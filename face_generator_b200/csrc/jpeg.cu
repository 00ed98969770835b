// Baseline JPEG decode straight into the device-resident dataset (fg_jpeg_info, fg_dataset_upload_jpeg) and the
// cache read-back (fg_dataset_download).
//
// Replaces dataset.lua:156-211 loadImagesFromDirs' image.load(path, nbChannels) for the .jpg training sets: the host
// only walks the markers; entropy decode, IDCT, upsampling and colour conversion run on the GPU, and the decoded
// planar uint8 lands in the cache rows.  Scope (T.81): SOF0 / SOF1, 8-bit, Huffman, one scan holding every
// component, 1 or 3 components, component 0 sampled 1x1, 2x1 or 2x2 with 1x1 chroma, DRI restarts; everything else
// is refused per file.  The arithmetic is k_jpeg.cuh; the output equals libjpeg-turbo's default decompression
// (islow IDCT, fancy upsampling) bit for bit.
//
// A call runs in chunks of at most kChunkImages files / kChunkBytes entropy bytes / kChunkCoefs coefficients (a
// larger single file is a chunk of its own):
//   host    parse every file of the chunk, split the scan at its RST markers, deduplicate the table sets and pack
//           table sets, descriptors and entropy bytes into one pinned buffer (two, alternating);
//   copy    one host-to-device copy on the dataset's copy stream, so chunk k+1 uploads while chunk k decodes;
//   decode  on the ctx stream: zero the coefficient scratch, jpeg_entropy_kernel (one thread per restart interval),
//           jpeg_idct_color_kernel (one CTA per band of MCU rows, usually the whole image), then the per-file
//           error flags back to pinned memory.
#include <algorithm>
#include <cstdarg>
#include <cstring>
#include <string>
#include <unordered_map>

#include "fg_internal.h"
#include "k_jpeg.cuh"
#include "k_jpeg_enc.cuh"

using jpg::BandDesc;
using jpg::ImageDesc;
using jpg::IntervalDesc;
using jpg::TableSet;

namespace {

constexpr int kChunkImages = 8192;
constexpr int64_t kChunkBytes = 32ll << 20;
constexpr int64_t kChunkCoefs = 32ll << 20;  // int16 coefficients (64 MB of scratch)
constexpr int kBandBudget = 64 * 1024;       // shared memory a band aims for; one MCU row may need more
constexpr int kEntropyThreads = 32, kIdctThreads = 128;

// ---- host marker walk ------------------------------------------------------------------------------------------
struct Header {
  int C = 0, H = 0, W = 0, hs = 1, vs = 1;
  int comp_id[3] = {0, 0, 0}, comp_q[3] = {0, 0, 0}, comp_dc[3] = {0, 0, 0}, comp_ac[3] = {0, 0, 0};
  int restart = 0;
  int64_t scan = 0;  // first entropy byte
  // table slots as defined when the scan starts: DQT in natural order, DHT counts + values
  uint16_t q[4][64];
  bool q_set[4] = {false, false, false, false};
  uint8_t hbits[2][2][17];  // [class: 0 DC, 1 AC][slot]
  uint8_t hvals[2][2][256];
  bool h_set[2][2] = {{false, false}, {false, false}};
};

enum { kOk = FG_OK, kBad = FG_ERR_INVALID, kUnsup = FG_ERR_UNSUPPORTED };
struct Parse {
  int rc = kOk;
  std::string why;
  int fail(int r, const char* fmt, ...) __attribute__((format(printf, 3, 4))) {
    char buf[256];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    rc = r;
    why = buf;
    return r;
  }
};

int u16be(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// Walks the markers from SOI to the first SOS and fills h.  Everything the decoder does not support is kUnsup with
// the reason; a malformed header is kBad.
int parse_header(const uint8_t* b, int64_t len, Header* h, Parse* ps) {
  if (len < 4 || b[0] != 0xFF || b[1] != 0xD8) return ps->fail(kBad, "not a JPEG file (no SOI marker)");
  int64_t p = 2;
  bool have_sof = false;
  bool adobe_rgb = false;
  while (true) {
    while (p < len && b[p] != 0xFF) ++p;  // tolerate junk between segments, as decoders do
    while (p < len && b[p] == 0xFF) ++p;  // fill bytes
    if (p >= len) return ps->fail(kBad, "truncated header (no SOS marker)");
    const int m = b[p++];
    if (m == 0xD8 || m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;  // standalone markers
    if (m == 0xD9) return ps->fail(kBad, "EOI before any scan");
    if (p + 2 > len) return ps->fail(kBad, "truncated header");
    const int L = u16be(b + p);
    if (L < 2 || p + L > len) return ps->fail(kBad, "truncated header (segment 0x%02X)", m);
    const uint8_t* s = b + p + 2;
    const int n = L - 2;
    if (m == 0xC0 || m == 0xC1) {
      if (have_sof) return ps->fail(kBad, "two frame headers");
      if (n < 6) return ps->fail(kBad, "short SOF");
      if (s[0] != 8) return ps->fail(kUnsup, "%d-bit samples (only 8-bit is supported)", s[0]);
      h->H = u16be(s + 1);
      h->W = u16be(s + 3);
      h->C = s[5];
      if (h->H == 0) return ps->fail(kUnsup, "height defined by a DNL marker");
      if (h->W == 0) return ps->fail(kBad, "zero width");
      if (h->C != 1 && h->C != 3) return ps->fail(kUnsup, "%d components (only 1 or 3 are supported)", h->C);
      if (n < 6 + 3 * h->C) return ps->fail(kBad, "short SOF");
      int hv[3][2];
      for (int c = 0; c < h->C; ++c) {
        h->comp_id[c] = s[6 + 3 * c];
        hv[c][0] = s[7 + 3 * c] >> 4;
        hv[c][1] = s[7 + 3 * c] & 15;
        h->comp_q[c] = s[8 + 3 * c];
        if (hv[c][0] < 1 || hv[c][0] > 4 || hv[c][1] < 1 || hv[c][1] > 4 || h->comp_q[c] > 3)
          return ps->fail(kBad, "bad component parameters");
      }
      if (h->C == 3) {
        const bool ok = (hv[1][0] == 1 && hv[1][1] == 1 && hv[2][0] == 1 && hv[2][1] == 1) &&
                        ((hv[0][0] == 1 && hv[0][1] == 1) || (hv[0][0] == 2 && hv[0][1] == 1) || (hv[0][0] == 2 && hv[0][1] == 2));
        if (!ok)
          return ps->fail(kUnsup, "sampling %dx%d,%dx%d,%dx%d (supported: 1x1, 2x1 or 2x2 luma with 1x1 chroma)", hv[0][0],
                          hv[0][1], hv[1][0], hv[1][1], hv[2][0], hv[2][1]);
        h->hs = hv[0][0];
        h->vs = hv[0][1];
        if (h->comp_id[0] == 'R' && h->comp_id[1] == 'G' && h->comp_id[2] == 'B')
          return ps->fail(kUnsup, "RGB-coded components (only YCbCr is supported)");
      }
      have_sof = true;
    } else if ((m >= 0xC2 && m <= 0xC3) || (m >= 0xC5 && m <= 0xC7) || (m >= 0xC9 && m <= 0xCB) || (m >= 0xCD && m <= 0xCF)) {
      const char* kind = m == 0xC2 || m == 0xC6 || m == 0xCA || m == 0xCE ? "progressive"
                         : m == 0xC3 || m == 0xC7 || m == 0xCB || m == 0xCF ? "lossless"
                                                                             : "hierarchical or arithmetic-coded";
      return ps->fail(kUnsup, "%s JPEG (SOF%d; only baseline / extended sequential Huffman is supported)", kind, m - 0xC0);
    } else if (m == 0xCC) {
      return ps->fail(kUnsup, "arithmetic coding (DAC marker)");
    } else if (m == 0xDC) {
      return ps->fail(kUnsup, "DNL marker");
    } else if (m == 0xC4) {
      int i = 0;
      while (i < n) {
        if (i + 17 > n) return ps->fail(kBad, "short DHT");
        const int tc = s[i] >> 4, th = s[i] & 15;
        if (tc > 1 || th > 3) return ps->fail(kBad, "bad DHT class / slot");
        if (th > 1) return ps->fail(kUnsup, "Huffman table slot %d (only slots 0 and 1 are supported)", th);
        int cnt = 0;
        h->hbits[tc][th][0] = 0;
        for (int l = 1; l <= 16; ++l) cnt += (h->hbits[tc][th][l] = s[i + l]);
        if (cnt > 256 || i + 17 + cnt > n) return ps->fail(kBad, "bad DHT");
        memset(h->hvals[tc][th], 0, 256);
        memcpy(h->hvals[tc][th], s + i + 17, cnt);
        h->h_set[tc][th] = true;
        i += 17 + cnt;
      }
    } else if (m == 0xDB) {
      int i = 0;
      while (i < n) {
        const int pq = s[i] >> 4, tq = s[i] & 15;
        if (pq > 1 || tq > 3 || i + 1 + 64 * (pq + 1) > n) return ps->fail(kBad, "bad DQT");
        for (int k = 0; k < 64; ++k)
          h->q[tq][jpg::natural_of(k)] = (uint16_t)(pq ? u16be(s + i + 1 + 2 * k) : s[i + 1 + k]);
        h->q_set[tq] = true;
        i += 1 + 64 * (pq + 1);
      }
    } else if (m == 0xDD) {
      if (n < 2) return ps->fail(kBad, "short DRI");
      h->restart = u16be(s);
    } else if (m == 0xEE) {  // Adobe APP14: transform 0 on 3 components means RGB-coded
      if (n >= 12 && !memcmp(s, "Adobe", 5) && s[11] == 0) adobe_rgb = true;
    } else if (m == 0xDA) {
      if (!have_sof) return ps->fail(kBad, "SOS before the frame header");
      if (n < 1) return ps->fail(kBad, "short SOS");
      const int ns = s[0];
      if (ns != h->C)
        return ps->fail(kUnsup, "a scan of %d of %d components (only one scan holding every component is supported)", ns, h->C);
      if (n < 1 + 2 * ns + 3) return ps->fail(kBad, "short SOS");
      for (int j = 0; j < ns; ++j) {
        if (s[1 + 2 * j] != h->comp_id[j]) return ps->fail(kUnsup, "scan components out of frame order");
        h->comp_dc[j] = s[2 + 2 * j] >> 4;
        h->comp_ac[j] = s[2 + 2 * j] & 15;
        if (h->comp_dc[j] > 1 || h->comp_ac[j] > 1)
          return ps->fail(kUnsup, "Huffman table slot > 1 (only slots 0 and 1 are supported)");
        if (!h->h_set[0][h->comp_dc[j]] || !h->h_set[1][h->comp_ac[j]]) return ps->fail(kBad, "scan uses an undefined Huffman table");
        if (!h->q_set[h->comp_q[j]]) return ps->fail(kBad, "component uses an undefined quantisation table");
      }
      const uint8_t* t = s + 1 + 2 * ns;
      if (t[0] != 0 || t[1] != 63 || t[2] != 0) return ps->fail(kUnsup, "spectral selection / successive approximation");
      if (adobe_rgb && h->C == 3) return ps->fail(kUnsup, "RGB-coded components (Adobe transform 0)");
      if (h->C == 1) h->hs = h->vs = 1;  // a 1-component scan is coded one block per MCU whatever its factors
      h->scan = p + L;
      return kOk;
    }
    p += L;
  }
}

void mcu_grid(const Header& h, int* mcux, int* mcuy) {
  *mcux = (h.W + 8 * h.hs - 1) / (8 * h.hs);
  *mcuy = (h.H + 8 * h.vs - 1) / (8 * h.vs);
}

// Finds the end of the scan and its restart intervals: iv[k] = byte range of interval k (RST markers excluded).
// The scan must be followed by EOI; RSTm markers must count 0..7 cyclically and match DRI.
int split_scan(const uint8_t* b, int64_t len, const Header& h, std::vector<std::pair<int64_t, int64_t>>* iv, Parse* ps) {
  iv->clear();
  int mcux, mcuy;
  mcu_grid(h, &mcux, &mcuy);
  const int64_t total = (int64_t)mcux * mcuy;
  const int64_t want = h.restart ? (total + h.restart - 1) / h.restart : 1;
  int64_t start = h.scan, p = h.scan;
  while (true) {
    const uint8_t* f = p < len ? (const uint8_t*)memchr(b + p, 0xFF, (size_t)(len - p)) : nullptr;
    if (!f) return ps->fail(kBad, "truncated entropy-coded data (no EOI marker)");
    int64_t q = f - b;
    int64_t r = q + 1;
    while (r < len && b[r] == 0xFF) ++r;  // fill bytes before a marker
    if (r >= len) return ps->fail(kBad, "truncated entropy-coded data (no EOI marker)");
    const int m = b[r];
    if (m == 0x00) {
      p = r + 1;
      continue;
    }
    iv->emplace_back(start, q);
    if (m >= 0xD0 && m <= 0xD7) {
      const int64_t k = (int64_t)iv->size() - 1;
      if (!h.restart || (int64_t)iv->size() >= want || m - 0xD0 != (int)(k & 7))
        return ps->fail(kBad, "corrupt entropy-coded data (unexpected RST%d marker)", m - 0xD0);
      start = p = r + 1;
      continue;
    }
    if (m != 0xD9) {
      if (m == 0xDA) return ps->fail(kUnsup, "more than one scan (only one scan holding every component is supported)");
      return ps->fail(kBad, "corrupt entropy-coded data (marker 0x%02X inside the scan)", m);
    }
    if ((int64_t)iv->size() != want)
      return ps->fail(kBad, "corrupt entropy-coded data (%lld restart intervals, DRI implies %lld)", (long long)iv->size(),
                      (long long)want);
    return kOk;
  }
}

// ---- chunk scratch ------------------------------------------------------------------------------------------------
// Two slots alternate: a pinned host buffer and a device buffer, each [sets][images][intervals][bands][bytes], and the
// per-file error flags the decode writes back.  Grows to the largest chunk seen; freed with the dataset.
struct Slot {
  uint8_t* host = nullptr;
  uint8_t* dev = nullptr;
  size_t cap = 0;
  int* err_host = nullptr;
  int* err_dev = nullptr;
  int err_cap = 0;
  cudaEvent_t uploaded = nullptr, done = nullptr;
  bool pending = false;  // launched, flags not checked yet
  int64_t first = 0;     // index (within the call) of the chunk's first file
  int n = 0;
};

}  // namespace

struct JpegScratch {
  Slot slot[2];
  int16_t* coef = nullptr;
  int64_t coef_cap = 0;
  cudaStream_t copy = nullptr;
};

void jpeg_scratch_free(JpegScratch* s) {
  if (!s) return;
  for (Slot& sl : s->slot) {
    cudaFreeHost(sl.host);
    cudaFree(sl.dev);
    cudaFreeHost(sl.err_host);
    cudaFree(sl.err_dev);
    if (sl.uploaded) cudaEventDestroy(sl.uploaded);
    if (sl.done) cudaEventDestroy(sl.done);
  }
  cudaFree(s->coef);
  if (s->copy) cudaStreamDestroy(s->copy);
  delete s;
}

namespace {

// ---- kernels ------------------------------------------------------------------------------------------------------
// One thread per restart interval.  When every interval of the CTA uses one table set, the set is staged in shared
// memory (a dataset from one encoder has one set); otherwise the threads read their sets from global memory.
__global__ void __launch_bounds__(kEntropyThreads) jpeg_entropy_kernel(const uint8_t* __restrict__ bytes, const TableSet* __restrict__ sets,
                                                                       const ImageDesc* __restrict__ imgs,
                                                                       const IntervalDesc* __restrict__ ivs, int n_iv,
                                                                       int16_t* __restrict__ coef, int* __restrict__ err) {
  __shared__ TableSet s_set;
  __shared__ int s_uniform;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int lo = blockIdx.x * blockDim.x, hi = min(n_iv, lo + (int)blockDim.x) - 1;
  const int set0 = imgs[ivs[lo].img].set;
  if (threadIdx.x == 0) s_uniform = imgs[ivs[hi].img].set == set0;  // intervals are ordered by table set
  __syncthreads();
  const bool uniform = s_uniform;
  if (uniform) {
    const int4* src = reinterpret_cast<const int4*>(sets + set0);
    int4* dst = reinterpret_cast<int4*>(&s_set);
    for (int k = threadIdx.x; k < (int)(sizeof(TableSet) / 16); k += blockDim.x) dst[k] = src[k];
  }
  __syncthreads();
  if (i >= n_iv) return;
  const IntervalDesc iv = ivs[i];
  const ImageDesc m = imgs[iv.img];
  const TableSet& ts = uniform ? s_set : sets[m.set];
  if (!jpg::decode_interval(bytes, iv, m, ts, coef + m.coef)) err[iv.img] = 1;
}

// One CTA per band of MCU rows: islow IDCT of every block the band needs into shared-memory component planes, then
// upsampling and colour conversion of the band's output rows, written planar into the cache row.
__global__ void __launch_bounds__(kIdctThreads) jpeg_idct_color_kernel(const TableSet* __restrict__ sets, const ImageDesc* __restrict__ imgs,
                                                                       const BandDesc* __restrict__ bands, const int16_t* __restrict__ coef,
                                                                       uint8_t* __restrict__ data) {
  extern __shared__ uint8_t planes[];
  const BandDesc bd = bands[blockIdx.x];
  const ImageDesc m = imgs[bd.img];
  const jpg::BandGeom g = jpg::band_geom(m, bd.mr0, bd.mr1);
  const TableSet& ts = sets[m.set];
  const int nb = jpg::band_blocks(m, g);
  for (int k = threadIdx.x; k < nb; k += blockDim.x) {
    int comp, so, stride;
    int64_t co;
    jpg::band_block(m, g, k, &comp, &co, &so, &stride);
    jpg::idct_islow(coef + m.coef + co, ts.q[comp], planes + so, stride);
  }
  __syncthreads();
  const int y1 = min(g.y1, m.H), W = m.W;
  const int64_t plane = (int64_t)m.H * W;
  uint8_t* out = data + m.out;
  for (int i = threadIdx.x; i < (y1 - g.y0) * W; i += blockDim.x) {
    const int y = g.y0 + i / W, x = i - (i / W) * W;
    uint8_t rgb[3];
    jpg::band_pixel(m, g, planes, y, x, rgb);
    const int64_t o = (int64_t)y * W + x;
    out[o] = rgb[0];
    if (m.Cs == 3) {
      out[plane + o] = rgb[1];
      out[2 * plane + o] = rgb[2];
    }
  }
}

// ---- host packing --------------------------------------------------------------------------------------------------
struct Chunk {
  std::vector<TableSet> sets;
  std::unordered_map<std::string, int> set_of;
  std::vector<ImageDesc> imgs;
  std::vector<IntervalDesc> ivs;
  std::vector<BandDesc> bands;
  std::vector<std::pair<const uint8_t*, int64_t>> spans;  // entropy bytes to copy, in order
  int64_t n_bytes = 0, n_coefs = 0;
  int smem = 0;
  void clear() {
    sets.clear();
    set_of.clear();
    imgs.clear();
    ivs.clear();
    bands.clear();
    spans.clear();
    n_bytes = n_coefs = 0;
    smem = 0;
  }
};

// the table-set key: for each component its quantisation table and both Huffman tables, as bytes
std::string set_key(const Header& h) {
  std::string k;
  k.reserve(h.C * (128 + 2 * 273));
  for (int c = 0; c < h.C; ++c) {
    k.append((const char*)h.q[h.comp_q[c]], 128);
    for (int cls = 0; cls < 2; ++cls) {
      const int slot = cls ? h.comp_ac[c] : h.comp_dc[c];
      k.push_back((char)(cls * 2 + slot));
      k.append((const char*)h.hbits[cls][slot], 17);
      k.append((const char*)h.hvals[cls][slot], 256);
    }
  }
  return k;
}

int add_set(Chunk& ch, const Header& h, Parse* ps) {
  std::string key = set_key(h);
  auto it = ch.set_of.find(key);
  if (it != ch.set_of.end()) return it->second;
  TableSet ts;
  memset(&ts, 0, sizeof(ts));
  for (int cls = 0; cls < 2; ++cls)
    for (int slot = 0; slot < 2; ++slot)
      if (h.h_set[cls][slot] && !jpg::build_huff(h.hbits[cls][slot], h.hvals[cls][slot], &ts.tab[cls * 2 + slot])) {
        ps->fail(kBad, "invalid Huffman table");
        return -1;
      }
  for (int c = 0; c < h.C; ++c) {
    memcpy(ts.q[c], h.q[h.comp_q[c]], 128);
    ts.dc[c] = (uint8_t)h.comp_dc[c];
    ts.ac[c] = (uint8_t)(2 + h.comp_ac[c]);
  }
  const int id = (int)ch.sets.size();
  ch.sets.push_back(ts);
  ch.set_of.emplace(std::move(key), id);
  return id;
}

size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

int grow(Slot& s, size_t bytes, int n) {
  if (bytes > s.cap) {
    cudaFreeHost(s.host);
    cudaFree(s.dev);
    s.host = nullptr;
    s.dev = nullptr;
    s.cap = 0;
    const size_t cap = std::max(bytes, s.cap + s.cap / 2);
    FG_CUDA(cudaHostAlloc((void**)&s.host, cap, cudaHostAllocDefault));
    FG_CUDA(cudaMalloc((void**)&s.dev, cap));
    s.cap = cap;
  }
  if (n > s.err_cap) {
    cudaFreeHost(s.err_host);
    cudaFree(s.err_dev);
    s.err_host = nullptr;
    s.err_dev = nullptr;
    s.err_cap = 0;
    FG_CUDA(cudaHostAlloc((void**)&s.err_host, sizeof(int) * n, cudaHostAllocDefault));
    FG_CUDA(cudaMalloc((void**)&s.err_dev, sizeof(int) * n));
    s.err_cap = n;
  }
  if (!s.uploaded) FG_CUDA(cudaEventCreateWithFlags(&s.uploaded, cudaEventDisableTiming));
  if (!s.done) FG_CUDA(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
  return FG_OK;
}

// waits for a launched chunk and returns the index (within the call) of its first failing file, or -1
int64_t finish(Slot& s, int* rc) {
  if (!s.pending) return -1;
  s.pending = false;
  const cudaError_t e = cudaEventSynchronize(s.done);
  if (e != cudaSuccess) {
    fg_set_error("fg_dataset_upload_jpeg: %s", cudaGetErrorString(e));
    *rc = FG_ERR_CUDA;
    return -1;
  }
  for (int i = 0; i < s.n; ++i)
    if (s.err_host[i]) return s.first + i;
  return -1;
}

}  // namespace

int jpeg_idct_band_rows(const ImageDesc& m, int* smem) {
  int rows = 1;
  while (rows < m.mcuy && jpg::band_bytes(m, 0, rows + 1) <= kBandBudget) ++rows;
  *smem = 0;
  for (int r0 = 0; r0 < m.mcuy; r0 += rows) *smem = std::max(*smem, jpg::band_bytes(m, r0, std::min(m.mcuy, r0 + rows)));
  return rows;
}

int jpeg_idct_launch(fg_ctx* c, const TableSet* sets, const ImageDesc* imgs, const BandDesc* bands, int n_bands, int smem,
                     const int16_t* coef, uint8_t* data) {
  if (smem > 48 * 1024) FG_CUDA(cudaFuncSetAttribute(jpeg_idct_color_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  jpeg_idct_color_kernel<<<n_bands, kIdctThreads, smem, c->stream>>>(sets, imgs, bands, coef, data);
  LAUNCH_CHECK(c);
  return FG_OK;
}

extern "C" {

int fg_jpeg_info(const uint8_t* bytes, int64_t len, int* C, int* H, int* W) {
  if (!bytes || len < 0) {
    fg_set_error("fg_jpeg_info: null argument");
    return FG_ERR_INVALID;
  }
  Header h;
  Parse ps;
  if (parse_header(bytes, len, &h, &ps) != kOk) {
    fg_set_error("fg_jpeg_info: %s", ps.why.c_str());
    return ps.rc;
  }
  if (C) *C = h.C;
  if (H) *H = h.H;
  if (W) *W = h.W;
  return FG_OK;
}

int fg_dataset_upload_jpeg(fg_dataset* d, int64_t first, int64_t count, const uint8_t* bytes, const int64_t* offsets,
                           int64_t* failed_out) {
  if (failed_out) *failed_out = -1;
  if (!d || !d->c) {
    fg_set_error("null fg_dataset");
    return FG_ERR_INVALID;
  }
  FG_REQUIRE(bytes && offsets && first >= 0 && count >= 1 && first + count <= d->N,
             "fg_dataset_upload_jpeg: range [%lld, %lld) outside [0, %lld)", (long long)first, (long long)(first + count),
             (long long)d->N);
  for (int64_t i = 0; i < count; ++i)
    FG_REQUIRE(offsets[i + 1] >= offsets[i] && offsets[i] >= 0, "fg_dataset_upload_jpeg: offsets[%lld..%lld] decrease",
               (long long)i, (long long)i + 1);
  auto refuse = [&](int64_t i, int rc, const std::string& why) {
    if (failed_out) *failed_out = i;
    fg_set_error("fg_dataset_upload_jpeg: file %lld: %s", (long long)i, why.c_str());
    return rc;
  };
  // every header first, before anything is launched
  for (int64_t i = 0; i < count; ++i) {
    Header h;
    Parse ps;
    if (parse_header(bytes + offsets[i], offsets[i + 1] - offsets[i], &h, &ps) != kOk) return refuse(i, ps.rc, ps.why);
    if (h.H != d->Hs || h.W != d->Ws) {
      char buf[128];
      snprintf(buf, sizeof(buf), "size %dx%d, the cache holds %dx%d", h.W, h.H, d->Ws, d->Hs);
      return refuse(i, FG_ERR_INVALID, buf);
    }
    if (h.C == 3 && d->Cs == 1) return refuse(i, FG_ERR_INVALID, "a 3-component file cannot go into a 1-channel cache");
  }
  fg_ctx* c = d->c;
  FG_CUDA(cudaSetDevice(c->device));
  if (!d->jpeg) d->jpeg = new JpegScratch();
  JpegScratch& js = *d->jpeg;
  if (!js.copy) FG_CUDA(cudaStreamCreateWithFlags(&js.copy, cudaStreamNonBlocking));
  const int64_t per = (int64_t)d->Cs * d->Hs * d->Ws;

  Chunk ch;
  std::vector<std::pair<int64_t, int64_t>> iv;
  int rc = FG_OK;
  int64_t bad = -1;
  std::string bad_why;
  int k = 0;  // chunk counter, selects the slot
  int64_t i = 0;
  while (i < count && bad < 0 && rc == FG_OK) {
    // ---- parse and pack one chunk; a file the host finds corrupt ends the chunk and the call, after the files
    // before it have been decoded (one of them may fail on the device, with a lower index)
    ch.clear();
    const int64_t chunk_first = i;
    for (; i < count && (int64_t)ch.imgs.size() < kChunkImages; ++i) {
      const uint8_t* f = bytes + offsets[i];
      const int64_t len = offsets[i + 1] - offsets[i];
      Header h;
      Parse ps;
      parse_header(f, len, &h, &ps);  // checked above
      if (split_scan(f, len, h, &iv, &ps) != kOk) {
        bad = i;
        bad_why = ps.why;
        break;
      }
      int mcux, mcuy;
      mcu_grid(h, &mcux, &mcuy);
      const int64_t ncoef = jpg::image_coefs(h.C, h.hs, h.vs, mcux, mcuy);
      int64_t nbytes = 0;
      for (auto& r : iv) nbytes += r.second - r.first;
      if (!ch.imgs.empty() && (ch.n_coefs + ncoef > kChunkCoefs || ch.n_bytes + nbytes > kChunkBytes)) break;
      const int set = add_set(ch, h, &ps);
      if (set < 0) {
        bad = i;
        bad_why = ps.why;
        break;
      }
      ImageDesc m;
      m.coef = ch.n_coefs;
      m.out = (first + i) * per;
      m.set = set;
      m.C = h.C;
      m.H = h.H;
      m.W = h.W;
      m.Cs = d->Cs;
      m.hs = h.hs;
      m.vs = h.vs;
      m.mcux = mcux;
      m.mcuy = mcuy;
      const int img = (int)ch.imgs.size();
      ch.imgs.push_back(m);
      const int64_t total = (int64_t)mcux * mcuy;
      const int64_t ri = h.restart ? h.restart : total;
      for (size_t r = 0; r < iv.size(); ++r) {
        IntervalDesc d_iv;
        d_iv.off = ch.n_bytes;
        d_iv.len = (int)(iv[r].second - iv[r].first);
        d_iv.img = img;
        d_iv.mcu0 = (int)(r * ri);
        d_iv.n = (int)std::min<int64_t>(ri, total - (int64_t)r * ri);
        ch.ivs.push_back(d_iv);
        ch.spans.emplace_back(f + iv[r].first, d_iv.len);
        ch.n_bytes += d_iv.len;
      }
      // bands: as many MCU rows as fit the budget, at least one
      int rows = 1;
      while (rows < mcuy && jpg::band_bytes(m, 0, rows + 1) <= kBandBudget) ++rows;
      for (int r0 = 0; r0 < mcuy; r0 += rows) {
        const int r1 = std::min(mcuy, r0 + rows);
        ch.bands.push_back({img, r0, r1});
        ch.smem = std::max(ch.smem, jpg::band_bytes(m, r0, r1));
      }
      ch.n_coefs += ncoef;
    }
    if (ch.imgs.empty()) break;
    // intervals ordered by table set, so that a CTA of the entropy kernel usually shares one set
    if (ch.sets.size() > 1)
      std::stable_sort(ch.ivs.begin(), ch.ivs.end(),
                       [&](const IntervalDesc& a, const IntervalDesc& b) { return ch.imgs[a.img].set < ch.imgs[b.img].set; });
    Slot& s = js.slot[k & 1];
    // the slot's previous chunk must be decoded before its buffers are rewritten
    const int64_t prev_bad = finish(s, &rc);
    if (rc != FG_OK) break;
    if (prev_bad >= 0) {  // an earlier chunk failed: nothing after it needs decoding
      bad = prev_bad;
      bad_why = "corrupt or truncated entropy-coded data";
      break;
    }
    const size_t o_img = align16(sizeof(TableSet) * ch.sets.size());
    const size_t o_iv = o_img + align16(sizeof(ImageDesc) * ch.imgs.size());
    const size_t o_band = o_iv + align16(sizeof(IntervalDesc) * ch.ivs.size());
    const size_t o_bytes = o_band + align16(sizeof(BandDesc) * ch.bands.size());
    const size_t total = o_bytes + (size_t)ch.n_bytes + 16;
    if ((rc = grow(s, total, (int)ch.imgs.size())) != FG_OK) break;
    memcpy(s.host, ch.sets.data(), sizeof(TableSet) * ch.sets.size());
    memcpy(s.host + o_img, ch.imgs.data(), sizeof(ImageDesc) * ch.imgs.size());
    memcpy(s.host + o_iv, ch.ivs.data(), sizeof(IntervalDesc) * ch.ivs.size());
    memcpy(s.host + o_band, ch.bands.data(), sizeof(BandDesc) * ch.bands.size());
    uint8_t* dst = s.host + o_bytes;
    for (auto& sp : ch.spans) {
      memcpy(dst, sp.first, (size_t)sp.second);
      dst += sp.second;
    }
    if (ch.n_coefs > js.coef_cap) {
      FG_CUDA(cudaStreamSynchronize(c->stream));
      cudaFree(js.coef);
      js.coef = nullptr;
      js.coef_cap = 0;
      FG_CUDA(cudaMalloc((void**)&js.coef, sizeof(int16_t) * (size_t)ch.n_coefs));
      js.coef_cap = ch.n_coefs;
    }
    // ---- upload on the copy stream, decode on the ctx stream once it has landed
    const cudaError_t e = cudaMemcpyAsync(s.dev, s.host, total, cudaMemcpyHostToDevice, js.copy);
    if (e != cudaSuccess) {
      fg_set_error("fg_dataset_upload_jpeg: upload: %s", cudaGetErrorString(e));
      rc = FG_ERR_CUDA;
      break;
    }
    FG_CUDA(cudaEventRecord(s.uploaded, js.copy));
    FG_CUDA(cudaStreamWaitEvent(c->stream, s.uploaded, 0));
    const int n_img = (int)ch.imgs.size(), n_iv = (int)ch.ivs.size();
    const TableSet* sets = reinterpret_cast<const TableSet*>(s.dev);
    const ImageDesc* imgs = reinterpret_cast<const ImageDesc*>(s.dev + o_img);
    FG_CUDA(cudaMemsetAsync(js.coef, 0, sizeof(int16_t) * (size_t)ch.n_coefs, c->stream));
    FG_CUDA(cudaMemsetAsync(s.err_dev, 0, sizeof(int) * n_img, c->stream));
    jpeg_entropy_kernel<<<(n_iv + kEntropyThreads - 1) / kEntropyThreads, kEntropyThreads, 0, c->stream>>>(
        s.dev + o_bytes, sets, imgs, reinterpret_cast<const IntervalDesc*>(s.dev + o_iv), n_iv, js.coef, s.err_dev);
    LAUNCH_CHECK(c);
    if (ch.smem > 48 * 1024)
      FG_CUDA(cudaFuncSetAttribute(jpeg_idct_color_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ch.smem));
    jpeg_idct_color_kernel<<<(int)ch.bands.size(), kIdctThreads, ch.smem, c->stream>>>(
        sets, imgs, reinterpret_cast<const BandDesc*>(s.dev + o_band), js.coef, d->data);
    LAUNCH_CHECK(c);
    FG_CUDA(cudaMemcpyAsync(s.err_host, s.err_dev, sizeof(int) * n_img, cudaMemcpyDeviceToHost, c->stream));
    FG_CUDA(cudaEventRecord(s.done, c->stream));
    s.pending = true;
    s.first = chunk_first;
    s.n = n_img;
    ++k;
  }
  // drain both slots in launch order (the older one first), so that the lowest failing index is reported
  for (int j = 0; j < 2; ++j) {
    Slot& s = js.slot[(k + j) & 1];
    int r2 = FG_OK;
    const int64_t b = finish(s, &r2);
    if (rc == FG_OK) rc = r2;
    if (b >= 0 && (bad < 0 || b < bad)) {
      bad = b;
      bad_why = "corrupt or truncated entropy-coded data";
    }
  }
  if (rc != FG_OK) return rc;
  if (bad >= 0) return refuse(bad, FG_ERR_INVALID, bad_why);
  return FG_OK;
}

int fg_dataset_download(fg_dataset* d, int64_t first, int64_t count, uint8_t* out) {
  if (!d || !d->c) {
    fg_set_error("null fg_dataset");
    return FG_ERR_INVALID;
  }
  FG_REQUIRE(out && first >= 0 && count >= 1 && first + count <= d->N, "fg_dataset_download: range [%lld, %lld) outside [0, %lld)",
             (long long)first, (long long)(first + count), (long long)d->N);
  FG_CUDA(cudaSetDevice(d->c->device));
  const size_t per = (size_t)d->Cs * d->Hs * d->Ws;
  FG_CUDA(cudaMemcpyAsync(out, d->data + (size_t)first * per, (size_t)count * per, cudaMemcpyDefault, d->c->stream));
  FG_CUDA(cudaStreamSynchronize(d->c->stream));
  return FG_OK;
}

}  // extern "C"
