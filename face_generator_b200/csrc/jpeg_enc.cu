// Baseline JPEG encode of the device-resident dataset (fg_dataset_encode_jpeg), of caller images (fg_jpeg_encode), and
// the dataset's round trip in place (fg_dataset_jpeg_roundtrip).
//
// Replaces dataset/generate_dataset.py's last step, misc.imsave(path, row), and image.save(path, grid) of sample.lua's
// sheets: Pillow's Image.save at its defaults (baseline JFIF 1.01, quality 75, YCbCr 4:2:0, standard Huffman tables,
// islow DCT, no restart markers), which every file train.lua, train_c2f.lua and sample.lua read or write went through.
// The arithmetic is k_jpeg_enc.cuh; the files equal Pillow's byte for byte (tests/jpeg_enc_ref.py restates the rules,
// tests/test_gpu_jpeg_encode.py and tests/test_gpu_sample_sheets.py hold the kernels to them).  A call runs in chunks
// of at most kChunkBlocks 8x8 blocks (at least one image), on the ctx stream:
//   jpeg_fdct_kernel   one CTA per band of MCU rows (usually the whole image): colour conversion into shared memory,
//                      then one thread per block: edge expansion, 2x2 downsampling, forward DCT, quantisation, written
//                      in the decoder's coefficient layout; then the dummy blocks
// then one of two entropy coders, chosen by the blocks per file (kMultiMinBlocks); both write the same bytes:
//   one CTA per file (small files, many per chunk)
//     jpeg_huff_kernel   the bit length of every block (its DC predictor is already in the scratch), a scan to bit
//                        offsets, every block's codes packed into the file's word buffer, the padding 1-bits, and the
//                        length after byte stuffing
//     jpeg_stuff_kernel  header, stuffed entropy bytes (0x00 after each 0xFF) and EOI at the file's offset in the
//                        chunk's output, which goes to the host in one copy
//   many CTAs per file (large files, such as sample sheets: one file per chunk)
//     jpeg_blen_kernel    kTileBlocks blocks per CTA: bit lengths, their scan within the tile, the tile's sum
//     jpeg_scan_kernel    one CTA: exclusive scan of the tile sums -> tile bit offsets and the file's bit count
//     jpeg_zero_kernel    zeroes the words the codes occupy
//     jpeg_pack_kernel    kTileBlocks blocks per CTA: codes OR-ed into the words at their offsets, the padding 1-bits
//     jpeg_ffcount_kernel kStuffSegs CTAs, one contiguous segment of words each: the 0xFF bytes of the segment
//     jpeg_scan_kernel    the segments' 0xFF counts -> their shifts, and the stuffed byte count
//     jpeg_scatter_kernel kStuffSegs CTAs: header, each segment's stuffed bytes at its shift, EOI
// The sizes are known only once a chunk is coded, and nothing may be written to the caller's buffer unless every file
// fits, so the encode codes the images twice: once for the sizes (no stuffing, no copy), once to write (a call of one
// chunk keeps its first pass).  The round trip runs jpeg_fdct_kernel and then the decoder's jpeg_idct_color_kernel on
// the same coefficients: decode(encode(row)) without the entropy coding, which is lossless.
#include <algorithm>
#include <cstring>
#include <vector>

#include "fg_internal.h"
#include "k_jpeg_enc.cuh"

using jpg::EncGeom;

namespace {

constexpr int64_t kChunkBlocks = 1 << 18;  // 32 MB of coefficients, 53 MB of worst-case code words
constexpr int kBandBudget = 64 * 1024;     // shared memory a band of the forward kernel aims for; one MCU row may need more
constexpr int kFdctThreads = 128, kHuffThreads = 128, kStuffThreads = 128;
constexpr int kBlockWords = (jpg::kMaxBlockBits + 31) / 32;  // code words one block may need
// Files of at least kMultiMinBlocks blocks are entropy-coded by many CTAs: one CTA of kHuffThreads would loop over
// 16 or more blocks per thread, and a chunk holds at most a few dozen such files, so most SMs would idle (a 1024x1024
// colour sheet has 24 576 blocks, 192 per thread).  Below it, files are small and a chunk holds many of them.
constexpr int kMultiMinBlocks = 2048;
constexpr int kTileBlocks = 128;  // blocks per CTA of jpeg_blen_kernel / jpeg_pack_kernel (one per thread)
constexpr int kScanThreads = 1024;
constexpr int kStuffSegs = 264;  // CTAs of jpeg_ffcount_kernel / jpeg_scatter_kernel: two per SM

// ---- kernels ------------------------------------------------------------------------------------------------------
// exclusive scan of v over the CTA (blockDim.x a multiple of 32, at most 1024); *total = the sum
__device__ int block_excl_scan(int v, int* total) {
  __shared__ int warp_sum[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sum[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int s = lane < nw ? warp_sum[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < nw) warp_sum[lane] = s;
  }
  __syncthreads();
  const int excl = x - v + (wid ? warp_sum[wid - 1] : 0);
  *total = warp_sum[nw - 1];
  __syncthreads();  // warp_sum is reused by the next call
  return excl;
}

// One CTA per band of MCU rows [mr0, mr1) of one row of the cache.  rows: the chunk's first cache row; coef: the
// chunk's scratch, g.nblk * 64 coefficients per row.
__global__ void __launch_bounds__(kFdctThreads) jpeg_fdct_kernel(const __grid_constant__ EncGeom g, const uint8_t* __restrict__ rows,
                                                                 int16_t* __restrict__ coef) {
  extern __shared__ uint8_t sp[];  // [Cs][ny][W]: Y (Cb, Cr) of the band's image rows [y0, y0 + ny)
  const int img = blockIdx.x / g.bands, band = blockIdx.x - img * g.bands;
  const int mr0 = band * g.rows, mr1 = min(g.mcuy, mr0 + g.rows);
  const int W = g.W, y0 = mr0 * 8 * g.vs, ny = min(mr1 * 8 * g.vs, g.H) - y0;
  const int64_t plane = (int64_t)g.H * W;
  const uint8_t* src = rows + (int64_t)img * g.Cs * plane + (int64_t)y0 * W;
  const int pn = ny * W;
  for (int i = threadIdx.x; i < pn; i += blockDim.x) {
    if (g.Cs == 3) jpg::rgb_to_ycc(src[i], src[plane + i], src[2 * plane + i], sp + i, sp + pn + i, sp + 2 * pn + i);
    else sp[i] = src[i];
  }
  __syncthreads();
  const int bw0 = g.mcux * g.hs, nl = (mr1 - mr0) * g.vs * bw0, nc = (mr1 - mr0) * g.mcux, nb = nl + (g.Cs - 1) * nc;
  const int64_t n0 = (int64_t)bw0 * g.mcuy * g.vs * 64, n1 = (int64_t)g.mcux * g.mcuy * 64;
  int16_t* out = coef + (int64_t)img * g.nblk * 64;
  const int hc = (g.H + 1) / 2;  // downsampled chroma rows
  for (int k = threadIdx.x; k < nb; k += blockDim.x) {
    int comp, by, bx;
    if (k < nl) {
      comp = 0;
      by = mr0 * g.vs + k / bw0;
      bx = k - (k / bw0) * bw0;
      if (bx >= g.bwr || by >= g.bhr) continue;  // a dummy block: below
    } else {
      const int k2 = k - nl;
      comp = 1 + k2 / nc;
      const int k3 = k2 - (comp - 1) * nc;
      by = mr0 + k3 / g.mcux;
      bx = k3 - (k3 / g.mcux) * g.mcux;
    }
    int32_t d[64];
    if (comp == 0) {
      for (int r = 0; r < 8; ++r) {
        const uint8_t* row = sp + (min(by * 8 + r, g.H - 1) - y0) * W;
        for (int c = 0; c < 8; ++c) d[r * 8 + c] = row[min(bx * 8 + c, W - 1)] - 128;
      }
    } else {
      const uint8_t* pl = sp + comp * pn;
      for (int r = 0; r < 8; ++r) {
        const int rr = min(by * 8 + r, hc - 1), ya = 2 * rr, yb = min(2 * rr + 1, g.H - 1);
        const uint8_t *ra = pl + (ya - y0) * W, *rb = pl + (yb - y0) * W;
        for (int c = 0; c < 8; ++c) {
          const int cx = bx * 8 + c, xa = min(2 * cx, W - 1), xb = min(2 * cx + 1, W - 1);
          d[r * 8 + c] = ((ra[xa] + ra[xb] + rb[xa] + rb[xb] + 1 + (c & 1)) >> 2) - 128;
        }
      }
    }
    jpg::fdct_islow(d);
    const uint16_t* q = g.q[comp ? 1 : 0];
    uint32_t packed[32];
    for (int i = 0; i < 32; ++i)
      packed[i] = (uint32_t)(uint16_t)jpg::quantize(d[2 * i], q[2 * i]) | ((uint32_t)(uint16_t)jpg::quantize(d[2 * i + 1], q[2 * i + 1]) << 16);
    int16_t* blk = out + (comp == 0 ? ((int64_t)by * bw0 + bx) * 64 : n0 + (comp - 1) * n1 + ((int64_t)by * g.mcux + bx) * 64);
    int4* dst = reinterpret_cast<int4*>(blk);
    for (int i = 0; i < 8; ++i) dst[i] = make_int4(packed[4 * i], packed[4 * i + 1], packed[4 * i + 2], packed[4 * i + 3]);
  }
  if (g.bwr == bw0 && g.bhr == g.mcuy * g.vs) return;  // no dummy blocks (uniform over the grid)
  __syncthreads();  // the real blocks' DCs are in global memory, visible to the CTA
  for (int k = threadIdx.x; k < nl; k += blockDim.x) {
    const int by = mr0 * g.vs + k / bw0, bx = k - (k / bw0) * bw0;
    if (bx < g.bwr && by < g.bhr) continue;
    // jccoefct.c: a right-edge dummy takes its left neighbour's DC, a bottom one the DC of the MCU's last block of
    // the row above, which is itself a real block or a right-edge dummy carrying its left neighbour's
    int sy = by, sx = bx - 1;
    if (by >= g.bhr) {
      sy = by - 1;
      sx = (bx / g.hs) * g.hs + g.hs - 1;
      if (sx >= g.bwr) sx = g.bwr - 1;
    }
    const int16_t dc = out[((int64_t)sy * bw0 + sx) * 64];
    int4* dst = reinterpret_cast<int4*>(out + ((int64_t)by * bw0 + bx) * 64);
    dst[0] = make_int4((int)(uint16_t)dc, 0, 0, 0);
    for (int i = 1; i < 8; ++i) dst[i] = make_int4(0, 0, 0, 0);
  }
}

// Packs bits MSB-first into 32-bit words starting at a bit offset.  The first and the last word may be shared with
// the neighbouring blocks' codes and are OR-ed atomically into zeroed words; the words in between are the block's own.
struct WordSink {
  uint32_t* w;
  uint64_t acc = 0;
  int n;
  bool first = true;
  __device__ WordSink(uint32_t* base, int bit) : w(base + (bit >> 5)), n(bit & 31) {}
  __device__ void put(uint32_t bits, int k) {
    acc = (acc << k) | bits;
    n += k;
    if (n >= 32) {
      n -= 32;
      const uint32_t v = (uint32_t)(acc >> n);
      if (first) atomicOr(w, v);
      else *w = v;
      first = false;
      ++w;
      acc &= (1ull << n) - 1;
    }
  }
  __device__ void flush() {
    if (n) atomicOr(w, (uint32_t)(acc << (32 - n)));
  }
};

// One CTA per row of the chunk: words[img] gets the row's entropy-coded bits (before stuffing, padded with 1-bits to a
// whole byte), nbits[img] their count and slen[img] the byte count after stuffing.
__global__ void __launch_bounds__(kHuffThreads) jpeg_huff_kernel(const __grid_constant__ EncGeom g, const int16_t* __restrict__ coef,
                                                                 const uint32_t* __restrict__ codes, uint32_t* __restrict__ words,
                                                                 int* __restrict__ boff, int* __restrict__ nbits,
                                                                 int* __restrict__ slen) {
  __shared__ uint32_t s_codes[4][256];
  __shared__ int s_ff;
  for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) (&s_codes[0][0])[i] = codes[i];
  if (threadIdx.x == 0) s_ff = 0;
  __syncthreads();
  const int img = blockIdx.x;
  const int16_t* cf = coef + (int64_t)img * g.nblk * 64;
  uint32_t* wd = words + (int64_t)img * g.nblk * kBlockWords;
  int* bo = boff + (int64_t)img * g.nblk;
  // bit offset of every block in scan order
  int carry = 0;
  for (int t = 0; t < g.nblk; t += blockDim.x) {
    const int s = t + threadIdx.x;
    int len = 0;
    if (s < g.nblk) {
      int64_t off, prev;
      const int comp = jpg::scan_block(g, s, &off, &prev);
      jpg::BitCount bc;
      jpg::huff_block(cf + off, prev < 0 ? 0 : cf[prev], s_codes[comp ? 2 : 0], s_codes[comp ? 3 : 1], bc);
      len = bc.n;
    }
    int total;
    const int ex = block_excl_scan(len, &total);
    if (s < g.nblk) bo[s] = carry + ex;
    carry += total;
  }
  const int T = carry, nw = (T + 31) >> 5;
  for (int i = threadIdx.x; i < nw; i += blockDim.x) wd[i] = 0;
  __syncthreads();
  for (int s = threadIdx.x; s < g.nblk; s += blockDim.x) {
    int64_t off, prev;
    const int comp = jpg::scan_block(g, s, &off, &prev);
    WordSink ws(wd, bo[s]);
    jpg::huff_block(cf + off, prev < 0 ? 0 : cf[prev], s_codes[comp ? 2 : 0], s_codes[comp ? 3 : 1], ws);
    ws.flush();
  }
  __syncthreads();
  const int nbytes = (T + 7) >> 3, pad = nbytes * 8 - T;
  if (threadIdx.x == 0 && pad) atomicOr(wd + (T >> 5), ((1u << pad) - 1) << (32 - (T & 31) - pad));  // 1-bits
  __syncthreads();
  int ff = 0;
  for (int i = threadIdx.x; i < nw; i += blockDim.x) {
    const uint32_t v = wd[i];
    for (int j = 0; j < 4 && 4 * i + j < nbytes; ++j) ff += ((v >> (24 - 8 * j)) & 0xff) == 0xff;
  }
  if (ff) atomicAdd(&s_ff, ff);
  __syncthreads();
  if (threadIdx.x == 0) {
    nbits[img] = T;
    slen[img] = nbytes + s_ff;
  }
}

// One CTA per row of the chunk: the file at out + off[img]: header, the stuffed entropy-coded bytes, EOI.
__global__ void __launch_bounds__(kStuffThreads) jpeg_stuff_kernel(int nblk, const uint32_t* __restrict__ words,
                                                                   const int* __restrict__ nbits, const uint8_t* __restrict__ hdr,
                                                                   int hdr_len, const int64_t* __restrict__ off,
                                                                   uint8_t* __restrict__ out) {
  const int img = blockIdx.x;
  const uint32_t* wd = words + (int64_t)img * nblk * kBlockWords;
  uint8_t* dst = out + off[img];
  for (int i = threadIdx.x; i < hdr_len; i += blockDim.x) dst[i] = hdr[i];
  dst += hdr_len;
  const int nbytes = (nbits[img] + 7) >> 3, nw = (nbytes + 3) >> 2;
  int carry = 0;
  for (int t = 0; t < nw; t += blockDim.x) {
    const int i = t + threadIdx.x;
    uint32_t v = 0;
    int nb = 0, ff = 0;
    if (i < nw) {
      v = wd[i];
      nb = min(4, nbytes - 4 * i);
      for (int j = 0; j < nb; ++j) ff += ((v >> (24 - 8 * j)) & 0xff) == 0xff;
    }
    int total;
    int p = 4 * i + carry + block_excl_scan(ff, &total);
    for (int j = 0; j < nb; ++j) {
      const uint8_t b = (uint8_t)(v >> (24 - 8 * j));
      dst[p++] = b;
      if (b == 0xff) dst[p++] = 0;
    }
    carry += total;
  }
  if (threadIdx.x == 0) {
    dst[nbytes + carry] = 0xff;
    dst[nbytes + carry + 1] = 0xd9;
  }
}

// ---- the multi-CTA coder of one file (the chunk's only image) ---------------------------------------------------------
// kTileBlocks blocks per CTA: boff[s] = the bit offset of block s within its tile, tsum[tile] = the tile's bits
__global__ void __launch_bounds__(kTileBlocks) jpeg_blen_kernel(const __grid_constant__ EncGeom g, const int16_t* __restrict__ coef,
                                                                const uint32_t* __restrict__ codes, int* __restrict__ boff,
                                                                int* __restrict__ tsum) {
  __shared__ uint32_t s_codes[4][256];
  for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) (&s_codes[0][0])[i] = codes[i];
  __syncthreads();
  const int s = blockIdx.x * kTileBlocks + threadIdx.x;
  int len = 0;
  if (s < g.nblk) {
    int64_t off, prev;
    const int comp = jpg::scan_block(g, s, &off, &prev);
    jpg::BitCount bc;
    jpg::huff_block(coef + off, prev < 0 ? 0 : coef[prev], s_codes[comp ? 2 : 0], s_codes[comp ? 3 : 1], bc);
    len = bc.n;
  }
  int total;
  const int ex = block_excl_scan(len, &total);
  if (s < g.nblk) boff[s] = ex;
  if (threadIdx.x == 0) tsum[blockIdx.x] = total;
}

// One CTA: v[0, n) replaced by its exclusive scan; *total = the sum, plus the whole bytes of *nbits bits when nbits is
// given (the stuffed length: entropy bytes + one 0x00 per 0xFF)
__global__ void __launch_bounds__(kScanThreads) jpeg_scan_kernel(int* __restrict__ v, int n, int* __restrict__ total,
                                                                 const int* __restrict__ nbits) {
  int carry = 0;
  for (int t = 0; t < n; t += blockDim.x) {
    const int i = t + threadIdx.x;
    const int x = i < n ? v[i] : 0;
    int sum;
    const int ex = block_excl_scan(x, &sum);
    if (i < n) v[i] = carry + ex;
    carry += sum;
  }
  if (threadIdx.x == 0) *total = carry + (nbits ? (*nbits + 7) >> 3 : 0);
}

// the words the file's *nbits bits occupy, zeroed for jpeg_pack_kernel's OR-ing
__global__ void jpeg_zero_kernel(const int* __restrict__ nbits, uint32_t* __restrict__ words) {
  const int nw = (*nbits + 31) >> 5;
  GRID_STRIDE(i, nw) words[i] = 0;
}

// kTileBlocks blocks per CTA: each block's codes at toff[tile] + boff[s], shared boundary words OR-ed atomically as
// in jpeg_huff_kernel; the thread of the last block adds the padding 1-bits
__global__ void __launch_bounds__(kTileBlocks) jpeg_pack_kernel(const __grid_constant__ EncGeom g, const int16_t* __restrict__ coef,
                                                                const uint32_t* __restrict__ codes, const int* __restrict__ boff,
                                                                const int* __restrict__ toff, const int* __restrict__ nbits,
                                                                uint32_t* __restrict__ words) {
  __shared__ uint32_t s_codes[4][256];
  for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) (&s_codes[0][0])[i] = codes[i];
  __syncthreads();
  const int s = blockIdx.x * kTileBlocks + threadIdx.x;
  if (s >= g.nblk) return;
  int64_t off, prev;
  const int comp = jpg::scan_block(g, s, &off, &prev);
  WordSink ws(words, toff[blockIdx.x] + boff[s]);
  jpg::huff_block(coef + off, prev < 0 ? 0 : coef[prev], s_codes[comp ? 2 : 0], s_codes[comp ? 3 : 1], ws);
  ws.flush();
  if (s == g.nblk - 1) {
    const int T = *nbits, pad = ((T + 7) >> 3) * 8 - T;
    if (pad) atomicOr(words + (T >> 5), ((1u << pad) - 1) << (32 - (T & 31) - pad));
  }
}

// the words [w0, w1) of segment blockIdx.x of the file's entropy bytes (kStuffSegs equal segments)
__device__ void stuff_segment(int nbytes, int* w0, int* w1) {
  const int nw = (nbytes + 3) >> 2, per = (nw + gridDim.x - 1) / gridDim.x;
  *w0 = min(nw, (int)blockIdx.x * per);
  *w1 = min(nw, *w0 + per);
}

// sff[seg] = the 0xFF bytes among the entropy bytes of segment seg
__global__ void __launch_bounds__(kStuffThreads) jpeg_ffcount_kernel(const uint32_t* __restrict__ words, const int* __restrict__ nbits,
                                                                     int* __restrict__ sff) {
  const int nbytes = (*nbits + 7) >> 3;
  int w0, w1;
  stuff_segment(nbytes, &w0, &w1);
  int ff = 0;
  for (int i = w0 + threadIdx.x; i < w1; i += blockDim.x) {
    const uint32_t v = words[i];
    for (int j = 0; j < 4 && 4 * i + j < nbytes; ++j) ff += ((v >> (24 - 8 * j)) & 0xff) == 0xff;
  }
  int total;
  block_excl_scan(ff, &total);
  if (threadIdx.x == 0) sff[blockIdx.x] = total;
}

// The file at out + off[0]: header (CTA 0), each segment's stuffed bytes shifted by the 0x00s of the segments before
// it (soff[seg]), EOI after the *slen stuffed bytes
__global__ void __launch_bounds__(kStuffThreads) jpeg_scatter_kernel(const uint32_t* __restrict__ words, const int* __restrict__ nbits,
                                                                     const int* __restrict__ soff, const int* __restrict__ slen,
                                                                     const uint8_t* __restrict__ hdr, int hdr_len,
                                                                     const int64_t* __restrict__ off, uint8_t* __restrict__ out) {
  uint8_t* dst = out + off[0];
  if (blockIdx.x == 0)
    for (int i = threadIdx.x; i < hdr_len; i += blockDim.x) dst[i] = hdr[i];
  dst += hdr_len;
  const int nbytes = (*nbits + 7) >> 3;
  int w0, w1;
  stuff_segment(nbytes, &w0, &w1);
  int carry = soff[blockIdx.x];
  for (int t = w0; t < w1; t += blockDim.x) {
    const int i = t + threadIdx.x;
    uint32_t v = 0;
    int nb = 0, ff = 0;
    if (i < w1) {
      v = words[i];
      nb = min(4, nbytes - 4 * i);
      for (int j = 0; j < nb; ++j) ff += ((v >> (24 - 8 * j)) & 0xff) == 0xff;
    }
    int total;
    int p = 4 * i + carry + block_excl_scan(ff, &total);
    for (int j = 0; j < nb; ++j) {
      const uint8_t b = (uint8_t)(v >> (24 - 8 * j));
      dst[p++] = b;
      if (b == 0xff) dst[p++] = 0;
    }
    carry += total;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    dst[*slen] = 0xff;
    dst[*slen + 1] = 0xd9;
  }
}

// ---- host side -----------------------------------------------------------------------------------------------------
void put16(std::vector<uint8_t>& v, int x) {
  v.push_back((uint8_t)(x >> 8));
  v.push_back((uint8_t)x);
}
void segment(std::vector<uint8_t>& h, int marker, const std::vector<uint8_t>& body) {
  h.push_back(0xff);
  h.push_back((uint8_t)marker);
  put16(h, (int)body.size() + 2);
  h.insert(h.end(), body.begin(), body.end());
}
// SOI, APP0 (JFIF 1.01, density 1:1, unit 0), one DQT per table, SOF0, one DHT per table, SOS: Pillow's header
std::vector<uint8_t> jfif_header(const EncGeom& g) {
  std::vector<uint8_t> h = {0xff, 0xd8};
  segment(h, 0xe0, {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0});
  const int nt = g.Cs == 3 ? 2 : 1;
  for (int t = 0; t < nt; ++t) {
    std::vector<uint8_t> b = {(uint8_t)t};
    for (int k = 0; k < 64; ++k) b.push_back((uint8_t)g.q[t][jpg::natural_of(k)]);
    segment(h, 0xdb, b);
  }
  std::vector<uint8_t> sof = {8};
  put16(sof, g.H);
  put16(sof, g.W);
  sof.push_back((uint8_t)g.Cs);
  for (int c = 0; c < g.Cs; ++c) {
    sof.push_back((uint8_t)(c + 1));
    sof.push_back(c == 0 && g.Cs == 3 ? 0x22 : 0x11);
    sof.push_back(c ? 1 : 0);
  }
  segment(h, 0xc0, sof);
  for (int t = 0; t < 2 * nt; ++t) {
    std::vector<uint8_t> b = {(uint8_t)(((t & 1) << 4) | (t >> 1))};
    int n = 0;
    for (int l = 0; l < 16; ++l) n += jpg::kStdBits[t][l];
    b.insert(b.end(), jpg::kStdBits[t], jpg::kStdBits[t] + 16);
    b.insert(b.end(), jpg::std_vals(t), jpg::std_vals(t) + n);
    segment(h, 0xc4, b);
  }
  std::vector<uint8_t> sos = {(uint8_t)g.Cs};
  for (int c = 0; c < g.Cs; ++c) {
    sos.push_back((uint8_t)(c + 1));
    sos.push_back(c ? 0x11 : 0x00);
  }
  sos.insert(sos.end(), {0, 63, 0});
  segment(h, 0xda, sos);
  return h;
}

EncGeom make_geom(int Cs, int H, int W, int quality, int* smem) {
  EncGeom g;
  memset(&g, 0, sizeof(g));
  g.Cs = Cs;
  g.H = H;
  g.W = W;
  g.hs = g.vs = Cs == 3 ? 2 : 1;
  g.mcux = (g.W + 8 * g.hs - 1) / (8 * g.hs);
  g.mcuy = (g.H + 8 * g.vs - 1) / (8 * g.vs);
  g.bwr = (g.W + 7) / 8;
  g.bhr = (g.H + 7) / 8;
  g.nblk = (int)(jpg::image_coefs(g.Cs, g.hs, g.vs, g.mcux, g.mcuy) / 64);
  g.rows = std::max(1, std::min(g.mcuy, kBandBudget / (g.Cs * 8 * g.vs * g.W)));
  g.bands = (g.mcuy + g.rows - 1) / g.rows;
  *smem = g.Cs * std::min(g.rows * 8 * g.vs, g.H) * g.W;
  jpg::quant_table(quality, 0, g.q[0]);
  jpg::quant_table(quality, 1, g.q[1]);
  return g;
}

template <typename T>
int dev_reserve(fg_ctx* c, T** p, int64_t* cap, int64_t n) {
  if (n <= *cap) return FG_OK;
  FG_CUDA(cudaStreamSynchronize(c->stream));
  cudaFree(*p);
  *p = nullptr;
  *cap = 0;
  FG_CUDA(cudaMalloc((void**)p, sizeof(T) * (size_t)n));
  *cap = n;
  return FG_OK;
}

int check_span(fg_dataset* d, const char* what, int64_t first, int64_t count, int quality) {
  if (!d || !d->c) {
    fg_set_error("null fg_dataset");
    return FG_ERR_INVALID;
  }
  FG_REQUIRE(first >= 0 && count >= 1 && first <= d->N - count, "%s: range [%lld, %lld) outside [0, %lld)", what,
             (long long)first, (long long)(first + count), (long long)d->N);
  FG_REQUIRE(quality >= 1 && quality <= 100, "%s: quality %d outside 1..100", what, quality);
  return FG_OK;
}

}  // namespace

// Chunk scratch of the encoder, grown to the largest chunk seen; freed with the dataset (fg_dataset_encode_jpeg,
// fg_dataset_jpeg_roundtrip) or the ctx (fg_jpeg_encode).
struct JpegEncScratch {
  int16_t* coef = nullptr;
  int64_t coef_cap = 0;
  uint32_t* words = nullptr;
  int64_t words_cap = 0;
  int* boff = nullptr;
  int64_t boff_cap = 0;
  int* lens = nullptr;  // [2][images]: bit counts, stuffed byte counts
  int64_t lens_cap = 0;
  int* lens_host = nullptr;  // pinned mirror of the stuffed byte counts
  int64_t lens_host_cap = 0;
  int64_t* off = nullptr;  // file offsets within the chunk's output
  int64_t off_cap = 0;
  uint8_t* out = nullptr;
  int64_t out_cap = 0;
  uint8_t* consts = nullptr;  // Huffman codes [4][256] u32, then the header; or the round trip's TableSet
  int64_t consts_cap = 0;
  uint8_t* desc = nullptr;  // the round trip's ImageDesc / BandDesc arrays
  int64_t desc_cap = 0;
  int* part = nullptr;  // the multi-CTA coder's tile sums, then its segment 0xFF counts
  int64_t part_cap = 0;
  uint8_t* src = nullptr;  // fg_jpeg_encode: the chunk's images when the caller's are in host memory
  int64_t src_cap = 0;
};

void jpeg_enc_scratch_free(JpegEncScratch* s) {
  if (!s) return;
  cudaFree(s->coef);
  cudaFree(s->words);
  cudaFree(s->boff);
  cudaFree(s->lens);
  cudaFreeHost(s->lens_host);
  cudaFree(s->off);
  cudaFree(s->out);
  cudaFree(s->consts);
  cudaFree(s->desc);
  cudaFree(s->part);
  cudaFree(s->src);
  delete s;
}

namespace {

// jpeg_fdct_kernel on n images at src (device, [n][Cs][H][W]) into the coefficient scratch
int run_fdct(fg_ctx* c, JpegEncScratch& s, const EncGeom& g, int smem, const uint8_t* src, int n) {
  FG_TRY(dev_reserve(c, &s.coef, &s.coef_cap, (int64_t)n * g.nblk * 64));
  if (smem > 48 * 1024) FG_CUDA(cudaFuncSetAttribute(jpeg_fdct_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  jpeg_fdct_kernel<<<n * g.bands, kFdctThreads, smem, c->stream>>>(g, src, s.coef);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// the multi-CTA coder: one file per chunk
bool multi_cta(const fg_ctx* c, const EncGeom& g) {
  return c->jpeg_route == 2 || (c->jpeg_route == 0 && g.nblk >= kMultiMinBlocks);
}

// forward kernel and entropy coding of n images at src: the bit and stuffed byte counts in s.lens, the stuffed byte
// count of each also in s.lens_host
int run_code(fg_ctx* c, JpegEncScratch& s, const EncGeom& g, int smem, const uint8_t* src, int n) {
  FG_TRY(run_fdct(c, s, g, smem, src, n));
  FG_TRY(dev_reserve(c, &s.words, &s.words_cap, (int64_t)n * g.nblk * kBlockWords));
  FG_TRY(dev_reserve(c, &s.boff, &s.boff_cap, (int64_t)n * g.nblk));
  FG_TRY(dev_reserve(c, &s.lens, &s.lens_cap, 2 * (int64_t)n));
  if (n > s.lens_host_cap) {
    cudaFreeHost(s.lens_host);
    s.lens_host = nullptr;
    s.lens_host_cap = 0;
    FG_CUDA(cudaHostAlloc((void**)&s.lens_host, sizeof(int) * (size_t)n, cudaHostAllocDefault));
    s.lens_host_cap = n;
  }
  const uint32_t* codes = reinterpret_cast<const uint32_t*>(s.consts);
  if (multi_cta(c, g)) {
    const int tiles = (g.nblk + kTileBlocks - 1) / kTileBlocks;
    FG_TRY(dev_reserve(c, &s.part, &s.part_cap, (int64_t)std::max(tiles, kStuffSegs)));
    jpeg_blen_kernel<<<tiles, kTileBlocks, 0, c->stream>>>(g, s.coef, codes, s.boff, s.part);
    LAUNCH_CHECK(c);
    jpeg_scan_kernel<<<1, kScanThreads, 0, c->stream>>>(s.part, tiles, s.lens, nullptr);
    LAUNCH_CHECK(c);
    jpeg_zero_kernel<<<grid_for((int64_t)g.nblk * kBlockWords, 256, c->sm_count * 4), 256, 0, c->stream>>>(s.lens, s.words);
    LAUNCH_CHECK(c);
    jpeg_pack_kernel<<<tiles, kTileBlocks, 0, c->stream>>>(g, s.coef, codes, s.boff, s.part, s.lens, s.words);
    LAUNCH_CHECK(c);
    jpeg_ffcount_kernel<<<kStuffSegs, kStuffThreads, 0, c->stream>>>(s.words, s.lens, s.part);
    LAUNCH_CHECK(c);
    jpeg_scan_kernel<<<1, kScanThreads, 0, c->stream>>>(s.part, kStuffSegs, s.lens + 1, s.lens);
    LAUNCH_CHECK(c);
  } else {
    jpeg_huff_kernel<<<n, kHuffThreads, 0, c->stream>>>(g, s.coef, codes, s.words, s.boff, s.lens, s.lens + n);
    LAUNCH_CHECK(c);
  }
  FG_CUDA(cudaMemcpyAsync(s.lens_host, s.lens + n, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

// The JFIF files of `count` images, each [Cs][H][W]: image i at images + i * Cs*H*W, device memory, or host memory
// staged a chunk at a time.  offsets / out / cap as fg_dataset_encode_jpeg.
int encode_files(fg_ctx* c, JpegEncScratch& s, const char* what, const uint8_t* images, bool host, int64_t count, int Cs,
                 int H, int W, int quality, uint8_t* out, int64_t cap, int64_t* offsets) {
  int smem;
  const EncGeom g = make_geom(Cs, H, W, quality, &smem);
  const int64_t per = (int64_t)Cs * H * W;
  const std::vector<uint8_t> hdr = jfif_header(g);
  std::vector<uint8_t> consts(4 * 256 * sizeof(uint32_t) + hdr.size());
  for (int t = 0; t < 4; ++t) jpg::huff_codes(t, reinterpret_cast<uint32_t*>(consts.data()) + 256 * t);
  memcpy(consts.data() + 4 * 256 * sizeof(uint32_t), hdr.data(), hdr.size());
  FG_TRY(dev_reserve(c, &s.consts, &s.consts_cap, (int64_t)consts.size()));
  FG_CUDA(cudaMemcpyAsync(s.consts, consts.data(), consts.size(), cudaMemcpyHostToDevice, c->stream));
  const uint8_t* hdr_dev = s.consts + 4 * 256 * sizeof(uint32_t);
  const int64_t fixed = (int64_t)hdr.size() + 2;  // header + EOI
  const bool multi = multi_cta(c, g);
  const int chunk = multi ? 1 : (int)std::max<int64_t>(1, std::min<int64_t>(count, kChunkBlocks / g.nblk));
  // the chunk's images on the device
  auto chunk_src = [&](int64_t i, int n, const uint8_t** src) -> int {
    *src = images + i * per;
    if (!host) return FG_OK;
    FG_TRY(dev_reserve(c, &s.src, &s.src_cap, n * per));
    FG_CUDA(cudaMemcpyAsync(s.src, *src, (size_t)(n * per), cudaMemcpyHostToDevice, c->stream));
    *src = s.src;
    return FG_OK;
  };

  // pass 1: every file's size
  offsets[0] = 0;
  for (int64_t i = 0; i < count; i += chunk) {
    const int n = (int)std::min<int64_t>(chunk, count - i);
    const uint8_t* src;
    FG_TRY(chunk_src(i, n, &src));
    FG_TRY(run_code(c, s, g, smem, src, n));
    for (int k = 0; k < n; ++k) offsets[i + k + 1] = offsets[i + k] + fixed + s.lens_host[k];
  }
  if (!out) return FG_OK;
  if (offsets[count] > cap) {
    fg_set_error("%s: the files take %lld bytes, the buffer holds %lld", what, (long long)offsets[count], (long long)cap);
    return FG_ERR_INVALID;
  }
  // pass 2: the files (a single chunk is still coded from pass 1)
  std::vector<int64_t> off(chunk);
  for (int64_t i = 0; i < count; i += chunk) {
    const int n = (int)std::min<int64_t>(chunk, count - i);
    if (count > chunk) {
      const uint8_t* src;
      FG_TRY(chunk_src(i, n, &src));
      FG_TRY(run_code(c, s, g, smem, src, n));
    }
    for (int k = 0; k < n; ++k) off[k] = offsets[i + k] - offsets[i];
    const int64_t bytes = offsets[i + n] - offsets[i];
    FG_TRY(dev_reserve(c, &s.off, &s.off_cap, (int64_t)n));
    FG_TRY(dev_reserve(c, &s.out, &s.out_cap, bytes));
    FG_CUDA(cudaMemcpyAsync(s.off, off.data(), sizeof(int64_t) * n, cudaMemcpyHostToDevice, c->stream));
    if (multi)
      jpeg_scatter_kernel<<<kStuffSegs, kStuffThreads, 0, c->stream>>>(s.words, s.lens, s.part, s.lens + 1, hdr_dev,
                                                                     (int)hdr.size(), s.off, s.out);
    else
      jpeg_stuff_kernel<<<n, kStuffThreads, 0, c->stream>>>(g.nblk, s.words, s.lens, hdr_dev, (int)hdr.size(), s.off, s.out);
    LAUNCH_CHECK(c);
    FG_CUDA(cudaMemcpyAsync(out + offsets[i], s.out, (size_t)bytes, cudaMemcpyDefault, c->stream));
    FG_CUDA(cudaStreamSynchronize(c->stream));
  }
  return FG_OK;
}

}  // namespace

extern "C" {

int fg_dataset_encode_jpeg(fg_dataset* d, int64_t first, int64_t count, int quality, uint8_t* out, int64_t cap,
                           int64_t* offsets) {
  FG_TRY(check_span(d, "fg_dataset_encode_jpeg", first, count, quality));
  FG_REQUIRE(offsets, "fg_dataset_encode_jpeg: null offsets");
  FG_REQUIRE(!out || cap >= 0, "fg_dataset_encode_jpeg: negative capacity");
  fg_ctx* c = d->c;
  FG_CUDA(cudaSetDevice(c->device));
  if (!d->jpeg_enc) d->jpeg_enc = new JpegEncScratch();
  const int64_t per = (int64_t)d->Cs * d->Hs * d->Ws;
  return encode_files(c, *d->jpeg_enc, "fg_dataset_encode_jpeg", d->data + first * per, false, count, d->Cs, d->Hs, d->Ws,
                      quality, out, cap, offsets);
}

int fg_jpeg_encode(fg_ctx* c, const uint8_t* images, int count, int C, int H, int W, int quality, uint8_t* out, int64_t cap,
                   int64_t* offsets) {
  if (!c) {
    fg_set_error("null fg_ctx");
    return FG_ERR_INVALID;
  }
  FG_REQUIRE(images && offsets && count >= 1, "fg_jpeg_encode: need images, offsets and count >= 1");
  FG_REQUIRE(C == 1 || C == 3, "fg_jpeg_encode: %d channels (1 or 3)", C);
  FG_REQUIRE(H >= 1 && W >= 1 && H <= 4096 && W <= 4096, "fg_jpeg_encode: size %dx%d outside [1, 4096]", H, W);
  FG_REQUIRE(quality >= 1 && quality <= 100, "fg_jpeg_encode: quality %d outside 1..100", quality);
  FG_REQUIRE(!out || cap >= 0, "fg_jpeg_encode: negative capacity");
  FG_CUDA(cudaSetDevice(c->device));
  if (!c->jpeg_enc) c->jpeg_enc = new JpegEncScratch();
  return encode_files(c, *c->jpeg_enc, "fg_jpeg_encode", images, !fg_is_dev(images), count, C, H, W, quality, out, cap,
                      offsets);
}

int fg_dataset_jpeg_roundtrip(fg_dataset* d, int64_t first, int64_t count, int quality) {
  FG_TRY(check_span(d, "fg_dataset_jpeg_roundtrip", first, count, quality));
  fg_ctx* c = d->c;
  FG_CUDA(cudaSetDevice(c->device));
  if (!d->jpeg_enc) d->jpeg_enc = new JpegEncScratch();
  JpegEncScratch& s = *d->jpeg_enc;
  int smem;
  const EncGeom g = make_geom(d->Cs, d->Hs, d->Ws, quality, &smem);
  // the decoder's view of one file: its quantisation tables (the Huffman tables are not read by the IDCT kernel)
  jpg::TableSet ts;
  memset(&ts, 0, sizeof(ts));
  for (int k = 0; k < g.Cs; ++k) memcpy(ts.q[k], g.q[k ? 1 : 0], sizeof(ts.q[k]));
  FG_TRY(dev_reserve(c, &s.consts, &s.consts_cap, (int64_t)sizeof(ts)));
  FG_CUDA(cudaMemcpyAsync(s.consts, &ts, sizeof(ts), cudaMemcpyHostToDevice, c->stream));
  jpg::ImageDesc m;
  m.coef = 0;
  m.out = 0;
  m.set = 0;
  m.C = g.Cs;
  m.H = g.H;
  m.W = g.W;
  m.Cs = g.Cs;
  m.hs = g.hs;
  m.vs = g.vs;
  m.mcux = g.mcux;
  m.mcuy = g.mcuy;
  int idct_smem;
  const int rows = jpeg_idct_band_rows(m, &idct_smem);
  const int bands = (g.mcuy + rows - 1) / rows;
  const int chunk = (int)std::max<int64_t>(1, std::min<int64_t>(count, kChunkBlocks / g.nblk));
  const int64_t per = (int64_t)g.Cs * g.H * g.W;
  std::vector<jpg::ImageDesc> imgs(chunk);
  std::vector<jpg::BandDesc> bds((size_t)chunk * bands);
  const size_t o_band = (sizeof(jpg::ImageDesc) * chunk + 15) & ~(size_t)15;
  FG_TRY(dev_reserve(c, &s.desc, &s.desc_cap, (int64_t)(o_band + sizeof(jpg::BandDesc) * bds.size())));
  for (int64_t i = 0; i < count; i += chunk) {
    const int n = (int)std::min<int64_t>(chunk, count - i);
    FG_TRY(run_fdct(c, s, g, smem, d->data + (first + i) * per, n));
    for (int k = 0; k < n; ++k) {
      imgs[k] = m;
      imgs[k].coef = (int64_t)k * g.nblk * 64;
      imgs[k].out = (first + i + k) * per;
      for (int b = 0; b < bands; ++b) bds[(size_t)k * bands + b] = {k, b * rows, std::min(g.mcuy, (b + 1) * rows)};
    }
    // the previous chunk's IDCT has read its descriptors: the stream orders the copies after it
    FG_CUDA(cudaMemcpyAsync(s.desc, imgs.data(), sizeof(jpg::ImageDesc) * n, cudaMemcpyHostToDevice, c->stream));
    FG_CUDA(cudaMemcpyAsync(s.desc + o_band, bds.data(), sizeof(jpg::BandDesc) * n * bands, cudaMemcpyHostToDevice, c->stream));
    FG_TRY(jpeg_idct_launch(c, reinterpret_cast<const jpg::TableSet*>(s.consts), reinterpret_cast<const jpg::ImageDesc*>(s.desc),
                            reinterpret_cast<const jpg::BandDesc*>(s.desc + o_band), n * bands, idct_smem, s.coef, d->data));
  }
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

}  // extern "C"
