-- sample_b200.lua -- drop-in for sample.lua's c2f(images, G, D, fineSize) (sample.lua:176-214): refines a table of
-- images through a trained coarse-to-fine G/D pair on the GPU, 10 tries per image, keeping the try D rates highest.
-- Same signature, a table of images in and a table of refined [C][fineSize][fineSize] FloatTensors out.
-- One fg_c2f per fine size is built from G:getParameters() / D:getParameters() on first use (and rebuilt when another
-- G / D is passed for that size).  D's dropout stays live, as sample.lua never calls evaluate().
-- sample_b200.main(OPT) is the drop-in for sample.lua's main() (sample.lua:69-115): every run's sheets are generated,
-- scored, laid out and JPEG-encoded on the GPU and only the files' bytes come back (face_generator_b200/sheets.py
-- sample_run is the executable mirror, with the same seeds and permutations).
-- Delivered untested-by-execution (no LuaJIT/Torch7 in the build image); face_generator_b200/pyramid.py (refine) and
-- face_generator_b200/sheets.py (sample_run) are the executable mirrors, and tests/test_gpu_c2f_refine.py and
-- tests/test_gpu_sample_sheets.py drive the same C calls through ctypes.
require 'torch'
local ffi = require 'ffi'
local F = require 'fg_ffi'
require 'b200'
local C = F.C

local sample_b200 = {}
local TRIES = 10         -- sample.lua:177 triesPerImage
local nets = {}          -- fineSize -> {net = fg_c2f*, G = G, D = D}
local calls = 0

local function c2f_net(ctx, G, D, fineSize, channels)
  local e = nets[fineSize]
  if e == nil or e.G ~= G or e.D ~= D then
    if e ~= nil then
      C.fg_c2f_destroy(e.net)
      nets[fineSize] = nil   -- if building the new net fails, no later call may get the destroyed one back
    end
    -- G and D may be any of models_c2f.lua's nets; their parameter vectors are checked against the recognised nets
    local pG = G:getParameters():float():contiguous()
    local pD = D:getParameters():float():contiguous()
    e = {net = b200.c2fNets(ctx, G, D, pG, pD, fineSize, channels), G = G, D = D}
    nets[fineSize] = e
  end
  return e.net
end

-- sample.lua:176-214
function sample_b200.c2f(images, G, D, fineSize)
  local N = #images
  local channels, inSize = images[1]:size(1), images[1]:size(2)
  local ctx = b200.context(OPT and OPT.gpu or 0, TRIES * 16, channels)
  local net = c2f_net(ctx, G, D, fineSize, channels)
  -- as many images per pass as the ctx's batch holds (the result does not depend on it)
  local chunk = math.max(1, math.floor(tonumber(C.fg_get_option(ctx, 'max_batch')) / TRIES))
  local batch = torch.FloatTensor(N, channels, inSize, inSize)
  for i = 1, N do batch[i]:copy(images[i]) end
  local refined = torch.FloatTensor(N, channels, fineSize, fineSize)
  calls = calls + 1
  -- noise and dropout masks from the device streams of seed `calls`: a fresh draw per call, as noiseInputs:uniform
  F.check(C.fg_c2f_refine(net, F.ptr(batch), N, inSize, TRIES, chunk, 1, nil, nil, calls, F.ptr(refined), nil, nil),
          'fg_c2f_refine')
  local result = {}
  for i = 1, N do table.insert(result, refined[i]:clone()) end
  return result
end

-- ---- sample.lua:main() --------------------------------------------------------------------------------------------
local U64 = ffi.typeof('uint64_t')
local NOISE_DIM = 100

-- sheets.run_streams: key = seed * 1000003 + run, then 8 * key + k (k = 0 noise, 1 / 2 the best / worst scoring
-- passes, 3 / 4 the random256 / random permutations)
local function run_streams(seed, run)
  local key = U64(seed) * 1000003ULL + U64(run)
  local s = {}
  for k = 0, 4 do s[k] = key * 8ULL + U64(k) end
  return s
end

-- sheets.permutation: 0..n-1 sorted by splitmix64(stream * 2^32 + i), ties by i (the stand-in for torch.randperm)
local function permutation(stream, n)
  local keys, idx = {}, {}
  for i = 0, n - 1 do
    local x = stream * 4294967296ULL + U64(i) + 0x9E3779B97F4A7C15ULL
    x = bit.bxor(x, bit.rshift(x, 30)) * 0xBF58476D1CE4E5B9ULL
    x = bit.bxor(x, bit.rshift(x, 27)) * 0x94D049BB133111EBULL
    keys[i] = bit.bxor(x, bit.rshift(x, 31))
    idx[i + 1] = i
  end
  table.sort(idx, function(a, b) if keys[a] ~= keys[b] then return keys[a] < keys[b] end return a < b end)
  return idx
end

local function int32s(t, n)
  local a = ffi.new('int32_t[?]', n)
  for i = 1, n do a[i - 1] = t[i] end
  return a
end

-- one sheet: fg_image_grid of images[order] into the device buffer `grid`, fg_jpeg_encode, written to path
local function write_sheet(ctx, path, images, N, ch, S, order, count, nrow, grid)
  local hg, wg = ffi.new('int[1]'), ffi.new('int[1]')
  F.check(C.fg_image_grid(ctx, images, N, ch, S, S, order, count, nrow, 0, ffi.cast('uint8_t*', grid), hg, wg), 'fg_image_grid')
  local offsets = ffi.new('int64_t[2]')
  F.check(C.fg_jpeg_encode(ctx, ffi.cast('const uint8_t*', grid), 1, ch, hg[0], wg[0], 75, nil, 0, offsets), 'fg_jpeg_encode')
  local bytes = ffi.new('uint8_t[?]', offsets[1])
  F.check(C.fg_jpeg_encode(ctx, ffi.cast('const uint8_t*', grid), 1, ch, hg[0], wg[0], 75, bytes, offsets[1], offsets),
          'fg_jpeg_encode')
  local f = assert(io.open(path, 'wb'))
  f:write(ffi.string(bytes, offsets[1]))
  f:close()
end

-- sample.lua:69-115 with MODEL_G / MODEL_D from loadModels() (or G, D given): OPT.runs runs of 1024 images, each
-- writing random256 / random1024 / best / worst / random _%04d_base.jpg into OPT.writeto, and with OPT.neighbours the
-- neighbour sheet against `dataset` (an fg_dataset* of the training set, b200.loadImagesToDevice of DATASET's dirs).
function sample_b200.main(OPT, G, D, dataset)
  if G == nil then G, D = loadModels() end
  local N, chunk, S = 1024, OPT.batchSize, OPT.scale
  assert(S == 32 or S == 16, 'sample_b200.main: --scale 32 or 16')
  local ch = OPT.grayscale and 1 or 3
  local ctx = b200.context(OPT.gpu, math.max(chunk, 16), ch)
  local pG = G:getParameters():float():contiguous()
  local pD = D:getParameters():float():contiguous()
  local s16 = S == 16 and b200.s16(ctx) or nil
  if s16 then
    F.check(C.fg_s16_set_params(s16, 0, F.ptr(pG)), 'fg_s16_set_params(G)')
    F.check(C.fg_s16_set_params(s16, 1, F.ptr(pD)), 'fg_s16_set_params(D)')
  else
    F.check(C.fg_set_params(ctx, 0, F.ptr(pG)), 'fg_set_params(G)')
    F.check(C.fg_set_params(ctx, 1, F.ptr(pD)), 'fg_set_params(D)')
  end
  local per = ch * S * S
  local noise = ffi.cast('float*', C.fg_dev_alloc(4 * N * NOISE_DIM))
  local images = ffi.cast('float*', C.fg_dev_alloc(4 * N * per))
  local pairs = ffi.cast('float*', C.fg_dev_alloc(4 * 32 * per))
  local nidx = ffi.cast('int32_t*', C.fg_dev_alloc(4 * 16))
  local ndist = ffi.cast('float*', C.fg_dev_alloc(4 * 16))
  local grid = C.fg_dev_alloc(ch * 32 * S * 32 * S)
  for run = 1, OPT.runs do
    local st = run_streams(OPT.seed, run)
    F.check(C.fg_noise_uniform(ctx, st[0], N * NOISE_DIM, noise), 'fg_noise_uniform')
    if s16 then
      for s = 0, N - 1, chunk do
        F.check(C.fg_s16_G_forward(s16, noise + s * NOISE_DIM, math.min(chunk, N - s), 1, images + s * per), 'fg_s16_G_forward')
      end
    else
      F.check(C.fg_sample(ctx, noise, N, chunk, images), 'fg_sample')
    end
    -- two sortImagesByPrediction calls (sample.lua:84-85): two passes with live dropout
    local preds = {}
    for k = 1, 2 do
      local p = ffi.new('float[?]', N)
      if s16 then
        F.check(C.fg_s16_D_score(s16, images, N, chunk, 1, st[k], p), 'fg_s16_D_score')
      else
        F.check(C.fg_D_score(ctx, images, N, chunk, 1, st[k], p), 'fg_D_score')
      end
      preds[k] = p
    end
    local function ranked(p, ascending)  -- a stable argsort, as scoring.sort_images_by_prediction
      local idx = {}
      for i = 0, N - 1 do idx[i + 1] = i end
      table.sort(idx, function(a, b)
        if p[a] ~= p[b] then if ascending then return p[a] < p[b] end return p[a] > p[b] end
        return a < b
      end)
      return idx
    end
    local best, worst = ranked(preds[1], false), ranked(preds[2], true)
    local name = function(f) return paths.concat(OPT.writeto, string.format(f, run)) end
    write_sheet(ctx, name('random256_%04d_base.jpg'), images, N, ch, S, int32s(permutation(st[3], N), 256), 256, 16, grid)
    write_sheet(ctx, name('random1024_%04d_base.jpg'), images, N, ch, S, nil, N, 32, grid)
    write_sheet(ctx, name('best_%04d_base.jpg'), images, N, ch, S, int32s(best, 64), 64, 8, grid)
    write_sheet(ctx, name('worst_%04d_base.jpg'), images, N, ch, S, int32s(worst, 64), 64, 8, grid)
    write_sheet(ctx, name('random_%04d_base.jpg'), images, N, ch, S, int32s(permutation(st[4], N), 64), 64, 8, grid)
    if OPT.neighbours then
      assert(dataset ~= nil, 'sample_b200.main: --neighbours needs the training set as an fg_dataset*')
      for i = 0, 15 do F.check(C.fg_memcpy(ctx, pairs + i * per, images + best[i + 1] * per, 4 * per), 'fg_memcpy') end
      F.check(C.fg_dataset_nearest_sized(dataset, S, pairs, 16, nidx, ndist), 'fg_dataset_nearest_sized')
      F.check(C.fg_dataset_gather_sized(dataset, nidx, 16, S, pairs + 16 * per), 'fg_dataset_gather_sized')
      local order = {}
      for i = 0, 15 do order[2 * i + 1], order[2 * i + 2] = i, 16 + i end
      write_sheet(ctx, name('best_%04d_neighbours_base.jpg'), pairs, 32, ch, S, int32s(order, 32), 32, 16, grid)
    end
    xlua.progress(run, OPT.runs)
  end
  for _, p in ipairs({noise, images, pairs, nidx, ndist, grid}) do C.fg_dev_free(p) end
  print("Finished.")
end

return sample_b200
