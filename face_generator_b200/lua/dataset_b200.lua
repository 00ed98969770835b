-- dataset_b200.lua -- dataset.lua's loadImagesFromDirs (dataset.lua:156-211) straight into the device-resident
-- training set: the .jpg files are read with io.open and decoded on the GPU (fg_dataset_upload_jpeg), so no image
-- is decoded on the host.  .pgm files (train_autoencoder.lua's lfwcrop_grey set) are parsed here and uploaded as
-- decoded planes (fg_dataset_upload).  The Python mirror is DeviceDataset.from_dirs (face_generator_b200/dataset.py).
-- Delivered untested-by-execution (no LuaJIT/Torch7 in the build image).
--
-- b200.loadLFWToDevice builds the augmented LFW set those trainers read (dataset/generate_dataset.py) from LFW itself.
--
--   local ds = b200.loadImagesToDevice(ctx, DATASET.dirs, 'jpg', 3, 1, 250000)
--   local ds = b200.loadLFWToDevice(ctx, {'/data/lfw'}, 19, 43)   -- out_aug_64x64, on the GPU
--   local ds = b200.loadLFWToDevice(ctx, {'/data/lfw'}, 19, 43, 64, 2048, 75)   -- ... as its .jpg files decode
--   b200.saveDatasetJPEG(ds, 'out_aug_64x64', 75, 20)               -- and those files, encoded on the GPU
--   F.check(C.fg_train_step_dataset(ctx, ds, hyper, B, seed, stats), 'fg_train_step_dataset')
require 'paths'
local ffi = require 'ffi'
local F = require 'fg_ffi'
local C = F.C

b200 = b200 or {}

local CHUNK = 16384  -- files per fg_dataset_upload_jpeg call: bounds the host bytes held at once

-- the file list of loadImagesFromDirs with doSort = true: every file of each dir whose name ends in ext, sorted by
-- full path, then files[startAt .. min(startAt+count-1, #files)]
function b200.listImageFiles(dirs, ext, startAt, count)
  local files = {}
  for i = 1, #dirs do
    for file in paths.files(dirs[i]) do
      if file:find(ext .. '$') then
        table.insert(files, paths.concat(dirs[i], file))
      end
    end
    if #files == 0 then
      error('given directory doesnt contain any files of type: ' .. ext)
    end
  end
  table.sort(files, function (a, b) return a < b end)
  local out = {}
  for i = startAt, math.min(startAt + count - 1, #files) do
    out[#out + 1] = files[i]
  end
  return out
end

local function readFile(path)
  local f = assert(io.open(path, 'rb'))
  local s = f:read('*a')
  f:close()
  return s
end

-- binary (P5) 8-bit PGM -> width, height, offset of the pixel bytes (1-based)
local function pgmHeader(s, path)
  assert(s:sub(1, 2) == 'P5', path .. ': not a binary PGM (P5) file')
  local fields, p = {}, 3
  while #fields < 3 do
    local a, b = s:find('^%s+', p)
    if a then p = b + 1 end
    if s:sub(p, p) == '#' then
      p = (s:find('[\r\n]', p) or #s) + 1
    else
      local num = s:match('^%d+', p)
      assert(num, path .. ': bad PGM header')
      fields[#fields + 1] = tonumber(num)
      p = p + #num
    end
  end
  assert(fields[3] > 0 and fields[3] < 256, path .. ': only 8-bit PGM is supported')
  assert(#s >= p + fields[1] * fields[2], path .. ': truncated PGM data')
  return fields[1], fields[2], p + 1
end

-- dataset.loadImagesFromDirs(dirs, ext, startAt, count, true) as an fg_dataset* of nbChannels planes at the files'
-- own size (image.load(path, nbChannels, 'byte')), sized from the first file; every file must have that size.
-- A colour JPEG under nbChannels = 1 is refused: load it with nbChannels = 3, a 1-channel ctx gathers rgb2y of it.
function b200.loadImagesToDevice(ctx, dirs, ext, nbChannels, startAt, count)
  ext = ext or 'jpg'
  startAt = startAt or 1
  count = count or math.huge
  local files = b200.listImageFiles(dirs, ext, startAt, count)
  assert(#files > 0, 'no ' .. ext .. ' files in the requested range')
  local pgm = ext:lower():find('pgm$') ~= nil
  local first = readFile(files[1])
  local H, W
  if pgm then
    W, H = pgmHeader(first, files[1])
  else
    local c, h, w = ffi.new('int[1]'), ffi.new('int[1]'), ffi.new('int[1]')
    F.check(C.fg_jpeg_info(ffi.cast('const uint8_t*', first), #first, c, h, w), 'fg_jpeg_info ' .. files[1])
    H, W = h[0], w[0]
  end
  local out = ffi.new('fg_dataset*[1]')
  F.check(C.fg_dataset_create(ctx, #files, nbChannels, H, W, out), 'fg_dataset_create')
  local ds = ffi.gc(out[0], C.fg_dataset_destroy)
  local failed = ffi.new('int64_t[1]')
  for s = 1, #files, CHUNK do
    local n = math.min(CHUNK, #files - s + 1)
    if pgm then
      local plane = H * W
      local buf = ffi.new('uint8_t[?]', n * nbChannels * plane)
      for i = 0, n - 1 do
        local data = readFile(files[s + i])
        local w, h, p = pgmHeader(data, files[s + i])
        assert(w == W and h == H, files[s + i] .. ': PGM files of different sizes')
        for c = 0, nbChannels - 1 do
          ffi.copy(buf + (i * nbChannels + c) * plane, ffi.cast('const uint8_t*', data) + p - 1, plane)
        end
      end
      F.check(C.fg_dataset_upload(ds, s - 1, n, buf), 'fg_dataset_upload')
    else
      local parts, offsets, total = {}, ffi.new('int64_t[?]', n + 1), 0
      for i = 1, n do
        parts[i] = readFile(files[s + i - 1])
        offsets[i - 1] = total
        total = total + #parts[i]
      end
      offsets[n] = total
      local bytes = table.concat(parts)
      parts = nil
      local rc = C.fg_dataset_upload_jpeg(ds, s - 1, n, ffi.cast('const uint8_t*', bytes), offsets, failed)
      if rc ~= 0 then
        local where = failed[0] >= 0 and files[s + tonumber(failed[0])] or ''
        error(string.format('fg_dataset_upload_jpeg failed (%d): %s %s', rc, ffi.string(C.fg_last_error()), where))
      end
      collectgarbage()
    end
  end
  return ds
end

-- dataset/generate_dataset.py's walk: the .jpg files of each dir and of its direct subdirectories, sorted by full path
-- (the reference's order came from a set() and os.listdir, which is unspecified)
function b200.listLFWFiles(dirs)
  local files, seen = {}, {}
  local function add(dir)
    for file in paths.files(dir) do
      local p = paths.concat(dir, file)
      if file:find('%.jpg$') and paths.filep(p) and not seen[p] then
        seen[p] = true
        files[#files + 1] = p
      end
    end
  end
  for i = 1, #dirs do
    add(dirs[i])
    for sub in paths.files(dirs[i]) do
      if sub ~= '.' and sub ~= '..' and paths.dirp(paths.concat(dirs[i], sub)) then
        add(paths.concat(dirs[i], sub))
      end
    end
  end
  table.sort(files, function (a, b) return a < b end)
  return files
end

-- generate_dataset.py on the GPU (the Python mirror is DeviceDataset.from_lfw): an fg_dataset* of
-- #files * (1 + augmentations) rows of 3 x size x size, row i * (1 + augmentations) + a = augmentation a of photo i
-- (a = 0: the photo itself), the order of the reference's {i:06}_{a:03}.jpg names.  augmentations = 19 (default) is
-- out_aug_64x64, 0 is out_unaug_64x64; seed defaults to generate_dataset.py's 43.  Photos are decoded on the GPU
-- `chunk` at a time into a scratch cache and augmented from there (fg_dataset_upload_jpeg, fg_lfw_aug_params,
-- fg_dataset_augment).
-- quality (optional, last): pass every row through fg_dataset_jpeg_roundtrip(quality) -- 75 gives the rows the
-- reference's quality-75 files decode to; nil keeps the rows before any JPEG encoding
function b200.loadLFWToDevice(ctx, dirs, augmentations, seed, size, chunk, quality)
  augmentations = augmentations or 19
  seed = seed or 43
  size = size or 64
  chunk = chunk or 2048
  local files = b200.listLFWFiles(dirs)
  assert(#files > 0, 'no .jpg files in the given directories or their direct subdirectories')
  local first = readFile(files[1])
  local c, h, w = ffi.new('int[1]'), ffi.new('int[1]'), ffi.new('int[1]')
  F.check(C.fg_jpeg_info(ffi.cast('const uint8_t*', first), #first, c, h, w), 'fg_jpeg_info ' .. files[1])
  local H, W = h[0], w[0]
  local per = 1 + augmentations
  local out = ffi.new('fg_dataset*[1]')
  F.check(C.fg_dataset_create(ctx, #files * per, 3, size, size, out), 'fg_dataset_create')
  local ds = ffi.gc(out[0], C.fg_dataset_destroy)
  local failed = ffi.new('int64_t[1]')
  for s = 1, #files, chunk do
    local n = math.min(chunk, #files - s + 1)
    local parts, offsets, total = {}, ffi.new('int64_t[?]', n + 1), 0
    for i = 1, n do
      parts[i] = readFile(files[s + i - 1])
      offsets[i - 1] = total
      total = total + #parts[i]
    end
    offsets[n] = total
    local bytes = table.concat(parts)
    parts = nil
    local sc = ffi.new('fg_dataset*[1]')
    F.check(C.fg_dataset_create(ctx, n, 3, H, W, sc), 'fg_dataset_create')
    local rc = C.fg_dataset_upload_jpeg(sc[0], 0, n, ffi.cast('const uint8_t*', bytes), offsets, failed)
    if rc ~= 0 then
      local msg = ffi.string(C.fg_last_error())
      C.fg_dataset_destroy(sc[0])
      local where = failed[0] >= 0 and files[s + tonumber(failed[0])] or ''
      error(string.format('fg_dataset_upload_jpeg failed (%d): %s %s', rc, msg, where))
    end
    local augs = ffi.new('fg_aug[?]', n * per)
    rc = C.fg_lfw_aug_params(seed, s - 1, n, augmentations, H, W, augs)
    if rc == 0 then
      for k = 0, n * per - 1 do
        augs[k].src = augs[k].src - (s - 1)  -- rows of the scratch cache
      end
      rc = C.fg_dataset_augment(sc[0], ds, (s - 1) * per, augs, n * per)
    end
    local msg = rc ~= 0 and ffi.string(C.fg_last_error()) or nil
    C.fg_dataset_destroy(sc[0])
    if msg then error(string.format('LFW augmentation failed (%d): %s', rc, msg)) end
    collectgarbage()
  end
  if quality then
    F.check(C.fg_dataset_jpeg_roundtrip(ds, 0, #files * per, quality), 'fg_dataset_jpeg_roundtrip')
  end
  return ds
end

-- every row of ds as a JPEG file in dir (which must exist), encoded on the GPU at quality (default 75): byte for byte
-- what generate_dataset.py's misc.imsave wrote, named {i:06}_{a:03}.jpg for per (default 20) rows per photo
function b200.saveDatasetJPEG(ds, dir, quality, per)
  quality = quality or 75
  per = per or 20
  local N = tonumber(C.fg_dataset_size(ds))
  for s = 0, N - 1, CHUNK do
    local n = math.min(CHUNK, N - s)
    local offsets = ffi.new('int64_t[?]', n + 1)
    F.check(C.fg_dataset_encode_jpeg(ds, s, n, quality, nil, 0, offsets), 'fg_dataset_encode_jpeg (sizes)')
    local total = tonumber(offsets[n])
    local out = ffi.new('uint8_t[?]', math.max(total, 1))
    F.check(C.fg_dataset_encode_jpeg(ds, s, n, quality, out, total, offsets), 'fg_dataset_encode_jpeg')
    for i = 0, n - 1 do
      local r = s + i
      local f = assert(io.open(paths.concat(dir, string.format('%06d_%03d.jpg', math.floor(r / per), r % per)), 'wb'))
      f:write(ffi.string(out + offsets[i], tonumber(offsets[i + 1] - offsets[i])))
      f:close()
    end
    out = nil
    collectgarbage()
  end
end

return b200
