-- sample_b200.lua -- drop-in for sample.lua's c2f(images, G, D, fineSize) (sample.lua:176-214): refines a table of
-- images through a trained coarse-to-fine G/D pair on the GPU, 10 tries per image, keeping the try D rates highest.
-- Same signature, a table of images in and a table of refined [C][fineSize][fineSize] FloatTensors out.
-- One fg_c2f per fine size is built from G:getParameters() / D:getParameters() on first use (and rebuilt when another
-- G / D is passed for that size).  D's dropout stays live, as sample.lua never calls evaluate().
-- Delivered untested-by-execution (no LuaJIT/Torch7 in the build image); face_generator_b200/pyramid.py (refine) is
-- the executable mirror and tests/test_gpu_c2f_refine.py drives the same C call through ctypes.
require 'torch'
local ffi = require 'ffi'
local F = require 'fg_ffi'
require 'b200'
local C = F.C

local sample_b200 = {}
local TRIES = 10         -- sample.lua:177 triesPerImage
local nets = {}          -- fineSize -> {net = fg_c2f*, G = G, D = D}
local calls = 0

local function c2f_net(ctx, G, D, fineSize)
  local e = nets[fineSize]
  if e == nil or e.G ~= G or e.D ~= D then
    if e ~= nil then C.fg_c2f_destroy(e.net) end
    local out = ffi.new('fg_c2f*[1]')
    F.check(C.fg_c2f_create_sized(ctx, fineSize, out), 'fg_c2f_create_sized')
    local pG = G:getParameters():float():contiguous()
    local pD = D:getParameters():float():contiguous()
    F.check(C.fg_c2f_set_params(out[0], 0, F.ptr(pG)), 'fg_c2f_set_params(G)')
    F.check(C.fg_c2f_set_params(out[0], 1, F.ptr(pD)), 'fg_c2f_set_params(D)')
    e = {net = out[0], G = G, D = D}
    nets[fineSize] = e
  end
  return e.net
end

-- sample.lua:176-214
function sample_b200.c2f(images, G, D, fineSize)
  local N = #images
  local channels, inSize = images[1]:size(1), images[1]:size(2)
  local ctx = b200.context(OPT and OPT.gpu or 0, TRIES * 16, channels)
  local net = c2f_net(ctx, G, D, fineSize)
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

return sample_b200
