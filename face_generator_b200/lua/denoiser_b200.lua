-- denoiser_b200.lua -- drop-in for train_denoiser.lua's train() (:230-370): every batch is ONE fg_dn_train_step
-- (fevalAE + optim.adam, then fevalAE2 + optim.adam on the one OPTSTATE.adam).  Keeps the script's globals (OPT,
-- IMG_DIMENSIONS, EPOCH) and its return value (the two mean losses).
--
-- The decoders train in the library, so the Torch modules never run a forward: their parameters AND their BatchNorm
-- running statistics live only there.  M.copyToDecoder(net, decoder) writes both into a DECODER module tree (before
-- torch.save, :360-362); M.copyFromDecoder(net, decoder) reads both back (after loading --network).  net is 0 for AE's
-- decoder (AE:get(2)), 1 for AE2.  Delivered untested-by-execution (no LuaJIT/Torch7 in the build image);
-- face_generator_b200/denoiser.py is the executable mirror.
require 'torch'
local ffi = require 'ffi'
local F = require 'fg_ffi'
require 'b200'
local C = F.C

local M = {}
local BN_STATE = 2 * (8 + 8 + 2048)  -- [mean1 8][var1 8][mean2 8][var2 8][mean3 2048][var3 2048]

function M.init()
  local ctx = b200.context(OPT.gpu or 0, OPT.batchSize, IMG_DIMENSIONS[1])
  local out = ffi.new('fg_dn*[1]')
  F.check(C.fg_dn_create(ctx, IMG_DIMENSIONS[2], out), 'fg_dn_create')
  M.dn = ffi.gc(out[0], C.fg_dn_destroy)
  M.hyper = ffi.new('fg_dn_hyper[1]')
  C.fg_dn_hyper_default(M.hyper)
  M.hyper[0].L1, M.hyper[0].L2, M.hyper[0].clamp = OPT.coefL1, OPT.coefL2, OPT.AE_clamp
  M.n = tonumber(C.fg_dn_param_count(IMG_DIMENSIONS[1], IMG_DIMENSIONS[2]))
  -- the step seed: --seed selects the noise and dropout streams, the batch counter advances them
  M.seedBase = (OPT.seed or 1) * 2 ^ 32
  M.step = 0
  return M
end

-- flat getParameters() vectors of one decoder (PARAMETERS_AE is DECODER's: WhiteNoise has no parameters)
function M.setParameters(net, flat)
  F.check(C.fg_dn_set_params(M.dn, net, F.ptr(flat:float():contiguous())), 'fg_dn_set_params')
end
function M.getParameters(net)
  local p = torch.FloatTensor(M.n)
  F.check(C.fg_dn_get_params(M.dn, net, F.ptr(p)), 'fg_dn_get_params')
  return p
end
-- the BatchNorm running statistics of one decoder, in the layout above
function M.setBNState(net, state)
  assert(state:nElement() == BN_STATE, 'denoiser_b200: the BatchNorm state has ' .. BN_STATE .. ' floats')
  F.check(C.fg_dn_set_bn_state(M.dn, net, F.ptr(state:float():contiguous())), 'fg_dn_set_bn_state')
end
function M.getBNState(net)
  local s = torch.FloatTensor(BN_STATE)
  F.check(C.fg_dn_get_bn_state(M.dn, net, F.ptr(s)), 'fg_dn_get_bn_state')
  return s
end

-- the modules of a DECODER that hold parameters, and those that hold running statistics, in module order
local function walk(decoder)
  local params, bns = {}, {}
  for _, m in ipairs(decoder:listModules()) do
    if m.weight then table.insert(params, m.weight) end
    if m.bias then table.insert(params, m.bias) end
    if m.running_mean then table.insert(bns, m) end
  end
  assert(#bns == 3, 'denoiser_b200: a DECODER has three BatchNorm layers')
  return params, bns
end

-- library -> modules: parameters (weight, bias per module: the getParameters() order) and running statistics.  The
-- 2015 nn stores running_std = 1/sqrt(var + eps) instead of running_var; both forms are written as the module has them.
function M.copyToDecoder(net, decoder)
  local params, bns = walk(decoder)
  local flat, st = M.getParameters(net), M.getBNState(net)
  local o = 1
  for _, t in ipairs(params) do
    t:copy(flat:narrow(1, o, t:nElement()):viewAs(t))
    o = o + t:nElement()
  end
  assert(o - 1 == M.n, 'denoiser_b200: the DECODER does not match the denoiser at this image size')
  o = 1
  for _, m in ipairs(bns) do
    local c = m.running_mean:nElement()
    local mean, var = st:narrow(1, o, c), st:narrow(1, o + c, c)
    m.running_mean:copy(mean)
    if m.running_var then
      m.running_var:copy(var)
    else
      m.running_std:copy(var:clone():add(m.eps or 1e-5):sqrt():pow(-1))
    end
    o = o + 2 * c
  end
end
-- modules -> library (resuming from a saved denoiser)
function M.copyFromDecoder(net, decoder)
  local params, bns = walk(decoder)
  local parts, st = {}, {}
  for _, t in ipairs(params) do table.insert(parts, t:float():contiguous():view(-1)) end
  M.setParameters(net, torch.cat(parts, 1))
  for _, m in ipairs(bns) do
    table.insert(st, m.running_mean:float())
    if m.running_var then
      table.insert(st, m.running_var:float())
    else
      table.insert(st, m.running_std:float():clone():pow(-2):add(-(m.eps or 1e-5)))
    end
  end
  M.setBNState(net, torch.cat(st, 1))
end

function M.train(usedDataset)
  EPOCH = EPOCH or 1
  local N = usedDataset:size()
  local shuffle = torch.randperm(N)
  local sum1, sum2 = 0, 0
  local stats = ffi.new('fg_dn_stats[1]')
  for t = 1, N, OPT.batchSize do
    local thisBatchSize = math.min(OPT.batchSize, N - t + 1)
    -- BatchNorm needs two samples: a last batch of one image would fail in Torch as well, so it is skipped
    if thisBatchSize >= 2 then
      local inputs = torch.FloatTensor(thisBatchSize, IMG_DIMENSIONS[1], IMG_DIMENSIONS[2], IMG_DIMENSIONS[3])
      for i = 1, thisBatchSize do inputs[i] = usedDataset[shuffle[t + i - 1]] end
      M.step = M.step + 1
      F.check(C.fg_dn_train_step(M.dn, M.hyper, thisBatchSize, F.ptr(inputs), nil, nil, M.seedBase + M.step, stats),
              'fg_dn_train_step')
      sum1, sum2 = sum1 + stats[0].loss_AE1, sum2 + stats[0].loss_AE2
    end
  end
  print(string.format("<trainer> loss AE1 = %.4f", sum1 / (N / OPT.batchSize)))
  print(string.format("<trainer> loss AE2 = %.4f", sum2 / (N / OPT.batchSize)))
  EPOCH = EPOCH + 1
  return sum1 / (N / OPT.batchSize), sum2 / (N / OPT.batchSize)
end

return M
