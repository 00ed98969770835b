-- adversarial_c2f_b200.lua -- drop-in for adversarial_c2f.lua's loop body (adversarial_c2f.lua:121-187): the
-- "OPT.D_iterations D iterations + OPT.G_iterations G iterations" of the coarse-to-fine GAN are ONE call
-- (fg_c2f_train_step for 1 + 1, fg_c2f_train_step_iters otherwise).  Keeps the globals
-- train_c2f.lua sets up (OPT, OPTSTATE, CONFUSION, IMG_DIMENSIONS, NOISE_DIM, COND_DIM) and the
-- adversarial.train(trainData) signature; batch assembly (random {diff, coarse} pairs, adversarial_c2f.lua:124-141,
-- :168-174) stays in Lua exactly as in the reference.
-- Delivered untested-by-execution (no LuaJIT/Torch7 in the build image); face_generator_b200/adversarial_c2f.py
-- is the executable mirror and tests/test_c2f.py drives the same C calls through ctypes.
require 'torch'
local ffi = require 'ffi'
local F = require 'fg_ffi'
require 'b200'
local C = F.C

local adversarial = {}
local net = nil   -- fg_c2f*, created on first use, parameters uploaded from PARAMETERS_G / PARAMETERS_D

local function c2f(ctx)
  if net == nil then
    -- train_c2f.lua --fineSize (16, 32 or 64) sizes both nets; IMG_DIMENSIONS / NOISE_DIM / COND_DIM follow it.
    -- MODEL_G / MODEL_D may be any of models_c2f.lua's nets (models_c2f.create_G / create_D); the flat vectors are
    -- already in getParameters() order (train_c2f.lua:131-132) and are checked against the recognised nets' lengths
    net = b200.c2fNets(ctx, MODEL_G, MODEL_D, PARAMETERS_G, PARAMETERS_D, OPT.fineSize, IMG_DIMENSIONS[1])
  end
  return net
end

function adversarial.train(trainData)
  EPOCH = EPOCH or 1
  local N_epoch = OPT.N_epoch
  if N_epoch <= 0 then N_epoch = trainData:size() end
  local dataBatchSize = OPT.batchSize / 2
  local ctx = b200.context(OPT.gpu, OPT.batchSize, IMG_DIMENSIONS[1])
  local n = c2f(ctx)
  local hyper = b200.hyperFromOPT(OPT, OPTSTATE)
  local stats = ffi.new('fg_step_stats[1]')
  local time = sys.clock()
  local seed = (EPOCH - 1) * 1000000
  local dims = IMG_DIMENSIONS
  -- train_c2f.lua --D_iterations / --G_iterations (train_c2f.lua:31-32): 1..16 each
  local dIters, gIters = OPT.D_iterations or 1, OPT.G_iterations or 1
  assert(dIters >= 1 and dIters <= 16 and gIters >= 1 and gIters <= 16, 'b200: --D_iterations / --G_iterations must lie in [1, 16]')
  for t = 1, N_epoch, dataBatchSize do
    local B = math.min(OPT.batchSize, N_epoch - t + 1)
    if B < 4 then break end                                  -- adversarial_c2f.lua:33-36
    B = B - B % 2
    local half = B / 2
    -- every D iteration draws its own pairs, coarse images and noise, every G iteration its own coarse images and
    -- noise (the reference's fevalD / fevalG_on_D draws, once per iteration); stacked per iteration
    local realDiff = torch.FloatTensor(dIters, half, dims[1], dims[2], dims[3])
    local condD = torch.FloatTensor(dIters, B, COND_DIM[1], COND_DIM[2], COND_DIM[3])
    local noiseD = torch.FloatTensor(dIters, half, NOISE_DIM[1], NOISE_DIM[2], NOISE_DIM[3])
    local condG = torch.FloatTensor(gIters, B, COND_DIM[1], COND_DIM[2], COND_DIM[3])
    local noiseG = torch.FloatTensor(gIters, B, NOISE_DIM[1], NOISE_DIM[2], NOISE_DIM[3])
    for j = 1, dIters do
      for i = 1, half do                                     -- (1.1) real pairs, :124-132
        local ex = trainData[math.random(trainData:size())]
        realDiff[j][i] = ex.diff
        condD[j][i] = ex.coarse
      end
      for i = half + 1, B do                                 -- (1.2) coarse images for the generated half, :136-141
        condD[j][i] = trainData[math.random(trainData:size())].coarse
      end
      noiseD[j]:uniform(-1, 1)
    end
    for j = 1, gIters do
      for i = 1, B do                                        -- (2) fresh coarse images for the G step, :170-174
        condG[j][i] = trainData[math.random(trainData:size())].coarse
      end
      noiseG[j]:uniform(-1, 1)
    end
    seed = seed + 1
    if dIters == 1 and gIters == 1 then
      F.check(C.fg_c2f_train_step(n, hyper, B, F.ptr(realDiff), F.ptr(condD), F.ptr(noiseD), F.ptr(condG), F.ptr(noiseG),
                                  nil, nil, seed, stats), 'fg_c2f_train_step')
    else
      F.check(C.fg_c2f_train_step_iters(n, hyper, B, dIters, gIters, F.ptr(realDiff), F.ptr(condD), F.ptr(noiseD),
                                        F.ptr(condG), F.ptr(noiseG), nil, nil, seed, stats), 'fg_c2f_train_step_iters')
    end
    local s = stats[0]
    CONFUSION.mat[2][2] = CONFUSION.mat[2][2] + s.conf[0]    -- adversarial_c2f.lua:66-70
    CONFUSION.mat[1][2] = CONFUSION.mat[1][2] + s.conf[1]
    CONFUSION.mat[2][1] = CONFUSION.mat[2][1] + s.conf[2]
    CONFUSION.mat[1][1] = CONFUSION.mat[1][1] + s.conf[3]
    OPTSTATE.adam.D.t, OPTSTATE.adam.G.t = s.t_D, s.t_G
    xlua.progress(t + B, N_epoch)
  end
  -- hand the trained parameters back to the Torch modules (for torch.save / plotting, adversarial_c2f.lua:200-230)
  F.check(C.fg_c2f_get_params(n, 0, F.ptr(PARAMETERS_G)), 'fg_c2f_get_params(G)')
  F.check(C.fg_c2f_get_params(n, 1, F.ptr(PARAMETERS_D)), 'fg_c2f_get_params(D)')
  time = sys.clock() - time
  print(string.format("<trainer> time required for this epoch = %d s", time))
  print(string.format("<trainer> time to learn 1 sample = %f ms", 1000 * time / N_epoch))
  print("Confusion of D:")
  print(CONFUSION)
  CONFUSION:zero()
  EPOCH = EPOCH + 1
end

return adversarial
