-- adversarial_b200.lua -- drop-in for adversarial.lua's loop body (adversarial.lua:54-300): the whole
-- "OPT.D_iterations D iterations + OPT.G_iterations G iterations" (batch assembly excluded) is ONE call, fg_train_step
-- for 1 + 1 and fg_train_step_iters otherwise.  Keeps the globals
-- train.lua sets up (OPT, OPTSTATE, CONFUSION, NN_UTILS, IMG_DIMENSIONS) and the ADVERSARIAL.train signature.
-- Delivered untested-by-execution (no LuaJIT/Torch7 in the build image); face_generator_b200/adversarial.py
-- is the executable mirror.
require 'torch'
local ffi = require 'ffi'
local F = require 'fg_ffi'
require 'b200'
local C = F.C

local adversarial = {}
adversarial.accs = {}

-- data parallel: N copies of train.lua, one per GPU (INTEGRATION.md "Launching a Lua host on N GPUs").
-- FG_DP_WORLD / FG_DP_RANK / FG_DP_ID_FILE: rank 0 publishes the 128-byte NCCL id through a file.
local function dp_init(ctx)
  local world, rank, path = tonumber(os.getenv('FG_DP_WORLD') or '1'), tonumber(os.getenv('FG_DP_RANK') or '0'), os.getenv('FG_DP_ID_FILE')
  if world <= 1 then return end
  assert(path, 'FG_DP_ID_FILE must name the rendezvous file')
  local id = ffi.new('uint8_t[128]')
  if rank == 0 then
    F.check(C.fg_dp_unique_id(id), 'fg_dp_unique_id')
    local f = assert(io.open(path .. '.tmp', 'wb'))
    f:write(ffi.string(id, 128)); f:close()
    assert(os.rename(path .. '.tmp', path))
  else
    local data
    for _ = 1, 600 do                                     -- wait up to ~60 s for rank 0
      local f = io.open(path, 'rb')
      if f then data = f:read('*a'); f:close() end
      if data and #data == 128 then break end
      sys.sleep(0.1)
    end
    assert(data and #data == 128, 'rank 0 did not publish the NCCL id')
    ffi.copy(id, data, 128)
  end
  F.check(C.fg_dp_init(ctx, id, world, rank), 'fg_dp_init')
  F.check(C.fg_dp_broadcast_params(ctx), 'fg_dp_broadcast_params')
end

function adversarial.train(dataset, maxAccuracyD, accsInterval)
  EPOCH = EPOCH or 1
  local N_epoch = OPT.N_epoch
  if N_epoch <= 0 then N_epoch = dataset:size() end
  local dataBatchSize = OPT.batchSize / 2
  local ctx = b200.context(OPT.gpu, OPT.batchSize, IMG_DIMENSIONS[1])
  -- train.lua --scale 16: models.create_G / create_D built the 16x16 nets (models.lua:87-104); same loop, fg_s16_* entry points
  local s16 = IMG_DIMENSIONS[2] == 16 and b200.s16(ctx) or nil
  local hyper = b200.hyperFromOPT(OPT, OPTSTATE)
  hyper[0].D_maxAcc, hyper[0].accs_interval = maxAccuracyD, accsInterval
  -- the stock models' parameters (MODELS.create_* + NN_UTILS.initializeWeights, train.lua:134-138) are uploaded once;
  -- from then on the device copy is authoritative and written back at every checkpoint (below)
  if not adversarial.uploaded then
    if s16 then
      F.check(C.fg_s16_set_params(s16, F.NET_D, F.ptr(PARAMETERS_D)), 'fg_s16_set_params')
      F.check(C.fg_s16_set_params(s16, F.NET_G, F.ptr(PARAMETERS_G)), 'fg_s16_set_params')
    else
      F.check(C.fg_set_params(ctx, F.NET_D, F.ptr(PARAMETERS_D)), 'fg_set_params')
      F.check(C.fg_set_params(ctx, F.NET_G, F.ptr(PARAMETERS_G)), 'fg_set_params')
    end
    dp_init(ctx)                                          -- after the upload: rank 0's parameters win
    if s16 then F.check(C.fg_s16_dp_broadcast_params(s16), 'fg_s16_dp_broadcast_params') end
    adversarial.uploaded = true
  end
  local stats = ffi.new('fg_step_stats[1]')
  local time = sys.clock()
  local seed = (EPOCH - 1) * 1000000
  -- train.lua --D_iterations / --G_iterations (train.lua:33-34): D and G optimizer steps per batch, 1..16 each
  local dIters, gIters = OPT.D_iterations or 1, OPT.G_iterations or 1
  assert(dIters >= 1 and dIters <= 16 and gIters >= 1 and gIters <= 16, 'b200: --D_iterations / --G_iterations must lie in [1, 16]')
  for t = 1, N_epoch, dataBatchSize do
    local thisBatchSize = math.min(OPT.batchSize, N_epoch - t + 1)
    if thisBatchSize < 4 then break end                      -- adversarial.lua:73-76
    thisBatchSize = thisBatchSize - thisBatchSize % 2        -- even batches only (SURVEY appendix 13)
    local half = thisBatchSize / 2
    local dims = IMG_DIMENSIONS
    -- every D iteration draws its own real half-batch (1.1, adversarial.lua:244-249) and its own noise for the fakes
    -- (1.2, nn_utils.lua:35-39); every G iteration its own noise (2, :276); stacked per iteration
    local real = torch.FloatTensor(dIters, half, dims[1], dims[2], dims[3])
    local noiseD = torch.FloatTensor(dIters, half, 100)
    for j = 1, dIters do
      for i = 1, half do real[j][i] = dataset[math.random(dataset:size())] end
      noiseD[j]:copy(NN_UTILS.createNoiseInputs(half))
    end
    local noiseG = torch.FloatTensor(gIters, thisBatchSize, 100)
    for j = 1, gIters do noiseG[j]:copy(NN_UTILS.createNoiseInputs(thisBatchSize)) end
    seed = seed + 1
    if dIters == 1 and gIters == 1 then
      if s16 then
        F.check(C.fg_s16_train_step(s16, hyper, thisBatchSize, F.ptr(real), F.ptr(noiseD), F.ptr(noiseG), nil, nil, seed, stats), 'fg_s16_train_step')
      else
        F.check(C.fg_train_step(ctx, hyper, thisBatchSize, F.ptr(real), F.ptr(noiseD), F.ptr(noiseG), nil, nil, seed, stats), 'fg_train_step')
      end
    elseif s16 then
      F.check(C.fg_s16_train_step_iters(s16, hyper, thisBatchSize, dIters, gIters, F.ptr(real), F.ptr(noiseD), F.ptr(noiseG),
                                        nil, nil, seed, stats), 'fg_s16_train_step_iters')
    else
      F.check(C.fg_train_step_iters(ctx, hyper, thisBatchSize, dIters, gIters, F.ptr(real), F.ptr(noiseD), F.ptr(noiseG),
                                    nil, nil, seed, stats), 'fg_train_step_iters')
    end
    local s = stats[0]
    -- feed optim.ConfusionMatrix exactly like adversarial.lua:112-117 (rows = predicted class, cols = target); conf
    -- sums over the call's D iterations, as CONFUSION:add does once per fevalD
    CONFUSION.mat[2][2] = CONFUSION.mat[2][2] + s.conf[0]
    CONFUSION.mat[1][2] = CONFUSION.mat[1][2] + s.conf[1]
    CONFUSION.mat[2][1] = CONFUSION.mat[2][1] + s.conf[2]
    CONFUSION.mat[1][1] = CONFUSION.mat[1][1] + s.conf[3]
    -- the optimizer state tables keep their step counters (interruptable_optimizers.lua:78, :29, :123)
    local stD, stG = OPTSTATE[OPT.D_optmethod or 'adam'].D, OPTSTATE[OPT.G_optmethod or 'adam'].G
    if (OPT.D_optmethod or 'adam') == 'adam' then stD.t = s.t_D else stD.evalCounter = s.t_D end
    if (OPT.G_optmethod or 'adam') == 'adam' then stG.t = s.t_G else stG.evalCounter = s.t_G end
    xlua.progress(t + thisBatchSize, N_epoch)
  end
  time = sys.clock() - time
  print(string.format("<trainer> time to learn 1 sample = %f ms", 1000 * time / N_epoch))
  print(CONFUSION)
  CONFUSION:updateValids()
  local tV = CONFUSION.totalValid                                      -- adversarial.lua:316
  CONFUSION:zero()
  -- the live device parameters are copied back into the flat tensors train.lua:151-152 obtained from
  -- MODEL_x:getParameters() at the end of every epoch (20 MB), so MODEL_D / MODEL_G -- which train.lua's plotting
  -- (NN_UTILS.visualizeProgress, train.lua:204) and the save sequence below use -- hold the trained weights
  if s16 then
    F.check(C.fg_s16_get_params(s16, F.NET_D, F.ptr(PARAMETERS_D)), 'fg_s16_get_params')
    F.check(C.fg_s16_get_params(s16, F.NET_G, F.ptr(PARAMETERS_G)), 'fg_s16_get_params')
  else
    F.check(C.fg_get_params(ctx, F.NET_D, F.ptr(PARAMETERS_D)), 'fg_get_params')
    F.check(C.fg_get_params(ctx, F.NET_G, F.ptr(PARAMETERS_G)), 'fg_get_params')
  end
  -- checkpoint every OPT.saveFreq epochs: the reference's own sequence (adversarial.lua:319-329)
  if EPOCH % OPT.saveFreq == 0 then
    local filename = paths.concat(OPT.save, 'adversarial.net')
    os.execute(string.format("mkdir -p %s", sys.dirname(filename)))
    if paths.filep(filename) then os.execute(string.format("mv %s %s.old", filename, filename)) end
    print(string.format("<trainer> saving network to %s", filename))
    NN_UTILS.prepareNetworkForSave(MODEL_D)
    NN_UTILS.prepareNetworkForSave(MODEL_G)
    torch.save(filename, {D = MODEL_D, G = MODEL_G, opt = OPT, epoch = EPOCH})
  end
  EPOCH = EPOCH + 1
  return tV                                                            -- adversarial.lua:334
end

return adversarial
