-- autoencoder_b200.lua -- drop-in for train_autoencoder.lua: MODEL_AE trains in the library, every batch is ONE
-- fg_ae_train_step (fevalAE + optim.adam with the script's empty config).  Keeps the script's globals (OPT, EPOCH) and
-- adds the layer shims b200.ReLU, b200.Tanh, b200.AbsCriterion and the net shim b200.Autoencoder.
--
-- The net trains in the library, so MODEL_AE's Torch modules never run: M.copyToModel(MODEL_AE) writes the trained
-- parameters into them (before torch.save, :234), M.copyFromModel(MODEL_AE) reads them back (after a load).
-- Delivered untested-by-execution (no LuaJIT/Torch7 in the build image); face_generator_b200/autoencoder.py is the
-- executable mirror.
require 'torch'
require 'nn'
local ffi = require 'ffi'
local F = require 'fg_ffi'
require 'b200'
local C = F.C

local M = {}

function M.init()
  local ctx = b200.context(OPT.gpu or 0, OPT.batchSize, 1)  -- OPT.geometry = {1, scale, scale} (:57)
  local out = ffi.new('fg_ae*[1]')
  F.check(C.fg_ae_create(ctx, OPT.scale, OPT.noiseDim, out), 'fg_ae_create')
  M.ae = ffi.gc(out[0], C.fg_ae_destroy)
  M.hyper = ffi.new('fg_ae_hyper[1]')
  C.fg_ae_hyper_default(M.hyper)
  M.hyper[0].L1, M.hyper[0].L2 = OPT.coefL1, OPT.coefL2
  M.n = tonumber(C.fg_ae_param_count(OPT.scale, OPT.noiseDim))
  -- the step seed: --seed selects the dropout stream, the batch counter advances it
  M.seedBase = (OPT.seed or 1) * 2 ^ 32
  M.step = 0
  return M
end

-- flat getParameters() vector (PARAMETERS_AE)
function M.setParameters(flat)
  assert(flat:nElement() == M.n, 'autoencoder_b200: MODEL_AE does not match this --scale / --noiseDim')
  F.check(C.fg_ae_set_params(M.ae, F.ptr(flat:float():contiguous())), 'fg_ae_set_params')
end
function M.getParameters()
  local p = torch.FloatTensor(M.n)
  F.check(C.fg_ae_get_params(M.ae, F.ptr(p)), 'fg_ae_get_params')
  return p
end
function M.copyFromModel(model) M.setParameters(model:getParameters()) end
function M.copyToModel(model) model:getParameters():copy(M.getParameters()) end

-- train() of the script (:148-239) without its save block: the caller copies the parameters out and saves
function M.train(usedDataset)
  EPOCH = EPOCH or 1
  local N = usedDataset:size()
  local shuffle = torch.randperm(N)
  local sum, batches = 0, 0
  local stats = ffi.new('fg_ae_stats[1]')
  for t = 1, N, OPT.batchSize do
    local thisBatchSize = math.min(OPT.batchSize, N - t + 1)
    local inputs = torch.FloatTensor(thisBatchSize, 1, OPT.scale, OPT.scale)
    for i = 1, thisBatchSize do inputs[i] = usedDataset[shuffle[t + i - 1]] end
    M.step = M.step + 1
    F.check(C.fg_ae_train_step(M.ae, M.hyper, thisBatchSize, F.ptr(inputs), nil, M.seedBase + M.step, stats), 'fg_ae_train_step')
    sum, batches = sum + stats[0].loss, batches + 1
  end
  print(string.format("<trainer> loss = %.4f", sum / batches))
  EPOCH = EPOCH + 1
  return sum / batches
end

-- getSamples (:137-145): the script forwards without evaluate(), so Dropout stays live (training = 1)
function M.getSamples(dataset, N)
  local images = torch.FloatTensor(N, 1, OPT.scale, OPT.scale)
  for i = 1, N do images[i] = dataset[i] end
  local decoded = torch.FloatTensor(N, 1, OPT.scale, OPT.scale)
  F.check(C.fg_ae_reconstruct(M.ae, F.ptr(images), N, math.min(N, OPT.batchSize), 1, M.seedBase + M.step, F.ptr(decoded)),
          'fg_ae_reconstruct')
  return {images, decoded}
end

-- ---- layer shims (FloatTensors or CudaTensors, as their neighbours in b200.lua) ----
local function unary(name, fwd, bwd, from_output)
  local cls, parent = torch.class('b200.' .. name, 'nn.Module')
  function cls:__init() parent.__init(self); self.ctx = b200.context() end
  function cls:updateOutput(input)
    input = input:contiguous()
    self.output:resizeAs(input)
    F.check(C[fwd](self.ctx, F.ptr(input), F.ptr(self.output), input:nElement()), fwd)
    return self.output
  end
  function cls:updateGradInput(input, gradOutput)
    self.gradInput:resizeAs(input)
    local from = from_output and self.output or input:contiguous()
    F.check(C[bwd](self.ctx, F.ptr(from), F.ptr(gradOutput:contiguous()), F.ptr(self.gradInput), input:nElement()), bwd)
    return self.gradInput
  end
end
unary('ReLU', 'fg_relu_forward', 'fg_relu_backward', false)  -- train_autoencoder.lua:84,89
unary('Tanh', 'fg_tanh_forward', 'fg_tanh_backward', true)   -- :86

local Abs, aparent = torch.class('b200.AbsCriterion', 'nn.Criterion')  -- :98
function Abs:__init() aparent.__init(self); self.ctx = b200.context() end
function Abs:updateOutput(input, target)
  local out = torch.FloatTensor(1)
  F.check(C.fg_abs_forward(self.ctx, F.ptr(input:contiguous()), F.ptr(target:contiguous()), input:nElement(), F.ptr(out)), 'fg_abs_forward')
  self.output = out[1]
  return self.output
end
function Abs:updateGradInput(input, target)
  self.gradInput:resizeAs(input)
  F.check(C.fg_abs_backward(self.ctx, F.ptr(input:contiguous()), F.ptr(target:contiguous()), input:nElement(), F.ptr(self.gradInput)), 'fg_abs_backward')
  return self.gradInput
end

-- MODEL_AE as one module: forward = fg_ae_forward (training-mode until :evaluate()), backward = fg_ae_backward into the
-- library's gradient buffer
local AE, eparent = torch.class('b200.Autoencoder', 'nn.Module')
function AE:__init(scale, noiseDim)
  eparent.__init(self)
  self.ctx = b200.context()
  self.S, self.d, self.train, self.seed = scale, noiseDim, true, 0
  local out = ffi.new('fg_ae*[1]')
  F.check(C.fg_ae_create(self.ctx, scale, noiseDim, out), 'fg_ae_create')
  self.ae = ffi.gc(out[0], C.fg_ae_destroy)
  self.output, self.code = torch.FloatTensor(), torch.FloatTensor()
end
function AE:training() self.train = true; return self end
function AE:evaluate() self.train = false; return self end
function AE:updateOutput(input)
  input = input:float():contiguous()
  local B = input:size(1)
  self.output:resize(B, 1, self.S, self.S)
  self.code:resize(B, self.d)
  self.seed = self.seed + 1
  F.check(C.fg_ae_forward(self.ae, F.ptr(input), B, self.train and 1 or 0, nil, self.seed, F.ptr(self.code), F.ptr(self.output)),
          'fg_ae_forward')
  return self.output
end
function AE:backward(input, gradOutput)
  F.check(C.fg_ae_backward(self.ae, F.ptr(gradOutput:float():contiguous())), 'fg_ae_backward')
end
function AE:zeroGradParameters() F.check(C.fg_ae_zero_grads(self.ae), 'fg_ae_zero_grads') end

return M
