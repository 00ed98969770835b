-- b200.lua -- nn.Module shims over libfg_b200.so so that train.lua / adversarial.lua / sample.lua keep their
-- plugin surface (SURVEY.md 8b):  MODEL:forward/backward, MODEL.modules[1].gradInput, MODEL:getParameters(),
-- :training()/:evaluate(), CRITERION:forward/backward, interruptableAdam(opfunc, x, config).
-- Delivered untested-by-execution (no LuaJIT/Torch7 in the build image); face_generator_b200/nn.py is the
-- executable mirror and tests/test_gpu_parity.py::test_modules_equal_fused_step exercises the same call order.
require 'nn'
local ffi = require 'ffi'
local F = require 'fg_ffi'
local C = F.C

b200 = b200 or {}

-- models.lua's discriminators by the name of the function that builds them (FG_DISC_*, include/fg_b200.h)
b200.DISCRIMINATORS = {create_D32b = 1, create_D16_d = 2, create_D32 = 3, create_D16 = 4, create_D16_b = 5,
                       create_D16_c = 6}
local function disc_id(name, default)
  local d = b200.DISCRIMINATORS[name or default]
  assert(d, 'unknown discriminator ' .. tostring(name))
  return d
end

-- models_c2f.lua's nets by the name of the function that builds them (FG_C2F_G_* / FG_C2F_D_*, include/fg_b200.h):
-- G's "same" SpatialConvolutionUpsample layers {planes out, kernel} after the C+1 joined planes (0 = the C image
-- channels), D's 3x3 convolutions {planes out, 2x2 max pool after}
b200.C2F_GENERATORS = {
  create_G_d = {id = 1, layers = {{64, 3}, {64, 3}, {128, 5}, {256, 5}, {0, 7}}},
  create_G_a = {id = 2, layers = {{64, 3}, {128, 7}, {0, 5}}},
  create_G_b = {id = 3, layers = {{64, 3}, {64, 3}, {256, 5}, {0, 7}}},
  create_G_c = {id = 4, layers = {{64, 3}, {128, 3}, {256, 5}, {0, 7}}},
}
b200.C2F_DISCRIMINATORS = {
  create_D_c = {id = 1, layers = {{64, false}, {64, true}, {128, false}, {256, true}}},
  create_D_a = {id = 2, layers = {{64, false}, {64, true}}},
  create_D_b = {id = 3, layers = {{64, false}, {64, true}, {128, false}, {128, true}}},
}

-- the convolutions of a module tree in module order, {planes out, planes in, kernel width, max pool after}; the
-- CUDA-mode nn.Copy layers and every other leaf are skipped
local function c2f_convs(net)
  local convs = {}
  local function walk(m)
    if m.modules then
      for _, child in ipairs(m.modules) do walk(child) end
      return
    end
    local t = torch.type(m)
    if t:find('Convolution') then
      table.insert(convs, {m.nOutputPlane, m.nInputPlane, m.kW, false})
    elseif t:find('SpatialMaxPooling') and #convs > 0 then
      convs[#convs][4] = true
    end
  end
  walk(net)
  return convs
end

local function c2f_describe(convs)
  local parts = {}
  for _, c in ipairs(convs) do
    table.insert(parts, string.format('%d->%d %dx%d%s', c[2], c[1], c[3], c[3], c[4] and ' pool' or ''))
  end
  return #parts > 0 and table.concat(parts, ', ') or 'none'
end

-- the entry of `nets` (C2F_GENERATORS or C2F_DISCRIMINATORS) whose layers the convolutions are, for `channels`
-- image channels: name, FG_C2F_* id
local function c2f_recognise(convs, channels, nets, isG)
  for name, e in pairs(nets) do
    if #e.layers == #convs then
      local ok, cin = true, isG and channels + 1 or channels
      for i, l in ipairs(e.layers) do
        local cout = (isG and l[1] == 0) and channels or l[1]
        local k, pool = isG and l[2] or 3, (not isG) and l[2] or false
        local c = convs[i]
        if c[1] ~= cout or c[2] ~= cin or c[3] ~= k or c[4] ~= pool then
          ok = false
          break
        end
        cin = cout
      end
      if ok then return name, e.id end
    end
  end
  return nil
end

-- the fg_c2f for the models_c2f.lua nets G and D (recognised from their convolutions' kernel sizes and plane counts)
-- at fineSize on ctx, with their flat parameter vectors pG / pD (G:getParameters() order) uploaded.  A net that is
-- none of models_c2f.lua's, or a vector of another length, is refused before anything is copied.
function b200.c2fNets(ctx, G, D, pG, pD, fineSize, channels)
  local gc, dc = c2f_convs(G), c2f_convs(D)
  local gName, gId = c2f_recognise(gc, channels, b200.C2F_GENERATORS, true)
  assert(gName, 'b200: G is not one of models_c2f.lua\'s generators for ' .. channels .. ' channels; its convolutions: '
         .. c2f_describe(gc))
  local dName, dId = c2f_recognise(dc, channels, b200.C2F_DISCRIMINATORS, false)
  assert(dName, 'b200: D is not one of models_c2f.lua\'s discriminators for ' .. channels .. ' channels; its convolutions: '
         .. c2f_describe(dc))
  local nG = tonumber(C.fg_c2f_gen_param_count(gId, channels))
  local nD = tonumber(C.fg_c2f_disc_param_count(dId, channels, fineSize))
  assert(nD >= 0, 'b200: fine size ' .. tostring(fineSize) .. ' is not supported (16, 32 or 64)')
  assert(pG:nElement() == nG, string.format('b200: G (%s) has %d parameters, the c2f net expects %d', gName,
                                            pG:nElement(), nG))
  assert(pD:nElement() == nD, string.format('b200: D (%s) has %d parameters, %s at fine size %d expects %d', dName,
                                            pD:nElement(), dName, fineSize, nD))
  local out = ffi.new('fg_c2f*[1]')
  F.check(C.fg_c2f_create_nets(ctx, fineSize, gId, dId, out), 'fg_c2f_create_nets')
  local net = out[0]
  for i, p in ipairs({pG, pD}) do
    local rc = C.fg_c2f_set_params(net, i - 1, F.ptr(p))
    if rc ~= 0 then
      local msg = ffi.string(C.fg_last_error())
      C.fg_c2f_destroy(net)   -- a failed upload leaves no half-initialised net behind
      error(string.format('fg_c2f_set_params(%s) failed (%d): %s', i == 1 and 'G' or 'D', rc, msg))
    end
  end
  return net, gName, dName
end

-- one context per process/GPU, created lazily from OPT (train.lua:16-50); discriminator: 'create_D32b' (default)
-- or 'create_D32'
function b200.context(device, maxBatch, channels, discriminator)
  if not b200._ctx then
    local out = ffi.new('fg_ctx*[1]')
    F.check(C.fg_create_disc(out, device or 0, maxBatch or 256, channels or 3, disc_id(discriminator, 'create_D32b')),
            'fg_create_disc')
    b200._ctx = ffi.gc(out[0], C.fg_destroy)
    b200._hyper = ffi.new('fg_hyper[1]')
    C.fg_hyper_default(b200._hyper)
  end
  return b200._ctx
end

-- the --scale 16 nets (models.lua:87-104 pick create_G_decoder_upsampling16 / create_D16_d for 16x16 images);
-- discriminator: 'create_D16_d' (default), 'create_D16', 'create_D16_b' or 'create_D16_c'
function b200.s16(ctx, discriminator)
  if not b200._s16 then
    local out = ffi.new('fg_s16*[1]')
    F.check(C.fg_s16_create_disc(ctx, disc_id(discriminator, 'create_D16_d'), out), 'fg_s16_create_disc')
    b200._s16 = ffi.gc(out[0], C.fg_s16_destroy)
  end
  return b200._s16
end

-- hyper-parameters from the reference's OPT / OPTSTATE tables; also selects the optimizer the fused step runs
-- (OPT.D_optmethod / OPT.G_optmethod, train.lua:38-39; adversarial.lua:259-266, :279-286)
local OPTMETHOD = {adam = 0, adagrad = 1, sgd = 2}
function b200.hyperFromOPT(OPT, OPTSTATE)
  local h = b200._hyper[0]
  h.D_L1, h.D_L2, h.G_L1, h.G_L2 = OPT.D_L1, OPT.D_L2, OPT.G_L1, OPT.G_L2
  h.D_clamp, h.G_clamp, h.D_maxAcc = OPT.D_clamp, OPT.G_clamp, OPT.D_maxAcc
  for _, net in ipairs({'D', 'G'}) do
    local method = OPT[net .. '_optmethod'] or 'adam'
    assert(OPTMETHOD[method], 'b200: unknown optimizer method ' .. tostring(method))
    F.check(C.fg_set_option(b200._ctx, 'optimizer_' .. net, OPTMETHOD[method]), 'fg_set_option')
    local st = OPTSTATE and OPTSTATE[method] and OPTSTATE[method][net] or {}
    -- adam: learningRate or 1e-3 (interruptable_optimizers.lua:53); adagrad: 1e-3 (:10); sgd: OPT.*_SGD_lr (train.lua:180-191)
    h['lr_' .. net] = st.learningRate or 1e-3
    if method == 'sgd' then
      F.check(C.fg_set_option_f(b200._ctx, 'sgd_momentum_' .. net, st.momentum or 0), 'fg_set_option_f')
    end
  end
  return b200._hyper
end

-- a CudaTensor over raw device memory: torch.CudaStorage(size, address) wraps existing memory without owning it
-- ([3P] cutorch shares torch7's generic/Storage.c constructor `Storage(size, ptr)`)
function b200.aliasCuda(ptr, n)
  local addr = tonumber(ffi.cast('intptr_t', ptr))
  return torch.CudaTensor(torch.CudaStorage(n, addr))
end
local function devptr(t) return ffi.cast('float*', t:data()) end

---------------------------------------------------------------------------------------------------------------
-- Fused networks.  train.lua / adversarial.lua stay UNMODIFIED when MODELS.create_G / create_D return these
-- (INTEGRATION.md section 2); face_generator_b200/nn.py is the executable mirror, tests/test_gpu_lnet_dropin.py
-- runs the transcribed reference flow through it.  What the reference does to a model, and how this class answers:
--   NN_UTILS.initializeWeights(model)  walks model.modules[m].weight/.bias (nn_utils.lua:17-29)
--        -> self.modules = one proxy per reference layer, weight/bias = views into the flat device vector
--   NN_UTILS.activateCuda(model)       net:clone(), :cuda(), wrapped into Sequential{Copy, net, Copy} (:328-363)
--        -> clone() returns self (one fused net per context), type()/cuda() are no-ops, CudaTensor in / out
--   MODEL:getParameters()              stock Module.flatten on the wrapping Sequential (train.lua:151-152): allocates
--        ONE new flat storage, copies, re-points self.weight / self.gradWeight at it
--        -> sync() sees weight:data() change and passes the new pointers to fg_bind_params: PARAMETERS_x /
--           GRAD_PARAMETERS_x (zeroed, penalised, clamped by adversarial.lua:92-123, updated in place by the stock
--           interruptable optimizers) then ARE the buffers the kernels read and write
--   MODEL_D.modules[1].gradInput       is the leading nn.Copy's gradInput (adversarial.lua:210): stock nn
--   torch.save({D = MODEL_D, ...})     write()/read() serialise the flat parameters + BN statistics
---------------------------------------------------------------------------------------------------------------
local Fused, parent = torch.class('b200.Fused', 'nn.Module')

function Fused:__init(net, channels, layers)
  parent.__init(self)
  self.net, self.channels, self.layers = net, channels, layers
  self:attach()
end
function Fused:attach()
  self.ctx = b200.context()
  -- D's length follows the discriminator the context holds (fg_create_disc), G's is fixed
  self.n = self.net == F.NET_D and tonumber(C.fg_disc_param_count(C.fg_get_disc(self.ctx), self.channels))
           or tonumber(C.fg_param_count(self.net, self.channels))
  self.train = true
  self.output, self.gradInput = torch.CudaTensor(), torch.CudaTensor()
  self.weight = b200.aliasCuda(C.fg_params_ptr(self.ctx, self.net), self.n)
  self.gradWeight = b200.aliasCuda(C.fg_grads_ptr(self.ctx, self.net), self.n)
  self._w, self._g = devptr(self.weight), devptr(self.gradWeight)
  self:views()
end
-- per-layer proxies in models.lua's module order; flat offsets follow getParameters() (weight, then bias)
function Fused:views()
  self.modules = {}
  local o = 1
  local function view(shape)
    local cnt = 1
    for _, d in ipairs(shape) do cnt = cnt * d end
    local w, g = self.weight:narrow(1, o, cnt):view(unpack(shape)), self.gradWeight:narrow(1, o, cnt):view(unpack(shape))
    o = o + cnt
    return w, g
  end
  for i, L in ipairs(self.layers) do
    local m = {typename = L[1]}
    if L[2] then m.weight, m.gradWeight = view(L[2]) end
    if L[3] then m.bias, m.gradBias = view(L[3]) end
    self.modules[i] = m
  end
  assert(o == self.n + 1)
end
function Fused:sync()
  local w, g = devptr(self.weight), devptr(self.gradWeight)
  if w ~= self._w or g ~= self._g then       -- Module.flatten moved us into the caller's flat storage
    F.check(C.fg_bind_params(self.ctx, self.net, w, g), 'fg_bind_params')
    self._w, self._g = w, g
    self:views()
  end
  F.check(C.fg_set_stream(self.ctx, cutorch.getStream and ffi.cast('void*', cutorch.getStream()) or nil), 'fg_set_stream')
end
function Fused:training() self.train = true; return self end
function Fused:evaluate() self.train = false; return self end
function Fused:type() return self end        -- :cuda() / :float(): the parameters live on the device
function Fused:clone() return self end       -- NN_UTILS.activateCuda (nn_utils.lua:352)
function Fused:listModules() return {self} end
function Fused:parameters() return {self.weight}, {self.gradWeight} end
function Fused:zeroGradParameters() self:sync(); F.check(C.fg_zero_grads(self.ctx, self.net), 'fg_zero_grads') end
function Fused:accGradParameters() end       -- folded into backward()
-- torch.save / torch.load (adversarial.lua:319-329): flat parameters (+ G's BatchNorm running statistics)
function Fused:write(file)
  local p = torch.FloatTensor(self.n)
  self:sync()
  F.check(C.fg_sync(self.ctx), 'fg_sync')
  p:copy(self.weight)
  local bn = torch.FloatTensor(768)
  F.check(C.fg_get_bn_state(self.ctx, F.ptr(bn)), 'fg_get_bn_state')
  file:writeObject({net = self.net, channels = self.channels, layers = self.layers, params = p, bn = bn, train = self.train})
end
function Fused:read(file)
  local t = file:readObject()
  self.net, self.channels, self.layers = t.net, t.channels, t.layers
  b200.context(nil, nil, t.channels)
  self:attach()
  self.train = t.train
  self.weight:copy(t.params)
  if self.net == F.NET_G then F.check(C.fg_set_bn_state(self.ctx, F.ptr(t.bn)), 'fg_set_bn_state') end
end

-- MODELS.create_G(dimensions, noiseDim)  (models.lua:87-93 -> create_G_decoder_upsampling32 :57-81)
local FusedG = torch.class('b200.FusedG', 'b200.Fused')
function FusedG:__init(dimensions, noiseDim)
  assert(noiseDim == 100 and dimensions[2] == 32, 'b200.FusedG implements create_G_decoder_upsampling32 with noiseDim 100')
  local c = dimensions[1]
  b200.Fused.__init(self, F.NET_G, c, {
    {'nn.Linear', {8192, 100}, {8192}}, {'nn.View'}, {'nn.PReLU', {1}}, {'nn.SpatialUpSamplingNearest'},
    {'cudnn.SpatialConvolution', {256, 128, 5, 5}, {256}}, {'nn.SpatialBatchNormalization', {256}, {256}}, {'nn.PReLU', {1}},
    {'nn.SpatialUpSamplingNearest'}, {'cudnn.SpatialConvolution', {128, 256, 5, 5}, {128}},
    {'nn.SpatialBatchNormalization', {128}, {128}}, {'nn.PReLU', {1}}, {'cudnn.SpatialConvolution', {c, 128, 3, 3}, {c}},
    {'nn.Sigmoid'}})
end
function FusedG:updateOutput(input)
  self:sync()
  local B = input:size(1)
  self.output:resize(B, self.channels, 32, 32)
  F.check(C.fg_G_forward(self.ctx, F.ptr(input:contiguous()), B, self.train and 1 or 0, F.ptr(self.output)), 'fg_G_forward')
  return self.output
end
function FusedG:backward(input, gradOutput)  -- updateGradInput + accGradParameters in one call
  self:sync()
  self.gradInput:resizeAs(input)
  F.check(C.fg_G_backward(self.ctx, F.ptr(gradOutput:contiguous()), F.ptr(self.gradInput)), 'fg_G_backward')
  return self.gradInput
end
FusedG.updateGradInput = FusedG.backward

-- MODELS.create_D(dimensions)  (models.lua:98-104 -> create_D32b :382-416), or with `name` another 32x32
-- discriminator of models.lua ('create_D32', :322-376).  The context is created with that D when this is its first
-- use; a context that already holds another D is refused, naming both.  The proxies list the parameterised leaves
-- in module order through the ConcatTable, which is getParameters() order.
local function d32b_layers(c)
  local layers, cin = {}, c
  for _, cout in ipairs({64, 128, 256, 512}) do
    for _, L in ipairs({{'nn.SpatialConvolution', {cout, cin, 3, 3}, {cout}}, {'nn.PReLU', {1}}, {'nn.SpatialDropout'},
                        {'nn.SpatialAveragePooling'}}) do layers[#layers + 1] = L end
    cin = cout
  end
  for _, L in ipairs({{'nn.View'}, {'nn.Linear', {512, 2048}, {512}}, {'nn.PReLU', {1}}, {'nn.Dropout'},
                      {'nn.Linear', {512, 512}, {512}}, {'nn.PReLU', {1}}, {'nn.Dropout'}, {'nn.Linear', {1, 512}, {1}},
                      {'nn.Sigmoid'}}) do layers[#layers + 1] = L end
  return layers
end
local function d32_layers(c)
  local conv = function(o, i, k) return {'nn.SpatialConvolution', {o, i, k, k}, {o}} end
  local lin = function(o, i) return {'nn.Linear', {o, i}, {o}} end
  local P = {'nn.PReLU', {1}}
  return {
    -- fine branch
    conv(64, c, 3), P, conv(64, 64, 3), P, {'nn.SpatialMaxPooling'}, {'nn.SpatialDropout'}, {'nn.View'}, lin(1024, 16384), P,
    -- coarse branch
    conv(32, c, 5), P, conv(32, 32, 5), P, {'nn.SpatialMaxPooling'}, conv(54, 32, 5), P, conv(54, 54, 5), P,
    {'nn.SpatialMaxPooling'}, {'nn.SpatialDropout'}, {'nn.View'}, lin(1024, 3456), P, {'nn.Dropout'}, lin(1024, 1024), P,
    -- dense branch
    {'nn.View'}, lin(1024, c * 1024), P, {'nn.Dropout'}, lin(1024, 1024), P,
    -- head
    {'nn.JoinTable'}, lin(1024, 3072), P, {'nn.Dropout'}, lin(1, 1024), {'nn.Sigmoid'}}
end
local D32_LAYERS = {create_D32b = d32b_layers, create_D32 = d32_layers}
local FusedD = torch.class('b200.FusedD', 'b200.Fused')
function FusedD:__init(dimensions, name)
  name = name or 'create_D32b'
  assert(dimensions[2] == 32 and D32_LAYERS[name], 'b200.FusedD implements create_D32b and create_D32 (32x32), not '
         .. tostring(name) .. ' at ' .. tostring(dimensions[2]))
  local ctx = b200.context(nil, nil, dimensions[1], name)
  local held = C.fg_get_disc(ctx)
  if held ~= disc_id(name) then
    local have = '?'
    for k, v in pairs(b200.DISCRIMINATORS) do if v == held then have = k end end
    error('b200.FusedD(' .. name .. '): the context already holds ' .. have .. '; create it with b200.context(..., \''
          .. name .. '\') first')
  end
  local layers = D32_LAYERS[name](dimensions[1])
  b200.Fused.__init(self, F.NET_D, dimensions[1], layers)
  self.seed = 0
  self.wantWeightGrads = true   -- set false inside fevalG_on_D to skip the D weight gradients the reference discards
end
function FusedD:updateOutput(input)
  self:sync()
  local B = input:size(1)
  self.output:resize(B, 1)
  self.seed = self.seed + 1
  F.check(C.fg_D_forward(self.ctx, F.ptr(input:contiguous()), B, self.train and 1 or 0, nil, self.seed, F.ptr(self.output)), 'fg_D_forward')
  return self.output
end
function FusedD:backward(input, gradOutput)
  self:sync()
  self.gradInput:resizeAs(input)
  F.check(C.fg_D_backward(self.ctx, F.ptr(gradOutput:contiguous()), self.wantWeightGrads and 1 or 0, F.ptr(self.gradInput)), 'fg_D_backward')
  return self.gradInput
end
FusedD.updateGradInput = FusedD.backward

---------------------------------------------------------------------------------------------------------------
-- nn.BCECriterion replacement (train.lua:148); optional: the stock CPU criterion keeps working on the
-- FloatTensor outputs of the wrapping Sequential
---------------------------------------------------------------------------------------------------------------
local BCE, bparent = torch.class('b200.BCECriterion', 'nn.Criterion')
function BCE:__init() bparent.__init(self); self.ctx = b200.context(); self.gradInput = torch.FloatTensor() end
function BCE:updateOutput(input, target)
  local out = torch.FloatTensor(1)
  F.check(C.fg_bce_forward(self.ctx, F.ptr(input:contiguous()), F.ptr(target:contiguous()), input:nElement(), F.ptr(out)), 'fg_bce_forward')
  self.output = out[1]
  return self.output
end
function BCE:updateGradInput(input, target)
  self.gradInput:resizeAs(input)
  F.check(C.fg_bce_backward(self.ctx, F.ptr(input:contiguous()), F.ptr(target:contiguous()), input:nElement(), F.ptr(self.gradInput)), 'fg_bce_backward')
  return self.gradInput
end

---------------------------------------------------------------------------------------------------------------
-- interruptableAdam(opfunc, x, config[, state]) (interruptable_optimizers.lua:49-94), optional drop-in for the
-- stock one (which also works: it updates the aliased flat tensor in place with cutorch ops).  x is the FLAT
-- PARAMETER TENSOR exactly as adversarial.lua:264 / :284 pass it; opfunc(x) returns f, dfdx or false, false.
-- The update is one fused kernel on the raw device pointers; penalty and clamp were already applied to dfdx by the
-- caller's opfunc (adversarial.lua:103-123), so none is applied here.
---------------------------------------------------------------------------------------------------------------
function b200.interruptableAdam(opfunc, x, config, state)
  local config = config or {}
  local state = state or config
  local lr = config.learningRate or 0.001
  local beta1, beta2, epsilon = config.beta1 or 0.9, config.beta2 or 0.999, config.epsilon or 1e-8
  local fx, dfdx = opfunc(x)
  if fx == false then return false end                                -- interruptable_optimizers.lua:64-66
  state.t = (state.t or 0) + 1
  state.m = state.m or x.new(dfdx:size()):zero()
  state.v = state.v or x.new(dfdx:size()):zero()
  F.check(C.fg_adam_step(b200.context(), devptr(x), devptr(dfdx), devptr(state.m), devptr(state.v), x:nElement(), lr, beta1,
                         beta2, epsilon, state.t, 0, 0, 0, 1), 'fg_adam_step')
  return x, {fx}
end

---------------------------------------------------------------------------------------------------------------
-- per-layer modules (L-op level): constructor-compatible with the classes models.lua instantiates
---------------------------------------------------------------------------------------------------------------
local Conv, cparent = torch.class('b200.SpatialConvolution', 'nn.Module')  -- cudnn./nn.SpatialConvolution, stride 1, same pad
function Conv:__init(nIn, nOut, kW, kH, dW, dH, padW, padH)
  cparent.__init(self)
  assert(kW == kH and (dW or 1) == 1 and (dH or 1) == 1 and (padW or 0) == (kW - 1) / 2, 'b200.SpatialConvolution: square, stride 1, same padding')
  self.nIn, self.nOut, self.k = nIn, nOut, kW
  self.weight, self.bias = torch.FloatTensor(nOut, nIn, kH, kW), torch.FloatTensor(nOut)
  self.gradWeight, self.gradBias = torch.FloatTensor(nOut, nIn, kH, kW):zero(), torch.FloatTensor(nOut):zero()
  self.ctx = b200.context()
  self:reset()
end
function Conv:reset()
  local stdv = 1 / math.sqrt(self.k * self.k * self.nIn)
  self.weight:uniform(-stdv, stdv); self.bias:uniform(-stdv, stdv)
end
function Conv:updateOutput(input)
  local N, H, W = input:size(1), input:size(3), input:size(4)
  self.output:resize(N, self.nOut, H, W)
  F.check(C.fg_conv2d_forward(self.ctx, F.ptr(input:contiguous()), F.ptr(self.weight), F.ptr(self.bias), F.ptr(self.output), N, self.nIn, H, W, self.nOut, self.k), 'fg_conv2d_forward')
  return self.output
end
function Conv:updateGradInput(input, gradOutput)
  local N, H, W = input:size(1), input:size(3), input:size(4)
  self.gradInput:resizeAs(input)
  F.check(C.fg_conv2d_backward_data(self.ctx, F.ptr(gradOutput:contiguous()), F.ptr(self.weight), F.ptr(self.gradInput), N, self.nIn, H, W, self.nOut, self.k), 'fg_conv2d_backward_data')
  return self.gradInput
end
function Conv:accGradParameters(input, gradOutput, scale)
  assert((scale or 1) == 1, 'b200.SpatialConvolution: scale must be 1')
  local N, H, W = input:size(1), input:size(3), input:size(4)
  F.check(C.fg_conv2d_backward_filter(self.ctx, F.ptr(input:contiguous()), F.ptr(gradOutput:contiguous()), F.ptr(self.gradWeight), F.ptr(self.gradBias), N, self.nIn, H, W, self.nOut, self.k), 'fg_conv2d_backward_filter')
end

-- layers/cudnnSpatialConvolutionUpsample.lua: a convolution to nOut*factor^2 planes (:14-15) whose contiguous output is
-- viewed as [N][nOut][h*factor][w*factor] (:18-30) and whose gradOutput is viewed back (:32-58).  The reference only
-- instantiates factor = 1 (models_c2f.lua:123-131); fg_scu_* takes any factor (default 2 like the reference's :5).
local SCU = torch.class('b200.SpatialConvolutionUpsample', 'b200.SpatialConvolution')
function SCU:__init(nIn, nOut, kW, kH, factor)
  factor = factor or 2
  assert(kW % 2 == 1 and kH % 2 == 1 and kW == kH, 'b200.SpatialConvolutionUpsample: odd square kernels')
  self.factor, self.nOutU = factor, nOut
  b200.SpatialConvolution.__init(self, nIn, nOut * factor * factor, kW, kH, 1, 1, (kW - 1) / 2, (kH - 1) / 2)
end
function SCU:updateOutput(input)
  local N, H, W = input:size(1), input:size(3), input:size(4)
  self.output:resize(N, self.nOutU, H * self.factor, W * self.factor)   -- the view of :24; same bytes as [N][nOut*f*f][H][W]
  F.check(C.fg_scu_forward(self.ctx, F.ptr(input:contiguous()), F.ptr(self.weight), F.ptr(self.bias), F.ptr(self.output), N, self.nIn, H, W, self.nOutU, self.k, self.factor), 'fg_scu_forward')
  return self.output
end
function SCU:updateGradInput(input, gradOutput)
  local N, H, W = input:size(1), input:size(3), input:size(4)
  self.gradInput:resizeAs(input)
  F.check(C.fg_scu_backward_data(self.ctx, F.ptr(gradOutput:contiguous()), F.ptr(self.weight), F.ptr(self.gradInput), N, self.nIn, H, W, self.nOutU, self.k, self.factor), 'fg_scu_backward_data')
  return self.gradInput
end
function SCU:accGradParameters(input, gradOutput, scale)
  assert((scale or 1) == 1, 'b200.SpatialConvolutionUpsample: scale must be 1')
  local N, H, W = input:size(1), input:size(3), input:size(4)
  F.check(C.fg_scu_backward_filter(self.ctx, F.ptr(input:contiguous()), F.ptr(gradOutput:contiguous()), F.ptr(self.gradWeight), F.ptr(self.gradBias), N, self.nIn, H, W, self.nOutU, self.k, self.factor), 'fg_scu_backward_filter')
end

local Lin, lparent = torch.class('b200.Linear', 'nn.Module')
function Lin:__init(inp, out)
  lparent.__init(self)
  self.inp, self.out = inp, out
  self.weight, self.bias = torch.FloatTensor(out, inp), torch.FloatTensor(out)
  self.gradWeight, self.gradBias = torch.FloatTensor(out, inp):zero(), torch.FloatTensor(out):zero()
  self.ctx = b200.context()
  local stdv = 1 / math.sqrt(inp)
  self.weight:uniform(-stdv, stdv); self.bias:uniform(-stdv, stdv)
end
function Lin:updateOutput(input)
  local N = input:size(1)
  self.output:resize(N, self.out)
  F.check(C.fg_linear_forward(self.ctx, F.ptr(input:contiguous()), F.ptr(self.weight), F.ptr(self.bias), F.ptr(self.output), N, self.inp, self.out), 'fg_linear_forward')
  return self.output
end
function Lin:updateGradInput(input, gradOutput)
  self.gradInput:resizeAs(input)
  F.check(C.fg_linear_backward(self.ctx, F.ptr(input:contiguous()), F.ptr(self.weight), F.ptr(gradOutput:contiguous()), F.ptr(self.gradInput), nil, nil, input:size(1), self.inp, self.out), 'fg_linear_backward')
  return self.gradInput
end
function Lin:accGradParameters(input, gradOutput)
  F.check(C.fg_linear_backward(self.ctx, F.ptr(input:contiguous()), F.ptr(self.weight), F.ptr(gradOutput:contiguous()), nil, F.ptr(self.gradWeight), F.ptr(self.gradBias), input:size(1), self.inp, self.out), 'fg_linear_backward')
end

local BN, bnparent = torch.class('b200.SpatialBatchNormalization', 'nn.Module')
function BN:__init(nFeature)
  bnparent.__init(self)
  self.n = nFeature
  self.weight, self.bias = torch.FloatTensor(nFeature):uniform(), torch.FloatTensor(nFeature):zero()
  self.gradWeight, self.gradBias = torch.FloatTensor(nFeature):zero(), torch.FloatTensor(nFeature):zero()
  self.running_mean, self.running_var = torch.FloatTensor(nFeature):zero(), torch.FloatTensor(nFeature):fill(1)
  self.save_mean, self.save_istd = torch.FloatTensor(nFeature), torch.FloatTensor(nFeature)
  self.ctx = b200.context()
end
function BN:updateOutput(input)
  local N, HW = input:size(1), input:size(3) * input:size(4)
  self.output:resizeAs(input)
  F.check(C.fg_bn_forward_train(self.ctx, F.ptr(input:contiguous()), F.ptr(self.weight), F.ptr(self.bias), F.ptr(self.output), F.ptr(self.save_mean), F.ptr(self.save_istd), F.ptr(self.running_mean), F.ptr(self.running_var), N, self.n, HW), 'fg_bn_forward_train')
  return self.output
end
function BN:backward(input, gradOutput)
  local N, HW = input:size(1), input:size(3) * input:size(4)
  self.gradInput:resizeAs(input)
  F.check(C.fg_bn_backward(self.ctx, F.ptr(input:contiguous()), F.ptr(self.weight), F.ptr(self.save_mean), F.ptr(self.save_istd), F.ptr(gradOutput:contiguous()), F.ptr(self.gradInput), F.ptr(self.gradWeight), F.ptr(self.gradBias), N, self.n, HW), 'fg_bn_backward')
  return self.gradInput
end

local PR, prparent = torch.class('b200.PReLU', 'nn.Module')  -- nn.PReLU(): one shared slope
function PR:__init()
  prparent.__init(self)
  self.weight, self.gradWeight = torch.FloatTensor(1):fill(0.25), torch.FloatTensor(1):zero()
  self.ctx = b200.context()
end
function PR:updateOutput(input)
  self.output:resizeAs(input)
  F.check(C.fg_prelu_forward(self.ctx, F.ptr(input:contiguous()), F.ptr(self.weight), F.ptr(self.output), input:nElement()), 'fg_prelu_forward')
  return self.output
end
function PR:backward(input, gradOutput)
  self.gradInput:resizeAs(input)
  F.check(C.fg_prelu_backward(self.ctx, F.ptr(input:contiguous()), F.ptr(self.weight), F.ptr(gradOutput:contiguous()), F.ptr(self.gradInput), F.ptr(self.gradWeight), input:nElement()), 'fg_prelu_backward')
  return self.gradInput
end


---------------------------------------------------------------------------------------------------------------
-- parameter-free layers (L-op level): resampling, pooling, dropout, sigmoid.  NCHW FloatTensors in and out.
---------------------------------------------------------------------------------------------------------------
local function dims4(t) return t:size(1), t:size(2), t:size(3), t:size(4) end

local Up, upparent = torch.class('b200.SpatialUpSamplingNearest', 'nn.Module')  -- models.lua:63,68 (scale 2 only)
function Up:__init(scale) upparent.__init(self); assert(scale == 2, 'b200.SpatialUpSamplingNearest: scale 2 only'); self.ctx = b200.context() end
function Up:updateOutput(input)
  local n, c, h, w = dims4(input)
  self.output:resize(n, c, 2 * h, 2 * w)
  F.check(C.fg_upsample2_forward(self.ctx, F.ptr(input), F.ptr(self.output), n, c, h, w), 'fg_upsample2_forward')
  return self.output
end
function Up:updateGradInput(input, gradOutput)
  local n, c, h, w = dims4(input)
  self.gradInput:resizeAs(input)
  F.check(C.fg_upsample2_backward(self.ctx, F.ptr(gradOutput), F.ptr(self.gradInput), n, c, h, w), 'fg_upsample2_backward')
  return self.gradInput
end

local function pool_class(name, fwd, bwd, needs_input)
  local P, pparent = torch.class('b200.' .. name, 'nn.Module')
  function P:__init(kW, kH, dW, dH)
    pparent.__init(self)
    assert(kW == 2 and kH == 2 and (dW or 2) == 2 and (dH or 2) == 2, 'b200.' .. name .. ': 2x2 window, stride 2 only')
    self.ctx = b200.context()
  end
  function P:updateOutput(input)
    local n, c, h, w = dims4(input)
    self.output:resize(n, c, math.floor(h / 2), math.floor(w / 2))
    F.check(C[fwd](self.ctx, F.ptr(input), F.ptr(self.output), n, c, h, w), fwd)
    return self.output
  end
  function P:updateGradInput(input, gradOutput)
    local n, c, h, w = dims4(input)
    self.gradInput:resizeAs(input)
    if needs_input then
      F.check(C[bwd](self.ctx, F.ptr(input), F.ptr(gradOutput), F.ptr(self.gradInput), n, c, h, w), bwd)
    else
      F.check(C[bwd](self.ctx, F.ptr(gradOutput), F.ptr(self.gradInput), n, c, h, w), bwd)
    end
    return self.gradInput
  end
end
pool_class('SpatialAveragePooling', 'fg_avgpool2_forward', 'fg_avgpool2_backward', false)  -- models.lua:388,...
pool_class('SpatialMaxPooling', 'fg_maxpool2_forward', 'fg_maxpool2_backward', true)       -- models_c2f.lua:251,256

-- nn.Dropout(p) (v2 rescale) and nn.SpatialDropout(p) (no rescale); the keep mask is drawn on the host with
-- torch.bernoulli like the reference modules do, so the reference's RNG stream is preserved
local function dropout_class(name, spatial, default_p)
  local D, dparent = torch.class('b200.' .. name, 'nn.Module')
  function D:__init(p) dparent.__init(self); self.p = p or default_p; self.train = true; self.ctx = b200.context(); self.noise = torch.FloatTensor() end
  function D:apply_(src, dst, fn)
    local n, c = src:size(1), src:size(2)
    local hw = src:nElement() / (n * c)
    dst:resizeAs(src)
    F.check(C[fn](self.ctx, F.ptr(src), self.train and F.ptr(self.noise) or nil, self.p, spatial and 1 or 0, F.ptr(dst), n, c, hw), fn)
    return dst
  end
  function D:updateOutput(input)
    if self.train then
      if spatial then self.noise:resize(input:size(1), input:size(2)) else self.noise:resizeAs(input) end
      self.noise:bernoulli(1 - self.p)
    end
    return self:apply_(input, self.output, 'fg_dropout_forward')
  end
  function D:updateGradInput(input, gradOutput) return self:apply_(gradOutput, self.gradInput, 'fg_dropout_backward') end
end
dropout_class('Dropout', false, 0.5)         -- models.lua:408,411; models_c2f.lua:258,264
dropout_class('SpatialDropout', true, 0.5)   -- models.lua:387,391,396,401 (p = 0.2 there)

local Sg, sgparent = torch.class('b200.Sigmoid', 'nn.Module')  -- models.lua:74,413
function Sg:__init() sgparent.__init(self); self.ctx = b200.context() end
function Sg:updateOutput(input)
  self.output:resizeAs(input)
  F.check(C.fg_sigmoid_forward(self.ctx, F.ptr(input), F.ptr(self.output), input:nElement()), 'fg_sigmoid_forward')
  return self.output
end
function Sg:updateGradInput(input, gradOutput)
  self.gradInput:resizeAs(input)
  F.check(C.fg_sigmoid_backward(self.ctx, F.ptr(self.output), F.ptr(gradOutput), F.ptr(self.gradInput), input:nElement()), 'fg_sigmoid_backward')
  return self.gradInput
end

-- train.lua --denoise (:101-110): DENOISER = AE1_DECODER:evaluate(), applied to G's images in
-- NN_UTILS.visualizeProgress (nn_utils.lua:144-155).  b200.Denoiser(IMG_DIMENSIONS, file, OPT.gpu, OPT.batchSize)
-- loads `denoiser_CxHxW.net` (AE1_DECODER's flat parameters and BatchNorm running statistics, read by the library's
-- Torch7 reader) and forwards through fg_dn_denoise; :training() switches to the training-mode forward (WhiteNoise,
-- batch statistics, drawn dropout).  It is built before the GAN's shims, so it creates the process's context: pass the
-- device and batch size the GAN will use (b200.context keeps the first context it creates).
local Denoiser, dparent = torch.class('b200.Denoiser', 'nn.Module')
function Denoiser:__init(dimensions, filename, device, maxBatch)
  dparent.__init(self)
  self.ctx = b200.context(device or 0, maxBatch or 256, dimensions[1])
  self.maxBatch = tonumber(C.fg_get_option(self.ctx, 'max_batch'))  -- the context's, whoever created it
  self.C, self.S, self.train, self.seed = dimensions[1], dimensions[2], false, 0
  local out = ffi.new('fg_dn*[1]')
  F.check(C.fg_dn_create(self.ctx, self.S, out), 'fg_dn_create')
  self.dn = ffi.gc(out[0], C.fg_dn_destroy)
  if filename then self:load(filename) end
  self.output = torch.FloatTensor()
end
function Denoiser:load(filename)
  local f = ffi.new('fg_t7*[1]')
  F.check(C.fg_t7_open(filename, f), 'fg_t7_open')
  local n = tonumber(C.fg_dn_param_count(self.C, self.S))
  local p, bn = torch.FloatTensor(n), torch.FloatTensor(2 * (8 + 8 + 2048))
  local got = C.fg_t7_net_params(f[0], 'AE1_DECODER', F.ptr(p), n)
  local gotbn = C.fg_t7_net_bn_state(f[0], 'AE1_DECODER', F.ptr(bn), bn:nElement())
  C.fg_t7_close(f[0])
  assert(tonumber(got) == n, 'b200.Denoiser: AE1_DECODER does not match the denoiser at this image size')
  assert(tonumber(gotbn) == bn:nElement(), 'b200.Denoiser: AE1_DECODER lacks its BatchNorm running statistics')
  F.check(C.fg_dn_set_params(self.dn, 0, F.ptr(p)), 'fg_dn_set_params')
  F.check(C.fg_dn_set_bn_state(self.dn, 0, F.ptr(bn)), 'fg_dn_set_bn_state')
end
function Denoiser:training() self.train = true; return self end
function Denoiser:evaluate() self.train = false; return self end
function Denoiser:type() return self end
function Denoiser:float() return self end
function Denoiser:updateOutput(input)
  input = input:float():contiguous()
  local B = input:size(1)
  self.output:resize(B, self.C, self.S, self.S)
  if self.train then
    self.seed = self.seed + 1
    F.check(C.fg_dn_forward(self.dn, 0, F.ptr(input), B, 1, nil, nil, self.seed, F.ptr(self.output)), 'fg_dn_forward')
  else
    F.check(C.fg_dn_denoise(self.dn, F.ptr(input), B, math.min(B, self.maxBatch), F.ptr(self.output)), 'fg_dn_denoise')
  end
  return self.output
end

return b200
