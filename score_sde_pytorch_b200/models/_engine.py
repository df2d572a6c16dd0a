"""Engine plumbing shared by the engine-backed score networks (``NCSNpp``, ``DDPM``).

A subclass builds its parameters in ``all_modules`` with the reference's names, shapes and
initialisers, calls :meth:`EngineModel._init_engine` at the end of its constructor and implements
``_family_config(c)``, which fills the family-specific fields of a ``b200_ncsnpp_config``.  Everything
else - creating and planning the native engine, repacking weights after in-place writes, the forward
through the C ABI, debug taps and per-op labels - lives here once.
"""
import ctypes
import math
import weakref

import torch
import torch.nn as nn

from .. import _lib

PDL_DEFAULT = False
HALO_DEFAULT = True      # halo form of the 3x3 mainloop in the swapped-operand kernel (csrc/gemm_tc.cu)


def positional_frequencies(nf):
  """Frequency table of the sinusoidal time embedding (``models/layers.py:515-529``), built with the reference's own
  torch ops so the engine multiplies by bit-identical fp32 frequencies."""
  half = nf // 2
  return torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000) / (half - 1)))


class EngineModel(nn.Module):
  """Base of the engine-backed networks.  ``precision``: ``'tf32'`` (wgmma tensor cores on TF32-rounded fp32 operands,
  default), ``'f16'`` (wgmma on fp16 operands: the same 11-bit significand as TF32 with fp32 accumulation and fp32
  activations between layers), ``'tf32x3'`` (split TF32: every operand as a hi + lo pair of TF32 values, three wgmma
  products per K step into an fp32 accumulator - close to fp32 accuracy at tensor-core rate) or ``'fp32'`` (strict fp32
  on CUDA cores; validation mode)."""
  takes_time_labels = True   # the label is a time / sigma value (False: integer noise-level indices, NCSNv2)

  def _set_engine_options(self, config, precision=None, keep_activations=False, lanes=1, cuda_core_head=None, pdl=None,
                          halo=None):
    m = config.model
    self.precision = (precision or getattr(m, 'precision', 'tf32')).lower()
    self.keep_activations = bool(keep_activations)
    self.lanes = int(getattr(m, 'lanes', lanes))   # 2: evaluate batches >= 128 as two half-batch lanes on two streams
    # per-engine execution options (fields of b200_ncsnpp_config; nothing is read from the environment)
    self.cuda_core_head = bool(getattr(m, 'cuda_core_head', False) if cuda_core_head is None else cuda_core_head)
    # programmatic dependent launch between the kernels of a forward / PC iteration (common.cuh)
    self.pdl = bool(getattr(m, 'pdl', PDL_DEFAULT) if pdl is None else pdl)
    # halo form of the 3x3 tensor-core mainloop (csrc/gemm_tc.cu): True (default) = in the swapped-operand kernel, False =
    # nine shifted tile loads per channel chunk (kept for A/B; bit-identical results)
    self.halo = bool(getattr(m, 'halo', HALO_DEFAULT) if halo is None else halo)

  def _init_engine(self):
    """Call once ``all_modules`` is complete."""
    self._engine = None        # (handle, blob, workspace, batch, weights_version)
    self._tan_engine = None    # the same for the tangent-enabled engine of jvp(), created on first use
    self._weights_version = 0
    self._link_parameters()    # lets models.ema.ExponentialMovingAverage tell this module to repack
    # fires for direct loads and for loads through a wrapper (DataParallel(model).load_state_dict calls
    # _load_from_state_dict on the children, not the override below)
    self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate_weights())

  # ---- native engine plumbing ------------------------------------------------
  def _family_config(self, c):
    raise NotImplementedError

  def _native_config(self):
    cfg, m = self.config, self.config.model
    c = _lib.NcsnppConfig()
    c.image_size, c.num_channels, c.nf, c.num_res_blocks = cfg.data.image_size, cfg.data.num_channels, m.nf, m.num_res_blocks
    c.num_levels = len(m.ch_mult)
    for i, v in enumerate(m.ch_mult):
      c.ch_mult[i] = int(v)
    c.num_attn_resolutions = len(m.attn_resolutions)
    for i, v in enumerate(m.attn_resolutions):
      c.attn_resolutions[i] = int(v)
    c.centered, c.scale_by_sigma = int(bool(cfg.data.centered)), int(bool(m.scale_by_sigma))
    c.conditional = int(bool(m.conditional))
    self._execution_config(c)
    self._family_config(c)
    return c

  def _execution_config(self, c):
    """The execution fields of a ``b200_ncsnpp_config``, shared by every family."""
    c.pdl = int(self.pdl)
    c.no_halo = int(not self.halo)
    if self.precision not in ('tf32', 'fp32', 'f16', 'tf32x3'):
      raise ValueError(f"precision must be 'tf32', 'fp32', 'f16' or 'tf32x3', got {self.precision!r}")
    c.precision = {'tf32': 0, 'fp32': 1, 'f16': 2, 'tf32x3': 3}[self.precision]
    c.keep_activations = int(self.keep_activations)
    c.lanes = self.lanes
    c.cuda_core_head = int(self.cuda_core_head)

  def native_param_table(self):
    """[(name, shape)] the engine expects, in its load order (no GPU needed)."""
    h = ctypes.c_void_p()
    cfg = self._native_config()
    _lib.call('b200_ncsnpp_create', ctypes.byref(cfg), ctypes.byref(h))
    try:
      return self._param_table(h)
    finally:
      _lib.load().b200_ncsnpp_destroy(h)

  @staticmethod
  def _param_table(h):
    lib = _lib.load()
    out = []
    for i in range(lib.b200_ncsnpp_num_params(h)):
      name = ctypes.create_string_buffer(256)
      shape = (ctypes.c_longlong * 4)()
      nd = ctypes.c_int()
      _lib.call('b200_ncsnpp_param_info', h, i, name, 256, shape, ctypes.byref(nd))
      out.append((name.value.decode(), tuple(shape[:nd.value])))
    return out

  def invalidate_weights(self):
    """Call after mutating parameters in place so the engine repacks its device copy.  This package's
    ``models.ema.ExponentialMovingAverage.copy_to`` / ``restore`` do it automatically (through the owner link
    set below); with any other in-place writer (the reference's EMA class, manual ``p.data.copy_``) call it."""
    self._weights_version += 1

  def _link_parameters(self):
    ref = weakref.ref(self)
    for p in self.parameters():
      p._b200_owner = ref

  def load_state_dict(self, state_dict, strict=True, **kw):
    sd = {(k[7:] if k.startswith('module.') else k): v for k, v in state_dict.items()}
    return super().load_state_dict(sd, strict=strict, **kw)   # the post hook invalidates the packed weights

  def _release(self):
    """Destroy the native engines.  Every cached PC plan holds a pointer to the primal one, so they are released first."""
    for plan in self.__dict__.get('_pc_plans', {}).values():
      plan._release()
    if self.__dict__.get('_engine') is not None:
      _lib.load().b200_ncsnpp_destroy(self._engine['h'])
      self._engine = None
    self._release_tangent()

  def _release_tangent(self):
    if self.__dict__.get('_tan_engine') is not None:
      _lib.load().b200_ncsnpp_destroy(self._tan_engine['h'])
      self._tan_engine = None

  def check_jvp_supported(self):
    """Raise ``NotImplementedError`` naming the field if this configuration has no forward-mode tangent pass (``jvp``).
    Creates and destroys a tangent-enabled engine handle; needs no GPU."""
    name = type(self).__name__
    if self.precision == 'f16':
      raise NotImplementedError(f"{name}.jvp: precision='f16' has no tangent pass; use precision='tf32' or 'fp32'")
    cfg = self._native_config()
    cfg.tangent = 1
    h = ctypes.c_void_p()
    lib = _lib.load()
    if lib.b200_ncsnpp_create(ctypes.byref(cfg), ctypes.byref(h)) != 0:
      raise NotImplementedError(f'{name}.jvp: {_lib.last_error()}')
    lib.b200_ncsnpp_destroy(h)

  @staticmethod
  def _explicit_device(device):
    """``torch.device('cuda') != torch.device('cuda:0')``: normalise to an explicit index so the engine cache
    does not thrash between a sampler created with ``device='cuda'`` and direct ``model(x, t)`` calls."""
    device = torch.device(device)
    if device.type == 'cuda' and device.index is None:
      device = torch.device('cuda', torch.cuda.current_device())
    return device

  def __del__(self):
    try:
      self._release()
    except Exception:
      pass

  def engine(self, batch, device, tangent=False):
    """Create / re-plan the native engine for ``batch`` images on ``device``.  ``eng['gen']`` is a monotonically
    increasing plan generation: it changes whenever the engine, its workspace or its plan is rebuilt, which is what
    dependants (captured CUDA graphs in ``native.PcPlan``) key their validity on.

    ``tangent=True``: the separate tangent-enabled engine of :meth:`jvp` (``b200_ncsnpp_config.tangent = 1``), with its own
    weights and workspace; the primal engine, its PC plans and the generation counter are not touched."""
    device = self._explicit_device(device)
    eng = self._tan_engine if tangent else self._engine
    if eng is not None and (eng['device'] != device or eng['precision'] != self.precision):
      self._release_tangent() if tangent else self._release()
      eng = None
    if eng is None:
      h = ctypes.c_void_p()
      cfg = self._native_config()
      if tangent:
        self.check_jvp_supported()
        cfg.tangent = 1
      _lib.call('b200_ncsnpp_create', ctypes.byref(cfg), ctypes.byref(h))
      nbytes = _lib.load().b200_ncsnpp_weights_bytes(h)
      blob = torch.zeros(nbytes // 4 + 64, dtype=torch.float32, device=device)
      _lib.call('b200_ncsnpp_bind_weights', h, _lib.ptr(blob))
      if not tangent:
        self._generation = getattr(self, '_generation', 0) + 1
      eng = dict(h=h, blob=blob, ws=None, batch=0, wver=-1, device=device, precision=self.precision,
                 table=self._param_table(h), gen=None if tangent else self._generation)
      if tangent:
        self._tan_engine = eng
      else:
        self._engine = eng
    if eng['wver'] != self._weights_version:
      sd = dict(self.named_parameters())
      pos_freqs = getattr(self, 'pos_freqs', None)   # the sinusoidal embedding's frequency table (a pseudo-parameter)
      if pos_freqs is not None:
        sd['pos_freqs'] = pos_freqs
      st = _lib.stream_ptr(device)
      for i, (name, shape) in enumerate(eng['table']):
        p = sd[name]
        if tuple(p.shape) != tuple(shape):
          raise RuntimeError(f'parameter {name}: module has {tuple(p.shape)}, engine expects {tuple(shape)}')
        src = p.detach().to(device=device, dtype=torch.float32).contiguous()
        _lib.call('b200_ncsnpp_load_param', eng['h'], i, _lib.ptr(src), st)
      torch.cuda.current_stream(device).synchronize()   # sources above are temporaries
      eng['wver'] = self._weights_version
    if eng['batch'] != batch:
      need = _lib.load().b200_ncsnpp_workspace_bytes(eng['h'], batch)
      if need < 0:
        raise RuntimeError(f'engine planning failed: {_lib.last_error()}')
      if eng['ws'] is None or eng['ws'].numel() * 4 < need:
        eng['ws'] = None
        eng['ws'] = torch.empty(need // 4 + 256, dtype=torch.float32, device=device)
      _lib.call('b200_ncsnpp_bind_workspace', eng['h'], batch, _lib.ptr(eng['ws']), eng['ws'].numel() * 4)
      eng['batch'] = batch
      if not tangent:
        self._generation += 1
        eng['gen'] = self._generation
    return eng

  def forward(self, x, time_cond, labels_uniform=False):
    name = type(self).__name__
    if not x.is_cuda:
      raise RuntimeError(f'{name} (score_sde_pytorch_b200) runs on CUDA devices only: there is no CPU path; '
                         'move the model and inputs to a CUDA device (the PyTorch restatement in oracle/ is test-only)')
    if x.dim() != 4 or x.shape[1] != self.config.data.num_channels or x.shape[2] != self.config.data.image_size \
        or x.shape[3] != self.config.data.image_size:
      raise RuntimeError(f'{name}: input shape {tuple(x.shape)} does not match the configured image geometry')
    with torch.cuda.device(x.device):
      eng = self.engine(x.shape[0], x.device)
      xin = x.detach().to(torch.float32).contiguous()
      lab = time_cond.detach().to(device=x.device, dtype=torch.float32).contiguous()
      if lab.numel() != x.shape[0]:
        raise RuntimeError(f'{name}: time_cond has {lab.numel()} entries for a batch of {x.shape[0]}')
      out = torch.empty_like(xin)
      _lib.call('b200_ncsnpp_forward', eng['h'], _lib.ptr(xin), _lib.ptr(lab), int(bool(labels_uniform)),
                _lib.ptr(out), _lib.stream_ptr(x.device))
    return out

  def jvp(self, x, time_cond, v, labels_uniform=False):
    """``(net(x), J_net(x) v)`` in one forward-mode pass of the tangent-enabled engine (``b200_ncsnpp_jvp``): the
    Jacobian-vector product the likelihood's divergence needs (``likelihood.py:26-35``), without autograd.  Configurations
    without a tangent pass raise ``NotImplementedError`` (:meth:`check_jvp_supported`)."""
    name = type(self).__name__
    if not x.is_cuda:
      raise RuntimeError(f'{name}.jvp runs on CUDA devices only')
    if x.dim() != 4 or x.shape[1] != self.config.data.num_channels or x.shape[2] != self.config.data.image_size \
        or x.shape[3] != self.config.data.image_size:
      raise RuntimeError(f'{name}: input shape {tuple(x.shape)} does not match the configured image geometry')
    if tuple(v.shape) != tuple(x.shape):
      raise RuntimeError(f'{name}.jvp: tangent shape {tuple(v.shape)} differs from the input shape {tuple(x.shape)}')
    with torch.cuda.device(x.device):
      eng = self.engine(x.shape[0], x.device, tangent=True)
      xin = x.detach().to(torch.float32).contiguous()
      vin = v.detach().to(device=x.device, dtype=torch.float32).contiguous()
      lab = time_cond.detach().to(device=x.device, dtype=torch.float32).contiguous()
      if lab.numel() != x.shape[0]:
        raise RuntimeError(f'{name}: time_cond has {lab.numel()} entries for a batch of {x.shape[0]}')
      out = torch.empty_like(xin)
      jv = torch.empty_like(xin)
      _lib.call('b200_ncsnpp_jvp', eng['h'], _lib.ptr(xin), _lib.ptr(lab), int(bool(labels_uniform)), _lib.ptr(vin),
                _lib.ptr(out), _lib.ptr(jv), _lib.stream_ptr(x.device))
    return out, jv

  def tap_tangent(self, module_index):
    """Debug (``keep_activations=True``, after :meth:`jvp`): the tangent of ``all_modules[module_index]``'s output, NCHW."""
    eng = self._tan_engine
    if eng is None:
      raise RuntimeError('tap_tangent: run jvp first')
    shape = (ctypes.c_int * 4)()
    buf = torch.empty(min(1 << 28, eng['ws'].numel()), dtype=torch.float32, device=eng['device'])
    _lib.call('b200_ncsnpp_tap_tangent', eng['h'], module_index, _lib.ptr(buf), buf.numel(), shape,
              _lib.stream_ptr(eng['device']))
    n = shape[0] * shape[1] * shape[2] * shape[3]
    return buf[:n].reshape(shape[0], shape[1], shape[2], shape[3]).clone()

  def activation_range_report(self, x, time_cond, limit=65504.0):
    """Largest magnitude of every module output of one evaluation, measured with an fp32-range (`'tf32'`) copy of this
    network.  `precision='f16'` stores the operands of every contraction - normalised activations, but also the raw block
    inputs of the skip projections - as IEEE fp16, which assumes |value| < 65504 (and loses precision below 6e-5);
    random-init and normalised activations are far inside, a trained checkpoint can be checked with this before it is
    sampled in fp16 mode.  Returns ``{'max_abs': {module_index: float}, 'worst': (index, value), 'fits_f16': bool}``."""
    probe = type(self)(self.config, precision='tf32', keep_activations=True, pdl=False).to(x.device)
    probe.load_state_dict(self.state_dict())
    with torch.no_grad():
      probe(x, time_cond)
    out = {}
    for i in range(len(self.all_modules)):
      try:
        out[i] = float(probe.tap(i).abs().max())
      except RuntimeError:
        continue
    probe._release()
    worst = max(out.items(), key=lambda kv: kv[1])
    return dict(max_abs=out, worst=worst, fits_f16=bool(worst[1] < limit))

  def tap(self, module_index):
    """Debug (``keep_activations=True``): output of ``all_modules[module_index]`` as NCHW."""
    eng = self._engine
    if eng is None:
      raise RuntimeError('tap: run a forward pass first')
    shape = (ctypes.c_int * 4)()
    cap = 1 << 28
    # query shape with a first call into a generous buffer sized from the workspace
    buf = torch.empty(min(cap, eng['ws'].numel()), dtype=torch.float32, device=eng['device'])
    _lib.call('b200_ncsnpp_tap', eng['h'], module_index, _lib.ptr(buf), buf.numel(), shape, _lib.stream_ptr(eng['device']))
    n = shape[0] * shape[1] * shape[2] * shape[3]
    return buf[:n].reshape(shape[0], shape[1], shape[2], shape[3]).clone()

  def launches_per_forward(self):
    return int(_lib.load().b200_ncsnpp_launches_per_forward(self._engine['h'])) if self._engine else 0

  def op_names(self, tangent=False):
    """Shape labels of the ops of the bound plan, in execution order (b200_ncsnpp_op_info); empty before the first call.
    ``tangent=True``: the plan of the tangent-enabled engine of :meth:`jvp`."""
    eng = self._tan_engine if tangent else self._engine
    if not eng:
      return []
    h = eng['h']
    n = int(_lib.load().b200_ncsnpp_num_ops(h))
    buf, kind, fl = ctypes.create_string_buffer(200), ctypes.c_int(), ctypes.c_double()
    names = []
    for i in range(n):
      _lib.call('b200_ncsnpp_op_info', h, i, buf, 200, ctypes.byref(kind), ctypes.byref(fl))
      names.append(buf.value.decode())
    return names
