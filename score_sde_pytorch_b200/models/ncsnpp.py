"""NCSN++ score network backed by the sm_90a engine.

Host-side mirror of ``models/ncsnpp.py:35-381``: ``NCSNpp(config)`` is an
``nn.Module`` registered as ``'ncsnpp'``; its parameters live in
``all_modules`` with the reference's names, shapes and initialisers, so
``state_dict()`` / ``load_state_dict()`` interoperate with reference checkpoints
(with or without the ``module.`` prefix DataParallel adds, ``utils.py:16``), and
``forward(x[B,C,H,W], time_cond[B]) -> [B,C,H,W]`` has the reference's meaning.

The forward itself is not PyTorch: parameters are repacked once into the
engine's blob (K-major, TF32-rounded where a layer runs on the tensor cores) and every
call replays the engine's kernel sequence on the current CUDA stream through the
C ABI (``include/scoresde_b200.h``).  CPU tensors are rejected — there is no CPU
path in the product (the plain-PyTorch restatement lives in ``oracle/`` and is
test infrastructure only).
"""
import ctypes

import numpy as np
import torch
import torch.nn as nn

from . import utils
from .. import _lib

PDL_DEFAULT = False
HALO_DEFAULT = True      # halo form of the 3x3 mainloop in the swapped-operand kernel (csrc/gemm_tc.cu)

_SUPPORTED = ("engine supports embedding_type in {'fourier','positional'}, conditional=True, resblock_type='biggan', "
              "fir in {True, False} (progressive_input='residual' needs fir=True), progressive in {'none','output_skip'}, "
              "progressive_input in {'none','residual','input_skip'} with progressive_combine='sum'; "
              "positional embeddings need scale_by_sigma=False")


def _variance_scaling_uniform(shape, scale, in_axis=1, out_axis=0):
  """fan_avg / uniform variance scaling, the reference's ``default_init``
  (``models/layers.py:54-91``; ``scale == 0`` is replaced by ``1e-10`` there, ``:88-91``)."""
  scale = 1e-10 if scale == 0 else scale
  rf = np.prod(shape) / shape[in_axis] / shape[out_axis]
  denom = (shape[in_axis] * rf + shape[out_axis] * rf) / 2
  return (torch.rand(*shape, dtype=torch.float32) * 2. - 1.) * np.sqrt(3 * scale / denom)


class _Holder(nn.Module):
  """Parameter container; submodule / parameter names follow the reference."""


def _conv(cin, cout, k, init_scale=1.):
  m = nn.Conv2d(cin, cout, kernel_size=k, stride=1, padding=k // 2)
  m.weight.data = _variance_scaling_uniform(m.weight.shape, init_scale)
  nn.init.zeros_(m.bias)
  return m


def _gn(c):
  return nn.GroupNorm(num_groups=min(c // 4, 32), num_channels=c, eps=1e-6)


def _dense(cin, cout):
  m = nn.Linear(cin, cout)
  m.weight.data = _variance_scaling_uniform(m.weight.shape, 1.)
  nn.init.zeros_(m.bias)
  return m


class _NIN(nn.Module):
  def __init__(self, cin, cout, init_scale=0.1):
    super().__init__()
    self.W = nn.Parameter(_variance_scaling_uniform((cin, cout), init_scale))
    self.b = nn.Parameter(torch.zeros(cout))


class _Fourier(nn.Module):
  def __init__(self, size, scale):
    super().__init__()
    self.W = nn.Parameter(torch.randn(size) * scale, requires_grad=False)


def _resblock(cin, cout, temb_dim, init_scale, up=False, down=False):
  h = _Holder()
  h.GroupNorm_0 = _gn(cin)
  h.Conv_0 = _conv(cin, cout, 3)
  h.Dense_0 = _dense(temb_dim, cout)
  h.GroupNorm_1 = _gn(cout)
  h.Conv_1 = _conv(cout, cout, 3, init_scale)
  if cin != cout or up or down:
    h.Conv_2 = _conv(cin, cout, 1)
  return h


def _attn(c, init_scale):
  h = _Holder()
  h.GroupNorm_0 = _gn(c)
  h.NIN_0, h.NIN_1, h.NIN_2 = _NIN(c, c), _NIN(c, c), _NIN(c, c)
  h.NIN_3 = _NIN(c, c, init_scale=init_scale)
  return h


def _combine(dim1, dim2):
  """``layerspp.Combine`` (``layerspp.py:44-59``): ``Conv_0`` is a 1x1 convolution dim1 -> dim2."""
  h = _Holder()
  h.Conv_0 = _conv(dim1, dim2, 1)
  return h


def _pyramid_down(cin, cout):
  h = _Holder()
  inner = _Holder()
  inner.weight = nn.Parameter(_variance_scaling_uniform((cout, cin, 3, 3), 1.))
  inner.bias = nn.Parameter(torch.zeros(cout))
  h.Conv2d_0 = inner
  return h


@utils.register_model(name='ncsnpp')
class NCSNpp(nn.Module):
  """NCSN++ model (engine-backed).  ``precision``: ``'tf32'`` (wgmma tensor cores on TF32-rounded
  fp32 operands, default), ``'f16'`` (wgmma on fp16 operands: the same 11-bit significand as TF32
  with fp32 accumulation and fp32 activations between layers, half the operand traffic and twice the
  MMA rate) or ``'fp32'`` (strict fp32 on CUDA cores; validation mode)."""

  def __init__(self, config, precision=None, keep_activations=False, lanes=1, cuda_core_head=None,
               separate_groupnorm=None, pdl=None, halo=None):
    super().__init__()
    self.config = config
    m = config.model
    emb = m.embedding_type.lower()
    if (emb not in ('fourier', 'positional') or not m.conditional or m.resblock_type.lower() != 'biggan'
        or m.progressive.lower() not in ('none', 'output_skip')
        or m.progressive_input.lower() not in ('none', 'residual', 'input_skip')
        or (m.progressive_input.lower() == 'input_skip' and str(getattr(m, 'progressive_combine', 'sum')).lower() != 'sum')
        or (not m.fir and m.progressive_input.lower() == 'residual')
        or (emb == 'positional' and m.scale_by_sigma)):
      raise NotImplementedError(f'NCSNpp: {_SUPPORTED}')
    if m.nonlinearity.lower() != 'swish':
      raise NotImplementedError('NCSNpp: engine implements the swish (SiLU) nonlinearity only')
    assert emb != 'fourier' or config.training.continuous, "Fourier features are only used for continuous training."
    self.register_buffer('sigmas', torch.tensor(utils.get_sigmas(config)))   # fp64, as ncsnpp.py:42
    self.embedding_type = emb
    self.precision = (precision or getattr(m, 'precision', 'tf32')).lower()
    self.keep_activations = bool(keep_activations)
    self.lanes = int(getattr(m, 'lanes', lanes))   # 2: evaluate batches >= 128 as two half-batch lanes on two streams
    # per-engine execution options (fields of b200_ncsnpp_config; nothing is read from the environment)
    self.cuda_core_head = bool(getattr(m, 'cuda_core_head', False) if cuda_core_head is None else cuda_core_head)
    # GroupNorm+SiLU of the tensor-core layers runs as a stand-alone streaming pass (True, default).  The convolution that
    # applied it on load (False) is not part of this build, so False is rejected rather than silently ignored.
    # (2: separate passes also in front of the memory-bound few-channel convolutions of the nf = 16 networks, which
    # otherwise normalise on load in tf32 mode - csrc/conv_lowc.cu; kept for A/B tests)
    sg = getattr(m, 'separate_groupnorm', True) if separate_groupnorm is None else separate_groupnorm
    if not sg:
      raise ValueError('NCSNpp: separate_groupnorm=False (GroupNorm applied on load by the tensor-core convolution) is not '
                       'available in this build; use True (separate pass) or 2')
    self.separate_groupnorm = 2 if (not isinstance(sg, bool) and sg == 2) else True
    # programmatic dependent launch between the kernels of a forward / PC iteration (common.cuh)
    self.pdl = bool(getattr(m, 'pdl', PDL_DEFAULT) if pdl is None else pdl)
    # halo form of the 3x3 tensor-core mainloop (csrc/gemm_tc.cu): True (default) = in the swapped-operand kernel, False =
    # nine shifted tile loads per channel chunk (kept for A/B); an int is the raw b200_ncsnpp_config.no_halo (tests: 8)
    hv = getattr(m, 'halo', HALO_DEFAULT) if halo is None else halo
    self.halo = hv if (isinstance(hv, int) and not isinstance(hv, bool)) else bool(hv)   # int: raw b200_ncsnpp_config.no_halo
    nf, ch_mult, nrb = m.nf, tuple(m.ch_mult), m.num_res_blocks
    L = len(ch_mult)
    all_res = [config.data.image_size // (2 ** i) for i in range(L)]
    channels = config.data.num_channels
    init_scale = m.init_scale
    temb_dim = nf * 4
    if emb == 'fourier':
      mods = [_Fourier(nf, m.fourier_scale), _dense(2 * nf, temb_dim), _dense(temb_dim, temb_dim)]
    else:
      # Sinusoidal embedding of the time label (models/layers.py:515-529): no parameters.  The frequency table is
      # built with the reference's own torch ops (so the engine multiplies by bit-identical fp32 frequencies) and kept
      # as a non-persistent buffer: it is not a state_dict key of the reference.
      mods = [_dense(nf, temb_dim), _dense(temb_dim, temb_dim)]
      half = nf // 2
      if nf % 2 or half < 2:
        raise NotImplementedError('NCSNpp: positional embedding needs an even nf >= 4')
      import math
      f = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000) / (half - 1)))
      self.register_buffer('pos_freqs', f, persistent=False)
    mods.append(_conv(channels, nf, 3))
    hs_c = [nf]
    in_ch, pyr_ch = nf, channels
    for lvl in range(L):
      for _ in range(nrb):
        out_ch = nf * ch_mult[lvl]
        mods.append(_resblock(in_ch, out_ch, temb_dim, init_scale))
        in_ch = out_ch
        if all_res[lvl] in m.attn_resolutions:
          mods.append(_attn(in_ch, init_scale))
        hs_c.append(in_ch)
      if lvl != L - 1:
        mods.append(_resblock(in_ch, in_ch, temb_dim, init_scale, down=True))
        if m.progressive_input.lower() == 'input_skip':
          mods.append(_combine(channels, in_ch))
        elif m.progressive_input.lower() == 'residual':
          mods.append(_pyramid_down(pyr_ch, in_ch))
          pyr_ch = in_ch
        hs_c.append(in_ch)
    in_ch = hs_c[-1]
    mods += [_resblock(in_ch, in_ch, temb_dim, init_scale), _attn(in_ch, init_scale),
             _resblock(in_ch, in_ch, temb_dim, init_scale)]
    for lvl in reversed(range(L)):
      for _ in range(nrb + 1):
        out_ch = nf * ch_mult[lvl]
        mods.append(_resblock(in_ch + hs_c.pop(), out_ch, temb_dim, init_scale))
        in_ch = out_ch
      if all_res[lvl] in m.attn_resolutions:
        mods.append(_attn(in_ch, init_scale))
      if m.progressive.lower() == 'output_skip':      # ncsnpp.py:190-203
        mods.append(_gn(in_ch))
        mods.append(_conv(in_ch, channels, 3, init_scale))
      if lvl != 0:
        mods.append(_resblock(in_ch, in_ch, temb_dim, init_scale, up=True))
    assert not hs_c
    if m.progressive.lower() != 'output_skip':
      mods.append(_gn(in_ch))
      mods.append(_conv(in_ch, channels, 3, init_scale))
    self.all_modules = nn.ModuleList(mods)
    self._engine = None        # (handle, blob, workspace, batch, weights_version)
    self._weights_version = 0
    self._link_parameters()    # lets models.ema.ExponentialMovingAverage tell this module to repack
    # fires for direct loads and for loads through a wrapper (DataParallel(model).load_state_dict calls
    # _load_from_state_dict on the children, not the override below)
    self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate_weights())

  # ---- native engine plumbing ------------------------------------------------
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
    c.skip_rescale, c.conditional = int(bool(m.skip_rescale)), int(bool(m.conditional))
    c.progressive_input = {'none': 0, 'residual': 1, 'input_skip': 2}[m.progressive_input.lower()]
    c.progressive = 1 if m.progressive.lower() == 'output_skip' else 0
    c.pdl = int(self.pdl)
    c.no_halo = self.halo if (isinstance(self.halo, int) and not isinstance(self.halo, bool)) else int(not self.halo)
    c.fir_taps = len(m.fir_kernel)
    for i, v in enumerate(m.fir_kernel):
      c.fir_kernel[i] = float(v)
    if self.precision not in ('tf32', 'fp32', 'f16'):
      raise ValueError(f"precision must be 'tf32', 'fp32' or 'f16', got {self.precision!r}")
    c.precision = {'tf32': 0, 'fp32': 1, 'f16': 2}[self.precision]
    c.keep_activations = int(self.keep_activations)
    c.lanes = self.lanes
    c.cuda_core_head = int(self.cuda_core_head)
    c.separate_groupnorm = int(self.separate_groupnorm)
    c.embedding_type = 1 if self.embedding_type == 'positional' else 0
    c.naive_resample = 0 if m.fir else 1
    return c

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
    import weakref
    ref = weakref.ref(self)
    for p in self.parameters():
      p._b200_owner = ref

  def load_state_dict(self, state_dict, strict=True, **kw):
    sd = {(k[7:] if k.startswith('module.') else k): v for k, v in state_dict.items()}
    return super().load_state_dict(sd, strict=strict, **kw)   # the post hook below invalidates the packed weights

  def _release(self):
    """Destroy the native engine.  Every cached PC plan holds a pointer to it, so they are released first."""
    for plan in self.__dict__.get('_pc_plans', {}).values():
      plan._release()
    if self._engine is not None:
      _lib.load().b200_ncsnpp_destroy(self._engine['h'])
      self._engine = None

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

  def engine(self, batch, device):
    """Create / re-plan the native engine for ``batch`` images on ``device``.  ``eng['gen']`` is a monotonically
    increasing plan generation: it changes whenever the engine, its workspace or its plan is rebuilt, which is what
    dependants (captured CUDA graphs in ``native.PcPlan``) key their validity on."""
    device = self._explicit_device(device)
    eng = self._engine
    if eng is not None and (eng['device'] != device or eng['precision'] != self.precision):
      self._release()
      eng = None
    if eng is None:
      h = ctypes.c_void_p()
      cfg = self._native_config()
      _lib.call('b200_ncsnpp_create', ctypes.byref(cfg), ctypes.byref(h))
      nbytes = _lib.load().b200_ncsnpp_weights_bytes(h)
      blob = torch.zeros(nbytes // 4 + 64, dtype=torch.float32, device=device)
      _lib.call('b200_ncsnpp_bind_weights', h, _lib.ptr(blob))
      self._generation = getattr(self, '_generation', 0) + 1
      eng = dict(h=h, blob=blob, ws=None, batch=0, wver=-1, device=device, precision=self.precision,
                 table=self._param_table(h), gen=self._generation)
      self._engine = eng
    if eng['wver'] != self._weights_version:
      sd = dict(self.named_parameters())
      if self.embedding_type == 'positional':
        sd['pos_freqs'] = self.pos_freqs
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
      self._generation += 1
      eng['gen'] = self._generation
    return eng

  def forward(self, x, time_cond, labels_uniform=False):
    if not x.is_cuda:
      raise RuntimeError('NCSNpp (score_sde_pytorch_b200) runs on CUDA devices only: there is no CPU path; '
                         'move the model and inputs to a CUDA device (the PyTorch restatement in oracle/ is test-only)')
    if x.dim() != 4 or x.shape[1] != self.config.data.num_channels or x.shape[2] != self.config.data.image_size \
        or x.shape[3] != self.config.data.image_size:
      raise RuntimeError(f'NCSNpp: input shape {tuple(x.shape)} does not match the configured image geometry')
    with torch.cuda.device(x.device):
      eng = self.engine(x.shape[0], x.device)
      xin = x.detach().to(torch.float32).contiguous()
      lab = time_cond.detach().to(device=x.device, dtype=torch.float32).contiguous()
      if lab.numel() != x.shape[0]:
        raise RuntimeError(f'NCSNpp: time_cond has {lab.numel()} entries for a batch of {x.shape[0]}')
      out = torch.empty_like(xin)
      _lib.call('b200_ncsnpp_forward', eng['h'], _lib.ptr(xin), _lib.ptr(lab), int(bool(labels_uniform)),
                _lib.ptr(out), _lib.stream_ptr(x.device))
    return out

  def activation_range_report(self, x, time_cond, limit=65504.0):
    """Largest magnitude of every module output of one evaluation, measured with an fp32-range (`'tf32'`) copy of this
    network.  `precision='f16'` stores the operands of every contraction - normalised activations, but also the raw block
    inputs of the skip projections - as IEEE fp16, which assumes |value| < 65504 (and loses precision below 6e-5);
    random-init and normalised activations are far inside, a trained checkpoint can be checked with this before it is
    sampled in fp16 mode.  Returns ``{'max_abs': {module_index: float}, 'worst': (index, value), 'fits_f16': bool}``."""
    probe = NCSNpp(self.config, precision='tf32', keep_activations=True, separate_groupnorm=True, pdl=False).to(x.device)
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
    buf = torch.empty(0, device=eng['device'])
    # query shape with a first call into a generous buffer sized from the workspace
    buf = torch.empty(min(cap, eng['ws'].numel()), dtype=torch.float32, device=eng['device'])
    _lib.call('b200_ncsnpp_tap', eng['h'], module_index, _lib.ptr(buf), buf.numel(), shape, _lib.stream_ptr(eng['device']))
    n = shape[0] * shape[1] * shape[2] * shape[3]
    return buf[:n].reshape(shape[0], shape[1], shape[2], shape[3]).clone()

  def launches_per_forward(self):
    return int(_lib.load().b200_ncsnpp_launches_per_forward(self._engine['h'])) if self._engine else 0

  def op_names(self):
    """Shape labels of the ops of the bound plan, in execution order (b200_ncsnpp_op_info); empty before the first call."""
    if not self._engine:
      return []
    import ctypes
    h = self._engine['h']
    n = int(_lib.load().b200_ncsnpp_num_ops(h))
    buf, kind, fl = ctypes.create_string_buffer(200), ctypes.c_int(), ctypes.c_double()
    names = []
    for i in range(n):
      _lib.call('b200_ncsnpp_op_info', h, i, buf, 200, ctypes.byref(kind), ctypes.byref(fl))
      names.append(buf.value.decode())
    return names
