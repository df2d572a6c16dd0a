"""Host driver of the native predictor–corrector loop.

``match_pc_plan`` decides whether a ``(sde, model, predictor, corrector)``
combination handed to :func:`sampling.get_pc_sampler` is one the sm_90a engine
implements end to end; if so it returns a :class:`PcPlan` whose ``run(x)``
executes all ``sde.N`` iterations on the device (one CUDA-graph replay per
iteration, noise from the in-kernel Philox stream that reproduces
``torch.randn_like`` under the current CUDA generator state).  Otherwise it
returns ``None`` and the caller runs the generic host loop.

What the loop computes per iteration ``i`` (``t_i = linspace(T, eps, N)[i]``),
citing the reference statements it replaces:

* corrector (``sampling.py:262-282``): ``g = s(x,t_i)``, ``z ~ N(0,I)``,
  ``eps = 2 alpha_i (snr * mean_b||z_b|| / mean_b||g_b||)^2``,
  ``x = x + eps g + sqrt(2 eps) z``;
* predictor, as the affine update ``x_mean = pa_i x + pb_i net(x, label_i)``,
  ``x = x_mean + pc_i z`` which covers ``ReverseDiffusionPredictor``
  (``sampling.py:195-200`` with ``sde_lib.py:102-107`` and the SDE's
  ``discretize``) and ``EulerMaruyamaPredictor`` (``sampling.py:181-187`` with
  ``sde_lib.py:93-100``), with or without ``probability_flow``;
* score adapter (``models/utils.py:129-178``): ``score = score_scale_i * net_out``
  with ``label_i = sigma(t_i)`` / ``score_scale = 1`` for VE and ``label_i = 999 t_i``
  / ``score_scale = -1/std(t_i)`` for (sub-)VP.

The per-step scalar tables are built here with the same torch fp32 ops the
reference evaluates inside its loop, then handed to the C ABI as host arrays.

``match_pc_plan(..., constraint='inpaint' | 'colorize')`` returns a
:class:`ConstrainedPcPlan` for ``controllable_generation``: the same loop with
the data-consistency blend (``controllable_generation.py:43-52`` / ``:137-146``)
after the corrector block and after the predictor block of every iteration.
"""
import ctypes

import numpy as np
import torch

from . import _lib, sde_lib


def _unwrap(model):
  return model.module if isinstance(model, torch.nn.DataParallel) else model


def build_tables(sde, predictor_kind, corrector_kind, probability_flow, eps, snr=0.16):
  """Per-step scalars (float32 numpy arrays of length N).  ``predictor_kind`` in
  {'none','reverse_diffusion','euler_maruyama','ancestral_sampling'}, ``corrector_kind`` in {'none','langevin','ald'}.
  Every update the native loop runs is affine in (x, network output, noise): x_mean = a x + b out, x = x_mean + c z;
  the tables are evaluated with the SDE's own torch ops, in the reference's operation order."""
  N, T = sde.N, sde.T
  t = torch.linspace(T, eps, N)
  half = 0.5 if probability_flow else 1.0
  ones = torch.ones(N)
  if isinstance(sde, sde_lib.VESDE):
    label = sde.marginal_prob(torch.zeros(N, 1, 1, 1), t)[1]            # sigma(t), models/utils.py:164-165
    ss = ones.clone()
    alpha = ones.clone()                                               # sampling.py:270-271
    if predictor_kind == 'reverse_diffusion':
      _, G = sde.discretize(torch.zeros(N, 1, 1, 1), t)                # sde_lib.py:246-254
      pa, pb, pc = ones.clone(), G ** 2 * half, G
    elif predictor_kind == 'euler_maruyama':
      _, g = sde.sde(torch.zeros(N, 1, 1, 1), t)                       # sde_lib.py:224-231
      pa, pb, pc = ones.clone(), g ** 2 * half * (1. / N), g * float(np.sqrt(1. / N))
    elif predictor_kind == 'ancestral_sampling':                       # sampling.py:213-223
      idx = (t * (N - 1) / T).long()
      sigma = sde.discrete_sigmas[idx]
      adj = torch.where(idx == 0, torch.zeros_like(t), sde.discrete_sigmas[idx - 1])
      pa, pb = ones.clone(), sigma ** 2 - adj ** 2
      pc = torch.sqrt((adj ** 2 * (sigma ** 2 - adj ** 2)) / (sigma ** 2))
    else:
      pa, pb, pc = ones.clone(), torch.zeros(N), torch.zeros(N)
  else:
    label = t * 999                                                    # models/utils.py:151
    std = sde.marginal_prob(torch.zeros(N, 1, 1, 1), t)[1]             # VP: sqrt(1-e^{2c}); sub-VP: 1-e^{2c}
    ss = -1. / std                                                     # models/utils.py:159
    if isinstance(sde, sde_lib.VPSDE):
      idx = (t * (N - 1) / T).long()
      alpha = sde.alphas[idx]                                          # sampling.py:267-269
    else:
      alpha = ones.clone()
    beta_t = sde.beta_0 + t * (sde.beta_1 - sde.beta_0)
    _, g = sde.sde(torch.zeros(N, 1, 1, 1), t)
    if predictor_kind == 'ancestral_sampling':                         # sampling.py:225-232 (VP only, like the reference)
      b_i = sde.discrete_betas[(t * (N - 1) / T).long()]
      pa, pb, pc = 1. / torch.sqrt(1. - b_i), b_i * ss / torch.sqrt(1. - b_i), torch.sqrt(b_i)
    elif predictor_kind == 'reverse_diffusion' and isinstance(sde, sde_lib.VPSDE):
      idx = (t * (N - 1) / T).long()
      a_i, b_i = sde.alphas[idx], sde.discrete_betas[idx]              # sde_lib.py:155-164
      pa, pb, pc = 2. - torch.sqrt(a_i), b_i * half * ss, torch.sqrt(b_i)
    elif predictor_kind in ('reverse_diffusion', 'euler_maruyama'):
      # default SDE.discretize is Euler–Maruyama with dt = 1/N (sde_lib.py:52-69)
      pa = 1. + 0.5 * beta_t * (1. / N)
      pb = g ** 2 * half * (1. / N) * ss
      pc = g * float(np.sqrt(1. / N))
    else:
      pa, pb, pc = ones.clone(), torch.zeros(N), torch.zeros(N)
  if probability_flow:
    pc = torch.zeros(N)
  f32 = lambda v: np.ascontiguousarray(v.to(torch.float32).numpy())
  out = dict(label=f32(label), score_scale=f32(ss), alpha=f32(alpha), pa=f32(pa), pb=f32(pb), pc=f32(pc))
  if corrector_kind == 'ald':
    # AnnealedLangevinDynamics (sampling.py:299-317): step_size = (snr * std)^2 * 2 * alpha with the marginal std of the
    # step - no norms - so x_mean = x + step_size * score, x = x_mean + sqrt(2 step_size) * z is affine as well
    std = sde.marginal_prob(torch.zeros(N, 1, 1, 1), t)[1]
    step = (snr * std) ** 2 * 2 * alpha
    out.update(ca=f32(ones.clone()), cb=f32(step * ss), cc=f32(torch.sqrt(step * 2)))
  return out


def build_constraint_tables(sde, eps):
  """Per-step scalars of controllable generation's data-consistency blend (float32 numpy arrays of length N):
  ``cm`` and ``cs`` with ``sde.marginal_prob(known, t_i) == (cm[i] * known, cs[i])`` (controllable_generation.py:44-45,
  :138-139).  VE: ``cm = 1``, ``cs = sigma(t)``; (sub-)VP: ``cm = exp(log_mean_coeff(t))`` and the SDE's std."""
  N = sde.N
  t = torch.linspace(sde.T, eps, N)
  cm, cs = sde.marginal_prob(torch.ones(N, 1, 1, 1), t)
  f32 = lambda v: np.ascontiguousarray(v.reshape(N).to(torch.float32).numpy())
  return dict(cm=f32(cm), cs=f32(cs))


class PcPlan:
  """A native PC loop bound to one model, SDE, sampler configuration and batch shape."""

  def __init__(self, model, sde, predictor_kind, corrector_kind, shape, snr, n_steps, probability_flow, eps, device):
    self.model, self.sde, self.shape, self.device = model, sde, tuple(shape), model._explicit_device(device)
    self.predictor_kind, self.corrector_kind = predictor_kind, corrector_kind
    self.snr, self.n_steps, self.probability_flow, self.eps = float(snr), int(n_steps), bool(probability_flow), float(eps)
    self.tables = build_tables(sde, predictor_kind, corrector_kind, probability_flow, eps, snr=float(snr))
    self._pc = None
    self._ws = None
    self._engine_id = None
    self._x = self._xm = None      # persistent state buffers: stable addresses keep the captured graph valid
    self.use_graph = True

  def _release(self):
    if self._pc is not None:
      _lib.load().b200_pc_destroy(self._pc)
      self._pc = None

  def __del__(self):
    try:
      self._release()
    except Exception:
      pass

  def _ensure(self):
    eng = self.model.engine(self.shape[0], self.device)
    key = eng['gen']   # monotonically increasing: bumped on engine re-create, workspace realloc and re-plan
    if self._pc is not None and self._engine_id == key:
      return eng
    self._release()
    cfg = _lib.PcConfig()
    cfg.n_steps = self.sde.N
    cfg.corrector = {'langevin': 1, 'ald': 2}.get(self.corrector_kind, 0)
    cfg.predictor = 0 if self.predictor_kind == 'none' else 1
    cfg.n_corrector_steps = self.n_steps
    cfg.snr = self.snr
    fp = ctypes.POINTER(ctypes.c_float)
    for k in ('label', 'score_scale', 'alpha', 'pa', 'pb', 'pc', 'ca', 'cb', 'cc', 'cm', 'cs'):
      if k in self.tables:
        setattr(cfg, k, self.tables[k].ctypes.data_as(fp))
    self._configure(cfg)
    h = ctypes.c_void_p()
    _lib.call('b200_pc_create', eng['h'], ctypes.byref(cfg), self.shape[0], ctypes.byref(h))
    self._pc = h
    need = _lib.load().b200_pc_workspace_bytes(h)
    self._ws = torch.zeros(need // 4 + 64, dtype=torch.float32, device=self.device)
    if self._x is None:
      self._x = torch.empty(self.shape, dtype=torch.float32, device=self.device)
      self._xm = torch.empty(self.shape, dtype=torch.float32, device=self.device)
    _lib.call('b200_pc_bind_workspace', h, _lib.ptr(self._ws), self._ws.numel() * 4, _lib.stream_ptr(self.device))
    self._bind(h)
    self._engine_id = key
    return eng

  def _configure(self, cfg):
    """Hook for variants: fill further ``PcConfig`` fields before the plan is created."""

  def _bind(self, h):
    """Hook for variants: bind further device buffers once the workspace is bound."""

  def _generator(self):
    idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
    return torch.cuda.default_generators[idx]

  def run(self, x, first_step=0, num_steps=None, clone=True):
    """Run iterations ``[first_step, first_step+num_steps)`` from state ``x`` (NCHW; a pinned host
    tensor is uploaded asynchronously).  Consumes the CUDA generator exactly as the reference loop
    would (same seed/offset bookkeeping).  Returns ``(x, x_mean)`` — fresh tensors, or with
    ``clone=False`` the plan's persistent buffers (overwritten by the next call)."""
    with torch.cuda.device(self.device):
      self._ensure()
      num_steps = self.sde.N - first_step if num_steps is None else num_steps
      self._x.copy_(x.detach().reshape(self.shape), non_blocking=True)
      self._xm.copy_(self._x)
      x, x_mean = self._x, self._xm
      gen = self._generator()
      seed, offset = gen.initial_seed(), gen.get_offset()
      off_out = ctypes.c_ulonglong(0)
      _lib.call('b200_pc_run', self._pc, _lib.ptr(x), _lib.ptr(x_mean), int(first_step), int(num_steps),
                ctypes.c_ulonglong(seed), ctypes.c_ulonglong(offset), ctypes.byref(off_out),
                int(self.use_graph), _lib.stream_ptr(self.device))
      gen.set_offset(int(off_out.value))
      if clone:
        x, x_mean = x.clone(), x_mean.clone()
    return x, x_mean

  def step_external(self, x, x_mean, step, noise_c, noise_p):
    """One iteration with caller-provided noise (parity tests against a CPU-generated trajectory)."""
    with torch.cuda.device(self.device):
      self._ensure()
      _lib.call('b200_pc_step_external', self._pc, _lib.ptr(x), _lib.ptr(x_mean), int(step),
                _lib.ptr(noise_c), _lib.ptr(noise_p), _lib.stream_ptr(self.device))
    return x, x_mean

  def launches_per_step(self):
    self._ensure()
    return int(_lib.load().b200_pc_launches_per_step(self._pc))


class ConstrainedPcPlan(PcPlan):
  """A :class:`PcPlan` for controllable generation: after the corrector block and after the predictor block of every
  iteration the state is blended with a fresh draw from the data marginal (``constraint`` 'inpaint' or 'colorize',
  controllable_generation.py:43-52 / :137-146).  ``known`` and ``mask`` live in persistent device buffers, so the
  captured graph stays valid from one call to the next.  ``channels_last``: the state the reference loop draws its
  ``randn_like`` noise on is channels-last, so torch fills it in NHWC memory order (the colorizer's einsum output)."""

  def __init__(self, model, sde, predictor_kind, corrector_kind, shape, snr, n_steps, probability_flow, eps, device,
               constraint, channels_last=False):
    if constraint not in ('inpaint', 'colorize'):
      raise ValueError(f'constraint must be inpaint or colorize, got {constraint!r}')
    super().__init__(model, sde, predictor_kind, corrector_kind, shape, snr, n_steps, probability_flow, eps, device)
    self.constraint, self.channels_last = constraint, bool(channels_last)
    self.tables.update(build_constraint_tables(sde, eps))
    self._known = self._mask = None

  def _configure(self, cfg):
    cfg.constraint = 1 if self.constraint == 'inpaint' else 2
    cfg.noise_nhwc = int(self.channels_last)
    if self.constraint == 'colorize':
      from .controllable_generation import _M
      m = torch.tensor(_M)
      cfg.color_m[:] = m.flatten().tolist()
      cfg.color_minv[:] = torch.inverse(m).flatten().tolist()   # the reference's invM, computed the same way

  def _bind(self, h):
    if self._known is None:
      self._known = torch.empty(self.shape, dtype=torch.float32, device=self.device)
      self._mask = torch.empty(self.shape, dtype=torch.float32, device=self.device)
    _lib.call('b200_pc_bind_constraint', h, _lib.ptr(self._known), _lib.ptr(self._mask), _lib.stream_ptr(self.device))

  def run(self, x, known, mask, first_step=0, num_steps=None, clone=True):
    """:meth:`PcPlan.run` with the blend's ``known`` (the data; for colorization ``decouple(gray)``) and ``mask``
    (1 where ``known`` is imposed).  A mask that broadcasts to the batch shape is expanded here."""
    with torch.cuda.device(self.device):
      self._ensure()
      self._known.copy_(known.detach().expand(self.shape))
      self._mask.copy_(mask.detach().expand(self.shape))
      return super().run(x, first_step=first_step, num_steps=num_steps, clone=clone)


def _kind_of_predictor(predictor):
  from . import sampling
  if predictor is None or predictor is sampling.NonePredictor:
    return 'none'
  if predictor is sampling.ReverseDiffusionPredictor:
    return 'reverse_diffusion'
  if predictor is sampling.EulerMaruyamaPredictor:
    return 'euler_maruyama'
  if predictor is sampling.AncestralSamplingPredictor:
    return 'ancestral_sampling'
  return None   # user classes run on the generic host loop


def _kind_of_corrector(corrector):
  from . import sampling
  if corrector is None or corrector is sampling.NoneCorrector:
    return 'none'
  if corrector is sampling.LangevinCorrector:
    return 'langevin'
  if corrector is sampling.AnnealedLangevinDynamics:
    return 'ald'
  return None


def match_pc_plan(sde, model, predictor, corrector, shape, snr, n_steps, probability_flow, continuous, eps, device,
                  constraint=None, channels_last=False):
  """Return a :class:`PcPlan` when the native engine implements this sampler, else ``None``.  With ``constraint``
  'inpaint' or 'colorize' (controllable generation) the plan is a :class:`ConstrainedPcPlan`; the rules are the same."""
  from .models._engine import EngineModel
  model = _unwrap(model)
  if not isinstance(model, EngineModel) or torch.device(device).type != 'cuda' or not torch.cuda.is_available():
    return None
  if not model.takes_time_labels:   # NCSNv2 evaluates noise-level indices: the host loop calls its forward
    return None
  if type(sde) not in (sde_lib.VESDE, sde_lib.VPSDE, sde_lib.subVPSDE) or not continuous:
    return None
  pk, ck = _kind_of_predictor(predictor), _kind_of_corrector(corrector)
  if pk is None or ck is None or (pk == 'none' and ck == 'none'):
    return None
  if ck in ('langevin', 'ald') and isinstance(sde, sde_lib.subVPSDE):
    return None   # the reference itself fails here (subVPSDE has no .alphas, sampling.py:267-269, :303-305)
  if pk == 'ancestral_sampling' and (isinstance(sde, sde_lib.subVPSDE) or probability_flow):
    return None   # the reference raises for these (sampling.py:208-211): let its host-side class do so
  if ck in ('langevin', 'ald') and n_steps < 1:
    return None
  # keyed on the SDE's parameters (not id(sde): a freed-and-reallocated SDE object must not hit a stale plan)
  sde_key = (type(sde).__name__, int(sde.N)) + tuple(
      float(getattr(sde, a)) for a in ('sigma_min', 'sigma_max', 'beta_0', 'beta_1') if hasattr(sde, a))
  key = (sde_key, pk, ck, tuple(shape), float(snr), int(n_steps), bool(probability_flow), float(eps),
         str(model._explicit_device(device)))
  if constraint is not None:
    key += (constraint, bool(channels_last))
  cache = model.__dict__.setdefault('_pc_plans', {})
  plan = cache.get(key)
  if plan is None:
    if constraint is None:
      plan = PcPlan(model, sde, pk, ck, shape, snr, n_steps, probability_flow, eps, device)
    else:
      plan = ConstrainedPcPlan(model, sde, pk, ck, shape, snr, n_steps, probability_flow, eps, device, constraint,
                               channels_last)
    cache[key] = plan
  return plan
