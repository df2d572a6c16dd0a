"""`-m gpu`: inpainting and colorization (controllable_generation.py) on the native PC loop.

* which loop runs (``last_stats``) for stock and non-stock combinations;
* native loop against the host loop over the same engine, same seeds: outputs and the CUDA generator offset;
* native loop against the oracle restatement of the reference, in fp32, tf32, f16 and with two lanes;
* graph replay against direct launches, and the refusal of caller-supplied noise on a constrained plan."""
import pytest
import torch

from helpers import golden, golden_config, seeded_model, rel_l2
from oracle import ncsnpp_oracle as NO
from oracle import sampling_oracle as SO

pytestmark = pytest.mark.gpu
TOL_PARITY = 1e-3      # tensor-core operand modes against the strict-fp32 oracle, as in the native PC sampler tests


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


def _sde(kind, N):
  from score_sde_pytorch_b200 import sde_lib
  return {'ve': lambda: sde_lib.VESDE(0.01, 50, N), 'vp': lambda: sde_lib.VPSDE(0.1, 20., N),
          'subvp': lambda: sde_lib.subVPSDE(0.1, 20., N)}[kind]()


def _osde(kind, N):
  return {'ve': lambda: SO.VE(0.01, 50, N), 'vp': lambda: SO.VP(0.1, 20., N), 'subvp': lambda: SO.SubVP(0.1, 20., N)}[kind]()


def _classes(pred, corr):
  from score_sde_pytorch_b200 import sampling
  P = {'reverse_diffusion': sampling.ReverseDiffusionPredictor, 'euler_maruyama': sampling.EulerMaruyamaPredictor,
       'ancestral_sampling': sampling.AncestralSamplingPredictor, 'none': sampling.NonePredictor}[pred]
  C = {'langevin': sampling.LangevinCorrector, 'ald': sampling.AnnealedLangevinDynamics,
       'none': sampling.NoneCorrector}[corr]
  return P, C


def _factory(task, sde, P, C, **kw):
  from score_sde_pytorch_b200 import controllable_generation as CG
  make = CG.get_pc_inpainter if task == 'inpaint' else CG.get_pc_colorizer
  return make(sde, P, C, lambda v: v, **kw)


def _inputs(dev, B=2):
  g = golden('controllable_tiny.npz')
  data, mask, gray = (torch.from_numpy(g[k]).to(dev) for k in ('data', 'mask', 'gray'))
  return data[:B], mask[:B], gray[:B]


def _call(fn, task, model, data, mask, gray, seed):
  torch.manual_seed(seed); torch.cuda.manual_seed(seed)
  out = fn(model, data, mask) if task == 'inpaint' else fn(model, gray)
  return out, torch.cuda.default_generators[0].get_offset()


def _decouple(v):
  from score_sde_pytorch_b200.controllable_generation import _M
  return torch.einsum('bihw,ij->bjhw', v, torch.tensor(_M, device=v.device))


# (sde, predictor, corrector, n_steps_each, probability_flow)
CASES = [('ve', 'reverse_diffusion', 'langevin', 1, False),
         ('ve', 'ancestral_sampling', 'ald', 2, False),
         ('ve', 'none', 'langevin', 2, False),
         ('ve', 'euler_maruyama', 'none', 1, False),
         ('vp', 'reverse_diffusion', 'langevin', 1, False),
         ('vp', 'euler_maruyama', 'ald', 2, False),
         ('vp', 'ancestral_sampling', 'none', 1, False),
         ('subvp', 'reverse_diffusion', 'none', 1, True)]


@pytest.mark.parametrize('task', ['inpaint', 'colorize'])
@pytest.mark.parametrize('case', CASES, ids=['-'.join(map(str, c)) for c in CASES])
def test_native_loop_matches_host_loop_on_the_engine(dev, task, case):
  """Same engine, same seeds: the native loop and the host loop (reached through a user subclass of the predictor) give
  the same x and x_mean to 1e-4 per image and leave the CUDA generator at the same offset."""
  kind, pred, corr, n_each, pflow = case
  N = 6 if kind == 've' else 30   # (sub-)VP: beta_max / N < 1 keeps the discrete alphas positive
  sde = _sde(kind, N)
  P, C = _classes(pred, corr)
  UserP = type('User' + P.__name__, (P,), {})
  model = seeded_model(golden_config('tiny' if kind == 've' else 'tiny_vp'), precision='fp32').to(dev)
  data, mask, gray = _inputs(dev)
  eps = 1e-5 if kind == 've' else 1e-3
  outs = {}
  for denoise in (True, False):
    kw = dict(snr=0.16, n_steps=n_each, probability_flow=pflow, continuous=True, denoise=denoise, eps=eps)
    fn_n, fn_h = _factory(task, sde, P, C, **kw), _factory(task, sde, UserP, C, **kw)
    out_n, off_n = _call(fn_n, task, model, data, mask, gray, 11)
    out_h, off_h = _call(fn_h, task, model, data, mask, gray, 11)
    assert fn_n.last_stats['loop'] == 'native' and fn_h.last_stats['loop'] == 'host'
    assert off_n == off_h, (off_n, off_h)
    assert torch.isfinite(out_n).all()
    e = rel_l2(out_n, out_h)
    print(f'{task} {case} denoise={denoise}: native vs host rel-L2 {e:.2e}, '
          f'{fn_n.last_stats["launches_per_step"]} launches/step')
    assert e <= 1e-4
    outs[denoise] = out_n
  if kind == 've':   # the last mean coefficient is exactly 1: the denoised output carries the data where it is known
    if task == 'inpaint':
      known = mask.bool()
      assert torch.allclose(outs[True][known], data[known], atol=1e-4)
    else:
      assert torch.allclose(_decouple(outs[True])[:, 0], _decouple(gray)[:, 0], atol=1e-4)


def test_non_stock_combinations_run_the_host_loop(dev):
  from score_sde_pytorch_b200 import sampling
  sde = _sde('ve', 3)
  model = seeded_model(golden_config('tiny'), precision='fp32').to(dev)
  data, mask, gray = _inputs(dev)
  cfg = golden_config('tiny')
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}

  class Plain(torch.nn.Module):
    def forward(self, x, labels):
      return NO.ncsnpp_forward(sd, cfg, x, labels)

  class UserCorrector(sampling.LangevinCorrector):
    pass

  for task in ('inpaint', 'colorize'):
    base = dict(snr=0.16, n_steps=1, probability_flow=False, denoise=True, eps=1e-5)
    runs = [(sampling.LangevinCorrector, dict(continuous=True), model, 'native'),
            (UserCorrector, dict(continuous=True), model, 'host'),
            (sampling.LangevinCorrector, dict(continuous=False), model, 'host'),
            (sampling.LangevinCorrector, dict(continuous=True), Plain(), 'host')]
    for C, extra, m, loop in runs:
      fn = _factory(task, sde, sampling.ReverseDiffusionPredictor, C, **base, **extra)
      out, _ = _call(fn, task, m, data, mask, gray, 3)
      assert fn.last_stats['loop'] == loop, (task, C.__name__, extra, type(m).__name__)


ORACLE_CASES = [('ve', 'reverse_diffusion', 'langevin'), ('vp', 'reverse_diffusion', 'langevin'),
                ('subvp', 'euler_maruyama', 'none')]


@pytest.mark.parametrize('task', ['inpaint', 'colorize'])
@pytest.mark.parametrize('case', ORACLE_CASES, ids=['-'.join(c) for c in ORACLE_CASES])
def test_native_loop_matches_oracle_fp32(dev, task, case):
  kind, pred, corr = case
  N = 8 if kind == 've' else 30
  cfg = golden_config('tiny' if kind == 've' else 'tiny_vp')
  model = seeded_model(cfg, precision='fp32').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  net = lambda a, l: NO.ncsnpp_forward(sd, cfg, a, l)
  P, C = _classes(pred, corr)
  eps = 1e-5 if kind == 've' else 1e-3
  kw = dict(snr=0.16, n_steps=1, continuous=True, denoise=True, eps=eps)
  fn = _factory(task, _sde(kind, N), P, C, probability_flow=False, **kw)
  data, mask, gray = _inputs(dev)
  out, off = _call(fn, task, model, data, mask, gray, 21)
  assert fn.last_stats['loop'] == 'native'
  torch.manual_seed(21); torch.cuda.manual_seed(21)
  if task == 'inpaint':
    ref = SO.inpaint_sample(_osde(kind, N), net, data, mask, predictor=pred, corrector=corr, **kw)
  else:
    ref = SO.colorize_sample(_osde(kind, N), net, gray, predictor=pred, corrector=corr, **kw)
  assert torch.cuda.default_generators[0].get_offset() == off
  e = rel_l2(out, ref)
  print(f'{task} {case} fp32: rel-L2 vs oracle {e:.2e}')
  assert e < 2e-4


@pytest.mark.parametrize('task,precision', [('inpaint', 'tf32'), ('colorize', 'f16')])
def test_native_loop_tensor_core_modes_cifar10(dev, task, precision):
  """The CIFAR-10 NCSN++ (VE, reverse diffusion + Langevin) in a tensor-core operand mode against the strict-fp32 oracle."""
  cfg = golden_config('cifar10_ve')
  model = seeded_model(cfg, precision=precision).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  net = lambda a, l: NO.ncsnpp_forward(sd, cfg, a, l)
  N, B = 20, 4
  torch.manual_seed(0)
  data = torch.rand(B, 3, 32, 32, device=dev)
  mask = (torch.rand(B, 1, 32, 32, device=dev) > 0.5).float()
  gray = data.mean(1, keepdim=True).expand(B, 3, 32, 32).contiguous()
  P, C = _classes('reverse_diffusion', 'langevin')
  kw = dict(snr=0.16, n_steps=1, continuous=True, denoise=True, eps=1e-5)
  fn = _factory(task, _sde('ve', N), P, C, probability_flow=False, **kw)
  out, _ = _call(fn, task, model, data, mask, gray, 31)
  assert fn.last_stats['loop'] == 'native'
  torch.manual_seed(31); torch.cuda.manual_seed(31)
  if task == 'inpaint':
    ref = SO.inpaint_sample(_osde('ve', N), net, data, mask, **kw)
  else:
    ref = SO.colorize_sample(_osde('ve', N), net, gray, **kw)
  e = rel_l2(out, ref)
  print(f'{task} CIFAR-10 [{precision}] {N} steps: rel-L2 vs oracle {e:.2e}')
  assert e < TOL_PARITY


def test_native_loop_two_lanes_broadcast_mask_matches_oracle(dev):
  """lanes=2 (batches >= 128 run as two half-batch lanes) with a per-pixel mask broadcast over the channels."""
  cfg = golden_config('tiny')
  model = seeded_model(cfg, precision='fp32', lanes=2).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  net = lambda a, l: torch.cat([NO.ncsnpp_forward(sd, cfg, a[i:i + 64], l[i:i + 64]) for i in range(0, a.shape[0], 64)])
  N, B = 4, 130
  torch.manual_seed(1)
  data = torch.rand(B, 3, 16, 16, device=dev)
  mask = (torch.rand(B, 1, 16, 16, device=dev) > 0.5).float()
  P, C = _classes('reverse_diffusion', 'langevin')
  kw = dict(snr=0.16, n_steps=1, continuous=True, denoise=True, eps=1e-5)
  fn = _factory('inpaint', _sde('ve', N), P, C, probability_flow=False, **kw)
  out, _ = _call(fn, 'inpaint', model, data, mask, None, 41)
  assert fn.last_stats['loop'] == 'native'
  torch.manual_seed(41); torch.cuda.manual_seed(41)
  ref = SO.inpaint_sample(_osde('ve', N), net, data, mask, **kw)
  e = rel_l2(out, ref)
  print(f'inpaint lanes=2 B={B}: rel-L2 vs oracle {e:.2e}')
  assert e < 2e-4


def _plan(model, task, shape, dev):
  from score_sde_pytorch_b200 import native
  P, C = _classes('reverse_diffusion', 'langevin')
  plan = native.match_pc_plan(sde=_sde('ve', 5), model=model, predictor=P, corrector=C, shape=shape, snr=0.16, n_steps=1,
                              probability_flow=False, continuous=True, eps=1e-5, device=dev, constraint=task)
  assert plan is not None
  return plan


@pytest.mark.parametrize('task', ['inpaint', 'colorize'])
def test_graph_replay_is_bit_identical_to_direct_launches(dev, task):
  model = seeded_model(golden_config('tiny'), precision='fp32').to(dev)
  data, mask, gray = _inputs(dev)
  known = data if task == 'inpaint' else _decouple(gray)
  if task == 'colorize':
    mask = torch.zeros_like(gray)
    mask[:, 0] = 1.
  plan = _plan(model, task, data.shape, dev)
  torch.manual_seed(0)
  x0 = torch.randn(data.shape, device=dev) * 50
  res = {}
  for trial, k in enumerate((known, known.flip(0))):   # second trial: same graph, new contents of the bound buffers
    for use_graph in (True, False):
      plan.use_graph = use_graph
      torch.cuda.manual_seed(7)
      res[trial, use_graph] = plan.run(x0, k, mask)
    for a, b in zip(res[trial, True], res[trial, False]):
      assert torch.equal(a, b)
  assert not torch.equal(res[0, True][0], res[1, True][0])


def test_step_external_refuses_a_constrained_plan(dev):
  model = seeded_model(golden_config('tiny'), precision='fp32').to(dev)
  data, mask, _ = _inputs(dev)
  plan = _plan(model, 'inpaint', data.shape, dev)
  x, xm, z = data.clone(), data.clone(), torch.zeros_like(data)
  with pytest.raises(RuntimeError, match='constrained'):
    plan.step_external(x, xm, 0, z, z)


@pytest.mark.parametrize('task', ['inpaint', 'colorize'])
def test_single_image_matches_host_loop(dev, task):
  """Batch 1: the colorizer's einsum returns a contiguous state there, so its draws are in NCHW order (channels-last
  order for larger batches); the plan follows the layout of the state it is given."""
  from score_sde_pytorch_b200 import sampling
  sde = _sde('ve', 6)
  model = seeded_model(golden_config('tiny'), precision='fp32').to(dev)
  data, mask, gray = _inputs(dev, B=1)

  class UserLangevin(sampling.LangevinCorrector):
    pass

  kw = dict(snr=0.16, n_steps=1, probability_flow=False, continuous=True, denoise=True, eps=1e-5)
  fn_n = _factory(task, sde, sampling.ReverseDiffusionPredictor, sampling.LangevinCorrector, **kw)
  fn_h = _factory(task, sde, sampling.ReverseDiffusionPredictor, UserLangevin, **kw)
  out_n, off_n = _call(fn_n, task, model, data, mask, gray, 13)
  out_h, off_h = _call(fn_h, task, model, data, mask, gray, 13)
  assert fn_n.last_stats['loop'] == 'native' and fn_h.last_stats['loop'] == 'host' and off_n == off_h
  e = rel_l2(out_n, out_h)
  print(f'{task} batch 1: native vs host rel-L2 {e:.2e}')
  assert e <= 1e-4
