"""`-m gpu`: precision='tf32x3' (split TF32 on the tensor cores) against float64 runs of the oracle networks, forward-mode AD
of the strict-fp32 oracle, the reference's bits/dim fixture (tests/golden/likelihood_tiny.npz), the engine's own fp32 mode
and the strict-fp32 oracle's PC sampler."""
import numpy as np
import pytest
import torch

from ddpm_helpers import golden_config as ddpm_config, seeded_ddpm
from helpers import golden, golden_config, seeded_model, rel_l2
from oracle import ddpm_oracle as DO, ncsnpp_oracle as NO, sampling_oracle as SO
from score_sde_pytorch_b200 import configs

pytestmark = pytest.mark.gpu
TOL = 1e-4          # the bound 'fp32' mode is held to


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


@pytest.fixture
def oracle64(monkeypatch):
  """The oracle networks in float64: their two float32 constants (the FIR taps, the sinusoidal frequencies) follow the
  input's dtype."""
  up, te = NO.upfirdn2d_native, NO.timestep_embedding
  monkeypatch.setattr(NO, 'upfirdn2d_native', lambda x, k, **kw: up(x, k.to(x.dtype), **kw))
  te64 = lambda t, dim, **kw: te(t, dim, **kw).double()
  monkeypatch.setattr(NO, 'timestep_embedding', te64)
  monkeypatch.setattr(DO, 'timestep_embedding', te64)

  def run(name, sd, cfg, x, labels):
    fwd = DO.ddpm_forward if name in ('cifar10_ddpm', 'tiny_ddpm') else NO.ncsnpp_forward
    with torch.no_grad():
      return fwd({k: v.double() for k, v in sd.items()}, cfg, x.double(), labels.double())
  return run


NETS = {
    'cifar10_ve': (lambda: golden_config('cifar10_ve'), seeded_model),
    'cifar10_ddpmpp': (lambda: golden_config('cifar10_ddpmpp'), seeded_model),
    'cifar10_ddpm': (lambda: ddpm_config('cifar10'), seeded_ddpm),
    'tiny_progressive': (lambda: golden_config('tiny_progressive'), seeded_model),
    'tiny_ddpm': (configs.tiny_ddpm, seeded_ddpm),
    'tiny_ddpmpp': (configs.tiny_ddpmpp, seeded_model),
}


def net(name, dev, **kw):
  cfg_fn, ctor = NETS[name]
  cfg = cfg_fn()
  return cfg, ctor(cfg, **kw).to(dev)


def inputs(cfg, dev, batch, seed=11):
  g = torch.Generator().manual_seed(seed)
  R, C = cfg.data.image_size, cfg.data.num_channels
  x = torch.randn(batch, C, R, R, generator=g).to(dev)
  v = torch.randn(batch, C, R, R, generator=g).to(dev)
  if cfg.model.name == 'ddpm' or getattr(cfg.model, 'embedding_type', 'fourier') == 'positional':
    labels = torch.tensor([3., 150., 600., 990.][:batch], device=dev)      # t * 999
  else:
    labels = torch.tensor([0.05, 0.9, 7., 40.][:batch], device=dev)        # sigma
  return x, v, labels


@pytest.mark.parametrize('name', ['cifar10_ve', 'cifar10_ddpmpp', 'cifar10_ddpm', 'tiny_progressive'])
def test_one_evaluation_matches_float64_oracle(dev, oracle64, name):
  cfg, _ = net(name, dev, precision='tf32')
  x, _, labels = inputs(cfg, dev, 4)
  ys, sd = {}, None
  for precision in ('tf32', 'tf32x3', 'fp32'):
    cfg, model = net(name, dev, precision=precision)
    sd = model.state_dict()
    with torch.no_grad():
      ys[precision] = model(x, labels)
    del model
  ref = oracle64(name, sd, cfg, x, labels)
  e = {p: rel_l2(y, ref) for p, y in ys.items()}
  print(f'{name}: rel-L2 vs float64 oracle ' + ', '.join(f'{p} {v:.2e}' for p, v in e.items()))
  assert e['tf32x3'] <= TOL and 20 * e['tf32x3'] <= e['tf32']


@pytest.mark.parametrize('name', ['tiny_ddpm', 'tiny_ddpmpp'])
def test_per_module_taps_match_oracle(dev, name):
  cfg, model = net(name, dev, precision='tf32x3', keep_activations=True)
  x, _, labels = inputs(cfg, dev, 2)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  fwd = DO.ddpm_forward if name == 'tiny_ddpm' else NO.ncsnpp_forward
  taps = {}
  with torch.no_grad():
    fwd(sd, cfg, x, labels, taps=taps)
    model(x, labels)
  rows = []
  for i, t in sorted(taps.items()):
    if t.dim() != 4:
      continue
    try:
      rows.append((i, rel_l2(model.tap(i), t)))
    except RuntimeError:
      continue                      # modules whose output the engine never materialises
  assert len(rows) > 5
  bad = [r for r in rows if not r[1] <= TOL]
  assert not bad, f'diverging module outputs (index, rel-L2): {bad[:6]}'


@pytest.mark.parametrize('name', ['cifar10_ddpm', 'cifar10_ddpmpp'])
def test_whole_network_jvp_matches_oracle_at_cifar10_size(dev, name):
  cfg, model = net(name, dev, precision='tf32x3')
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  fwd = DO.ddpm_forward if name == 'cifar10_ddpm' else NO.ncsnpp_forward
  x, v, labels = inputs(cfg, dev, 2)
  with torch.no_grad():
    y_ref, jv_ref = torch.func.jvp(lambda xx: fwd(sd, cfg, xx, labels), (x,), (v,))
    y, jv = model.jvp(x, labels, v)
  e_y, e_jv = rel_l2(y, y_ref), rel_l2(jv, jv_ref)
  print(f'{name} [tf32x3] jvp: rel-L2 out {e_y:.3e}, J v {e_jv:.3e}')
  assert e_y <= TOL and e_jv <= TOL
  names = model.op_names(tangent=True)
  assert any(n.startswith('tangent[separate]: gn_tangent') for n in names)
  assert any('3xtf32' in n for n in names if n.startswith('tangent[separate]: conv'))


def likelihood_setup(name, sde_name, hutch, dev, precision):
  from score_sde_pytorch_b200 import sde_lib
  g = golden('likelihood_tiny.npz')
  cfg, model = net(name, dev, precision=precision)
  key = f'{name}_{sde_name}_{hutch}'
  data = torch.from_numpy(g[f'{name}_data']).to(dev)
  eps = torch.from_numpy(g[key + '_eps']).to(dev)
  inv = (lambda v: (v + 1.) / 2.) if cfg.data.centered else (lambda v: v)
  sde = sde_lib.VPSDE(0.1, 20., 1000) if sde_name == 'vp' else sde_lib.subVPSDE(0.1, 20., 1000)
  return g, key, model, data, eps, inv, sde


@pytest.mark.parametrize('hutch', ['rademacher', 'gaussian'])
@pytest.mark.parametrize('sde_name', ['vp', 'subvp'])
@pytest.mark.parametrize('name', ['tiny_ddpm', 'tiny_ddpmpp'])
def test_likelihood_matches_reference_golden_and_fp32(dev, name, sde_name, hutch):
  from score_sde_pytorch_b200 import likelihood
  g, key, model, data, eps, inv, sde = likelihood_setup(name, sde_name, hutch, dev, 'tf32x3')
  fn = likelihood.get_likelihood_fn(sde, inv)
  bpd, _, nfe = fn(model, data, epsilon=eps)
  assert fn.last_stats['solver'] == 'device'
  ref_bpd = g[key + '_bpd']
  e = float(np.max(np.abs(bpd.cpu().numpy() - ref_bpd) / np.abs(ref_bpd)))
  print(f'{key} [tf32x3]: bpd {bpd.tolist()} golden {ref_bpd.tolist()} (rel {e:.2e}); nfe {nfe} / {int(g[key + "_nfe"])}')
  assert e < 1e-2                   # the bound of the fp32 mode (test_gpu_likelihood.py)
  # at rtol = atol = 1e-3 against the engine's fp32 mode on the same draw
  fn3 = likelihood.get_likelihood_fn(sde, inv, rtol=1e-3, atol=1e-3)
  bpd3, _, nfe3 = fn3(model, data, epsilon=eps)
  assert fn3.last_stats['solver'] == 'device'
  _, _, model32, _, _, _, _ = likelihood_setup(name, sde_name, hutch, dev, 'fp32')
  bpd32, _, nfe32 = fn3(model32, data, epsilon=eps)
  e32 = ((bpd3 - bpd32).abs() / bpd32.abs()).max().item()
  print(f'  rtol=atol=1e-3: nfe {nfe3} vs fp32 {nfe32}, bpd rel {e32:.2e}')
  assert abs(nfe3 - nfe32) <= 0.02 * nfe32 and e32 <= 1e-3


def test_native_pc_loop_matches_strict_fp32_oracle(dev):
  from score_sde_pytorch_b200 import native, sampling, sde_lib
  cfg, model = net('cifar10_ve', dev, precision='tf32x3')
  sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
  sde, osde = sde_lib.VESDE(0.01, 50, 1000), SO.VE(0.01, 50, 1000)
  shape, N = (64, 3, 32, 32), 10
  torch.manual_seed(2)
  x0 = sde.prior_sampling(shape).to(dev)
  plan = native.match_pc_plan(sde=sde, model=model, predictor=sampling.ReverseDiffusionPredictor,
                              corrector=sampling.LangevinCorrector, shape=shape, snr=0.16, n_steps=1,
                              probability_flow=False, continuous=True, eps=1e-5, device=dev)
  torch.cuda.manual_seed(3)
  _, xm = plan.run(x0, first_step=0, num_steps=N)
  torch.cuda.synchronize()
  with torch.no_grad():
    torch.cuda.manual_seed(3)
    r, _ = SO.pc_sample(osde, lambda a, l: NO.ncsnpp_forward(sd, cfg, a, l), shape, eps=1e-5, device=dev, x_init=x0, num_iters=N)
  e = rel_l2(xm, r)
  print(f'NCSN++ VE PC loop [tf32x3] {N} steps, batch 64: rel-L2 vs strict-fp32 oracle {e:.2e}')
  assert e <= TOL


@pytest.mark.parametrize('name', ['cifar10_ve', 'cifar10_ddpm'])
def test_plans_run_attention_as_separate_contractions_and_carry_the_mode_tag(dev, name):
  cfg, model = net(name, dev, precision='tf32x3')
  x, _, labels = inputs(cfg, dev, 2)
  with torch.no_grad():
    model(x, labels)
  names = model.op_names()
  assert not any('attention core' in n or 'attn_small' in n for n in names)
  contractions = [n for n in names if n.startswith(('conv', 'gemm')) and '[' in n and 'cuda-core' not in n and 'small-n' not in n]
  assert contractions and all('3xtf32' in n for n in contractions), [n for n in contractions if '3xtf32' not in n][:4]
  assert any(n.startswith('split 3xtf32') for n in names)
  assert any(n.startswith('softmax') for n in names)
