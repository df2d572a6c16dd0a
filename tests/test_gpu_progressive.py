"""`-m gpu`: the high-resolution NCSN++ family: progressive='output_skip',
progressive_input='input_skip', Combine 'sum' (models/ncsnpp.py:163-166, 190-203, 289-292, 325-341, 366-367;
layerspp.py:44-59) through the engine - against the oracle, against a golden written by the REAL reference
(tools/make_golden_progressive.py), and at full size for the two reference configurations of the family."""
import pytest
import torch

from helpers import golden, golden_config, seeded_model, rel_l2
from oracle import ncsnpp_oracle as NO
from oracle import sampling_oracle as SO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


@pytest.mark.parametrize('precision', ['fp32', 'tf32'])     # (32/64-channel layers: off the fp16 tiling; full-size f16 below)
def test_progressive_tiny_matches_oracle_and_reference_golden(dev, precision):
  g = golden('ncsnpp_tiny_progressive.npz')
  cfg = golden_config('tiny_progressive')
  model = seeded_model(cfg, precision=precision, keep_activations=True).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  x, sigma = torch.from_numpy(g['x']).to(dev), torch.from_numpy(g['sigma']).to(dev)
  taps = {}
  with torch.no_grad():
    ref = NO.ncsnpp_forward(sd, cfg, x, sigma, taps=taps)
    y = model(x, sigma)
  tol_mod, tol_out = (1e-4, 1e-4) if precision == 'fp32' else (5e-3, 2.5e-3)
  rows = []
  for i in sorted(taps):
    if taps[i].dim() != 4:
      continue
    try:
      rows.append((i, rel_l2(model.tap(i), taps[i])))
    except RuntimeError:
      continue
  worst = sorted(rows, key=lambda r: -r[1])[:4]
  e_or, e_gold = rel_l2(y, ref), rel_l2(y, torch.from_numpy(g['y']).to(dev))
  print(f'progressive tiny [{precision}]: rel-L2 vs oracle {e_or:.3e}, vs reference CPU golden {e_gold:.3e}; {len(rows)} module taps, worst {worst}')
  assert len(rows) >= 10
  assert all(r[1] < tol_mod for r in rows), f'worst modules: {worst}'
  assert e_or < tol_out and e_gold < tol_out


def test_progressive_nofir_matches_oracle(dev):
  """fir=False member (avg-pool / nearest pyramids): oracle only - the reference's own Upsample(fir=False) does not run
  on current PyTorch (F.interpolate called with the mode in the scale_factor slot, layerspp.py:116)."""
  from score_sde_pytorch_b200 import configs
  cfg = configs.tiny_progressive(fir=False)
  model = seeded_model(cfg, precision='fp32').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  torch.manual_seed(3)
  x = torch.randn(2, 3, 32, 32, device=dev) * 2
  sigma = torch.tensor([9.0, 0.2], device=dev)
  with torch.no_grad():
    assert rel_l2(model(x, sigma), NO.ncsnpp_forward(sd, cfg, x, sigma)) < 1e-4


def test_few_channel_levels_groupnorm_on_load_matches_oracle(dev):
  """nf = 16 network in tf32 mode: the 16/32-channel 3x3 convolutions run on conv_lowc.cu and apply GroupNorm+SiLU while
  they stage their input.  Held against the oracle at 7.5e-4: the same network with a separate GroupNorm pass in front of
  those convolutions measured 5.3e-4 on these inputs (H100), and the two plans differ only by rare one-ulp flips of 11-bit
  operands (ex2/rcp SiLU approximations vs expf/divide, both followed by the TF32 rounding)."""
  from score_sde_pytorch_b200 import configs
  cfg = configs.tiny_progressive(nf=16, image_size=64, num_res_blocks=2, ch_mult=(1, 2, 2, 4), attn_resolutions=(8,))
  torch.manual_seed(3)
  model = seeded_model(cfg, precision='tf32').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  torch.manual_seed(5)
  x = torch.randn(3, 3, 64, 64, device=dev) * 3
  sigma = torch.tensor([20.0, 1.5, 0.05], device=dev)
  with torch.no_grad():
    y = model(x, sigma)
    ref = NO.ncsnpp_forward(sd, cfg, x, sigma)
  e = rel_l2(y, ref)
  print(f'few-channel GroupNorm on load: vs oracle {e:.3e}; {model.launches_per_forward()} launches')
  assert any('gn+silu' in n for n in model.op_names())
  assert e < 7.5e-4


@pytest.mark.parametrize('name,precision', [('celebahq_256', 'tf32'), ('celebahq_256', 'f16'), ('ffhq_1024', 'tf32')])
def test_high_resolution_reference_configs_full_size(dev, name, precision):
  """configs/ve/celebahq_256_ncsnpp_continuous.py (65.6 M parameters, 256x256, seven levels) and
  configs/ve/ffhq_ncsnpp_continuous.py (105.8 M parameters, 1024x1024, eight levels, nf=16: the 16/32/64-channel levels run on
  the few-channel TF32 MMA kernel, the rest on the wgmma kernels), one evaluation at batch 1 against the strict-fp32 oracle."""
  cfg = golden_config(name)
  model = seeded_model(cfg, precision=precision).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  R = cfg.data.image_size
  torch.manual_seed(4)
  x = torch.randn(1, 3, R, R, device=dev) * 5
  sigma = torch.tensor([3.0], device=dev)
  with torch.no_grad():
    y = model(x, sigma)
    ref = NO.ncsnpp_forward(sd, cfg, x, sigma)
  e = rel_l2(y, ref)
  print(f'{name} [{precision}] 1x3x{R}x{R}: rel-L2 vs oracle {e:.3e}, {model.launches_per_forward()} launches')
  assert torch.isfinite(y).all()
  assert e < 2.5e-3


@pytest.mark.parametrize('precision', ['tf32', 'f16'])
def test_deep_cifar10_variant_matches_oracle(dev, precision):
  """configs/ve/cifar10_ncsnpp_deep_continuous.py: eight residual blocks per level ("deep")."""
  cfg = golden_config('cifar10_deep')
  model = seeded_model(cfg, precision=precision).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  torch.manual_seed(6)
  x = torch.randn(2, 3, 32, 32, device=dev) * 4
  sigma = torch.tensor([12.0, 0.4], device=dev)
  with torch.no_grad():
    e = rel_l2(model(x, sigma), NO.ncsnpp_forward(sd, cfg, x, sigma))
  print(f'cifar10 deep [{precision}]: rel-L2 vs oracle {e:.3e}, {model.launches_per_forward()} launches, '
        f'{sum(p.numel() for p in model.parameters())} parameters')
  assert e < 2.5e-3


def test_baseline_config3_ddpmpp_celebahq256_subvp_ode_sampler(dev):
  """Benchmark configuration 3 at batch 1: DDPM++ cont. (fir=False, positional embedding) at 256x256 under the sub-VP SDE,
  probability-flow ODE sampler with the state on the device.  One evaluation against the strict-fp32 oracle, then the
  device RK45 solve against this package's scipy host loop on the same network (looser tolerances than the default
  1e-5 keep the oracle-free comparison to a few dozen evaluations)."""
  from score_sde_pytorch_b200 import sampling, sde_lib
  cfg = golden_config('celebahq_256_ddpmpp_subvp')
  model = seeded_model(cfg, precision='f16').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  shape = (1, 3, 256, 256)
  torch.manual_seed(8)
  x = torch.randn(*shape, device=dev)
  lab = torch.tensor([500.3], device=dev)
  with torch.no_grad():
    e = rel_l2(model(x, lab), NO.ncsnpp_forward(sd, cfg, x, lab))
  sde = sde_lib.subVPSDE(0.1, 20., 1000)
  z = sde.prior_sampling(shape).to(dev)
  kw = dict(denoise=False, rtol=1e-2, atol=1e-2, eps=1e-3, device=dev)
  s_dev, nfe_dev = sampling.get_ode_sampler(sde, shape, lambda v: v, **kw)(model, z=z.clone())
  s_host, nfe_host = sampling.get_ode_sampler(sde, shape, lambda v: v, device_solver=False, **kw)(model, z=z.clone())
  print(f'configs[3] (DDPM++ 256 sub-VP, f16): forward rel-L2 {e:.3e}; ODE nfe device {nfe_dev} / scipy {nfe_host}, rel-L2 {rel_l2(s_dev, s_host):.2e}')
  assert e < 2.5e-3
  assert nfe_dev == nfe_host and rel_l2(s_dev, s_host) < 1e-5


def test_baseline_config4_ffhq1024_pc_sampler_steps(dev):
  """Benchmark configuration 4 at batch 1: NCSN++ FFHQ 1024x1024 VE-SDE PC sampler (reverse diffusion + Langevin) through
  the native loop in tf32 mode, two iterations (four 1024x1024 evaluations) against the oracle loop on the same noise."""
  from score_sde_pytorch_b200 import native, sampling, sde_lib
  cfg = golden_config('ffhq_1024')
  model = seeded_model(cfg, precision='tf32').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  shape = (1, 3, 1024, 1024)
  sde, osde = sde_lib.VESDE(0.01, 1348, 2000), SO.VE(0.01, 1348, 2000)
  torch.manual_seed(9)
  x0 = osde.prior_sampling(shape).to(dev)
  plan = native.match_pc_plan(sde=sde, model=model, predictor=sampling.ReverseDiffusionPredictor, corrector=sampling.LangevinCorrector,
                              shape=shape, snr=0.15, n_steps=1, probability_flow=False, continuous=True, eps=1e-5, device=dev)
  assert plan is not None
  torch.cuda.manual_seed(77)
  _, xm = plan.run(x0, first_step=0, num_steps=2)
  torch.cuda.manual_seed(77)
  with torch.no_grad():
    ref, _ = SO.pc_sample(osde, lambda a, l: NO.ncsnpp_forward(sd, cfg, a, l), shape, snr=0.15, eps=1e-5, device=dev, x_init=x0, num_iters=2)
  e = rel_l2(xm, ref)
  print(f'configs[4] (FFHQ-1024 PC, tf32): 2 iterations rel-L2 {e:.3e}')
  assert e < 1e-3
