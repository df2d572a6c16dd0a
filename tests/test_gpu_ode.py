"""`-m gpu`: probability-flow ODE sampler with the state on the device (sampling.py:414-485).

The device solver (score_sde_pytorch_b200/ode.py + csrc/ode.cu) is held to
  * this package's own host loop over scipy.integrate.solve_ivp on the SAME engine network (`device_solver=False`): same
    right-hand side, so the number of function evaluations must agree to +-2 % and the samples to round-off;
  * the oracle's restatement of the reference sampler (oracle/sampling_oracle.py:ode_sample, pinned on CPU to goldens
    from the real reference) run on the GPU with the strict-fp32 oracle network;
  * the reference's own CPU result (tests/golden/ode_tiny.npz), loosely (different hardware => different round-off
    in an adaptive integrator)."""
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


def _case(case):
  from score_sde_pytorch_b200 import sde_lib
  return {'ve': ('tiny', sde_lib.VESDE(0.01, 50, 1000), SO.VE(0.01, 50, 1000), 1e-5, False),
          'vp': ('tiny_ddpmpp', sde_lib.VPSDE(0.1, 20., 1000), SO.VP(0.1, 20., 1000), 1e-3, False),
          'subvp': ('tiny_ddpmpp', sde_lib.subVPSDE(0.1, 20., 1000), SO.SubVP(0.1, 20., 1000), 1e-3, True)}[case]


@pytest.mark.parametrize('case', ['ve', 'vp', 'subvp'])
def test_device_ode_sampler_matches_scipy_host_loop_oracle_and_reference(dev, case):
  from score_sde_pytorch_b200 import sampling
  g = golden('ode_tiny.npz')
  name, sde, osde, eps, denoise = _case(case)
  cfg = golden_config(name)
  model = seeded_model(cfg, precision='fp32').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  z = torch.from_numpy(g[case + '_z']).to(dev)
  shape = tuple(z.shape)
  ident = lambda v: v
  fn_dev = sampling.get_ode_sampler(sde, shape, ident, denoise=denoise, eps=eps, device=dev)
  fn_host = sampling.get_ode_sampler(sde, shape, ident, denoise=denoise, eps=eps, device=dev, device_solver=False)
  torch.manual_seed(52); torch.cuda.manual_seed(52)
  s_dev, nfe_dev = fn_dev(model, z=z.clone())
  stats = dict(fn_dev.last_stats)
  torch.manual_seed(52); torch.cuda.manual_seed(52)
  s_host, nfe_host = fn_host(model, z=z.clone())
  torch.manual_seed(52); torch.cuda.manual_seed(52)
  s_or, nfe_or = SO.ode_sample(osde, lambda a, l: NO.ncsnpp_forward(sd, cfg, a, l), shape, z=z.clone(), denoise=denoise, eps=eps, device=dev)
  e_host, e_or, e_gold = rel_l2(s_dev, s_host), rel_l2(s_dev, s_or), rel_l2(s_dev, torch.from_numpy(g[case]).to(dev))
  print(f'ode [{case}] nfe: device {nfe_dev}, scipy host loop {nfe_host}, oracle(GPU) {nfe_or}, reference(CPU) {int(g[case + "_nfe"])}; '
        f'rel-L2 vs host loop {e_host:.2e}, vs oracle {e_or:.2e}, vs reference CPU golden {e_gold:.2e}; '
        f'host scalar reads {stats["host_scalar_reads"]}')
  assert stats['solver'] == 'device' and fn_host.last_stats['solver'] == 'scipy'
  assert abs(nfe_dev - nfe_host) <= 0.02 * nfe_host
  assert abs(nfe_dev - nfe_or) <= 0.05 * nfe_or
  assert e_host < 1e-4            # same network, same controller: round-off of the float64 stage sums only
  assert e_or < 1e-3              # north-star bound against the reference restatement (strict fp32) on the same GPU
  assert e_gold < 1e-2
  # one double per attempted step (6 evaluations each after the first), plus the three norms of the initial step
  assert stats['host_scalar_reads'] == (nfe_dev - 2) // 6 + 3


@pytest.mark.parametrize('precision', ['f16', 'tf32'])
def test_device_ode_sampler_cifar10_tensor_core_modes(dev, precision):
  """The headline network (62.8 M parameters) in the tensor-core operand modes, VE SDE, rtol = atol = 1e-5 as in the
  reference's default: samples against the strict-fp32 oracle sampler, NFE against the fp32 oracle's."""
  from score_sde_pytorch_b200 import sampling, sde_lib
  cfg = golden_config('cifar10_ve')
  model = seeded_model(cfg, precision=precision).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  shape = (4, 3, 32, 32)
  sde, osde = sde_lib.VESDE(0.01, 50, 1000), SO.VE(0.01, 50, 1000)
  torch.manual_seed(61)
  z = sde.prior_sampling(shape).to(dev)
  fn_dev = sampling.get_ode_sampler(sde, shape, lambda v: v, eps=1e-5, device=dev)
  s_dev, nfe_dev = fn_dev(model, z=z.clone())
  s_or, nfe_or = SO.ode_sample(osde, lambda a, l: NO.ncsnpp_forward(sd, cfg, a, l), shape, z=z.clone(), eps=1e-5, device=dev)
  e = rel_l2(s_dev, s_or)
  print(f'ode cifar10 [{precision}]: nfe device {nfe_dev} vs fp32 oracle {nfe_or}; rel-L2 {e:.3e}')
  assert e < 1e-3
  assert nfe_dev <= 1.25 * nfe_or
