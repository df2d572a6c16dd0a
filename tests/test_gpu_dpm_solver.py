"""`-m gpu`: the multistep DPM-Solver / DPM-Solver++ sampler on the native loop (`b200_pc_config.predictor = 2`,
`pc_multistep_kernel`), held to
  * the host loop over the same engine network in 'fp32' (same tables, same network evaluations): per-image rel-L2 1e-5;
  * the float64 oracle loop over the strict-fp32 oracle network for the CIFAR-10 NCSN++ VE / DDPM++ VP networks in
    'tf32' and 'f16': per-image rel-L2 1e-3 of the final state;
  * itself: bit-identical graph replays, no generator use, the launch count, and repacked weights after
    invalidate_weights()."""
import pytest
import torch

from helpers import golden_config, rel_l2, seeded_model
from oracle import dpm_solver_oracle as DO, ncsnpp_oracle as NO

pytestmark = pytest.mark.gpu
KINDS = ('ve', 'vp', 'subvp')


def make_sde(kind):
  from score_sde_pytorch_b200 import sde_lib
  return {'ve': lambda: sde_lib.VESDE(0.01, 50., 1000), 'vp': lambda: sde_lib.VPSDE(0.1, 20., 1000),
          'subvp': lambda: sde_lib.subVPSDE(0.1, 20., 1000)}[kind]()


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


@pytest.fixture(scope='module')
def tiny(dev):
  cache = {}

  def get(kind):
    name = 'tiny' if kind == 've' else 'tiny_ddpmpp'
    if name not in cache:
      cache[name] = (seeded_model(golden_config(name), precision='fp32').to(dev), golden_config(name))
    return cache[name]
  return get


class Plain(torch.nn.Module):
  """The same engine network behind a plain module: the sampler then runs its host loop."""

  def __init__(self, net):
    super().__init__()
    self.net = net

  def forward(self, x, labels):
    return self.net(x, labels)


def prior(sde, shape, dev, seed=5):
  torch.manual_seed(seed)
  return sde.prior_sampling(shape).to(dev)


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('order', [1, 2, 3])
@pytest.mark.parametrize('algorithm', ['dpmsolver++', 'dpmsolver'])
def test_native_loop_matches_host_loop(dev, tiny, kind, order, algorithm):
  from score_sde_pytorch_b200 import native, sampling
  model, cfg = tiny(kind)
  sde = make_sde(kind)
  shape = (3, cfg.data.num_channels, cfg.data.image_size, cfg.data.image_size)
  z = prior(sde, shape, dev)
  fn = sampling.get_dpm_solver_sampler(sde, shape, lambda v: v, steps=10, order=order, algorithm=algorithm, device=dev)
  gen = torch.cuda.default_generators[dev.index or 0]
  off = gen.get_offset()
  x, nfe = fn(model, z=z.clone())
  assert fn.last_stats == dict(loop='native', steps=10, order=order, nfe=10) and nfe == 10
  assert gen.get_offset() == off
  x2, _ = fn(model, z=z.clone())                       # the cached plan's graph replayed
  assert torch.equal(x, x2)
  plan = native.match_multistep_plan(sde, model, shape, 10, order, algorithm, 'logSNR', 1e-3, dev)
  assert plan.launches_per_step() == model.launches_per_forward() + 3
  xh, _ = fn(Plain(model), z=z.clone())
  assert fn.last_stats['loop'] == 'host'
  err = rel_l2(x, xh)
  print(f'{kind} {algorithm} order {order}: native vs host loop (fp32 engine) rel-L2 {err:.2e}')
  assert torch.isfinite(x).all() and err <= 1e-5


def cifar_case(kind):
  from score_sde_pytorch_b200 import configs
  cfg = configs.ve_cifar10_ncsnpp_continuous() if kind == 've' else configs.vp_cifar10_ddpmpp_continuous()
  cfg.model.init_scale = 1.0
  return cfg


@pytest.mark.parametrize('kind', ['ve', 'vp'])
@pytest.mark.parametrize('precision', ['tf32', 'f16'])
@pytest.mark.parametrize('algorithm', ['dpmsolver++', 'dpmsolver'])
def test_tensor_core_native_loop_matches_oracle(dev, kind, precision, algorithm):
  from score_sde_pytorch_b200 import sampling
  cfg = cifar_case(kind)
  model = seeded_model(cfg, precision=precision).to(dev)
  sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
  sde = make_sde(kind)
  shape = (2, 3, 32, 32)
  z = prior(sde, shape, dev)
  fn = sampling.get_dpm_solver_sampler(sde, shape, lambda v: v, steps=10, order=3, algorithm=algorithm, device=dev)
  x, _ = fn(model, z=z.clone())
  assert fn.last_stats['loop'] == 'native'
  mg = DO.Marginal(kind)

  def score(xs, t):
    xf = xs.float()
    if kind == 've':
      return NO.ncsnpp_forward(sd, cfg, xf, mg.sigma(t).to(dev).float()).double()
    return -NO.ncsnpp_forward(sd, cfg, xf, (t * 999).to(dev).float()).double() / mg.sigma(t).to(dev)[:, None, None, None]

  with torch.no_grad():
    ref = DO.sample(mg, score, z.double(), 10, 3, algorithm)
  err = rel_l2(x, ref)
  print(f'CIFAR-10 {kind} {precision} {algorithm} order 3, 10 steps: native vs oracle loop rel-L2 {err:.2e}')
  assert err <= 1e-3


def test_cached_plan_sees_new_weights(dev, tiny):
  from score_sde_pytorch_b200 import sampling
  cfg = golden_config('tiny')
  model = seeded_model(cfg, precision='fp32').to(dev)
  sde = make_sde('ve')
  shape = (2, 3, cfg.data.image_size, cfg.data.image_size)
  z = prior(sde, shape, dev)
  fn = sampling.get_dpm_solver_sampler(sde, shape, lambda v: v, steps=6, order=2, device=dev)
  before, _ = fn(model, z=z.clone())
  with torch.no_grad():
    for p in model.parameters():
      p.mul_(1.05)
  model.invalidate_weights()
  after, _ = fn(model, z=z.clone())
  fresh = seeded_model(cfg, precision='fp32').to(dev)
  fresh.load_state_dict(model.state_dict())
  want, _ = fn(fresh, z=z.clone())
  assert not torch.equal(before, after)
  assert torch.equal(after, want)


def test_ncsnv2_is_refused(dev):
  from score_sde_pytorch_b200 import configs, sampling
  from score_sde_pytorch_b200.models.ncsnv2 import NCSNv2
  cfg = configs.tiny_ncsnv2()
  net = NCSNv2(cfg).to(dev)
  shape = (1, cfg.data.num_channels, cfg.data.image_size, cfg.data.image_size)
  fn = sampling.get_dpm_solver_sampler(make_sde('ve'), shape, lambda v: v, device=dev)
  with pytest.raises(NotImplementedError, match='noise-level indices'):
    fn(net)
