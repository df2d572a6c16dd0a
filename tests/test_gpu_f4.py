"""`-m gpu`: gradients of the two native ops (op/upfirdn2d.py:19-141, op/fused_act.py:20-72) through the
package's autograd Functions on the sm_90a kernels, and the evaluation losses (losses.py:55-210, train=False) through
the engine, all against goldens written by the REAL reference (tools/make_golden_f4.py) and against the oracle."""
import pytest
import torch

from helpers import golden, golden_config, seeded_model
from oracle import losses_oracle as LO
from oracle import ncsnpp_oracle as NO
from oracle import sampling_oracle as SO
from tools_f4_cases import FIR_CASES, StandIn

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


@pytest.mark.parametrize('case', FIR_CASES, ids=lambda c: c[0])
def test_upfirdn2d_first_and_second_derivative_match_the_reference(dev, case):
  """y, d<y, go>/dx and d<grad_input, v>/d go: three launches of b200_upfirdn2d_f32 (forward; adjoint = flipped FIR with
  up and down exchanged and the padding of op/upfirdn2d.py:106-111; adjoint of the adjoint = forward)."""
  from score_sde_pytorch_b200.op import upfirdn2d
  name = case[0]
  g = golden('f4_op_grads.npz')
  up, down, p0, p1 = (int(v) for v in g[f'fir_{name}_cfg'])
  t = lambda k: torch.from_numpy(g[f'fir_{name}_{k}']).to(dev)
  x = t('x').requires_grad_(True)
  go = t('go').requires_grad_(True)
  y = upfirdn2d(x, torch.from_numpy(g[f'fir_{name}_k']), up=up, down=down, pad=(p0, p1))
  gi, = torch.autograd.grad(y, x, go, create_graph=True)
  ggo, = torch.autograd.grad((gi * t('v')).sum(), go)
  for got, key in ((y, 'y'), (gi, 'gi'), (ggo, 'ggo')):
    assert got.shape == t(key).shape, (name, key)
    err = (got.detach() - t(key)).abs().max().item()
    assert err <= 2e-6 * max(1.0, t(key).abs().max().item()), (name, key, err)
  # .backward() accumulates into .grad like any differentiable op
  x2 = t('x').requires_grad_(True)
  upfirdn2d(x2, torch.from_numpy(g[f'fir_{name}_k']), up=up, down=down, pad=(p0, p1)).backward(t('go'))
  assert torch.allclose(x2.grad, t('gi'), rtol=2e-6, atol=2e-6)


def test_upfirdn2d_gradient_of_the_network_resampling_layers(dev):
  """The three parameterisations NCSN++ uses (upsample_2d / downsample_2d / conv_downsample_2d's FIR,
  up_or_down_sampling.py:216-257) on a larger tensor, against autograd of the oracle's pure-torch form."""
  from score_sde_pytorch_b200.op import upfirdn2d
  k = torch.as_tensor(NO.setup_kernel([1, 3, 3, 1]), dtype=torch.float32)
  torch.manual_seed(4)
  for kk, up, down, pad in ((k * 4, 2, 1, (2, 1)), (k, 1, 2, (1, 1)), (k, 1, 1, (2, 1))):
    x = torch.randn(3, 5, 32, 32)
    go_shape = NO.upfirdn2d_native(x, kk, up=up, down=down, pad=pad).shape
    go, v = torch.randn(go_shape), torch.randn(x.shape)
    y_ref, gi_ref, ggo_ref = LO.upfirdn2d_grads(x, kk, up, down, pad, go, v)
    xd, god = x.to(dev).requires_grad_(True), go.to(dev).requires_grad_(True)
    y = upfirdn2d(xd, kk, up=up, down=down, pad=pad)
    gi, = torch.autograd.grad(y, xd, god, create_graph=True)
    ggo, = torch.autograd.grad((gi * v.to(dev)).sum(), god)
    for got, ref in ((y, y_ref), (gi, gi_ref), (ggo, ggo_ref)):
      assert torch.allclose(got.detach().cpu(), ref, rtol=2e-6, atol=2e-6)


def test_fused_leaky_relu_first_and_second_derivative_match_the_reference(dev):
  from score_sde_pytorch_b200.op import fused_leaky_relu, FusedLeakyReLU
  g = golden('f4_op_grads.npz')
  t = lambda k: torch.from_numpy(g[f'lrelu_{k}']).to(dev)
  x, b, go = t('x').requires_grad_(True), t('b').requires_grad_(True), t('go').requires_grad_(True)
  y = fused_leaky_relu(x, b)
  gi, gb = torch.autograd.grad(y, (x, b), go, create_graph=True)
  ggo, = torch.autograd.grad((gi * t('vi')).sum() + (gb * t('vb')).sum(), go)
  for got, key in ((y, 'y'), (gi, 'gi'), (gb, 'gb'), (ggo, 'ggo')):
    assert torch.allclose(got.detach(), t(key), rtol=2e-6, atol=2e-6), key
  mod = FusedLeakyReLU(6).to(dev)
  with torch.no_grad():
    mod.bias.copy_(t('b'))
  mod(t('x')).backward(t('go'))
  assert torch.allclose(mod.bias.grad, t('gb'), rtol=2e-6, atol=2e-5)


def _sdes(name):
  from score_sde_pytorch_b200 import sde_lib
  return {'ve': (sde_lib.VESDE(0.01, 50, 1000), SO.VE(0.01, 50, 1000)), 'vp': (sde_lib.VPSDE(0.1, 20, 1000), SO.VP(0.1, 20, 1000)),
          'subvp': (sde_lib.subVPSDE(0.1, 20, 1000), SO.SubVP(0.1, 20, 1000))}[name]


@pytest.mark.parametrize('mname,sname', [('tiny', 've'), ('tiny_vp', 'vp'), ('tiny_vp', 'subvp'), ('tiny_ddpmpp', 'vp')])
def test_sde_evaluation_losses_match_the_reference(dev, mname, sname):
  """get_sde_loss_fn(train=False) with the reference's own draws (t, z): perturbation kernel -> engine forward (strict fp32
  mode) -> reduction kernel.  (a) the perturbed batch is bit-equal to the reference's unfused torch arithmetic, (b) the
  loss equals the reference's CPU value to fp32 network noise, (c) the TF32 tensor-core mode stays within its operand
  rounding (fp16 operand mode needs the fused attention shape, which these 16x16 test networks do not have)."""
  from score_sde_pytorch_b200 import losses
  g = golden('f4_losses.npz')
  cfg = golden_config(mname)
  sde, osde = _sdes(sname)
  batch = torch.from_numpy(g[f'{mname}_batch']).to(dev)
  t, z = torch.from_numpy(g[f'{mname}_{sname}_t']).to(dev), torch.from_numpy(g[f'{mname}_{sname}_z']).to(dev)
  mean, std = sde.marginal_prob(batch, t)
  want = mean + std[:, None, None, None] * z                                  # losses.py:86-87 on the GPU
  one = torch.ones(batch.shape[0], 1, 1, 1, device=dev)
  got = losses._perturb(batch, z, sde.marginal_prob(one, t)[0].reshape(-1), std)
  assert torch.equal(got, want)
  for precision, tol in (('fp32', 2e-5), ('tf32', 3e-3)):
    model = seeded_model(cfg, precision=precision).to(dev)
    for rm in (False, True):
      for lw in (False, True):
        fn = losses.get_sde_loss_fn(sde, train=False, reduce_mean=rm, continuous=True, likelihood_weighting=lw)
        loss = fn(model, batch, t=t, z=z).item()
        ref = float(g[f'{mname}_{sname}_loss_rm{int(rm)}_lw{int(lw)}'])
        assert abs(loss - ref) <= tol * abs(ref), (precision, rm, lw, loss, ref)
    if precision == 'fp32':
      # and against the oracle on the same device, same weights
      sd = {k: v.to(dev) for k, v in model.state_dict().items()}
      net = lambda a, l: NO.ncsnpp_forward(sd, cfg, a, l)
      with torch.no_grad():
        ol, _ = LO.sde_loss(osde, lambda a, tt: osde.score(net, a, tt), batch, t, z, reduce_mean=False, likelihood_weighting=True)
      fn = losses.get_sde_loss_fn(sde, train=False, reduce_mean=False, continuous=True, likelihood_weighting=True)
      assert abs(fn(model, batch, t=t, z=z).item() - ol.item()) <= 2e-5 * abs(ol.item())
    del model


def test_ddpm_evaluation_loss_and_internal_draws(dev):
  from score_sde_pytorch_b200 import losses
  g = golden('f4_losses.npz')
  cfg = golden_config('tiny_ddpmpp')
  sde, _ = _sdes('vp')
  model = seeded_model(cfg, precision='fp32').to(dev)
  batch = torch.from_numpy(g['tiny_ddpmpp_batch']).to(dev)
  labels, z = torch.from_numpy(g['tiny_ddpmpp_ddpm_labels']).to(dev), torch.from_numpy(g['tiny_ddpmpp_ddpm_z']).to(dev)
  for rm in (False, True):
    loss = losses.get_ddpm_loss_fn(sde, train=False, reduce_mean=rm)(model, batch, labels=labels, z=z).item()
    ref = float(g[f'tiny_ddpmpp_ddpm_loss_rm{int(rm)}'])
    assert abs(loss - ref) <= 2e-5 * abs(ref), (rm, loss, ref)
  # internal draws consume torch's CUDA generator in the reference's order: t (or labels) first, then z
  fn = losses.get_sde_loss_fn(sde, train=False, reduce_mean=True, likelihood_weighting=False)
  torch.manual_seed(31)
  a = fn(model, batch).item()
  torch.manual_seed(31)
  t = torch.rand(batch.shape[0], device=dev) * (sde.T - 1e-5) + 1e-5
  zz = torch.randn_like(batch)
  assert fn(model, batch, t=t, z=zz).item() == a
  dfn = losses.get_ddpm_loss_fn(sde, train=False)
  torch.manual_seed(32)
  b = dfn(model, batch).item()
  torch.manual_seed(32)
  lab = torch.randint(0, sde.N, (batch.shape[0],), device=dev)
  zz = torch.randn_like(batch)
  assert dfn(model, batch, labels=lab, z=zz).item() == b


def test_smld_evaluation_loss_matches_the_reference(dev):
  """get_smld_loss_fn(train=False) (losses.py:105-126) through the device kernels (perturbation with mean coefficient 1,
  residual mode 2: score + (z sigma) / sigma^2) on the goldens' stand-in model, with the reference's own draws."""
  from score_sde_pytorch_b200 import losses
  g = golden('f4_losses.npz')
  sde, _ = _sdes('ve')
  model = StandIn().to(dev)
  batch = torch.from_numpy(g['smld_batch']).to(dev)
  labels, z = torch.from_numpy(g['smld_labels']).to(dev), torch.from_numpy(g['smld_z']).to(dev)
  sig = torch.flip(sde.discrete_sigmas, dims=(0,)).to(dev)[labels]
  assert torch.equal(losses._perturb(batch, z, None, sig), z * sig[:, None, None, None] + batch)   # noise + batch (:111-112)
  for rm in (False, True):
    loss = losses.get_smld_loss_fn(sde, train=False, reduce_mean=rm)(model, batch, labels=labels, z=z).item()
    ref = float(g[f'smld_loss_rm{int(rm)}'])
    assert abs(loss - ref) <= 2e-5 * abs(ref), (rm, loss, ref)
  # the discrete step function picks this loss for a VE SDE (losses.py:176-183) and evaluates the EMA weights
  from score_sde_pytorch_b200.models.ema import ExponentialMovingAverage
  state = dict(model=model, ema=ExponentialMovingAverage(model.parameters(), decay=0.999), step=0, optimizer=None)
  step_fn = losses.get_step_fn(sde, train=False, reduce_mean=False, continuous=False)
  torch.manual_seed(8)
  a = step_fn(state, batch).item()
  torch.manual_seed(8)
  assert losses.get_smld_loss_fn(sde, train=False, reduce_mean=False)(model, batch).item() == a


def test_evaluation_step_swaps_the_ema_weights_in_and_out(dev):
  """get_step_fn(train=False) (losses.py:200-206): the loss is that of the EMA weights - the engine repacks them - and the
  model's own parameters are back afterwards."""
  from score_sde_pytorch_b200 import losses
  from score_sde_pytorch_b200.models.ema import ExponentialMovingAverage
  cfg = golden_config('tiny')
  sde, _ = _sdes('ve')
  model = seeded_model(cfg, precision='fp32').to(dev)
  other = seeded_model(cfg, precision='fp32').to(dev)                         # stands in for the averaged weights: every
  torch.manual_seed(5)                                                        # TRAINABLE parameter moved (the frozen Fourier
  with torch.no_grad():                                                       # projection is not part of the EMA, models/ema.py:24)
    for p in other.parameters():
      if p.requires_grad:
        p.add_(0.02 * torch.randn_like(p))
  ema = ExponentialMovingAverage(other.parameters(), decay=0.999)
  state = dict(model=model, ema=ema, step=0, optimizer=None)
  torch.manual_seed(1)
  batch = torch.rand(4, 3, 16, 16, device=dev)
  before = [p.detach().clone() for p in model.parameters()]
  step_fn = losses.get_step_fn(sde, train=False, reduce_mean=True, continuous=True, likelihood_weighting=False)
  loss_fn = losses.get_sde_loss_fn(sde, train=False, reduce_mean=True, continuous=True, likelihood_weighting=False)
  torch.manual_seed(9)
  l_step = step_fn(state, batch).item()
  torch.manual_seed(9)
  l_other = loss_fn(other, batch).item()
  torch.manual_seed(9)
  l_own = loss_fn(model, batch).item()
  assert l_step == l_other and l_step != l_own
  for p, q in zip(model.parameters(), before):
    assert torch.equal(p.detach(), q)
  torch.manual_seed(9)
  assert loss_fn(model, batch).item() == l_own                                # the engine holds the model's own weights again
