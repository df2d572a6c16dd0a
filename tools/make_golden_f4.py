"""Golden fixtures for the losses and op gradients from the REAL reference, run on CPU (same recipe as tools/make_golden.py):

  f4_op_grads.npz   first and second derivatives of the reference's two native ops through its own CPU forms under autograd
                    (op/upfirdn2d.py:159-200 `upfirdn2d_native`; op/fused_act.py:85-93) - what its CUDA autograd Functions
                    (op/upfirdn2d.py:19-141, op/fused_act.py:20-72) compute with the kernels
  f4_losses.npz     losses.get_sde_loss_fn / get_ddpm_loss_fn (train=False) of the reference's NCSNpp holding this repository's
                    deterministic weights, with the draws (t / labels, z) the loss made; get_smld_loss_fn on a deterministic
                    stand-in model (the reference's positional-embedding VE network does not run on current PyTorch)

    python tools/make_golden_f4.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG   # noqa: E402
from score_sde_pytorch_b200 import configs as our_configs   # noqa: E402

FIR_CASES = [   # name, input HxW, FIR, up, down, pad
    ('up2', (8, 8), 'fir4x2', 2, 1, (2, 1)),       # upsample_2d (up_or_down_sampling.py:216-219)
    ('down2', (8, 8), 'fir4', 1, 2, (1, 1)),       # downsample_2d (:248-252)
    ('same', (6, 10), 'fir4', 1, 1, (2, 1)),
    ('generic', (5, 7), 'k3x5', 2, 3, (1, 2)),     # odd sizes, rectangular FIR, both factors
    ('crop', (9, 6), 'k3x5', 1, 1, (-1, 0)),       # negative padding crops
]


def fir(name):
  k1 = torch.tensor([1., 3., 3., 1.])
  k = torch.outer(k1, k1); k = k / k.sum()
  if name == 'fir4':
    return k
  if name == 'fir4x2':
    return k * 4
  g = torch.Generator().manual_seed(3)
  return torch.randn(3, 5, generator=g)


def op_grads(ref_upfirdn2d_mod):
  import torch.nn.functional as F
  out = {}
  g = torch.Generator().manual_seed(11)
  for name, (h, w), kn, up, down, pad in FIR_CASES:
    k = fir(kn)
    x = torch.randn(2, 3, h, w, generator=g, requires_grad=True)
    y = ref_upfirdn2d_mod.upfirdn2d(x, k, up=up, down=down, pad=pad)          # CPU input -> upfirdn2d_native
    go = torch.randn(y.shape, generator=g, requires_grad=True)
    gi, = torch.autograd.grad(y, x, go, create_graph=True)
    v = torch.randn(x.shape, generator=g)
    ggo, = torch.autograd.grad((gi * v).sum(), go)
    for key, val in (('x', x), ('k', k), ('y', y), ('go', go), ('gi', gi), ('v', v), ('ggo', ggo)):
      out[f'fir_{name}_{key}'] = val.detach().numpy()
    out[f'fir_{name}_cfg'] = np.array([up, down, pad[0], pad[1]])
  ref_fused = sys.modules['op.fused_act']
  x = torch.randn(4, 6, 5, 5, generator=g, requires_grad=True)
  b = torch.randn(6, generator=g, requires_grad=True)
  y = ref_fused.fused_leaky_relu(x, b)                                         # CPU form
  go = torch.randn(y.shape, generator=g, requires_grad=True)
  gi, gb = torch.autograd.grad(y, (x, b), go, create_graph=True)
  vi, vb = torch.randn(x.shape, generator=g), torch.randn(6, generator=g)
  ggo, = torch.autograd.grad((gi * vi).sum() + (gb * vb).sum(), go)
  for key, val in (('x', x), ('b', b), ('y', y), ('go', go), ('gi', gi), ('gb', gb), ('vi', vi), ('vb', vb), ('ggo', ggo)):
    out[f'lrelu_{key}'] = val.detach().numpy()
  return out


def loss_goldens(sde_lib, mutils):
  import losses as ref_losses
  out = {}
  tiny_vp = our_configs.tiny_ncsnpp(); tiny_vp.model.scale_by_sigma = False; tiny_vp.data.centered = True
  models = {'tiny': our_configs.tiny_ncsnpp(), 'tiny_vp': tiny_vp, 'tiny_ddpmpp': our_configs.tiny_ddpmpp()}
  B = 4
  for mname, cfg in models.items():
    cfg.device = torch.device('cpu')
    sd = MG.our_weights(cfg)
    torch.manual_seed(0)
    model = mutils.get_model('ncsnpp')(cfg).eval()
    model.load_state_dict(sd, strict=True)
    R, C = cfg.data.image_size, cfg.data.num_channels
    g = torch.Generator().manual_seed(21)
    batch = torch.rand(B, C, R, R, generator=g) * 2 - 1
    out[f'{mname}_batch'] = batch.numpy()
    if mname == 'tiny':
      sdes = {'ve': sde_lib.VESDE(sigma_min=0.01, sigma_max=50, N=1000)}
    elif mname == 'tiny_vp':
      sdes = {'vp': sde_lib.VPSDE(beta_min=0.1, beta_max=20, N=1000), 'subvp': sde_lib.subVPSDE(beta_min=0.1, beta_max=20, N=1000)}
    else:
      sdes = {'vp': sde_lib.VPSDE(beta_min=0.1, beta_max=20, N=1000)}
    for sname, sde in sdes.items():
      seed = 100 + len(out)
      torch.manual_seed(seed)
      t = torch.rand(B) * (sde.T - 1e-5) + 1e-5
      z = torch.randn_like(batch)
      out[f'{mname}_{sname}_t'], out[f'{mname}_{sname}_z'] = t.numpy(), z.numpy()
      for rm in (False, True):
        for lw in (False, True):
          fn = ref_losses.get_sde_loss_fn(sde, train=False, reduce_mean=rm, continuous=True, likelihood_weighting=lw)
          torch.manual_seed(seed)
          with torch.no_grad():
            out[f'{mname}_{sname}_loss_rm{int(rm)}_lw{int(lw)}'] = np.float64(fn(model, batch).item())
      # the evaluation step: EMA weights (here: a perturbed copy) swapped in around the loss (losses.py:200-206)
    if mname == 'tiny_ddpmpp':
      sde = sdes['vp']
      seed = 777
      torch.manual_seed(seed)
      labels = torch.randint(0, sde.N, (B,))
      z = torch.randn_like(batch)
      out['tiny_ddpmpp_ddpm_labels'], out['tiny_ddpmpp_ddpm_z'] = labels.numpy(), z.numpy()
      for rm in (False, True):
        fn = ref_losses.get_ddpm_loss_fn(sde, train=False, reduce_mean=rm)
        torch.manual_seed(seed)
        with torch.no_grad():
          out[f'tiny_ddpmpp_ddpm_loss_rm{int(rm)}'] = np.float64(fn(model, batch).item())
  return out


class StandIn(torch.nn.Module):
  """A deterministic stand-in score model for the SMLD loss: the reference's own positional-embedding VE network raises a
  dtype error on current PyTorch , and the loss arithmetic does not care what the model is."""

  def forward(self, x, labels):
    return 0.3 * torch.flip(x, dims=(3,)) + (0.001 * labels.float())[:, None, None, None] * x


def smld_goldens(sde_lib):
  import losses as ref_losses
  out = {}
  sde = sde_lib.VESDE(sigma_min=0.01, sigma_max=50, N=1000)
  g = torch.Generator().manual_seed(33)
  batch = torch.rand(5, 3, 8, 8, generator=g)
  out['smld_batch'] = batch.numpy()
  seed = 555
  torch.manual_seed(seed)
  labels = torch.randint(0, sde.N, (batch.shape[0],))
  z = torch.randn_like(batch)
  out['smld_labels'], out['smld_z'] = labels.numpy(), z.numpy()
  for rm in (False, True):
    fn = ref_losses.get_smld_loss_fn(sde, train=False, reduce_mean=rm)
    torch.manual_seed(seed)
    with torch.no_grad():
      out[f'smld_loss_rm{int(rm)}'] = np.float64(fn(StandIn(), batch).item())
  return out


def main():
  torch.set_num_threads(8)
  sde_lib, sampling, ncsnpp, mutils, _ = MG.import_reference()
  import op   # noqa: F401  (op/__init__.py binds the name `upfirdn2d` to the function, so fetch the module itself)
  og = op_grads(sys.modules['op.upfirdn2d'])
  np.savez_compressed(os.path.join(MG.OUT, 'f4_op_grads.npz'), **og)
  print('op grads', len(og), 'arrays')
  lg = loss_goldens(sde_lib, mutils)
  lg.update(smld_goldens(sde_lib))
  np.savez_compressed(os.path.join(MG.OUT, 'f4_losses.npz'), **lg)
  print({k: float(v) for k, v in lg.items() if 'loss' in k})


if __name__ == '__main__':
  main()
