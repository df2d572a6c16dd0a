"""Golden fixtures for controllable generation (controllable_generation.py:8-198) from the REAL
reference: get_pc_inpainter and get_pc_colorizer with the reverse-diffusion predictor + Langevin corrector under the VE
SDE (N = 12) on the reference's own tiny NCSNpp, CPU, fixed seeds.  controllable_tiny.npz: data, mask, inpainted,
gray, colorized.

    python tools/make_golden_controllable.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG   # noqa: E402


def main():
  torch.set_num_threads(8)
  sde_lib, sampling, ncsnpp, mutils, _ = MG.import_reference()
  import controllable_generation as CG     # the reference's module (sys.path[0] is the reference tree)
  cfg, B = MG.golden_configs()['tiny']
  cfg.device = torch.device('cpu')
  sd = MG.our_weights(cfg)
  torch.manual_seed(0)
  m = mutils.get_model('ncsnpp')(cfg).eval()
  m.load_state_dict(sd, strict=True)
  R = cfg.data.image_size
  g = torch.Generator().manual_seed(70)
  data = torch.rand(B, 3, R, R, generator=g)
  mask = torch.ones(B, 3, R, R)
  mask[:, :, :, R // 2:] = 0.                     # right half unknown
  sde = sde_lib.VESDE(sigma_min=0.01, sigma_max=50, N=12)
  inp = CG.get_pc_inpainter(sde, sampling.ReverseDiffusionPredictor, sampling.LangevinCorrector, lambda v: v, snr=0.16,
                            n_steps=1, probability_flow=False, continuous=True, denoise=True, eps=1e-5)
  torch.manual_seed(71)
  out_i = inp(m, data, mask)
  gray = data.mean(dim=1, keepdim=True).repeat(1, 3, 1, 1)
  col = CG.get_pc_colorizer(sde, sampling.ReverseDiffusionPredictor, sampling.LangevinCorrector, lambda v: v, snr=0.16,
                            n_steps=1, probability_flow=False, continuous=True, denoise=True, eps=1e-5)
  torch.manual_seed(72)
  out_c = col(m, gray)
  np.savez_compressed(os.path.join(MG.OUT, 'controllable_tiny.npz'), data=data.numpy(), mask=mask.numpy(), inpainted=out_i.numpy(),
                      gray=gray.numpy(), colorized=out_c.numpy())
  print('inpainted', float(out_i.abs().mean()), 'colorized', float(out_c.abs().mean()))


if __name__ == '__main__':
  main()
