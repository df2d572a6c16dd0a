"""Attribute-style config trees for the sampling engine.

The reference describes experiments with ``ml_collections.ConfigDict`` objects
(``configs/default_cifar10_configs.py:5-71``).  ``ml_collections`` is not a
dependency here: any object with attribute access works (the engine only reads
fields), and :class:`ConfigDict` below is the small stand-in we ship.
"""
import torch


class ConfigDict(dict):
  """dict with attribute access (duck-type of ``ml_collections.ConfigDict``)."""

  def __getattr__(self, key):
    try:
      return self[key]
    except KeyError as e:
      raise AttributeError(key) from e

  def __setattr__(self, key, value):
    self[key] = value

  def copy(self):
    out = ConfigDict()
    for k, v in self.items():
      out[k] = v.copy() if isinstance(v, ConfigDict) else v
    return out


def _default_device():
  return torch.device('cuda:0') if torch.cuda.is_available() else torch.device('cpu')


def cifar10_defaults():
  """Field-for-field equivalent of ``configs/default_cifar10_configs.py:5-71``
  restricted to what the sampling path reads (training/optim bookkeeping that
  the sampler never touches is kept only where the model constructor reads it)."""
  c = ConfigDict()
  c.training = ConfigDict(batch_size=128, continuous=True, reduce_mean=False,
                          likelihood_weighting=False, sde='vesde')
  c.sampling = ConfigDict(method='pc', predictor='reverse_diffusion', corrector='langevin',
                          n_steps_each=1, noise_removal=True, probability_flow=False, snr=0.16)
  c.eval = ConfigDict(batch_size=1024, num_samples=50000)
  c.data = ConfigDict(dataset='CIFAR10', image_size=32, centered=False, num_channels=3,
                      random_flip=True, uniform_dequantization=False)
  c.model = ConfigDict(sigma_min=0.01, sigma_max=50, num_scales=1000, beta_min=0.1,
                       beta_max=20., dropout=0.1, embedding_type='fourier')
  # configs/default_cifar10_configs.py:59-67 - read by losses.get_optimizer / optimization_manager
  c.optim = ConfigDict(weight_decay=0, optimizer='Adam', lr=2e-4, beta1=0.9, eps=1e-8, warmup=5000, grad_clip=1.)
  c.seed = 42
  c.device = _default_device()
  return c


def ve_cifar10_ncsnpp_continuous():
  """``configs/ve/cifar10_ncsnpp_continuous.py:19-59`` — the headline workload."""
  c = cifar10_defaults()
  c.training.sde = 'vesde'
  c.training.continuous = True
  c.sampling.method = 'pc'
  c.sampling.predictor = 'reverse_diffusion'
  c.sampling.corrector = 'langevin'
  m = c.model
  m.name = 'ncsnpp'
  m.scale_by_sigma = True
  m.ema_rate = 0.999
  m.normalization = 'GroupNorm'
  m.nonlinearity = 'swish'
  m.nf = 128
  m.ch_mult = (1, 2, 2, 2)
  m.num_res_blocks = 4
  m.attn_resolutions = (16,)
  m.resamp_with_conv = True
  m.conditional = True
  m.fir = True
  m.fir_kernel = [1, 3, 3, 1]
  m.skip_rescale = True
  m.resblock_type = 'biggan'
  m.progressive = 'none'
  m.progressive_input = 'residual'
  m.progressive_combine = 'sum'
  m.attention_type = 'ddpm'
  m.init_scale = 0.
  m.fourier_scale = 16
  m.conv_size = 3
  return c


def ve_cifar10_ncsnpp_deep_continuous():
  """``configs/ve/cifar10_ncsnpp_deep_continuous.py`` — 8 blocks per level."""
  c = ve_cifar10_ncsnpp_continuous()
  c.model.num_res_blocks = 8
  return c


def tiny_ncsnpp(nf=32, image_size=16, num_res_blocks=1, ch_mult=(1, 2), attn_resolutions=(8,)):
  """A small NCSN++ of the same family (test fixture sized; not a reference config)."""
  c = ve_cifar10_ncsnpp_continuous()
  c.model.nf = nf
  c.model.ch_mult = tuple(ch_mult)
  c.model.num_res_blocks = num_res_blocks
  c.model.attn_resolutions = tuple(attn_resolutions)
  c.model.init_scale = 1.0
  c.data.image_size = image_size
  return c


def vp_cifar10_ddpmpp_continuous():
  """``configs/vp/cifar10_ddpmpp_continuous.py:21-63`` — DDPM++ cont. (VP): naive 2x resampling (``fir=False``),
  sinusoidal positional time embedding, no input pyramid, centred data, Euler-Maruyama predictor only."""
  c = ve_cifar10_ncsnpp_continuous()
  c.training.sde = 'vpsde'
  c.training.reduce_mean = True
  c.sampling.predictor = 'euler_maruyama'
  c.sampling.corrector = 'none'
  c.data.centered = True
  m = c.model
  m.scale_by_sigma = False
  m.ema_rate = 0.9999
  m.fir = False
  m.progressive_input = 'none'
  m.embedding_type = 'positional'
  return c


def subvp_cifar10_ddpmpp_continuous():
  """``configs/subvp/cifar10_ddpmpp_continuous.py`` — the same network under the sub-VP SDE."""
  c = vp_cifar10_ddpmpp_continuous()
  c.training.sde = 'subvpsde'
  return c


def tiny_ddpmpp(nf=32, image_size=16, num_res_blocks=1, ch_mult=(1, 2), attn_resolutions=(8,)):
  """A small DDPM++ of the same family (test fixture sized; not a reference config)."""
  c = vp_cifar10_ddpmpp_continuous()
  c.model.nf = nf
  c.model.ch_mult = tuple(ch_mult)
  c.model.num_res_blocks = num_res_blocks
  c.model.attn_resolutions = tuple(attn_resolutions)
  c.model.init_scale = 1.0
  c.data.image_size = image_size
  return c


def ve_ffhq_1024_ncsnpp_continuous():
  """``configs/ve/ffhq_ncsnpp_continuous.py`` over ``configs/default_lsun_configs.py``: the 1024x1024 NCSN++ -
  nf=16, eight levels, ``progressive='output_skip'``, ``progressive_input='input_skip'``, attention at 16x16."""
  c = ve_cifar10_ncsnpp_continuous()
  c.data.dataset = 'FFHQ'
  c.data.image_size = 1024
  c.training.batch_size = 8
  c.eval.batch_size = 8
  m = c.model
  m.sigma_max = 1348
  m.num_scales = 2000
  m.ema_rate = 0.9999
  m.nf = 16
  m.ch_mult = (1, 2, 4, 8, 16, 32, 32, 32)
  m.num_res_blocks = 1
  m.attn_resolutions = (16,)
  m.dropout = 0.
  m.progressive = 'output_skip'
  m.progressive_input = 'input_skip'
  m.progressive_combine = 'sum'
  return c


def ve_celebahq_256_ncsnpp_continuous():
  """``configs/ve/celebahq_256_ncsnpp_continuous.py``: 256x256, nf=128, ch_mult (1,1,2,2,2,2,2), two blocks per level,
  output_skip / input_skip pyramids."""
  c = ve_cifar10_ncsnpp_continuous()
  c.data.dataset = 'CelebAHQ'
  c.data.image_size = 256
  c.eval.batch_size = 64
  m = c.model
  m.sigma_max = 348
  m.ema_rate = 0.999
  m.nf = 128
  m.ch_mult = (1, 1, 2, 2, 2, 2, 2)
  m.num_res_blocks = 2
  m.attn_resolutions = (16,)
  m.progressive = 'output_skip'
  m.progressive_input = 'input_skip'
  m.progressive_combine = 'sum'
  return c


def tiny_progressive(nf=32, image_size=32, num_res_blocks=1, ch_mult=(1, 1, 2), attn_resolutions=(8,), fir=True):
  """A small member of the high-resolution family (three levels, output_skip + input_skip); test fixture sized."""
  c = tiny_ncsnpp(nf=nf, image_size=image_size, num_res_blocks=num_res_blocks, ch_mult=ch_mult, attn_resolutions=attn_resolutions)
  c.model.progressive = 'output_skip'
  c.model.progressive_input = 'input_skip'
  c.model.progressive_combine = 'sum'
  c.model.fir = fir
  return c


def vp_cifar10_ddpm_continuous():
  """``configs/vp/ddpm/cifar10_continuous.py`` — DDPM cont. (VP): the ``models/ddpm.py`` network, centred data,
  Euler-Maruyama predictor, no corrector."""
  c = cifar10_defaults()
  c.training.sde = 'vpsde'
  c.training.continuous = True
  c.training.reduce_mean = True
  c.sampling.method = 'pc'
  c.sampling.predictor = 'euler_maruyama'
  c.sampling.corrector = 'none'
  c.data.centered = True
  m = c.model
  m.name = 'ddpm'
  m.scale_by_sigma = False
  m.ema_rate = 0.9999
  m.normalization = 'GroupNorm'
  m.nonlinearity = 'swish'
  m.nf = 128
  m.ch_mult = (1, 2, 2, 2)
  m.num_res_blocks = 2
  m.attn_resolutions = (16,)
  m.resamp_with_conv = True
  m.conditional = True
  return c


def subvp_cifar10_ddpm_continuous():
  """``configs/subvp/cifar10_ddpm_continuous.py`` — the same network under the sub-VP SDE."""
  c = vp_cifar10_ddpm_continuous()
  c.training.sde = 'subvpsde'
  return c


def vp_cifar10_ddpm():
  """``configs/vp/ddpm/cifar10.py`` — discrete-time DDPM (``continuous=False``), ancestral sampling.  Samples through the
  generic host loop over the engine network."""
  c = vp_cifar10_ddpm_continuous()
  c.training.continuous = False
  c.sampling.predictor = 'ancestral_sampling'
  return c


def vp_celebahq_256_ddpm():
  """``configs/vp/ddpm/celebahq.py`` over ``configs/default_lsun_configs.py``: 256x256, ch_mult (1,1,2,2,4,4), two blocks
  per level, attention at 16x16, discrete time, ancestral sampling."""
  c = vp_cifar10_ddpm()
  c.data.dataset = 'CelebAHQ'
  c.data.image_size = 256
  c.training.batch_size = 64
  c.eval.batch_size = 512
  m = c.model
  m.sigma_max = 378          # configs/default_lsun_configs.py:51-56
  m.dropout = 0.
  m.num_scales = 1000        # configs/vp/ddpm/celebahq.py
  m.ch_mult = (1, 1, 2, 2, 4, 4)
  m.num_res_blocks = 2
  m.attn_resolutions = (16,)
  return c


def tiny_ddpm(nf=32, image_size=16, num_res_blocks=1, ch_mult=(1, 2), attn_resolutions=(8,)):
  """A small DDPM of the same family (test fixture sized; not a reference config)."""
  c = vp_cifar10_ddpm_continuous()
  c.model.nf = nf
  c.model.ch_mult = tuple(ch_mult)
  c.model.num_res_blocks = num_res_blocks
  c.model.attn_resolutions = tuple(attn_resolutions)
  c.data.image_size = image_size
  return c


def subvp_celebahq_256_ddpmpp_continuous():
  """DDPM++ cont. CelebA-HQ 256 sub-VP.  The reference ships no such config file; it is composed from ``configs/subvp/cifar10_ddpmpp_continuous.py`` (DDPM++: ``fir=False``, positional
  embedding, no pyramids, sub-VP SDE, Euler-Maruyama predictor) with the 256-pixel data / ``ch_mult`` fields of
  ``configs/ve/celebahq_256_ncsnpp_continuous.py``."""
  c = subvp_cifar10_ddpmpp_continuous()
  c.data.dataset = 'CelebAHQ'
  c.data.image_size = 256
  c.eval.batch_size = 64
  c.model.ch_mult = (1, 1, 2, 2, 2, 2, 2)
  c.model.num_res_blocks = 2
  c.model.attn_resolutions = (16,)
  return c


def ve_cifar10_ncsnv2():
  """``configs/ve/ncsnv2/cifar10.py`` — NCSNv2 (``model.name = 'ncsnv2_64'``): InstanceNorm++, ELU, nf=128, 232 noise
  levels, discrete time (``continuous=False``) with annealed Langevin dynamics (predictor ``none``, corrector ``ald``,
  5 steps per level, snr 0.176).  ``data.channels`` mirrors ``data.num_channels``: the reference's NCSNv2 constructor
  reads that name (models/ncsnv2.py:55)."""
  c = cifar10_defaults()
  c.training.sde = 'vesde'
  c.training.continuous = False
  c.sampling.method = 'pc'
  c.sampling.predictor = 'none'
  c.sampling.corrector = 'ald'
  c.sampling.n_steps_each = 5
  c.sampling.snr = 0.176
  c.data.channels = c.data.num_channels
  m = c.model
  m.name = 'ncsnv2_64'
  m.scale_by_sigma = True
  m.num_scales = 232
  m.ema_rate = 0.999
  m.normalization = 'InstanceNorm++'
  m.nonlinearity = 'elu'
  m.nf = 128
  m.interpolation = 'bilinear'
  c.optim = ConfigDict(weight_decay=0, optimizer='Adam', lr=1e-4, beta1=0.9, amsgrad=False, eps=1e-8, warmup=0, grad_clip=-1.)
  return c


def ve_celeba_ncsnv2():
  """``configs/ve/ncsnv2/celeba.py`` over ``configs/default_celeba_configs.py``: the same network at 64x64, sigma_max 90,
  500 noise levels, snr 0.128."""
  c = ve_cifar10_ncsnv2()
  c.data.dataset = 'CELEBA'
  c.data.image_size = 64
  c.model.sigma_max = 90.
  c.model.num_scales = 500
  c.sampling.snr = 0.128
  return c


def ve_bedroom_ncsnv2():
  """``configs/ve/ncsnv2/bedroom.py`` over ``configs/default_lsun_configs.py``: NCSNv2_128 (``model.name = 'ncsnv2_128'``)
  at 128x128, sigma_max 190, 1086 noise levels, 3 Langevin steps per level, snr 0.095, EMA 0.9999."""
  c = ve_cifar10_ncsnv2()
  c.data.dataset = 'LSUN'
  c.data.category = 'bedroom'
  c.data.image_size = 128
  c.training.batch_size = 128
  c.eval.batch_size = 512
  c.sampling.n_steps_each = 3
  c.sampling.snr = 0.095
  m = c.model
  m.name = 'ncsnv2_128'
  m.sigma_max = 190
  m.sigma_min = 0.01
  m.num_scales = 1086
  m.ema_rate = 0.9999
  return c


def tiny_ncsnv2(nf=32, image_size=16, num_scales=20):
  """A small NCSNv2 (``ncsnv2_64`` walk; test fixture sized, not a reference config)."""
  c = ve_cifar10_ncsnv2()
  c.model.nf = nf
  c.model.num_scales = num_scales
  c.data.image_size = image_size
  return c
