"""ORACLE (test infrastructure, not product code): float64 plain-PyTorch restatement of the multistep DPM-Solver
(Lu et al., arXiv:2206.00927) and DPM-Solver++ (arXiv:2211.01095) samplers of the probability-flow ODE, written from the
papers' equations and independently of ``score_sde_pytorch_b200.native.build_multistep_tables``:

* the marginal ``x_t = alpha_t x_0 + sigma_t eps`` from the SDE's own formulas (``sde_lib.py``), and ``t(lambda)`` by
  bisection of the monotone log-SNR ``lambda_t = log alpha_t - log sigma_t`` instead of its closed form;
* each step in divided-difference form: ``D1_0 = (M_0 - M_1) / r0``, ``D1_1 = (M_1 - M_2) / r1``,
  ``D1 = D1_0 + r0 / (r0 + r1) (D1_0 - D1_1)``, ``D2 = (D1_0 - D1_1) / (r0 + r1)`` (so ``D1 ~ h M'`` and
  ``D2 ~ h^2 M'' / 2``), against the exponential-integrator weights of the Taylor terms.

``score(x, t)`` is any callable returning the score at float64 ``x`` and the batch of times ``t``.
"""
import math

import torch


class Marginal:
  """alpha_t, sigma_t of a stock SDE given by kind ('ve', 'vp', 'subvp') and its parameters."""

  def __init__(self, kind, sigma_min=0.01, sigma_max=50., beta_min=0.1, beta_max=20.):
    self.kind, self.sigma_min, self.sigma_max, self.beta_0, self.beta_1 = kind, sigma_min, sigma_max, beta_min, beta_max

  def log_alpha(self, t):
    t = torch.as_tensor(t, dtype=torch.float64)
    if self.kind == 've':
      return torch.zeros_like(t)
    return -0.25 * t ** 2 * (self.beta_1 - self.beta_0) - 0.5 * t * self.beta_0

  def alpha(self, t):
    return torch.exp(self.log_alpha(t))

  def sigma(self, t):
    t = torch.as_tensor(t, dtype=torch.float64)
    if self.kind == 've':
      return self.sigma_min * (self.sigma_max / self.sigma_min) ** t
    one_minus_a2 = -torch.expm1(2. * self.log_alpha(t))   # 1 - alpha^2 without cancellation near t = 0
    return torch.sqrt(one_minus_a2) if self.kind == 'vp' else one_minus_a2

  def lam(self, t):
    return self.log_alpha(t) - torch.log(self.sigma(t))

  def t_of_lambda(self, lam, lo=0., hi=1., iters=200):
    """lambda_t decreases in t: bisection on [lo, hi] to the float64 resolution."""
    lam = torch.as_tensor(lam, dtype=torch.float64)
    a, b = torch.full_like(lam, lo), torch.full_like(lam, hi)
    for _ in range(iters):
      m = 0.5 * (a + b)
      above = self.lam(m) > lam
      a, b = torch.where(above, m, a), torch.where(above, b, m)
    return 0.5 * (a + b)


def time_grid(mg, steps, skip_type, T=1., eps=1e-3):
  if skip_type == 'logSNR':
    lam = torch.linspace(float(mg.lam(T)), float(mg.lam(eps)), steps + 1, dtype=torch.float64)
    t = mg.t_of_lambda(lam)
  elif skip_type == 'time_uniform':
    t = torch.linspace(T, eps, steps + 1, dtype=torch.float64)
  else:
    t = torch.linspace(math.sqrt(T), math.sqrt(eps), steps + 1, dtype=torch.float64) ** 2
  t[0], t[-1] = T, eps
  return t


def step_orders(steps, order):
  return [min(order, i + 1, steps - i) if steps < 10 else min(order, i + 1) for i in range(steps)]


def prediction(mg, algorithm, x, score, t):
  """The model's data prediction x0 = (x + sigma^2 score) / alpha ('dpmsolver++') or noise prediction
  eps = -sigma score ('dpmsolver')."""
  a, s = float(mg.alpha(t)), float(mg.sigma(t))
  return (x + s * s * score) / a if algorithm == 'dpmsolver++' else -s * score


def update(mg, algorithm, order, t_hist, t_next, x, m_hist):
  """One multistep step from t_hist[0] to t_next.  t_hist = (t_i, t_{i-1}, t_{i-2})[:order], m_hist the predictions at
  those times, most recent first."""
  s, t = t_hist[0], t_next
  lam_s, lam_t = float(mg.lam(s)), float(mg.lam(t))
  h = lam_t - lam_s
  a_s, a_t, sg_s, sg_t = float(mg.alpha(s)), float(mg.alpha(t)), float(mg.sigma(s)), float(mg.sigma(t))
  if algorithm == 'dpmsolver++':
    # x_t = sigma_t/sigma_s x_s + sigma_t int_{lam_s}^{lam_t} e^lam x0(lam) dlam, x0 expanded in (lam - lam_s)
    e1 = math.expm1(-h)
    w0, w1, w2 = -a_t * e1, a_t * (e1 / h + 1.), -a_t * ((e1 / h + 1.) / h - 0.5)
    base = (sg_t / sg_s) * x
  else:
    # x_t = alpha_t/alpha_s x_s - alpha_t int_{lam_s}^{lam_t} e^-lam eps(lam) dlam
    e1 = math.expm1(h)
    w0, w1, w2 = -sg_t * e1, -sg_t * (e1 / h - 1.), -sg_t * ((e1 / h - 1.) / h - 0.5)
    base = (a_t / a_s) * x
  m0 = m_hist[0]
  if order == 1:
    return base + w0 * m0
  r0 = (lam_s - float(mg.lam(t_hist[1]))) / h
  d1_0 = (m0 - m_hist[1]) / r0
  if order == 2:
    return base + w0 * m0 + 0.5 * w0 * d1_0
  r1 = (float(mg.lam(t_hist[1])) - float(mg.lam(t_hist[2]))) / h
  d1_1 = (m_hist[1] - m_hist[2]) / r1
  d1 = d1_0 + (r0 / (r0 + r1)) * (d1_0 - d1_1)
  d2 = (d1_0 - d1_1) / (r0 + r1)
  return base + w0 * m0 + w1 * d1 + w2 * 2. * d2   # w2 weighs h^2 M'' = 2 D2


def sample(mg, score, x, steps, order, algorithm='dpmsolver++', skip_type='logSNR', T=1., eps=1e-3):
  """The multistep loop: returns x at t = eps (no final denoising step)."""
  t = time_grid(mg, steps, skip_type, T, eps)
  orders = step_orders(steps, order)
  ts, ms = [], []
  for i in range(steps):
    vec_t = torch.full((x.shape[0],), float(t[i]), dtype=x.dtype, device=x.device)
    ts.insert(0, float(t[i]))
    ms.insert(0, prediction(mg, algorithm, x, score(x, vec_t), float(t[i])))
    ts, ms = ts[:3], ms[:3]
    x = update(mg, algorithm, orders[i], ts, float(t[i + 1]), x, ms)
  return x


def coefficients(mg, steps, order, algorithm='dpmsolver++', skip_type='logSNR', T=1., eps=1e-3):
  """The affine tables of each step read off the update by probing it with unit inputs:
  x_{i+1} = pa x_i + pb M_i + pm1 M_{i-1} + pm2 M_{i-2}, and M_i = mq x_i + ms score_i.  float64 tensors."""
  t = time_grid(mg, steps, skip_type, T, eps)
  orders = step_orders(steps, order)
  one, zero = torch.ones(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)
  out = {k: torch.zeros(steps, dtype=torch.float64) for k in ('pa', 'pb', 'pm1', 'pm2', 'mq', 'ms')}
  for i in range(steps):
    k = orders[i]
    ts = [float(t[i - j]) for j in range(k)]
    for name, (xv, hist) in {'pa': (one, [zero] * k), 'pb': (zero, [one] + [zero] * (k - 1)),
                             'pm1': (zero, [zero, one, zero][:k]), 'pm2': (zero, [zero, zero, one][:k])}.items():
      if name == 'pm1' and k < 2 or name == 'pm2' and k < 3:
        continue
      out[name][i] = update(mg, algorithm, k, ts, float(t[i + 1]), xv, hist)
    out['mq'][i] = prediction(mg, algorithm, one, zero, ts[0])
    out['ms'][i] = prediction(mg, algorithm, zero, one, ts[0])
  out['t'] = t
  return out
