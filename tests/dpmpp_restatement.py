"""TEST INFRASTRUCTURE ONLY -- CPU restatement of DPM-Solver++(2M) sampling (Lu et al. 2022, "DPM-Solver++: Fast Solver for
Guided Sampling of Diffusion Probabilistic Models", Algorithm 2), which the reference does not have.  It reuses the pinned
pieces of oracle/restatement.py (x0 prediction, dynamic threshold), like ddim_restatement.py, and writes the update in the
paper's form -- log-SNR lambda, step h, ratio r, the combined data prediction D -- not in the product's affine-table form,
with its own grid code, so that the tests check the algebra as well as the wiring."""
import math

import torch

import ddim_restatement as D
from oracle import restatement as R


def lambdas(timesteps):
    """log-SNR lambda_t = log(alpha_t / sigma_t) = 0.5 (log a_t - log(1 - a_t)), fp64, as a list (-inf where a_t = 0)."""
    return [0.5 * (math.log(a) - math.log1p(-a)) if a > 0 else -math.inf
            for a in D.alphas_cumprod_fp64(timesteps).tolist()]


def dpm_grid(timesteps, steps):
    """Descending walk T-1 .. 0 over points uniform in log-SNR: built ascending from u_0 = 0, each inner point the t with
    lambda_t closest to its target (first such t on a tie), pushed up to keep the points distinct and capped so that the
    remaining points still fit below T; the last point is T-1."""
    lam = lambdas(timesteps)
    lo, hi = lam[0], lam[timesteps - 1]
    if hi == -math.inf:                         # T = 20: the last beta is 1; the targets end one timestep earlier
        hi = lam[timesteps - 2]
    up = [0]
    for j in range(1, steps - 1):
        target = lo + (hi - lo) * j / (steps - 1)
        best = min(range(timesteps), key=lambda t: abs(lam[t] - target))
        up.append(min(max(best, up[-1] + 1), timesteps - steps + j))
    return (up + [timesteps - 1])[::-1]


def thresholded_x0(tabs, x, t, eps, percentile=0.9):
    """restatement.p_sample_step's x0 prediction and dynamic threshold (fp32), returned in fp64."""
    x0 = R._ext(tabs['sqrt_recip_alphas_cumprod'], t, x) * x - R._ext(tabs['sqrt_recipm1_alphas_cumprod'], t, x) * eps
    s = torch.quantile(x0.flatten(1).abs(), percentile, dim=-1)
    s.clamp_(min=1.)
    s = s.reshape(-1, *((1,) * (x.dim() - 1)))
    return (x0.clamp(-s, s) / s).double()


def dpmpp_step(acp, lam, x, t, t_next, x0, x0_prev, h_prev):
    """One step of Algorithm 2 from t to t_next (python ints; t_next < 0: the last step, which returns x0 itself).
    x0: this step's thresholded data prediction, x0_prev / h_prev: the previous step's (None at the first step).
        h = lambda(t_next) - lambda(t),  r = h_prev / h,  D = (1 + 1/(2r)) x0 - x0_prev / (2r)   (D = x0 at the first step)
        x' = (sigma_next / sigma) x - alpha_next (e^{-h} - 1) D,   alpha = sqrt(a), sigma = sqrt(1 - a).
    Evaluated in fp64; returns (x' in fp32, h)."""
    if t_next < 0:
        return x0.float(), None
    h = lam[t_next] - lam[t]
    if x0_prev is None:
        d = x0
    else:
        r = h_prev / h
        d = (1. + 1. / (2. * r)) * x0 - x0_prev / (2. * r)
    a, a_next = float(acp[t]), float(acp[t_next])
    out = math.sqrt(1. - a_next) / math.sqrt(1. - a) * x.double() - math.sqrt(a_next) * math.expm1(-h) * d
    return out.float(), h


def dpmpp_loop(sd, cfg, shape, timesteps, steps, noise_fn, cond_scale=3., **unet_kw):
    """DPM-Solver++(2M) sampling loop over restatement.unet_forward with classifier-free guidance; x_T through
    `noise_fn('init', shape, -1)` like Imagen's (the solver takes no other draws).  unet_kw as in ddim_restatement.ddim_loop.
    Returns the finalised images in [0, 1]."""
    tabs = R.ddpm_tables(timesteps)
    acp = D.alphas_cumprod_fp64(timesteps)
    lam = lambdas(timesteps)
    grid = dpm_grid(timesteps, steps)
    x = noise_fn("init", shape, -1).float().cpu()
    b = shape[0]
    x0_prev = h_prev = None
    with torch.no_grad():
        for i, tau in enumerate(grid):
            t = torch.full((b,), tau, dtype=torch.long)
            cond = R.unet_forward(sd, cfg, x, t, **unet_kw)
            null = R.unet_forward(sd, cfg, x, t, cond_drop_prob=1., **unet_kw)
            x0 = thresholded_x0(tabs, x, t, R.cfg_combine(cond, null, cond_scale))
            x, h_prev = dpmpp_step(acp, lam, x, tau, grid[i + 1] if i + 1 < len(grid) else -1, x0, x0_prev, h_prev)
            x0_prev = x0
    return (x.clamp(-1, 1) + 1) * 0.5
