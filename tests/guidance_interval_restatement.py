"""TEST INFRASTRUCTURE ONLY -- CPU restatement of guidance intervals (Kynkaanniemi et al. 2024, "Applying Guidance in a
Limited Interval Improves Sample and Distribution Quality in Diffusion Models") and guidance-weight schedules (after Wang
et al. 2024, "Analysis of Classifier-Free Guidance Weight Schedulers"), which the reference does not have.  Written from
the formulas of Imagen.sample's docstring in plain Python floats, not from GaussianDiffusion.guidance_table:
    sigma_t = sqrt((1 - a_t) / a_t)   (inf where a_t = 0),   tau = t / (T - 1),
    shape(t) = 1, 2 (1 - tau) or 1 + cos(pi tau),   s[t] = shape(t) if lo < sigma_t <= hi else 0   (fp64, then fp32),
    w_b(t) = w_b if s[t] == 1 else fp32(1 + fp32(fp32(w_b - 1) s[t])),
and a grid point with s[t] == 0 takes the conditional prediction alone.  The sampling loop runs the restated U-Net
(oracle/restatement.py) with the negative prompt (or the null conditioning) as the guidance pass, then the DDPM, DDIM or
DPM-Solver++(2M) step of the restatements next to this file."""
import math

import numpy as np
import torch

import ddim_restatement as D
import dpmpp_restatement as P
from oracle import restatement as R


def sigmas(timesteps):
    """The VE noise level of every timestep, fp64 Python floats."""
    return [math.sqrt((1. - a) / a) if a > 0 else math.inf for a in D.alphas_cumprod_fp64(timesteps).tolist()]


def table(timesteps, interval=None, schedule=None):
    """s[t] for t = 0 .. T-1 as a list of fp32 values (Python floats holding fp32 numbers)."""
    out = []
    for t, sig in enumerate(sigmas(timesteps)):
        tau = t / (timesteps - 1)
        shape = {None: 1., 'linear': 2. * (1. - tau), 'cosine': 1. + math.cos(math.pi * tau)}[schedule]
        inside = interval is None or interval[0] < sig <= interval[1]
        out.append(float(np.float32(shape if inside else 0.)))
    return out


def guided_points(grid, tab):
    """The points of `grid` that run the guidance pass."""
    return [t for t in grid if tab[t] != 0.]


def weights(w, s):
    """w_b(t) for the per-image weights w (a sequence of floats) at a table value s, fp32 op by op."""
    f = np.float32
    return [float(wb) if s == 1. else float(f(1.) + f(f(f(wb) - f(1.)) * f(s))) for wb in w]


def interval_loop(sd, cfg, shape, timesteps, noise_fn, w, *, interval=None, schedule=None, sampler='ddpm', steps=None,
                  eta=0., text_embeds=None, text_mask=None, negative_text_embeds=None, negative_text_mask=None):
    """The DDPM loop over every timestep, the DDIM loop over ddim_grid(timesteps, steps) or the 2M loop over
    dpm_grid(timesteps, steps), with per-image weights w ([b] floats) scheduled by the table of (interval, schedule); the
    guidance pass conditions on the negative prompt when given, else on the null conditioning.  Draws through
    `noise_fn(kind, shape, step)` like Imagen's.  Returns (finalised images in [0, 1], the guided grid points)."""
    tabs = R.ddpm_tables(timesteps)
    acp = D.alphas_cumprod_fp64(timesteps)
    tab = table(timesteps, interval, schedule)
    if sampler == 'ddpm':
        grid = list(range(timesteps - 1, -1, -1))
    elif sampler == 'ddim':
        grid = D.ddim_grid(timesteps, steps)
    else:
        grid = P.dpm_grid(timesteps, steps)
        lam = P.lambdas(timesteps)
    b = shape[0]
    x = noise_fn("init", shape, -1).float().cpu()
    x0_prev = h_prev = None
    kw = dict(text_embeds=text_embeds, text_mask=text_mask)
    neg = dict(text_embeds=negative_text_embeds, text_mask=negative_text_mask, cond_drop_prob=0.) \
        if negative_text_embeds is not None else dict(kw, cond_drop_prob=1.)
    with torch.no_grad():
        for i, tau in enumerate(grid):
            t = torch.full((b,), tau, dtype=torch.long)
            eps = R.unet_forward(sd, cfg, x, t, **kw)
            if tab[tau] != 0.:
                g = R.unet_forward(sd, cfg, x, t, **neg)
                wb = torch.tensor(weights(w, tab[tau]), dtype=torch.float32).reshape(b, 1, 1, 1)
                eps = R.cfg_combine(eps, g, wb)
            t_next = grid[i + 1] if i + 1 < len(grid) else -1
            if sampler == 'dpmpp_2m':
                x0 = P.thresholded_x0(tabs, x, t, eps)
                x, h_prev = P.dpmpp_step(acp, lam, x, tau, t_next, x0, x0_prev, h_prev)
                x0_prev = x0
                continue
            z = noise_fn("step", shape, tau).float().cpu()
            if sampler == 'ddpm':
                x = R.p_sample_step(tabs, x, t, eps, z)
            else:
                x = D.ddim_step(tabs, acp, x, t, torch.full((b,), t_next, dtype=torch.long), eps, z, eta)
    return (x.clamp(-1, 1) + 1) * 0.5, guided_points(grid, tab)
