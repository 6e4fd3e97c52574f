"""TEST INFRASTRUCTURE ONLY -- CPU restatement of RePaint inpainting (Lugmayr et al. 2022, jump length 1), which the
reference does not have.  It is written in RePaint's form: the re-noising is q(x_t | x_t') with a_t / a_t' evaluated in
fp64, the known region is q(x_t | k) in fp64, and the step between them is the golden-pinned restatement.p_sample_step
(DDPM) or ddim_restatement.ddim_step (DDIM) over restatement.unet_forward.  The product's form (fp32 ra / rb tables,
fused select) is not used.  Pinned in tests/test_inpaint.py: with R = 1 and nothing known it is the plain loop."""
import torch

import ddim_restatement as D
from oracle import restatement as R


def walk(timesteps, steps=None):
    """The grid points T-1 > ... > 0 of a stage: every timestep (DDPM) or the DDIM grid of `steps` points."""
    return list(range(timesteps - 1, -1, -1)) if steps is None else D.ddim_grid(timesteps, steps)


def plan(timesteps, resample_times, steps=None):
    """The iterations (t, r) in order: R per grid point t > 0, one at t = 0."""
    return [(t, r) for t in walk(timesteps, steps) for r in range(resample_times if t > 0 else 1)]


def inpaint_loop(sd, cfg, shape, timesteps, known, mask, resample_times, noise_fn, steps=None, eta=0., cond_scale=3.,
                 **unet_kw):
    """RePaint sampling over restatement.unet_forward with classifier-free guidance, draws taken through
    `noise_fn(kind, shape, step)` in Imagen's order and labels (t * R + r).  known: the NORMALISED known image
    (b, c, s, s); mask: bool (b, s, s), True = known.  steps: None for the DDPM loop, else the DDIM grid with `eta`.
    unet_kw as in ddim_restatement.ddim_loop.  Returns the finalised images in [0, 1]."""
    tabs = R.ddpm_tables(timesteps)
    acp = D.alphas_cumprod_fp64(timesteps)
    grid = walk(timesteps, steps)
    b = shape[0]
    m = mask.bool()[:, None].expand(shape)
    k = known.double()
    x = noise_fn("init", shape, -1).float().cpu()
    with torch.no_grad():
        for i, tau in enumerate(grid):
            t_next = grid[i + 1] if i + 1 < len(grid) else -1
            t = torch.full((b,), tau, dtype=torch.long)
            for r in range(resample_times if tau > 0 else 1):
                label = tau * resample_times + r
                if r > 0:
                    # q(x_t | x_t'): back from the next grid point to t
                    a = acp[tau] / acp[t_next]
                    z = noise_fn("renoise", shape, label).double().cpu()
                    x = (a.sqrt() * x.double() + (1. - a).sqrt() * z).float()
                # q(x_t | k) on the known region
                z = noise_fn("inpaint", shape, label).double().cpu()
                x = torch.where(m, (acp[tau].sqrt() * k + (1. - acp[tau]).sqrt() * z).float(), x)
                cond = R.unet_forward(sd, cfg, x, t, **unet_kw)
                null = R.unet_forward(sd, cfg, x, t, cond_drop_prob=1., **unet_kw)
                eps = R.cfg_combine(cond, null, cond_scale)
                z = noise_fn("step", shape, label).float().cpu()
                if steps is None:
                    x = R.p_sample_step(tabs, x, t, eps, z)
                else:
                    x = D.ddim_step(tabs, acp, x, t, torch.full((b,), t_next, dtype=torch.long), eps, z, eta)
    x = torch.where(m, known.float(), x)
    return (x.clamp(-1, 1) + 1) * 0.5
