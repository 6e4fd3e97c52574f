"""TEST INFRASTRUCTURE ONLY -- CPU restatement of image-to-image sampling (SDEdit, Meng et al. 2022, "SDEdit: Guided
Image Synthesis and Editing with Stochastic Differential Equations"), which the reference does not have.  A stage starts
from the given image diffused to t0 by q(x_t0 | x_0), written here in fp64 from alphas_cumprod (not the product's fp32
tables and mi_q_sample), then runs the reverse steps of its walk from t0 down to 0: the golden-pinned
restatement.p_sample_step (DDPM), ddim_restatement.ddim_step (DDIM) or dpmpp_restatement.dpmpp_step (DPM-Solver++(2M),
whose history starts empty at t0, so its first step is first order) over restatement.unet_forward."""
import torch

import ddim_restatement as D
import dpmpp_restatement as P
from oracle import restatement as R


def walk(timesteps, steps=None, sampler="ddim"):
    """A stage's full walk T-1 .. 0: every timestep (steps None), the DDIM grid or the 2M log-SNR grid."""
    if steps is None:
        return list(range(timesteps - 1, -1, -1))
    return P.dpm_grid(timesteps, steps) if sampler == "dpmpp_2m" else D.ddim_grid(timesteps, steps)


def diffuse(acp, image, t0, z):
    """q(x_t0 | x_0 = image) with the draw z: sqrt(a_t0) image + sqrt(1 - a_t0) z, in fp64, returned in fp32."""
    return (acp[t0].sqrt() * image.double() + (1. - acp[t0]).sqrt() * z.double()).float()


def sdedit_loop(sd, cfg, shape, timesteps, image, skip, noise_fn, steps=None, eta=0., sampler="ddim", cond_scale=3.,
                **unet_kw):
    """SDEdit over restatement.unet_forward with classifier-free guidance: the walk's points from grid[skip] on, started
    from `image` (NORMALISED, (b, c, s, s)) diffused to grid[skip] with noise_fn('init', shape, -1); the steps take
    noise_fn('step', shape, t) like Imagen's (2M takes none).  unet_kw as in ddim_restatement.ddim_loop.  Returns the
    finalised images in [0, 1]."""
    tabs = R.ddpm_tables(timesteps)
    acp = D.alphas_cumprod_fp64(timesteps)
    lam = P.lambdas(timesteps)
    grid = walk(timesteps, steps, sampler)[skip:]
    b = shape[0]
    x = diffuse(acp, image.cpu(), grid[0], noise_fn("init", shape, -1).cpu())
    x0_prev = h_prev = None
    with torch.no_grad():
        for i, tau in enumerate(grid):
            t_next = grid[i + 1] if i + 1 < len(grid) else -1
            t = torch.full((b,), tau, dtype=torch.long)
            eps = R.cfg_combine(R.unet_forward(sd, cfg, x, t, **unet_kw),
                                R.unet_forward(sd, cfg, x, t, cond_drop_prob=1., **unet_kw), cond_scale)
            if sampler == "dpmpp_2m":
                x0 = P.thresholded_x0(tabs, x, t, eps)
                x, h_prev = P.dpmpp_step(acp, lam, x, tau, t_next, x0, x0_prev, h_prev)
                x0_prev = x0
                continue
            z = noise_fn("step", shape, tau).float().cpu()
            if steps is None:
                x = R.p_sample_step(tabs, x, t, eps, z)
            else:
                x = D.ddim_step(tabs, acp, x, t, torch.full((b,), t_next, dtype=torch.long), eps, z, eta)
    return (x.clamp(-1, 1) + 1) * 0.5
