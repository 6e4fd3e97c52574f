"""TEST INFRASTRUCTURE ONLY -- CPU restatement of classifier-free guidance with a negative prompt and per-image weights,
which the reference does not have: the guidance pass is the restated U-Net conditioned on the negative prompt
(cond_drop_prob 0, so no RNG) instead of the null conditioning, combined by restatement.cfg_combine with the weights
broadcast per image, then the DDPM step (restatement.p_sample_step) or the DDIM step (ddim_restatement.ddim_step)."""
import torch

import ddim_restatement as D
from oracle import restatement as R


def negprompt_loop(sd, cfg, shape, timesteps, noise_fn, w, *, text_embeds, text_mask, negative_text_embeds,
                   negative_text_mask, steps=None, eta=0., **unet_kw):
    """The DDPM loop over every timestep (steps=None) or the DDIM loop over ddim_grid(timesteps, steps), draws taken
    through `noise_fn(kind, shape, step)` like Imagen's; w: [b] guidance weights.  Returns the finalised images in [0, 1]."""
    tabs = R.ddpm_tables(timesteps)
    acp = D.alphas_cumprod_fp64(timesteps)
    grid = list(range(timesteps - 1, -1, -1)) if steps is None else D.ddim_grid(timesteps, steps)
    x = noise_fn("init", shape, -1).float().cpu()
    b = shape[0]
    wb = w.float().reshape(b, 1, 1, 1)
    with torch.no_grad():
        for i, tau in enumerate(grid):
            t = torch.full((b,), tau, dtype=torch.long)
            cond = R.unet_forward(sd, cfg, x, t, text_embeds=text_embeds, text_mask=text_mask, **unet_kw)
            neg = R.unet_forward(sd, cfg, x, t, text_embeds=negative_text_embeds, text_mask=negative_text_mask,
                                 cond_drop_prob=0., **unet_kw)
            eps = R.cfg_combine(cond, neg, wb)
            z = noise_fn("step", shape, tau).float().cpu()
            if steps is None:
                x = R.p_sample_step(tabs, x, t, eps, z)
            else:
                t_prev = torch.full((b,), grid[i + 1] if i + 1 < len(grid) else -1, dtype=torch.long)
                x = D.ddim_step(tabs, acp, x, t, t_prev, eps, z, eta)
    return (x.clamp(-1, 1) + 1) * 0.5
