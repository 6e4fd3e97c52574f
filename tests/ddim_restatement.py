"""TEST INFRASTRUCTURE ONLY -- CPU restatement of fewer-step DDIM sampling (Song et al. 2021, eq. 12), which the reference
does not have.  It reuses the pinned pieces of oracle/restatement.py (schedule, x0 prediction, dynamic threshold) and
writes the update in the paper's form, not in the product's affine-table form, so that the tests check the algebra as
well as the wiring.  Pinned in tests/test_respaced.py: at S = T, eta = 1 a step equals the golden-pinned
restatement.p_sample_step."""
import torch

from oracle import restatement as R


def ddim_grid(timesteps, steps):
    """Respaced sampling grid: round(linspace(0, T-1, S)), descending."""
    return torch.linspace(0, timesteps - 1, steps, dtype=torch.float64).round().long().flip(0).tolist()


def alphas_cumprod_fp64(timesteps):
    """alphas_cumprod of restatement.ddpm_tables before its fp32 cast."""
    scale = 1000 / timesteps
    betas = torch.linspace(scale * 0.0001, scale * 0.02, timesteps, dtype=torch.float64)
    return torch.cumprod(1. - betas, 0)


def ddim_step(tabs, acp, x, t, t_prev, eps, noise, eta, percentile=0.9):
    """After the same x0 prediction and dynamic threshold as restatement.p_sample_step, eps is re-derived from the clamped
    x0 and
        x_prev = sqrt(a_prev) x0 + sqrt(1 - a_prev - sigma^2) eps' + sigma z,
        sigma^2 = eta^2 (1 - a_prev) / (1 - a_t) (1 - a_t / a_prev).
    tabs: restatement.ddpm_tables; acp: fp64 alphas_cumprod; t_prev < 0 marks the last step (a_prev = 1).  The update is
    evaluated in fp64 and returned in fp32."""
    x0 = R._ext(tabs['sqrt_recip_alphas_cumprod'], t, x) * x - R._ext(tabs['sqrt_recipm1_alphas_cumprod'], t, x) * eps
    s = torch.quantile(x0.flatten(1).abs(), percentile, dim=-1)
    s.clamp_(min=1.)
    s = s.reshape(-1, *((1,) * (x.dim() - 1)))
    x0 = (x0.clamp(-s, s) / s).double()
    shp = (x.shape[0], *((1,) * (x.dim() - 1)))
    a_t = acp[t].reshape(shp)
    a_prev = torch.where(t_prev >= 0, acp[t_prev.clamp(min=0)], torch.ones_like(acp[t])).reshape(shp)
    sig2 = eta ** 2 * (1. - a_prev) / (1. - a_t) * (1. - a_t / a_prev)
    eps_prime = (x.double() - a_t.sqrt() * x0) / (1. - a_t).sqrt()
    out = a_prev.sqrt() * x0 + (1. - a_prev - sig2).clamp(min=0.).sqrt() * eps_prime + sig2.sqrt() * noise.double()
    return out.float()


def ddim_loop(sd, cfg, shape, timesteps, steps, eta, noise_fn, cond_scale=3., **unet_kw):
    """DDIM sampling loop over restatement.unet_forward + ddim_step with classifier-free guidance, draws taken through
    `noise_fn(kind, shape, step)` like Imagen's.  unet_kw: CPU conditioning (text_embeds, text_mask; for SR U-Nets the
    NORMALISED lowres_cond_img and lowres_noise_times).  Returns the finalised images in [0, 1]."""
    tabs = R.ddpm_tables(timesteps)
    acp = alphas_cumprod_fp64(timesteps)
    grid = ddim_grid(timesteps, steps)
    x = noise_fn("init", shape, -1).float().cpu()
    b = shape[0]
    with torch.no_grad():
        for i, tau in enumerate(grid):
            t = torch.full((b,), tau, dtype=torch.long)
            t_prev = torch.full((b,), grid[i + 1] if i + 1 < len(grid) else -1, dtype=torch.long)
            cond = R.unet_forward(sd, cfg, x, t, **unet_kw)
            null = R.unet_forward(sd, cfg, x, t, cond_drop_prob=1., **unet_kw)
            eps = R.cfg_combine(cond, null, cond_scale)
            x = ddim_step(tabs, acp, x, t, t_prev, eps, noise_fn("step", shape, tau).float().cpu(), eta)
    return (x.clamp(-1, 1) + 1) * 0.5
