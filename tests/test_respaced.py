"""Fewer-step DDIM sampling (Imagen.sample(sampling_timesteps=, ddim_eta=)) on the CPU, through the torch emulation of
the ops interface.  The anchor: at S = T, eta = 1 the respaced tables ARE the DDPM tables, so the respaced loop is the
DDPM sampler; below that, the loop is checked against ddim_restatement.ddim_step (written in the paper's form, not the
product's affine one) over the restated U-Net.  (The CPU emulation runs the eager loop; the captured graph and its
mi_step_advance_t_table walk are covered on the GPU in test_gpu_respaced.py.)"""
import pytest
import torch

import ddim_restatement as D
from conftest import load_golden, rel_l2
from oracle import restatement as R


def _tiny_imagen(g, timesteps, device="cpu"):
    """The tiny base U-Net of sample_loop.pt in an Imagen with `timesteps` training steps."""
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet
    u = Unet(**g["cfg"]).eval()
    u.load_state_dict(g["state_dict"])
    im = Imagen(unets=u, text_encoder_name="t5_small", image_sizes=(64,), timesteps=timesteps,
                cond_drop_prob=0.15).eval().to(device)
    im.unets[0].load_state_dict(g["state_dict"])
    return im


def _bank(seed, shape=(2, 3, 64, 64)):
    """noise_fn over a seeded bank: one tensor per (kind, step); records the calls in order."""
    gen = torch.Generator().manual_seed(seed)
    bank, calls = {}, []

    def noise_fn(kind, shp, step):
        assert tuple(shp) == tuple(shape)
        calls.append((kind, step))
        if (kind, step) not in bank:
            bank[(kind, step)] = torch.randn(shape, generator=gen)
        return bank[(kind, step)]
    noise_fn.calls = calls
    noise_fn.bank = bank
    return noise_fn


def restated_tiny_loop(g, timesteps, steps, eta, noise_fn):
    return D.ddim_loop(g["state_dict"], g["cfg"], (2, 3, 64, 64), timesteps, steps, eta, noise_fn,
                       text_embeds=g["text_embeds"].cpu(), text_mask=g["text_mask"].cpu())


# ------------------------------------------------------------------------------------------------ schedule
@pytest.mark.parametrize("T", [20, 25, 1000])
@pytest.mark.parametrize("S", [2, 10, "T"])
def test_grid_descending_unique_endpoints(T, S):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    S = T if S == "T" else S
    sch = GaussianDiffusion(timesteps=T).sampling_schedule(S, 0.5, "cpu")
    grid = list(sch.grid)
    assert len(grid) == S and len(set(grid)) == S
    assert grid[0] == T - 1 and grid[-1] == 0
    assert all(a > b for a, b in zip(grid, grid[1:]))
    assert grid == D.ddim_grid(T, S)
    # next_t walks the grid and stays at 0
    assert [int(sch.next_t[t]) for t in grid] == grid[1:] + [0]
    assert sch.c1.shape == sch.c2.shape == sch.sigma.shape == sch.next_t.shape == (T,)
    assert sch.c1.dtype == torch.float32 and sch.next_t.dtype == torch.int64


@pytest.mark.parametrize("T", [20, 25, 100, 1000, 4000])
def test_tables_at_full_steps_are_the_ddpm_tables(T):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    gd = GaussianDiffusion(timesteps=T)
    sch = gd.sampling_schedule(T, 1., "cpu")
    assert torch.equal(sch.c1, gd.posterior_mean_coef1)
    assert torch.equal(sch.c2, gd.posterior_mean_coef2)
    assert torch.equal(sch.sigma[1:], gd.sigma[1:])
    assert sch.sigma[0] == 0                                  # the step kernel masks t == 0 either way
    assert torch.equal(sch.next_t, (torch.arange(T) - 1).clamp(min=0))
    det = gd.sampling_schedule(max(2, T // 7), 0., "cpu")
    assert torch.count_nonzero(det.sigma) == 0                # eta = 0: no noise at any step
    assert gd.sampling_schedule(T, 1., "cpu") is sch          # cached per (steps, eta, device)


# ------------------------------------------------------------------------------------------------ sampling loop
def test_respaced_loop_at_full_steps_equals_ddpm_loop(emu):
    """S = T = 25, eta = 1 on sample_loop.pt's tiny U-Net (CFG w = 3), eager: the respaced path gives the DDPM loop's output
    bit for bit, and both take one 'step' draw per iteration labelled T-1 .. 0."""
    g = load_golden("sample_loop.pt")
    outs, calls = [], []
    for respaced in (False, True):
        im = _tiny_imagen(g, 25)
        im.use_cuda_graph = False
        im.noise_fn = _bank(5)
        sched = im.noise_schedulers[0].sampling_schedule(25, 1., "cpu") if respaced else None
        outs.append(im._p_sample_loop(im.unets[0], (2, 3, 64, 64), noise_scheduler=im.noise_schedulers[0],
                                      text_embeds=g["text_embeds"], text_mask=g["text_mask"], cond_scale=3.,
                                      schedule=sched))
        calls.append(im.noise_fn.calls)
    assert torch.equal(outs[1], outs[0])
    assert calls[0] == calls[1] == [("init", -1)] + [("step", t) for t in range(24, -1, -1)]


def test_respaced_loop_max_steps_takes_the_first_grid_points(emu):
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    im.use_cuda_graph = False
    im.noise_fn = _bank(6)
    sched = im.noise_schedulers[0].sampling_schedule(10, 0.5, "cpu")
    im._p_sample_loop(im.unets[0], (2, 3, 64, 64), noise_scheduler=im.noise_schedulers[0],
                      text_embeds=g["text_embeds"], text_mask=g["text_mask"], cond_scale=3., schedule=sched, max_steps=3)
    assert im.noise_fn.calls == [("init", -1), ("step", 999), ("step", 888), ("step", 777)]


@pytest.mark.parametrize("eta", [0., 0.5])
def test_respaced_loop_vs_restated_ddim(emu, eta):
    """S = 8 over T = 1000 with CFG w = 3: the product's affine tables through the fused-step contract vs the paper-form
    restatement over the restated U-Net."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    im.use_cuda_graph = False
    im.noise_fn = _bank(7)
    sched = im.noise_schedulers[0].sampling_schedule(8, eta, "cpu")
    out = im._p_sample_loop(im.unets[0], (2, 3, 64, 64), noise_scheduler=im.noise_schedulers[0],
                            text_embeds=g["text_embeds"], text_mask=g["text_mask"], cond_scale=3., schedule=sched)
    assert im.noise_fn.calls == [("init", -1)] + [("step", t) for t in D.ddim_grid(1000, 8)]
    ref = restated_tiny_loop(g, 1000, 8, eta, im.noise_fn)
    err = rel_l2(out, ref)
    print(f"respaced S=8 eta={eta}: rel-L2 vs restated DDIM = {err:.3e}")
    assert err < 1e-3
    if eta == 0.:
        # deterministic given x_T: a different bank of step draws (same x_T) changes nothing
        first, other = im.noise_fn, _bank(8)
        other.bank[("init", -1)] = first.bank[("init", -1)]
        im.noise_fn = other
        out2 = im._p_sample_loop(im.unets[0], (2, 3, 64, 64), noise_scheduler=im.noise_schedulers[0],
                                 text_embeds=g["text_embeds"], text_mask=g["text_mask"], cond_scale=3., schedule=sched)
        assert not torch.equal(other.bank[("step", 999)], first.bank[("step", 999)])
        assert torch.equal(out2, out)


def test_cascade_sample_at_full_steps_vs_reference_golden(emu):
    """Imagen.sample(sampling_timesteps=25, ddim_eta=1) over the tiny 2-stage cascade (lowres augmentation, inter-stage
    resize, CFG w = 2) reproduces the reference's DDPM output and consumes its recorded draws in order."""
    from test_host_logic import _cascade_from_golden
    g = load_golden("cascade_tiny.pt")
    im, it = _cascade_from_golden(g, "cpu")
    out = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=g["cond_scale"],
                    lowres_sample_noise_level=g["lowres_noise_level"], sampling_timesteps=25, ddim_eta=1.)
    assert next(it, None) is None
    assert out.shape == g["out"].shape
    assert rel_l2(out, g["out"]) < 1e-3
    assert "step_epilogue" in emu.calls


def test_cascade_sample_per_stage_steps(emu):
    """One entry per U-Net, None keeping a stage on the DDPM loop; PIL output works on the respaced path."""
    g = load_golden("cascade_tiny.pt")
    from test_host_logic import _cascade_from_golden
    im, _ = _cascade_from_golden(g, "cpu")
    steps = []
    im.noise_fn = lambda kind, shape, step: steps.append((kind, step)) or torch.randn(shape)
    imgs = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=2.,
                     sampling_timesteps=(None, 5), ddim_eta=0.3, return_pil_images=True)
    assert len(imgs) == 2 and imgs[0].size == (32, 32)
    kinds = [s for s in steps if s[0] == "step"]
    assert [s[1] for s in kinds] == list(range(24, -1, -1)) + D.ddim_grid(25, 5)


def test_restated_ddim_step_at_full_steps_is_p_sample_step():
    """Pin of ddim_restatement.ddim_step (the reference has no DDIM): at S = T, eta = 1 it is the golden-pinned p_sample_step."""
    for T in (25, 1000):
        g = load_golden("ddpm_step.pt")[T]
        tabs = R.ddpm_tables(T)
        t = g["t"]
        t_prev = torch.where(t > 0, t - 1, torch.full_like(t, -1))
        ddim = D.ddim_step(tabs, D.alphas_cumprod_fp64(T), g["x"], t, t_prev, g["eps"], g["noise"], 1.)
        ddpm = R.p_sample_step(tabs, g["x"], t, g["eps"], g["noise"])
        assert rel_l2(ddpm, g["out"]) < 1e-6
        err = rel_l2(ddim, ddpm)
        print(f"T={T}: restated DDIM (S=T, eta=1) vs DDPM step rel-L2 = {err:.3e}")
        assert err <= 1e-6
        for i in range(t.shape[0]):                           # per image as well (t = T-1, T/3, 0)
            assert rel_l2(ddim[i], ddpm[i]) <= 1e-6


def test_sample_validation_asserts(emu):
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet, BaseTest, SuperTest
    im = Imagen(unets=(Unet(**BaseTest.defaults), Unet(**SuperTest.defaults)), text_encoder_name="t5_small",
                image_sizes=(16, 32), timesteps=25, cond_drop_prob=0.1)
    te = torch.zeros(1, 4, 512)
    with pytest.raises(AssertionError, match="one entry per unet"):
        im.sample(text_embeds=te, sampling_timesteps=(10,))
    with pytest.raises(AssertionError, match="between 2 and"):
        im.sample(text_embeds=te, sampling_timesteps=1)
    with pytest.raises(AssertionError, match="between 2 and the unet's 25 timesteps, got 31"):
        im.sample(text_embeds=te, sampling_timesteps=(None, 31))
    with pytest.raises(AssertionError, match="between 2 and the unet's 25 timesteps"):
        im.sample(text_embeds=te, sampling_timesteps=26)
    for eta in (-0.1, 1.5):
        with pytest.raises(AssertionError, match="ddim_eta must be between 0 and 1"):
            im.sample(text_embeds=te, sampling_timesteps=10, ddim_eta=eta)
    with pytest.raises(AssertionError, match="ddim_eta must be in"):
        im.noise_schedulers[0].sampling_schedule(10, 2., "cpu")
    with pytest.raises(AssertionError, match="between 2 and 25"):
        im.noise_schedulers[0].sampling_schedule(1, 0., "cpu")
