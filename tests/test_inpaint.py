"""Inpainting with RePaint resampling (Imagen.sample(inpaint_images=, inpaint_masks=, inpaint_resample_times=)) on the CPU,
through the torch emulation of the ops interface extended by the three inpainting entry points.  Covers the re-noising
tables, the iteration plan and its draws, the argument checks, the pin of inpaint_restatement to the plain loops, and the
emulated sampler against that restatement.  (The kernels, the captured graph and the cascade are covered on the GPU in
test_gpu_inpaint.py.)"""
import pytest
import torch

import ddim_restatement as D
import inpaint_restatement as P
from conftest import load_golden, rel_l2
from oracle import restatement as R
from test_respaced import _bank, _tiny_imagen

SHAPE = (2, 3, 64, 64)


def known_and_mask(seed, shape=SHAPE, frac=0.5):
    """A known image in [0, 1] and a random bool mask (True = known)."""
    gen = torch.Generator().manual_seed(seed)
    img = torch.rand(shape, generator=gen)
    mask = torch.rand((shape[0], *shape[2:]), generator=gen) < frac
    return img, mask


def sample_tiny(im, g, img, mask, R, steps=None, eta=0.):
    return im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=3., inpaint_images=img,
                     inpaint_masks=mask, inpaint_resample_times=R, sampling_timesteps=steps, ddim_eta=eta)


def restated_tiny(g, T, img, mask, R, noise_fn, steps=None, eta=0.):
    return P.inpaint_loop(g["state_dict"], g["cfg"], SHAPE, T, img * 2 - 1, mask, R, noise_fn, steps=steps, eta=eta,
                          text_embeds=g["text_embeds"].cpu(), text_mask=g["text_mask"].cpu())


# ------------------------------------------------------------------------------------------------ tables
@pytest.mark.parametrize("T", [20, 25, 1000])
def test_ddpm_tables(T):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    gd = GaussianDiffusion(timesteps=T)
    next_t, ra, rb = gd.inpaint_tables(None, "cpu")
    assert ra.dtype == rb.dtype == torch.float32 and next_t.dtype == torch.int64
    assert ra.shape == rb.shape == next_t.shape == (T,)
    assert torch.equal(next_t, (torch.arange(T) - 1).clamp(min=0))
    assert ra[0] == 1 and rb[0] == 0
    eps = torch.finfo(torch.float32).eps
    assert ((ra.double() ** 2 + rb.double() ** 2 - 1).abs() <= 4 * eps).all()
    assert ((ra.double() - (1. - gd.betas.double()).sqrt())[1:].abs() <= eps).all()
    assert gd.inpaint_tables(None, "cpu")[1] is ra                  # cached per walk


@pytest.mark.parametrize("S", [2, 8, 25])
def test_ddim_tables_follow_the_grid(S):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    T = 25
    gd = GaussianDiffusion(timesteps=T)
    sched = gd.sampling_schedule(S, 0.5, "cpu")
    next_t, ra, rb = gd.inpaint_tables(sched, "cpu")
    assert next_t is sched.next_t
    acp = D.alphas_cumprod_fp64(T)
    grid = D.ddim_grid(T, S)
    for t, t_next in zip(grid, grid[1:]):
        a = acp[t] / acp[t_next]
        assert ra[t] == a.sqrt().float() and rb[t] == (1. - a).sqrt().float()
    off = [t for t in range(T) if t not in grid[:-1]]               # t = 0 and the timesteps off the grid
    assert (ra[off] == 1).all() and (rb[off] == 0).all()


# ------------------------------------------------------------------------------------------------ plan and draws
@pytest.mark.parametrize("R_", [1, 3])
def test_plan_and_draw_sequence(emu, R_):
    """(S - 1) R + 1 iterations, draws 'renoise' (r > 0), 'inpaint', 'step' labelled t * R + r; at R = 1 the 'step'
    labels are those of the plain DDIM loop."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 25)
    im.use_cuda_graph = False
    im.noise_fn = _bank(1)
    img, mask = known_and_mask(1)
    sample_tiny(im, g, img, mask, R_, steps=4)
    grid = D.ddim_grid(25, 4)
    want = [("init", -1)]
    for t in grid:
        for r in range(R_ if t > 0 else 1):
            want += ([("renoise", t * R_ + r)] if r > 0 else []) + [("inpaint", t * R_ + r), ("step", t * R_ + r)]
    assert im.noise_fn.calls == want
    assert len(P.plan(25, R_, 4)) == (4 - 1) * R_ + 1 == emu.calls.count("inpaint_prologue")
    assert emu.calls.count("step_epilogue") == (4 - 1) * R_ + 1
    if R_ == 1:
        assert [c for c in want if c[0] == "step"] == [("step", t) for t in grid]


def test_max_steps_counts_iterations(emu):
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 25)
    im.use_cuda_graph = False
    im.noise_fn = _bank(2)
    img, mask = known_and_mask(2)
    k, m = (img * 2 - 1).contiguous(), mask.float().reshape(2, -1)
    im._p_sample_loop(im.unets[0], SHAPE, noise_scheduler=im.noise_schedulers[0], text_embeds=g["text_embeds"],
                      text_mask=g["text_mask"], cond_scale=3., max_steps=4, inpaint=(k, m, 3))
    assert im.noise_fn.calls == [("init", -1), ("inpaint", 72), ("step", 72), ("renoise", 73), ("inpaint", 73),
                                 ("step", 73), ("renoise", 74), ("inpaint", 74), ("step", 74), ("inpaint", 69),
                                 ("step", 69)]


def test_graph_key_ignores_the_walk():
    """DDPM and DDIM lookups of one signature hit the same cached text-only graph, which installs the walk it is given on
    every hit; the inpainting graph has its own key.  Graphs stand in for captured ones in the cache (no GPU needed)."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 25)
    sch = im.noise_schedulers[0]
    args = (im.unets[0], SHAPE, sch, g["text_embeds"], g["text_mask"], None, None, 3.)
    assert im._graph_key(*args, inpaint=True) == im._graph_key(*args) + ("inpaint",)

    class Cached:
        def __init__(self):
            self.walks, self.inpaints = [], []

        def set_cond(self, **cond):
            pass

        def set_schedule(self, sched):
            self.walks.append(sched)

        def set_inpaint(self, *args):
            self.inpaints.append(args)

    text, inp = Cached(), Cached()
    im._graphs = {im._graph_key(*args): text, im._graph_key(*args, inpaint=True): inp}
    kw = dict(noise_scheduler=sch, text_embeds=g["text_embeds"], text_mask=g["text_mask"], lowres_cond_img=None,
              lowres_noise_times=None, cond_scale=3.)
    ddim = sch.sampling_schedule(8, 0.5, "cpu")
    assert im._step_graph(im.unets[0], SHAPE, **kw) is text
    assert im._step_graph(im.unets[0], SHAPE, schedule=ddim, **kw) is text
    assert im._step_graph(im.unets[0], SHAPE, **kw) is text
    ddpm = sch.ddpm_schedule("cpu")
    assert len(text.walks) == 3 and all(w is want for w, want in zip(text.walks, (ddpm, ddim, ddpm)))
    assert not text.inpaints
    img, mask = known_and_mask(0)
    k, m = (img * 2 - 1).contiguous(), mask.float().reshape(2, -1)
    assert im._step_graph(im.unets[0], SHAPE, schedule=ddim, inpaint=(k, m, 3), **kw) is inp
    _, ra, rb = sch.inpaint_tables(ddim, "cpu")
    assert len(inp.walks) == 1 and inp.walks[0] is ddim and len(inp.inpaints) == 1
    assert all(a is b for a, b in zip(inp.inpaints[0], (k, m, 3, ra, rb)))
    assert len(im._graphs) == 2


# ------------------------------------------------------------------------------------------------ argument checks
def test_inpaint_asserts(emu):
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet, BaseTest, SuperTest
    im = Imagen(unets=(Unet(**BaseTest.defaults), Unet(**SuperTest.defaults)), text_encoder_name="t5_small",
                image_sizes=(16, 32), timesteps=25, cond_drop_prob=0.1)
    te = torch.zeros(2, 4, 512)
    img, mask = torch.rand(2, 3, 32, 32), torch.ones(2, 32, 32, dtype=torch.bool)
    with pytest.raises(AssertionError, match="inpaint_images and inpaint_masks must be given together"):
        im.sample(text_embeds=te, inpaint_images=img)
    with pytest.raises(AssertionError, match="inpaint_images and inpaint_masks must be given together"):
        im.sample(text_embeds=te, inpaint_masks=mask)
    for bad in (0, -1, 2.0, True, None):
        with pytest.raises(AssertionError, match="inpaint_resample_times must be an int >= 1, got"):
            im.sample(text_embeds=te, inpaint_images=img, inpaint_masks=mask, inpaint_resample_times=bad)
    with pytest.raises(AssertionError, match="inpaint_images must be a float tensor"):
        im.sample(text_embeds=te, inpaint_images=(img * 255).to(torch.uint8), inpaint_masks=mask)
    for bad in (torch.rand(3, 3, 32, 32), torch.rand(2, 1, 32, 32), torch.rand(2, 3, 32, 16), torch.rand(2, 3, 32)):
        with pytest.raises(AssertionError, match=r"inpaint_images must be \(b, channels, s, s\) = \(2, 3, s, s\), got"):
            im.sample(text_embeds=te, inpaint_images=bad, inpaint_masks=mask)
    with pytest.raises(AssertionError, match="inpaint_masks must be a bool tensor"):
        im.sample(text_embeds=te, inpaint_images=img, inpaint_masks=mask.float())
    for bad in (mask[:1], mask[:, :16], mask[:, None]):
        with pytest.raises(AssertionError, match=r"inpaint_masks must be \(b, s, s\) = \(2, 32, 32\), got"):
            im.sample(text_embeds=te, inpaint_images=img, inpaint_masks=bad)


# ------------------------------------------------------------------------------------------------ restatement pin
def test_restatement_r1_nothing_known_is_the_plain_loop():
    """R = 1 with an all-False mask: inpaint_restatement is ddim_restatement.ddim_loop (DDIM) and the loop over the
    golden-pinned restatement.p_sample_step (DDPM), bit for bit."""
    g = load_golden("sample_loop.pt")
    img, _ = known_and_mask(3)
    none = torch.zeros(2, 64, 64, dtype=torch.bool)
    bank = _bank(3)
    got = restated_tiny(g, 25, img, none, 1, bank, steps=6, eta=0.5)
    want = D.ddim_loop(g["state_dict"], g["cfg"], SHAPE, 25, 6, 0.5, bank, text_embeds=g["text_embeds"],
                       text_mask=g["text_mask"])
    assert torch.equal(got, want)

    T = 25
    bank = _bank(4)
    got = restated_tiny(g, T, img, none, 1, bank)
    tabs = R.ddpm_tables(T)
    x = bank("init", SHAPE, -1)
    kw = dict(text_embeds=g["text_embeds"], text_mask=g["text_mask"])
    with torch.no_grad():
        for tau in range(T - 1, -1, -1):
            t = torch.full((2,), tau, dtype=torch.long)
            eps = R.cfg_combine(R.unet_forward(g["state_dict"], g["cfg"], x, t, **kw),
                                R.unet_forward(g["state_dict"], g["cfg"], x, t, cond_drop_prob=1., **kw), 3.)
            x = R.p_sample_step(tabs, x, t, eps, bank("step", SHAPE, tau))
    assert torch.equal(got, (x.clamp(-1, 1) + 1) * 0.5)


# ------------------------------------------------------------------------------------------------ emulated sampler
@pytest.mark.parametrize("T,S,R_", [(25, None, 2), (25, 5, 3)])
def test_emulated_sample_vs_restatement(emu, T, S, R_):
    """Imagen.sample with inpainting (CFG w = 3, random mask) on sample_loop.pt's tiny U-Net, DDPM and DDIM (eta 0.5),
    against the RePaint-form restatement over the restated U-Net; the known pixels are the inputs."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, T)
    im.use_cuda_graph = False
    im.noise_fn = _bank(10 + R_)
    img, mask = known_and_mask(5)
    out = sample_tiny(im, g, img, mask, R_, steps=S, eta=0.5)
    ref = restated_tiny(g, T, img, mask, R_, im.noise_fn, steps=S, eta=0.5)
    err = rel_l2(out, ref)
    print(f"T={T} S={S} R={R_}: emulated sample vs restated RePaint rel-L2 = {err:.3e}")
    assert err < 1e-3
    keep = mask[:, None].expand(SHAPE)
    assert (out - img)[keep].abs().max() <= 1.2e-7
