"""Negative prompts and per-image guidance weights on the GPU: mi_step_epilogue_w / mi_step_epilogue_multistep_w bit for bit
against the scalar entry points image by image (fused and three-kernel forms), the captured loop against the eager one
with a negative prompt and per-image weights in the three graph flavours, one captured graph serving every scale and
negative prompt, and the native path against the CPU emulation."""
import pytest
import torch

from conftest import load_golden, rel_l2
from emu_ops import EmuOps
from test_gpu_inpaint import _inp
from test_guidance import _negative
from test_respaced import _bank, _tiny_imagen

pytestmark = pytest.mark.gpu
SHAPE = (2, 3, 64, 64)


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("B,side", [(3, 64), (2, 288)])            # 3 x 288^2 > 196 608: the three-kernel form
@pytest.mark.parametrize("multistep", [False, True])
def test_weight_array_is_the_scalar_per_image(native, B, side, multistep):
    from minimagen_b200.Imagen import quantile_rank
    from minimagen_b200.diffusion_model import GaussianDiffusion
    n = 3 * side * side
    gd = GaussianDiffusion(timesteps=1000).cuda()
    sch = gd.dpm_solver_schedule(10, "cuda")
    gen = torch.Generator().manual_seed(B * side + multistep)
    rn = lambda: torch.randn(B, n, generator=gen).cuda()
    x, eps, eps_null, noise, hist = rn() * 1.3, rn(), rn(), rn(), rn()
    grid = list(sch.grid)
    t = torch.tensor([grid[3], grid[1], 0][:B], device="cuda")
    lo, hi, wq = quantile_rank(n, 0.9)
    tabs = (t, gd.sqrt_recip_alphas_cumprod, gd.sqrt_recipm1_alphas_cumprod, sch.c1, sch.c2, gd.sigma)
    scales = [3., 0.5, 7.25][:B]

    def run(cond_scale, h):
        out = torch.empty_like(x)
        if multistep:
            native.step_epilogue_multistep(x, eps, eps_null, cond_scale, *tabs, sch.c3, noise, h, B, n, lo, hi, wq, 1.0, out)
        else:
            native.step_epilogue(x, eps, eps_null, cond_scale, *tabs, noise, B, n, lo, hi, wq, 1.0, out)
        return out

    h = hist.clone()
    got = run(torch.tensor(scales, device="cuda"), h)
    for i, w in enumerate(scales):
        h_i = hist.clone()
        want = run(w, h_i)
        assert torch.equal(got[i], want[i]), (i, w)
        if multistep:
            assert torch.equal(h[i], h_i[i])
    # the scale is ignored without a guidance pass: any weights give the unguided bits
    out = torch.empty_like(x)
    native.step_epilogue(x, eps, None, torch.full((B,), 5., device="cuda"), *tabs, noise, B, n, lo, hi, wq, 1.0, out)
    plain = torch.empty_like(x)
    native.step_epilogue(x, eps, None, 1., *tabs, noise, B, n, lo, hi, wq, 1.0, plain)
    assert torch.equal(out, plain)


def test_weight_array_checks(native):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    gd = GaussianDiffusion(timesteps=25).cuda()
    B, n = 2, 3 * 16 * 16
    x = torch.zeros(B, n, device="cuda")
    t = torch.zeros(B, dtype=torch.long, device="cuda")
    args = lambda w: (x, x, x, w, t, gd.sqrt_recip_alphas_cumprod, gd.sqrt_recipm1_alphas_cumprod,
                      gd.posterior_mean_coef1, gd.posterior_mean_coef2, gd.sigma, x, B, n, 0, 1, 0.5, 1.0, x.clone())
    with pytest.raises(ValueError, match="expected 2 per-image weights, got 3"):
        native.step_epilogue(*args(torch.ones(3, device="cuda")))
    with pytest.raises(TypeError, match="cond_scale: expected torch.float32"):
        native.step_epilogue(*args(torch.ones(2, device="cuda", dtype=torch.float64)))
    with pytest.raises(ValueError, match="contiguous"):
        native.step_epilogue(*args(torch.ones(4, device="cuda")[::2]))
    with pytest.raises(ValueError, match="CUDA device"):
        native.step_epilogue(*args(torch.ones(2)))


# ------------------------------------------------------------------------------------------------ captured loops
def _flavour_loop(im, g, flavour, graph, w, nte, ntm):
    im.use_cuda_graph = graph
    im.noise_fn = _bank(9)
    sch = im.noise_schedulers[0]
    inpaint = None
    if flavour == "multistep":
        walk = sch.dpm_solver_schedule(8, "cuda")
    else:
        walk = sch.sampling_schedule(8, 0.5, "cuda")
    if flavour == "inpaint":
        gen = torch.Generator().manual_seed(2)
        mask = torch.zeros(2, 64, 64, dtype=torch.bool)
        mask[:, 16:48, 8:40] = True
        inpaint = _inp(torch.rand(2, 3, 64, 64, generator=gen), mask, 2)
    return im._p_sample_loop(im.unets[0], SHAPE, noise_scheduler=sch, text_embeds=g["text_embeds"].cuda(),
                             text_mask=g["text_mask"].cuda(), cond_scale=w, schedule=walk, inpaint=inpaint,
                             negative_text_embeds=None if nte is None else nte.cuda(),
                             negative_text_mask=None if ntm is None else ntm.cuda())


@pytest.mark.parametrize("flavour", ["text", "inpaint", "multistep"])
def test_graph_vs_eager_negative_per_image(native, flavour):
    g = load_golden("sample_loop.pt")
    nte, ntm = _negative()
    w = torch.tensor([2., 4.5], device="cuda")
    outs = {}
    for graph in (False, True):
        im = _tiny_imagen(g, 1000, "cuda")
        outs[graph] = _flavour_loop(im, g, flavour, graph, w, nte, ntm)
        if graph:
            assert len(im._graphs) == 1
    null = _flavour_loop(_tiny_imagen(g, 1000, "cuda"), g, flavour, True, w, None, None)
    err = rel_l2(outs[True], outs[False])
    print(f"{flavour}: graph vs eager rel-L2 = {err:.3e}; vs null guidance {rel_l2(outs[True], null):.3e}")
    assert err <= 1e-5
    assert rel_l2(outs[True], null) > 1e-2


def test_one_graph_serves_every_scale_and_negative(native):
    """Loops at 3, then 5, then a per-image vector, then a new negative prompt leave one captured graph; each output equals
    a fresh Imagen's."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000, "cuda")
    nte, ntm = _negative()
    nte2, ntm2 = _negative(seed=12)
    runs = [(3., nte, ntm), (5., nte, ntm), (torch.tensor([1.5, 6.], device="cuda"), nte, ntm), (4., nte2, ntm2)]
    outs = []
    for w, a, m in runs:
        out = _flavour_loop(im, g, "text", True, w, a, m)
        want = _flavour_loop(_tiny_imagen(g, 1000, "cuda"), g, "text", True, w, a, m)
        err = rel_l2(out, want)
        print(f"w={w}: reused graph vs fresh Imagen rel-L2 = {err:.3e}")
        assert err <= 1e-5
        outs.append(out)
    assert len(im._graphs) == 1
    assert all(rel_l2(a, b) > 1e-3 for a, b in zip(outs, outs[1:]))


def test_native_vs_emulated(native):
    """sample() with a negative prompt and per-image weights on the tiny golden config: GPU (captured graph) vs the CPU
    emulation with the same draws."""
    import minimagen_b200.ops as ops_mod
    g = load_golden("sample_loop.pt")
    nte, ntm = _negative()
    outs = {}
    for dev in ("cuda", "cpu"):
        prev = ops_mod._OPS
        if dev == "cpu":
            ops_mod.set_ops(EmuOps())
        try:
            im = _tiny_imagen(g, 1000, dev)
            im.noise_fn = _bank(4)
            outs[dev] = im.sample(text_embeds=g["text_embeds"].to(dev), text_masks=g["text_mask"].to(dev),
                                  cond_scale=torch.tensor([2., 4.5]), sampling_timesteps=8,
                                  negative_text_embeds=nte.to(dev), negative_text_masks=ntm.to(dev)).cpu()
        finally:
            ops_mod.set_ops(prev)
    err = rel_l2(outs["cuda"], outs["cpu"])
    print(f"native vs emulated: rel-L2 = {err:.3e}")
    assert err < 1e-3
