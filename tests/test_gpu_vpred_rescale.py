"""v-prediction, zero-terminal-SNR schedules and guidance rescale on the GPU: mi_guidance_rescale_factor within one fp32
ulp of float64 from 3 x 64^2 to 3 x 1024^2 per image and B up to 64 (with an SS_g = 0 image, a NaN image and an image
offset to mean 10^3 std), deterministic; mi_step_epilogue_rescaled bit for bit the plain epilogue fed fp32(g * f) and
within the step's float64 bounds, fused and three-kernel; the captured rescaled loops bit for bit the eager ones, one
graph serving every phi; one guided cfg-3 sampling step at the benchmark's size and one 'v' zero-SNR training step with
every kernel call of the loop (resp. the step) checked against float64."""
import time

import pytest
import torch

import fp64_ref as R
from checking_ops import ALLOWED, CheckingOps
from conftest import load_golden, rel_l2
from test_gpu_inpaint import _inp
from test_guidance import _negative
from test_respaced import _bank, _tiny_imagen

pytestmark = pytest.mark.gpu
SHAPE = (2, 3, 64, 64)
F32 = torch.float32


def _pred_pair(B, n, seed, edge=False):
    gen = torch.Generator().manual_seed(seed)
    c = torch.randn(B, n, generator=gen) * (0.5 + torch.rand(B, 1, generator=gen))
    u = torch.randn(B, n, generator=gen) * 0.8 + 0.1
    if edge:
        c[1], u[1] = 0.25, 0.25                                   # SS_g = 0 (and SS_c = 0): f = 1
        c[2, n // 3] = float("nan")                               # f = NaN
        c[3] = 1e3 + c[3] / c[3].std()                            # mean 10^3 std: a one-pass sum of squares cancels
        u[3] = 1e3 + u[3]
    return c, u


# ------------------------------------------------------------------------------------------------ factor kernel
FACTOR_CASES = [(1, 64), (32, 256), (64, 64), (64, 256), (1, 1024), (2, 1024)]


@pytest.mark.parametrize("B,side", FACTOR_CASES)
@pytest.mark.parametrize("table", [False, True])
def test_factor_within_one_ulp(native, B, side, table):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    n = 3 * side * side
    c, u = _pred_pair(B, n, B * side + table)
    gen = torch.Generator().manual_seed(7)
    w = (1. + 7. * torch.rand(B, generator=gen)).cuda()
    t = torch.randint(0, 1000, (B,), generator=gen).cuda()
    w_sched = GaussianDiffusion(timesteps=1000).guidance_table(None, "cosine", "cuda") if table else None
    phi = torch.rand(B, generator=gen).cuda()
    f = torch.empty(B, device="cuda")
    native.guidance_rescale_factor(c.cuda(), u.cuda(), w, w_sched, t, phi, B, n, f)
    ref, bound = R.rescale_factor_ref(c, u, w, w_sched, t, phi, B, n)
    R.check(f, ref, bound, f"factor B={B} n={n}")
    f2 = torch.empty(B, device="cuda")
    native.guidance_rescale_factor(c.cuda(), u.cuda(), w, w_sched, t, phi, B, n, f2)
    assert torch.equal(f, f2)                                       # a fixed reduction order


@pytest.mark.parametrize("side", [64, 1024])
def test_factor_edge_images(native, side):
    B, n = 4, 3 * side * side
    c, u = _pred_pair(B, n, side, edge=True)
    w = torch.tensor([3., 5., 2., 4.], device="cuda")
    t = torch.zeros(B, dtype=torch.long, device="cuda")
    phi = torch.tensor([0.7, 0.7, 0.7, 1.], device="cuda")
    f = torch.empty(B, device="cuda")
    native.guidance_rescale_factor(c.cuda(), u.cuda(), w, None, t, phi, B, n, f)
    assert f[1] == 1 and torch.isnan(f[2])
    ref, bound = R.rescale_factor_ref(c, u, w, None, t, phi, B, n)
    keep = torch.tensor([0, 3])
    print(f"offset image: f = {float(f[3]):.9g}, float64 {float(ref[3]):.9g}")
    R.check(f[keep.cuda()], ref[keep], bound[keep], f"factor edge images n={n}")


# ------------------------------------------------------------------------------------------------ rescaled epilogue
@pytest.mark.parametrize("B,side", [(4, 256), (2, 1024)])         # fused, and 3 x 1024^2 > 196 608: three kernels
@pytest.mark.parametrize("multistep", [False, True])
@pytest.mark.parametrize("table", [False, True])
def test_rescaled_epilogue_is_the_plain_epilogue(native, B, side, multistep, table):
    """Bit for bit mi_step_epilogue(_multistep) fed eps = fp32(g * f) and no guidance pass, and within its float64 bounds
    (the per-call checker), on the v tables of a zero-SNR schedule at per-image t (T-1 included)."""
    from minimagen_b200.Imagen import quantile_rank
    from minimagen_b200.diffusion_model import ZeroTerminalSNRDiffusion
    n = 3 * side * side
    gd = ZeroTerminalSNRDiffusion(timesteps=1000).cuda()
    sch = gd.dpm_solver_schedule(10, "cuda")
    grid = list(sch.grid)
    t = torch.tensor([grid[0], grid[2], grid[5], grid[9]][:B], device="cuda")
    c, u = (v.cuda() for v in _pred_pair(B, n, side + 10 * multistep))
    gen = torch.Generator().manual_seed(side)
    x = (torch.randn(B, n, generator=gen) * 1.2).cuda()
    noise, hist = torch.randn(B, n, generator=gen).cuda(), (torch.randn(B, n, generator=gen) * 0.3).cuda()
    w = torch.tensor([3., 7.5, 1.5, 5.][:B], device="cuda")
    w_sched = gd.guidance_table(None, "linear", "cuda") if table else None
    phi = torch.tensor([0.7, 1., 0.3, 0.5][:B], device="cuda")
    f = torch.empty(B, device="cuda")
    native.guidance_rescale_factor(c, u, w, w_sched, t, phi, B, n, f)
    lo, hi, wq = quantile_rank(n, 0.9)
    a, b = gd.sqrt_alphas_cumprod, gd.sqrt_one_minus_alphas_cumprod
    c3 = sch.c3 if multistep else None
    out, h, s = torch.empty_like(x), hist.clone() if multistep else None, torch.empty(B, device="cuda")
    native.step_epilogue_rescaled(x, c, u, w, w_sched, f, t, a, b, sch.c1, sch.c2, sch.sigma, c3, noise, h, B, n, lo, hi,
                                  wq, 1.0, out, s_out=s)
    eps = R.rescaled_eps_fp32(c, u, w, w_sched, t, f, B, n).cuda()
    want, wh = torch.empty_like(x), hist.clone() if multistep else None
    if multistep:
        native.step_epilogue_multistep(x, eps, None, 1.0, t, a, b, sch.c1, sch.c2, sch.sigma, c3, noise, wh, B, n, lo, hi,
                                       wq, 1.0, want)
    else:
        native.step_epilogue(x, eps, None, 1.0, t, a, b, sch.c1, sch.c2, sch.sigma, noise, B, n, lo, hi, wq, 1.0, want)
    assert torch.equal(out, want) and (not multistep or torch.equal(h, wh))
    proxy = CheckingOps(native)
    h = hist.clone() if multistep else None
    proxy.step_epilogue_rescaled(x, c, u, w, w_sched, f, t, a, b, sch.c1, sch.c2, sch.sigma, c3, noise, h, B, n, lo, hi,
                                 wq, 1.0, torch.empty_like(x), s_out=torch.empty(B, device="cuda"))
    proxy.guidance_rescale_factor(c, u, w, w_sched, t, phi, B, n, torch.empty(B, device="cuda"))
    assert proxy.checked == {"step_epilogue_rescaled", "guidance_rescale_factor"}
    proxy.report()


# ------------------------------------------------------------------------------------------------ captured loops
def _imagen_v(g):
    return _tiny_imagen(g, 1000, "cuda").set_objectives('v', True)


def _run(im, g, flavour, graph, phi, table=None, seed=None):
    im.use_cuda_graph = graph
    im.noise_fn = None if seed is not None else _bank(9)
    sch = im.noise_schedulers[0]
    walk = sch.dpm_solver_schedule(8, "cuda") if flavour == "multistep" else sch.sampling_schedule(8, 0.5, "cuda")
    inpaint = None
    if flavour == "inpaint":
        gen = torch.Generator().manual_seed(2)
        mask = torch.zeros(2, 64, 64, dtype=torch.bool)
        mask[:, 16:48, 8:40] = True
        inpaint = _inp(torch.rand(2, 3, 64, 64, generator=gen), mask, 2)
    tab = None if table is None else sch.guidance_table(table[0], table[1], "cuda")
    nte, ntm = _negative()
    seeds = None if seed is None else torch.arange(seed, seed + 2, device="cuda")
    return im._p_sample_loop(im.unets[0], SHAPE, noise_scheduler=sch, text_embeds=g["text_embeds"].cuda(),
                             text_mask=g["text_mask"].cuda(), cond_scale=torch.tensor([2., 4.5], device="cuda"),
                             schedule=walk, inpaint=inpaint, negative_text_embeds=nte.cuda(),
                             negative_text_mask=ntm.cuda(), guidance_table=tab, seeds=seeds, stage=1,
                             **({} if phi is None else dict(guidance_rescale=phi)))


CAPTURED = [("text", None, None), ("multistep", None, None), ("inpaint", None, None),
            ("text", ((0.4, 20.), "linear"), None), ("text", None, 5)]


@pytest.mark.parametrize("flavour,table,seed", CAPTURED, ids=["ddim", "2m", "inpaint", "table_pair", "seeded"])
def test_rescaled_graph_vs_eager(native, flavour, table, seed):
    """v on a zero-SNR schedule, per-image phi: the captured loop equals the eager loop bit for bit; a second phi replays
    the same graph (no recapture) and equals its eager loop too."""
    g = load_golden("sample_loop.pt")
    im = _imagen_v(g)
    outs = []
    for phi in (torch.tensor([0.7, 1.], device="cuda"), 0.25):
        graph = _run(im, g, flavour, True, phi, table, seed)
        assert len(im._graphs) == 1
        (key, sg), = im._graphs.items()
        if not outs:
            first = (sg.graph, sg.graph_unguided)
        assert (sg.graph, sg.graph_unguided) == first and 'rescaled' in key
        eager = _run(_imagen_v(g), g, flavour, False, phi, table, seed)
        print(f"{flavour} phi={phi}: graph vs eager rel-L2 = {rel_l2(graph, eager):.3e}")
        assert torch.equal(graph, eager)
        outs.append(graph)
    assert rel_l2(outs[0], outs[1]) > 1e-4
    if table is not None:
        assert sg.graph_unguided is not None


def test_phi_zero_is_the_plain_graph(native):
    g = load_golden("sample_loop.pt")
    im = _imagen_v(g)
    want = _run(im, g, "text", True, None)
    keys = list(im._graphs)
    got = _run(im, g, "text", True, 0.)
    assert list(im._graphs) == keys and 'rescaled' not in keys[0] and torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ per-call checks
LOOP = {"step_epilogue", "step_epilogue_multistep", "step_advance_t", "step_advance_t_table", "step_finalize",
        "resize_separable", "q_sample", "guidance_rescale_factor", "step_epilogue_rescaled"}


def test_one_rescaled_cfg3_sampling_step_at_benchmark_size(native):
    """Imagen.sample(start_at_unet_number=2) with bench.py's cfg-3 U-Net as a 'v', zero-SNR second stage, b = 32 at
    256 x 256, two DDIM steps (eager) with w = 5 and phi = 0.7: every kernel of the loop -- the resize, q_sample, the
    rescale factor, the rescaled step, the finalize -- checked against float64.  The U-Net calls at this size are checked
    by test_gpu_flagship_calls.py."""
    import bench
    import minimagen_b200.ops as ops_mod
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import BaseTest, Unet
    wl = bench.workload("cfg3")
    size, low, b = wl["size"], wl["size"] // 4, 32
    torch.manual_seed(0)
    u = Unet(**wl["cfg"]).eval()
    first = Unet(**dict(BaseTest.defaults, text_embed_dim=wl["E"])).eval()
    im = Imagen(unets=(first, u), text_encoder_name="t5_base", image_sizes=(low, size), timesteps=1000,
                cond_drop_prob=0.1).eval().cuda().set_objectives(('noise', 'v'), (False, True))
    im.use_cuda_graph = False
    g = torch.Generator().manual_seed(11)
    te = torch.randn(b, 20, wl["E"], generator=g).cuda()
    tm = torch.ones(b, 20, dtype=torch.bool)
    tm[-1, 5:] = False
    start = torch.rand(b, 3, low, low, generator=g).cuda()
    proxy = CheckingOps(native, only=LOOP)
    ops_mod.set_ops(proxy)                                  # the `native` fixture restores the previous backend afterwards
    t0 = time.time()
    out = im.sample(text_embeds=te, text_masks=tm.cuda(), cond_scale=5., sampling_timesteps=2, start_at_unet_number=2,
                    start_images=start, guidance_rescale=0.7)
    torch.cuda.synchronize()
    print(f"\ntwo rescaled cfg3 sampling steps, b = {b}: {time.time() - t0:.1f} s")
    proxy.report()
    assert tuple(out.shape) == (b, 3, size, size) and torch.isfinite(out).all()
    assert proxy.family["step_epilogue_rescaled"][0] == 2 and proxy.family["guidance_rescale_factor"][0] == 2
    assert {"step_epilogue_rescaled", "guidance_rescale_factor", "step_finalize", "q_sample"} <= proxy.checked


def test_every_call_of_a_v_zero_snr_training_step(native):
    """The two-stage tiny cascade of train_tiny.pt with 'v' and zero-SNR schedules: one eager training step of each U-Net,
    every kernel call checked against float64 (the v target is q_sample with the tables (-sqrt(1 - a), sqrt(a)))."""
    import minimagen_b200.ops as ops_mod
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet
    g = load_golden("train_tiny.pt")
    im = Imagen(unets=[Unet(**c["cfg"]) for c in g["cases"]], text_encoder_name="t5_small", image_sizes=g["image_sizes"],
                timesteps=g["timesteps"], cond_drop_prob=g["cond_drop_prob"]).set_objectives('v', True)
    for u, c in zip(im.unets, g["cases"]):
        u.load_state_dict(c["state_dict"])
    im = im.cuda().train()
    images = torch.rand(3, 3, 40, 40, generator=torch.Generator().manual_seed(3)).cuda()
    for unet_number in (1, 2):
        proxy = CheckingOps(native, fresh_accumulators=True)
        ops_mod.set_ops(proxy)
        torch.manual_seed(5)
        loss = im(images, text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda(), unet_number=unet_number)
        loss.backward()
        torch.cuda.synchronize()
        assert torch.isfinite(loss.detach())
        proxy.report()
        unchecked = proxy.called - proxy.checked - ALLOWED
        assert not unchecked, f"kernels that ran without a float64 check: {sorted(unchecked)}"
        assert proxy.family["q_sample"][0] >= 2                 # x_t and the v target
        im.zero_grad(set_to_none=True)
