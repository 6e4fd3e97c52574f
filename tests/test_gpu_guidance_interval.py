"""Guidance intervals and guidance-weight schedules on the GPU: mi_step_epilogue_ws / mi_step_epilogue_multistep_ws bit for
bit against the _w entry points called with the scheduled weights (fused and three-kernel forms), the captured graph pair
against the eager loop, one pair serving every interval and schedule, one guided replay per guided point, the graph keys
of the two identities, and one eager Imagen.sample with every kernel call checked against float64."""
import pytest
import torch

import guidance_interval_restatement as G
from fp64_ref import scheduled_weights
from checking_ops import ALLOWED, CheckingOps
from conftest import load_golden, rel_l2
from test_gpu_inpaint import _inp
from test_guidance import _negative
from test_respaced import _bank, _tiny_imagen

pytestmark = pytest.mark.gpu
SHAPE = (2, 3, 64, 64)
INF = float("inf")


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("B,side", [(4, 64), (2, 288)])            # 3 x 288^2 > 196 608: the three-kernel form
@pytest.mark.parametrize("multistep", [False, True])
def test_scheduled_is_the_weight_array(native, B, side, multistep):
    """Per-image t at table values 0, 1 and between, one image at w = 1: the _ws call equals the _w call with
    w_eff[b] = w_b(t[b]) bit for bit, and so does the history of the multistep form."""
    from minimagen_b200.Imagen import quantile_rank
    from minimagen_b200.diffusion_model import GaussianDiffusion
    n = 3 * side * side
    gd = GaussianDiffusion(timesteps=1000).cuda()
    sch = gd.dpm_solver_schedule(10, "cuda")
    grid = list(sch.grid)
    tab = gd.guidance_table(None, "cosine", "cuda").clone()
    t = torch.tensor([grid[1], grid[3], grid[5], grid[7]][:B], device="cuda")
    tab[grid[1]], tab[grid[3]] = 0., 1.                             # s = 0 and s = 1; grid[5], grid[7] in between
    s = tab[t].tolist()
    assert s[:2] == [0., 1.] and all(0. < v < 2. and v != 1. for v in s[2:])
    gen = torch.Generator().manual_seed(B * side + multistep)
    rn = lambda: torch.randn(B, n, generator=gen).cuda()
    x, eps, eps_null, noise, hist = rn() * 1.3, rn(), rn(), rn(), rn()
    lo, hi, wq = quantile_rank(n, 0.9)
    tabs = (gd.sqrt_recip_alphas_cumprod, gd.sqrt_recipm1_alphas_cumprod, sch.c1, sch.c2, gd.sigma)
    w = torch.tensor([3., 0.5, 7.25, 1.][:B], device="cuda")
    if B == 2:
        w[1] = 1.
    w_eff = scheduled_weights(w, tab, t, B).cuda()
    assert w_eff.tolist() == [G.weights([wb], sb)[0] for wb, sb in zip(w.tolist(), s)]

    def run(scheduled):
        out, h = torch.empty_like(x), hist.clone()
        if multistep:
            if scheduled:
                native.step_epilogue_multistep_scheduled(x, eps, eps_null, w, tab, t, *tabs, sch.c3, noise, h, B, n, lo,
                                                         hi, wq, 1.0, out)
            else:
                native.step_epilogue_multistep(x, eps, eps_null, w_eff, t, *tabs, sch.c3, noise, h, B, n, lo, hi, wq, 1.0,
                                               out)
        elif scheduled:
            native.step_epilogue_scheduled(x, eps, eps_null, w, tab, t, *tabs, noise, B, n, lo, hi, wq, 1.0, out)
        else:
            native.step_epilogue(x, eps, eps_null, w_eff, t, *tabs, noise, B, n, lo, hi, wq, 1.0, out)
        return out, h

    (got, gh), (want, wh) = run(True), run(False)
    assert torch.equal(got, want) and torch.equal(gh, wh)
    # a scalar cond_scale is every image's weight
    out = torch.empty_like(x)
    native.step_epilogue_scheduled(x, eps, eps_null, 3., tab, t, *tabs, noise, B, n, lo, hi, wq, 1.0, out)
    ref = torch.empty_like(x)
    native.step_epilogue(x, eps, eps_null, scheduled_weights(3., tab, t, B).cuda(), t, *tabs, noise, B, n, lo, hi, wq,
                         1.0, ref)
    assert torch.equal(out, ref)


def test_scheduled_checks(native):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    gd = GaussianDiffusion(timesteps=25).cuda()
    B, n = 2, 3 * 16 * 16
    x = torch.zeros(B, n, device="cuda")
    t = torch.zeros(B, dtype=torch.long, device="cuda")
    args = lambda tab: (x, x, x, 3., tab, t, gd.sqrt_recip_alphas_cumprod, gd.sqrt_recipm1_alphas_cumprod,
                        gd.posterior_mean_coef1, gd.posterior_mean_coef2, gd.sigma, x, B, n, 0, 1, 0.5, 1.0, x.clone())
    with pytest.raises(TypeError, match="w_sched: expected torch.float32"):
        native.step_epilogue_scheduled(*args(torch.ones(25, device="cuda", dtype=torch.float64)))
    with pytest.raises(ValueError, match="w_sched: the guidance table must be an fp32 tensor on a CUDA device"):
        native.step_epilogue_scheduled(*args(torch.ones(25)))


# ------------------------------------------------------------------------------------------------ captured loops
def _run(im, g, flavour, graph, interval, schedule, w=3., seed=None):
    im.use_cuda_graph = graph
    im.noise_fn = None if seed is not None else _bank(9)
    sch = im.noise_schedulers[0]
    inpaint = None
    walk = sch.dpm_solver_schedule(8, "cuda") if flavour == "multistep" else sch.sampling_schedule(8, 0.5, "cuda")
    if flavour == "inpaint":
        gen = torch.Generator().manual_seed(2)
        mask = torch.zeros(2, 64, 64, dtype=torch.bool)
        mask[:, 16:48, 8:40] = True
        inpaint = _inp(torch.rand(2, 3, 64, 64, generator=gen), mask, 2)
    tab = None if interval is None and schedule is None else sch.guidance_table(interval, schedule, "cuda")
    nte, ntm = _negative()
    seeds = None if seed is None else torch.arange(seed, seed + 2, device="cuda")
    return im._p_sample_loop(im.unets[0], SHAPE, noise_scheduler=sch, text_embeds=g["text_embeds"].cuda(),
                             text_mask=g["text_mask"].cuda(), cond_scale=w, schedule=walk, inpaint=inpaint,
                             negative_text_embeds=nte.cuda(), negative_text_mask=ntm.cuda(), guidance_table=tab,
                             seeds=seeds, stage=1)


CAPTURED = [("text", (0.4, 20.), None, None), ("multistep", None, "cosine", None), ("inpaint", (0.4, 20.), None, None),
            ("text", (0.4, 20.), "linear", 5)]


@pytest.mark.parametrize("flavour,interval,schedule,seed", CAPTURED,
                         ids=["ddim_interval", "2m_cosine", "inpaint_interval", "seeded_linear"])
def test_graph_pair_vs_eager(native, flavour, interval, schedule, seed):
    """The captured pair against the eager loop, bit for bit; one cache entry holding both graphs, one guided replay per
    guided iteration."""
    from minimagen_b200.Imagen import _StepGraph
    g = load_golden("sample_loop.pt")
    w = torch.tensor([2., 4.5], device="cuda")
    eager = _run(_tiny_imagen(g, 1000, "cuda"), g, flavour, False, interval, schedule, w, seed)
    im = _tiny_imagen(g, 1000, "cuda")
    replays = []
    orig = _StepGraph.replay
    _StepGraph.replay = lambda self, guided=True: replays.append(guided) or orig(self, guided)
    try:
        graph = _run(im, g, flavour, True, interval, schedule, w, seed)
    finally:
        _StepGraph.replay = orig
    (key, pair), = im._graphs.items()
    print(f"{flavour}: graph vs eager rel-L2 = {rel_l2(graph, eager):.3e}, {sum(replays)} of {len(replays)} replays "
          f"guided")
    assert torch.equal(graph, eager)
    assert key[-1] == "guidance_table" or key[-2] == "guidance_table"
    assert pair.graph is not None and pair.graph_unguided is not None
    sch = im.noise_schedulers[0]
    grid = list((sch.dpm_solver_schedule(8, "cuda") if flavour == "multistep" else sch.sampling_schedule(8, 0.5, "cuda"))
                .grid)
    iters = [t for t in grid for _ in range(2 if flavour == "inpaint" and t > 0 else 1)]
    tab = G.table(1000, interval, schedule)
    assert replays == [tab[t] != 0. for t in iters]
    assert 0 < sum(replays) < len(replays)


def test_one_pair_serves_every_interval_and_schedule(native):
    """Loops with other intervals and schedules reuse the cached pair (the same two graphs, no recapture) and equal a
    fresh Imagen's loops."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000, "cuda")
    runs = [((0.4, 20.), None), ((1., 50.), "linear"), (None, "cosine"), ((0.1, 3.), "cosine")]
    graphs, outs = None, []
    for interval, schedule in runs:
        out = _run(im, g, "text", True, interval, schedule)
        assert len(im._graphs) == 1
        (pair,) = im._graphs.values()
        if graphs is None:
            graphs = (pair.graph, pair.graph_unguided)
        assert (pair.graph, pair.graph_unguided) == graphs
        want = _run(_tiny_imagen(g, 1000, "cuda"), g, "text", True, interval, schedule)
        print(f"{interval} {schedule}: reused pair vs fresh Imagen rel-L2 = {rel_l2(out, want):.3e}")
        assert torch.equal(out, want)
        outs.append(out)
    assert all(rel_l2(a, b) > 1e-3 for a, b in zip(outs, outs[1:]))


def test_identity_graph_keys(native):
    """A covering interval captures the plain graph (the key and bits of the loop without it); an empty one the key of
    the cond_scale = 1 loop, with its bits."""
    g = load_golden("sample_loop.pt")
    for (w, interval, schedule) in ((3., (0., INF), None), (1., (1000., 2000.), "linear")):
        im = _tiny_imagen(g, 1000, "cuda")
        want = _run(im, g, "text", True, None, None, w=w)
        keys = list(im._graphs)
        got = _run(im, g, "text", True, interval, schedule)
        assert list(im._graphs) == keys and torch.equal(got, want)
        assert keys[0][2] == (w != 1.)                                   # guided only in the covering case


# ------------------------------------------------------------------------------------------------ per-call check
@pytest.mark.parametrize("sampler", ["ddim", "dpmpp_2m"])
def test_every_call_of_an_interval_sample(native, sampler):
    """One eager Imagen.sample with an interval and the 'linear' schedule on the tiny golden U-Net: every kernel call
    checked against float64, the plain and the scheduled step epilogues both reached."""
    import minimagen_b200.ops as ops_mod
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000, "cuda")
    im.use_cuda_graph = False
    im.noise_fn = _bank(4)
    proxy = CheckingOps(native)
    ops_mod.set_ops(proxy)                              # the `native` fixture restores the previous backend afterwards
    out = im.sample(text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda(),
                    cond_scale=torch.tensor([2., 4.5]), sampling_timesteps=4, sampler=sampler,
                    guidance_interval=(0.4, 20.), guidance_schedule="linear")
    torch.cuda.synchronize()
    proxy.report()
    assert torch.isfinite(out).all()
    unchecked = proxy.called - proxy.checked - ALLOWED
    assert not unchecked, f"kernels that ran without a float64 check: {sorted(unchecked)}"
    step = "step_epilogue_multistep" if sampler == "dpmpp_2m" else "step_epilogue"
    assert {step, step + "_scheduled", "step_finalize"} <= proxy.checked
