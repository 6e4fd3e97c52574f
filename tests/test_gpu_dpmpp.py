"""DPM-Solver++(2M) sampling on the GPU: mi_step_epilogue_multistep bit for bit against its torch contract (fused and
three-kernel forms, eagerly and captured), the multistep graph against the eager loop, the paper-form restatement, DDIM at
S = 2 and the analytic ODE end point; graph flavours side by side on one Imagen; batch sharding; a cascade against the
CPU emulation."""
import pytest
import torch

import dpmpp_restatement as P
from conftest import load_golden, rel_l2
from emu_ops import EmuOps, multistep_ref
from test_dpmpp import SHAPE, AnalyticEps, analytic_errors
from test_gpu_inpaint import _capture
from test_respaced import _bank, _tiny_imagen

pytestmark = pytest.mark.gpu


def _loop(im, g, sched, graph=True, unet=None, cond_scale=3.):
    im.use_cuda_graph = graph
    return im._p_sample_loop(im.unets[0] if unet is None else unet, SHAPE, noise_scheduler=im.noise_schedulers[0],
                             text_embeds=g["text_embeds"].cuda(), text_mask=g["text_mask"].cuda(), cond_scale=cond_scale,
                             schedule=sched)


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("B,side", [(3, 64), (2, 288)])            # 3 x 288^2 > 196 608: the three-kernel form
@pytest.mark.parametrize("cfg", [False, True])
def test_multistep_kernel_bitwise(native, B, side, cfg):
    from minimagen_b200.Imagen import quantile_rank
    from minimagen_b200.diffusion_model import GaussianDiffusion
    n = 3 * side * side
    gd = GaussianDiffusion(timesteps=1000).cuda()
    sch = gd.dpm_solver_schedule(10, "cuda")
    c3 = sch.c3.clone()
    sigma = gd.sigma.clone()                                       # nonzero: the noise term is exercised too
    gen = torch.Generator().manual_seed(B * side + cfg)
    rn = lambda: torch.randn(B, n, generator=gen).cuda()
    x, eps, noise, hist = rn() * 1.3, rn(), rn(), rn()
    eps0 = rn() if cfg else None
    grid = list(sch.grid)
    t = torch.tensor([grid[3], grid[0], grid[-1]][:B], device="cuda")            # c3 != 0, c3 == 0 (T-1), c3 == 0 (t = 0)
    hist[1:] = float("nan")                                        # NaN history where c3 == 0: ignored
    lo, hi, w = quantile_rank(n, 0.9)
    a, b_ = gd.sqrt_recip_alphas_cumprod, gd.sqrt_recipm1_alphas_cumprod
    x0 = torch.empty_like(x)
    s = torch.empty(B, device="cuda")
    native.step_x0(x, eps, eps0, 7.0, t, a, b_, B, n, x0)
    native.step_quantile(x0, B, n, lo, hi, w, 1.0, s)
    want, want_hist = multistep_ref(x0, s, x, noise, hist, t, sch.c1, sch.c2, sigma, c3, B, n)
    assert torch.isfinite(want).all()

    args = (eps, eps0, 7.0, t, a, b_, sch.c1, sch.c2, sigma, c3, noise)
    out, h = torch.empty_like(x), hist.clone()
    s2 = torch.empty(B, device="cuda")
    native.step_epilogue_multistep(x, *args, h, B, n, lo, hi, w, 1.0, out, s_out=s2)
    assert torch.equal(out, want) and torch.equal(h, want_hist) and torch.equal(s2, s)
    xin, h = x.clone(), hist.clone()
    native.step_epilogue_multistep(xin, *args, h, B, n, lo, hi, w, 1.0, xin)          # out aliases x_t
    assert torch.equal(xin, want) and torch.equal(h, want_hist)
    # captured: one replay = one step over the buffers' current contents
    xin, h = x.clone(), hist.clone()
    graph = _capture(lambda: native.step_epilogue_multistep(xin, *args, h, B, n, lo, hi, w, 1.0, xin))
    xin.copy_(x)
    h.copy_(hist)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(xin, want) and torch.equal(h, want_hist)
    # c3 = 0 everywhere: mi_step_epilogue's bits, whatever the history holds
    plain = torch.empty_like(x)
    native.step_epilogue(x, eps, eps0, 7.0, t, a, b_, sch.c1, sch.c2, sigma, noise, B, n, lo, hi, w, 1.0, plain)
    out, h = torch.empty_like(x), torch.full_like(hist, float("nan"))
    native.step_epilogue_multistep(x, eps, eps0, 7.0, t, a, b_, sch.c1, sch.c2, sigma, torch.zeros_like(c3), noise, h, B,
                                   n, lo, hi, w, 1.0, out)
    assert torch.equal(out, plain) and torch.equal(h, want_hist)


# ------------------------------------------------------------------------------------------------ the loop
def test_graph_vs_eager_analytic_bitwise(native):
    """With the analytic stand-in (no atomics) the captured multistep loop equals the eager one bit for bit."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000, "cuda")
    standin = AnalyticEps(1000).cuda()
    outs = []
    for graph in (False, True):
        im.noise_fn = _bank(4)
        outs.append(_loop(im, g, im.noise_schedulers[0].dpm_solver_schedule(12, "cuda"), graph, standin, 1.))
    assert torch.equal(outs[0], outs[1])
    assert len(im._graphs) == 1 and next(iter(im._graphs))[-1] == "multistep"


def test_graph_eager_and_restatement(native):
    g = load_golden("sample_loop.pt")
    outs = {}
    for graph in (False, True):
        im = _tiny_imagen(g, 1000, "cuda")
        im.noise_fn = _bank(7)
        outs[graph] = _loop(im, g, im.noise_schedulers[0].dpm_solver_schedule(8, "cuda"), graph)
        assert im.noise_fn.calls == [("init", -1)] + [("step", t) for t in P.dpm_grid(1000, 8)]
    ref = P.dpmpp_loop(g["state_dict"], g["cfg"], SHAPE, 1000, 8, _bank(7), text_embeds=g["text_embeds"],
                       text_mask=g["text_mask"])
    e_ge, e_ref = rel_l2(outs[True], outs[False]), rel_l2(outs[True], ref)
    print(f"2M S=8: graph vs eager {e_ge:.3e}; vs restated DPM-Solver++(2M) {e_ref:.3e}")
    assert e_ge <= 1e-6 and e_ref < 1e-3


def test_two_steps_equal_ddim(native):
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 25, "cuda")
    standin = AnalyticEps(25).cuda()
    gd = im.noise_schedulers[0]
    outs = []
    for sched in (gd.dpm_solver_schedule(2, "cuda"), gd.sampling_schedule(2, 0., "cuda")):
        im.noise_fn = _bank(5)
        outs.append(_loop(im, g, sched, True, standin, 1.))
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("S", [10, 20, 50])
def test_analytic_convergence_native(native, S):
    errs, _ = analytic_errors("cuda", S, graph=True)
    print(f"S={S} (native, graph): DDIM {errs['ddim']:.3e}, first order {errs['first']:.3e}, 2M {errs['2m']:.3e}")
    assert errs["2m"] * 10 <= errs["ddim"] and errs["2m"] * 5 <= errs["first"]


def test_ddim_2m_ddim_leaves_two_graphs(native):
    """DDIM -> 2M -> DDIM on one Imagen: a text-only and a multistep graph; each loop equals its eager run."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000, "cuda")
    ref = _tiny_imagen(g, 1000, "cuda")
    outs = []
    for kind in ("ddim", "2m", "ddim"):
        sched_of = (lambda gd: gd.sampling_schedule(8, 0., "cuda")) if kind == "ddim" else \
            (lambda gd: gd.dpm_solver_schedule(8, "cuda"))
        im.noise_fn, ref.noise_fn = _bank(11), _bank(11)
        out = _loop(im, g, sched_of(im.noise_schedulers[0]), True)
        want = _loop(ref, g, sched_of(ref.noise_schedulers[0]), False)
        err = rel_l2(out, want)
        print(f"{kind}: graph vs eager {err:.3e}")
        assert err <= 1e-6
        outs.append(out)
    assert len(im._graphs) == 2
    assert rel_l2(outs[2], outs[0]) <= 1e-6 and rel_l2(outs[1], outs[0]) > 1e-3


def test_tensor_core_sr_config_vs_restatement(native):
    """The sr_d64 configuration of test_gpu_unet.CFGS (tensor-core convs, lowres conditioning) at 64x64, b = 2, CFG w = 3,
    S = 5, against the restated 2M loop.  fp16 operand budget: 2e-3."""
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import BaseTest, Unet
    from test_gpu_unet import CFGS
    _, cfg, s, lowres, b = next(c for c in CFGS if c[0] == "sr_d64")
    torch.manual_seed(0)
    im = Imagen(unets=(Unet(**BaseTest.defaults), Unet(**cfg)), text_encoder_name="t5_small", image_sizes=(16, s),
                timesteps=1000, cond_drop_prob=0.1).eval()
    sd = {k: v.clone() for k, v in im.unets[1].state_dict().items()}
    im = im.cuda()
    gen = torch.Generator().manual_seed(3)
    te = torch.randn(b, 20, 512, generator=gen)
    tm = torch.ones(b, 20, dtype=torch.bool)
    tm[-1, 5:] = False
    lowres_img = torch.rand(b, 3, s, s, generator=gen)
    lnt = torch.full((b,), 200)
    shape = (b, 3, s, s)
    im.noise_fn = _bank(4, shape)
    out = im._p_sample_loop(im.unets[1], shape, noise_scheduler=im.noise_schedulers[1], text_embeds=te.cuda(),
                            text_mask=tm.cuda(), lowres_cond_img=lowres_img.cuda(), lowres_noise_times=lnt.cuda(),
                            cond_scale=3., schedule=im.noise_schedulers[1].dpm_solver_schedule(5, "cuda"))
    ref = P.dpmpp_loop(sd, cfg, shape, 1000, 5, im.noise_fn, text_embeds=te, text_mask=tm,
                       lowres_cond_img=lowres_img * 2 - 1, lowres_noise_times=lnt)
    err = rel_l2(out, ref)
    print(f"sr_d64 2M S=5: rel-L2 vs restated loop = {err:.3e}")
    assert err < 2e-3


def test_sample_sharding_invariance(native):
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet
    g = load_golden("sample_loop.pt")
    u = Unet(**g["cfg"]).eval()
    u.load_state_dict(g["state_dict"])
    im = Imagen(unets=u.cuda(), text_encoder_name="t5_small", image_sizes=(64,), timesteps=25, cond_drop_prob=0.15).cuda()
    im.unets[0].load_state_dict(g["state_dict"])
    gen = torch.Generator().manual_seed(0)
    bank = {}

    def noise_fn(kind, shape, step):
        if (kind, step) not in bank:
            bank[(kind, step)] = torch.randn(4, *shape[1:], generator=gen)
        return bank[(kind, step)][noise_fn.lo:noise_fn.lo + shape[0]]
    noise_fn.lo = 0
    im.noise_fn = noise_fn
    te = torch.randn(4, 9, 512, generator=gen).cuda()
    tm = torch.ones(4, 9, dtype=torch.bool).cuda()
    kw = dict(cond_scale=3., sampling_timesteps=6, sampler="dpmpp_2m")
    full = im.sample(text_embeds=te, text_masks=tm, **kw)
    assert full.shape == (4, 3, 64, 64) and torch.isfinite(full).all()
    parts = []
    for lo in (0, 2):
        noise_fn.lo = lo
        parts.append(im.sample(text_embeds=te[lo:lo + 2], text_masks=tm[lo:lo + 2], **kw))
    err = rel_l2(torch.cat(parts), full)
    print(f"2M sample b=4 vs two shards of 2: rel-L2 = {err:.3e}")
    assert err <= 1e-5


def test_cascade_vs_cpu_emulation(native):
    """The two-stage cascade of cascade_tiny.pt (16 -> 32, CFG w = 2, lowres augmentation), both stages on 2M, S = 6:
    GPU sample (captured graphs) vs the same call on the CPU emulation with the same draw bank."""
    import minimagen_b200.ops as ops_mod
    from test_host_logic import _cascade_from_golden
    g = load_golden("cascade_tiny.pt")
    gen = torch.Generator().manual_seed(6)
    bank = {}

    def noise_fn(kind, shape, step):
        key = (kind, step, tuple(shape))
        if key not in bank:
            bank[key] = torch.randn(shape, generator=gen)
        return bank[key]

    outs = {}
    for dev in ("cuda", "cpu"):
        prev = ops_mod._OPS
        if dev == "cpu":
            ops_mod.set_ops(EmuOps())
        try:
            im, _ = _cascade_from_golden(g, dev)
            im.noise_fn = noise_fn
            im.use_cuda_graph = True
            outs[dev] = im.sample(text_embeds=g["text_embeds"].to(dev), text_masks=g["text_mask"].to(dev),
                                  cond_scale=g["cond_scale"], lowres_sample_noise_level=g["lowres_noise_level"],
                                  sampling_timesteps=6, sampler="dpmpp_2m").cpu()
        finally:
            ops_mod.set_ops(prev)
    err = rel_l2(outs["cuda"], outs["cpu"])
    print(f"cascade 2M S=6: GPU vs CPU emulation rel-L2 = {err:.3e}")
    assert err < 1e-3
