"""DPM-Solver++(2M) sampling (Imagen.sample(sampling_timesteps=, sampler='dpmpp_2m')) on the CPU, through the torch
emulation of the ops interface extended by mi_step_epilogue_multistep.  Covers the log-SNR grid, the tables against the
paper-form restatement (dpmpp_restatement.py), the argument checks, the three graph flavours' keys, the emulated loop
against the restatement over the restated U-Net, and convergence on an analytic denoiser whose ODE end point is known in
closed form.  (The kernel, the captured graph and the cascade are covered on the GPU in test_gpu_dpmpp.py.)"""
import pytest
import torch
from torch import nn

import ddim_restatement as D
import dpmpp_restatement as P
from conftest import load_golden, rel_l2
from test_respaced import _bank, _tiny_imagen

F32 = torch.float32
SHAPE = (2, 3, 64, 64)


# ------------------------------------------------------------------------------------------------ analytic denoiser
MU, SD = 0.1, 0.15          # per-pixel Gaussian data N(MU, SD^2): |x0| < 1, so the dynamic threshold does nothing


class AnalyticEps(nn.Module):
    """Stand-in U-Net returning the exact E[eps | x_t] for per-pixel N(MU, SD^2) data on the linear schedule of
    `timesteps`, computed on the tensors' device without host syncs.  The parameter and the no-op static-text hooks let
    the captured-graph path take it like a U-Net."""

    def __init__(self, timesteps):
        super().__init__()
        self.anchor = nn.Parameter(torch.zeros(1))
        self.register_buffer("acp", D.alphas_cumprod_fp64(timesteps), persistent=False)

    def forward(self, x, t, **kw):
        a = self.acp[t].reshape(-1, 1, 1, 1)
        xd = x.double()
        x0 = MU + a.sqrt() * SD ** 2 / (a * SD ** 2 + 1. - a) * (xd - a.sqrt() * MU)
        return ((xd - a.sqrt() * x0) / (1. - a).sqrt()).to(F32)

    def register_static_text(self, te):
        pass

    def unregister_static_text(self, te):
        pass


def exact_end(x_T, timesteps):
    """Where the probability-flow ODE takes x_T (at t = T-1) by t = 0, denoised by the final x0 prediction: the ODE keeps
    z = (x_t - sqrt(a_t) MU) / sqrt(a_t SD^2 + 1 - a_t) fixed, and E[x0 | x_0] = MU + sqrt(a_0) SD^2 / sqrt(a_0 SD^2 + 1 - a_0) z."""
    acp = D.alphas_cumprod_fp64(timesteps)
    aT, a0 = acp[timesteps - 1], acp[0]
    z = (x_T.double() - aT.sqrt() * MU) / (aT * SD ** 2 + 1. - aT).sqrt()
    return MU + a0.sqrt() * SD ** 2 / (a0 * SD ** 2 + 1. - a0).sqrt() * z


def first_order_walk(gd, steps, device):
    """The 2M grid walked to first order: c3 = 0 and c1 = phi (DDIM's eta = 0 coefficient over the 2M grid), fp64 -> fp32."""
    s = gd.dpm_solver_schedule(steps, "cpu")
    acp = D.alphas_cumprod_fp64(gd.num_timesteps)
    walk = list(s.grid)
    c1 = torch.zeros(gd.num_timesteps, dtype=torch.float64)
    for t, t_next in zip(walk, walk[1:] + [-1]):
        a, a_next = acp[t], (acp[t_next] if t_next >= 0 else torch.tensor(1., dtype=torch.float64))
        c1[t] = a_next.sqrt() - (1. - a_next).sqrt() * a.sqrt() / (1. - a).sqrt()
    return s._replace(c1=c1.to(F32).to(device), c2=s.c2.to(device), sigma=s.sigma.to(device), next_t=s.next_t.to(device),
                      c3=torch.zeros_like(s.c3).to(device))


def analytic_errors(device, steps, graph):
    """rel-L2 of the final x0 against exact_end for DDIM eta = 0, the first-order log-SNR walk and 2M, at cond_scale 1."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000, device)
    im.use_cuda_graph = graph
    gd = im.noise_schedulers[0]
    standin = AnalyticEps(1000).to(device)
    te = g["text_embeds"].to(device)
    errs, outs = {}, {}
    for name, sched in (("ddim", gd.sampling_schedule(steps, 0., device)), ("first", first_order_walk(gd, steps, device)),
                        ("2m", gd.dpm_solver_schedule(steps, device))):
        im.noise_fn = _bank(21)
        out = im._p_sample_loop(standin, SHAPE, noise_scheduler=gd, text_embeds=te, cond_scale=1., schedule=sched)
        outs[name] = out
        errs[name] = rel_l2(out.double() * 2 - 1, exact_end(im.noise_fn.bank[("init", -1)], 1000))
    return errs, outs


# ------------------------------------------------------------------------------------------------ schedule
@pytest.mark.parametrize("T,steps", [(20, list(range(2, 21))), (25, list(range(2, 26))), (1000, [2, 3, 10, 20, 50, 200, 999, 1000])])
def test_grid_distinct_points_from_T_minus_1_to_0(T, steps):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    gd = GaussianDiffusion(timesteps=T)
    for S in steps:
        sch = gd.dpm_solver_schedule(S, "cpu")
        grid = list(sch.grid)
        assert len(grid) == S and len(set(grid)) == S
        assert grid[0] == T - 1 and grid[-1] == 0
        assert all(a > b for a, b in zip(grid, grid[1:]))
        assert grid == P.dpm_grid(T, S)
        assert [int(sch.next_t[t]) for t in grid] == grid[1:] + [0]
        assert sch.c1.shape == sch.c2.shape == sch.c3.shape == sch.sigma.shape == sch.next_t.shape == (T,)
        assert sch.c3.dtype == F32 and sch.next_t.dtype == torch.int64
        off = [t for t in range(T) if t not in grid]
        assert not sch.c1[off].any() and not sch.c2[off].any() and not sch.c3[off].any()


@pytest.mark.parametrize("T,S", [(20, 6), (25, 3), (25, 7), (1000, 10), (1000, 20), (1000, 50)])
def test_tables_match_the_restated_step(T, S):
    """c1 x0 + c2 x + c3 x0_prev with the fp32 tables == dpmpp_step in fp64, at every grid point."""
    from minimagen_b200.diffusion_model import GaussianDiffusion
    sch = GaussianDiffusion(timesteps=T).dpm_solver_schedule(S, "cpu")
    acp, lam = D.alphas_cumprod_fp64(T), P.lambdas(T)
    gen = torch.Generator().manual_seed(S)
    x0_prev = h_prev = None
    grid = list(sch.grid)
    for i, t in enumerate(grid):
        x, x0 = torch.randn(4096, generator=gen), torch.rand(4096, generator=gen, dtype=torch.float64) * 2 - 1
        want, h = P.dpmpp_step(acp, lam, x, t, grid[i + 1] if i + 1 < S else -1, x0, x0_prev, h_prev)
        got = sch.c1[t].double() * x0 + sch.c2[t].double() * x.double()
        if x0_prev is not None:
            got = got + sch.c3[t].double() * x0_prev
        assert rel_l2(got, want.double()) < 1e-6, (t, rel_l2(got, want.double()))
        x0_prev, h_prev = x0, h
    assert sch.c3[T - 1] == 0 and sch.c3[0] == 0                       # first order at T-1; x = x0 at t = 0
    assert sch.c1[0] == 1 and sch.c2[0] == 0
    assert not sch.sigma.any()


@pytest.mark.parametrize("T", [20, 25, 1000])
def test_two_steps_are_ddim_eta_0(T):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    gd = GaussianDiffusion(timesteps=T)
    sch, ddim = gd.dpm_solver_schedule(2, "cpu"), gd.sampling_schedule(2, 0., "cpu")
    assert sch.grid == ddim.grid == (T - 1, 0)
    for name in ("c1", "c2", "sigma", "next_t"):
        assert torch.equal(getattr(sch, name), getattr(ddim, name)), name
    assert not sch.c3.any() and ddim.c3 is None
    assert gd.dpm_solver_schedule(2, "cpu") is sch                     # cached per (steps, device)


# ------------------------------------------------------------------------------------------------ argument checks
def test_sampler_asserts(emu):
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet, BaseTest, SuperTest
    im = Imagen(unets=(Unet(**BaseTest.defaults), Unet(**SuperTest.defaults)), text_encoder_name="t5_small",
                image_sizes=(16, 32), timesteps=25, cond_drop_prob=0.1)
    te = torch.zeros(2, 4, 512)
    for bad in ("dpm", "DDIM", None, 2):
        with pytest.raises(AssertionError, match="sampler must be 'ddim' or 'dpmpp_2m', got"):
            im.sample(text_embeds=te, sampling_timesteps=5, sampler=bad)
    for steps in (None, (None, None)):
        with pytest.raises(AssertionError, match="sampler='dpmpp_2m' needs sampling_timesteps"):
            im.sample(text_embeds=te, sampling_timesteps=steps, sampler="dpmpp_2m")
    with pytest.raises(AssertionError, match="sampler='dpmpp_2m' is deterministic: ddim_eta must be 0, got 0.5"):
        im.sample(text_embeds=te, sampling_timesteps=5, ddim_eta=0.5, sampler="dpmpp_2m")
    img, mask = torch.rand(2, 3, 32, 32), torch.ones(2, 32, 32, dtype=torch.bool)
    with pytest.raises(AssertionError, match="sampler='dpmpp_2m' cannot be combined with inpainting"):
        im.sample(text_embeds=te, sampling_timesteps=5, sampler="dpmpp_2m", inpaint_images=img, inpaint_masks=mask)
    with pytest.raises(AssertionError, match="between 2 and 25"):
        im.noise_schedulers[0].dpm_solver_schedule(1, "cpu")
    # the loop itself refuses a multistep walk with inpainting
    sch = im.noise_schedulers[0]
    k, m = torch.zeros(2, 3, 16, 16), torch.ones(2, 16 * 16)
    with pytest.raises(AssertionError, match="a multistep schedule cannot be combined with inpainting"):
        im._p_sample_loop(im.unets[0], (2, 3, 16, 16), noise_scheduler=sch, text_embeds=te,
                          schedule=sch.dpm_solver_schedule(5, "cpu"), inpaint=(k, m, 2))


# ------------------------------------------------------------------------------------------------ graph keys
def test_graph_keys_of_the_three_flavours():
    """Text-only, inpainting and multistep keys differ; a 2M lookup takes the multistep graph and installs its walk, and a
    DDIM lookup after it hits the text-only graph.  Stand-ins take the place of captured graphs (no GPU needed)."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 25)
    sch = im.noise_schedulers[0]
    args = (im.unets[0], SHAPE, sch, g["text_embeds"], g["text_mask"], None, None, 3.)
    keys = {im._graph_key(*args), im._graph_key(*args, inpaint=True), im._graph_key(*args, multistep=True)}
    assert len(keys) == 3
    assert im._graph_key(*args, multistep=True) == im._graph_key(*args) + ("multistep",)

    class Cached:
        def __init__(self):
            self.walks = []

        def set_cond(self, **cond):
            pass

        def set_schedule(self, sched):
            self.walks.append(sched)

    text, multi = Cached(), Cached()
    im._graphs = {im._graph_key(*args): text, im._graph_key(*args, multistep=True): multi}
    kw = dict(noise_scheduler=sch, text_embeds=g["text_embeds"], text_mask=g["text_mask"], lowres_cond_img=None,
              lowres_noise_times=None, cond_scale=3.)
    dpm, ddim = sch.dpm_solver_schedule(8, "cpu"), sch.sampling_schedule(8, 0., "cpu")
    assert im._step_graph(im.unets[0], SHAPE, schedule=dpm, **kw) is multi
    assert im._step_graph(im.unets[0], SHAPE, schedule=ddim, **kw) is text
    assert im._step_graph(im.unets[0], SHAPE, schedule=sch.dpm_solver_schedule(5, "cpu"), **kw) is multi
    assert [w.grid for w in multi.walks] == [dpm.grid, tuple(P.dpm_grid(25, 5))] and text.walks == [ddim]
    assert len(im._graphs) == 2


# ------------------------------------------------------------------------------------------------ emulated sampler
def test_emulated_loop_vs_restatement(emu):
    """S = 8 over T = 1000 with CFG w = 3 on sample_loop.pt's tiny U-Net: the product's tables through the multistep
    contract vs the paper-form restatement over the restated U-Net; one 'step' draw per grid point, like DDIM."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    im.noise_fn = _bank(7)
    sched = im.noise_schedulers[0].dpm_solver_schedule(8, "cpu")
    out = im._p_sample_loop(im.unets[0], SHAPE, noise_scheduler=im.noise_schedulers[0], text_embeds=g["text_embeds"],
                            text_mask=g["text_mask"], cond_scale=3., schedule=sched)
    assert im.noise_fn.calls == [("init", -1)] + [("step", t) for t in P.dpm_grid(1000, 8)]
    assert emu.calls.count("step_epilogue_multistep") == 8 and "step_epilogue" not in emu.calls
    ref = P.dpmpp_loop(g["state_dict"], g["cfg"], SHAPE, 1000, 8, _bank(7), text_embeds=g["text_embeds"].cpu(),
                       text_mask=g["text_mask"].cpu())
    err = rel_l2(out, ref)
    print(f"2M S=8: rel-L2 vs restated DPM-Solver++(2M) = {err:.3e}")
    assert err < 1e-3
    ddim = im._p_sample_loop(im.unets[0], SHAPE, noise_scheduler=im.noise_schedulers[0], text_embeds=g["text_embeds"],
                             text_mask=g["text_mask"], cond_scale=3., schedule=im.noise_schedulers[0].sampling_schedule(8, 0., "cpu"))
    assert rel_l2(ddim, out) > 1e-3                                   # a different sampler, not DDIM again


def test_two_steps_equal_ddim_loop(emu):
    g = load_golden("sample_loop.pt")
    outs = []
    for sched_of in (lambda gd: gd.dpm_solver_schedule(2, "cpu"), lambda gd: gd.sampling_schedule(2, 0., "cpu")):
        im = _tiny_imagen(g, 25)
        im.noise_fn = _bank(3)
        outs.append(im._p_sample_loop(im.unets[0], SHAPE, noise_scheduler=im.noise_schedulers[0],
                                      text_embeds=g["text_embeds"], text_mask=g["text_mask"], cond_scale=3.,
                                      schedule=sched_of(im.noise_schedulers[0])))
    assert torch.equal(outs[0], outs[1])


def test_cascade_sample_per_stage(emu):
    """sampler='dpmpp_2m' applies to the stages with a sampling_timesteps entry; a None entry keeps the DDPM loop.  Each
    stage makes one U-Net evaluation pair per grid point (CFG w = 2, unbatched)."""
    from test_host_logic import _cascade_from_golden
    g = load_golden("cascade_tiny.pt")
    im, _ = _cascade_from_golden(g, "cpu")
    steps = []
    im.noise_fn = lambda kind, shape, step: steps.append((kind, step)) or torch.randn(shape)
    calls = []
    for u in im.unets:
        fwd = u.forward
        u.forward = (lambda f: lambda *a, **kw: calls.append(1) or f(*a, **kw))(fwd)
    out = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=2., sampling_timesteps=(None, 5),
                    sampler="dpmpp_2m")
    assert out.shape == (2, 3, 32, 32) and torch.isfinite(out).all()
    assert [s[1] for s in steps if s[0] == "step"] == list(range(24, -1, -1)) + P.dpm_grid(25, 5)
    assert len(calls) == 2 * (25 + 5)
    assert emu.calls.count("step_epilogue") == 25 and emu.calls.count("step_epilogue_multistep") == 5


# ------------------------------------------------------------------------------------------------ analytic convergence
@pytest.mark.parametrize("S", [10, 20, 50])
def test_analytic_convergence(emu, S):
    """On the analytic denoiser (cond_scale 1), 2M's final x0 is at least 10x closer to the exact ODE end point than DDIM
    eta = 0's and 5x closer than the first-order walk over the same log-SNR grid (fp64 ratios: 46 / 23 / 69 and
    18 / 8 / 21 at S = 10 / 20 / 50)."""
    errs, _ = analytic_errors("cpu", S, graph=False)
    print(f"S={S}: rel-L2 vs exact end point: DDIM {errs['ddim']:.3e}, first order {errs['first']:.3e}, "
          f"2M {errs['2m']:.3e}")
    assert errs["2m"] * 10 <= errs["ddim"]
    assert errs["2m"] * 5 <= errs["first"]
