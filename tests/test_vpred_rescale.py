"""v-prediction, zero-terminal-SNR schedules and guidance rescale (Imagen.set_objectives(pred_objectives=,
zero_terminal_snr=), Imagen.sample(guidance_rescale=)) on the CPU, through the torch emulation of the ops interface
with mi_guidance_rescale_factor and mi_step_epilogue_rescaled (tests/emu_ops.py).  Covers the schedule against Lin et al.'s Algorithm 1 and the
finiteness of every walk's tables at alphas_cumprod = 0; an exact v-denoiser under 'v' against the exact eps-denoiser
under 'noise'; the v training target; the argument checks; the rescaled loop against the float64 restatement
(rescale_restatement.py) on DDPM, DDIM, DPM-Solver++(2M), a guidance table, per-image phi and a negative prompt, and
phi = 0 as the loop without it; and the per-call checkers of the two new entry points against planted defects.
(The kernels and the captured graphs are covered on the GPU in test_gpu_vpred_rescale.py.)"""
import math

import pytest
import torch
import torch.nn.functional as F
from torch import nn

import fp64_ref as R
import rescale_restatement as RS
from conftest import load_golden, rel_l2
from checking_ops import CheckingOps
from emu_ops import EmuOps

F32, F64 = torch.float32, torch.float64
SHAPE = (2, 3, 64, 64)
INF = float("inf")


def _imagen(T=1000, objective='noise', zero_snr=False, device="cpu"):
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet
    g = load_golden("sample_loop.pt")
    u = Unet(**g["cfg"]).eval()
    u.load_state_dict(g["state_dict"])
    im = Imagen(unets=u, text_encoder_name="t5_small", image_sizes=(64,), timesteps=T,
                cond_drop_prob=0.15).eval().to(device).set_objectives(objective, zero_snr)
    im.unets[0].load_state_dict(g["state_dict"])
    im.use_cuda_graph = False
    return im


# ------------------------------------------------------------------------------------------------ stand-in U-Net
MU, SD = 0.1, 0.15            # the data of the conditional pass: per-pixel N(MU + shift_b, SD^2), shift_b from the text
MU_N, SD_N = -0.05, 0.3       # the data of the null pass


class TwoPass(nn.Module):
    """A stand-in U-Net that outputs, under `objective`, the exact denoiser of per-pixel Gaussian data: N(MU + shift_b,
    SD^2) for a conditional pass (shift_b = 0.2 text_embeds[b, 0, 0], so a negative prompt differs from the prompt) and
    N(MU_N, SD_N^2) for the null pass (cond_drop_prob = 1).  `double(x, t, null, te)` is the same in float64."""

    def __init__(self, acp, objective):
        super().__init__()
        self.anchor = nn.Parameter(torch.zeros(1))
        self.objective = objective
        self.register_buffer("acp", acp.to(F64), persistent=False)

    def double(self, x, t, null, te=None):
        a = self.acp[t].reshape(-1, 1, 1, 1)
        mu, sd = (MU_N, SD_N) if null else (MU, SD)
        if not null and te is not None:
            mu = mu + 0.2 * te[:, 0, 0].to(F64).reshape(-1, 1, 1, 1)
        xd = x.to(F64)
        x0 = mu + a.sqrt() * sd ** 2 / (a * sd ** 2 + 1. - a) * (xd - a.sqrt() * mu)
        eps = (xd - a.sqrt() * x0) / (1. - a).sqrt()
        return eps if self.objective == 'noise' else RS.v_target(x0, eps, a)

    def forward(self, x, t, cond_drop_prob=0., text_embeds=None, **kw):
        return self.double(x, t, cond_drop_prob == 1., text_embeds).to(F32)

    def register_static_text(self, te):
        pass

    def unregister_static_text(self, te):
        pass


def _bank(seed, shape=SHAPE):
    gen = torch.Generator().manual_seed(seed)
    bank = {}

    def noise_fn(kind, shp, step):
        if (kind, step) not in bank:
            bank[(kind, step)] = torch.randn(tuple(shp), generator=gen)
        return bank[(kind, step)]
    noise_fn.bank = bank
    return noise_fn


def _walk(gd, sampler, steps):
    if sampler == "ddpm":
        return gd.ddpm_schedule("cpu")
    if sampler == "dpmpp_2m":
        return gd.dpm_solver_schedule(steps, "cpu")
    return gd.sampling_schedule(steps, 0., "cpu")


# ------------------------------------------------------------------------------------------------ schedule
@pytest.mark.parametrize("T", [20, 25, 1000])
def test_zero_snr_schedule_is_algorithm_1(T):
    from minimagen_b200.diffusion_model import GaussianDiffusion, ZeroTerminalSNRDiffusion, _betas_fp64
    base, z = GaussianDiffusion(timesteps=T), ZeroTerminalSNRDiffusion(timesteps=T)
    assert torch.equal(base.alphas_cumprod_fp64, torch.cumprod(1. - _betas_fp64(T), dim=0))     # default untouched
    acp = z.alphas_cumprod_fp64
    assert acp[T - 1] == 0 and z.alphas_cumprod[T - 1] == 0 and z.betas[T - 1] == 1
    assert acp[0] == base.alphas_cumprod_fp64[0] and z.alphas_cumprod[0] == base.alphas_cumprod[0]
    assert bool((acp[1:] < acp[:-1]).all())
    ref = RS.zero_snr_acp(T)
    assert float((acp - ref).abs().max()) <= 1e-15
    # the eps-only tables are inf at SNR 0; every other buffer is finite
    assert math.isinf(z.sqrt_recip_alphas_cumprod[T - 1]) and math.isinf(z.sqrt_recipm1_alphas_cumprod[T - 1])
    for name, buf in z.named_buffers():
        if name not in ("sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod"):
            assert bool(torch.isfinite(buf).all()), name
    assert z.sqrt_alphas_cumprod[T - 1] == 0 and z.sqrt_one_minus_alphas_cumprod[T - 1] == 1


@pytest.mark.parametrize("T", [20, 25, 1000])
def test_zero_snr_walk_tables_are_finite(T):
    from minimagen_b200.diffusion_model import ZeroTerminalSNRDiffusion
    gd = ZeroTerminalSNRDiffusion(timesteps=T)
    walks = [gd.ddpm_schedule("cpu")]
    for S in sorted({2, 3, 10, T // 2, T}):
        walks += [gd.sampling_schedule(S, 0., "cpu"), gd.sampling_schedule(S, 1., "cpu"), gd.dpm_solver_schedule(S, "cpu")]
    for walk in walks:
        for tab in (walk.c1, walk.c2, walk.sigma) + ((walk.c3,) if walk.c3 is not None else ()):
            assert bool(torch.isfinite(tab).all()), walk.grid
        _, ra, rb = gd.inpaint_tables(None if walk is walks[0] else walk, "cpu")
        assert bool(torch.isfinite(ra).all() and torch.isfinite(rb).all())
        assert ra[T - 1] == 0 and rb[T - 1] == 1                  # back to t = T-1 is pure noise
    for interval in (None, (0.3, 5.), (0., INF), (2., INF)):
        for schedule in (None, "linear", "cosine"):
            assert bool(torch.isfinite(gd.guidance_table(interval, schedule, "cpu")).all())


# ------------------------------------------------------------------------------------------------ objective, analytic
LOOPS = [("ddpm", 25, None), ("ddim", 1000, 10), ("dpmpp_2m", 1000, 10)]


def _analytic_loop(im, sampler, steps, seed=21):
    gd = im.noise_schedulers[0]
    standin = TwoPass(gd.alphas_cumprod_fp64, im.pred_objectives[0])
    im.noise_fn = _bank(seed)
    out = im._p_sample_loop(standin, SHAPE, noise_scheduler=gd, text_embeds=torch.zeros(2, 4, 8), cond_scale=1.,
                            schedule=_walk(gd, sampler, steps))
    return out, im.noise_fn.bank[("init", -1)]


@pytest.mark.parametrize("sampler,T,steps", LOOPS, ids=[c[0] for c in LOOPS])
def test_v_denoiser_tracks_eps_denoiser(emu, sampler, T, steps):
    """The same exact denoiser, output as v under 'v' and as eps under 'noise': the two loops differ only by the fp32
    rounding of the two x0 formulas."""
    eps_out, _ = _analytic_loop(_imagen(T, 'noise'), sampler, steps)
    v_out, _ = _analytic_loop(_imagen(T, 'v'), sampler, steps)
    err = rel_l2(v_out, eps_out)
    print(f"\n{sampler}: rel-L2(v loop, eps loop) = {err:.3g}")
    assert err < 1e-5


def _exact_end(x_T, acp):
    aT, a0 = acp[-1], acp[0]
    z = (x_T.to(F64) - aT.sqrt() * MU) / (aT * SD ** 2 + 1. - aT).sqrt()
    return MU + a0.sqrt() * SD ** 2 / (a0 * SD ** 2 + 1. - a0).sqrt() * z


@pytest.mark.parametrize("sampler", ["ddim", "dpmpp_2m"])
def test_zero_snr_v_loop_converges_to_the_ode_end_point(emu, sampler):
    """Under zero terminal SNR the 'v' loop starts at SNR 0 (x0 = -v there) and stays finite; its distance to the exact
    ODE end point shrinks with the step count like the linear schedule's.  It is not smaller than the linear schedule's
    at equal steps on this problem (measured, 10 / 50 steps: DDIM 0.484 / 0.128 against 0.483 / 0.127, 2M 0.039 / 0.0040
    against 0.011 / 0.0019): the last interval of the walk, from SNR 0, is the hardest to integrate."""
    errs = {}
    for zero in (False, True):
        im = _imagen(1000, 'v', zero)
        for steps in (10, 50):
            out, x_T = _analytic_loop(im, sampler, steps)
            assert bool(torch.isfinite(out).all())
            errs[zero, steps] = rel_l2(out.to(F64) * 2 - 1, _exact_end(x_T, im.noise_schedulers[0].alphas_cumprod_fp64))
    print(f"\n{sampler}: rel-L2 to the exact ODE end point {errs}")
    assert errs[True, 50] * (2.5 if sampler == "dpmpp_2m" else 3.5) <= errs[True, 10]
    assert errs[True, 50] <= 2.5 * errs[False, 50]


# ------------------------------------------------------------------------------------------------ objective, training
def _f32_sum_of_products(a, x, b, y):
    """fp32(fp32(a x) + fp32(b y)) restated in float64: the products of fp32 values are exact in float64, and rounding a
    float64 sum to fp32 is the fp32 sum (float64 has more than 2 * 24 + 2 bits)."""
    p = (a.to(F64) * x.to(F64)).to(F32).to(F64)
    q = (b.to(F64) * y.to(F64)).to(F32).to(F64)
    return (p + q).to(F32)


@pytest.mark.parametrize("zero_snr", [False, True])
def test_v_training_loss_is_the_restatement(emu, zero_snr):
    im = _imagen(1000, 'v', zero_snr)
    gd = im.noise_schedulers[0]
    standin = TwoPass(gd.alphas_cumprod_fp64, 'v')
    gen = torch.Generator().manual_seed(3)
    images = torch.rand(SHAPE, generator=gen)
    noise = torch.randn(SHAPE, generator=gen)
    times = torch.tensor([999, 417])
    te = torch.randn(2, 4, 8, generator=gen)
    loss = im._p_losses(standin, images, times, noise_scheduler=gd, text_embeds=te, noise=noise)
    x0 = images * 2 - 1
    col = lambda tab: tab[times].reshape(-1, 1, 1, 1).expand(SHAPE)
    x_t = _f32_sum_of_products(col(gd.sqrt_alphas_cumprod), x0, col(gd.sqrt_one_minus_alphas_cumprod), noise)
    target = _f32_sum_of_products(col(gd.sqrt_alphas_cumprod), noise, -col(gd.sqrt_one_minus_alphas_cumprod), x0)
    assert torch.equal(loss, F.mse_loss(standin(x_t, times, text_embeds=te), target))
    if zero_snr:
        assert torch.equal(target[0], -x0[0])                     # t = T-1: the target is -x0 exactly
    # and in float64, the definition sqrt(a) noise - sqrt(1 - a) x0
    a = gd.alphas_cumprod_fp64[times].reshape(-1, 1, 1, 1)
    assert float((target.to(F64) - RS.v_target(x0.to(F64), noise.to(F64), a)).abs().max()) < 1e-6


# ------------------------------------------------------------------------------------------------ validation
def test_constructor_checks():
    with pytest.raises(AssertionError, match="noise prediction is undefined at SNR 0"):
        _imagen(1000, 'noise', True)
    with pytest.raises(AssertionError, match="pred_objectives of unet 1 must be 'noise' or 'v'"):
        _imagen(1000, 'x_start')
    with pytest.raises(AssertionError, match="pred_objectives must have one entry per unet"):
        _imagen(1000, ('v', 'v'))
    with pytest.raises(AssertionError, match="zero_terminal_snr must have one entry per unet"):
        _imagen(1000, 'v', (True, True))
    im = _imagen(1000, ('v',), (True,))
    assert im.pred_objectives == ('v',) and im.noise_schedulers[0].zero_terminal_snr
    assert im.lowres_noise_schedule.alphas_cumprod[-1] > 0          # the augmentation schedule keeps its own


@pytest.mark.parametrize("phi,match", [(-0.1, "in \\[0, 1\\]"), (1.5, "in \\[0, 1\\]"), (float("nan"), "in \\[0, 1\\]"),
                                       (INF, "in \\[0, 1\\]"), (True, "in \\[0, 1\\]"), ((0.5, 0.5), "one entry per unet"),
                                       (torch.tensor([0.5, 1.5]), "must be in \\[0, 1\\]"),
                                       (torch.tensor([0.5]), "b = 2 per-image values")])
def test_guidance_rescale_checks(emu, phi, match):
    im = _imagen(25)
    with pytest.raises(AssertionError, match=match):
        im.sample(text_embeds=torch.zeros(2, 4, 512), cond_scale=3., guidance_rescale=phi)


# ------------------------------------------------------------------------------------------------ rescaled loop
FLAVOURS = [("ddpm", 25, None, None), ("ddim", 1000, 8, None), ("dpmpp_2m", 1000, 6, None),
            ("ddim", 1000, 8, ((0.4, 20.), "linear")), ("dpmpp_2m", 1000, 6, (None, "cosine"))]


@pytest.mark.parametrize("objective,zero_snr", [("noise", False), ("v", True)])
@pytest.mark.parametrize("sampler,T,steps,table", FLAVOURS,
                         ids=[f"{c[0]}{'-table' if c[3] else ''}" for c in FLAVOURS])
@pytest.mark.parametrize("negative", [False, True])
def test_rescaled_loop_vs_restatement(emu, sampler, T, steps, table, objective, zero_snr, negative):
    """Per-image w (2, 6) and phi (0.7, 1) against the float64 loop; the factor and rescaled step run once per guided
    point and the existing epilogues never."""
    im = _imagen(T, objective, zero_snr)
    gd = im.noise_schedulers[0]
    standin = TwoPass(gd.alphas_cumprod_fp64, objective)
    walk = _walk(gd, sampler, steps)
    gtab = None if table is None else gd.guidance_table(table[0], table[1], "cpu")
    te = torch.randn(2, 4, 8, generator=torch.Generator().manual_seed(5))
    nte = -te if negative else None
    w, phi = torch.tensor([2., 6.]), torch.tensor([0.7, 1.])
    im.noise_fn = _bank(11)
    emu.calls.clear()
    out = im._p_sample_loop(standin, SHAPE, noise_scheduler=gd, text_embeds=te, cond_scale=w, schedule=walk,
                            guidance_table=gtab, negative_text_embeds=nte, guidance_rescale=phi)
    x_T = im.noise_fn.bank[("init", -1)]
    guided_at = None if gtab is None else (lambda t: float(gtab[t]) != 0.)
    # the stand-in's fp32 outputs, as the loop reads them: near SNR 0 the predictions are nearly constant images, and
    # their sums of squares (so f) are set by the fp32 rounding of the outputs
    model = lambda x, t, null: (standin.double(x, t, False, nte) if (null and negative) else
                                standin.double(x, t, null, te)).to(F32).to(F64)
    ref = RS.loop(model, x_T, walk, gd.alphas_cumprod_fp64, objective, w, phi,
                  lambda t: im.noise_fn.bank[("step", t)], guided_at=guided_at, gtab=gtab, c3=sampler == "dpmpp_2m")
    err = rel_l2(out, ref)
    n_guided = sum(1 for t in walk.grid if guided_at is None or guided_at(t))
    print(f"\nrel-L2 vs restatement {err:.3g}, {n_guided} guided points of {len(walk.grid)}")
    assert err < 1e-6
    assert emu.calls.count("guidance_rescale_factor") == emu.calls.count("step_epilogue_rescaled") == n_guided
    plain = [c for c in emu.calls if c.startswith("step_epilogue") and c != "step_epilogue_rescaled"]
    assert len(plain) == len(walk.grid) - n_guided


@pytest.mark.parametrize("sampler", ["ddpm", "ddim", "dpmpp_2m"])
@pytest.mark.parametrize("phi", [0., torch.zeros(2)])
def test_phi_zero_is_the_loop_without_it(emu, sampler, phi):
    im = _imagen(25 if sampler == "ddpm" else 1000, 'v', True)
    gd = im.noise_schedulers[0]
    standin = TwoPass(gd.alphas_cumprod_fp64, 'v')
    te = torch.randn(2, 4, 8, generator=torch.Generator().manual_seed(5))
    outs = []
    for kw in ({}, dict(guidance_rescale=phi)):
        im.noise_fn = _bank(13)
        emu.calls.clear()
        outs.append(im._p_sample_loop(standin, SHAPE, noise_scheduler=gd, text_embeds=te, cond_scale=4.,
                                      schedule=_walk(gd, sampler, 6), **kw))
        assert "guidance_rescale_factor" not in emu.calls and "step_epilogue_rescaled" not in emu.calls
    assert torch.equal(outs[0], outs[1])


def test_unguided_stage_never_rescales(emu):
    im = _imagen(25, 'v', True)
    gd = im.noise_schedulers[0]
    im.noise_fn = _bank(2)
    im._p_sample_loop(TwoPass(gd.alphas_cumprod_fp64, 'v'), SHAPE, noise_scheduler=gd,
                      text_embeds=torch.zeros(2, 4, 8), cond_scale=1., guidance_rescale=0.7)
    assert "guidance_rescale_factor" not in emu.calls and "step_epilogue_rescaled" not in emu.calls


def test_rescaled_graph_key():
    im = _imagen(25)
    gd = im.noise_schedulers[0]
    args = (im.unets[0], SHAPE, gd, torch.zeros(2, 4, 8), None, None, None, 3.)
    base = im._graph_key(*args)
    assert im._graph_key(*args, rescaled=True) == base + ('rescaled',)
    assert im._graph_key(*args, True, rescaled=True)[-2:] == ('rescaled', 'inpaint')


# ------------------------------------------------------------------------------------------------ planted defects
SMS = 132
B, N = 3, 3 * 64 * 64


def _call_data(seed=0, table=False):
    gen = torch.Generator().manual_seed(seed)
    c = torch.randn(B, N, generator=gen) * torch.tensor([[1.], [0.5], [2.]]) + 0.3
    u = torch.randn(B, N, generator=gen) * 0.8
    w = torch.tensor([3., 7.5, 1.5])
    t = torch.tensor([999, 500, 0])
    w_sched = torch.linspace(0.2, 1.7, 1000).to(F32) if table else None
    phi = torch.tensor([0.7, 1., 0.3])
    return c, u, w, w_sched, t, phi


def _factor(defect):
    def run(eps_cond, eps_null, cond_scale, w_sched, t, phi, Bn, n, f):
        c, u = eps_cond.reshape(Bn, n).double(), eps_null.reshape(Bn, n)
        wt = cond_scale if defect == "unscheduled" else (
            cond_scale if w_sched is None else torch.where(w_sched[t] == 1, cond_scale, 1 + (cond_scale - 1) * w_sched[t]))
        g = (u + (eps_cond.reshape(Bn, n) - u) * wt[:, None]).double()
        ssc = ((c - c.mean(1, keepdim=True)) ** 2).sum(1)
        ssg = ((g - g.mean(1, keepdim=True)) ** 2).sum(1)
        if defect == "biased":
            ssc = ssc * n / (n - 1)                                 # the unbiased std in one of the two terms only
        ph = phi.double()
        fv = ph * (ssc / ssg).sqrt() + (1 - ph)
        if defect == "neighbour":
            fv = fv.roll(1)
        f.copy_(fv.to(F32))
    return run


@pytest.mark.parametrize("table", [False, True])
def test_factor_passes_and_planted_defects_fail_its_check(table):
    c, u, w, w_sched, t, phi = _call_data(1, table)
    proxy = CheckingOps(EmuOps(), sms=SMS)
    f = torch.empty(B)
    proxy.guidance_rescale_factor(c, u, w, w_sched, t, phi, B, N, f)
    assert "guidance_rescale_factor" in proxy.checked and bool((f != 1).all())
    defects = ["biased", "neighbour"] + (["unscheduled"] if table else [])
    for defect in defects:
        proxy = CheckingOps(type("P", (), {"guidance_rescale_factor": staticmethod(_factor(defect))})(), sms=SMS,
                            strict=False)
        proxy.guidance_rescale_factor(c, u, w, w_sched, t, phi, B, N, torch.empty(B))
        assert proxy.failures and proxy.failures[0].startswith("guidance_rescale_factor("), defect


def _tables():
    from minimagen_b200.diffusion_model import ZeroTerminalSNRDiffusion
    gd = ZeroTerminalSNRDiffusion(timesteps=1000)
    s = gd.dpm_solver_schedule(10, "cpu")
    s = s._replace(c3=s.c3.clone())
    s.c3[999] = 0.
    s.c3[500] = -0.3
    return gd, s


@pytest.mark.parametrize("multi", [False, True])
@pytest.mark.parametrize("defect", [None, "neighbour", "unscaled"])
def test_rescaled_epilogue_check(multi, defect):
    from minimagen_b200.Imagen import quantile_rank
    gd, s = _tables()
    c, u, w, w_sched, t, phi = _call_data(2, True)
    x = torch.randn(B, N, generator=torch.Generator().manual_seed(4))
    z = torch.randn(B, N, generator=torch.Generator().manual_seed(5))
    hist = torch.randn(B, N, generator=torch.Generator().manual_seed(6)) * 0.1 if multi else None
    f = torch.tensor([0.8, 1.25, 0.6])
    lo, hi, wt = quantile_rank(N, 0.9)
    emu = EmuOps()

    def planted(x_t, eps_cond, eps_null, cond_scale, w_sched, f, *rest, **kw):
        if defect == "neighbour":
            f = f.roll(1)
        elif defect == "unscaled":
            f = torch.ones_like(f)
        emu.step_epilogue_rescaled(x_t, eps_cond, eps_null, cond_scale, w_sched, f, *rest, **kw)

    proxy = CheckingOps(type("P", (), {"step_epilogue_rescaled": staticmethod(planted)})(), sms=SMS, strict=False)
    proxy.step_epilogue_rescaled(x, c, u, w, w_sched, f, t, gd.sqrt_alphas_cumprod, gd.sqrt_one_minus_alphas_cumprod,
                                 s.c1, s.c2, s.sigma, s.c3 if multi else None, z, hist, B, N, lo, hi, wt, 1.0,
                                 torch.empty_like(x), s_out=torch.empty(B))
    if defect is None:
        assert not proxy.failures and proxy.checked == {"step_epilogue_rescaled"}
    else:
        assert proxy.failures and proxy.failures[0].startswith("step_epilogue_rescaled(")


def test_rescaled_epilogue_is_the_plain_epilogue_of_the_rescaled_prediction():
    from minimagen_b200.Imagen import quantile_rank
    gd, s = _tables()
    c, u, w, w_sched, t, phi = _call_data(7, True)
    x = torch.randn(B, N, generator=torch.Generator().manual_seed(8))
    z = torch.randn(B, N, generator=torch.Generator().manual_seed(9))
    emu, lo_hi = EmuOps(), quantile_rank(N, 0.9)
    f = torch.empty(B)
    emu.guidance_rescale_factor(c, u, w, w_sched, t, phi, B, N, f)
    a, b = gd.sqrt_alphas_cumprod, gd.sqrt_one_minus_alphas_cumprod
    out1, out2 = torch.empty_like(x), torch.empty_like(x)
    emu.step_epilogue_rescaled(x, c, u, w, w_sched, f, t, a, b, s.c1, s.c2, s.sigma, None, z, None, B, N, *lo_hi, 1.0, out1)
    eps = R.guided_fp32(c, u, w, w_sched, t, B, N) * f[:, None]
    emu.step_epilogue(x, eps, None, 1.0, t, a, b, s.c1, s.c2, s.sigma, z, B, N, *lo_hi, 1.0, out2)
    assert torch.equal(out1, out2)
