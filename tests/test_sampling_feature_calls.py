"""The sampling features under one CheckingOps (tests/checking_ops.py), on a machine without a GPU:

  * completeness over the interface: every public method of minimagen_b200.ops.NativeOps has a `_check_` method in
    CheckingOps or is in ALLOWED (no kernel: capability queries and the launch-mode setting), and an emulation in
    tests/emu_ops.py with the same parameters, so a kernel added to the interface later fails here until it gets both;
  * the emulated combined samples of test_gpu_sampling_feature_calls.py on the tiny golden U-Nets, every call checked:
    a non-square two-stage DDIM cascade (RePaint at R = 2 with mask values of exactly 0.5, per-image seeds, weights and
    guidance tables, a negative prompt, then a v-prediction zero-SNR stage with a guidance interval, a cosine schedule,
    per-image rescale and img2img), the same on DPM-Solver++(2M) without inpainting, and DDPM inpainting at R = 3;
  * the device-side RePaint walk (mi_inpaint_advance and the keyed draws labelled t * R + r read on the device, which
    only the captured step runs) over a whole plan;
  * planted defects: each fails its own method's check only.
"""
import inspect

import numpy as np
import pytest
import torch

import keyed_noise_restatement as K
from checking_ops import ALLOWED, CheckingOps
from conftest import load_golden
from emu_ops import EmuOps
from test_host_logic import _cascade_from_golden
from test_respaced import _tiny_imagen

SMS = 132
F32, I64 = torch.float32, torch.int64


# ------------------------------------------------------------------------------------------------ completeness
def _public_methods():
    from minimagen_b200.ops import NativeOps
    return {n: f for n, f in inspect.getmembers(NativeOps, inspect.isfunction) if not n.startswith("_")}


def test_every_ops_method_has_a_checker():
    """Every public method of NativeOps: a checker, or in ALLOWED.  ALLOWED methods launch no kernel (their source makes no
    library call but queries), and every other method makes one."""
    methods = _public_methods()
    missing = sorted(n for n in methods if n not in ALLOWED and not hasattr(CheckingOps, "_check_" + n))
    assert not missing, f"NativeOps methods without a float64 checker in CheckingOps: {missing}"
    assert ALLOWED <= set(methods), f"ALLOWED names methods NativeOps does not have: {sorted(ALLOWED - set(methods))}"
    for n in ALLOWED:
        assert "call(" not in inspect.getsource(methods[n]), f"{n} is in ALLOWED but launches a kernel"
    for n in set(methods) - ALLOWED:
        src = inspect.getsource(methods[n])
        assert "call(" in src or "self._scheduled(" in src, f"{n} has a checker but launches nothing"


def test_emulation_covers_every_ops_method():
    """Every public method of NativeOps exists on EmuOps with the same parameters (names, order, kinds, defaults), so the
    CPU tests can run any host code path on the emulation."""
    params = lambda f: list(inspect.signature(f).parameters.values())
    methods = _public_methods()
    missing = sorted(n for n in methods if not hasattr(EmuOps, n))
    assert not missing, f"NativeOps methods EmuOps does not emulate: {missing}"
    differ = sorted(n for n, f in methods.items() if params(f) != params(getattr(EmuOps, n)))
    assert not differ, f"EmuOps methods whose parameters differ from NativeOps's: {differ}"


# ------------------------------------------------------------------------------------------------ combined samples
def _negative(b, D, L=5, seed=11):
    gen = torch.Generator().manual_seed(seed)
    nte = torch.randn(b, L, D, generator=gen)
    ntm = torch.ones(b, L, dtype=torch.bool)
    ntm[0, 3:] = False
    return nte, ntm


def half_mask(b, h, w):
    """A bool mask at (h, w) whose 2x downsample (the base stage of a cascade sampled at (h / 2, w / 2)) has pixels of
    exactly 0.5: the left 5 / 12 known, and the top half, so the edge at an odd column falls midway between output
    pixels."""
    m = torch.zeros(b, h, w, dtype=torch.bool)
    m[:, :, :5 * w // 12 + 1] = True
    m[:, :h // 2 + 1, :] = True
    m[-1, h // 4:, w // 2:] = False
    return m


def cascade_case(im, flavour, b, sizes, D, device, cfg_batched=False):
    """Imagen.sample arguments of the combined cases on the cascade `im` (objectives set here: stage 2 'v' on a zero-SNR
    schedule).  'ddim': stage 1 inpainting R = 2 (mask values of exactly 0.5), per-image seeds, per-image w, a negative
    prompt and a 'linear' guidance schedule; stage 2 a guidance interval with a 'cosine' schedule, per-image rescale and
    an init image with skip_steps = 1.  'dpmpp_2m': the same without inpainting (2M rejects it), on the multistep walk."""
    im.set_objectives(['noise', 'v'], zero_terminal_snr=[False, True])
    im.cfg_batched = cfg_batched
    im.use_cuda_graph = False
    im.noise_fn = None
    gen = torch.Generator().manual_seed(17)
    (h1, w1), (h2, w2) = sizes
    nte, ntm = _negative(1, D)
    on = lambda v: v.to(device)
    w1s = torch.tensor([2., 4.5, 1., 3.][:b])
    kw = dict(cond_scale=(on(w1s), on(torch.tensor([3., 1.5, 5., 2.][:b]))),
              guidance_interval=(None, (0.3, float("inf"))), guidance_schedule=("linear", "cosine"),
              guidance_rescale=(0., on(torch.tensor([0.7, 0.3, 1., 0.5][:b]))),
              init_images=(None, on(torch.rand(b, 3, h1, w1, generator=gen))), skip_steps=(0, 1),
              sampling_timesteps=(4, 4), seed=[5, 2 ** 40 + 1, 123, 7][:b], negative_text_embeds=on(nte),
              negative_text_masks=on(ntm), image_sizes=sizes)
    if flavour == "ddim":
        kw.update(ddim_eta=0.5, inpaint_images=on(torch.rand(b, 3, 2 * h1, 2 * w1, generator=gen)),
                  inpaint_masks=on(half_mask(b, 2 * h1, 2 * w1)), inpaint_resample_times=2)
    else:
        kw.update(sampler="dpmpp_2m")
    return kw


# the families (CheckingOps.family / features) each combined case must reach
REACH = {
    "ddim": {"inpaint_prologue", "inpaint_finalize", "randn_keyed", "step_epilogue", "step_epilogue_scheduled",
             "guidance_rescale_factor", "step_epilogue_rescaled", "q_sample", "resize_separable",
             "inpaint_prologue m = 0.5", "inpaint_prologue re-noise", "inpaint_prologue r = 0",
             "step_epilogue_rescaled plain scheduled", "randn_keyed renoise stage 1", "randn_keyed inpaint stage 2",
             "randn_keyed lowres stage 2", "randn_keyed init stage 2"},
    "dpmpp_2m": {"randn_keyed", "step_epilogue_multistep", "step_epilogue_multistep_scheduled",
                 "guidance_rescale_factor", "step_epilogue_rescaled", "q_sample", "resize_separable", "step_finalize",
                 "step_epilogue_rescaled multistep scheduled", "randn_keyed step stage 1", "randn_keyed init stage 2"},
    "ddpm_inpaint": {"inpaint_prologue", "inpaint_finalize", "randn_keyed", "step_epilogue", "inpaint_prologue re-noise",
                     "randn_keyed renoise stage 1"},
}


def reached(proxy):
    return set(proxy.checked) | proxy.features


def _cpu_cascade():
    g = load_golden("cascade_tiny.pt")
    im, _ = _cascade_from_golden(g, "cpu")
    return im, g


@pytest.mark.parametrize("flavour,cfg_batched", [("ddim", False), ("ddim", True), ("dpmpp_2m", False)])
def test_emulated_combined_cascade_passes_every_call_check(emu, flavour, cfg_batched):
    import minimagen_b200.ops as ops_mod
    im, g = _cpu_cascade()
    kw = cascade_case(im, flavour, 2, ((32, 48), (64, 96)), g["text_embeds"].shape[-1], "cpu", cfg_batched)
    proxy = CheckingOps(emu, sms=SMS)
    ops_mod.set_ops(proxy)
    out = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], **kw)
    print(f"\n{flavour} cascade, cfg_batched={cfg_batched} (emulated)")
    proxy.report()
    assert out.shape == (2, 3, 64, 96) and torch.isfinite(out).all()
    unchecked = proxy.called - proxy.checked - ALLOWED
    assert not unchecked, f"kernels that ran without a float64 check: {sorted(unchecked)}"
    assert REACH[flavour] <= reached(proxy), sorted(REACH[flavour] - reached(proxy))
    # the keyed draws of the walks: RePaint labels t * 2 + r on the base stage's grid, the stage-2 walk from grid[1]
    if flavour == "ddim":
        renoise = {lab for kind, st, labs in proxy.keyed if kind == "renoise" and st == 1 for lab in labs}
        assert renoise == {t * 2 + 1 for t in (24, 16, 8)}
        steps2 = [labs[0] for kind, st, labs in proxy.keyed if kind == "step" and st == 2]
        assert steps2 == [t * 2 + r for t, r in ((16, 0), (16, 1), (8, 0), (8, 1), (0, 0))]


def test_emulated_ddpm_inpaint_r3_passes_every_call_check(emu):
    import minimagen_b200.ops as ops_mod
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 25)
    im.use_cuda_graph = False
    proxy = CheckingOps(emu, sms=SMS)
    ops_mod.set_ops(proxy)
    gen = torch.Generator().manual_seed(3)
    mask = torch.zeros(2, 64, 64, dtype=torch.bool)
    mask[:, 8:40, 16:48] = True
    out = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=torch.tensor([3., 1.5]),
                    inpaint_images=torch.rand(2, 3, 64, 64, generator=gen), inpaint_masks=mask,
                    inpaint_resample_times=3, seed=[9, 10])
    proxy.report()
    assert torch.isfinite(out).all()
    assert not proxy.called - proxy.checked - ALLOWED
    assert REACH["ddpm_inpaint"] <= reached(proxy)
    renoise = sorted({labs[0] for kind, _, labs in proxy.keyed if kind == "renoise"})
    assert renoise == [t * 3 + r for t in range(1, 25) for r in (1, 2)]
    assert proxy.family["inpaint_prologue"][0] == 24 * 3 + 1


def device_walk(ops, T, R, B, seeds, n, next_t):
    """The captured RePaint step's bookkeeping without the U-Net: per iteration the three keyed draws at the labels read on
    the device (t * R + r), then mi_inpaint_advance, from t = T - 1, r = 0 until t = 0 has run.  Returns the (t, r) of
    every iteration."""
    dev = seeds.device
    t = torch.full((B,), T - 1, dtype=I64, device=dev)
    r = torch.zeros(B, dtype=I64, device=dev)
    Rt = torch.tensor([R], dtype=I64, device=dev)
    z = torch.empty(B, n, device=dev)
    walk = []
    while True:
        walk.append((int(t[0]), int(r[0])))
        for kind in ("renoise", "inpaint", "step"):
            ops.randn_keyed(z, seeds, B, n, K.KINDS[kind], 1, t=t, r=r, R=Rt)
        last = int(t[0]) == 0
        ops.inpaint_advance(t, r, next_t, Rt, T, B)
        if last:
            return walk


def test_device_side_repaint_walk_passes_its_checks():
    from minimagen_b200.diffusion_model import GaussianDiffusion
    T, R_ = 20, 3
    proxy = CheckingOps(EmuOps(), sms=SMS)
    walk = device_walk(proxy, T, R_, 2, torch.tensor([4, 2 ** 33]), 3 * 8 * 8,
                       GaussianDiffusion(timesteps=T).ddpm_schedule("cpu").next_t)
    assert walk == [(t, r) for t in range(T - 1, -1, -1) for r in range(R_ if t > 0 else 1)]
    assert {"inpaint_advance repeat", "inpaint_advance next point", "randn_keyed renoise stage 1 device labels"} <= \
        proxy.features
    assert {f"randn_keyed renoise stage 1 label {t * 3 + r}" for t in range(1, T) for r in range(3)} <= proxy.features
    assert proxy.checked == {"randn_keyed", "inpaint_advance"}


def test_three_kernel_step_passes_its_checks():
    """mi_step_x0, mi_step_quantile and mi_step_posterior (the pieces of the step the ABI runs for large images) through
    their checkers."""
    from minimagen_b200.Imagen import quantile_rank
    from minimagen_b200.diffusion_model import GaussianDiffusion
    gd = GaussianDiffusion(timesteps=50)
    B, n = 3, 3 * 16 * 16
    gen = torch.Generator().manual_seed(8)
    x, e, u, z = (torch.randn(B, n, generator=gen) for _ in range(4))
    t = torch.tensor([49, 20, 0])
    lo, hi, wq = quantile_rank(n, 0.9)
    proxy = CheckingOps(EmuOps(), sms=SMS)
    x0, s, out = torch.empty(B, n), torch.empty(B), torch.empty(B, n)
    proxy.step_x0(x, e, u, 3., t, gd.sqrt_recip_alphas_cumprod, gd.sqrt_recipm1_alphas_cumprod, B, n, x0)
    proxy.step_quantile(x0, B, n, lo, hi, wq, 1.0, s)
    proxy.step_posterior(x0, x, z, s, t, gd.posterior_mean_coef1, gd.posterior_mean_coef2, gd.sigma, B, n, out)
    assert proxy.checked == {"step_x0", "step_quantile", "step_posterior"}


# ------------------------------------------------------------------------------------------------ planted defects
class _Planted:
    def __init__(self, **methods):
        self.__dict__.update(methods)


def _prologue(defect):
    """mi_inpaint_prologue's contract op by op (emu_ops.prologue_ref) with one defect; every t in range."""
    def run(x, t, r, ra, rb, sqrt_acp, sqrt_1m_acp, k, m, z_renoise, z_known, T, B, C, hw):
        xv = x.reshape(B, C, hw)
        col = lambda tab, tt=t: tab[tt.clamp(0, T - 1)][:, None, None]
        ren = (r >= 0 if defect == "renoise at r = 0" else r > 0)[:, None, None]
        v = torch.where(ren, col(ra) * xv + col(rb) * z_renoise.reshape(B, C, hw), xv)
        mm = m.reshape(B, 1, hw)
        paste = mm > 0.5 if defect == "paste at m > 0.5" else mm >= 0.5
        a = col(sqrt_acp, t - 1) if defect == "sqrt_acp[t - 1]" else col(sqrt_acp)
        v = torch.where(paste, a * k.reshape(B, C, hw) + col(sqrt_1m_acp) * z_known.reshape(B, C, hw), v)
        x.copy_(v.reshape(x.shape))
    return run


def _prologue_call(ops):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    T, B, C, hw = 20, 3, 3, 64
    gd = GaussianDiffusion(timesteps=T)
    sch = gd.sampling_schedule(4, 0., "cpu")
    _, ra, rb = gd.inpaint_tables(sch, "cpu")
    gen = torch.Generator().manual_seed(6)
    x, k, zr, zk = (torch.randn(B, C, hw, generator=gen) for _ in range(4))
    m = torch.tensor([0., 0.25, 0.5, 0.75, 1.])[torch.randint(0, 5, (B, hw), generator=gen)]
    m[:, :4] = 0.5
    ops.inpaint_prologue(x, torch.tensor([6, 3, 9]), torch.tensor([0, 1, 2]), ra, rb, gd.sqrt_alphas_cumprod,
                         gd.sqrt_one_minus_alphas_cumprod, k, m, zr, zk, T, B, C, hw)


def _advance(defect):
    def run(t, r, next_t, R, T, B):
        valid = (t >= 0) & (t < T)
        rep = valid & (r + 1 < R[0]) & ((t >= 0) if defect else (t > 0))
        nt = torch.where(valid, next_t[t.clamp(0, T - 1)], torch.zeros_like(t))
        t.copy_(torch.where(rep, t, nt))
        r.copy_(torch.where(rep, r + 1, torch.zeros_like(r)))
    return run


def _advance_call(ops):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    next_t = GaussianDiffusion(timesteps=20).sampling_schedule(4, 0., "cpu").next_t
    ops.inpaint_advance(torch.tensor([0, 6, 6, 19, -1, 20]), torch.tensor([0, 0, 2, 1, 0, 0]), next_t, torch.tensor([3]),
                        20, 6)


def _finalize(defect):
    def run(x, k, m, B, C, hw, unnormalize, out):
        v = torch.where(m.reshape(B, 1, hw) >= 0.5, k.reshape(B, C, hw), x.reshape(B, C, hw))
        v = v if defect else v.clamp(-1., 1.)
        out.copy_(((v + 1) * 0.5 if unnormalize else v).reshape(out.shape))
    return run


def _finalize_call(ops):
    gen = torch.Generator().manual_seed(2)
    x, k = torch.randn(2, 3, 64, generator=gen) * 2, torch.rand(2, 3, 64, generator=gen) * 2 - 1
    x[0, 1, 5] = float("nan")
    m = (torch.rand(2, 64, generator=gen) < 0.5).float()
    m[0, 5] = 0.
    for unnormalize in (0, 1):
        ops.inpaint_finalize(x, k, m, 2, 3, 64, unnormalize, torch.empty_like(x))


def _randn(defect):
    def run(out, seeds, B, n, kind, stage, t=None, r=None, R=None, label=0):
        s = seeds[:B].roll(1) if defect == "neighbour seed" else seeds[:B]
        lab = t * int(R[0]) + (0 if defect == "label t * R" else r)
        out.copy_(torch.from_numpy(K.randn_keyed(s.tolist(), n, kind, stage, lab.tolist(), np.float32)).reshape(out.shape))
    return run


def _randn_call(ops):
    ops.randn_keyed(torch.empty(3, 100), torch.tensor([3, 99, 2 ** 50]), 3, 100, K.KINDS["renoise"], 2,
                    t=torch.tensor([5, 5, 7]), r=torch.tensor([1, 2, 0]), R=torch.tensor([3]))


def _scheduled(defect):
    emu = EmuOps()

    def run(x_t, eps_cond, eps_null, cond_scale, w_sched, t, *rest, **kw):
        if defect:
            t0 = t[:1].expand(t.shape[0])          # the guidance table read at image 0's t for every image
            emu.step_epilogue(x_t, eps_cond, eps_null, torch.where(w_sched[t0] == 1, cond_scale,
                              1 + (cond_scale - 1) * w_sched[t0]), t, *rest, **kw)
        else:
            emu.step_epilogue_scheduled(x_t, eps_cond, eps_null, cond_scale, w_sched, t, *rest, **kw)
    return run


def _scheduled_call(ops):
    from minimagen_b200.Imagen import quantile_rank
    from minimagen_b200.diffusion_model import GaussianDiffusion
    gd = GaussianDiffusion(timesteps=1000)
    sch = gd.sampling_schedule(10, 0.5, "cpu")
    tab = gd.guidance_table(None, "cosine", "cpu")
    B, n = 3, 3 * 16 * 16
    gen = torch.Generator().manual_seed(4)
    x, e, u, z = (torch.randn(B, n, generator=gen) for _ in range(4))
    t = torch.tensor([sch.grid[1], sch.grid[4], sch.grid[8]])
    lo, hi, wq = quantile_rank(n, 0.9)
    ops.step_epilogue_scheduled(x, e, u, torch.tensor([3., 6., 1.5]), tab, t, gd.sqrt_recip_alphas_cumprod,
                                gd.sqrt_recipm1_alphas_cumprod, sch.c1, sch.c2, sch.sigma, z, B, n, lo, hi, wq, 1.0,
                                torch.empty_like(x))


def _factor(defect):
    def run(eps_cond, eps_null, cond_scale, w_sched, t, phi, B, n, f):
        c, u = eps_cond.reshape(B, n), eps_null.reshape(B, n)
        g = (u + (c - u) * cond_scale[:, None]).double()
        cd = c.double()
        if defect:                                  # sums of squares about 0 instead of the mean
            ssc, ssg = (cd ** 2).sum(1), (g ** 2).sum(1)
        else:
            ssc, ssg = ((cd - cd.mean(1, keepdim=True)) ** 2).sum(1), ((g - g.mean(1, keepdim=True)) ** 2).sum(1)
        f.copy_((phi.double() * (ssc / ssg).sqrt() + (1 - phi.double())).to(F32))
    return run


def _factor_call(ops):
    gen = torch.Generator().manual_seed(1)
    B, n = 3, 3 * 32 * 32
    c = torch.randn(B, n, generator=gen) * torch.tensor([[1.], [0.5], [2.]]) + 0.3
    u = torch.randn(B, n, generator=gen) * 0.8 - 0.2
    ops.guidance_rescale_factor(c, u, torch.tensor([3., 7.5, 1.5]), None, torch.tensor([999, 500, 0]),
                                torch.tensor([0.7, 1., 0.3]), B, n, torch.empty(B))


PLANTED = {   # name -> (method, implementation factory (defect or None), the call)
    "prologue pastes at m > 0.5": ("inpaint_prologue", _prologue, "paste at m > 0.5", _prologue_call),
    "prologue re-noises at r == 0": ("inpaint_prologue", _prologue, "renoise at r = 0", _prologue_call),
    "prologue uses sqrt_acp[t - 1]": ("inpaint_prologue", _prologue, "sqrt_acp[t - 1]", _prologue_call),
    "advance increments r at t == 0": ("inpaint_advance", _advance, True, _advance_call),
    "finalize skips the clamp": ("inpaint_finalize", _finalize, True, _finalize_call),
    "randn_keyed uses the neighbouring image's seed": ("randn_keyed", _randn, "neighbour seed", _randn_call),
    "randn_keyed labels t * R without + r": ("randn_keyed", _randn, "label t * R", _randn_call),
    "scheduled step reads the table at image 0's t": ("step_epilogue_scheduled", _scheduled, True, _scheduled_call),
    "rescale factor without subtracting the mean": ("guidance_rescale_factor", _factor, True, _factor_call),
}


@pytest.mark.parametrize("name", sorted(PLANTED))
def test_planted_feature_defect_fails_its_call_check(name):
    """The correct implementation passes the method's check on the call's data; the planted defect fails it, and only it:
    a proxy over an ops object holding every planted method runs the calls of all the other methods too."""
    method, make, defect, call = PLANTED[name]
    good = CheckingOps(_Planted(**{method: make(None)}), sms=SMS)
    call(good)
    assert good.checked == {method}
    others = {m: make_(None) for m, make_, _, _ in PLANTED.values() if m != method}
    proxy = CheckingOps(_Planted(**others, **{method: make(defect)}), sms=SMS, strict=False)
    for c in dict.fromkeys(p[3] for p in PLANTED.values()):
        c(proxy)
    with pytest.raises(AssertionError) as e:
        proxy.raise_failures()
    print(f"\nplanted {name}: {str(e.value)[:300]}")
    assert all(f.startswith(method + "(") for f in proxy.failures), proxy.failures
