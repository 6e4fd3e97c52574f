"""Every kernel call of the workloads bench.py reports, at the benchmark's sizes, against float64: the flagship cfg-3
super-resolution U-Net (`Unet(**Super.defaults, lowres_cond=True, text_embed_dim=768)`) at 256 x 256 with b = 32, and the
secondary rows cfg 2b, cfg 4's base stage and cfg 5, each as `bench.workload` defines it.

test_gpu_lowering_calls.py checks every call of a forward at 32 - 64 px with b <= 16.  `conv_tc_launch` (csrc/conv_tc.cu)
picks the conv schedule from the problem size and the SM count, so those sizes never reach the schedules that carry the
benchmark's conv time: the 256-wide cooperative tiles, the transposed C_out = 128 schedule and the 128-wide ping-pong tiles
(at b = 2 nearly every conv steps down to 64-wide tiles, and at 64 px the deepest level runs on the fp32 direct conv).  Here:

  * test_every_call_of_the_cfg3_forward_at_benchmark_size, test_every_call_of_a_secondary_forward_at_benchmark_size[row]:
    one forward of each bench.py row (FORWARDS: cfg 3's conditional and null pass; cfg 2b at b = 64; cfg 4's base stage
    as one cfg_batched 2 x 64 batch, half of it on the null-text rows; cfg 5 at b = 2, 1024 x 1024) through
    `CheckingOps` (tests/checking_ops.py), with the assertions of
    test_every_call_of_a_forward, and the routes the row exists for.  A Python restatement of the schedule choice
    (`conv_schedule`) names the kernel instance of every conv call, and one profiler session over the whole checked run
    counts the conv_wg_kernel launches per instance: the two counts must agree, so the per-schedule table (calls, worst
    |err| / bound) is about the schedules that actually ran;
  * test_step_epilogue_many_cluster_waves: the step epilogue at B = 32 and 64 -- the fused cluster kernel (8 CTAs per
    image) then launches several waves of clusters -- and the three-kernel form, at cfg 5's n = 3 x 1024^2 too, against
    float64, with non-finite images past the first wave;
  * test_one_cfg3_sampling_step_at_benchmark_size, test_two_cfg5_sampling_steps_at_benchmark_size: Imagen.sample's eager
    loop (64 -> 256 px at b = 32; 256 -> 1024 px at b = 2), the loop's own kernels checked.

The float64 references of the image-sized calls are computed a few images, or at 1024 px a band of rows, at a time
(checking_ops._bands).  Each test prints its wall time and peak device memory.
"""
import collections
import inspect
import time

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import fp64_ref as R
from checking_ops import ALLOWED, CheckingOps
from emu_ops import EmuOps
from fp64_ref import check, check_rel_l2
from test_gpu_conv_transposed import conv_instance
from test_gpu_lowering_calls import _inputs
from test_gpu_sampler_ops import FUSED_MAX, _nan_equal, _tabs_cuda

pytestmark = pytest.mark.gpu

INT32_MAX = 2 ** 31 - 1
TRANSPOSED, COOP256, PINGPONG128 = (256, False, True), (256, False, False), (128, False, False)


# ------------------------------------------------------------------------------------------------ schedule restatement
# conv_tc_launch's choice of conv_wg_kernel<BLOCK_N, GN, TR> (csrc/conv_tc.cu), restated
def _ilog2_exact(v):
    lg = 0
    while (1 << lg) < v:
        lg += 1
    return lg if (1 << lg) == v else -1


def tile_geometry(H, W, B, tile_pix):
    """(BW, BH, tiles_w * tiles_h * tiles_b): a box of tile_pix pixels, BW x BH pixels x BB images."""
    BW = tile_pix if W >= tile_pix else W
    BH = min(tile_pix // BW, H)
    BB = tile_pix // (BW * BH)
    return BW, BH, -(-W // BW) * (H // BH) * -(-B // BB)


def pick_block_n(c_out, tiles_m, hint, sms):
    """The largest of 256 / 128 / 64 / 32 / 16 dividing C_out that still gives every SM a tile, never below 64 for that;
    a hint that divides C_out wins."""
    hint = abs(hint)
    if hint in (256, 128, 64, 32, 16) and c_out % hint == 0:
        return hint
    block_n = 16
    for c in (256, 128, 64, 32, 16):
        if c_out % c:
            continue
        block_n = c
        if tiles_m * (c_out // c) >= sms or c <= 64:
            break
    return block_n


def transposed_ok(c_out, n_valid, out_sc, H, W, in_stride, out_sh, out_sw):
    if c_out != 128 or n_valid != c_out or out_sc != 1:
        return False
    BW = 256 if W >= 256 else W
    if W % BW or _ilog2_exact(BW) < 3 or BW * in_stride > 256:
        return False
    BH = 256 // BW
    if BH * out_sh + BW * out_sw + c_out > INT32_MAX:
        return False
    return H % BH == 0 and BH * in_stride <= 256


def conv_schedule(B, H, W, c_out, sms, hint=0, n_valid=0, out_sc=1, in_stride=1, out_sh=0, out_sw=0):
    """The (BLOCK_N, GN, transposed) instance conv_tc_launch launches for this problem."""
    nv, sc, h = n_valid if n_valid > 0 else c_out, out_sc if out_sc > 0 else 1, abs(hint)
    ok = transposed_ok(c_out, nv, sc, H, W, in_stride, out_sh, out_sw)
    tr = ok if h == 256 else (h == 0 or c_out % h != 0) and ok and B * H * W // 256 >= sms
    if tr:
        return TRANSPOSED
    return pick_block_n(c_out, tile_geometry(H, W, B, 128)[2], hint, sms), False, False


def instance_name(inst):
    bn, gn, tr = inst
    if tr:
        return "transposed 128x256"
    if gn:
        return f"{bn}-wide GroupNorm prologue"
    return f"{bn}-wide " + ("cooperative" if bn == 256 else "ping-pong")


class ScheduleLog:
    """Wraps the checking proxy: names the kernel instance of every tensor-core conv call by the restatement, and keeps
    per instance the number of calls and their worst |err| / bound (the proxy's ratio of that call)."""

    def __init__(self, inner, sms):
        from minimagen_b200.ops import NativeOps
        self.inner, self.sms = inner, sms
        self.sig = {m: inspect.signature(getattr(NativeOps, m)) for m in ("conv_igemm", "conv_res1x1")}
        self.per = {}                                       # instance -> [calls, worst]

    def _instance(self, name, args, kwargs):
        if name == "conv_gn":
            return 128, True, False
        a = self.sig[name].bind(None, *args, **kwargs)
        a.apply_defaults()
        p = a.arguments
        if name == "conv_res1x1":
            return conv_schedule(p["B"], p["H"], p["W"], p["c_out"], self.sms, out_sh=p["W"] * p["c_out"],
                                 out_sw=p["c_out"])
        _, sh, sw = p["out_strides"]
        return conv_schedule(p["B"], p["H"], p["W"], p["c_out"], self.sms, hint=p["block_n"], n_valid=p["n_valid"],
                             out_sc=p["out_sc"], in_stride=2 if p["mode"] == 6 else 1, out_sh=sh, out_sw=sw)

    def __getattr__(self, name):
        target = getattr(self.inner, name)
        if name not in ("conv_igemm", "conv_res1x1", "conv_gn"):
            return target

        def call(*args, **kwargs):
            inst = self._instance(name, args, kwargs)
            ret = target(*args, **kwargs)
            rec = self.per.setdefault(inst, [0, 0.0])
            rec[0] += 1
            rec[1] = max(rec[1], self.inner.last)
            return ret
        return call

    def counts(self):
        return collections.Counter({inst: calls for inst, (calls, _) in self.per.items()})


def _profiled_launches(fn):
    """fn() under one profiler session; (its result, Counter of conv_wg_kernel launches per instance).  A session that
    returns no kernel record at all is repeated (up to three sessions) rather than read as "no conv ran"; fn builds
    fresh state each time."""
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            res = fn()
            torch.cuda.synchronize()
        launches = collections.Counter(conv_instance(ev.name) for ev in prof.events())
        launches.pop(None, None)
        if launches:
            break
    return res, launches


# ------------------------------------------------------------------------------------------------ the forward
# bench.py row -> (workload, batch, how the batch runs, the routes the case exists for: CheckingOps features)
FORWARDS = {
    # the headline: the conditional and the null pass of one guided step
    "cfg3": ("cfg3", 32, "guided", set()),
    # Base.defaults at dim 128: C_out = 384 convs, LayerNorm rows of 384 (the generic ln_rows kernel), the 8x8 level's
    # 128-pixel tiles spanning two images
    "cfg2b": ("cfg2b", 64, "one pass", {"conv_igemm c_out=384", "ln_rows C=384", "conv_igemm multi-image tiles"}),
    # cfg 4's base stage: the cfg-2a U-Net with both halves of a guided step in one 2B = 128 batch (Imagen.cfg_batched), the
    # second half on the null-text rows; its 4096-token self-attention at B = 128
    "cfg4_base": ("cfg2a", 64, "cfg_batched", {"attention B=128 n=4096", "text_tokens null rows B=128"}),
    # cfg 5 as measure_config(per_gpu=16, micro=2, cond_scale=1) runs it: 1024-wide rows, the 2048 + 2048-channel concat
    # convs at 64x64 (K = 36 864), the 4096-token self-attention and its LayerNorm rows at 2048 channels
    "cfg5": ("cfg5", 2, "one pass", {"conv_igemm W=1024", "conv_igemm K=36864", "attention B=2 n=4096", "ln_rows C=2048"}),
}


def _check_forward(native, row):
    """Every call of one forward of a bench.py row at the row's size (bench.workload: config, image size, text width)
    through CheckingOps, with the schedule restatement checked against the profiler's launch counts; the case must reach
    the routes it is listed for."""
    import bench
    import minimagen_b200.ops as ops_mod
    from minimagen_b200.Unet import Unet
    name, b, how, routes = FORWARDS[row]
    wl = bench.workload(name)
    cfg, s = wl["cfg"], wl["size"]
    assert cfg["text_embed_dim"] == wl["E"]
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    torch.manual_seed(0)
    u = Unet(**cfg).eval().cuda()
    x, t, kw = _inputs(cfg, s, b)
    tm = kw["text_mask"]
    tm[b // 2, 11:] = False                                 # ragged rows besides _inputs' last one, one with a single token
    tm[min(3, b - 1), 1:] = False

    def run():
        proxy = CheckingOps(native)
        log = ScheduleLog(proxy, sms)
        ops_mod.set_ops(log)                                # the `native` fixture restores the previous backend afterwards
        with torch.no_grad():
            if how == "guided":
                out = u.forward_with_cond_scale(x, t, cond_scale=3., **kw)   # the conditional and the null pass
            elif how == "cfg_batched":
                two = lambda v: torch.cat((v, v))
                keep = torch.cat((torch.ones(b, dtype=torch.uint8), torch.zeros(b, dtype=torch.uint8))).cuda()
                out = u._forward_impl(two(x), two(t), cond_keep=keep, **{k: two(v) for k, v in kw.items()})
            else:
                out = u(x, t, **kw)
        return out, proxy, log

    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    (out, proxy, log), launches = _profiled_launches(run)
    dt = time.time() - t0
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    assert torch.isfinite(out).all()
    n_acc = proxy.assert_accumulators_disjoint()
    passes = 2 if how == "guided" else 1
    print(f"\n{row} U-Net ({name}), b = {b} at {s}x{s}, {how} on {props.name} ({sms} SMs): {dt:.1f} s under the "
          f"profiler, peak {peak:.1f} GiB allocated, {n_acc} statistics accumulators (zero when handed out, disjoint)")
    proxy.report()
    predicted = log.counts()
    print("  conv schedule                      calls   worst |err|/bound   profiler launches   per forward")
    for inst in sorted(set(predicted) | set(launches), key=lambda i: (-i[2], -i[0], i[1])):
        calls, worst = log.per.get(inst, (0, 0.0))
        print(f"  {instance_name(inst):32s} {calls:7d}   {worst:17.3g}   {launches[inst]:17d}   {calls / passes:11g}")
    if "conv_direct" in proxy.family:
        calls, worst = proxy.family["conv_direct"]
        print(f"  {'fp32 direct':32s} {calls:7d}   {worst:17.3g}")
    unchecked = proxy.called - proxy.checked - ALLOWED
    assert not unchecked, f"kernels that ran without a float64 check: {sorted(unchecked)}"
    assert {"conv_igemm", "gn_apply_silu", "attention", "ln_rows", "linear_f32"} <= proxy.checked
    assert launches == predicted, f"profiler {dict(launches)} vs restatement {dict(predicted)}"
    missing = routes - proxy.features
    assert not missing, f"routes not reached: {sorted(missing)}; reached: {sorted(proxy.features)}"
    return sms, launches


def test_every_call_of_the_cfg3_forward_at_benchmark_size(native):
    sms, launches = _check_forward(native, "cfg3")
    if sms == 132:
        assert {TRANSPOSED, COOP256, PINGPONG128} <= set(launches), "a schedule of the benchmark was not reached"


@pytest.mark.parametrize("row", [r for r in FORWARDS if r != "cfg3"])
def test_every_call_of_a_secondary_forward_at_benchmark_size(native, row):
    _check_forward(native, row)


# ------------------------------------------------------------------------------------------------ the step epilogue
def _step_call(native, multi, x, eps, eps0, w, t, tabs, noise, hist, lo, hi, wt, out, s):
    a, b_, c1, c2, sigma, c3 = tabs
    B, n = x.shape
    if multi:
        native.step_epilogue_multistep(x, eps, eps0, w, t, a, b_, c1, c2, sigma, c3, noise, hist, B, n, lo, hi, wt, 1.0,
                                       out, s_out=s)
    else:
        native.step_epilogue(x, eps, eps0, w, t, a, b_, c1, c2, sigma, noise, B, n, lo, hi, wt, 1.0, out, s_out=s)


CFG5_N = 3 * 1024 * 1024                                    # one cfg-5 image: 3 x 1024 x 1024, 16 x FUSED_MAX


@pytest.mark.parametrize("kind", ["ddpm", "dpmpp"])
@pytest.mark.parametrize("B,n", [(32, FUSED_MAX), (32, FUSED_MAX + 1), (64, FUSED_MAX), (64, FUSED_MAX + 1), (2, CFG5_N),
                                 (16, CFG5_N)])
def test_step_epilogue_many_cluster_waves(native, B, n, kind):
    """At n = FUSED_MAX the fused cluster kernel runs B clusters of 8 CTAs, several waves at B = 32 and 64; n + 1 takes
    the three-kernel form, and so does cfg 5's n = 3 x 1024^2 (at its benchmark batch, 2, and at 16).  out, s and the
    history against float64 (test_step_epilogue_bounds' references and bounds) for scalar and per-image guidance weights,
    out separate from x_t and aliasing it; s bit for bit torch.quantile of step_x0's output.  Then (B >= 4) images B - 4
    (one NaN), B - 3 (15 % +inf) and B - 2 (two +-inf), past the first wave, must give the NaN pattern the torch
    restatement gives (as test_step_nan_and_inf_parity at B = 4), and the clean images the bits of a run without them."""
    assert n <= 2 ** 24, "torch.quantile, the reference of s, takes rows of up to 2^24 elements"
    from minimagen_b200.Imagen import quantile_rank
    tabs, grid = _tabs_cuda(kind)
    multi = kind == "dpmpp"
    t0 = time.time()
    g = torch.Generator().manual_seed(B + n + len(kind))
    x = torch.randn(B, n, generator=g) * 1.3
    x[-1] *= 0.2                                            # its threshold falls below min_s = 1 at t = 0
    eps, eps0, noise, hist = (torch.randn(B, n, generator=g) for _ in range(4))
    t = torch.tensor([grid[(7 * i) % len(grid)] for i in range(B)])
    t[-1] = 0
    lo, hi, wt = quantile_rank(n, 0.9)
    xc, tc, ec, e0c, zc = x.cuda(), t.cuda(), eps.cuda(), eps0.cuda(), noise.cuda()
    for guidance in ("scalar", "per_image"):
        w = torch.linspace(1.5, 7.5, B) if guidance == "per_image" else 3.0
        wn = w.cuda() if torch.is_tensor(w) else w
        x0r, bx0 = R.step_x0_ref(x, eps, eps0, w, t, tabs[0], tabs[1])
        sr, bs = R.step_threshold_ref(x0r, bx0, lo, hi, wt, 1.0)
        outr, bo, xsr, bxs = R.step_posterior_ref(x0r, bx0, sr, bs, x, noise, t, *tabs[2:5], tabs[5] if multi else None,
                                                  hist if multi else None)
        results = []
        for alias in (False, True):
            xin = xc.clone()
            out, s, h = (xin if alias else torch.empty_like(xc)), torch.empty(B, device="cuda"), hist.cuda()
            _step_call(native, multi, xin, ec, e0c, wn, tc, tabs, zc, h, lo, hi, wt, out, s)
            results.append((out.clone(), s.clone(), h.clone()))
        (out, s, h), (out2, s2, h2) = results
        assert torch.equal(out, out2) and torch.equal(s, s2) and torch.equal(h, h2), "aliasing out and x_t changed the result"
        what = f"{kind} B={B} n={n} {guidance}"
        check(s, sr, bs, f"{what} s")
        check(out, outr, bo, f"{what} out")
        check_rel_l2(out, outr, 1e-6, f"{what} out")
        if multi:
            check(h, xsr, bxs, f"{what} hist")
        if guidance == "scalar":
            x0n = torch.empty_like(xc)
            native.step_x0(xc, ec, e0c, w, tc, tabs[0], tabs[1], B, n, x0n)
            assert torch.equal(s.cpu(), torch.quantile(x0n.abs().cpu(), 0.9, dim=-1).clamp(min=1.0)), f"{what}: s not exact"

    if B < 4:
        print(f"{kind} B={B} n={n}: {time.time() - t0:.1f} s")
        return
    # non-finite images past the first wave of clusters
    xb, eb = x.clone(), eps.clone()
    eb[B - 4, n // 2] = float("nan")
    xb[B - 3, torch.randperm(n, generator=g)[:(15 * n + 99) // 100]] = float("inf")
    xb[B - 2, :2] = torch.tensor([float("inf"), -float("inf")])
    h = hist.cuda()
    on, sn = torch.empty(B, n, device="cuda"), torch.empty(B, device="cuda")
    _step_call(native, multi, xb.cuda(), eb.cuda(), e0c, 3.0, tc, tabs, zc, h, lo, hi, wt, on, sn)
    oe, se, he = torch.empty(B, n), torch.empty(B), hist.clone()
    ct = [v.cpu() if v is not None else None for v in tabs]
    if multi:
        EmuOps().step_epilogue_multistep(xb, eb, eps0, 3.0, t, *ct, noise, he, B, n, lo, hi, wt, 1.0, oe, s_out=se)
    else:
        EmuOps().step_epilogue(xb, eb, eps0, 3.0, t, *ct[:5], noise, B, n, lo, hi, wt, 1.0, oe, s_out=se)
    bad = torch.zeros(B, dtype=torch.bool)
    bad[B - 4:B - 2] = True
    assert torch.equal(sn.cpu().isnan(), bad), f"NaN thresholds at {sn.cpu().isnan().nonzero().flatten().tolist()}"
    assert on[bad.cuda()].isnan().all(), "an image with a NaN x0 or >= 10 % inf must come out all NaN"
    _nan_equal(sn, se, f"{kind} B={B} n={n} s_out")
    _nan_equal(on, oe, f"{kind} B={B} n={n} out")
    if multi:
        _nan_equal(h, he, f"{kind} B={B} n={n} hist")
    oc, sc, hc = torch.empty(B, n, device="cuda"), torch.empty(B, device="cuda"), hist.cuda()
    _step_call(native, multi, xc, ec, e0c, 3.0, tc, tabs, zc, hc, lo, hi, wt, oc, sc)
    clean = ~bad
    clean[B - 2] = False
    assert torch.equal(on[clean.cuda()], oc[clean.cuda()]) and torch.equal(sn[clean.cuda()], sc[clean.cuda()])
    assert torch.equal(h[clean.cuda()], hc[clean.cuda()])
    print(f"{kind} B={B} n={n}: {time.time() - t0:.1f} s")


# ------------------------------------------------------------------------------------------------ one sampling step
LOOP = {"step_epilogue", "step_epilogue_multistep", "step_advance_t", "step_advance_t_table", "step_finalize",
        "resize_separable", "q_sample"}


def _two_sampling_steps(native, name, b):
    """Imagen.sample(start_at_unet_number=2) with the bench.py row's U-Net as the second stage, from random images of the
    first stage's size, two DDIM steps with guidance w = 3, eager (a loop of two steps is not captured): the loop's own
    kernels -- the cascade resize of the start images, q_sample of the low-res conditioning, the step epilogue, the
    finalize -- checked against float64; the U-Net calls run unchecked (see the forward test above)."""
    import bench
    import minimagen_b200.ops as ops_mod
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import BaseTest, Unet
    wl = bench.workload(name)
    size, low = wl["size"], wl["size"] // 4
    torch.manual_seed(0)
    u = Unet(**wl["cfg"]).eval()
    first = Unet(**dict(BaseTest.defaults, text_embed_dim=wl["E"])).eval()
    im = Imagen(unets=(first, u), text_encoder_name="t5_base", image_sizes=(low, size), timesteps=1000,
                cond_drop_prob=0.1).eval().cuda()
    im.use_cuda_graph = False
    g = torch.Generator().manual_seed(11)
    te = torch.randn(b, 20, wl["E"], generator=g).cuda()
    tm = torch.ones(b, 20, dtype=torch.bool)
    tm[-1, 5:] = False
    start = torch.rand(b, 3, low, low, generator=g).cuda()
    proxy = CheckingOps(native, only=LOOP)
    ops_mod.set_ops(proxy)                                  # the `native` fixture restores the previous backend afterwards
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    out = im.sample(text_embeds=te, text_masks=tm.cuda(), cond_scale=3., sampling_timesteps=2, start_at_unet_number=2,
                    start_images=start)
    torch.cuda.synchronize()
    print(f"\ntwo {name} sampling steps, b = {b}, {low} -> {size} px: {time.time() - t0:.1f} s, peak "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB allocated")
    proxy.report()
    assert tuple(out.shape) == (b, 3, size, size) and torch.isfinite(out).all()
    assert proxy.family["step_epilogue"][0] == 2
    assert {"step_epilogue", "step_finalize", "resize_separable", "q_sample"} <= proxy.checked


def test_one_cfg3_sampling_step_at_benchmark_size(native):
    _two_sampling_steps(native, "cfg3", 32)


def test_two_cfg5_sampling_steps_at_benchmark_size(native):
    """cfg 5's loop at its benchmark batch: the resize 256 -> 1024 and images of n = 3 x 1024^2 in the step epilogue's
    three-kernel form."""
    _two_sampling_steps(native, "cfg5", 2)
