"""FootprintOps (tests/footprint_ops.py) on a machine without a GPU, over the torch emulation (tests/emu_ops.py):

  * completeness: every public method of minimagen_b200.ops.NativeOps has a write footprint (`_writes_<method>`) or is in
    checking_ops.ALLOWED (no kernel), so a kernel added to the interface later fails here until it gets one;
  * the footprints are not too narrow: the emulated lowering forwards, training steps and a combined sampling cascade pass
    under CheckingOps(FootprintOps(EmuOps())), every call both float64- and footprint-checked, and so does the boundary
    call list (`boundary_calls`, which tests/test_gpu_footprint.py runs on the native kernels);
  * the checks are not vacuous: each planted stray write on EmuOps fails its own method's footprint check only, with a
    message naming the region it landed in.
"""
import inspect
import types

import pytest
import torch

import minimagen_b200.ops as ops_mod
from checking_ops import ALLOWED, CheckingOps, run_training_step, train_cases
from emu_ops import EmuOps, _strided
from footprint_ops import FootprintOps, installed, unchecked

SMS = 132
F16, F32, F64, I64, U8 = torch.float16, torch.float32, torch.float64, torch.int64, torch.uint8


# ------------------------------------------------------------------------------------------------ completeness
def test_every_ops_method_has_a_write_footprint():
    from minimagen_b200.ops import NativeOps
    methods = {n for n, _ in inspect.getmembers(NativeOps, inspect.isfunction) if not n.startswith("_")}
    missing = sorted(n for n in methods - ALLOWED if not hasattr(FootprintOps, "_writes_" + n))
    assert not missing, f"NativeOps methods without a write footprint in FootprintOps: {missing}"
    stale = sorted(n[len("_writes_"):] for n in dir(FootprintOps) if n.startswith("_writes_")
                   and n[len("_writes_"):] not in methods)
    assert not stale, f"write footprints of methods NativeOps does not have: {stale}"
    params = lambda f: [p.name for p in inspect.signature(f).parameters.values()]
    differ = sorted(n for n in methods - ALLOWED
                    if params(getattr(FootprintOps, "_writes_" + n)) != params(getattr(NativeOps, n)))
    assert not differ, f"write footprints whose parameters differ from NativeOps's: {differ}"


# ------------------------------------------------------------------------------------------------ the boundary calls
def boundary_calls(ops, dev):
    """Direct calls at the shapes where a store goes astray: every output sized exactly (so the first stray element lands in
    a guard) or a view inside a buffer whose other elements hold data."""
    from minimagen_b200.Imagen import quantile_rank
    from minimagen_b200.diffusion_model import GaussianDiffusion
    g = torch.Generator().manual_seed(0)

    def rn(*shape, dt=F32, scale=1.0):
        return (torch.randn(*shape, generator=g) * scale).to(dt).to(dev)

    def conv(B, H, W, c_in=64, c_out=64, block_n=0, n_valid=0, res=True, stats=True, out_stats=None):
        nv = n_valid or c_out
        st = out_stats if out_stats is not None else (
            torch.zeros(B, c_out // 16, 2, dtype=F64, device=dev) if stats else None)
        ops.conv_igemm(rn(B, H, W, c_in, dt=F16), B, H, W, c_in, 0, c_in, rn(c_out, 9 * c_in, dt=F16, scale=0.05), c_out,
                       3, 3, 0, rn(c_out), rn(B, H, W, c_out) if res else None, None,
                       torch.empty(B, H, W, nv, dtype=F16, device=dev), (H * W * nv, W * nv, nv), block_n=block_n,
                       n_valid=n_valid, out_stats=st)

    # partial multi-image tiles (a 128-pixel tile covers 2 images at 8 x 8, 4 at 4 x 8), ragged widths
    conv(1, 8, 8)
    conv(3, 8, 8)
    conv(5, 4, 8)
    conv(2, 4, 130, stats=False)
    conv(2, 8, 200)
    # the schedules: 256-wide cooperative, transposed 128 x 256, 64 / 32 / 16-wide ping-pong with n_valid < c_out (a
    # channel-contiguous output pitch is a multiple of 4 elements)
    conv(2, 8, 8, c_out=256, block_n=256)
    conv(2, 16, 16, c_out=128, block_n=256)
    conv(2, 8, 8, c_out=128, block_n=64, n_valid=100, res=False, stats=False)
    conv(2, 8, 8, c_out=64, block_n=32, n_valid=52, res=False, stats=False)
    conv(2, 8, 8, c_out=32, block_n=16, n_valid=12, res=False, stats=False)
    # statistics carved next to each other: the neighbours hold data
    arena = rn(3 * 2 * 4 * 2, dt=F64)
    arena[16:32] = 0
    conv(2, 8, 8, out_stats=arena[16:32].view(2, 4, 2))
    # the NCHW final conv: n_valid = 3 of 16 channels, out_sc = H W, into an exact [B, 3, H, W]
    B, H, W = 2, 8, 8
    out = torch.empty(B, 3, H, W, device=dev)
    ops.conv_igemm(rn(B, H, W, 64, dt=F16), B, H, W, 64, 0, 64, rn(16, 9 * 64, dt=F16, scale=0.05), 16, 3, 3, 0, rn(16),
                   None, out, None, (3 * H * W, W, 1), out_sc=H * W, n_valid=3)
    # a channel slice of a concat buffer whose other channels hold data
    cat = rn(B, H, W, 192, dt=F16)
    ops.conv_igemm(rn(B, H, W, 64, dt=F16), B, H, W, 64, 0, 64, rn(64, 9 * 64, dt=F16, scale=0.05), 64, 3, 3, 0, rn(64),
                   None, None, cat[..., 64:], (H * W * 192, W * 192, 192),
                   out_stats=torch.zeros(B, 4, 2, dtype=F64, device=dev))
    # the four sub-pixel phases into one interleaved output, one accumulator
    Ho, Wo, C = 2 * H, 2 * W, 64
    o32 = torch.empty(B, Ho, Wo, C, device=dev)
    st = torch.zeros(B, C // 16, 2, dtype=F64, device=dev)
    a16 = rn(B, H, W, 64, dt=F16)
    for p in range(4):
        off = ((p >> 1) * Wo + (p & 1)) * C
        ops.conv_igemm(a16, B, H, W, 64, 0, 64, rn(C, 4 * 64, dt=F16, scale=0.05), C, 2, 2, 2 + p, rn(C), None,
                       o32.reshape(-1)[off:], None, (Ho * Wo * C, 2 * Wo * C, 2 * C), out_stats=st)
    # conv_gn and conv_res1x1 at their smallest accepted shapes
    B, H, W, c0, c_out, groups = 2, 32, 8, 64, 128, 4
    assert ops.conv_gn_supported(H, W, c0, 0, c_out, groups)
    src = rn(B, H, W, c0)
    blk = src.double().reshape(B, H * W, c0 // 16, 16)
    stats0 = torch.stack((blk.sum(dim=(1, 3)), (blk * blk).sum(dim=(1, 3))), dim=-1).contiguous()
    ops.conv_gn(src, c0, None, 0, 1.0, B, H, W, groups, stats0, None, rn(c0), rn(c0), rn(B, 2 * c0, scale=0.1), 2 * c0,
                1e-5, rn(c_out, 9 * c0, dt=F16, scale=0.05), c_out, rn(c_out), rn(B, H, W, c_out), None,
                torch.empty(B, H, W, c_out, dtype=F16, device=dev), torch.zeros(B, c_out // 16, 2, dtype=F64, device=dev))
    B, H, W = 2, 16, 16
    assert ops.conv_res1x1_supported(H, W, 64, 128, 64)
    ops.conv_res1x1(rn(B, H, W, 64, dt=F16), B, H, W, 64, 64, None, 0, 0, rn(B, H, W, 64, dt=F16), 64, 64, None, 0, 0,
                    rn(128, 9 * 64 + 64, dt=F16, scale=0.05), 128, rn(128), None, torch.empty(B, H, W, 128, device=dev),
                    None, torch.zeros(B, 8, 2, dtype=F64, device=dev))
    # attention on both paths (the wgmma one at n % 128 == 0, m >= 128), ragged m, a strided output with o_bs > n ldo
    for n, m in ((128, 130), (70, 77)):
        B, heads = 2, 2
        ldo = heads * 64 + 64
        o_bs = n * ldo + 192
        q, kv = rn(B, n, heads * 64, dt=F16), rn(B, m, 2 * heads * 64, dt=F16)
        mask = (torch.rand(B, m, generator=g) < 0.8).to(U8).to(dev)
        out = torch.empty((B - 1) * o_bs + (heads - 1) * 64 + (n - 1) * ldo + 64, dtype=F16, device=dev)
        ops.attention(q, n * heads * 64, heads * 64, kv, kv[..., heads * 64:], m * 2 * heads * 64, 2 * heads * 64, 64,
                      rn(2, 64), mask, B, heads, n, m, out, o_bs, ldo)
    # the step-epilogue family, fused and in three kernels, at B = 3 (not a multiple of the cluster size) and odd n; then
    # n past the fused limit (the x0 workspace)
    gd = GaussianDiffusion(timesteps=50)
    d = lambda v: v.to(dev)
    sch, msch = gd.sampling_schedule(10, 0.5, dev), gd.dpm_solver_schedule(10, dev)
    wsch = d(gd.guidance_table(None, "cosine", "cpu"))
    tab_a, tab_b = d(gd.sqrt_recip_alphas_cumprod), d(gd.sqrt_recipm1_alphas_cumprod)
    for B, n in ((3, 3 * 17 * 17), (3, 3 * 256 * 256 + 1)):
        x, e, u, z, hist = (rn(B, n) for _ in range(5))
        t = d(torch.tensor([sch.grid[1], sch.grid[4], 0][:B]))
        lo, hi, wq = quantile_rank(n, 0.9)
        w = d(torch.tensor([3., 6., 1.5][:B]))
        common = (tab_a, tab_b, sch.c1, sch.c2, sch.sigma)
        ops.step_epilogue(x, e, u, 3., t, *common, z, B, n, lo, hi, wq, 1.0, torch.empty(B, n, device=dev),
                          s_out=torch.empty(B, device=dev))
        xa = x.clone()                                                  # out is x_t
        ops.step_epilogue(xa, e, u, w, t, *common, z, B, n, lo, hi, wq, 1.0, xa)
        mt = (tab_a, tab_b, msch.c1, msch.c2, msch.sigma, msch.c3)
        ops.step_epilogue_multistep(x, e, u, w, t, *mt[:5], mt[5], z, hist, B, n, lo, hi, wq, 1.0,
                                    torch.empty(B, n, device=dev))
        ops.step_epilogue_scheduled(x, e, u, w, wsch, t, *common, z, B, n, lo, hi, wq, 1.0, torch.empty(B, n, device=dev),
                                    s_out=torch.empty(B, device=dev))
        ops.step_epilogue_multistep_scheduled(x, e, u, w, wsch, t, *mt[:5], mt[5], z, hist, B, n, lo, hi, wq, 1.0,
                                              torch.empty(B, n, device=dev))
        f = torch.empty(B, device=dev)
        ops.guidance_rescale_factor(e, u, w, wsch, t, d(torch.tensor([0.7, 1., 0.3][:B])), B, n, f)
        ops.step_epilogue_rescaled(x, e, u, w, wsch, f, t, *common, None, z, None, B, n, lo, hi, wq, 1.0,
                                   torch.empty(B, n, device=dev))
        ops.step_epilogue_rescaled(x, e, u, w, None, f, t, *mt[:5], mt[5], z, hist, B, n, lo, hi, wq, 1.0,
                                   torch.empty(B, n, device=dev), s_out=torch.empty(B, device=dev))
        x0, s = torch.empty(B, n, device=dev), torch.empty(B, device=dev)
        ops.step_x0(x, e, u, 3., t, tab_a, tab_b, B, n, x0)
        ops.step_quantile(x0, B, n, lo, hi, wq, 1.0, s)
        ops.step_posterior(x0, x, z, s, t, sch.c1, sch.c2, sch.sigma, B, n, torch.empty(B, n, device=dev))
    # the loop's bookkeeping on state tensors longer than B (only [:B] is the call's), and its per-image kernels
    import keyed_noise_restatement as K
    B, T, n = 3, 50, 3 * 8 * 8
    t, r = d(torch.tensor([sch.grid[2], 7, 0, 11, 12])), d(torch.tensor([0, 1, 0, 5, 5]))
    ops.step_advance_t(t.clone(), B)
    ops.step_advance_t_table(t.clone(), sch.next_t, T, B)
    ops.inpaint_advance(t.clone(), r.clone(), sch.next_t, d(torch.tensor([2])), T, B)
    ops.randn_keyed(torch.empty(B, n, device=dev), d(torch.tensor([3, 99, 2 ** 50])), B, n, K.KINDS["renoise"], 1, t=t,
                    r=r, R=d(torch.tensor([2])))
    _, ra, rb = gd.inpaint_tables(sch, dev)
    x, k, zr, zk = (rn(B, 3, 64) for _ in range(4))
    msk = d((torch.rand(B, 64, generator=g) < 0.5).float())
    ops.inpaint_prologue(x, t[:B].clone(), r[:B].clone(), ra, rb, d(gd.sqrt_alphas_cumprod),
                         d(gd.sqrt_one_minus_alphas_cumprod), k, msk, zr, zk, T, B, 3, 64)
    ops.inpaint_finalize(x, k, msk, B, 3, 64, 1, torch.empty(B, 3, 64, device=dev))
    ops.step_finalize(x, B * 3 * 64, 1, torch.empty(B, 3, 64, device=dev))
    ops.q_sample(x, zr, t[:B].clone(), d(gd.sqrt_alphas_cumprod), d(gd.sqrt_one_minus_alphas_cumprod), B, 3 * 64, 1.0,
                 0.0, torch.empty(B, 3, 64, device=dev))
    # text_tokens / place_rows with row_off > 0 inside rows that hold data
    B, L, D, max_len, m = 2, 7, 64, 6, 11
    c_out = rn(B, m, D)
    keep = d(torch.tensor([1, 0], dtype=U8))
    mask = d(torch.tensor([[1] * 7, [1] * 4 + [0] * 3], dtype=U8))
    ops.text_tokens(rn(B, L, D), B, L, D, mask, keep, rn(max_len, D), max_len, c_out, m, 2, torch.empty(B, D, device=dev))
    ops.place_rows(rn(B, 2, D), B, 2, D, c_out, m, 8)
    # cast_act in its three modes into an oversized output
    B, H, W, c0, c1 = 2, 4, 6, 64, 64
    for mode in (0, 1, 2):
        n_out = B * H * W * (c0 + c1) * (4 if mode == 1 else 1)
        ops.cast_act(rn(B, H, W, c0), c0, rn(B, H, W, c1), c1, 0.7, B, H, W, mode,
                     torch.empty(n_out + 1000, dtype=F16, device=dev))
    # gemm_f32: ragged M, N, K into a strided C inside a larger buffer, two batches
    M, N_, K, ld = 37, 45, 29, 53
    Cbuf = rn(2, M + 3, ld)
    ops.gemm_f32(rn(2, M, K), rn(2, K, N_), Cbuf[:, 1:], M, N_, K, (K, 1), (N_, 1), (ld, 1), Z1=2, a_b=(M * K, 0),
                 b_b=(K * N_, 0), c_b=((M + 3) * ld, 0))
    # gn_silu_bwd with dss_ld > 2C, into an exact [B - 1 rows of dss_ld + 2C]
    B, hw, C, groups, ld = 2, 64, 64, 8, 2 * 64 + 32
    x = rn(B, hw, C)
    xg = x.double().reshape(B, hw, groups, C // groups)
    sums = torch.stack((xg.sum(dim=(1, 3)), (xg * xg).sum(dim=(1, 3))), dim=-1).contiguous()
    ops.gn_silu_bwd(x, rn(B, hw, C), sums, B, hw, C, groups, rn(C), rn(C), rn(B, 2 * C, scale=0.1), 2 * C, 1e-5,
                    torch.empty(B, hw, C, device=dev), torch.zeros(C, device=dev), torch.zeros(C, device=dev),
                    torch.empty((B - 1) * ld + 2 * C, device=dev), ld)
    # conv_wgrad_tc at both strides
    for stride, k in ((1, 3), (2, 4)):
        B, Ho, Wo, c_in, co = 2, 8, 8, 64, 128
        ops.conv_wgrad_tc(rn(B, Ho, Wo, co, dt=F16), rn(B, stride * Ho, stride * Wo, c_in, dt=F16), B, Ho, Wo, c_in, co, k,
                          k, torch.empty(co, c_in, k, k, device=dev), stride=stride)


def test_boundary_calls_pass_on_the_emulation():
    proxy = FootprintOps(EmuOps())
    boundary_calls(CheckingOps(proxy, sms=SMS), "cpu")
    proxy.report()
    assert not unchecked(proxy)


# ------------------------------------------------------------------------------------------------ emulated real runs
def test_emulated_forwards_pass(emu):
    from test_gpu_lowering_calls import forward_case, run_forward
    for name in ("cfg_batched", "base_d64_mid_attn"):
        fp = FootprintOps(emu)
        proxy = CheckingOps(fp, sms=SMS)
        out = run_forward(proxy, *forward_case(name, "cpu"))
        assert torch.isfinite(out).all()
        print(f"\n{name} (emulated)")
        fp.report()
        assert not unchecked(fp) and not proxy.called - proxy.checked - ALLOWED


@pytest.mark.parametrize("case", ["base_d64_mid_attn", "cascade_unet1", "cascade_unet2"])
def test_emulated_training_steps_pass(monkeypatch, case):
    import minimagen_b200.autograd as ag
    monkeypatch.setattr(ag, "ROUTE_TC_ON_CPU", True)
    fp = FootprintOps(EmuOps())
    with installed(CheckingOps(fp, sms=SMS, fresh_accumulators=True)):
        run_training_step(train_cases()[case][0], "cpu")
    fp.report()
    assert not unchecked(fp)


def test_emulated_combined_cascade_passes(emu):
    from test_sampling_feature_calls import _cpu_cascade, cascade_case
    im, g = _cpu_cascade()
    kw = cascade_case(im, "ddim", 2, ((32, 48), (64, 96)), g["text_embeds"].shape[-1], "cpu", False)
    fp = FootprintOps(emu)
    with installed(CheckingOps(fp, sms=SMS)):
        out = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], **kw)
    fp.report()
    assert torch.isfinite(out).all()
    assert not unchecked(fp)
    assert {"inpaint_prologue", "step_epilogue_rescaled", "randn_keyed", "conv_igemm"} <= fp.checked


# ------------------------------------------------------------------------------------------------ planted stray writes
def _after_conv(extra):
    """conv_igemm as emulated, then `extra` (the call's bound arguments) writes where it must not."""
    def method(self, *args, **kwargs):
        EmuOps.conv_igemm(self, *args, **kwargs)
        a = inspect.signature(EmuOps.conv_igemm).bind(self, *args, **kwargs)
        a.apply_defaults()
        extra(a.arguments)
    return method


def _with_plain_conv(name):
    """EmuOps.<name>, its inner conv_igemm the unplanted one."""
    def method(self, *args, **kwargs):
        self.conv_igemm = types.MethodType(EmuOps.conv_igemm, self)
        try:
            return getattr(EmuOps, name)(self, *args, **kwargs)
        finally:
            del self.conv_igemm
    return method


def _image_B(a):        # the store for image B, past the last image
    o = a["out_f16"] if a["out_f16"] is not None else a["out_f32"]
    if a["out_sc"] == 1 and a["mode"] == 0 and o.dtype == F16:
        sb, sh, sw = a["out_strides"]
        nv = a["n_valid"] or a["c_out"]
        o.as_strided((a["H"], a["W"], nv), (sh, sw, 1), o.storage_offset() + a["B"] * sb).fill_(-7)


def _channel_n_valid(a):  # the NCHW final conv's channel n_valid
    if a["out_sc"] > 1:
        sb, sh, sw = a["out_strides"]
        o = a["out_f32"]
        o.as_strided((a["B"], a["H"], a["W"]), (sb, sh, sw), o.storage_offset() + a["n_valid"] * a["out_sc"]).fill_(-7)


def _beside_slice(a):   # the channel after its slice of a concat buffer
    o = a["out_f16"]
    sb, sh, sw = a["out_strides"]
    if o is not None and sw > a["c_out"]:
        o.as_strided((a["B"], a["H"], a["W"]), (sb, sh, sw), o.storage_offset() + a["c_out"]).fill_(-7)


def _neighbour_phase(a):  # phase p writing the neighbouring pixel's parity
    if a["mode"] == 2:
        sb, sh, sw = a["out_strides"]
        o = a["out_f32"]
        o.as_strided((a["B"], a["H"], a["W"], a["c_out"]), (sb, sh, sw, 1), o.storage_offset() + sw // 2).fill_(-7)


def _next_stats(a):     # statistics incremented into the next accumulator
    s = a["out_stats"]
    if s is not None and s.storage_offset() > 0:                        # the accumulator carved from the middle
        n = s.numel()
        s.as_strided((n,), (1,), s.storage_offset() + n).add_(1.0)


def _text_row_before(self, proj, B, L, D, mask, keep, null_embed, max_len, c_out, m, row_off, pooled):
    EmuOps.text_tokens(self, proj, B, L, D, mask, keep, null_embed, max_len, c_out, m, row_off, pooled)
    c_out.reshape(B, m, D)[:, row_off - 1] = -7


def _step_eps_cond(self, x_t, eps_cond, *args, **kwargs):
    EmuOps.step_epilogue(self, x_t, eps_cond, *args, **kwargs)
    eps_cond.reshape(-1)[1] = -7


def _attention_workspace(self, q, q_bs, ldq, k, v, kv_bs, ldkv, kv_hs, null_kv, mask, B, heads, n, m, out, o_bs, ldo):
    ws = ops_mod.torch.empty(B * heads * m, dtype=F32, device=q.device)
    ws.as_strided((ws.numel() + 1,), (1,), ws.storage_offset()).fill_(0.5)       # one element past its end
    EmuOps.attention(self, q, q_bs, ldq, k, v, kv_bs, ldkv, kv_hs, null_kv, mask, B, heads, n, m, out, o_bs, ldo)


PLANTED = {   # name -> (method, planted implementation, the region the message must name, and more it must contain)
    "conv stores image B into the guard": ("conv_igemm", _after_conv(_image_B), "guard after", "element [1, 0, 0, 0]"),
    "NCHW final conv writes channel n_valid": ("conv_igemm", _after_conv(_channel_n_valid), "guard after", "`out_f32`"),
    "conv writes beside its concat slice": ("conv_igemm", _after_conv(_beside_slice), "outside the footprint",
                                            "element [0, 0, 0, 64]"),
    "sub-pixel phase writes its neighbour's parity": ("conv_igemm", _after_conv(_neighbour_phase),
                                                      "outside the footprint", "`out_f32`"),
    "statistics into the next accumulator": ("conv_igemm", _after_conv(_next_stats), "outside the footprint",
                                             "`out_stats`"),
    "text_tokens writes row row_off - 1": ("text_tokens", _text_row_before, "outside the footprint",
                                           "element [0, 1, 0]"),
    "step epilogue modifies eps_cond": ("step_epilogue", _step_eps_cond, "outside the footprint", "`eps_cond`"),
    "a workspace written one element past its end": ("attention", _attention_workspace, "guard after", "workspace"),
}


@pytest.mark.parametrize("name", sorted(PLANTED))
def test_planted_stray_write_fails_its_footprint_check(name):
    method, impl, region, detail = PLANTED[name]
    methods = {method: impl}
    if method == "conv_igemm":                  # the emulated conv_gn / conv_res1x1 run the emulated conv_igemm inside
        methods.update({m: _with_plain_conv(m) for m in ("conv_gn", "conv_res1x1")})
    planted = type("Planted", (EmuOps,), methods)()
    proxy = FootprintOps(planted, strict=False)
    boundary_calls(proxy, "cpu")
    with pytest.raises(AssertionError) as e:
        proxy.raise_failures()
    print(f"\nplanted {name}: {str(e.value)[:400]}")
    assert all(f.startswith(method + ":") for f in proxy.failures), proxy.failures
    assert all(region in f for f in proxy.failures), proxy.failures
    assert any(detail in f for f in proxy.failures), proxy.failures
