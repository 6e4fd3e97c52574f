"""GPU: the image-side forward kernels -- the implicit-GEMM convolution in every mode and tile width, its epilogue GroupNorm
statistics, the folded res_conv, the fused GroupNorm conv, the fp32 direct convolution, the tensor-core stem, mi_gn_stats and
mi_gn_apply_silu -- against float64 references with elementwise error bounds (tests/fp64_ref.py; tests/test_error_bounds.py
shows on the CPU that the bounds catch subtly wrong kernels).

Every check prints the worst |err| / bound of its case and the rel-L2 beside it.  The op tests compare these kernels with the
emulation by whole-tensor rel-L2 only, so a wrong halo tap in one tile's border column, a k-block dropped from one tile, one
warp's rows missing from one statistics block or an image's statistics credited to its neighbour is only visible here.
Outputs are NaN-prefilled: every element the kernel should write is checked to be finite, the rest to be still NaN."""
import pytest
import torch

import fp64_ref as R
from emu_ops import EmuOps
from fp64_ref import check, check_rel_l2, half_out
from test_gpu_conv_pingpong import RING_CASES
from test_gpu_conv_tiles import HINTED_CASES
from test_gpu_ops import DIRECT_CASES

pytestmark = pytest.mark.gpu
F16, F32, F64 = torch.float16, torch.float32, torch.float64
NAN = float("nan")
EMU = EmuOps()
# whole-tensor rel-L2 limits next to the elementwise bounds: fp32 conv outputs, fp16 outputs, fp32 GroupNorm outputs
REL_CONV, REL_F16, REL_GN = 2e-5, 1e-3, 5e-6


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).cuda()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _rejects(out, ref, bound, what):
    """A defect planted into the native output on the host must fail the check: the bound has teeth at this size."""
    with pytest.raises(AssertionError):
        check(out, ref, bound, "planted: " + what)


def _nan(*shape, dtype=F32):
    return torch.full(shape, NAN, dtype=dtype, device="cuda")


# ---------------------------------------------------------------------------------------------- implicit-GEMM conv
def _run_conv(native, B, H, W, C0, C1, Cout, k, mode, bias, res, f16, stats, block_n, seed):
    """One conv (modes 2..5: the four phases into one interleaved 2H x 2W output, statistics accumulated over them) into
    NaN-prefilled outputs; checks the fp32 output, the fp16 output and the statistics.  Returns (a0, wp, out, ref, bound,
    stats) for planted defects ((H, W) is the grid of one launch)."""
    Cin = C0 + C1
    lead = (B, 2 * H, 2 * W) if mode == 6 else (B, 4, H, W) if mode == 1 else (B, H, W)
    a0 = _rand(*lead, C0, seed=seed).half()
    a1 = _rand(*lead, C1, seed=seed + 1).half() if C1 else None
    kh = 2 if 2 <= mode <= 5 else k
    w = _rand(Cout, Cin, kh, kh, seed=seed + 2, scale=(kh * kh * Cin) ** -0.5)
    w[:, C0:] *= 0.7071                                       # the skip scale, folded into the packed weight
    b = _rand(Cout, seed=seed + 3) if bias else None
    a = torch.cat((a0, a1), dim=-1) if C1 else a0
    kw = dict(act2=a1, lda2=C1, c_in1=C0) if C1 else {}
    phases = (2, 3, 4, 5) if mode == 2 else (mode,)
    Ho, Wo = (2 * H, 2 * W) if mode == 2 else (H, W)
    r = _rand(B, Ho, Wo, Cout, seed=seed + 4) if res else None
    o = _nan(B, Ho, Wo, Cout)
    o16 = _nan(B, Ho, Wo, Cout, dtype=F16) if f16 else None
    st = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda") if stats else None
    ref = torch.zeros(B, Ho, Wo, Cout, dtype=F64, device="cuda")
    bound = torch.zeros_like(ref)
    for p, m in enumerate(phases):
        wp = EMU.pack_conv_weight(w.cpu() + 0.1 * p if mode == 2 else w.cpu()).cuda()
        if mode == 2:
            off = ((p >> 1) * Wo + (p & 1)) * Cout
            view = lambda t: None if t is None else t.view(-1)[off:]
            native.conv_igemm(a0, B, H, W, C0, 0, Cin, wp, Cout, 2, 2, m, b, None, view(o), view(o16),
                              (Ho * Wo * Cout, 2 * Wo * Cout, 2 * Cout), block_n=block_n, out_stats=st, **kw)
            rr, bb = R.conv_fwd_ref(a, wp, 2, 2, m, b)
            ref[:, p >> 1::2, p & 1::2], bound[:, p >> 1::2, p & 1::2] = rr, bb
        else:
            native.conv_igemm(a0, B, H, W, C0, 0, Cin, wp, Cout, kh, kh, m, b, r, o, o16, (H * W * Cout, W * Cout, Cout),
                              block_n=block_n, out_stats=st, **kw)
            ref, bound = R.conv_fwd_ref(a, wp, kh, kh, m, b, r)
    torch.cuda.synchronize()
    what = f"conv mode {mode} k {kh} B={B} {H}x{W} {C0}+{C1}->{Cout} block_n={block_n}"
    check(o, ref, bound, what)
    check_rel_l2(o, ref, REL_CONV, what)
    if f16:
        check(o16, *half_out(ref, bound), what + " fp16")
        check_rel_l2(o16, ref, REL_F16, what + " fp16")
    if stats:
        check(st, *R.conv_stats_ref(o), what + " statistics")
    return a, wp, o, ref, bound, st


@pytest.mark.parametrize("block_n", [256, 128, 64])
@pytest.mark.parametrize("case", HINTED_CASES)
def test_conv_fwd_hinted(native, case, block_n):
    """Every mode (0 at k = 1 and 3, 1, 2..5, 6), the two-source concat, two images per tile with a batch tail, W > 128, at
    the cooperative 256-wide tile and the 128- and 64-wide ping-pong tiles."""
    B, H, W, C0, C1, Cout, k, mode, bias, res, f16, stats = case
    a, wp, o, ref, bound, st = _run_conv(native, B, H, W, C0, C1, Cout, k, mode, bias, res, f16, stats, block_n, seed=100)
    if case == HINTED_CASES[0]:
        # the second 64-channel k-block of tap (1, 2) missing in the first 128-pixel tile of image 1 (rows 0..7)
        w = R.unpack_conv_weight(wp, 3, 3, C0)
        part = torch.zeros_like(w)
        part[:, 64:128, 1, 2] = w[:, 64:128, 1, 2]
        d = o.clone()
        d[1, :8] -= R.conv_nhwc(a.double(), part, 0)[1, :8].float()
        _rejects(d, ref, bound, f"block_n={block_n}: one k-block of one tap missing in one tile")
        # one warp's 16 rows missing from statistics block 1 of image 0
        sref, sbound = R.conv_stats_ref(o)
        f = o.double().reshape(B, H * W, Cout)[0, 16:32, 16:32]
        d = st.clone()
        d[0, 1, 0] -= f.sum()
        d[0, 1, 1] -= (f * f).sum()
        _rejects(d, sref, sbound, f"block_n={block_n}: one warp's 16 rows missing from one statistics block")
    if mode == 2:
        d = o.clone()
        d[0, 0::2, 1::2], d[0, 1::2, 0::2] = o[0, 1::2, 0::2], o[0, 0::2, 1::2]
        _rejects(d, ref, bound, f"block_n={block_n}: sub-pixel phases (0, 1) and (1, 0) of image 0 swapped")


@pytest.mark.parametrize("name", list(RING_CASES))
def test_conv_fwd_ring(native, name):
    """The ping-pong ring and tile bookkeeping: fewer k-blocks than stages, k-blocks not a multiple of the stage count, one
    to five tiles per CTA, two images per tile."""
    B, H, W, Cin, Cout, k, block_n = RING_CASES[name](_sms())
    _run_conv(native, B, H, W, Cin, 0, Cout, k, 0, True, True, True, True, block_n, seed=600)


# B, H, W, C0, C1, C_out, k, statistics
SHAPE_CASES = {
    "block_n_32": (2, 16, 16, 64, 0, 32, 3, True),          # C_out = 32 selects the 32-wide tile
    "block_n_16": (2, 16, 16, 64, 0, 48, 3, False),         # C_out = 48: the 16-wide tile
    "ragged_w_136": (3, 4, 136, 64, 0, 128, 3, True),       # two 128-pixel tiles per row, the second 8 columns wide
    "ragged_w_520": (2, 1, 520, 128, 0, 256, 1, False),
    "two_images_per_tile": (5, 8, 8, 64, 0, 128, 3, True),
    "four_images_per_tile": (7, 4, 8, 64, 0, 128, 3, True),
    "eight_images_per_tile": (13, 2, 8, 64, 0, 128, 3, False),
    "deep_k": (2, 16, 16, 1024, 0, 512, 3, True),
    "concat_3x3": (2, 16, 16, 128, 64, 128, 3, True),
    "concat_1x1": (2, 16, 16, 128, 64, 128, 1, True),
}


@pytest.mark.parametrize("name", list(SHAPE_CASES))
def test_conv_fwd_shapes(native, name):
    B, H, W, C0, C1, Cout, k, stats = SHAPE_CASES[name]
    a, wp, o, ref, bound, st = _run_conv(native, B, H, W, C0, C1, Cout, k, 0, True, True, True, stats, 0, seed=200)
    if name == "ragged_w_136":
        # the masked columns 136..255 of every row's second tile counted with their bias value (the accumulator is 0)
        sref, sbound = R.conv_stats_ref(o)
        bias = _rand(Cout, seed=203).double().reshape(-1, 16)
        d = st.clone()
        d[..., 0] += (256 - W) * H * bias.sum(dim=1)
        d[..., 1] += (256 - W) * H * (bias * bias).sum(dim=1)
        _rejects(d, sref, sbound, name + ": masked ragged-W rows counted")
    if name == "four_images_per_tile":
        # the statistics of image 0 credited to image 1 (a tile holds images 0..3)
        sref, sbound = R.conv_stats_ref(o)
        d = st.clone()
        d[1] += st[0]
        d[0] = 0
        _rejects(d, sref, sbound, name + ": image 0's statistics credited to image 1")


def test_conv_fwd_strided_io(native):
    """A channel-offset input; a channel-slice output between NaN sentinels; an output pointer that is not 8-byte aligned
    (the scalar epilogue), with a residual holding a few +-1e5 elements: the fp32 output stays inside its bound and the fp16
    output saturates to +-65504."""
    B, H, W, lda, c_off, Cin, Cout = 2, 16, 16, 192, 64, 128, 64
    act = _rand(B, H, W, lda, seed=5).half()
    w = _rand(Cout, Cin, 3, 3, seed=6, scale=(9 * Cin) ** -0.5)
    wp = EMU.pack_conv_weight(w.cpu()).cuda()
    bias = _rand(Cout, seed=7)
    ref, bound = R.conv_fwd_ref(act[..., c_off:c_off + Cin], wp, 3, 3, 0, bias)
    # channel slice [32, 96) of a 160-channel buffer
    ldo = 160
    buf = _nan(B, H, W, ldo)
    native.conv_igemm(act, B, H, W, lda, c_off, Cin, wp, Cout, 3, 3, 0, bias, None, buf[..., 32:32 + Cout], None,
                      (H * W * ldo, W * ldo, ldo))
    torch.cuda.synchronize()
    sentinel = torch.ones(B, H, W, ldo, dtype=torch.bool, device="cuda")
    sentinel[..., 32:32 + Cout] = False
    rbuf, bbuf = torch.zeros(B, H, W, ldo, dtype=F64, device="cuda"), torch.ones(B, H, W, ldo, dtype=F64, device="cuda")
    rbuf[..., 32:32 + Cout], bbuf[..., 32:32 + Cout] = ref, bound
    check(buf, rbuf, bbuf, "conv channel-offset input, channel-slice output", sentinel=sentinel)
    check_rel_l2(buf[..., 32:32 + Cout], ref, REL_CONV, "conv channel-offset input, channel-slice output")
    # output, fp16 output and residual at channel 1 of a (C_out + 4)-channel row: 4- and 2-byte aligned only
    ldo = Cout + 4
    res_buf = _rand(B, H, W, ldo, seed=8)
    res = res_buf[..., 1:1 + Cout]
    res[0, 3, 5, :4] = torch.tensor([1e5, -1e5, 7e4, -7e4], device="cuda")
    ref, bound = R.conv_fwd_ref(act[..., c_off:c_off + Cin], wp, 3, 3, 0, bias, res)
    buf, buf16 = _nan(B, H, W, ldo), _nan(B, H, W, ldo, dtype=F16)
    st = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda")
    o, o16 = buf[..., 1:1 + Cout], buf16[..., 1:1 + Cout]
    assert o.data_ptr() % 8 == 4 and o16.data_ptr() % 4 == 2
    native.conv_igemm(act, B, H, W, lda, c_off, Cin, wp, Cout, 3, 3, 0, bias, res, o, o16, (H * W * ldo, W * ldo, ldo),
                      out_stats=st)
    torch.cuda.synchronize()
    sentinel = torch.ones(B, H, W, ldo, dtype=torch.bool, device="cuda")
    sentinel[..., 1:1 + Cout] = False
    rbuf, bbuf = torch.zeros(B, H, W, ldo, dtype=F64, device="cuda"), torch.ones(B, H, W, ldo, dtype=F64, device="cuda")
    rbuf[..., 1:1 + Cout], bbuf[..., 1:1 + Cout] = ref, bound
    check(buf, rbuf, bbuf, "conv unaligned output (scalar epilogue)", sentinel=sentinel)
    check_rel_l2(o, ref, REL_CONV, "conv unaligned output (scalar epilogue)")
    r16, b16 = half_out(rbuf, bbuf)
    check(buf16, r16, b16, "conv unaligned fp16 output (scalar epilogue)", sentinel=sentinel)
    assert torch.equal(o16[0, 3, 5, :4].float().cpu(), torch.tensor([65504.0, -65504.0, 65504.0, -65504.0]))
    check(st, *R.conv_stats_ref(o), "conv unaligned output statistics")
    d = o.clone()
    d[1] = d[1] - bias + bias.roll(16)
    _rejects(d, ref, bound, "bias shifted by one 16-channel block in image 1")


def test_conv_fwd_nchw_final(native):
    """The final conv: C_out = 3 zero-padded to 16 in the packed weight, stored NCHW with n_valid = 3 into a 16-plane
    buffer: planes 3..15 must stay NaN."""
    B, H, W, Cin, Cout = 2, 32, 32, 128, 3
    act = _rand(B, H, W, Cin, seed=41).half()
    w = _rand(Cout, Cin, 3, 3, seed=42, scale=0.03)
    bias = torch.zeros(16, device="cuda")
    bias[:Cout] = _rand(Cout, seed=43)
    wp = torch.zeros(16, 9 * Cin, dtype=F16, device="cuda")
    wp[:Cout] = EMU.pack_conv_weight(w.cpu()).cuda()
    buf = _nan(B, 16, H, W)
    native.conv_igemm(act, B, H, W, Cin, 0, Cin, wp, 16, 3, 3, 0, bias, None, buf, None, (16 * H * W, W, 1), out_sc=H * W,
                      n_valid=Cout)
    torch.cuda.synchronize()
    ref, bound = R.conv_fwd_ref(act, wp, 3, 3, 0, bias)
    sentinel = torch.ones(B, 16, H, W, dtype=torch.bool, device="cuda")
    sentinel[:, :Cout] = False
    rbuf, bbuf = ref.permute(0, 3, 1, 2).contiguous(), bound.permute(0, 3, 1, 2).contiguous()
    check(buf, rbuf, bbuf, "final conv NCHW n_valid=3", sentinel=sentinel)
    check_rel_l2(buf[:, :Cout], rbuf[:, :Cout], REL_CONV, "final conv NCHW n_valid=3")


@pytest.mark.parametrize("tile", [128, 256])
def test_conv_res1x1(native, tile):
    """mi_conv3x3_res1x1_f16 (3x3 + folded 1x1 over a virtual concat x) at the 128-wide ping-pong and the auto-selected
    256-wide cooperative tile."""
    if tile == 128:
        B, H, W, Cin, Cout, Cx0, Cx1 = _sms() // 4 + 1, 32, 32, 128, 128, 64, 128
    else:
        B, H, W, Cin, Cout, Cx0, Cx1 = -(-_sms() // 8), 32, 32, 64, 256, 64, 64
    Cx = Cx0 + Cx1
    assert native.conv_res1x1_supported(H, W, Cin, Cout, Cx)
    a = _rand(B, H, W, Cin, seed=801).half()
    x0, x1 = _rand(B, H, W, Cx0, seed=802).half(), _rand(B, H, W, Cx1, seed=803).half()
    w3 = _rand(Cout, Cin, 3, 3, seed=804, scale=(9 * Cin) ** -0.5)
    w1 = _rand(Cout, Cx, 1, 1, seed=805, scale=Cx ** -0.5)
    bias, r = _rand(Cout, seed=806), _rand(B, H, W, Cout, seed=807)
    wp = torch.cat((EMU.pack_conv_weight(w3.cpu()), EMU.pack_conv_weight(w1.cpu())), dim=1).contiguous().cuda()
    o, o16 = _nan(B, H, W, Cout), _nan(B, H, W, Cout, dtype=F16)
    st = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda")
    native.conv_res1x1(a, B, H, W, Cin, Cin, None, 0, 0, x0, Cx0, Cx, x1, Cx1, Cx0, wp, Cout, bias, r, o, o16, st)
    torch.cuda.synchronize()
    ref, bound = R.conv_fwd_ref(a, wp, 3, 3, 0, bias, r, x=torch.cat((x0, x1), dim=-1))
    what = f"conv res1x1 B={B} {Cin}+{Cx}->{Cout}"
    check(o, ref, bound, what)
    check_rel_l2(o, ref, REL_CONV, what)
    check(o16, *half_out(ref, bound), what + " fp16")
    check_rel_l2(o16, ref, REL_F16, what + " fp16")
    check(st, *R.conv_stats_ref(o), what + " statistics")
    d = o.clone()
    d[-1] -= (x1[-1].double() @ wp[:, 9 * Cin + Cx0:].double().t()).float()
    _rejects(d, ref, bound, what + ": the second x source dropped in the last image")


# ---------------------------------------------------------------------------------------------- fused GroupNorm conv
@pytest.mark.parametrize("B,H,W,C0,C1,Cout,res,ss", [
    (2, 32, 16, 128, 0, 128, False, False), (2, 32, 16, 256, 128, 256, True, True), (3, 32, 8, 128, 128, 128, True, True),
    (1, 64, 64, 128, 0, 256, False, True), (2, 32, 16, 128, 256, 128, True, True), (1, 32, 32, 512, 512, 512, True, True),
    (5, 64, 32, 128, 0, 128, True, False), (2, 64, 32, 256, 0, 256, True, True), (3, 32, 8, 128, 128, 512, False, True),
    (1, 32, 32, 512, 512, 1024, True, True),
])
def test_conv_gn(native, B, H, W, C0, C1, Cout, res, ss):
    """mi_conv3x3_gn_silu_f16 against GroupNorm -> FiLM -> SiLU -> 3x3 conv in float64 (conv_gn_ref) from the same block
    statistics; the epilogue statistics against the kernel's own output."""
    G, C = 8, C0 + C1
    assert native.conv_gn_supported(H, W, C0, C1, Cout, G)
    x0 = _rand(B, H, W, C0, seed=80) * 1.5 + 0.3
    x1 = _rand(B, H, W, C1, seed=81) if C1 else None
    gamma, beta = _rand(C, seed=82), _rand(C, seed=83)
    ssv = _rand(B, 2 * C, seed=84, scale=0.3) if ss else None
    w = _rand(Cout, C, 3, 3, seed=85, scale=(9 * C) ** -0.5)
    bias = _rand(Cout, seed=86)
    r = _rand(B, H, W, Cout, seed=87) if res else None
    wp = EMU.pack_conv_weight(w.cpu()).cuda()

    def blockstats(t):
        tb = t.double().reshape(B, H * W, -1, 16)
        return torch.stack((tb.sum(dim=(1, 3)), (tb * tb).sum(dim=(1, 3))), dim=-1).contiguous()
    st0, st1 = blockstats(x0), (blockstats(x1) if C1 else None)
    o, o16 = _nan(B, H, W, Cout), _nan(B, 1, H, W, Cout, dtype=F16)
    ost = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda")
    native.conv_gn(x0, C0, x1, C1, 0.7071, B, H, W, G, st0, st1, gamma, beta, ssv, 2 * C, 1e-5, wp, Cout, bias, r, o, o16,
                   ost)
    torch.cuda.synchronize()
    sums = R.group_sums(st0, C0, G, st1, C1, 0.7071)
    ref, bound = R.conv_gn_ref(x0, G, gamma, beta, ssv, 1e-5, sums, wp, bias, r, src1=x1, scale1=0.7071)
    what = f"conv_gn B={B} {H}x{W} {C0}+{C1}->{Cout}"
    check(o, ref, bound, what)
    check_rel_l2(o, ref, 5e-4, what)                   # the fp16 rounding of the activated operand can flip one ulp
    check(o16.reshape(B, H, W, Cout), *half_out(ref, bound), what + " fp16")
    check_rel_l2(o16.reshape(B, H, W, Cout), ref, 1.5e-3, what + " fp16")
    check(ost, *R.conv_stats_ref(o), what + " statistics")
    if ss and B == 2 and C1 == 128:
        ss2 = ssv.clone()
        ss2[0, :C] -= 1.0
        d = o.clone()
        d[0] = R.conv_gn_ref(x0, G, gamma, beta, ss2, 1e-5, sums, wp, bias, r, src1=x1, scale1=0.7071)[0][0].float()
        _rejects(d, ref, bound, what + ": FiLM scale without +1 in image 0")


# ---------------------------------------------------------------------------------------------- fp32 direct conv, stem
@pytest.mark.parametrize("case", DIRECT_CASES)
def test_conv_direct(native, case):
    """mi_conv2d_direct_f32: an fma chain over taps x ceil4(C_in), the conv_fwd_ref form with fp32 operands."""
    B, Hin, Win, Cin, ldi, Cout, k, stride, pad, residual, nchw = case
    Hout, Wout = (Hin + 2 * pad - k) // stride + 1, (Win + 2 * pad - k) // stride + 1
    assert (stride == 1 and pad == k // 2) or (stride == 2 and k == 4 and pad == 1)
    x = torch.zeros(B, Hin, Win, ldi, device="cuda")
    x[..., :Cin] = _rand(B, Hin, Win, Cin, seed=7)
    w = _rand(Cout, Cin, k, k, seed=8, scale=(k * k * Cin) ** -0.5)
    b = _rand(Cout, seed=9)
    if nchw:
        shape, strides = (B, Cout, Hout, Wout), (Cout * Hout * Wout, Wout, 1, Hout * Wout)
    else:
        shape, strides = (B, Hout, Wout, Cout), (Hout * Wout * Cout, Wout * Cout, Cout, 1)
    r = _rand(*shape, seed=10) if residual else None
    o = _nan(*shape)
    native.conv_direct(x, B, Hin, Win, Cin, ldi, w, Cout, k, k, stride, pad, b, r, o, Hout, Wout, strides)
    torch.cuda.synchronize()
    wpad = torch.zeros(Cout, ldi, k, k, device="cuda")
    wpad[:, :Cin] = w
    wp = wpad.permute(0, 2, 3, 1).reshape(Cout, -1)            # fp32, packed like the tensor-core weight
    nhwc = (lambda t: t.permute(0, 2, 3, 1)) if nchw else (lambda t: t)
    ref, bound = R.conv_fwd_ref(x, wp, k, k, 6 if stride == 2 else 0, b, None if r is None else nhwc(r))
    what = f"conv_direct B={B} {Hin}x{Win} {Cin}->{Cout} k={k} stride={stride}"
    check(nhwc(o), ref, bound, what)
    check_rel_l2(nhwc(o), ref, REL_CONV, what)
    d = nhwc(o).clone()
    d[..., 0] -= R.conv_nhwc(x[..., Cin - 1:Cin].double(), w[:1, Cin - 1:Cin].double(), 6 if stride == 2 else 0)[..., 0].float()
    _rejects(d, ref, bound, what + ": last input channel dropped in output channel 0")


@pytest.mark.parametrize("Ca,Cb,dim", [(3, 3, 128), (3, 0, 64)])
def test_stem(native, Ca, Cb, dim):
    """CrossEmbedLayer.run_stem on the tensor cores (stem_unroll, then the 15-tap GEMM over 128 unrolled channels, n = 15 x
    128) against the float64 k = 3 / 7 / 15 convs of its fp16 operands; the fp16 copy and the epilogue statistics."""
    from minimagen_b200.layers import CrossEmbedLayer
    B, H, W = 2, 32, 32
    x, lr = _rand(B, Ca, H, W, seed=44), (_rand(B, Cb, H, W, seed=45) if Cb else None)
    torch.manual_seed(0)
    layer = CrossEmbedLayer(Ca + Cb, (3, 7, 15), dim_out=dim, stride=1).cuda()
    assert layer.stem_tc_ok(H, W)
    with torch.no_grad():
        out = layer.run_stem(x, lr)
        torch.cuda.synchronize()
        a = torch.empty(B, H, W, 128, dtype=F16, device="cuda")
        native.stem_unroll(x, Ca, lr, Cb, B, H, W, a)
        wp, bias = layer._stem_weights()
        ref, bound = R.conv_fwd_ref(a, wp, 15, 1, 0, bias)
        xin = (torch.cat((x, lr), dim=1) if Cb else x).half().double()
        direct = torch.cat([torch.nn.functional.conv2d(xin, c.weight.half().double(), c.bias.double(), padding=c.padding)
                            for c in layer.convs], dim=1).permute(0, 2, 3, 1)
    assert float((direct - ref).abs().max()) <= 1e-9 * float(ref.abs().max())      # the unrolled GEMM is the three convs
    what = f"stem {Ca}+{Cb}->{dim}"
    check(out.f32, direct, bound, what)
    check_rel_l2(out.f32, direct, REL_CONV, what)
    check(out.f16.reshape(B, H, W, dim), *half_out(direct, bound), what + " fp16")
    check(out.stats, *R.conv_stats_ref(out.f32), what + " statistics")
    # the top row of the 15 x 15 window (tap 0 of the k = 15 conv) dropped
    c15 = layer.convs[-1]
    w0 = torch.zeros_like(c15.weight)
    w0[:, :, 0] = c15.weight[:, :, 0]
    d = out.f32.clone()
    d[..., dim - c15.out_channels:] -= torch.nn.functional.conv2d(xin, w0.half().double(), padding=7).permute(0, 2, 3, 1).float()
    _rejects(d, direct, bound, what + ": tap row 0 of the 15-tap GEMM dropped")


# ---------------------------------------------------------------------------------------------- GroupNorm statistics
# B, HW, C0, C1, groups, fp16 input: Cg = 3, 6, 1, 16, 48 (the concat), C = 4096 (one plane per thread); HW is not a
# multiple of the chunk except where noted
GN_STATS_CASES = [(2, 1000, 48, 0, 16, False), (2, 1000, 48, 0, 8, True), (2, 256, 32, 0, 32, False),
                  (2, 500, 128, 0, 8, True), (2, 1024, 256, 128, 8, False), (2, 1024, 256, 128, 8, True),
                  (1, 300, 4096, 0, 32, False)]


@pytest.mark.parametrize("B,HW,C0,C1,groups,in16", GN_STATS_CASES)
def test_gn_stats(native, B, HW, C0, C1, groups, in16):
    C = C0 + C1
    dt = F16 if in16 else F32
    s0 = (_rand(B, HW, C0, seed=11) * 2 + 0.5).to(dt)
    s1 = _rand(B, HW, C1, seed=12).to(dt) if C1 else None
    scale1 = 0.7071 if C1 else 1.0
    sums = torch.zeros(B, groups, 2, dtype=F64, device="cuda")
    native.gn_stats(s0, C0, s1, C1, scale1, B, HW, groups, sums)
    torch.cuda.synchronize()
    chunk, planes, L = R.gn_stats_plan(C, HW)
    ref, bound = R.gn_stats_ref(s0, groups, s1, scale1, L)
    what = f"gn_stats B={B} HW={HW} C={C0}+{C1} G={groups} fp16={in16} chunk={chunk} planes={planes}"
    check(sums, ref, bound, what)
    check_rel_l2(sums, ref, 1e-6, what)
    if HW > chunk:
        lost = R.gn_stats_ref(s0[:, chunk:2 * chunk], groups, None if s1 is None else s1[:, chunk:2 * chunk], scale1)[0]
        _rejects(sums - lost, ref, bound, what + ": the second chunk lost")


# ---------------------------------------------------------------------------------------------- GroupNorm apply
def _gn_apply_inputs(in16):
    """Concat of 96 + 48 channels, G = 8 (Cg = 18: groups straddle the sources and the 8-channel vectors); image 0 group 2
    near-constant (std << sqrt(eps)), image 1 group 6 at |mean| / std ~ 100; gamma = 3e4 in channel 126 drives v beyond
    65504 and below -88; HW = 1000 is not a multiple of the pixels per CTA."""
    B, HW, C0, C1, G = 2, 1000, 96, 48, 8
    C = C0 + C1
    dt = F16 if in16 else F32
    s0 = _rand(B, HW, C0, seed=21) * 2 + 0.5
    s1 = _rand(B, HW, C1, seed=22)
    s0[0, :, 36:54] = 2.5 + 1e-4 * _rand(HW, 18, seed=23)
    s1[1, :, 12:30] = 100.0 / 0.7071 + _rand(HW, 18, seed=24)
    gamma, beta = _rand(C, seed=25), _rand(C, seed=26)
    gamma[126] = 3e4
    return B, HW, C0, C1, G, C, s0.to(dt), s1.to(dt), gamma, beta


@pytest.mark.parametrize("film", [True, False])
@pytest.mark.parametrize("in16,out16", [(False, False), (False, True), (True, False), (True, True)])
def test_gn_apply_silu(native, in16, out16, film):
    """mi_gn_apply_silu with global statistics: (a) given the exact float64 statistics, (b) end to end from mi_gn_stats.
    FiLM rows with ss_ld > 2C and NaN gaps (must not be read)."""
    B, HW, C0, C1, G, C, s0, s1, gamma, beta = _gn_apply_inputs(in16)
    ss_ld = 2 * C + 24
    ss_buf = _nan(B, ss_ld)
    ss_buf[:, :2 * C] = _rand(B, 2 * C, seed=27, scale=0.3)
    ss = ss_buf[:, :2 * C] if film else None
    exact, err = R.gn_stats_ref(s0, G, s1, 0.7071)
    kst = torch.zeros(B, G, 2, dtype=F64, device="cuda")
    native.gn_stats(s0, C0, s1, C1, 0.7071, B, HW, G, kst)
    for form, stats, sums_err in (("a", exact, None), ("b", kst, err)):
        out = _nan(B, HW, C, dtype=F16 if out16 else F32)
        native.gn_apply_silu(s0, C0, s1, C1, 0.7071, B, HW, G, stats, 0, None, 0, gamma, beta, ss_buf if film else None,
                             ss_ld if film else 0, 1e-5, out)
        torch.cuda.synchronize()
        ref, bound = R.gn_apply_silu_ref(s0, G, gamma, beta, ss, 1e-5, exact, sums_err, src1=s1, scale1=0.7071, out16=out16)
        what = f"gn_apply_silu ({form}) in16={in16} out16={out16} film={film}"
        check(out, ref, bound, what)
        check(out[1, :, 108:126], ref[1, :, 108:126], bound[1, :, 108:126], what + " the |mean|/std ~ 100 group")
        check(out[0, :, 36:54], ref[0, :, 36:54], bound[0, :, 36:54], what + " the near-constant group")
        agg = torch.ones(B, HW, C, dtype=torch.bool, device="cuda")
        agg[..., 126], agg[0, :, 36:54], agg[1, :, 108:126] = False, False, False
        check_rel_l2(out[agg], ref[agg], REL_F16 if out16 else REL_GN, what)
        if out16:
            assert float(out[..., 126].float().abs().max()) == 65504.0
        if form == "a" and film:
            # image 1, group 3 normalised with group 4's mean
            wrong = exact.clone()
            wrong[1, 3, 0] = exact[1, 4, 0]
            wrong[1, 3, 1] = exact[1, 3, 1] - exact[1, 3, 0] ** 2 / (18 * HW) + exact[1, 4, 0] ** 2 / (18 * HW)
            d = out.clone()
            d[1, :, 54:72] = R.gn_apply_silu_ref(s0, G, gamma, beta, ss, 1e-5, wrong, src1=s1, scale1=0.7071,
                                                 out16=out16)[0][1, :, 54:72].to(out.dtype)
            _rejects(d, ref, bound, what + ": the neighbouring group's mean in image 1, group 3")


@pytest.mark.parametrize("out16", [True, False])
def test_gn_apply_silu_conv_block_stats(native, out16):
    """(b) with per-source block statistics written by two conv epilogues (C0 = 256, C1 = 128, G = 8: groups of 48 channels
    straddle the sources) over their fp16 outputs: the reference normalises with the exact statistics of the convs' fp32
    outputs, and conv_stats_ref bounds the epilogues' error."""
    B, H, W, Cin = 2, 16, 16, 64
    C0, C1, G = 256, 128, 8
    srcs = []
    for i, Cout in enumerate((C0, C1)):
        act = _rand(B, H, W, Cin, seed=50 + i).half()
        wp = EMU.pack_conv_weight(_rand(Cout, Cin, 3, 3, seed=52 + i, scale=0.05).cpu()).cuda()
        o16 = torch.empty(B, H, W, Cout, dtype=F16, device="cuda")
        o32 = torch.empty(B, H, W, Cout, device="cuda")
        st = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda")
        native.conv_igemm(act, B, H, W, Cin, 0, Cin, wp, Cout, 3, 3, 0, None, None, o32, o16, (H * W * Cout, W * Cout, Cout),
                          out_stats=st)
        srcs.append((o32, o16, st))
    gamma, beta = _rand(C0 + C1, seed=60), _rand(C0 + C1, seed=61)
    ss = _rand(B, 2 * (C0 + C1), seed=62, scale=0.3)
    out = _nan(B, H * W, C0 + C1, dtype=F16 if out16 else F32)
    native.gn_apply_silu(srcs[0][1], C0, srcs[1][1], C1, 0.7071, B, H * W, G, srcs[0][2], 16, srcs[1][2], 16, gamma, beta,
                         ss, 2 * (C0 + C1), 1e-5, out)
    torch.cuda.synchronize()
    (r0, e0), (r1, e1) = R.conv_stats_ref(srcs[0][0]), R.conv_stats_ref(srcs[1][0])
    sums = R.group_sums(r0, C0, G, r1, C1, 0.7071)
    sums_err = R.group_sums(e0, C0, G, e1, C1, 0.7071)
    flat = lambda t: t.reshape(B, H * W, -1)
    ref, bound = R.gn_apply_silu_ref(flat(srcs[0][1]), G, gamma, beta, ss, 1e-5, sums, sums_err, src1=flat(srcs[1][1]),
                                     scale1=0.7071, out16=out16)
    what = f"gn_apply_silu (b) conv block statistics out16={out16}"
    check(out, ref, bound, what)
    check_rel_l2(out, ref, REL_F16 if out16 else REL_GN, what)
    # the second source's block statistics gathered without scale1 (groups 5..7, channels 240..383, include them)
    wrong = R.group_sums(r0, C0, G, r1, C1, 1.0)
    d = out.clone()
    d[..., 240:] = R.gn_apply_silu_ref(flat(srcs[0][1]), G, gamma, beta, ss, 1e-5, wrong, src1=flat(srcs[1][1]),
                                       scale1=0.7071, out16=out16)[0][..., 240:].to(out.dtype)
    _rejects(d, ref, bound, what + ": block statistics of the second source unscaled")
