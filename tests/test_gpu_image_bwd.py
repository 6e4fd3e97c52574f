"""GPU: the image-side training kernels -- GroupNorm/FiLM/SiLU backward, the convolution weight gradient on the tensor cores
and on the CUDA cores, the tensor-core data gradients of Conv2dFn, the fp32 data-gradient kernels and the nearest x2
upsample backward -- against float64 references with elementwise error bounds (tests/fp64_ref.py; tests/test_error_bounds.py
shows on the CPU that the bounds catch subtly wrong kernels).

Every check prints the worst |err| / bound of its case and the rel-L2 beside it.  The model-level gradient tests compare
against unrounded fp32 at 2e-3 to 5e-3, so a defect below that in one group, one tap or one pixel box is only visible here."""
import pytest
import torch

import fp64_ref as R
from fp64_ref import check, check_rel_l2

pytestmark = pytest.mark.gpu
F16, F64 = torch.float16, torch.float64
# whole-tensor rel-L2 limits next to the elementwise bounds: the fp32 conv kernels and the tensor-core data gradient at equal
# operands, the tensor-core weight gradient, GroupNorm backward
REL_CONV, REL_WGRAD_TC, REL_GN = 2e-5, 1e-5, 5e-5


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).cuda()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _rejects(out, ref, bound, what):
    """A defect planted into the native output on the host must fail the check: the bound has teeth at this size."""
    with pytest.raises(AssertionError):
        check(out, ref, bound, "planted: " + what)


def _record_fallbacks(native):
    """Wrap the fp32 fallback kernels of Conv2dFn.backward so that a test sees which of them ran."""
    calls = []
    for name in ("conv_dgrad", "conv_wgrad"):
        orig = getattr(native, name)
        setattr(native, name, lambda *a, _n=name, _o=orig, **k: (calls.append(_n), _o(*a, **k))[1])
    return calls


def _restore(native):
    for name in ("conv_dgrad", "conv_wgrad"):
        delattr(native, name)


# ---------------------------------------------------------------------------------------------- GroupNorm/FiLM/SiLU backward
# (H, W, C): HW = 30 runs one pixel split (Z = 1); the others split the pixel sums (Z > 1: memset + fp32 atomics).
# C = 32 with G = 32 and C = 48 with G = 8 (Cg = 1, 6) take the per-element path of the dx kernel's channel quads.
GN_CASES = [(hw, C) for hw in ((5, 6), (64, 64), (48, 40), (128, 128)) for C in (32, 48, 128, 1024)
            if not (hw == (128, 128) and C == 1024)]


@pytest.mark.parametrize("hw,C", GN_CASES)
def test_gn_silu_bwd(native, hw, C):
    """Every G in {1, 8, 32} dividing C, with and without FiLM; ss / dss rows with ss_ld, dss_ld > 2C (NaN in the gaps:
    ss's must not be read, dss's must not be written); dgamma / dbeta accumulate onto non-zero values; the last group of
    the last image has |mean| / std ~ 100."""
    H, W = hw
    HW = H * W
    B = 4 if HW < 64 else 2
    eps = 1e-5
    Z = R.gn_bwd_splits(B, HW, C, _sms())
    assert (Z == 1) == (HW < 64), Z
    acc_len = R.gn_bwd_acc_len(B, HW, C, _sms())
    x = _rand(B, HW, C, seed=40, scale=2.0) + 0.5
    dy = _rand(B, HW, C, seed=41)
    gamma, beta = _rand(C, seed=42), _rand(C, seed=43)
    dg0, db0 = _rand(C, seed=44), _rand(C, seed=45)
    ss_ld, dss_ld = 2 * C + 24, 2 * C + 40
    ss_buf = torch.full((B, ss_ld), float("nan"), device="cuda")
    ss_buf[:, :2 * C] = _rand(B, 2 * C, seed=46, scale=0.3)
    for G in (1, 8, 32):
        if C % G:
            continue
        Cg = C // G
        xg = x.clone()
        xg[-1, :, C - Cg:] = 100.0 + _rand(HW, Cg, seed=47)
        xd = xg.double().reshape(B, HW, G, Cg)
        sums = torch.stack((xd.sum(dim=(1, 3)), (xd * xd).sum(dim=(1, 3))), dim=-1).contiguous()       # as gn_stats makes them
        for has_ss in (False, True):
            ss = ss_buf if has_ss else None
            dx = torch.full((B, HW, C), float("nan"), device="cuda")
            dg, db = dg0.clone(), db0.clone()
            dss = torch.full((B, dss_ld), float("nan"), device="cuda") if has_ss else None
            native.gn_silu_bwd(xg, dy, sums, B, HW, C, G, gamma, beta, ss, ss_ld if has_ss else 0, eps, dx, dg, db, dss,
                               dss_ld if has_ss else 0)
            torch.cuda.synchronize()
            refs = R.gn_silu_bwd_ref(xg, dy, gamma, beta, ss_buf[:, :2 * C] if has_ss else None, G, eps, dg0, db0, acc_len)
            what = f"gn_silu_bwd B={B} HW={HW} C={C} G={G} ss={has_ss} Z={Z}"
            for name, out, (ref, bound) in zip(("dx", "dgamma", "dbeta"), (dx, dg, db), refs[:3]):
                check(out, ref, bound, f"{what} {name}")
                check_rel_l2(out, ref, REL_GN, f"{what} {name}")
            if has_ss:
                ref_buf = torch.zeros((B, dss_ld), dtype=F64, device="cuda")
                bound_buf = torch.ones((B, dss_ld), dtype=F64, device="cuda")
                sentinel = torch.ones((B, dss_ld), dtype=torch.bool, device="cuda")
                (rs, bs), (rh, bh) = refs[3], refs[4]
                ref_buf[:, :C], ref_buf[:, C:2 * C] = rs, rh
                bound_buf[:, :C], bound_buf[:, C:2 * C] = bs, bh
                sentinel[:, :2 * C] = False
                check(dss, ref_buf, bound_buf, f"{what} dss", sentinel=sentinel)
                check_rel_l2(dss[:, :2 * C], ref_buf[:, :2 * C], REL_GN, f"{what} dss")
                if hw == (128, 128) and G == 32 and C == 128:
                    # the second pixel split of (b, c) = (0, 5) lost from d(shift)
                    chunk = -(-HW // Z)
                    c, g0 = 5, 5 // Cg
                    xs = xd[0, chunk:2 * chunk, g0]
                    mu = xd[0, :, g0].mean()
                    rstd = 1.0 / torch.sqrt(((xd[0, :, g0] - mu) ** 2).mean() + eps)
                    v = ((xs[:, c % Cg] - mu) * rstd * gamma[c].double() + beta[c].double()) * (ss_buf[0, c].double() + 1) \
                        + ss_buf[0, C + c].double()
                    sg = torch.sigmoid(v)
                    d = dss.clone()
                    d[0, C + c] -= float((dy[0, chunk:2 * chunk, c].double() * sg * (1 + v * (1 - sg))).sum())
                    _rejects(d, ref_buf, bound_buf, f"{what}: one pixel split missing from d(shift) of (0, 5)")


# ---------------------------------------------------------------------------------------------- weight gradient, tensor cores
WGRAD_TC_CASES = [
    # stride 1 (the former test_training.py::test_conv_wgrad_tensor_core cases)
    (2, 32, 32, 128, 128, 3, 1), (3, 16, 24, 64, 256, 3, 1), (2, 8, 8, 256, 128, 1, 1), (1, 64, 64, 128, 256, 3, 1),
    (5, 8, 16, 192, 384, 3, 1),
    (2, 128, 128, 128, 128, 1, 1),      # 256 splits of two boxes
    (1, 8, 8, 128, 128, 3, 1),          # one box: one split
    # stride 2, the 4x4 pad-1 Downsample: TMA element-stride boxes, padding row at coordinate -1
    (2, 16, 16, 128, 128, 4, 2), (3, 8, 16, 64, 256, 4, 2), (1, 32, 32, 192, 128, 4, 2), (2, 32, 32, 256, 256, 4, 2),
    (2, 8, 8, 1024, 512, 3, 1),         # the 8x8 level of the cfg-3 U-Net's training step
]


@pytest.mark.parametrize("B,Ho,Wo,cin,cout,k,stride", WGRAD_TC_CASES)
def test_conv_wgrad_tc(native, B, Ho, Wo, cin, cout, k, stride):
    """mi_conv2d_wgrad_f16 (wgmma, MN-major operands, contraction over pixels split over CTAs, split reduction) into a
    NaN-prefilled dW, against the float64 weight gradient of the same fp16 dy / x.  N tiles of 64 (C_in = 64, 192) and 128
    channels, one to three C_out tiles, one split to 256 splits, box counts not divisible by the boxes per split."""
    gen = torch.Generator().manual_seed(B * 1000 + Ho + cin)
    x16 = torch.randn(B, stride * Ho, stride * Wo, cin, generator=gen).cuda().half()
    dy16 = torch.randn(B, Ho, Wo, cout, generator=gen).cuda().half()
    pad = 1 if stride == 2 else k // 2
    assert native.conv_wgrad_tc_supported(Ho, Wo, cin, cout, k, k, stride)
    dw = torch.full((cout, cin, k, k), float("nan"), device="cuda")
    native.conv_wgrad_tc(dy16, x16, B, Ho, Wo, cin, cout, k, k, dw, stride)
    torch.cuda.synchronize()
    per, splits = R.wgrad_tc_plan(B, Ho, Wo, cin, cout, k, _sms())
    ref, bound = R.conv_wgrad_ref(dy16, x16, stride, pad, k, k, R.wgrad_tc_acc_len(B, Ho, Wo, cin, cout, k, _sms()))
    what = f"conv_wgrad_tc B={B} {Ho}x{Wo} {cin}->{cout} k={k} stride={stride} splits={splits} boxes/split={per}"
    check(dw, ref, bound, what)
    check_rel_l2(dw, ref, REL_WGRAD_TC, what)
    last = torch.zeros_like(dy16)
    last[-1, -8:, -8:] = dy16[-1, -8:, -8:]
    _rejects(dw - R.conv_wgrad_ref(last, x16, stride, pad, k, k, 1)[0], ref, bound, what + ": last 8x8 box dropped")


@pytest.mark.parametrize("B,Ho,Wo,cin,cout,k,stride", [(2, 8, 8, 1024, 512, 3, 1), (2, 16, 16, 128, 128, 4, 2)])
def test_conv_wgrad_tc_subnormal_dy(native, B, Ho, Wo, cin, cout, k, stride):
    """dy of the deep levels of a training step is small enough to round to fp16 subnormals (the cfg-3 U-Net's 8x8
    1024 -> 512 conv: |dy| ~ 1e-8).  The wgmma k-group aligns such a product as if its subnormal factor were 2^-14
    (fp64_ref.align_mag), so the error is measured against that; the bound must hold and still see a dropped box."""
    gen = torch.Generator().manual_seed(B * 1000 + Ho + cin + 7)
    x16 = torch.randn(B, stride * Ho, stride * Wo, cin, generator=gen).cuda().half()
    dy16 = (torch.randn(B, Ho, Wo, cout, generator=gen) * 2.0 ** -22).cuda().half()
    sub = (dy16 != 0) & (dy16.abs() < R.FP16_MIN_NORMAL)
    assert sub.float().mean() > 0.85
    pad = 1 if stride == 2 else k // 2
    dw = torch.full((cout, cin, k, k), float("nan"), device="cuda")
    native.conv_wgrad_tc(dy16, x16, B, Ho, Wo, cin, cout, k, k, dw, stride)
    torch.cuda.synchronize()
    ref, bound = R.conv_wgrad_ref(dy16, x16, stride, pad, k, k, R.wgrad_tc_acc_len(B, Ho, Wo, cin, cout, k, _sms()))
    what = f"conv_wgrad_tc subnormal dy B={B} {Ho}x{Wo} {cin}->{cout} k={k} stride={stride}"
    check(dw, ref, bound, what)
    check_rel_l2(dw, ref, REL_WGRAD_TC, what)
    last = torch.zeros_like(dy16)
    last[-1, -8:, -8:] = dy16[-1, -8:, -8:]
    _rejects(dw - R.conv_wgrad_ref(last, x16, stride, pad, k, k, 1)[0], ref, bound, what + ": last 8x8 box dropped")


# ---------------------------------------------------------------------------------------------- data gradients, tensor cores
@pytest.mark.parametrize("B,Hi,Wi,cin,cout,k,stride", [
    (2, 32, 32, 128, 128, 3, 1), (2, 64, 64, 64, 128, 3, 1), (1, 16, 32, 64, 256, 3, 1),
    (2, 32, 32, 128, 128, 4, 2), (3, 16, 32, 64, 256, 4, 2), (1, 64, 64, 128, 256, 4, 2),
])
def test_conv_dgrad_tensor_core(native, B, Hi, Wi, cin, cout, k, stride):
    """Conv2dFn.backward on tensor-core shapes: the 'same' conv's data gradient on the implicit-GEMM kernel with the flipped,
    transposed packed weight, the Downsample's as four sub-pixel 2x2 phases -- no fp32 fallback runs -- against float64 on
    the fp16-rounded dy and weight the kernels read; the weight gradient of the same call against float64 too."""
    from minimagen_b200.autograd import Conv2dFn
    pad = 1 if stride == 2 else k // 2
    gen = torch.Generator().manual_seed(Hi * 100 + cin + k)
    x = torch.randn(B, Hi, Wi, cin, generator=gen).cuda().requires_grad_(True)
    w = (torch.randn(cout, cin, k, k, generator=gen) * 0.05).cuda().requires_grad_(True)
    dy = torch.randn(B, Hi // stride, Wi // stride, cout, generator=gen).cuda()
    calls = _record_fallbacks(native)
    try:
        y = Conv2dFn.apply(x, w, None, stride, pad)
        dx, dw = torch.autograd.grad(y, (x, w), dy)
        torch.cuda.synchronize()
    finally:
        _restore(native)
    assert calls == [], calls
    Ho, Wo = Hi // stride, Wi // stride
    what = f"Conv2dFn tensor-core B={B} {Hi}x{Wi} {cin}->{cout} k={k} stride={stride}"
    ref, bound = R.conv_dgrad_ref(dy.half(), w.detach().half(), stride, pad, Hi, Wi)
    check(dx, ref, bound, what + " dx")
    check_rel_l2(dx, ref, REL_CONV, what + " dx")
    rw, bw = R.conv_wgrad_ref(dy.half(), x.detach().half(), stride, pad, k, k, R.wgrad_tc_acc_len(B, Ho, Wo, cin, cout, k, _sms()))
    check(dw, rw, bw, what + " dW")
    check_rel_l2(dw, rw, REL_WGRAD_TC, what + " dW")
    last = torch.zeros_like(dy)
    last[:, :, -1] = dy[:, :, -1]
    _rejects(dx - R.conv_dgrad_ref(last.half(), w.detach().half(), stride, pad, Hi, Wi)[0], ref, bound,
             what + ": last dy column's contribution dropped")
    if stride == 2:
        d = dx.clone()
        d[0, 0::2, 0::2], d[0, 0::2, 1::2] = dx[0, 0::2, 1::2], dx[0, 0::2, 0::2]
        _rejects(d, ref, bound, what + ": output parities (0, 0) and (0, 1) of image 0 swapped")


@pytest.mark.parametrize("k", [1, 3, 4])
def test_pack_conv_weight_dgrad(native, k):
    """mi_pack_conv_weight_dgrad_f16 is a permute (taps flipped, in / out channels swapped) and one fp16 rounding: bit for bit
    the emulation's flip + transpose + pack, including values that round to subnormals and ties."""
    from emu_ops import EmuOps
    w = _rand(192, 64, k, k, seed=50 + k)
    w[0, :, 0, 0] = torch.tensor([2.0 ** -20, 3 * 2.0 ** -25, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11] * 16, device="cuda")
    got = native.pack_conv_weight_dgrad(w)
    torch.cuda.synchronize()
    exp = EmuOps().pack_conv_weight_dgrad(w.cpu())
    assert got.shape == exp.shape == (64, k * k * 192)
    assert torch.equal(got.cpu().view(torch.int16), exp.view(torch.int16))


# ---------------------------------------------------------------------------------------------- fp32 fallbacks
@pytest.mark.parametrize("k,cout", [(3, 32), (7, 64), (15, 32), (15, 64)])
def test_conv_wgrad_f32_stem(native, k, cout):
    """conv2d_wgrad_f32's flat path (C_in < 32: the (C_in, tap) axis flattened into 32-wide tiles) at the stem's shape:
    6 input channels (image + low-res conditioning image), 64x64, 'same' k x k; dW NaN-prefilled."""
    B, H, W, cin = 2, 64, 64, 6
    x, dy = _rand(B, H, W, cin, seed=60), _rand(B, H, W, cout, seed=61)
    dw = torch.full((cout, cin, k, k), float("nan"), device="cuda")
    native.conv_wgrad(dy, x, B, H, W, cin, H, W, cout, k, k, 1, k // 2, dw)
    torch.cuda.synchronize()
    ppb, splits = R.wgrad_f32_plan(B, H, W, cin, cout, k, k, _sms())
    ref, bound = R.conv_wgrad_ref(dy, x, 1, k // 2, k, k, ppb + splits)
    what = f"conv_wgrad_f32 flat B={B} {H}x{W} {cin}->{cout} k={k} splits={splits}"
    check(dw, ref, bound, what)
    check_rel_l2(dw, ref, REL_CONV, what)
    part = torch.zeros_like(dy)
    part.view(-1, cout)[ppb:2 * ppb] = dy.view(-1, cout)[ppb:2 * ppb]
    d = dw.clone()
    d[:, :, k // 2, k // 2] -= R.conv_wgrad_ref(part, x, 1, k // 2, k, k, 1)[0][:, :, k // 2, k // 2]
    _rejects(d, ref, bound, what + ": the second split missing from the centre tap")


@pytest.mark.parametrize("B,Hi,Wi,cin,cout", [(2, 32, 32, 64, 96), (3, 16, 24, 48, 40)])
def test_conv_gradients_f32_stride2(native, B, Hi, Wi, cin, cout):
    """The 4x4 stride-2 pad-1 conv on the fp32 kernels: conv2d_wgrad_f32's tiled path (one tap per block) and
    conv2d_dgrad_f32's general kernel (C_out > 8), with the stride's parity tests at every border."""
    k, stride, pad = 4, 2, 1
    Ho, Wo = Hi // 2, Wi // 2
    x, dy = _rand(B, Hi, Wi, cin, seed=70), _rand(B, Ho, Wo, cout, seed=71)
    w = _rand(cout, cin, k, k, seed=72, scale=0.1)
    dw = torch.full((cout, cin, k, k), float("nan"), device="cuda")
    dx = torch.full((B, Hi, Wi, cin), float("nan"), device="cuda")
    native.conv_wgrad(dy, x, B, Hi, Wi, cin, Ho, Wo, cout, k, k, stride, pad, dw)
    native.conv_dgrad(dy, B, Ho, Wo, cout, w, cin, k, k, stride, pad, dx, Hi, Wi)
    torch.cuda.synchronize()
    what = f"B={B} {Hi}x{Wi} {cin}->{cout} k=4 stride=2"
    ref, bound = R.conv_wgrad_ref(dy, x, stride, pad, k, k, R.wgrad_f32_acc_len(B, Ho, Wo, cin, cout, k, k, _sms()))
    check(dw, ref, bound, "conv_wgrad_f32 tiled " + what)
    check_rel_l2(dw, ref, REL_CONV, "conv_wgrad_f32 tiled " + what)
    rx, bx = R.conv_dgrad_ref(dy, w, stride, pad, Hi, Wi)
    check(dx, rx, bx, "conv_dgrad_f32 general " + what)
    check_rel_l2(dx, rx, REL_CONV, "conv_dgrad_f32 general " + what)
    wf = w.clone()
    wf[:, 5] = w[:, 5].flip(1, 2)
    d = dx.clone()
    d[..., 5] = R.conv_dgrad_ref(dy, wf, stride, pad, Hi, Wi)[0][..., 5]
    _rejects(d, rx, bx, "conv_dgrad_f32 general " + what + ": taps of channel 5 not flipped")


@pytest.mark.parametrize("B,H,W", [(2, 64, 64), (1, 40, 24)])
def test_final_conv_gradients(native, B, H, W):
    """The U-Net's final conv (3x3, 128 -> 3) through Conv2dFn.backward: the data gradient on conv_dgrad_smallco_kernel
    (C_out <= 8: the weight in shared memory), the weight gradient by the swapped-operand route (conv_wgrad(x, dy, ...) on
    the flat path, then flipped and transposed) -- against float64."""
    from minimagen_b200.autograd import Conv2dFn
    cin, cout, k = 128, 3, 3
    x = _rand(B, H, W, cin, seed=80).requires_grad_(True)
    w = _rand(cout, cin, k, k, seed=81, scale=0.05).requires_grad_(True)
    b = _rand(cout, seed=82).requires_grad_(True)
    dy = _rand(B, H, W, cout, seed=83)
    calls = _record_fallbacks(native)
    try:
        y = Conv2dFn.apply(x, w, b, 1, 1)
        dx, dw = torch.autograd.grad(y, (x, w), dy)
        torch.cuda.synchronize()
    finally:
        _restore(native)
    assert calls == ["conv_dgrad", "conv_wgrad"], calls
    what = f"final conv B={B} {H}x{W} {cin}->{cout}"
    rx, bx = R.conv_dgrad_ref(dy, w.detach(), 1, 1, H, W)
    check(dx, rx, bx, what + " dx (smallco)")
    check_rel_l2(dx, rx, REL_CONV, what + " dx (smallco)")
    # the kernel ran with x and dy swapped: C_in = 3 (flat), C_out = 128
    rw, bw = R.conv_wgrad_ref(dy, x.detach(), 1, 1, k, k, R.wgrad_f32_acc_len(B, H, W, cout, cin, k, k, _sms()))
    check(dw, rw, bw, what + " dW (swapped)")
    check_rel_l2(dw, rw, REL_CONV, what + " dW (swapped)")
    d = dw.clone()
    d[1] = dw[1].flip(1, 2)
    _rejects(d, rw, bw, what + ": dW taps of output channel 1 not flipped back")


# ---------------------------------------------------------------------------------------------- upsample backward
@pytest.mark.parametrize("B,H,W,C", [(2, 32, 32, 64), (3, 5, 7, 64), (2, 33, 17, 3), (1, 64, 64, 3)])
def test_upsample2x_bwd(native, B, H, W, C):
    """mi_upsample2x_bwd: (d00 + d01) + (d10 + d11) in fp32, bit for bit, into a NaN-prefilled dx (ragged H, W: element
    counts that are not a multiple of the block)."""
    dy = _rand(B, 2 * H, 2 * W, C, seed=90, scale=1e3)
    dx = torch.full((B, H, W, C), float("nan"), device="cuda")
    native.upsample2x_bwd(dy, B, H, W, C, dx)
    torch.cuda.synchronize()
    ref = R.upsample2x_bwd_ref(dy)
    n_diff = int((dx != ref).sum())
    print(f"upsample2x_bwd B={B} {H}x{W} C={C}: {n_diff} elements differ from the fixed-order fp32 sum")
    assert n_diff == 0
    q = dy.reshape(B, H, 2, W, 2, C)
    assert not torch.equal((q[:, :, 0, :, 0] + q[:, :, 1, :, 0]) + (q[:, :, 0, :, 1] + q[:, :, 1, :, 1]), ref)
