"""GPU parity, op by op, through the C ABI: every native kernel vs the torch restatement of its contract
(tests/emu_ops.py) on identical seeded inputs.  Integer / index work (quantile order statistics, timestep gathers) is
checked bit-exactly; floating point within the stated tolerances."""
import pytest
import torch

from conftest import rel_l2
from emu_ops import EmuOps

pytestmark = pytest.mark.gpu
F16, F32, F64 = torch.float16, torch.float32, torch.float64
EMU = EmuOps()


def _cu(t):
    return None if t is None else t.cuda()


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed + sum(shape))
    return torch.randn(*shape, generator=g) * scale


# ---------------------------------------------------------------------------------------------- conv (tensor cores)
IGEMM_CASES = [
    # B, H, W, Cin, Cout, k, mode, bias, residual, f16out
    (2, 16, 16, 64, 128, 3, 0, True, True, False),
    (1, 32, 32, 128, 64, 3, 0, True, False, True),
    (3, 8, 8, 64, 64, 3, 0, False, True, False),       # tile spans two images + batch tail
    (1, 64, 64, 64, 16, 3, 0, True, False, False),     # narrow N
    (2, 16, 16, 256, 256, 1, 0, True, True, False),    # 1x1
    (2, 16, 16, 64, 128, 4, 1, True, False, False),    # Downsample 4x4 s2 via phase split
    (1, 4, 256, 64, 64, 3, 0, True, False, False),     # W > 128
    (1, 1, 520, 128, 1024, 1, 0, False, False, True),  # GEMM with ragged M (8320-like token rows)
    (2, 16, 16, 1024, 512, 3, 0, True, True, False),   # deep K, 2 N tiles
]


@pytest.mark.parametrize("case", IGEMM_CASES)
def test_conv_igemm(native, case):
    B, H, W, Cin, Cout, k, mode, bias, residual, f16out = case
    assert native.igemm_supported(H, W, Cin, Cout)
    P = 4 if mode == 1 else 1
    act = _rand(B, P, H, W, Cin, seed=1).to(F16)
    w = _rand(Cout, Cin, k, k, seed=2, scale=(k * k * Cin) ** -0.5)
    b = _rand(Cout, seed=3) if bias else None
    r = _rand(B, H, W, Cout, seed=4) if residual else None
    strides = (H * W * Cout, W * Cout, Cout)
    wp_e = EMU.pack_conv_weight(w)
    wp_n = native.pack_conv_weight(w.cuda())
    assert torch.equal(wp_n.cpu(), wp_e)
    o_e = torch.zeros(B, H, W, Cout)
    o16_e = torch.zeros(B, H, W, Cout, dtype=F16) if f16out else None
    EMU.conv_igemm(act, B, H, W, Cin, 0, Cin, wp_e, Cout, k, k, mode, b, r, o_e, o16_e, strides)
    o_n = torch.full((B, H, W, Cout), float("nan"), device="cuda")
    o16_n = torch.zeros(B, H, W, Cout, dtype=F16, device="cuda") if f16out else None
    native.conv_igemm(act.cuda(), B, H, W, Cin, 0, Cin, wp_n, Cout, k, k, mode, _cu(b), _cu(r), o_n, o16_n, strides)
    torch.cuda.synchronize()
    assert rel_l2(o_n, o_e) < 2e-5          # same fp16 operands, fp32 accumulation order differs
    if f16out:
        assert rel_l2(o16_n, o_e) < 1e-3


def test_conv_igemm_channel_offset_and_strided_output(native):
    """operand = a channel slice of a wider buffer; result written into a channel slice of a wider NHWC buffer"""
    B, H, W, lda, c_off, Cin, Cout, ldo = 1, 16, 16, 192, 64, 128, 64, 160
    act = _rand(B, 1, H, W, lda, seed=5).to(F16)
    w = _rand(Cout, Cin, 3, 3, seed=6, scale=0.03)
    wp = EMU.pack_conv_weight(w)
    strides = (H * W * ldo, W * ldo, ldo)
    o_e = torch.zeros(B, H, W, ldo)
    EMU.conv_igemm(act, B, H, W, lda, c_off, Cin, wp, Cout, 3, 3, 0, None, None, o_e[..., 32:], None, strides)
    o_n = torch.zeros(B, H, W, ldo, device="cuda")
    native.conv_igemm(act.cuda(), B, H, W, lda, c_off, Cin, wp.cuda(), Cout, 3, 3, 0, None, None, o_n[..., 32:], None,
                      strides)
    assert rel_l2(o_n, o_e) < 2e-5
    assert torch.count_nonzero(o_n[..., :32]) == 0 and torch.count_nonzero(o_n[..., 96:]) == 0


def test_conv_igemm_nchw_ragged_n(native):
    """final_conv: C_out = 3 zero-padded to 16 in the packed weight, stored NCHW with n_valid = 3"""
    B, H, W, Cin, Cout = 2, 32, 32, 128, 3
    act = _rand(B, 1, H, W, Cin, seed=41).to(F16)
    w = _rand(Cout, Cin, 3, 3, seed=42, scale=0.03)
    b = torch.zeros(16)
    b[:Cout] = _rand(Cout, seed=43)
    wp = torch.zeros(16, 9 * Cin, dtype=F16)
    wp[:Cout] = EMU.pack_conv_weight(w)
    strides = (Cout * H * W, W, 1)
    o_e = torch.zeros(B, Cout, H, W)
    EMU.conv_igemm(act, B, H, W, Cin, 0, Cin, wp, 16, 3, 3, 0, b, None, o_e, None, strides, out_sc=H * W, n_valid=Cout)
    ref = torch.nn.functional.conv2d(act[:, 0].float().permute(0, 3, 1, 2), w.half().float(), b[:Cout], padding=1)
    assert rel_l2(o_e, ref) < 1e-6
    o_n = torch.full((B, Cout, H, W), float("nan"), device="cuda")
    native.conv_igemm(act.cuda(), B, H, W, Cin, 0, Cin, wp.cuda(), 16, 3, 3, 0, b.cuda(), None, o_n, None, strides,
                      out_sc=H * W, n_valid=Cout)
    assert rel_l2(o_n, o_e) < 2e-5


@pytest.mark.parametrize("Ca,Cb,dim", [(3, 3, 128), (3, 0, 64)])
def test_stem_tensor_core_path(native, Ca, Cb, dim):
    """CrossEmbedLayer (k = 3/7/15) as unroll + 15-tap implicit GEMM vs three torch convs"""
    from minimagen_b200.layers import CrossEmbedLayer
    B, H, W = 2, 32, 32
    x, lr = _rand(B, Ca, H, W, seed=44), (_rand(B, Cb, H, W, seed=45) if Cb else None)
    a_e = torch.zeros(B, H, W, 128, dtype=F16)
    EMU.stem_unroll(x, Ca, lr, Cb, B, H, W, a_e)
    a_n = torch.zeros(B, H, W, 128, dtype=F16, device="cuda")
    native.stem_unroll(x.cuda(), Ca, _cu(lr), Cb, B, H, W, a_n)
    assert torch.equal(a_n.cpu(), a_e)
    torch.manual_seed(0)
    layer = CrossEmbedLayer(Ca + Cb, (3, 7, 15), dim_out=dim, stride=1)
    xin = torch.cat((x, lr), dim=1) if Cb else x
    ref = torch.cat([torch.nn.functional.conv2d(xin, c.weight, c.bias, padding=c.padding) for c in layer.convs], dim=1)
    layer = layer.cuda()
    assert layer.stem_tc_ok(H, W)
    with torch.no_grad():
        out = layer.run_stem(x.cuda(), _cu(lr))
    assert rel_l2(out.need_f32().permute(0, 3, 1, 2), ref) < 1e-3          # fp16 operands, one layer


def test_silu(native):
    x = _rand(37, 1024, seed=46) * 4
    o = torch.zeros(37, 1024, device="cuda")
    native.silu(x.cuda(), o)
    assert rel_l2(o, torch.nn.functional.silu(x)) < 1e-6


# ---------------------------------------------------------------------------------------------- conv (direct)
DIRECT_CASES = [
    # B, Hin, Win, Cin, ldi, Cout, k, stride, pad, residual, nchw_out
    (2, 32, 32, 6, 8, 32, 15, 1, 7, False, False),     # stem k=15 on 6 (padded to 8) channels
    (2, 32, 32, 3, 4, 4, 7, 1, 3, False, False),
    (1, 20, 20, 128, 128, 3, 3, 1, 1, False, True),    # final conv -> NCHW
    (2, 16, 16, 24, 24, 16, 3, 1, 1, True, False),     # tiny-config style
    (2, 16, 16, 8, 8, 16, 4, 2, 1, False, False),      # Downsample on the small-channel path
    (1, 8, 8, 16, 16, 8, 1, 1, 0, True, False),
]


@pytest.mark.parametrize("case", DIRECT_CASES)
def test_conv_direct(native, case):
    B, Hin, Win, Cin, ldi, Cout, k, stride, pad, residual, nchw = case
    Hout = (Hin + 2 * pad - k) // stride + 1
    Wout = (Win + 2 * pad - k) // stride + 1
    x = torch.zeros(B, Hin, Win, ldi)
    x[..., :Cin] = _rand(B, Hin, Win, Cin, seed=7)
    w = _rand(Cout, Cin, k, k, seed=8, scale=(k * k * Cin) ** -0.5)
    b = _rand(Cout, seed=9)
    if nchw:
        shape, strides = (B, Cout, Hout, Wout), (Cout * Hout * Wout, Wout, 1, Hout * Wout)
    else:
        shape, strides = (B, Hout, Wout, Cout), (Hout * Wout * Cout, Wout * Cout, Cout, 1)
    r = _rand(*shape, seed=10) if residual else None
    o_e = torch.zeros(shape)
    EMU.conv_direct(x, B, Hin, Win, Cin, ldi, w, Cout, k, k, stride, pad, b, r, o_e, Hout, Wout, strides)
    o_n = torch.full(shape, float("nan"), device="cuda")
    native.conv_direct(x.cuda(), B, Hin, Win, Cin, ldi, w.cuda(), Cout, k, k, stride, pad, b.cuda(), _cu(r), o_n, Hout,
                       Wout, strides)
    assert rel_l2(o_n, o_e) < 1e-5


# ---------------------------------------------------------------------------------------------- GroupNorm / casts
@pytest.mark.parametrize("B,HW,C0,C1,groups", [(2, 256, 128, 0, 8), (2, 1024, 256, 128, 8), (3, 100, 8, 0, 8),
                                               (2, 64, 16, 8, 8), (1, 4096, 2048, 0, 8), (2, 256, 32, 0, 8)])
@pytest.mark.parametrize("f16", [True, False])
@pytest.mark.parametrize("in16", [False, True])
def test_groupnorm_silu(native, B, HW, C0, C1, groups, f16, in16):
    if in16 and (C0 % 8 or (C1 and C1 % 8)):
        pytest.skip("fp16 sources need 8-channel alignment")
    C = C0 + C1
    dt_in = F16 if in16 else F32
    s0 = (_rand(B, HW, C0, seed=11) * 2 + 0.5).to(dt_in)
    s1 = _rand(B, HW, C1, seed=12).to(dt_in) if C1 else None
    gamma, beta = _rand(C, seed=13), _rand(C, seed=14)
    ss = _rand(B, 2 * C, seed=15, scale=0.3)
    sums_e = torch.zeros(B, groups, 2, dtype=F64)
    EMU.gn_stats(s0, C0, s1, C1, 0.7071, B, HW, groups, sums_e)
    sums_n = torch.zeros(B, groups, 2, dtype=F64, device="cuda")
    native.gn_stats(s0.cuda(), C0, _cu(s1), C1, 0.7071, B, HW, groups, sums_n)
    assert rel_l2(sums_n, sums_e) < 1e-6
    dt = F16 if f16 else F32
    big = torch.zeros(B, 2 * C + 24)
    big[:, 8:8 + 2 * C] = ss
    ssv_e = big[:, 8:8 + 2 * C]                 # a column slice of a wider buffer (row pitch != 2C)
    o_e = torch.zeros(B, HW, C, dtype=dt)
    EMU.gn_apply_silu(s0, C0, s1, C1, 0.7071, B, HW, groups, sums_e, 0, None, 0, gamma, beta, ssv_e, big.stride(0),
                      1e-5, o_e)
    o_n = torch.zeros(B, HW, C, dtype=dt, device="cuda")
    big_n = big.cuda()
    native.gn_apply_silu(s0.cuda(), C0, _cu(s1), C1, 0.7071, B, HW, groups, sums_n, 0, None, 0, gamma.cuda(),
                         beta.cuda(), big_n[:, 8:8 + 2 * C], big_n.stride(0), 1e-5, o_n)
    assert rel_l2(o_n, o_e) < (1e-3 if f16 else 5e-6)
    # and against torch's own GroupNorm (the op the reference calls)
    x = torch.cat((s0.float(), s1.float() * 0.7071), dim=-1) if C1 else s0.float()
    gn = torch.nn.functional.group_norm(x.transpose(1, 2).reshape(B, C, HW, 1), groups, gamma, beta, 1e-5)
    y = gn * (ss[:, :C, None, None] + 1) + ss[:, C:, None, None]
    y = torch.nn.functional.silu(y).reshape(B, C, HW).transpose(1, 2)
    assert rel_l2(o_n, y) < (1e-3 if f16 else 1e-5)


def test_groupnorm_block_statistics_from_conv_epilogue(native):
    """conv epilogue block statistics (per 16 channels) of two producers -> GroupNorm over their virtual concat"""
    B, H, W, Cin = 2, 16, 16, 64
    C0, C1, G = 256, 128, 8                      # concat of 384 channels: groups of 48 straddle the two sources
    outs = []
    for i, Cout in enumerate((C0, C1)):
        act = _rand(B, 1, H, W, Cin, seed=50 + i).to(F16)
        w = _rand(Cout, Cin, 3, 3, seed=52 + i, scale=0.05)
        wp = EMU.pack_conv_weight(w)
        strides = (H * W * Cout, W * Cout, Cout)
        o16 = torch.zeros(B, 1, H, W, Cout, dtype=F16, device="cuda")
        o32 = torch.zeros(B, H, W, Cout, device="cuda")
        st = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda")
        native.conv_igemm(act.cuda(), B, H, W, Cin, 0, Cin, wp.cuda(), Cout, 3, 3, 0, None, None, o32, o16, strides,
                          out_stats=st)
        blk = o32.double().reshape(B, H * W, Cout // 16, 16)
        assert rel_l2(st[:, :, 0], blk.sum(dim=(1, 3))) < 1e-6
        assert rel_l2(st[:, :, 1], (blk * blk).sum(dim=(1, 3))) < 1e-6
        # stand-alone pass with groups = C/16 yields the same block statistics
        st2 = torch.zeros_like(st)
        native.gn_stats(o32, Cout, None, 0, 1.0, B, H * W, Cout // 16, st2)
        assert rel_l2(st2, st) < 1e-6
        outs.append((o32, o16, st))
    gamma, beta = _rand(C0 + C1, seed=60), _rand(C0 + C1, seed=61)
    a = torch.zeros(B, H * W, C0 + C1, dtype=F16, device="cuda")
    native.gn_apply_silu(outs[0][1], C0, outs[1][1], C1, 0.7071, B, H * W, G, outs[0][2], 16, outs[1][2], 16,
                         gamma.cuda(), beta.cuda(), None, 0, 1e-5, a)
    x = torch.cat((outs[0][0].cpu(), outs[1][0].cpu() * 0.7071), dim=-1).reshape(B, H * W, C0 + C1)
    ref = torch.nn.functional.silu(torch.nn.functional.group_norm(x.transpose(1, 2), G, gamma, beta, 1e-5)).transpose(1, 2)
    assert rel_l2(a, ref) < 2e-3              # fp16 inputs and outputs


@pytest.mark.parametrize("B,H,W,C0,C1,Cout,res,ss", [
    (2, 32, 16, 128, 0, 128, False, False), (2, 32, 16, 256, 128, 256, True, True), (3, 32, 8, 128, 128, 128, True, True),
    (1, 64, 64, 128, 0, 256, False, True),
    (2, 32, 16, 128, 256, 128, True, True),          # GroupNorm groups (48 channels) straddle the two sources
    (1, 32, 32, 512, 512, 512, True, True),          # deep K (16 chunks), 4 channel tiles
    (5, 64, 32, 128, 0, 128, True, False),           # two chunks, many tiles per image
    (2, 64, 32, 256, 0, 256, True, True),            # C_out % 256 == 0, several tiles per image
    (3, 32, 8, 128, 128, 512, False, True),          # four 128-channel tiles, concat
    (1, 32, 32, 512, 512, 1024, True, True),         # eight channel tiles, deep K
])
def test_fused_groupnorm_conv(native, B, H, W, C0, C1, Cout, res, ss):
    """mi_conv3x3_gn_silu_f16 == mi_gn_apply_silu (block statistics) followed by mi_conv2d_igemm_f16"""
    G, C = 8, C0 + C1
    assert native.conv_gn_supported(H, W, C0, C1, Cout, G)
    x0 = _rand(B, H, W, C0, seed=80) * 1.5 + 0.3
    x1 = _rand(B, H, W, C1, seed=81) if C1 else None
    gamma, beta = _rand(C, seed=82), _rand(C, seed=83)
    ssv = _rand(B, 2 * C, seed=84, scale=0.3) if ss else None
    w = _rand(Cout, C, 3, 3, seed=85, scale=(9 * C) ** -0.5)
    bias = _rand(Cout, seed=86)
    r = _rand(B, H, W, Cout, seed=87) if res else None
    wp = EMU.pack_conv_weight(w)

    def blockstats(t, Cc):
        st = torch.zeros(B, Cc // 16, 2, dtype=F64)
        EMU.gn_stats(t, Cc, None, 0, 1.0, B, H * W, Cc // 16, st)
        return st
    st0, st1 = blockstats(x0, C0), (blockstats(x1, C1) if C1 else None)
    o_e, o16_e = torch.zeros(B, H, W, Cout), torch.zeros(B, 1, H, W, Cout, dtype=F16)
    os_e = torch.zeros(B, Cout // 16, 2, dtype=F64)
    EMU.conv_gn(x0, C0, x1, C1, 0.7071, B, H, W, G, st0, st1, gamma, beta, ssv, 2 * C, 1e-5, wp, Cout, bias, r, o_e, o16_e,
                os_e)
    o_n = torch.full((B, H, W, Cout), float("nan"), device="cuda")
    o16_n = torch.zeros(B, 1, H, W, Cout, dtype=F16, device="cuda")
    os_n = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda")
    native.conv_gn(x0.cuda(), C0, _cu(x1), C1, 0.7071, B, H, W, G, st0.cuda(), _cu(st1), gamma.cuda(), beta.cuda(), _cu(ssv),
                   2 * C, 1e-5, wp.cuda(), Cout, bias.cuda(), _cu(r), o_n, o16_n, os_n)
    torch.cuda.synchronize()
    assert rel_l2(o_n, o_e) < 5e-4          # the fp16 rounding of the activated operand can differ in the last bit
    assert rel_l2(o16_n.reshape(B, H, W, Cout), o_e) < 1.5e-3
    assert rel_l2(os_n, os_e) < 1e-3
    # and against the reference ops in fp32 (GroupNorm -> FiLM -> SiLU -> conv2d)
    x = torch.cat((x0, x1 * 0.7071), dim=-1) if C1 else x0
    y = torch.nn.functional.group_norm(x.permute(0, 3, 1, 2), G, gamma, beta, 1e-5)
    if ss:
        y = y * (ssv[:, :C, None, None] + 1) + ssv[:, C:, None, None]
    y = torch.nn.functional.conv2d(torch.nn.functional.silu(y), w, bias, padding=1).permute(0, 2, 3, 1)
    if res:
        y = y + r
    assert rel_l2(o_n, y) < 1.5e-3


def test_conv_igemm_two_sources(native):
    """virtual concat as two TMA sources (skip connection), skip scale folded into the packed weight"""
    B, H, W, C0, C1, Cout = 2, 16, 16, 128, 64, 128
    a0, a1 = _rand(B, 1, H, W, C0, seed=70).to(F16), _rand(B, 1, H, W, C1, seed=71).to(F16)
    for k in (1, 3):
        w = _rand(Cout, C0 + C1, k, k, seed=72 + k, scale=0.05)
        wsc = w.clone()
        wsc[:, C0:] *= 0.7071
        wp = EMU.pack_conv_weight(wsc)
        strides = (H * W * Cout, W * Cout, Cout)
        o_e = torch.zeros(B, H, W, Cout)
        EMU.conv_igemm(a0, B, H, W, C0, 0, C0 + C1, wp, Cout, k, k, 0, None, None, o_e, None, strides, act2=a1, lda2=C1,
                       c_in1=C0)
        ref = torch.nn.functional.conv2d(torch.cat((a0[:, 0].float(), a1[:, 0].float()), dim=-1).permute(0, 3, 1, 2),
                                         wsc.half().float(), None, padding=k // 2).permute(0, 2, 3, 1)
        assert rel_l2(o_e, ref) < 1e-6
        o_n = torch.zeros(B, H, W, Cout, device="cuda")
        native.conv_igemm(a0.cuda(), B, H, W, C0, 0, C0 + C1, wp.cuda(), Cout, k, k, 0, None, None, o_n, None, strides,
                          act2=a1.cuda(), lda2=C1, c_in1=C0)
        assert rel_l2(o_n, o_e) < 2e-5


@pytest.mark.parametrize("B,H,W,C0,C1,Cout", [(2, 32, 32, 128, 0, 128),     # one source, 4 x 32-pixel tiles
                                               (1, 64, 16, 64, 0, 256),      # 16-wide images, two channel tiles
                                               (2, 32, 32, 64, 64, 128),     # two TMA sources
                                               (3, 16, 16, 128, 64, 128)])   # two TMA sources, 16 x 16 images
def test_conv3x3_swapped_halo_paths(native, B, H, W, C0, C1, Cout):
    """3x3 convs with C_out % 128 == 0, one or two TMA sources: bias, residual, both output copies and the epilogue
    GroupNorm statistics.  (The name is kept from when these shapes selected separate halo kernels; every case now runs on
    the one implicit-GEMM kernel of csrc/conv_tc.cu.)"""
    Cin = C0 + C1
    a0 = _rand(B, 1, H, W, C0, seed=90).to(F16)
    a1 = _rand(B, 1, H, W, C1, seed=91).to(F16) if C1 else None
    w = _rand(Cout, Cin, 3, 3, seed=92, scale=(9 * Cin) ** -0.5)
    b, r = _rand(Cout, seed=93), _rand(B, H, W, Cout, seed=94)
    wp = EMU.pack_conv_weight(w)
    strides = (H * W * Cout, W * Cout, Cout)
    kw = dict(act2=a1, lda2=C1, c_in1=C0) if C1 else {}
    o_e, o16_e = torch.zeros(B, H, W, Cout), torch.zeros(B, H, W, Cout, dtype=F16)
    st_e = torch.zeros(B, Cout // 16, 2, dtype=F64)
    EMU.conv_igemm(a0, B, H, W, C0, 0, Cin, wp, Cout, 3, 3, 0, b, r, o_e, o16_e, strides, out_stats=st_e, **kw)
    o_n = torch.full((B, H, W, Cout), float("nan"), device="cuda")
    o16_n = torch.zeros(B, H, W, Cout, dtype=F16, device="cuda")
    st_n = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda")
    kwn = dict(act2=a1.cuda(), lda2=C1, c_in1=C0) if C1 else {}
    native.conv_igemm(a0.cuda(), B, H, W, C0, 0, Cin, wp.cuda(), Cout, 3, 3, 0, b.cuda(), r.cuda(), o_n, o16_n, strides,
                      out_stats=st_n, **kwn)
    torch.cuda.synchronize()
    assert rel_l2(o_n, o_e) < 2e-5
    assert rel_l2(o16_n, o_e) < 1e-3
    assert rel_l2(st_n, st_e) < 1e-5


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 16, 16, 64, 128), (1, 32, 32, 128, 256), (2, 8, 8, 64, 64),
                                           (3, 64, 16, 128, 128), (2, 32, 8, 64, 128), (1, 64, 64, 256, 128)])   # last three: C_out % 128 == 0 grids
def test_conv_igemm_subpixel_upsample_phases(native, B, H, W, Cin, Cout):
    """modes 2..5: the four 2x2 sub-pixel phases of 'nearest x2 upsample + 3x3 conv' on the low-res tensor, written
    interleaved into the 2H x 2W output; vs the emulation and vs the literal upsample + conv"""
    act = _rand(B, 1, H, W, Cin, seed=95).to(F16)
    k2 = [_rand(Cout, Cin, 2, 2, seed=96 + p, scale=(4 * Cin) ** -0.5) for p in range(4)]
    bias = _rand(Cout, seed=99)
    Ho, Wo = 2 * H, 2 * W
    strides = (Ho * Wo * Cout, 2 * Wo * Cout, 2 * Cout)
    o_e = torch.zeros(B, Ho, Wo, Cout)
    o_n = torch.full((B, Ho, Wo, Cout), float("nan"), device="cuda")
    st_e = torch.zeros(B, Cout // 16, 2, dtype=F64)
    st_n = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda")
    for p in range(4):
        off = ((p >> 1) * Wo + (p & 1)) * Cout
        wp = EMU.pack_conv_weight(k2[p])
        EMU.conv_igemm(act, B, H, W, Cin, 0, Cin, wp, Cout, 2, 2, 2 + p, bias, None, o_e.reshape(-1)[off:], None, strides,
                       out_stats=st_e)
        native.conv_igemm(act.cuda(), B, H, W, Cin, 0, Cin, wp.cuda(), Cout, 2, 2, 2 + p, bias.cuda(), None,
                          o_n.reshape(-1)[off:], None, strides, out_stats=st_n)
    torch.cuda.synchronize()
    assert rel_l2(o_n, o_e) < 2e-5
    assert rel_l2(st_n, st_e) < 1e-5


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("f16", [True, False])
@pytest.mark.parametrize("in16", [False, True])
def test_cast_act(native, mode, f16, in16):
    B, H, W, C0, C1 = 2, 8, 16, 64, 32
    dt_in = F16 if in16 else F32
    s0, s1 = _rand(B, H, W, C0, seed=16).to(dt_in), _rand(B, H, W, C1, seed=17).to(dt_in)
    dt = F16 if f16 else F32
    numel = B * H * W * (C0 + C1) * (4 if mode == 1 else 1)
    o_e = torch.zeros(numel, dtype=dt)
    EMU.cast_act(s0, C0, s1, C1, 0.5, B, H, W, mode, o_e)
    o_n = torch.zeros(numel, dtype=dt, device="cuda")
    native.cast_act(s0.cuda(), C0, s1.cuda(), C1, 0.5, B, H, W, mode, o_n)
    assert torch.equal(o_n.cpu(), o_e)


# ---------------------------------------------------------------------------------------------- conditioning
def test_posemb_and_text_tokens(native):
    t = torch.tensor([0, 1, 17, 500, 999])
    for dim in (8, 128, 256):
        o_e = torch.zeros(5, dim)
        EMU.posemb(t, 5, dim, o_e)
        o_n = torch.zeros(5, dim, device="cuda")
        native.posemb(t.cuda(), 5, dim, o_n)
        assert (o_n.cpu() - o_e).abs().max() < 2e-4          # sin/cos of arguments up to 999 rad, fp32
    B, L, D, m, nt = 3, 11, 16, 260, 4
    proj = _rand(B, L, D, seed=26)
    mask = torch.ones(B, L, dtype=torch.uint8)
    mask[0, 5:] = 0
    keep = torch.tensor([1, 0, 1], dtype=torch.uint8)
    null = _rand(256, D, seed=27)
    for mk in (mask, None):
        c_e, p_e = torch.zeros(B, m, D), torch.zeros(B, D)
        EMU.text_tokens(proj, B, L, D, mk, keep, null, 256, c_e, m, nt, p_e)
        c_n, p_n = torch.zeros(B, m, D, device="cuda"), torch.zeros(B, D, device="cuda")
        native.text_tokens(proj.cuda(), B, L, D, _cu(mk), keep.cuda(), null.cuda(), 256, c_n, m, nt, p_n)
        assert torch.equal(c_n.cpu(), c_e)                   # pure select: exact
        assert rel_l2(p_n, p_e) < 1e-6
    src = _rand(B, 2, D, seed=28)
    d_e, d_n = torch.zeros(B, m, D), torch.zeros(B, m, D, device="cuda")
    EMU.place_rows(src, B, 2, D, d_e, m, 2)
    native.place_rows(src.cuda(), B, 2, D, d_n, m, 2)
    assert torch.equal(d_n.cpu(), d_e)
    a, nl, ad = _rand(B, 32, seed=29), _rand(32, seed=30), _rand(B, 32, seed=31)
    s_e, s_n = torch.zeros(B, 32), torch.zeros(B, 32, device="cuda")
    EMU.select_rows(a, nl, keep, ad, B, 32, s_e)
    native.select_rows(a.cuda(), nl.cuda(), keep.cuda(), ad.cuda(), B, 32, s_n)
    assert torch.equal(s_n.cpu(), s_e)
    x, lr = _rand(2, 3, 10, 10, seed=32), _rand(2, 3, 10, 10, seed=33)
    n_e, n_n = torch.ones(2, 100, 8), torch.ones(2, 100, 8, device="cuda")
    EMU.nchw_to_nhwc(x, 3, lr, 3, 2, 100, 8, n_e)
    native.nchw_to_nhwc(x.cuda(), 3, lr.cuda(), 3, 2, 100, 8, n_n)
    assert torch.equal(n_n.cpu(), n_e)


# ---------------------------------------------------------------------------------------------- cascade resize
@pytest.mark.parametrize("n_in,n_out,pad,clamp", [(64, 256, "reflect", None), (128, 64, "reflect", (-1., 1.)),
                                                  (24, 36, "constant", (0., 1.))])
def test_resize_separable(native, n_in, n_out, pad, clamp):
    from minimagen_b200.helpers import resize_tables
    x = _rand(2, 3, n_in, n_in, seed=120)
    scale = n_out / n_in
    ho, iy, wy = resize_tables(n_in, scale, pad, torch.device("cpu"))
    o_e = torch.zeros(2, 3, ho, ho)
    EMU.resize_separable(x, 6, n_in, n_in, o_e, ho, ho, iy, wy, iy, wy, clamp=clamp)
    o_n = torch.zeros(2, 3, ho, ho, device="cuda")
    native.resize_separable(x.cuda(), 6, n_in, n_in, o_n, ho, ho, iy.cuda(), wy.cuda(), iy.cuda(), wy.cuda(), clamp=clamp)
    assert (o_n.cpu() - o_e).abs().max().item() < 2e-6


# ---------------------------------------------------------------------------------------------- DDPM step
@pytest.mark.parametrize("n,B", [(3 * 64 * 64, 4), (3 * 256 * 256, 2), (1000, 3), (3 * 1024 * 1024, 1)])
def test_quantile_is_exact(native, n, B):
    """Order statistics are integer work: the selected elements must be bit-identical to a full sort."""
    from minimagen_b200.Imagen import quantile_rank
    g = torch.Generator().manual_seed(n)
    x0 = torch.randn(B, n, generator=g) * 1.7
    x0[0, : n // 3] = 0.75                      # long runs of equal values around / below the rank
    if B > 1:
        x0[1] = x0[1].round()                   # heavy ties everywhere
    lo, hi, w = quantile_rank(n, 0.9)
    s_n = torch.zeros(B, device="cuda")
    native.step_quantile(x0.cuda(), B, n, lo, hi, w, 0.0, s_n)
    srt = x0.abs().sort(dim=-1).values
    expect = torch.lerp(srt[:, lo], srt[:, hi], torch.tensor(w))
    assert torch.equal(s_n.cpu(), expect), (s_n.cpu(), expect)
    assert torch.equal(s_n.cpu(), torch.quantile(x0.abs(), 0.9, dim=-1))
    # w = 0 selects one element exactly
    native.step_quantile(x0.cuda(), B, n, lo, lo, 0.0, 0.0, s_n)
    assert torch.equal(s_n.cpu(), srt[:, lo])
    native.step_quantile(x0.cuda(), B, n, n - 1, n - 1, 0.0, 0.0, s_n)
    assert torch.equal(s_n.cpu(), srt[:, -1])
    native.step_quantile(x0.cuda(), B, n, 0, 1, 0.5, 0.0, s_n)
    assert torch.equal(s_n.cpu(), torch.lerp(srt[:, 0], srt[:, 1], torch.tensor(0.5)))


@pytest.mark.parametrize("T", [25, 1000])
def test_step_kernels_vs_golden(native, T):
    from conftest import load_golden
    g = load_golden("ddpm_step.pt")[T]
    tabs = {k: v.cuda() for k, v in g["tables"].items()}
    sigma = (0.5 * g["tables"]["posterior_log_variance_clipped"]).exp().cuda()
    B, n = 3, 3 * 64 * 64
    x, eps, noise, t = g["x"].cuda(), g["eps"].cuda(), g["noise"].cuda(), g["t"].cuda()
    x0 = torch.zeros_like(x)
    native.step_x0(x, eps, None, 1.0, t, tabs["sqrt_recip_alphas_cumprod"], tabs["sqrt_recipm1_alphas_cumprod"], B, n,
                   x0)
    assert torch.equal(x0.cpu(), g["x0"])                                  # un-fused fp32 ops: bit exact
    s = torch.zeros(B, device="cuda")
    native.step_quantile(x0, B, n, 11058, 11059, 0.2998046875, 0.0, s)
    assert torch.equal(s.cpu(), g["s_quantile"])
    native.step_quantile(x0, B, n, 11058, 11059, 0.2998046875, 1.0, s)
    out = torch.zeros_like(x)
    native.step_posterior(x0, x, noise, s, t, tabs["posterior_mean_coef1"], tabs["posterior_mean_coef2"], sigma, B, n,
                          out)
    assert torch.equal(out.cpu(), g["out"])
    # CFG combine inside step_x0
    nl = torch.randn(3, 3, 64, 64, generator=torch.Generator().manual_seed(9))
    native.step_x0(x, eps, nl.cuda(), 7.0, t, tabs["sqrt_recip_alphas_cumprod"], tabs["sqrt_recipm1_alphas_cumprod"],
                   B, n, x0)
    e = nl + (g["eps"] - nl) * 7.0
    a = g["tables"]["sqrt_recip_alphas_cumprod"][g["t"]].reshape(3, 1, 1, 1)
    b = g["tables"]["sqrt_recipm1_alphas_cumprod"][g["t"]].reshape(3, 1, 1, 1)
    assert torch.equal(x0.cpu(), a * g["x"] - b * e)
    fin = torch.zeros_like(x)
    native.step_finalize(out, out.numel(), 1, fin)
    assert torch.equal(fin.cpu(), (g["out"].clamp(-1, 1) + 1) * 0.5)
    q = torch.zeros_like(x)
    native.q_sample(x, noise, t, tabs["sqrt_alphas_cumprod"], tabs["sqrt_one_minus_alphas_cumprod"], B, n, 1.0, 0.0, q)
    sa = g["tables"]["sqrt_alphas_cumprod"][g["t"]].reshape(3, 1, 1, 1)
    sb = g["tables"]["sqrt_one_minus_alphas_cumprod"][g["t"]].reshape(3, 1, 1, 1)
    assert torch.equal(q.cpu(), sa * g["x"] + sb * g["noise"])


# ---------------------------------------------------------------------------------------------- round 2 additions
@pytest.mark.parametrize("case", [(2, 32, 32, 64, 128), (1, 64, 64, 128, 256), (3, 16, 16, 256, 512)])
def test_conv_igemm_mode6_inplace_downsample(native, case):
    """ABI mode 6: the 4x4 stride-2 pad-1 Downsample conv reading the un-split fp16 input in place (TMA element strides)."""
    B, H, W, Cin, Cout = case                         # (H, W) = OUTPUT grid, input is 2H x 2W
    act = _rand(B, 1, 2 * H, 2 * W, Cin, seed=21).to(F16)
    w = _rand(Cout, Cin, 4, 4, seed=22, scale=(16 * Cin) ** -0.5)
    b = _rand(Cout, seed=23)
    wp = EMU.pack_conv_weight(w)
    strides = (H * W * Cout, W * Cout, Cout)
    o_e = torch.zeros(B, H, W, Cout)
    EMU.conv_igemm(act, B, H, W, Cin, 0, Cin, wp, Cout, 4, 4, 6, b, None, o_e, None, strides)
    o_n = torch.full((B, H, W, Cout), float("nan"), device="cuda")
    st = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda")
    native.conv_igemm(act.cuda(), B, H, W, Cin, 0, Cin, wp.cuda(), Cout, 4, 4, 6, b.cuda(), None, o_n, None, strides,
                      out_stats=st)
    assert rel_l2(o_n, o_e) < 2e-5
    ref_st = o_e.double().reshape(B, H * W, Cout // 16, 16)
    assert rel_l2(st[:, :, 0], ref_st.sum(dim=(1, 3))) < 1e-4 and rel_l2(st[:, :, 1], (ref_st ** 2).sum(dim=(1, 3))) < 1e-5


@pytest.mark.parametrize("case", [(2, 16, 16, 128, 64, 128, 1), (1, 32, 32, 64, 192, 256, 1), (2, 32, 32, 128, 128, 128, 3)])
def test_conv_igemm_two_source_virtual_concat(native, case):
    """1x1 (res_conv of the up path) and 3x3 convs over the VIRTUAL concat of two activation tensors (act / act2)."""
    B, H, W, C0, C1, Cout, k = case
    a0 = _rand(B, 1, H, W, C0, seed=31).to(F16)
    a1 = _rand(B, 1, H, W, C1, seed=32).to(F16)
    w = _rand(Cout, C0 + C1, k, k, seed=33, scale=(k * k * (C0 + C1)) ** -0.5)
    wp = EMU.pack_conv_weight(w)
    strides = (H * W * Cout, W * Cout, Cout)
    o_e = torch.zeros(B, H, W, Cout)
    EMU.conv_igemm(a0, B, H, W, C0, 0, C0 + C1, wp, Cout, k, k, 0, None, None, o_e, None, strides, act2=a1, lda2=C1,
                   c_in1=C0)
    o_n = torch.full((B, H, W, Cout), float("nan"), device="cuda")
    native.conv_igemm(a0.cuda(), B, H, W, C0, 0, C0 + C1, wp.cuda(), Cout, k, k, 0, None, None, o_n, None, strides,
                      act2=a1.cuda(), lda2=C1, c_in1=C0)
    assert rel_l2(o_n, o_e) < 2e-5


@pytest.mark.parametrize("B,n,cfg", [(3, 3 * 64 * 64, True), (2, 3 * 256 * 256, False), (1, 3 * 272 * 272, True)])
def test_step_epilogue_fused_is_bit_exact(native, B, n, cfg):
    """mi_step_epilogue (one cluster kernel; or, beyond 196 608 values per image, its three-kernel form) == the x0 ->
    quantile -> posterior chain bit for bit, also when it updates x_t in place; mi_step_advance_t."""
    from minimagen_b200.Imagen import quantile_rank
    from oracle import restatement as R
    tabs = {k: v.cuda() for k, v in R.ddpm_tables(1000).items()}
    sigma = torch.exp(0.5 * tabs["posterior_log_variance_clipped"])
    g = torch.Generator().manual_seed(B * 7 + n)
    x = (torch.randn(B, n, generator=g) * 1.3).cuda()
    eps = torch.randn(B, n, generator=g).cuda()
    eps0 = torch.randn(B, n, generator=g).cuda() if cfg else None
    noise = torch.randn(B, n, generator=g).cuda()
    t = torch.tensor([999, 0, 417][:B]).cuda()
    lo, hi, w = quantile_rank(n, 0.9)
    x0 = torch.empty_like(x)
    s = torch.empty(B, device="cuda")
    ref = torch.empty_like(x)
    a, b_ = tabs["sqrt_recip_alphas_cumprod"], tabs["sqrt_recipm1_alphas_cumprod"]
    c1, c2 = tabs["posterior_mean_coef1"], tabs["posterior_mean_coef2"]
    native.step_x0(x, eps, eps0, 7.0, t, a, b_, B, n, x0)
    native.step_quantile(x0, B, n, lo, hi, w, 1.0, s)
    native.step_posterior(x0, x, noise, s, t, c1, c2, sigma, B, n, ref)
    out = torch.empty_like(x)
    s2 = torch.empty(B, device="cuda")
    native.step_epilogue(x, eps, eps0, 7.0, t, a, b_, c1, c2, sigma, noise, B, n, lo, hi, w, 1.0, out, s_out=s2)
    assert torch.equal(out, ref) and torch.equal(s2, s)
    xin = x.clone()
    native.step_epilogue(xin, eps, eps0, 7.0, t, a, b_, c1, c2, sigma, noise, B, n, lo, hi, w, 1.0, xin)   # in place
    assert torch.equal(xin, ref)
    tt = t.clone()
    native.step_advance_t(tt, B)
    assert torch.equal(tt, (t - 1).clamp(min=0))


@pytest.mark.parametrize("case", [
    # B, H, W, Cin, Cout, Cx0, Cx1, residual, stats
    (2, 32, 16, 128, 128, 256, 0, False, True),        # G32x8, single-tensor x
    (2, 16, 16, 256, 256, 256, 256, True, True),       # G16x16, x = virtual concat (up-path ResnetBlock)
    (1, 64, 32, 128, 128, 128, 128, False, False),     # G32x8, concat x
    (3, 32, 32, 512, 512, 512, 512, False, True),      # deep K
])
def test_conv_res1x1_folded(native, case):
    """mi_conv3x3_res1x1_f16 == conv3x3(act) + conv1x1(cat(x0, x1)) (+bias sum, +residual, block statistics)."""
    B, H, W, Cin, Cout, Cx0, Cx1, res, stats = case
    Cx = Cx0 + Cx1
    assert native.conv_res1x1_supported(H, W, Cin, Cout, Cx)
    a = _rand(B, 1, H, W, Cin, seed=41).to(F16)
    x0 = _rand(B, 1, H, W, Cx0, seed=42).to(F16)
    x1 = _rand(B, 1, H, W, Cx1, seed=43).to(F16) if Cx1 else None
    w3 = _rand(Cout, Cin, 3, 3, seed=44, scale=(9 * Cin) ** -0.5)
    w1 = _rand(Cout, Cx, 1, 1, seed=45, scale=Cx ** -0.5)
    bias = _rand(Cout, seed=46)
    r = _rand(B, H, W, Cout, seed=47) if res else None
    wp = torch.cat((EMU.pack_conv_weight(w3), EMU.pack_conv_weight(w1)), dim=1).contiguous()
    o_e = torch.zeros(B, H, W, Cout)
    st_e = torch.zeros(B, Cout // 16, 2, dtype=F64) if stats else None
    EMU.conv_res1x1(a, B, H, W, Cin, Cin, None, 0, 0, x0, Cx0, Cx, x1, Cx1, Cx0 if Cx1 else 0, wp, Cout, bias, r, o_e, None, st_e)
    o_n = torch.full((B, H, W, Cout), float("nan"), device="cuda")
    o16_n = torch.zeros(B, 1, H, W, Cout, dtype=F16, device="cuda")
    st_n = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda") if stats else None
    native.conv_res1x1(a.cuda(), B, H, W, Cin, Cin, None, 0, 0, x0.cuda(), Cx0, Cx, _cu(x1), Cx1, Cx0 if Cx1 else 0, wp.cuda(),
                       Cout, bias.cuda(), _cu(r), o_n, o16_n, st_n)
    torch.cuda.synchronize()
    assert rel_l2(o_n, o_e) < 2e-5
    assert rel_l2(o16_n.reshape(B, H, W, Cout), o_e) < 1e-3
    if stats:
        assert rel_l2(st_n, st_e) < 1e-4
