"""The implicit-GEMM conv's 256-wide tiles (csrc/conv_tc.cu) against the emulation of the same fp16 operands
(tests/emu_ops.py): every conv mode at BLOCK_N = 256 through the block_n hint, and the auto-selected 256-wide tile
(including the folded res_conv, which takes no hint) on shapes sized from the device's SM count; bias, residual, fp16
output and GroupNorm statistics, an odd number of M tiles, fewer tiles than SMs, and images smaller than a tile."""
import pytest
import torch

from conftest import rel_l2
from emu_ops import EmuOps

pytestmark = pytest.mark.gpu
F16, F64 = torch.float16, torch.float64
EMU = EmuOps()


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed + sum(shape))
    return torch.randn(*shape, generator=g) * scale


def _cu(t):
    return None if t is None else t.cuda()


def _batch_for_256(tiles_per_image):
    """smallest batch whose 256-wide tiles (C_out = 256) give every SM one: pick_block_n then selects 256"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return -(-sms // tiles_per_image)


def _run(native, B, H, W, C0, C1, Cout, k, mode, bias, res, f16, stats, block_n, seed):
    """one conv through conv_igemm vs the emulation; (H, W) is the output grid"""
    Cin = C0 + C1
    P = 4 if mode == 1 else 1
    ishape = (B, 1, 2 * H, 2 * W, C0) if mode == 6 else (B, P, H, W, C0)
    a0 = _rand(*ishape, seed=seed).to(F16)
    a1 = _rand(B, P, H, W, C1, seed=seed + 1).to(F16) if C1 else None
    kh = 2 if 2 <= mode <= 5 else k
    w = _rand(Cout, Cin, kh, kh, seed=seed + 2, scale=(kh * kh * Cin) ** -0.5)
    b = _rand(Cout, seed=seed + 3) if bias else None
    r = _rand(B, H, W, Cout, seed=seed + 4) if res else None
    wp = EMU.pack_conv_weight(w)
    strides = (H * W * Cout, W * Cout, Cout)
    kw = dict(act2=a1, lda2=C1, c_in1=C0) if C1 else {}
    o_e = torch.zeros(B, H, W, Cout)
    o16_e = torch.zeros(B, H, W, Cout, dtype=F16) if f16 else None
    st_e = torch.zeros(B, Cout // 16, 2, dtype=F64) if stats else None
    EMU.conv_igemm(a0, B, H, W, C0, 0, Cin, wp, Cout, kh, kh, mode, b, r, o_e, o16_e, strides, out_stats=st_e, **kw)
    o_n = torch.full((B, H, W, Cout), float("nan"), device="cuda")
    o16_n = torch.zeros(B, H, W, Cout, dtype=F16, device="cuda") if f16 else None
    st_n = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda") if stats else None
    kwn = dict(act2=a1.cuda(), lda2=C1, c_in1=C0) if C1 else {}
    native.conv_igemm(a0.cuda(), B, H, W, C0, 0, Cin, wp.cuda(), Cout, kh, kh, mode, _cu(b), _cu(r), o_n, o16_n, strides,
                      block_n=block_n, out_stats=st_n, **kwn)
    torch.cuda.synchronize()
    assert rel_l2(o_n, o_e) < 2e-5
    if f16:
        assert rel_l2(o16_n, o_e) < 1e-3
    if stats:
        assert rel_l2(st_n, st_e) < 1e-5


HINTED_CASES = [
    # B, H, W, C0, C1, Cout, k, mode, bias, residual, f16out, stats
    (2, 16, 16, 128, 0, 256, 3, 0, True, True, True, True),       # 4 tiles: fewer tiles than SMs
    (1, 24, 16, 64, 0, 256, 3, 0, True, False, False, True),      # tiles_m = 3
    (5, 8, 8, 64, 0, 512, 3, 0, False, True, True, True),         # 2 images per tile, tiles_m = 3, batch tail
    (1, 4, 256, 64, 0, 256, 1, 0, True, False, False, False),     # W > 128, 1x1
    (2, 16, 16, 128, 64, 256, 3, 0, True, True, False, True),     # two-source virtual concat
    (2, 16, 16, 64, 0, 256, 4, 1, True, False, False, True),      # Downsample via phase split
    (2, 16, 16, 64, 0, 256, 4, 6, True, False, True, True),       # Downsample read in place
    (1, 8, 16, 64, 0, 512, 2, 2, True, False, False, True),       # sub-pixel phases (one launch per phase below)
]


@pytest.mark.parametrize("case", HINTED_CASES)
def test_conv_block_n_256(native, case):
    B, H, W, C0, C1, Cout, k, mode, bias, res, f16, stats = case
    modes = (2, 3, 4, 5) if mode == 2 else (mode,)
    for i, m in enumerate(modes):
        _run(native, B, H, W, C0, C1, Cout, k, m, bias, res, f16, stats, 256, seed=100 + 10 * i)


@pytest.mark.parametrize("H,W", [(32, 32), (24, 16)])
def test_conv_auto_256(native, H, W):
    """no hint: C_out = 256 with a 256-wide tile for every SM selects the 256-wide tile"""
    B = _batch_for_256(H * W // 128)
    _run(native, B, H, W, 64, 0, 256, 3, 0, True, True, True, True, 0, seed=300)


def test_conv_res1x1_auto_256(native):
    """the folded res_conv (3x3 + 1x1 over a virtual concat) on a shape that auto-selects the 256-wide tile"""
    B, H, W, Cin, Cout, Cx0, Cx1 = _batch_for_256(8), 32, 32, 64, 256, 64, 64
    Cx = Cx0 + Cx1
    assert native.conv_res1x1_supported(H, W, Cin, Cout, Cx)
    a = _rand(B, 1, H, W, Cin, seed=401).to(F16)
    x0 = _rand(B, 1, H, W, Cx0, seed=402).to(F16)
    x1 = _rand(B, 1, H, W, Cx1, seed=403).to(F16)
    w3 = _rand(Cout, Cin, 3, 3, seed=404, scale=(9 * Cin) ** -0.5)
    w1 = _rand(Cout, Cx, 1, 1, seed=405, scale=Cx ** -0.5)
    bias = _rand(Cout, seed=406)
    r = _rand(B, H, W, Cout, seed=407)
    wp = torch.cat((EMU.pack_conv_weight(w3), EMU.pack_conv_weight(w1)), dim=1).contiguous()
    o_e = torch.zeros(B, H, W, Cout)
    st_e = torch.zeros(B, Cout // 16, 2, dtype=F64)
    EMU.conv_res1x1(a, B, H, W, Cin, Cin, None, 0, 0, x0, Cx0, Cx, x1, Cx1, Cx0, wp, Cout, bias, r, o_e, None, st_e)
    o_n = torch.full((B, H, W, Cout), float("nan"), device="cuda")
    o16_n = torch.zeros(B, H, W, Cout, dtype=F16, device="cuda")
    st_n = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda")
    native.conv_res1x1(a.cuda(), B, H, W, Cin, Cin, None, 0, 0, x0.cuda(), Cx0, Cx, x1.cuda(), Cx1, Cx0, wp.cuda(), Cout,
                       bias.cuda(), r.cuda(), o_n, o16_n, st_n)
    torch.cuda.synchronize()
    assert rel_l2(o_n, o_e) < 2e-5
    assert rel_l2(o16_n, o_e) < 1e-3
    assert rel_l2(st_n, st_e) < 1e-4
