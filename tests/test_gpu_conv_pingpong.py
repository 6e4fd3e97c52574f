"""The implicit-GEMM conv's ping-pong schedule (csrc/conv_tc.cu, TMA kernel at BLOCK_N <= 128: each consumer warpgroup
owns every second tile of its CTA) against the emulation of the same fp16 operands (tests/emu_ops.py): every conv mode at
the 128- and 64-wide tiles, and the ring and tile bookkeeping -- fewer k-blocks per tile than ring stages, k-blocks not a
multiple of the stage count, CTAs with one tile, an odd number of tiles and many ring wraps, two images per tile, the
folded res_conv and the two-source concat."""
import pytest
import torch

from conftest import rel_l2
from emu_ops import EmuOps
from test_gpu_conv_tiles import HINTED_CASES, _rand, _run

pytestmark = pytest.mark.gpu
F16, F64 = torch.float16, torch.float64
EMU = EmuOps()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("block_n", [128, 64])
@pytest.mark.parametrize("case", HINTED_CASES)
def test_conv_block_n_pingpong(native, case, block_n):
    B, H, W, C0, C1, Cout, k, mode, bias, res, f16, stats = case
    modes = (2, 3, 4, 5) if mode == 2 else (mode,)
    for i, m in enumerate(modes):
        _run(native, B, H, W, C0, C1, Cout, k, m, bias, res, f16, stats, block_n, seed=500 + 10 * i)


# (B, H, W, C_in, C_out, k, block_n): one 128-pixel tile per image at 8 x 16, two per image at 16 x 16, two images per
# tile at 8 x 8; the ring has 6 stages at 128 wide and 8 at 64 wide
RING_CASES = {
    "one_kblock": lambda s: (2, 16, 16, 64, 128, 1, 128),          # 1x1, C_in = 64: num_kb = 1 < stages
    "kb9_of_6_stages": lambda s: (3, 16, 16, 64, 128, 3, 128),     # num_kb = 9, not a multiple of the stage count
    "kb18_of_8_stages": lambda s: (3, 16, 16, 128, 64, 3, 64),
    "one_tile_per_cta": lambda s: (2, 16, 16, 128, 128, 3, 128),   # 4 tiles: consumer 1 of every CTA idles
    "three_tiles_per_cta": lambda s: (3 * s, 8, 16, 64, 128, 3, 128),
    "many_tiles_per_cta": lambda s: (4 * s + 3, 8, 16, 64, 128, 3, 128),   # 4-5 tiles x 9 k-blocks: several ring wraps
    "two_images_per_tile": lambda s: (2 * s + 1, 8, 8, 64, 128, 3, 128),
    "two_images_per_tile_64": lambda s: (5, 8, 8, 128, 128, 3, 64),
}


@pytest.mark.parametrize("name", list(RING_CASES))
def test_conv_pingpong_ring(native, name):
    B, H, W, Cin, Cout, k, block_n = RING_CASES[name](_sms())
    _run(native, B, H, W, Cin, 0, Cout, k, 0, True, True, True, True, block_n, seed=600)


def test_conv_pingpong_auto_128(native):
    """no hint: C_out = 128 runs the 128-wide ping-pong tile, several tiles per CTA"""
    B = -(-3 * _sms() // 8)
    _run(native, B, 32, 32, 128, 0, 128, 3, 0, True, True, True, True, 0, seed=700)


def test_conv_res1x1_pingpong(native):
    """the folded res_conv (3x3 + 1x1 over a virtual concat) at C_out = 128, which runs 128-wide tiles"""
    B, H, W, Cin, Cout, Cx0, Cx1 = _sms() // 4 + 1, 32, 32, 128, 128, 64, 128
    Cx = Cx0 + Cx1
    assert native.conv_res1x1_supported(H, W, Cin, Cout, Cx)
    a = _rand(B, 1, H, W, Cin, seed=801).to(F16)
    x0 = _rand(B, 1, H, W, Cx0, seed=802).to(F16)
    x1 = _rand(B, 1, H, W, Cx1, seed=803).to(F16)
    w3 = _rand(Cout, Cin, 3, 3, seed=804, scale=(9 * Cin) ** -0.5)
    w1 = _rand(Cout, Cx, 1, 1, seed=805, scale=Cx ** -0.5)
    bias = _rand(Cout, seed=806)
    r = _rand(B, H, W, Cout, seed=807)
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
