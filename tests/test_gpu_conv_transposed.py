"""GPU: the implicit-GEMM conv's transposed schedule (csrc/conv_tc.cu, C_out = 128 computed as D^T = W . A^T on the
cooperative 256-wide kernel: output channels on M, 256 pixels of one image on N) against the float64 references and
per-element bounds of tests/fp64_ref.py.  The block_n hint 256 forces it at C_out = 128; every case also checks, from the
profiler's kernel records, that the transposed instance is the one that ran.  Covered: the four tile geometries (BW = 256,
BW = 128 / BH = 2, BW = 64 / BH = 4, and BW = 8 / BH = 32), more tiles than SMs x ring stages, b > 1, bias, residual, fp32
and fp16 outputs, statistics, the two-source concat, the folded res_conv, the stride-2 Downsample read in place and from
the phase split, the four sub-pixel phases into a strided output, and the 15x1 stem; and the transposed against the
128-wide ping-pong schedule on identical inputs."""
import re

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import fp64_ref as R
from emu_ops import EmuOps
from fp64_ref import check, check_rel_l2, half_out
from test_gpu_image_fwd import REL_CONV, REL_F16, _nan, _rand, _run_conv, _sms

pytestmark = pytest.mark.gpu
F16, F64 = torch.float16, torch.float64
EMU = EmuOps()
STAGES = 4        # ring stages of the 256-wide kernel (48 KiB each)
CONV_WG_KERNEL = re.compile(r"conv_wg_kernel<(\d+), *(?:\(bool\))?(\w+), *(?:\(bool\))?(\w+)>")


def conv_instance(name):
    """(BLOCK_N, GN, transposed) of a conv_wg_kernel record's name, or None for any other kernel."""
    m = CONV_WG_KERNEL.search(name)
    return None if m is None else (int(m.group(1)), m.group(2) in ("true", "1"), m.group(3) in ("true", "1"))


def _schedules(fn):
    """Run fn under the profiler; the set of conv_wg_kernel instances (BLOCK_N, GN, transposed) it launched.  fn must
    give the same result when run again: a profiling session that returns no kernel record at all is repeated (up to
    three sessions) rather than read as "no conv ran"."""
    found = set()
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        for ev in prof.events():
            inst = conv_instance(ev.name)
            if inst:
                found.add(inst)
        if found:
            break
    return found


TRANSPOSED, PINGPONG = (256, False, True), (128, False, False)


def _assert_ran(found, inst):
    assert found == {inst}, f"expected only conv_wg_kernel{inst}, the profiler saw {sorted(found)}"


# name: B, H, W, C0, C1, k, mode, bias, residual, fp16 out, statistics  ((H, W) the grid of one launch, C_out = 128)
CASES = {
    "bw256": lambda s: (2, 4, 256, 128, 0, 3, 0, True, True, True, True),
    "bw256_two_tiles_per_row_1x1": lambda s: (2, 2, 512, 128, 0, 1, 0, True, False, True, True),
    "bh2_more_tiles_than_sms_x_stages": lambda s: (s * STAGES // 64 + 1, 128, 128, 128, 0, 3, 0, True, True, True, True),
    "bh4_concat": lambda s: (3, 64, 64, 128, 128, 3, 0, True, False, True, True),
    "bh32_w8": lambda s: (2, 32, 8, 64, 0, 3, 0, False, True, False, True),
    "downsample_in_place": lambda s: (2, 64, 128, 128, 0, 4, 6, True, False, True, True),
    "downsample_phase_split": lambda s: (2, 32, 64, 128, 0, 4, 1, True, False, True, True),
    "subpixel_phases_strided_out": lambda s: (2, 32, 64, 128, 0, 2, 2, True, False, True, True),
}


@pytest.mark.parametrize("name", list(CASES))
def test_conv_transposed(native, name):
    B, H, W, C0, C1, k, mode, bias, res, f16, stats = CASES[name](_sms())
    if name == "bh2_more_tiles_than_sms_x_stages":
        assert B * H * W // 256 > _sms() * STAGES
    found = _schedules(lambda: _run_conv(native, B, H, W, C0, C1, 128, k, mode, bias, res, f16, stats, 256, seed=900))
    _assert_ran(found, TRANSPOSED)


def test_conv_transposed_vs_pingpong(native):
    """The same conv (bias, residual, fp32 + fp16 out, statistics) on both schedules: each within its bound of the float64
    reference, and the two within float rounding of each other."""
    B, H, W, Cin, Cout = 4, 128, 128, 256, 128
    a = _rand(B, H, W, Cin, seed=910).half()
    w = _rand(Cout, Cin, 3, 3, seed=911, scale=(9 * Cin) ** -0.5)
    wp = EMU.pack_conv_weight(w.cpu()).cuda()
    bias, r = _rand(Cout, seed=912), _rand(B, H, W, Cout, seed=913)
    ref, bound = R.conv_fwd_ref(a, wp, 3, 3, 0, bias, r)
    outs = {}
    for inst, hint in ((TRANSPOSED, 256), (PINGPONG, 128)):
        o, o16 = _nan(B, H, W, Cout), _nan(B, H, W, Cout, dtype=F16)
        st = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda")
        found = _schedules(lambda: (st.zero_(), native.conv_igemm(a, B, H, W, Cin, 0, Cin, wp, Cout, 3, 3, 0, bias, r, o, o16,
                                                                  (H * W * Cout, W * Cout, Cout), block_n=hint,
                                                                  out_stats=st)))
        _assert_ran(found, inst)
        what = f"conv 3x3 {Cin}->{Cout} @{H}x{W} block_n={hint}"
        check(o, ref, bound, what)
        check_rel_l2(o, ref, REL_CONV, what)
        check(o16, *half_out(ref, bound), what + " fp16")
        check(st, *R.conv_stats_ref(o), what + " statistics")
        outs[hint] = (o, o16, st)
    (o_t, o16_t, st_t), (o_p, o16_p, st_p) = outs[256], outs[128]
    check_rel_l2(o_t, o_p, 1e-6, "transposed vs ping-pong fp32 output")
    check_rel_l2(o16_t, o16_p, 1e-3, "transposed vs ping-pong fp16 output")
    check_rel_l2(st_t, st_p, 1e-6, "transposed vs ping-pong statistics")


def test_conv_res1x1_transposed(native):
    """The folded res_conv (3x3 + 1x1 over a virtual concat x) at C_out = 128 with a 256-pixel tile for every SM: it takes
    no hint and selects the transposed schedule by itself."""
    B, H, W, Cin, Cout, Cx0, Cx1 = -(-_sms() // 4), 32, 32, 128, 128, 64, 128
    Cx = Cx0 + Cx1
    assert native.conv_res1x1_supported(H, W, Cin, Cout, Cx)
    a = _rand(B, H, W, Cin, seed=921).half()
    x0, x1 = _rand(B, H, W, Cx0, seed=922).half(), _rand(B, H, W, Cx1, seed=923).half()
    w3 = _rand(Cout, Cin, 3, 3, seed=924, scale=(9 * Cin) ** -0.5)
    w1 = _rand(Cout, Cx, 1, 1, seed=925, scale=Cx ** -0.5)
    bias, r = _rand(Cout, seed=926), _rand(B, H, W, Cout, seed=927)
    wp = torch.cat((EMU.pack_conv_weight(w3.cpu()), EMU.pack_conv_weight(w1.cpu())), dim=1).contiguous().cuda()
    o, o16 = _nan(B, H, W, Cout), _nan(B, H, W, Cout, dtype=F16)
    st = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda")
    found = _schedules(lambda: (st.zero_(), native.conv_res1x1(a, B, H, W, Cin, Cin, None, 0, 0, x0, Cx0, Cx, x1, Cx1, Cx0, wp,
                                                               Cout, bias, r, o, o16, st)))
    _assert_ran(found, TRANSPOSED)
    ref, bound = R.conv_fwd_ref(a, wp, 3, 3, 0, bias, r, x=torch.cat((x0, x1), dim=-1))
    what = f"conv res1x1 transposed B={B} {Cin}+{Cx}->{Cout}"
    check(o, ref, bound, what)
    check_rel_l2(o, ref, REL_CONV, what)
    check(o16, *half_out(ref, bound), what + " fp16")
    check_rel_l2(o16, ref, REL_F16, what + " fp16")
    check(st, *R.conv_stats_ref(o), what + " statistics")


def test_stem_transposed(native):
    """The stem's 15x1 GEMM over the 128-wide unrolled operand (30 k-blocks) on 256-wide image rows."""
    B, H, W, C, Cout = 2, 16, 256, 128, 128
    a = _rand(B, H, W, C, seed=931).half()
    w = _rand(Cout, C, 15, 1, seed=932, scale=(15 * C) ** -0.5)
    wp = EMU.pack_conv_weight(w.cpu()).cuda()
    bias = _rand(Cout, seed=933)
    o, o16 = _nan(B, H, W, Cout), _nan(B, H, W, Cout, dtype=F16)
    st = torch.zeros(B, Cout // 16, 2, dtype=F64, device="cuda")
    found = _schedules(lambda: (st.zero_(), native.conv_igemm(a, B, H, W, C, 0, C, wp, Cout, 15, 1, 0, bias, None, o, o16,
                                                              (H * W * Cout, W * Cout, Cout), block_n=256, out_stats=st)))
    _assert_ran(found, TRANSPOSED)
    ref, bound = R.conv_fwd_ref(a, wp, 15, 1, 0, bias)
    what = "stem 15x1 128->128 transposed"
    check(o, ref, bound, what)
    check_rel_l2(o, ref, REL_CONV, what)
    check(o16, *half_out(ref, bound), what + " fp16")
    check(st, *R.conv_stats_ref(o), what + " statistics")
