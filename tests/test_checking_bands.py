"""The row bands of the per-call checkers (tests/checking_ops.py), on the CPU over the torch emulation (tests/emu_ops.py).

At 1024 x 1024 one image's float64 conv reference is 8 - 16x SLICE_ELEMENTS, so the image-sized checkers compute it in
bands of rows, each reading the halo rows its taps reach.  Here SLICE_ELEMENTS is forced low enough that every case bands
(bands of 3 rows: band edges that do not fall on tile or phase boundaries):

  * test_banded_and_whole_image_checks_agree: every image-sized checker -- the conv modes (3 x 3, the 15 x 1 stem conv, the
    phase-split and the in-place stride-2 conv, the sub-pixel Upsample phases, the folded 1x1 conv), their epilogue
    statistics, gn_stats, gn_apply_silu, cast_act, stem_unroll, nchw_to_nhwc -- gives the same verdict and the same worst
    |err| / bound, to 1e-9 relative, banded and on whole images;
  * test_halo_defect_at_a_band_edge_fails: a conv whose first or last output row of an interior band reads its halo row
    as zero (the band's neighbour treated as the image border, the defect a wrong banded reference would share) fails the
    banded check.
"""
import pytest
import torch

import checking_ops
from checking_ops import CheckingOps
from emu_ops import EmuOps

F16, F32, F64 = torch.float16, torch.float32, torch.float64
B, H, W = 3, 16, 16
ROWS = 3                                                # rows per band in the banded runs


def _rand(g, *shape, dtype=F32, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(dtype)


# ------------------------------------------------------------------------------------------------ the calls
def _conv(mode, kh, kw, c_in=64, c_out=32, h=H, f32=True, f16=True, stats=True, residual=True):
    """(halo, per_row, call): one conv_igemm of the given mode at h x W, with the per_row / halo its checker bands by."""
    def call(ops, g):
        inp = {6: (B, 2 * h, 2 * W, c_in), 1: (B, 4, h, W, c_in)}.get(mode, (B, h, W, c_in))
        act = _rand(g, *inp, dtype=F16)
        wp = _rand(g, c_out, kh * kw * c_in, dtype=F16, scale=0.05)
        st = (h * W * c_out, W * c_out, c_out)
        out32 = torch.empty(B, h, W, c_out) if f32 else None
        out16 = torch.empty(B, h, W, c_out, dtype=F16) if f16 else None
        ops.conv_igemm(act, B, h, W, c_in, 0, c_in, wp, c_out, kh, kw, mode, _rand(g, c_out),
                       _rand(g, B, h, W, c_out) if residual else None, out32, out16, st,
                       out_stats=torch.zeros(B, c_out // 16, 2, dtype=F64) if stats else None)
    halo = 2 if mode == 6 else (kh // 2 if mode == 0 else 1)
    return halo, W * max(4 * c_in, c_out), call


def _res1x1(ops, g):
    c_in, x_cin, c_out = 64, 64, 128
    ops.conv_res1x1(_rand(g, B, H, W, c_in, dtype=F16), B, H, W, c_in, c_in, None, 0, 0,
                    _rand(g, B, H, W, x_cin, dtype=F16), x_cin, x_cin, None, 0, 0,
                    _rand(g, c_out, 9 * c_in + x_cin, dtype=F16, scale=0.05), c_out, _rand(g, c_out),
                    _rand(g, B, H, W, c_out), torch.empty(B, H, W, c_out), None, torch.zeros(B, c_out // 16, 2, dtype=F64))


def _gn_stats(ops, g):
    ops.gn_stats(_rand(g, B, H * W, 64), 64, _rand(g, B, H * W, 32), 32, 0.7071, B, H * W, 8,
                 torch.zeros(B, 8, 2, dtype=F64))


def _gn_apply(out_dtype):
    def call(ops, g):
        C, G = 128, 8
        s0, s1 = _rand(g, B, H * W, 64, dtype=F16), _rand(g, B, H * W, 64, dtype=F16)
        x = torch.cat((s0.double(), s1.double() * 0.7071), dim=-1).reshape(B, H * W, G, C // G)
        sums = torch.stack((x.sum(dim=(1, 3)), (x * x).sum(dim=(1, 3))), dim=-1).contiguous()
        ops.gn_apply_silu(s0, 64, s1, 64, 0.7071, B, H * W, G, sums, 0, None, 0, 1 + _rand(g, C, scale=0.1),
                          _rand(g, C, scale=0.1), _rand(g, B, 2 * C, scale=0.1), 2 * C, 1e-5,
                          torch.empty(B, H * W, C, dtype=out_dtype))
    return call


def _cast(mode):
    def call(ops, g):
        n = B * H * W * 96 * (4 if mode == 1 else 1)
        ops.cast_act(_rand(g, B, H, W, 64), 64, _rand(g, B, H, W, 32), 32, 0.7071, B, H, W, mode,
                     torch.empty(n, dtype=F16))
    return call


def _stem_unroll(ops, g):
    ops.stem_unroll(_rand(g, B, 3, H, W), 3, _rand(g, B, 3, H, W), 3, B, H, W, torch.empty(B, H, W, 128, dtype=F16))


def _nchw_to_nhwc(ops, g):
    ops.nchw_to_nhwc(_rand(g, B, 3, H * W), 3, _rand(g, B, 3, H * W), 3, B, H * W, 8, torch.empty(B, H * W, 8))


# name -> (halo, per_row, call): SLICE_ELEMENTS = per_row (ROWS + 2 halo) gives bands of ROWS rows (of pixels, for the
# checkers that band the pixel dimension)
CASES = {
    "conv 3x3": _conv(0, 3, 3),
    "conv 15x1 stem": _conv(0, 15, 1, c_in=128, c_out=64, h=32),
    "conv phase-split stride 2": _conv(1, 4, 4),
    "conv stride 2 in place, fp16 out": _conv(6, 4, 4, f32=False),
    "conv sub-pixel phase 2": _conv(2, 2, 2),
    "conv sub-pixel phase 5, fp16 out": _conv(5, 2, 2, f32=False, residual=False),
    "conv_res1x1": (1, W * 128, _res1x1),
    "gn_stats": (0, 96 * 8, _gn_stats),
    "gn_apply_silu fp16": (0, 128 * 8, _gn_apply(F16)),
    "gn_apply_silu fp32": (0, 128 * 8, _gn_apply(F32)),
    "cast_act mode 0": (0, 4 * W * 96, _cast(0)),
    "cast_act mode 1": (0, 4 * W * 96, _cast(1)),
    "cast_act mode 2": (0, 4 * W * 96, _cast(2)),
    "stem_unroll": (0, W * 128, _stem_unroll),
    "nchw_to_nhwc": (0, 2 * 8 * 8, _nchw_to_nhwc),
}


def _run(ops, case, slice_elements, monkeypatch, **kw):
    """One call of `case` through CheckingOps with SLICE_ELEMENTS = slice_elements; returns (proxy, most bands per image)."""
    seen = []
    bands = checking_ops._bands

    def counting(*a, **k):
        pieces = bands(*a, **k)
        seen.append(max(len(rows) for _, rows in pieces))
        return pieces
    monkeypatch.setattr(checking_ops, "SLICE_ELEMENTS", slice_elements)
    monkeypatch.setattr(checking_ops, "_bands", counting)
    proxy = CheckingOps(ops, sms=132, **kw)
    CASES[case][2](proxy, torch.Generator().manual_seed(7))
    return proxy, max(seen)


@pytest.mark.parametrize("case", list(CASES))
def test_banded_and_whole_image_checks_agree(case, monkeypatch):
    halo, per_row, _ = CASES[case]
    whole, n1 = _run(EmuOps(), case, 1 << 26, monkeypatch)
    banded, n2 = _run(EmuOps(), case, per_row * (ROWS + 2 * halo), monkeypatch)
    assert n1 == 1 and n2 > 1, f"{case}: {n1} / {n2} bands per image"
    print(f"\n{case}: {n2} bands per image")
    assert whole.family.keys() == banded.family.keys() and whole.family
    for fam, (calls, worst) in whole.family.items():
        bc, bw = banded.family[fam]
        print(f"  {fam:24s} worst |err|/bound {worst:.6g} whole, {bw:.6g} banded")
        # to 1e-9 of the bound (every ratio here is <= 1).  The emulation's statistics are the float64 sums of its own
        # output, so their ratio is 0 whole and the float64 summation order, ~1e-10, banded
        assert calls == bc and abs(bw - worst) <= 1e-9 * max(worst, 1.0), f"{fam}: {worst!r} whole vs {bw!r} banded"


# ------------------------------------------------------------------------------------------------ planted halo defects
def _halo_defect(emu, edge, band):
    """conv_igemm whose output row `band[0]` (edge "first") or `band[1] - 1` ("last") is computed from the input with every
    row outside the band's own input rows zeroed: the neighbouring band's halo row read as the image border."""
    orig = emu.conv_igemm

    def f(act, B_, H_, W_, lda, c_off, c_in, wp, c_out, kh, kw, mode, bias, residual, out_f32, out_f16, out_strides,
          **k):
        orig(act, B_, H_, W_, lda, c_off, c_in, wp, c_out, kh, kw, mode, bias, residual, out_f32, out_f16, out_strides, **k)
        s = 2 if mode == 6 else 1
        h0, h1 = band
        cut = act.clone()
        rows = cut.reshape(B_, -1, s * H_, cut.shape[-2], cut.shape[-1])      # [B, phases, input rows, W, C]
        rows[:, :, :s * h0] = 0
        rows[:, :, s * h1:] = 0
        o32 = None if out_f32 is None else torch.empty_like(out_f32)
        o16 = None if out_f16 is None else torch.empty_like(out_f16)
        orig(cut, B_, H_, W_, lda, c_off, c_in, wp, c_out, kh, kw, mode, bias, residual, o32, o16, out_strides)
        r = h0 if edge == "first" else h1 - 1
        for o, d in ((out_f32, o32), (out_f16, o16)):
            if o is not None:
                o[:, r] = d[:, r]
    return f


DEFECT_CASES = [(c, e) for c in CASES if c.startswith("conv ") for e in ("first", "last")
                if not (c.startswith("conv sub-pixel phase 2") and e == "last")      # phase 2 reads rows y - 1 and y
                and not (c.startswith("conv sub-pixel phase 5") and e == "first")]   # phase 5 reads rows y and y + 1


@pytest.mark.parametrize("case,edge", DEFECT_CASES)
def test_halo_defect_at_a_band_edge_fails(case, edge, monkeypatch):
    halo, per_row, _ = CASES[case]
    band = (ROWS, 2 * ROWS)                                             # the second band: a neighbour on either side
    emu = EmuOps()
    emu.conv_igemm = _halo_defect(emu, edge, band)
    proxy, n = _run(emu, case, per_row * (ROWS + 2 * halo), monkeypatch, strict=False)
    assert n > 2
    with pytest.raises(AssertionError) as e:
        proxy.raise_failures()
    print(f"\n{case}, {edge} row of band {band}: {str(e.value)[:200]}")
    assert all(f.startswith("conv_igemm(") for f in proxy.failures)
