"""Micro-benchmarks of single kernels at the cfg-3 (SR 64->256, dim 128, batch 32) shapes.  GPU only.

Diagnostics for kernel tuning, not a bench value: CUDA events around `reps` back-to-back launches, rotating over enough
buffer sets that the working set exceeds the 50 MB L2 ("cold") or re-using one set ("warm").
Usage: python tools/bench_ops.py [gn ln linear step attn cast final stem]
       python tools/bench_ops.py conv [block_n ...]   (implicit-GEMM convs; block_n 0 = the library's choice; ends with
                                                       the k-block sweep and its per-tile cost fit)
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from minimagen_b200 import _native, ops as ops_mod   # noqa: E402

F16, F32, F64 = torch.float16, torch.float32, torch.float64
dev = torch.device("cuda", 0)

def _hbm_gbs():
    """HBM bandwidth of the roofline: MEASURED_PEAKS.json when present, else the H100 SXM data sheet (3.35 TB/s)."""
    import json
    try:
        return float(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                  "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 3350.0


HBM = _hbm_gbs()   # GB/s


def timeit(fn_list, reps=20):
    """fn_list: callables doing the same work on different buffers; returns ms per call."""
    for f in fn_list:
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(reps):
        fn_list[i % len(fn_list)]()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def report(name, ms_cold, ms_warm, nbytes):
    print(f"{name:44s} cold {ms_cold * 1e3:8.1f} us ({nbytes / ms_cold / 1e6:7.0f} GB/s, {nbytes / ms_cold / 1e6 / HBM * 100:5.1f}% HBM)"
          f"   warm {ms_warm * 1e3:8.1f} us   [{nbytes / 1e6:.0f} MB]", flush=True)


def bench_gn(ops):
    B = 32
    for (hw, c0, c1) in [(128 * 128, 128, 0), (128 * 128, 128, 128), (64 * 64, 256, 0), (64 * 64, 256, 256),
                         (32 * 32, 512, 0), (32 * 32, 512, 512), (16 * 16, 1024, 0), (16 * 16, 1024, 1024),
                         (256 * 256, 128, 0)]:
        C = c0 + c1
        n = B * hw * C
        nbytes = n * 6
        nset = max(1, int(300e6 // nbytes) + 1)
        sets = []
        for _ in range(nset):
            s0 = torch.randn(B, hw, c0, device=dev)
            s1 = torch.randn(B, hw, c1, device=dev) if c1 else None
            st0 = torch.rand(B, c0 // 16, 2, device=dev, dtype=F64) * hw * 16
            st0[..., 1] += hw * 16
            st1 = None
            if c1:
                st1 = torch.rand(B, c1 // 16, 2, device=dev, dtype=F64) * hw * 16
                st1[..., 1] += hw * 16
            out = torch.empty(B, hw, C, device=dev, dtype=F16)
            sets.append((s0, s1, st0, st1, out))
        gamma, beta = torch.randn(C, device=dev), torch.randn(C, device=dev)
        ss = torch.randn(B, 2 * C, device=dev)

        def mk(t):
            s0, s1, st0, st1, out = t
            return lambda: ops.gn_apply_silu(s0, c0, s1, c1, 0.7071, B, hw, 8, st0, 16, st1, 16 if c1 else 0, gamma, beta,
                                             ss, 2 * C, 1e-5, out)
        fns = [mk(t) for t in sets]
        report(f"gn_apply hw={hw} C={c0}+{c1}", timeit(fns), timeit(fns[:1]), nbytes)


def bench_ln(ops):
    for (rows, C) in [(8192, 1024), (32 * 59, 512)]:
        nbytes = rows * C * (4 + 2)
        nset = max(1, int(300e6 // nbytes) + 1)
        g, b = torch.randn(C, device=dev), torch.randn(C, device=dev)
        sets = [(torch.randn(rows, C, device=dev), torch.empty(rows, C, device=dev, dtype=F16)) for _ in range(nset)]
        fns = [(lambda t=t: ops.ln_rows(t[0], rows, C, g, b, 1e-5, 0, None, None, t[1])) for t in sets]
        report(f"ln_rows rows={rows} C={C} (f16 out)", timeit(fns), timeit(fns[:1]), nbytes)


def bench_linear(ops):
    for (M, K, Nn) in [(32, 512, 518 * 128), (32, 768, 1024), (32 * 59, 768, 128), (32, 512, 256), (32, 128, 512)]:
        x = torch.randn(M, K, device=dev)
        nbytes = Nn * K * 4 + M * K * 4 + M * Nn * 4
        nset = max(1, int(300e6 // nbytes) + 1)
        nset = min(nset, 8)
        sets = [(torch.randn(Nn, K, device=dev), torch.randn(Nn, device=dev), torch.empty(M, Nn, device=dev)) for _ in range(nset)]
        fns = [(lambda t=t: ops.linear_f32(x, M, K, t[0], t[1], Nn, 0, 0, None, t[2], None)) for t in sets]
        report(f"linear_f32 M={M} K={K} N={Nn}", timeit(fns), timeit(fns[:1]), nbytes)


def bench_step(ops):
    """The two selects sampling runs: the fused step epilogue at the cfg-3 step (cond_scale 1: no eps_null), and the
    single-CTA step_quantile of the three-kernel form that 3 x 1024 x 1024 images (cfg 5, batch 2) fall back to."""
    from minimagen_b200.Imagen import quantile_rank
    B, n = 32, 3 * 256 * 256
    x, eps, noise, out = (torch.randn(B, n, device=dev) for _ in range(4))
    t = torch.randint(0, 1000, (B,), device=dev)
    tab_a, tab_b, c1, c2, sigma = (torch.rand(1000, device=dev) for _ in range(5))
    lo, hi, w = quantile_rank(n, 0.9)
    f = lambda: ops.step_epilogue(x, eps, None, 1.0, t, tab_a, tab_b, c1, c2, sigma, noise, B, n, lo, hi, w, 1.0, out)
    ms = timeit([f], reps=500)                                              # ~150 us a launch: a window of tens of ms
    report(f"step_epilogue B={B} n={n}", ms, ms, B * n * 4 * 4)          # x_t, eps, noise in; out
    B, n = 2, 3 * 1024 * 1024
    x = torch.randn(B, n, device=dev)
    s = torch.empty(B, device=dev)
    lo, hi, w = quantile_rank(n, 0.9)
    f = lambda: ops.step_quantile(x, B, n, lo, hi, w, 1.0, s)
    ms = timeit([f])
    report(f"step_quantile B={B} n={n}", ms, ms, B * n * 4)


def bench_attn(ops):
    heads, d = 8, 64
    inner = heads * d
    for (B, n, m, shared) in [(32, 256, 256, True), (32, 256, 59, False), (64, 1024, 1024, True), (64, 4096, 4096, True),
                              (64, 1024, 258, False), (64, 4096, 258, False)]:
        q = torch.randn(B, n, inner, device=dev, dtype=F16) * 0.125
        out = torch.empty(B, n, inner, device=dev, dtype=F16)
        null_kv = torch.randn(2, d, device=dev)
        if shared:      # self-attention (layers.py:14-104): one shared k/v head (multi-query)
            kv = torch.randn(B, m, 2 * d, device=dev, dtype=F16)
            args = (kv, kv[..., d:], m * 2 * d, 2 * d, 0)
        else:           # cross-attention (layers.py:180-251): per-head k/v over m text tokens
            kv = torch.randn(B, m, 2 * inner, device=dev, dtype=F16)
            args = (kv, kv[..., inner:], m * 2 * inner, 2 * inner, d)
        fl = 4.0 * B * heads * n * (m + 1) * d
        res = []
        for tc in (True, False):
            ops.attention_tc = tc
            f = lambda: ops.attention(q, n * inner, inner, *args, null_kv, None, B, heads, n, m, out, n * inner, inner)
            ms = timeit([f], reps=5)
            res.append(f"{'wgmma' if tc else 'mma.sync'} {ms * 1e3:9.1f} us ({fl / ms / 1e9:6.1f} TFLOP/s)")
        ops.attention_tc = True
        print(f"attention B={B} n={n} m={m} {'multi-query' if shared else 'per-head kv'}:  " + "   ".join(res), flush=True)


def bench_cast(ops):
    B = 32
    for (H, c0, c1, mode) in [(128, 128, 0, 2), (64, 256, 0, 2), (64, 256, 0, 1), (128, 128, 0, 1), (32, 512, 0, 1), (16, 1024, 0, 1)]:
        C = c0 + c1
        n = B * H * H * C
        mult = 4 if mode == 1 else 1
        nbytes = n * 2 + n * 2 * mult
        src = torch.randn(B, H, H, c0, device=dev, dtype=F16)
        out = torch.empty(B * mult, H, H, C, device=dev, dtype=F16)
        f = lambda: ops.cast_act(src, c0, None, 0, 1.0, B, H, H, mode, out)
        ms = timeit([f])
        report(f"cast_act f16->f16 H={H} C={C} mode={mode}", ms, ms, nbytes)


def bench_final(ops):
    B, H, C = 32, 256, 128
    act = torch.randn(B, H, H, C, device=dev, dtype=F16)
    w = torch.randn(16, C, 3, 3, device=dev)
    w[3:] = 0
    wp = ops.pack_conv_weight(w)
    bias = torch.zeros(16, device=dev)
    out = torch.empty(B, 3, H, H, device=dev)
    f = lambda: ops.conv_igemm(act, B, H, H, C, 0, C, wp, 16, 3, 3, 0, bias, None, out, None, (3 * H * H, H, 1),
                               out_sc=H * H, n_valid=3)
    ms = timeit([f])
    report("final_conv 3x3 128->3 (N=16) 256x256 b32", ms, ms, B * H * H * C * 2 + B * 3 * H * H * 4)


def bench_stem(ops):
    B, H = 32, 256
    a, b = torch.randn(B, 3, H, H, device=dev), torch.randn(B, 3, H, H, device=dev)
    out = torch.empty(B, H, H, 128, device=dev, dtype=F16)
    f = lambda: ops.stem_unroll(a, 3, b, 3, B, H, H, out)
    ms = timeit([f])
    report("stem_unroll 6ch -> 128-wide f16, 256x256 b32", ms, ms, B * H * H * (6 * 4 + 128 * 2))


# cfg-3 conv shape classes at b=32: (label, H=W, C_in of source 0, C_in of source 1 (virtual concat), C_out, kernel)
CONV_SHAPES = [("3x3 1024->1024 @16", 16, 1024, 0, 1024, 3), ("3x3 2048->1024 @16 concat", 16, 1024, 1024, 1024, 3),
               ("3x3 512->512 @32", 32, 512, 0, 512, 3), ("3x3 1024->512 @32", 32, 1024, 0, 512, 3),
               ("3x3 256->256 @64", 64, 256, 0, 256, 3), ("3x3 512->256 @64", 64, 512, 0, 256, 3),
               ("3x3 128->128 @256", 256, 128, 0, 128, 3), ("3x3 128->128 @128", 128, 128, 0, 128, 3),
               ("3x3 256->128 @128", 128, 256, 0, 128, 3), ("1x1 1024->512 @32", 32, 1024, 0, 512, 1)]


def conv_tile(c_out, pixels, hint, num_sms):
    """(label, pixels per tile, output channels per tile) of the schedule conv_tc.cu's conv_tc_launch selects, for the
    shapes here (C_out % 64 == 0, grids that tile by 256 pixels inside one image): the transposed tile "t256" (256 pixels
    x 128 channels) at C_out = 128 for the hint 256, or without a hint when it gives every SM a tile; else the 128-pixel
    tile of the width the hint or pick_block_n selects."""
    hint = abs(hint)
    if c_out == 128 and (hint == 256 or ((hint == 0 or c_out % hint) and pixels // 256 >= num_sms)):
        return "t256", 256, 128
    if hint and c_out % hint == 0:
        return f"n{hint}", 128, hint
    for bn in (256, 128):
        if c_out % bn == 0 and pixels // 128 * (c_out // bn) >= num_sms:
            return f"n{bn}", 128, bn
    return "n64", 128, 64


# k-block sweep: 3x3 convs at b=32 whose k-blocks per tile (9 C_in / 64) run from 9 to 72, at the two cfg-3 geometries
# of the short-K layers; per-tile time against k-blocks fits a line whose intercept is the cost paid once per tile
SWEEP_SHAPES = [(128, 128, (64, 128, 256, 512)), (64, 256, (64, 128, 256, 512))]   # (H = W, C_out, C_in sweep)


def conv_operand_bytes(pixels, c_out, k_blocks, tile_px, tile_ch):
    """L2 -> SM operand bytes of one launch: per tile and k-block one TMA stage, a tile_px x 64 activation box and a
    tile_ch x 64 weight box."""
    return pixels // tile_px * (c_out // tile_ch) * k_blocks * (tile_px + tile_ch) * 64 * 2


def bench_conv(ops, hints=(0,)):
    """Usage: bench_ops.py conv [block_n ...] -- 0 = the library's own choice (default); 256 runs the C_out = 128 shapes on
    the transposed tile, 128 on the 128-wide ping-pong one."""
    B = 32
    num_sms = torch.cuda.get_device_properties(dev).multi_processor_count
    rows = [(lbl, H, c0, c1, co, k, False) for (lbl, H, c0, c1, co, k) in CONV_SHAPES]
    rows.append(("3x3 512->512 @32 + res 1x1 1024 concat", 32, 512, 0, 512, 3, True))
    for (lbl, H, c0, c1, c_out, k, res) in rows:
        c_in = c0 + c1
        act = torch.randn(B, H, H, c0, device=dev).to(F16)
        act2 = torch.randn(B, H, H, c1, device=dev).to(F16) if c1 else None
        out = torch.empty(B, H, H, c_out, device=dev, dtype=F16)
        stats = torch.zeros(B, c_out // 16, 2, device=dev, dtype=F64)
        bias = torch.randn(c_out, device=dev)
        k_blocks = k * k * c_in // 64
        flop = 2.0 * B * H * H * c_out * k * k * c_in
        if res:
            x = torch.randn(B, H, H, 512, device=dev).to(F16)
            x2 = torch.randn(B, H, H, 512, device=dev).to(F16)
            wp = torch.randn(c_out, 9 * c_in + 1024, device=dev).to(F16) * 0.01
            k_blocks += 1024 // 64
            flop += 2.0 * B * H * H * c_out * 1024
        else:
            wp = torch.randn(c_out, k * k * c_in, device=dev).to(F16) * 0.01
        res_line = []
        for hint in ((0,) if res else hints):        # the folded res_conv takes no hint
            if res:
                f = lambda: ops.conv_res1x1(act, B, H, H, c_in, c_in, None, 0, 0, x, 512, 1024, x2, 512, 512, wp, c_out,
                                            bias, None, None, out, stats)
            else:
                f = lambda hint=hint: ops.conv_igemm(act, B, H, H, c0, 0, c_in, wp, c_out, k, k, 0, bias, None, None, out,
                                                     (H * H * c_out, H * c_out, c_out), block_n=hint, act2=act2, lda2=c1,
                                                     c_in1=c0 if c1 else 0, out_stats=stats)
            ms = timeit([f], reps=20)
            lbl_t, tpx, tch = conv_tile(c_out, B * H * H, hint, num_sms)
            nbytes = conv_operand_bytes(B * H * H, c_out, k_blocks, tpx, tch)
            res_line.append(f"{lbl_t:4s} {ms * 1e3:8.1f} us {flop / ms / 1e9:6.1f} TFLOP/s L2->SM {nbytes / ms / 1e9:5.2f} TB/s")
        print(f"conv {lbl:40s} " + "  |  ".join(res_line), flush=True)
    bench_conv_phases(ops, hints, num_sms)
    bench_conv_sweep(ops, hints, num_sms)


def bench_conv_phases(ops, hints, num_sms):
    """One sub-pixel phase of the Upsample conv (2x2 taps on the low-res grid, every second pixel of every second row of
    the 2H x 2W output), with the fp16 + statistics epilogue: the cfg-3 classes 128->128 onto 256x256 and 256->128 onto
    128x128."""
    B, c_out = 32, 128
    for (H, c_in) in ((128, 128), (64, 256)):
        act = torch.randn(B, H, H, c_in, device=dev).to(F16)
        wp = (torch.randn(c_out, 4 * c_in, device=dev) * 0.01).to(F16)
        bias = torch.randn(c_out, device=dev)
        out = torch.empty(B, 2 * H, 2 * H, c_out, device=dev, dtype=F16)
        stats = torch.zeros(B, c_out // 16, 2, device=dev, dtype=F64)
        flop = 2.0 * B * H * H * c_out * 4 * c_in
        line = []
        for hint in hints:
            f = lambda hint=hint: ops.conv_igemm(act, B, H, H, c_in, 0, c_in, wp, c_out, 2, 2, 2, bias, None, None, out,
                                                 (4 * H * H * c_out, 4 * H * c_out, 2 * c_out), block_n=hint,
                                                 out_stats=stats)
            ms = timeit([f], reps=20)
            lbl_t = conv_tile(c_out, B * H * H, hint, num_sms)[0]
            line.append(f"{lbl_t:4s} {ms * 1e3:8.1f} us {flop / ms / 1e9:6.1f} TFLOP/s")
        print(f"conv sub-pixel phase {c_in}->{c_out} onto {2 * H}x{2 * H}{'':14s} " + "  |  ".join(line), flush=True)


def bench_conv_sweep(ops, hints, num_sms):
    """Per-tile cost against k-blocks per tile, with the fp16 + statistics epilogue most convs write ("f16") and with what
    ResnetBlock.block2 writes ("block2": bias, fp32 residual in, fp32 + fp16 out, statistics).  us/tile is the launch time
    over its tiles per SM; the fit per (shape, epilogue, width) is  us/tile = F + c * k-blocks."""
    import numpy as np
    B = 32
    for (H, c_out, c_ins) in SWEEP_SHAPES:
        for epi in ("f16", "block2"):
            pts = {}
            for c_in in c_ins:
                act = torch.randn(B, H, H, c_in, device=dev).to(F16)
                wp = (torch.randn(c_out, 9 * c_in, device=dev) * 0.01).to(F16)
                bias = torch.randn(c_out, device=dev)
                out16 = torch.empty(B, H, H, c_out, device=dev, dtype=F16)
                stats = torch.zeros(B, c_out // 16, 2, device=dev, dtype=F64)
                res = torch.randn(B, H, H, c_out, device=dev) if epi == "block2" else None
                out32 = torch.empty(B, H, H, c_out, device=dev) if epi == "block2" else None
                k_blocks = 9 * c_in // 64
                line = []
                for hint in hints:
                    lbl_t, tpx, tch = conv_tile(c_out, B * H * H, hint, num_sms)
                    f = lambda hint=hint: ops.conv_igemm(act, B, H, H, c_in, 0, c_in, wp, c_out, 3, 3, 0, bias, res, out32,
                                                         out16, (H * H * c_out, H * c_out, c_out), block_n=hint,
                                                         out_stats=stats)
                    ms = timeit([f], reps=20)
                    per_tile = ms * 1e3 / (B * H * H // tpx * (c_out // tch) / num_sms)
                    pts.setdefault((hint, lbl_t), []).append((k_blocks, per_tile))
                    line.append(f"{lbl_t:4s} {ms * 1e3:8.1f} us {per_tile:6.2f} us/tile "
                                f"{2.0 * B * H * H * c_out * 9 * c_in / ms / 1e9:6.1f} TFLOP/s")
                print(f"conv sweep 3x3 {c_in:4d}->{c_out} @{H} {epi:6s} kb={k_blocks:3d} " + "  |  ".join(line), flush=True)
            for (hint, lbl_t), p in sorted(pts.items()):
                kb, us = np.array(p).T
                c, F = np.polyfit(kb, us, 1)
                print(f"conv sweep fit C_out={c_out} @{H} {epi:6s} {lbl_t:4s}{'' if hint else ' (auto)'}: F = {F:5.2f} us/tile, "
                      f"{c:5.3f} us per k-block",
                      flush=True)


def main():
    _native.load()
    ops = ops_mod.get_ops()
    which = sys.argv[1:] or ["gn", "ln", "linear", "step", "attn", "cast", "final", "stem"]
    if which[0] == "conv":           # conv [block_n ...]
        with torch.no_grad():
            bench_conv(ops, tuple(int(h) for h in which[1:]) or (0,))
        return
    table = {"gn": bench_gn, "ln": bench_ln, "linear": bench_linear, "step": bench_step, "attn": bench_attn,
             "cast": bench_cast, "final": bench_final, "stem": bench_stem}
    with torch.no_grad():
        for w in which:
            table[w](ops)


if __name__ == "__main__":
    main()
