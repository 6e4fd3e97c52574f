"""Micro-benchmark: conv weight gradient, wgmma kernel (csrc/wgrad_tc.cu) vs the fp32 CUDA-core kernel (csrc/backward.cu)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from minimagen_b200.ops import NativeOps

ops = NativeOps()
shapes = [(8, 64, 64, 128, 128, 3), (8, 32, 32, 256, 256, 3), (8, 16, 16, 512, 512, 3), (8, 32, 32, 512, 256, 3),
          (8, 64, 64, 256, 128, 3), (8, 64, 64, 128, 128, 1), (32, 128, 128, 128, 128, 3)]
for B, H, W, ci, co, k in shapes:
    x = torch.randn(B, H, W, ci, device="cuda"); dy = torch.randn(B, H, W, co, device="cuda")
    x16, dy16 = x.half(), dy.half()
    dw = torch.empty(co, ci, k, k, device="cuda"); dw2 = torch.empty_like(dw)
    def t(fn, n=5):
        fn(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n): fn()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n
    t_tc = t(lambda: ops.conv_wgrad_tc(dy16, x16, B, H, W, ci, co, k, k, dw))
    t_f32 = t(lambda: ops.conv_wgrad(dy, x, B, H, W, ci, H, W, co, k, k, 1, k // 2, dw2), n=2)
    fl = 2.0 * B * H * W * ci * co * k * k
    err = float((dw - dw2).norm() / dw2.norm())
    print(f"B{B} {H}x{W} {ci}->{co} k{k}: tc {t_tc:.3f} ms ({fl / t_tc / 1e9:.0f} TFLOP/s)  fp32 {t_f32:.3f} ms ({fl / t_f32 / 1e9:.1f} TFLOP/s)  rel diff {err:.2e}", flush=True)
