"""Time per-image seeds (keyed noise drawn on the device) against torch's generator, on one GPU.

  (a) The workload's SR U-Net (cfg 3: 64 -> 256, b = 32) in the captured S-point DDIM loop at `--cond-scale`, seeded
      (mi_randn_keyed inside the step graph) and unseeded (normal_ inside it), after one warm-up of each alternated
      `--repeats` times with CUDA events around each loop; reports the median ratio.
  (b) mi_randn_keyed alone against torch's `normal_` on one [b, 3, 256, 256] fp32 draw: CUDA events around `--launches`
      back-to-back launches of each, in µs per launch and achieved GB/s of writes against the H100 SXM data-sheet
      3.35 TB/s.
Writes nothing; prints one JSON line with the card's name and power limit.
Usage: python tools/bench_seeded.py [--workload cfg3] [--cond-scale 3] [--sampling-timesteps 50] [--repeats 3]
                                    [--launches 2000]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True            # leave the tree as it is (no __pycache__ for bench.py)
from bench import synth_inputs, workload   # noqa: E402
from tools.bench_inpaint import power_limit_w   # noqa: E402

HBM_BYTES_PER_S = 3.35e12                 # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--cond-scale", type=float, default=3.)
    ap.add_argument("--sampling-timesteps", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--launches", type=int, default=2000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_seeded.py needs a CUDA device"
    assert args.launches >= 1000, "time at least 1000 launches of each draw"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)

    from minimagen_b200 import _native
    from minimagen_b200.Imagen import NOISE_KINDS, Imagen
    from minimagen_b200.Unet import BaseTest, Unet
    from minimagen_b200.ops import get_ops
    _native.load()
    wl = workload(args.workload)
    assert wl["lowres"], f"{args.workload} is not a super-resolution workload"
    B, T, S, s, w = wl["batch"], wl["T"], args.sampling_timesteps, wl["size"], args.cond_scale
    torch.manual_seed(0)
    with torch.device(dev):
        u = Unet(**wl["cfg"]).eval()
        base = Unet(**dict(BaseTest.defaults, text_embed_dim=wl["E"])).eval()
    im = Imagen(unets=(base, u), text_encoder_name="t5_base" if wl["E"] == 768 else "t5_small",
                image_sizes=(s // 4, s), timesteps=T, cond_drop_prob=0.1).eval().to(dev)
    inp = synth_inputs(wl, B, 1000)
    te, tm = inp["text_embeds"].to(dev), inp["text_mask"].to(dev)
    lowres = inp["lowres_img01"].to(dev)                         # the loop normalises it
    lowres_t = torch.full((B,), int(0.2 * T), dtype=torch.long, device=dev)
    sch = im.noise_schedulers[1]
    walk = sch.sampling_schedule(S, 0., dev)
    seeds = torch.arange(1000, 1000 + B, dtype=torch.long, device=dev)
    loop_kw = dict(noise_scheduler=sch, text_embeds=te, text_mask=tm, lowres_cond_img=lowres,
                   lowres_noise_times=lowres_t, schedule=walk, cond_scale=w)
    shape = (B, 3, s, s)

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    runs = {"unseeded_loop": lambda: im._p_sample_loop(u, shape, **loop_kw),
            "seeded_loop": lambda: im._p_sample_loop(u, shape, seeds=seeds, stage=2, **loop_kw)}
    outs = {}
    with torch.no_grad():
        for name, fn in runs.items():                              # warm-up: captures the two graphs
            outs[name] = fn()
        graphs = len(im._graphs)
        ms = {k: [] for k in runs}
        for _ in range(args.repeats):
            for name, fn in runs.items():
                t, outs[name] = timed(fn)
                ms[name].append(t)
        assert len(im._graphs) == graphs == 2
    for name, out in outs.items():
        assert torch.isfinite(out).all(), name

    # (b) one draw of the step's shape, alone
    ops = get_ops()
    n = 3 * s * s
    buf = torch.empty(shape, dtype=torch.float32, device=dev)
    draws = {"randn_keyed": lambda: ops.randn_keyed(buf, seeds, B, n, NOISE_KINDS["step"], 2, label=999),
             "torch_normal": lambda: buf.normal_()}
    us = {}
    for name, fn in draws.items():
        for _ in range(20):
            fn()

        def many():
            for _ in range(args.launches):
                fn()
        t, _ = timed(many)
        us[name] = 1e3 * t / args.launches
    nbytes = buf.numel() * 4
    gbs = {k: nbytes / (v * 1e-6) / 1e9 for k, v in us.items()}
    med = {k: statistics.median(v) for k, v in ms.items()}
    print(json.dumps({
        "workload": f"{args.workload}: {wl['desc']}", "device": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(), "sampling_timesteps": S, "cond_scale": w, "repeats": args.repeats,
        "unseeded_loop_ms": ms["unseeded_loop"], "seeded_loop_ms": ms["seeded_loop"],
        "seeded_over_unseeded_median": med["seeded_loop"] / med["unseeded_loop"],
        "draw_shape": list(shape), "draw_mbytes": nbytes / 1e6, "launches": args.launches,
        "randn_keyed_us": us["randn_keyed"], "torch_normal_us": us["torch_normal"],
        "randn_keyed_gbs": gbs["randn_keyed"], "torch_normal_gbs": gbs["torch_normal"],
        "randn_keyed_share_of_3_35_tbs": gbs["randn_keyed"] * 1e9 / HBM_BYTES_PER_S,
        "torch_normal_share_of_3_35_tbs": gbs["torch_normal"] * 1e9 / HBM_BYTES_PER_S}))


if __name__ == "__main__":
    main()
