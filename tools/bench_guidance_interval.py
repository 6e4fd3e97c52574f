"""Time guidance intervals and guidance-weight schedules (Imagen.sample(guidance_interval=, guidance_schedule=)) on one GPU.

The workload's SR U-Net (cfg 3: 64 -> 256, b = 32) at cond_scale 3, a captured S-point DDIM loop (eta = 0).  After one
warm-up of each (which captures the graphs), three loops are alternated `--repeats` times, CUDA events around each:
  full      guidance at every point (no table: today's loop);
  interval  guidance only where sigma_lo < sigma_t <= sigma_hi (`--interval`, default (0.25, 5.5]: k = 25 of the 50
            points), the other points without the guidance pass -- with unbatched guidance a loop that guides k of S
            points is expected to take about (S + k) / (2 S) of the full loop;
  linear    the 'linear' weight schedule, no interval: guided at every point but the first (where the ramp is 0), through
            mi_step_epilogue_ws -- expected (2 S - 1) / (2 S) of the full loop if the scheduled epilogue costs nothing.
Writes nothing; prints one JSON line with the card's name and power limit.
Usage: python tools/bench_guidance_interval.py [--workload cfg3] [--sampling-timesteps 50] [--interval 0.25 5.5]
                                               [--repeats 3]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--cond-scale", type=float, default=3.)
    ap.add_argument("--sampling-timesteps", type=int, default=50)
    ap.add_argument("--interval", type=float, nargs=2, default=(0.25, 5.5))
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_guidance_interval.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)

    from minimagen_b200 import _native
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import BaseTest, Unet
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
    im.max_cached_graphs = 8
    inp = synth_inputs(wl, B, 1000)
    te, tm = inp["text_embeds"].to(dev), inp["text_mask"].to(dev)
    lowres = inp["lowres_img01"].to(dev)                         # the loop normalises it
    lowres_t = torch.full((B,), int(0.2 * T), dtype=torch.long, device=dev)
    sch = im.noise_schedulers[1]
    walk = sch.sampling_schedule(S, 0., dev)
    interval = tuple(args.interval)
    tables = {"full": None, "interval": sch.guidance_table(interval, None, dev),
              "linear": sch.guidance_table(None, "linear", dev)}
    guided = {k: S if v is None else sum(bool(v[t] != 0) for t in walk.grid) for k, v in tables.items()}
    loop_kw = dict(noise_scheduler=sch, text_embeds=te, text_mask=tm, lowres_cond_img=lowres, lowres_noise_times=lowres_t,
                   schedule=walk, cond_scale=w)

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    runs = {k: (lambda tab=tab: im._p_sample_loop(u, (B, 3, s, s), guidance_table=tab, **loop_kw))
            for k, tab in tables.items()}
    outs = {}
    with torch.no_grad():
        for name, fn in runs.items():                              # warm-up: captures the graphs
            outs[name] = fn()
        graphs = len(im._graphs)
        ms = {k: [] for k in runs}
        for _ in range(args.repeats):
            for name, fn in runs.items():
                t, outs[name] = timed(fn)
                ms[name].append(t)
        assert len(im._graphs) == graphs, "a repeat must replay the captured graphs, not capture others"
    for name, out in outs.items():
        assert torch.isfinite(out).all(), name
    med = {k: statistics.median(v) for k, v in ms.items()}
    print(json.dumps({
        "workload": f"{args.workload}: {wl['desc']}", "device": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(), "sampling_timesteps": S, "cond_scale": w, "repeats": args.repeats,
        "interval": interval, "guided_points": guided, "captured_graphs": graphs,
        "full_ms": ms["full"], "interval_ms": ms["interval"], "linear_ms": ms["linear"],
        "interval_over_full_median": med["interval"] / med["full"],
        "interval_expected": (S + guided["interval"]) / (2 * S),
        "linear_over_full_median": med["linear"] / med["full"],
        "linear_expected": (S + guided["linear"]) / (2 * S)}))


if __name__ == "__main__":
    main()
