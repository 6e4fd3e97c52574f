"""Time guidance with a negative prompt and per-image weights, and what a new `cond_scale` costs, on one GPU.

The workload's SR U-Net (cfg 3: 64 -> 256, b = 32) in a two-stage cascade whose small base stage never runs.  After one
warm-up of each, four things are alternated `--repeats` times, CUDA events around each:
  (a) the captured S-point DDIM loop guided by the null conditioning at `--cond-scale`;
  (b) the same loop guided by a negative prompt (its own random embeddings, same length) with a per-image weight vector
      (a sweep over [1, 2 * cond_scale - 1]): the guidance pass has the same shapes as (a)'s;
  (c) `Imagen.sample` (SR stage only, from random 64x64 images) at a weight that differs from the previous call's: it
      replays the graph (a) captured, it does not capture;
  (d) the same call on an Imagen over the same U-Nets right after its `clear_graphs()`: what every new weight cost when
      the weight was part of the graph key (warm-up and capture of the two-pass step, then the loop).
Writes nothing; prints one JSON line with the card's name and power limit.
Usage: python tools/bench_guidance.py [--workload cfg3] [--cond-scale 3] [--sampling-timesteps 50] [--repeats 3]
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
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_guidance.py needs a CUDA device"
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
    make = lambda: Imagen(unets=(base, u), text_encoder_name="t5_base" if wl["E"] == 768 else "t5_small",
                          image_sizes=(s // 4, s), timesteps=T, cond_drop_prob=0.1).eval().to(dev)
    im, fresh = make(), make()
    assert im.unets[1] is u and fresh.unets[1] is u
    inp = synth_inputs(wl, B, 1000)
    gen = torch.Generator().manual_seed(1)
    te, tm = inp["text_embeds"].to(dev), inp["text_mask"].to(dev)
    neg = (torch.randn(te.shape, generator=gen) * inp["text_mask"][..., None]).to(dev)
    start = torch.rand(B, 3, s // 4, s // 4, generator=gen).to(dev)
    lowres = inp["lowres_img01"].to(dev)                         # the loop normalises it
    lowres_t = torch.full((B,), int(0.2 * T), dtype=torch.long, device=dev)
    sch = im.noise_schedulers[1]
    walk = sch.sampling_schedule(S, 0., dev)
    sweep = torch.linspace(1., 2 * w - 1, B, device=dev)
    loop_kw = dict(noise_scheduler=sch, text_embeds=te, text_mask=tm, lowres_cond_img=lowres,
                   lowres_noise_times=lowres_t, schedule=walk)
    sample_kw = dict(text_embeds=te, text_masks=tm, sampling_timesteps=S, start_at_unet_number=2, start_images=start)
    calls = [0]

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    def new_scale():                       # a weight the previous call did not use
        calls[0] += 1
        return w + 0.25 * calls[0]

    def after_clear():
        fresh.clear_graphs()
        return fresh.sample(cond_scale=new_scale(), **sample_kw)

    runs = {"null_loop": lambda: im._p_sample_loop(u, (B, 3, s, s), cond_scale=w, **loop_kw),
            "negative_loop": lambda: im._p_sample_loop(u, (B, 3, s, s), cond_scale=sweep, negative_text_embeds=neg,
                                                       negative_text_mask=tm, **loop_kw),
            "new_scale_sample": lambda: im.sample(cond_scale=new_scale(), **sample_kw),
            "new_scale_after_clear": after_clear}
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
        assert len(im._graphs) == graphs, "a new cond_scale must replay the captured graph, not capture another"
    for name, out in outs.items():
        assert torch.isfinite(out).all(), name
    med = {k: statistics.median(v) for k, v in ms.items()}
    print(json.dumps({
        "workload": f"{args.workload}: {wl['desc']}", "device": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(), "sampling_timesteps": S, "cond_scale": w, "repeats": args.repeats,
        "captured_graphs": graphs,
        "null_loop_ms": ms["null_loop"], "negative_loop_ms": ms["negative_loop"],
        "new_scale_sample_ms": ms["new_scale_sample"], "new_scale_after_clear_ms": ms["new_scale_after_clear"],
        "negative_over_null_median": med["negative_loop"] / med["null_loop"],
        "recapture_cost_ms_median": med["new_scale_after_clear"] - med["new_scale_sample"]}))


if __name__ == "__main__":
    main()
