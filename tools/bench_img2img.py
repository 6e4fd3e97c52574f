"""Time SR-only and image-to-image sampling (`Imagen.sample(..., start_at_unet_number=2, start_images=)`) on one GPU.

A two-stage cascade whose SR stage is the workload's U-Net (cfg 3: 64 -> 256, b = 32) and whose base stage, a small U-Net,
never runs: every call starts at the SR stage from random 64x64 start images.  Three things are alternated `--repeats`
times after one warm-up each, CUDA events around each:
  (a) `Imagen.sample` end to end with DDIM over S points (the resize, the low-res augmentation, the loop, the finalize);
  (b) the same with `init_images` (random 256x256) and `skip_steps` = `--skip`, so S - skip points from a noised image;
  (c) the bare captured loop, S replays of the cached step graph from x_T.
(a) - (c) is the per-call cost outside the loop.  Writes nothing; prints one JSON line with the card's name and power
limit.
Usage: python tools/bench_img2img.py [--workload cfg3] [--cond-scale 3] [--sampling-timesteps 50] [--skip 25] [--repeats 3]
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
    ap.add_argument("--skip", type=int, default=25)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_img2img.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)

    from minimagen_b200 import _native
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import BaseTest, Unet
    _native.load()
    wl = workload(args.workload)
    assert wl["lowres"], f"{args.workload} is not a super-resolution workload"
    B, T, S, s = wl["batch"], wl["T"], args.sampling_timesteps, wl["size"]
    torch.manual_seed(0)
    with torch.device(dev):
        u = Unet(**wl["cfg"]).eval()
        base = Unet(**dict(BaseTest.defaults, text_embed_dim=wl["E"])).eval()
    im = Imagen(unets=(base, u), text_encoder_name="t5_base" if wl["E"] == 768 else "t5_small",
                image_sizes=(s // 4, s), timesteps=T, cond_drop_prob=0.1).eval().to(dev)
    assert im.unets[1] is u
    inp = synth_inputs(wl, B, 1000)
    gen = torch.Generator().manual_seed(1)
    start = torch.rand(B, 3, s // 4, s // 4, generator=gen).to(dev)
    init = torch.rand(B, 3, s, s, generator=gen).to(dev)
    x = inp["x"].to(dev)
    kw = dict(text_embeds=inp["text_embeds"].to(dev), text_masks=inp["text_mask"].to(dev), cond_scale=args.cond_scale,
              sampling_timesteps=S, start_at_unet_number=2, start_images=start)

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    def bare_loop():
        g = next(iter(im._graphs.values()))
        g.x.copy_(x)
        g.t.fill_(T - 1)
        for _ in range(S):
            g.replay()

    runs = {"sr_only": lambda: im.sample(**kw),
            "img2img": lambda: im.sample(init_images=init, skip_steps=args.skip, **kw),
            "bare_loop": bare_loop}
    outs = {}
    with torch.no_grad():
        for name in runs:                                         # warm-up: captures the step graph on the first call
            outs[name] = runs[name]()
        assert len(im._graphs) == 1, "SR-only and image-to-image calls share one captured step graph"
        ms = {k: [] for k in runs}
        for _ in range(args.repeats):
            for name, fn in runs.items():
                ms[name].append(timed(fn))
    for name in ("sr_only", "img2img"):
        assert outs[name].shape == (B, 3, s, s) and torch.isfinite(outs[name]).all(), name
    med = {k: statistics.median(v) for k, v in ms.items()}
    print(json.dumps({
        "workload": f"{args.workload}: {wl['desc']}", "device": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(), "sampling_timesteps": S, "skip_steps": args.skip, "cond_scale": args.cond_scale,
        "repeats": args.repeats, "sr_only_sample_ms": ms["sr_only"], "img2img_sample_ms": ms["img2img"],
        "bare_loop_ms": ms["bare_loop"], "step_ms_median": med["bare_loop"] / S,
        "sample_overhead_ms_median": med["sr_only"] - med["bare_loop"],
        "img2img_over_sr_only_median": med["img2img"] / med["sr_only"]}))


if __name__ == "__main__":
    main()
