"""Time fewer-step DDIM sampling against the DDPM step on one GPU.

One whole captured sampling loop of S replays of the respaced step graph (`Imagen.sample(..., sampling_timesteps=S)`,
DDIM tables, t advanced through next_t) against S replays of the DDPM step graph of the same workload, alternated
`--repeats` times after one warm-up loop each, CUDA events around each loop.  The two loops run the same U-Net launches
and the same fused step epilogue; only the timestep-advance kernel differs.  Writes nothing; prints one JSON line.
Usage: python tools/bench_respaced.py [--workload cfg3] [--sampling-timesteps 50] [--eta 0] [--repeats 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True            # leave the tree as it is (no __pycache__ for bench.py)
from bench import make_cond, workload   # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--sampling-timesteps", type=int, default=50)
    ap.add_argument("--eta", type=float, default=0.)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_respaced.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)

    from minimagen_b200 import _native
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import BaseTest, Unet
    from minimagen_b200.ops import get_ops
    _native.load()
    wl = workload(args.workload)
    B, T, S = wl["batch"], wl["T"], args.sampling_timesteps
    shape = (B, 3, wl["size"], wl["size"])
    torch.manual_seed(0)
    with torch.device(dev):
        u = Unet(**wl["cfg"]).eval()
        # an SR U-Net sits behind a base stage (Imagen treats unets[0] as the base model); the stand-in never runs
        stages = (Unet(**dict(BaseTest.defaults, text_embed_dim=wl["E"])).eval(), u) if wl["lowres"] else (u,)
    sizes = (wl["size"] // 4, wl["size"]) if wl["lowres"] else (wl["size"],)
    im = Imagen(unets=stages, text_encoder_name="t5_base" if wl["E"] == 768 else "t5_small", image_sizes=sizes,
                timesteps=T, cond_drop_prob=0.1).eval().to(dev)
    assert im.unets[-1] is u
    sch = im.noise_schedulers[-1]
    inp, ckw = make_cond(dict(wl, name=args.workload), B, 1000, dev, sch, get_ops())
    x = inp["x"].to(dev)

    with torch.no_grad():
        graphs = {"ddpm": im._step_graph(u, shape, noise_scheduler=sch, cond_scale=1.0, **ckw),
                  "respaced": im._step_graph(u, shape, noise_scheduler=sch, cond_scale=1.0, respaced=True, **ckw)}
        graphs["respaced"].set_schedule(sch.sampling_schedule(S, args.eta, dev))

        def loop(g):
            """S replays from x_T at t = T-1; returns ms."""
            g.x.copy_(x)
            g.t.fill_(T - 1)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(S):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1)

        for g in graphs.values():
            loop(g)                                               # warm-up loop
        ms = {k: [] for k in graphs}
        for _ in range(args.repeats):
            for k, g in graphs.items():
                ms[k].append(loop(g))
        gr = graphs["respaced"]
        assert torch.isfinite(gr.x).all() and int(gr.t.max()) == 0, "the respaced loop did not reach t = 0"
        assert int(graphs["ddpm"].t.min()) == T - 1 - S, "the DDPM loop did not take S steps"

    per_step = {k: [v / S for v in vals] for k, vals in ms.items()}
    print(json.dumps({
        "workload": f"{args.workload}: {wl['desc']}", "device": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(), "sampling_timesteps": S, "ddim_eta": args.eta, "repeats": args.repeats,
        "respaced_loop_ms": ms["respaced"], "respaced_ms_per_step": per_step["respaced"],
        "ddpm_ms_per_step": per_step["ddpm"],
        "ratio_median": statistics.median(r / d for r, d in zip(per_step["respaced"], per_step["ddpm"]))}))


if __name__ == "__main__":
    main()
