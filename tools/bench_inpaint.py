"""Time inpainting with RePaint resampling against text-only sampling on one GPU.

One whole captured inpainting loop -- (S - 1) * R + 1 replays of the inpainting step graph (`Imagen.sample(...,
sampling_timesteps=S, inpaint_images=, inpaint_masks=, inpaint_resample_times=R)`: three draws, mi_inpaint_prologue, the
U-Net and step epilogue, mi_inpaint_advance) -- against S replays of the respaced text-only step graph of the same
workload, alternated `--repeats` times after one warm-up loop each, CUDA events around each loop.  The inpainting loop
runs more U-Net evaluations by design, so the comparison is per U-Net evaluation (one per replay at cond_scale 1): the
ratio is the cost of the two extra draws and the prologue.  Writes nothing; prints one JSON line.
Usage: python tools/bench_inpaint.py [--workload cfg3] [--sampling-timesteps 50] [--resample 2] [--eta 0] [--repeats 3]
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
    ap.add_argument("--resample", type=int, default=2)
    ap.add_argument("--eta", type=float, default=0.)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_inpaint.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)

    from minimagen_b200 import _native
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import BaseTest, Unet
    from minimagen_b200.ops import get_ops
    _native.load()
    wl = workload(args.workload)
    B, T, S, R = wl["batch"], wl["T"], args.sampling_timesteps, args.resample
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
    gen = torch.Generator(device=dev).manual_seed(1)
    known = torch.rand(shape, generator=gen, device=dev) * 2 - 1                      # normalised known image
    mask = (torch.rand((B, shape[2] * shape[3]), generator=gen, device=dev) < 0.5).float()
    sched = sch.sampling_schedule(S, args.eta, dev)
    n_iter = {"inpaint": (S - 1) * R + 1, "respaced": S}

    with torch.no_grad():
        kw = dict(noise_scheduler=sch, cond_scale=1.0, schedule=sched, **ckw)
        graphs = {"inpaint": im._step_graph(u, shape, inpaint=(known, mask, R), **kw),
                  "respaced": im._step_graph(u, shape, **kw)}

        def loop(name):
            """One whole loop from x_T at t = T-1; returns ms."""
            g = graphs[name]
            g.x.copy_(x)
            g.t.fill_(T - 1)
            if g.inp is not None:
                g.inp["r"].zero_()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n_iter[name]):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1)

        for name in graphs:
            loop(name)                                            # warm-up loop
        ms = {k: [] for k in graphs}
        for _ in range(args.repeats):
            for name in graphs:
                ms[name].append(loop(name))
        gi = graphs["inpaint"]
        assert torch.isfinite(gi.x).all() and int(gi.t.max()) == 0 and int(gi.inp["r"].max()) == 0, \
            "the inpainting loop did not end at t = 0, r = 0"
        assert int(graphs["respaced"].t.max()) == 0, "the respaced loop did not reach t = 0"

    per_eval = {k: [v / n_iter[k] for v in vals] for k, vals in ms.items()}
    print(json.dumps({
        "workload": f"{args.workload}: {wl['desc']}", "device": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(), "sampling_timesteps": S, "resample_times": R, "ddim_eta": args.eta,
        "repeats": args.repeats, "inpaint_unet_evals": n_iter["inpaint"], "inpaint_loop_ms": ms["inpaint"],
        "inpaint_ms_per_eval": per_eval["inpaint"], "respaced_ms_per_eval": per_eval["respaced"],
        "ratio_median": statistics.median(i / r for i, r in zip(per_eval["inpaint"], per_eval["respaced"]))}))


if __name__ == "__main__":
    main()
