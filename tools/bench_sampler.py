"""Time DPM-Solver++(2M) sampling against DDIM (eta = 0) on one GPU.

One whole captured 2M loop -- S replays of the multistep step graph (`Imagen.sample(..., sampling_timesteps=S,
sampler='dpmpp_2m')`: the draw, the U-Net pass(es) and mi_step_epilogue_multistep, mi_step_advance_t_table) -- against S
replays of the text-only step graph walking DDIM's grid at eta = 0, same workload and guidance, alternated `--repeats`
times after one warm-up loop each, CUDA events around each loop.  Both loops make S U-Net evaluations (2S with unbatched
guidance), so the comparison is per U-Net evaluation: the ratio is the cost of the history read and write.  Writes
nothing; prints one JSON line with the card's name and power limit.
Usage: python tools/bench_sampler.py [--workload cfg3] [--cond-scale 3] [--sampling-timesteps 20] [--repeats 5]
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
from bench import make_cond, workload   # noqa: E402
from tools.bench_inpaint import power_limit_w   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--cond-scale", type=float, default=3.)
    ap.add_argument("--sampling-timesteps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_sampler.py needs a CUDA device"
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
    walks = {"dpmpp_2m": sch.dpm_solver_schedule(S, dev), "ddim": sch.sampling_schedule(S, 0., dev)}
    evals = S * (2 if args.cond_scale != 1 and not im.cfg_batched else 1)

    with torch.no_grad():
        kw = dict(noise_scheduler=sch, cond_scale=args.cond_scale, **ckw)
        graphs = {}
        for name, walk in walks.items():
            graphs[name] = im._step_graph(u, shape, schedule=walk, **kw)
        assert graphs["dpmpp_2m"] is not graphs["ddim"] and graphs["dpmpp_2m"].hist is not None

        def loop(name):
            """One whole loop from x_T at t = T-1; returns ms."""
            g = graphs[name]
            g.set_schedule(walks[name])
            g.x.copy_(x)
            g.t.fill_(T - 1)
            if g.hist is not None:
                g.hist.zero_()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(S):
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
        for name, g in graphs.items():
            assert torch.isfinite(g.x).all() and int(g.t.max()) == 0, f"the {name} loop did not reach t = 0"

    per_eval = {k: [v / evals for v in vals] for k, vals in ms.items()}
    print(json.dumps({
        "workload": f"{args.workload}: {wl['desc']}", "device": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(), "sampling_timesteps": S, "cond_scale": args.cond_scale,
        "unet_evals_per_loop": evals, "repeats": args.repeats, "dpmpp_2m_loop_ms": ms["dpmpp_2m"], "ddim_loop_ms": ms["ddim"],
        "dpmpp_2m_ms_per_eval": per_eval["dpmpp_2m"], "ddim_ms_per_eval": per_eval["ddim"],
        "ratio_median": statistics.median(a / b for a, b in zip(per_eval["dpmpp_2m"], per_eval["ddim"]))}))


if __name__ == "__main__":
    main()
