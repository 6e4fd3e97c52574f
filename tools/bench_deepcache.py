"""Time DeepCache feature reuse (Imagen.sample(cache_interval=N)) on one GPU.

The workload's SR U-Net (cfg 3: 64 -> 256, b = 32) at cond_scale 3 with per-image seeds, a captured S-point DDIM loop
(eta = 0), at N = 1 (no caching: today's loop), 2, 3 and 5.  After one warm-up of each (which captures the graphs), the
loops are alternated `--repeats` times, CUDA events around each.  Then the DeepCache entry's full and cached graphs are
replayed alone, alternated, `--replays` times each (CUDA events around each replay, the step's static x and t reset
before it), which gives r = cached / full per evaluation and the loop ratio it predicts, (1 + (N - 1) r) / N.  The final
images' rel-L2 to the N = 1 loop is reported as a distance only: the network is randomly initialised, so it says
nothing about sample quality.
Writes nothing; prints one JSON line with the card's name and power limit.
Usage: python tools/bench_deepcache.py [--workload cfg3] [--sampling-timesteps 50] [--intervals 1 2 3 5] [--repeats 3]
                                       [--replays 20]
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
    ap.add_argument("--intervals", type=int, nargs="+", default=(1, 2, 3, 5))
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--replays", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_deepcache.py needs a CUDA device"
    assert 1 in args.intervals and any(n > 1 for n in args.intervals), "--intervals needs 1 and some N > 1"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)

    from minimagen_b200 import _native
    from minimagen_b200.Imagen import Imagen, deepcache_plan
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
    inp = synth_inputs(wl, B, 1000)
    te, tm = inp["text_embeds"].to(dev), inp["text_mask"].to(dev)
    lowres = inp["lowres_img01"].to(dev)                         # the loop normalises it
    lowres_t = torch.full((B,), int(0.2 * T), dtype=torch.long, device=dev)
    sch = im.noise_schedulers[1]
    walk = sch.sampling_schedule(S, 0., dev)
    seeds = torch.arange(1000, 1000 + B, device=dev)
    loop_kw = dict(noise_scheduler=sch, text_embeds=te, text_mask=tm, lowres_cond_img=lowres, lowres_noise_times=lowres_t,
                   schedule=walk, cond_scale=w, seeds=seeds, stage=2)

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    runs = {n: (lambda n=n: im._p_sample_loop(u, (B, 3, s, s), cache_interval=n, **loop_kw).clone())
            for n in args.intervals}
    outs = {}
    with torch.no_grad():
        for n, fn in runs.items():                                  # warm-up: captures the graphs
            outs[n] = fn()
        graphs = len(im._graphs)
        ms = {n: [] for n in runs}
        for _ in range(args.repeats):
            for n, fn in runs.items():
                t, outs[n] = timed(fn)
                ms[n].append(t)
        assert len(im._graphs) == graphs, "a repeat must replay the captured graphs, not capture others"
        # the full and the cached graph of the DeepCache entry alone
        (g,) = [e for k, e in im._graphs.items() if 'deepcache' in k]
        x0 = outs[1].clone()
        rep = {True: [], False: []}
        for _ in range(args.replays):
            for full in (True, False):
                g.x.copy_(x0)
                g.t.fill_(walk.grid[1])
                t, _ = timed(lambda: g.replay(True, full))
                rep[full].append(t)
    for n, out in outs.items():
        assert torch.isfinite(out).all(), n
    med = {n: statistics.median(v) for n, v in ms.items()}
    full_ms, cached_ms = statistics.median(rep[True]), statistics.median(rep[False])
    r = cached_ms / full_ms
    rel = lambda a, b: ((a.double() - b.double()).norm() / b.double().norm()).item()
    print(json.dumps({
        "workload": f"{args.workload}: {wl['desc']}", "device": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(), "sampling_timesteps": S, "cond_scale": w, "batch": B,
        "repeats": args.repeats, "captured_graphs": graphs,
        "loop_ms": {n: ms[n] for n in runs},
        "loop_over_n1_median": {n: med[n] / med[1] for n in runs},
        "full_evaluations": {n: sum(deepcache_plan([True] * S, n)) for n in runs},
        "full_replay_ms_median": full_ms, "cached_replay_ms_median": cached_ms, "cached_over_full": r,
        "predicted_loop_ratio": {n: (1 + (n - 1) * r) / n for n in runs},
        "rel_l2_to_n1": {n: rel(outs[n], outs[1]) for n in runs}}))


if __name__ == "__main__":
    main()
