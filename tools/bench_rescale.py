"""Guidance rescale and v-prediction on the GPU: what they cost in the cfg-3 sampling loop, and the factor kernel's rate.

  * rescale: the captured DDIM loop (`--steps` steps, cond_scale 5) of the cfg-3 SR U-Net (Super.defaults, lowres_cond,
    text_embed_dim 768) at b = `--batch`, 256 x 256, with guidance_rescale 0.7 against 0, alternated `--rounds` times;
  * objective: the same loop ('v' tables) against the 'noise' loop, phi = 0, alternated `--rounds` times;
  * factor: mi_guidance_rescale_factor alone under CUDA events, at B = 32 x 3 x 256^2 and B = 2 x 3 x 1024^2: the time and
    the bytes it must read (both predictions once, 2 B n fp32) per second, against the H100 SXM data sheet's 3.35 TB/s.

Prints one JSON line per part (the first names the card, its power limit and clocks, read in the same run) and writes
them to `--out` (default: a temporary file).  Needs a CUDA device.
"""
import argparse
import collections
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet


def _device_info():
    p = torch.cuda.get_device_properties(0)
    info = dict(gpu=p.name, sms=p.multi_processor_count)
    try:
        import subprocess
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        info["power_limit_clocks"] = q[0] if q else None
    except Exception as e:  # noqa: BLE001 -- the numbers are still valid without the query
        info["power_limit_clocks"] = f"unavailable: {e}"
    return info


def _sr_imagen(objective):
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import BaseTest, Super, Unet
    torch.manual_seed(0)
    # the SR U-Net sits behind a base stage (Imagen treats unets[0] as the base model), a tiny stand-in never run
    u = Unet(**dict(Super.defaults, lowres_cond=True, text_embed_dim=768)).eval()
    first = Unet(**dict(BaseTest.defaults, text_embed_dim=768)).eval()
    im = Imagen(unets=(first, u), text_encoder_name="t5_base", image_sizes=(64, 256), timesteps=1000,
                cond_drop_prob=0.1).eval().cuda()
    im.set_objectives(('noise', objective))
    im.use_cuda_graph = True
    return im


def _cond(b, seed=0):
    g = torch.Generator().manual_seed(seed)
    te = torch.randn(b, 32, 768, generator=g).cuda()
    tm = torch.ones(b, 32, dtype=torch.bool).cuda()
    low = torch.rand(b, 3, 256, 256, generator=g).cuda()
    return te, tm, low


def _loop(im, a, cond, phi):
    sch = im.noise_schedulers[-1]
    te, tm, low = cond
    lt = torch.full((a.batch,), 200, dtype=torch.long, device="cuda")
    torch.manual_seed(1)
    return im._p_sample_loop(im.unets[-1], (a.batch, 3, 256, 256), noise_scheduler=sch, text_embeds=te, text_mask=tm,
                             lowres_cond_img=low, lowres_noise_times=lt, cond_scale=5.,
                             schedule=sch.sampling_schedule(a.steps, 0., "cuda"), guidance_rescale=phi)


def _alternate(a, variants):
    """variants: name -> (imagen, phi).  Warm-up (capture) of each, then `rounds` alternated timed loops."""
    cond = _cond(a.batch)
    for im, phi in variants.values():
        _loop(im, a, cond, phi)
    torch.cuda.synchronize()
    times = collections.defaultdict(list)
    for _ in range(a.rounds):
        for name, (im, phi) in variants.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _loop(im, a, cond, phi)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1))
    res = {}
    for name, ms in times.items():
        ms = sorted(ms)
        res[name] = dict(loop_ms=ms, ms_per_step_median=ms[len(ms) // 2] / a.steps)
    return res


def part_rescale(a):
    im = _sr_imagen('noise')
    res = _alternate(a, {"phi_0": (im, 0.), "phi_0.7": (im, 0.7)})
    res["ratio_per_step"] = res["phi_0.7"]["ms_per_step_median"] / res["phi_0"]["ms_per_step_median"]
    return dict(part="rescale", batch=a.batch, steps=a.steps, rounds=a.rounds, cond_scale=5., graphs=len(im._graphs),
                **res)


def part_objective(a):
    res = _alternate(a, {"noise": (_sr_imagen('noise'), 0.), "v": (_sr_imagen('v'), 0.)})
    res["ratio_per_step"] = res["v"]["ms_per_step_median"] / res["noise"]["ms_per_step_median"]
    return dict(part="objective", batch=a.batch, steps=a.steps, rounds=a.rounds, cond_scale=5., **res)


def part_factor(a):
    from minimagen_b200.ops import get_ops
    ops = get_ops()
    res = {}
    for B, side in ((32, 256), (2, 1024)):
        n = 3 * side * side
        g = torch.Generator().manual_seed(side)
        c = torch.randn(B, n, generator=g).cuda()
        u = torch.randn(B, n, generator=g).cuda()
        w = torch.full((B,), 5., device="cuda")
        t = torch.full((B,), 500, dtype=torch.long, device="cuda")
        phi = torch.full((B,), 0.7, device="cuda")
        f = torch.empty(B, device="cuda")
        for _ in range(10):
            ops.guidance_rescale_factor(c, u, w, None, t, phi, B, n, f)
        torch.cuda.synchronize()
        reps = 200
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            ops.guidance_rescale_factor(c, u, w, None, t, phi, B, n, f)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / reps
        nbytes = 2 * B * n * 4
        res[f"B{B}_3x{side}x{side}"] = dict(us_per_call=us, bytes=nbytes, bytes_per_s=nbytes / (us * 1e-6),
                                            share_of_3_35TBps=nbytes / (us * 1e-6) / HBM_BYTES_PER_S)
    return dict(part="factor", what="two launches per call (partials, merge), host enqueue included, 200 calls "
                                    "back to back", **res)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--parts", default="factor,rescale,objective")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rescale.py needs a CUDA device")
    torch.cuda.set_device(0)
    out = a.out or os.path.join(tempfile.mkdtemp(prefix="bench_rescale_"), "bench_rescale.jsonl")
    lines = [dict(part="device", **_device_info())]
    print(json.dumps(lines[0]), flush=True)
    for p in a.parts.split(","):
        t0 = time.time()
        r = dict(globals()[f"part_{p}"](a), wall_s=round(time.time() - t0, 1))
        lines.append(r)
        print(json.dumps(r), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, "w") as f:
        f.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
