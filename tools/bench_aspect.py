"""Non-square sampling on the GPU: what a 2:3 image costs next to a square one, and what the exact BW x BH conv tiles gain.

  * loop: a captured DDIM loop (`--steps` steps, CFG w = 3) of the cfg-3 SR U-Net (Super.defaults, lowres_cond,
    text_embed_dim 768) at b = `--batch`, at 256 x 256 and at 256 x 384, alternated `--rounds` times in one session;
    ms per step and ms per megapixel;
  * kernels: one eager guided step's conv calls at 256 x 384, timed per call with CUDA events, summed per (level, conv
    schedule) -- the schedule named by tests/test_aspect.conv_schedule;
  * base: one eager forward of a dim-64 base U-Net (mults 1, 2, 4) at 64 x 96, b = `--batch`, with the tensor-core
    predicates as they are and with the parent rule (only power-of-two widths below 128: the 96 / 48 / 24-wide levels
    then run the fp32 direct convolution, as they did before exact tiles existed).

Prints one JSON line per part and writes them to `--out` (default: a temporary file).  Needs a CUDA device.
"""
import argparse
import collections
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import torch  # noqa: E402


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


def _sr_imagen():
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import BaseTest, Super, Unet
    torch.manual_seed(0)
    # the SR U-Net sits behind a base stage (Imagen treats unets[0] as the base model), a tiny stand-in never run
    u = Unet(**dict(Super.defaults, lowres_cond=True, text_embed_dim=768)).eval()
    first = Unet(**dict(BaseTest.defaults, text_embed_dim=768)).eval()
    im = Imagen(unets=(first, u), text_encoder_name="t5_base", image_sizes=(64, 256), timesteps=1000,
                cond_drop_prob=0.1).eval().cuda()
    assert im.unets[-1].lowres_cond
    return im


def _cond(b, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    te = torch.randn(b, 32, 768, generator=g).cuda()
    tm = torch.ones(b, 32, dtype=torch.bool).cuda()
    low = torch.rand(b, 3, h, w, generator=g).cuda()
    return te, tm, low


def _loop(im, shape, steps, te, tm, low):
    sch = im.noise_schedulers[-1]
    lt = torch.full((shape[0],), 200, dtype=torch.long, device="cuda")
    return im._p_sample_loop(im.unets[-1], shape, noise_scheduler=sch, text_embeds=te, text_mask=tm,
                             lowres_cond_img=low, lowres_noise_times=lt, cond_scale=3.,
                             schedule=sch.sampling_schedule(steps, 0., "cuda"))


def part_loop(a):
    im = _sr_imagen()
    im.use_cuda_graph = True
    shapes = {"256x256": (256, 256), "256x384": (256, 384)}
    conds = {k: _cond(a.batch, *hw) for k, hw in shapes.items()}
    for k, hw in shapes.items():                 # capture + warm-up of both shapes
        _loop(im, (a.batch, 3, *hw), a.steps, *conds[k])
    torch.cuda.synchronize()
    times = collections.defaultdict(list)
    for _ in range(a.rounds):
        for k, hw in shapes.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _loop(im, (a.batch, 3, *hw), a.steps, *conds[k])
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
    res = {}
    for k, hw in shapes.items():
        ms = sorted(times[k])
        step = [t / a.steps for t in ms]
        mpix = a.batch * hw[0] * hw[1] / 1e6
        res[k] = dict(loop_ms=ms, ms_per_step_median=step[len(step) // 2], ms_per_step_min=step[0],
                      ms_per_megapixel_step=step[len(step) // 2] / mpix)
    res["ratio_per_step"] = res["256x384"]["ms_per_step_median"] / res["256x256"]["ms_per_step_median"]
    return dict(part="loop", batch=a.batch, steps=a.steps, rounds=a.rounds, **res)


class _Timed:
    """Wraps the ops backend: each conv call between two CUDA events, keyed by (H, W, c_out, schedule)."""

    def __init__(self, inner, sms):
        import inspect
        from minimagen_b200.ops import NativeOps
        self.inner, self.sms, self.rec = inner, sms, []
        self.sig = {m: inspect.signature(getattr(NativeOps, m)) for m in ("conv_igemm", "conv_res1x1", "conv_gn",
                                                                           "conv_direct")}

    def _key(self, name, args, kwargs):
        from test_aspect import conv_schedule
        from test_gpu_flagship_calls import instance_name
        a = self.sig[name].bind(None, *args, **kwargs)
        a.apply_defaults()
        p = a.arguments
        if name == "conv_direct":
            return p["Hout"], p["Wout"], p["c_out"], "fp32 direct"
        if name == "conv_gn":
            return p["H"], p["W"], p["c_out"], "128-wide GroupNorm prologue"
        if name == "conv_res1x1":
            inst = conv_schedule(p["B"], p["H"], p["W"], p["c_out"], self.sms, out_sh=p["W"] * p["c_out"],
                                 out_sw=p["c_out"])
            return p["H"], p["W"], p["c_out"], instance_name(inst) + " +res1x1"
        _, sh, sw = p["out_strides"]
        inst = conv_schedule(p["B"], p["H"], p["W"], p["c_out"], self.sms, hint=p["block_n"], n_valid=p["n_valid"],
                             out_sc=p["out_sc"], in_stride=2 if p["mode"] == 6 else 1, out_sh=sh, out_sw=sw)
        return p["H"], p["W"], p["c_out"], f"{instance_name(inst)} mode {p['mode']}"

    def __getattr__(self, name):
        target = getattr(self.inner, name)
        if name not in self.sig:
            return target

        def call(*args, **kwargs):
            key = self._key(name, args, kwargs)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ret = target(*args, **kwargs)
            e1.record()
            self.rec.append((key, e0, e1))
            return ret
        return call


def part_kernels(a):
    import minimagen_b200.ops as ops_mod
    im = _sr_imagen()
    u = im.unets[-1]
    b, (h, w) = a.batch, (256, 384)
    te, tm, low = _cond(b, h, w)
    x = torch.randn(b, 3, h, w, device="cuda")
    t = torch.full((b,), 500, device="cuda")
    lt = torch.full((b,), 200, device="cuda")
    run = lambda: u.forward_with_cond_scale(x, t, cond_scale=3., text_embeds=te, text_mask=tm, lowres_cond_img=low,
                                            lowres_noise_times=lt)
    native = ops_mod.get_ops()
    with torch.no_grad():
        run()
        timed = _Timed(native, torch.cuda.get_device_properties(0).multi_processor_count)
        ops_mod.set_ops(timed)
        try:
            run()
        finally:
            ops_mod.set_ops(native)
        torch.cuda.synchronize()
    table = collections.defaultdict(lambda: [0, 0.0])
    for key, e0, e1 in timed.rec:
        table[key][0] += 1
        table[key][1] += e0.elapsed_time(e1)
    rows = [dict(H=k[0], W=k[1], c_out=k[2], schedule=k[3], calls=n, ms=round(ms, 4))
            for k, (n, ms) in sorted(table.items(), key=lambda kv: (-kv[0][1], kv[0][2], kv[0][3]))]
    return dict(part="kernels", batch=b, size=[h, w], what="one guided step (cond + null pass), eager, per-call events",
                conv_ms_total=round(sum(r["ms"] for r in rows), 3), rows=rows)


def part_base(a):
    import minimagen_b200.ops as ops_mod
    from minimagen_b200.Unet import Unet
    from test_aspect import _old_supported

    class ParentRule:
        """The predicates as they were before exact tiles: power-of-two widths below 128 only."""

        def __init__(self, inner):
            self.inner = inner

        def __getattr__(self, name):
            return getattr(self.inner, name)

        def igemm_supported(self, H, W, c_in, c_out):
            return self.inner.igemm_supported(H, W, c_in, c_out) and _old_supported(H, W)

        def conv_res1x1_supported(self, H, W, c_in, c_out, x_cin):
            return self.inner.conv_res1x1_supported(H, W, c_in, c_out, x_cin) and _old_supported(H, W)

        def conv_gn_supported(self, H, W, c0, c1, c_out, groups):
            return self.inner.conv_gn_supported(H, W, c0, c1, c_out, groups) and _old_supported(H, W)

    def net():          # a fresh network per backend: nothing the lowering prepares is shared between the two
        torch.manual_seed(0)
        return Unet(dim=64, dim_mults=(1, 2, 4), layer_attns=(False, True, True), layer_cross_attns=(False, True, True),
                    text_embed_dim=768).eval().cuda()
    b = a.batch
    g = torch.Generator().manual_seed(1)
    x = torch.randn(b, 3, 64, 96, generator=g).cuda()
    te = torch.randn(b, 32, 768, generator=g).cuda()
    t = torch.full((b,), 500, device="cuda")
    native = ops_mod.get_ops()
    res, outs = {}, {}
    for name, backend in (("exact_tiles", native), ("parent_rule_fp32_fallback", ParentRule(native))):
        u = net()
        ops_mod.set_ops(backend)
        try:
            with torch.no_grad():
                for _ in range(3):
                    outs[name] = u(x, t, text_embeds=te)
                torch.cuda.synchronize()
                ms = []
                for _ in range(a.rounds * 4):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    u(x, t, text_embeds=te)
                    e1.record()
                    torch.cuda.synchronize()
                    ms.append(e0.elapsed_time(e1))
        finally:
            ops_mod.set_ops(native)
        ms.sort()
        res[name] = dict(ms_median=ms[len(ms) // 2], ms_min=ms[0])
    d = (outs["exact_tiles"].double() - outs["parent_rule_fp32_fallback"].double()).norm()
    res["rel_l2_between"] = float(d / outs["parent_rule_fp32_fallback"].double().norm())
    res["speedup"] = res["parent_rule_fp32_fallback"]["ms_median"] / res["exact_tiles"]["ms_median"]
    return dict(part="base", batch=b, size=[64, 96], what="one eager forward, dim-64 base U-Net mults (1, 2, 4)", **res)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--parts", default="base,kernels,loop")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_aspect.py needs a CUDA device")
    torch.cuda.set_device(0)
    out = a.out or os.path.join(tempfile.mkdtemp(prefix="bench_aspect_"), "bench_aspect.jsonl")
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
