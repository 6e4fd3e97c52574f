"""Non-square images on the GPU: the implicit-GEMM convolution on the exact BW x BH tiles of widths that are multiples of 8
but not powers of two (csrc/conv_tc.cu tile_box), every kernel call of rectangular forwards, and Imagen.sample at 64 x 96
and 64 x 96 -> 256 x 384.

  * test_conv_rect: every conv route (mode 0 at k = 3 and 1, the two-source concat, the sub-pixel phases, the in-place
    stride-2 Downsample) at widths 24, 48, 96 and 384 on the 2:3 grid, on the 256-wide cooperative, the transposed
    C_out = 128 and the 128- / 64-wide ping-pong tiles, each with its GroupNorm statistics, against float64
    (test_gpu_image_fwd._run_conv); statistics credited to the wrong image or 16-channel block must fail the bound;
  * test_every_call_of_a_rectangular_forward: the conditional and null pass of a dim-64 base U-Net at 64 x 96 and of the
    cfg-3 SR structure at 256 x 384 (b = 2) under CheckingOps: every call checked, no conv_direct, the profiler's conv
    launches per kernel instance equal to test_aspect.conv_schedule's prediction, and the whole output within 2e-3 rel-L2
    of the float64 restatement;
  * sampling: the captured loop against the eager one (DDIM, 2M, inpainting, a guidance table) and a seeded image alone
    against inside a batch, at 64 x 96 and for the cascade 64 x 96 -> 256 x 384.
"""
import collections
import json
import os
import subprocess
import sys

import pytest
import torch

from checking_ops import ALLOWED, CheckingOps
from conftest import rel_l2
from oracle import restatement as OR
from test_aspect import conv_schedule
from test_gpu_flagship_calls import ScheduleLog, _profiled_launches, instance_name
from test_gpu_image_fwd import _rejects, _run_conv
import fp64_ref as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ kernel bounds
ROUTES = {   # name -> (C0, C1, C_out, k, mode, bias, residual, fp16 out)
    "k3": (128, 0, 128, 3, 0, True, True, True),
    "k1": (64, 0, 256, 1, 0, True, False, False),
    "concat": (64, 64, 128, 3, 0, True, False, True),
    "subpixel": (128, 0, 64, 2, 2, True, False, True),
    "downsample": (64, 0, 128, 4, 6, True, False, True),
}


@pytest.mark.parametrize("block_n", [256, 128, 64])
@pytest.mark.parametrize("route", sorted(ROUTES))
@pytest.mark.parametrize("W", [24, 48, 96, 384])
def test_conv_rect(native, W, route, block_n):
    C0, C1, Cout, k, mode, bias, res, f16 = ROUTES[route]
    H = 2 * W // 3
    B = 2
    if mode == 2:                       # the phases' low-res grid: a 2:3 image of half the size
        H, W = H // 2, W // 2
    if W % 8 or H % (128 // (W & -W)):
        pytest.skip(f"{H} x {W} has no exact 128-pixel box")
    a, wp, o, ref, bound, st = _run_conv(native, B, H, W, C0, C1, Cout, k, mode, bias, res, f16, True, block_n, seed=W)
    Ho, Wo = o.shape[1:3]
    sref, sbound = R.conv_stats_ref(o)
    # statistics credited to the wrong image, or to the wrong 16-channel block
    d = st.clone()
    f = o.double()[0, : Ho // 2].reshape(-1, Cout)[:, :16]
    d[0, 0, 0] -= f.sum()
    d[1, 0, 0] += f.sum()
    _rejects(d, sref, sbound, f"{route} W={W}: half of image 0's block-0 sum credited to image 1")
    d = st.clone()
    d[:, [0, 1]] = st[:, [1, 0]]
    _rejects(d, sref, sbound, f"{route} W={W}: statistics blocks 0 and 1 swapped")


# ------------------------------------------------------------------------------------------------ real forwards
def _cfgs():
    from minimagen_b200.Unet import Super
    return {"base_64x96": (dict(dim=64, dim_mults=(1, 2, 4), layer_attns=(False, True, True),
                                layer_cross_attns=(False, True, True), text_embed_dim=768), 64, 96),
            "cfg3_256x384": (dict(Super.defaults, lowres_cond=True, text_embed_dim=768), 256, 384)}


class RectScheduleLog(ScheduleLog):
    """ScheduleLog naming each conv's kernel instance by the new geometry's restatement.  Over a backend without a
    per-call error ratio (the native one, in the profiled run) it only counts the calls."""

    def _instance(self, name, args, kwargs):
        if name == "conv_gn":
            return 128, True, False
        a = self.sig[name].bind(None, *args, **kwargs)
        a.apply_defaults()
        p = a.arguments
        if name == "conv_res1x1":
            return conv_schedule(p["B"], p["H"], p["W"], p["c_out"], self.sms, out_sh=p["W"] * p["c_out"],
                                 out_sw=p["c_out"])
        _, sh, sw = p["out_strides"]
        return conv_schedule(p["B"], p["H"], p["W"], p["c_out"], self.sms, hint=p["block_n"], n_valid=p["n_valid"],
                             out_sc=p["out_sc"], in_stride=2 if p["mode"] == 6 else 1, out_sh=sh, out_sw=sw)

    def __getattr__(self, name):
        if name in ("conv_igemm", "conv_res1x1", "conv_gn") and not isinstance(self.inner, CheckingOps):
            target = getattr(self.inner, name)

            def count(*args, **kwargs):
                rec = self.per.setdefault(self._instance(name, args, kwargs), [0, 0.0])
                rec[0] += 1
                return target(*args, **kwargs)
            return count
        return super().__getattr__(name)


def _forward_case(case, b=2):
    """(cfg, the CUDA U-Net, its float64 state dict, x, t, conditioning) of a case, the same in every process."""
    from minimagen_b200.Unet import Unet
    cfg, H, W = _cfgs()[case]
    torch.manual_seed(0)
    u = Unet(**cfg).eval()
    sd = {k: v.detach().double().cuda() for k, v in u.state_dict().items()}
    g = torch.Generator().manual_seed(3)
    x = torch.randn(b, 3, H, W, generator=g).cuda()
    tm = torch.ones(b, 20, dtype=torch.bool)
    tm[-1, 5:] = False
    kw = dict(text_embeds=torch.randn(b, 20, 768, generator=g).cuda(), text_mask=tm.cuda())
    if cfg.get("lowres_cond"):
        kw.update(lowres_cond_img=torch.randn(b, 3, H, W, generator=g).cuda(),
                  lowres_noise_times=torch.full((b,), 200).cuda())
    return cfg, u.cuda(), sd, x, torch.tensor([999, 3][:b]).cuda(), kw


def _run_forward(case, backend, u, x, t, kw):
    """The conditional and the null pass with `backend` behind a RectScheduleLog; (outputs, log)."""
    import minimagen_b200.ops as ops_mod
    log = RectScheduleLog(backend, torch.cuda.get_device_properties(0).multi_processor_count)
    prev = ops_mod._OPS
    ops_mod.set_ops(log)
    try:
        with torch.no_grad():
            outs = (u(x, t, **kw), u(x, t, cond_drop_prob=1., **kw))
    finally:
        ops_mod.set_ops(prev)
    return outs, log


def _profiled_counts(case):
    """Profiler launch counts and predicted counts per conv instance of one native forward of `case` (the weights packed
    by a forward before the profiled one).  Runs in a process of its own (`python test_gpu_aspect.py case`): profiler
    sessions leave state behind in the process that ran them, which the profiler-based tests of other files must not
    inherit."""
    import minimagen_b200.ops as ops_mod
    from minimagen_b200 import _native
    _native.load()
    native = ops_mod.NativeOps()
    ops_mod.set_ops(native)
    _, u, _, x, t, kw = _forward_case(case)
    _run_forward(case, native, u, x, t, kw)
    torch.cuda.synchronize()
    (_, log), launches = _profiled_launches(lambda: _run_forward(case, native, u, x, t, kw))
    return log.counts(), launches


def _counts_in_child(case):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), case]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    d = json.loads(r.stdout.strip().splitlines()[-1])
    inst = lambda k: tuple(json.loads(k))
    return (collections.Counter({inst(k): v for k, v in d["predicted"].items()}),
            collections.Counter({inst(k): v for k, v in d["launches"].items()}))


@pytest.mark.parametrize("case", ["base_64x96", "cfg3_256x384"])
def test_every_call_of_a_rectangular_forward(native, case):
    """One native forward (conditional + null pass) under the profiler, in a child process: its conv launches per kernel
    instance against the restatement's prediction.  Then the same forward here with every call through CheckingOps: the
    lowering is the same, so the schedules the profiler counted are those checked."""
    predicted, launches = _counts_in_child(case)
    cfg, u, sd, x, t, kw = _forward_case(case)
    proxy = CheckingOps(native)
    outs, log = _run_forward(case, proxy, u, x, t, kw)
    proxy.report()
    print(f"\n{case}, b = {x.shape[0]}: conv schedule / calls / worst |err|/bound / profiler launches")
    for inst in sorted(set(predicted) | set(launches), key=lambda i: (-i[2], -i[0], i[1])):
        calls, worst = log.per.get(inst, (0, 0.0))
        print(f"  {instance_name(inst):32s} {calls:7d}   {worst:10.3g}   {launches[inst]:7d}")
    unchecked = proxy.called - proxy.checked - ALLOWED
    assert not unchecked, f"kernels that ran without a float64 check: {sorted(unchecked)}"
    assert "conv_direct" not in proxy.called
    assert {"conv_igemm", "stem_unroll"} <= proxy.checked
    assert log.counts() == predicted, f"checked run {dict(log.counts())} vs profiled run {dict(predicted)}"
    assert launches == predicted, f"profiler {dict(launches)} vs restatement {dict(predicted)}"
    with torch.no_grad():
        k64 = {k: (v.double() if v.is_floating_point() else v) for k, v in kw.items()}
        for out, drop in zip(outs, (0., 1.)):
            ref = OR.unet_forward(sd, cfg, x.double(), t, cond_drop_prob=drop, **k64)
            err = rel_l2(out, ref)
            print(f"  cond_drop_prob={drop}: rel-L2 vs float64 restatement {err:.3e}")
            assert err < 2e-3


# ------------------------------------------------------------------------------------------------ sampling
def _imagen(cascade):
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet
    torch.manual_seed(0)
    base = Unet(dim=64, dim_mults=(1, 2, 4), layer_attns=(False, False, True), layer_cross_attns=(False, True, True))
    unets = (base,)
    if cascade:
        unets += (Unet(dim=64, dim_mults=(1, 2, 4), num_resnet_blocks=(1, 1, 1), layer_attns=False,
                       layer_cross_attns=(False, False, True), lowres_cond=True, memory_efficient=True),)
    return Imagen(unets=unets, text_encoder_name="t5_small", image_sizes=(64, 256)[:len(unets)], timesteps=100,
                  cond_drop_prob=0.1).eval().cuda()


def _prompts(b, seed=21):
    gen = torch.Generator().manual_seed(seed)
    te = torch.randn(b, 9, 512, generator=gen)
    tm = torch.ones(b, 9, dtype=torch.bool)
    tm[1, 5:] = False
    return te.cuda(), tm.cuda()


FLAVOURS = {
    "ddim": dict(sampling_timesteps=6, ddim_eta=0.5),
    "dpmpp_2m": dict(sampling_timesteps=6, sampler="dpmpp_2m"),
    "inpaint": dict(sampling_timesteps=4, inpaint_resample_times=2),
    "guidance_table": dict(sampling_timesteps=6, guidance_interval=(0.5, 10.), guidance_schedule="linear"),
}


@pytest.mark.parametrize("cascade", [False, True])
@pytest.mark.parametrize("flavour", sorted(FLAVOURS))
def test_rectangular_graph_vs_eager(native, flavour, cascade):
    sizes = ((64, 96), (256, 384))[:1 + cascade]
    te, tm = _prompts(2)
    kw = dict(FLAVOURS[flavour], text_embeds=te, text_masks=tm, cond_scale=3., seed=[4, 2 ** 40], image_sizes=sizes)
    if flavour == "inpaint":
        mask = torch.zeros(2, 64, 96, dtype=torch.bool)
        mask[:, 16:48, 8:60] = True
        kw.update(inpaint_images=torch.rand(2, 3, 64, 96, generator=torch.Generator().manual_seed(5)).cuda(),
                  inpaint_masks=mask.cuda())
    outs = {}
    for graph in (False, True):
        im = _imagen(cascade)
        im.use_cuda_graph = graph
        outs[graph] = im.sample(**kw)
        if graph:
            assert len(im._graphs) >= 1 and all(k[1][2:] in sizes for k in im._graphs)
            im.clear_graphs()
    assert outs[True].shape == (2, 3, *sizes[-1])
    err = rel_l2(outs[True], outs[False])
    print(f"{flavour} {sizes}: graph vs eager rel-L2 = {err:.3e}, bitwise {torch.equal(outs[True], outs[False])}")
    assert err <= 1e-5


@pytest.mark.parametrize("cascade", [False, True])
def test_rectangular_batch_invariance(native, cascade):
    """A seeded image alone equals the same image inside a batch of 3 (captured graphs at batch 3 and 1)."""
    sizes = ((64, 96), (256, 384))[:1 + cascade]
    te, tm = _prompts(3)
    kw = dict(cond_scale=3., sampling_timesteps=6, ddim_eta=0.5, image_sizes=sizes)
    im = _imagen(cascade)
    full = im.sample(text_embeds=te, text_masks=tm, seed=[11, 2 ** 35, 3], **kw)
    one = im.sample(text_embeds=te[1:2], text_masks=tm[1:2], seed=[2 ** 35], **kw)
    err = rel_l2(one[0], full[1])
    print(f"{sizes}: row 1 alone vs in a batch of 3: rel-L2 {err:.3e}, bitwise {torch.equal(one[0], full[1])}")
    assert err <= 1e-5
    assert rel_l2(full[0], full[1]) > 0.1
    im.clear_graphs()


if __name__ == "__main__":
    # the profiled run of test_every_call_of_a_rectangular_forward: one JSON line of counts per instance
    predicted, launches = _profiled_counts(sys.argv[1])
    key = lambda c: {json.dumps(list(k)): v for k, v in c.items()}
    print(json.dumps(dict(predicted=key(predicted), launches=key(launches))))
