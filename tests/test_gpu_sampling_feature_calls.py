"""Samples that combine the sampling features, with every kernel call checked against float64 by one CheckingOps
(tests/checking_ops.py), on the GPU:

  (a) a two-stage non-square DDIM cascade, 64 x 96 -> 256 x 384 at b = 4 (test_gpu_aspect's networks): stage 1 RePaint
      at R = 2 with mask pixels of exactly 0.5, per-image seeds and weights, a negative prompt and a 'linear' guidance
      schedule; stage 2 a v-prediction U-Net on a zero-terminal-SNR schedule with a guidance interval, a 'cosine'
      schedule, per-image guidance rescale and an init image skipping one point; with cfg_batched on and off;
  (b) the same cascade on DPM-Solver++(2M) without inpainting, so the multistep history, the scheduled and the rescaled
      multistep epilogues meet the first-order restart of img2img;
  (c) DDPM inpainting at R = 3 on the tiny golden U-Net (T = 25), eager, and then through the captured step's body run
      eagerly (the graph replaced by a direct call), so mi_inpaint_advance walks r through 0..2 at every grid point and
      the keyed draws read their labels t * 3 + r on the device.

Each case asserts that no call went unchecked and that the families it exists for were reached, and prints the checked
families, its wall time and its peak memory.  Then the captured loops of (a) and (b) on analytic stand-in U-Nets (no
atomics, so bit for bit) against the eager ones.
"""
import time

import pytest
import torch

from checking_ops import ALLOWED, CheckingOps
from conftest import load_golden, rel_l2
from test_dpmpp import AnalyticEps
from test_gpu_aspect import _imagen, _prompts
from test_gpu_inpaint import _inp
from test_respaced import _tiny_imagen
from test_sampling_feature_calls import REACH, cascade_case, half_mask, reached
from test_vpred_rescale import TwoPass

pytestmark = pytest.mark.gpu
SIZES = ((64, 96), (256, 384))
INF = float("inf")


def _checked_run(native, name, fn):
    import minimagen_b200.ops as ops_mod
    proxy = CheckingOps(native)
    ops_mod.set_ops(proxy)                              # the `native` fixture restores the previous backend afterwards
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    print(f"\n{name}: {wall:.1f} s, peak memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    proxy.report()
    assert torch.isfinite(out).all()
    unchecked = proxy.called - proxy.checked - ALLOWED
    assert not unchecked, f"kernels that ran without a float64 check: {sorted(unchecked)}"
    return proxy, out


@pytest.mark.parametrize("flavour,cfg_batched", [("ddim", False), ("ddim", True), ("dpmpp_2m", True)],
                         ids=["a-ddim-unbatched", "a-ddim-cfg_batched", "b-dpmpp_2m"])
def test_every_call_of_a_combined_cascade(native, flavour, cfg_batched):
    im = _imagen(True)
    te, tm = _prompts(4)
    kw = cascade_case(im, flavour, 4, SIZES, 512, "cuda", cfg_batched)
    proxy, out = _checked_run(native, f"{flavour} cascade, cfg_batched={cfg_batched}",
                              lambda: im.sample(text_embeds=te, text_masks=tm, **kw))
    assert out.shape == (4, 3, *SIZES[-1])
    assert REACH[flavour] <= reached(proxy), sorted(REACH[flavour] - reached(proxy))
    if flavour == "ddim":
        renoise = {lab for kind, st, labs in proxy.keyed if kind == "renoise" and st == 1 for lab in labs}
        assert renoise == {t * 2 + 1 for t in (99, 66, 33)}


class _EagerGraph:
    """Stands in for a captured CUDA graph: replay() runs the captured step's body eagerly, so every call it makes goes
    through the checks."""

    def __init__(self, body):
        self.body = body

    def replay(self):
        self.body()

    def pool(self):
        return None


def test_every_call_of_ddpm_inpainting_r3(native, monkeypatch):
    from minimagen_b200.Imagen import Imagen
    g = load_golden("sample_loop.pt")
    T, R_ = 25, 3
    gen = torch.Generator().manual_seed(3)
    mask = torch.zeros(2, 64, 64, dtype=torch.bool)
    mask[:, 8:40, 16:48] = True
    kw = dict(text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda(), cond_scale=torch.tensor([3., 1.5]),
              inpaint_images=torch.rand(2, 3, 64, 64, generator=gen).cuda(), inpaint_masks=mask.cuda(),
              inpaint_resample_times=R_, seed=[9, 2 ** 40])
    outs = {}
    for body in (False, True):
        im = _tiny_imagen(g, T, "cuda")
        im.use_cuda_graph = body
        if body:
            monkeypatch.setattr(Imagen, "_capture", staticmethod(lambda fn, device, pool=None: _EagerGraph(fn)))
        proxy, outs[body] = _checked_run(native, f"DDPM inpainting R = 3, {'the graph body' if body else 'eager'}",
                                         lambda: im.sample(**kw))
        assert REACH["ddpm_inpaint"] <= reached(proxy)
        assert proxy.family["inpaint_prologue"][0] == (T - 1) * R_ + 1
        if body:
            labels = {f"randn_keyed {kind} stage 1 label {t * R_ + r}" for kind in ("renoise", "inpaint", "step")
                      for t in range(T) for r in range(R_ if t > 0 else 1)}
            assert labels <= proxy.features
            assert {"inpaint_advance", "inpaint_advance repeat", "inpaint_advance next point",
                    "randn_keyed renoise stage 1 device labels"} <= reached(proxy)
            assert proxy.family["inpaint_advance"][0] == (T - 1) * R_ + 1
    err = rel_l2(outs[True], outs[False])
    print(f"graph body vs eager loop: rel-L2 {err:.3e}, bitwise {torch.equal(outs[True], outs[False])}")
    assert err <= 1e-6


# ------------------------------------------------------------------------------------------------ analytic, captured
def _standin_cascade(flavour, graph):
    """The loops of case (a) or (b) on analytic stand-ins through _p_sample_loop: stage 1 AnalyticEps (per-pixel Gaussian
    data, linear schedule), stage 2 the 'v' TwoPass of test_vpred_rescale on the zero-SNR schedule, fed stage 1's output.
    Returns both stages' outputs."""
    from minimagen_b200.helpers import resize_image_to
    im = _imagen(True).set_objectives(['noise', 'v'], zero_terminal_snr=[False, True])
    im.cfg_batched = False
    im.use_cuda_graph = graph
    im.noise_fn = None
    s1, s2 = im.noise_schedulers
    u1 = AnalyticEps(s1.num_timesteps).cuda()
    u2 = TwoPass(s2.alphas_cumprod_fp64, 'v').cuda()
    te, tm = _prompts(4)
    gen = torch.Generator().manual_seed(17)
    nte = torch.randn(1, 5, 512, generator=gen).expand(4, 5, 512).contiguous().cuda()
    ntm = torch.ones(4, 5, dtype=torch.bool).cuda()
    seeds = torch.tensor([5, 2 ** 40 + 1, 123, 7], device="cuda")
    cond = dict(text_embeds=te, text_mask=tm, negative_text_embeds=nte, negative_text_mask=ntm, seeds=seeds)
    (h1, w1), (h2, w2) = SIZES
    if flavour == "ddim":
        walk1, walk2 = s1.sampling_schedule(4, 0.5, "cuda"), s2.sampling_schedule(4, 0.5, "cuda")
        walk2 = walk2._replace(grid=walk2.grid[1:])
        mask = half_mask(4, h1, w1)
        inpaint = _inp(torch.rand(4, 3, h1, w1, generator=gen), mask, 2)
    else:
        walk1, walk2 = s1.dpm_solver_schedule(4, "cuda"), s2.dpm_solver_schedule(4, "cuda", skip=1)
        inpaint = None
    x1 = im._p_sample_loop(u1, (4, 3, h1, w1), noise_scheduler=s1, cond_scale=torch.tensor([2., 4.5, 1., 3.]).cuda(),
                           schedule=walk1, inpaint=inpaint, stage=1,
                           guidance_table=s1.guidance_table(None, "linear", "cuda"), **cond)
    init = resize_image_to(x1, (h2, w2), clamp_range=(0., 1.)) * 2 - 1
    x2 = im._p_sample_loop(u2, (4, 3, h2, w2), noise_scheduler=s2, cond_scale=torch.tensor([3., 1.5, 5., 2.]).cuda(),
                           schedule=walk2, init_image=init.contiguous(), stage=2,
                           guidance_table=s2.guidance_table((0.3, INF), "cosine", "cuda"),
                           guidance_rescale=torch.tensor([0.7, 0.3, 1., 0.5]).cuda(), **cond)
    if graph:
        assert len(im._graphs) == 2 and all('guidance_table' in k and ('seeded', s) in k
                                            for k, s in zip(im._graphs, (1, 2)))
        assert ('rescaled' in list(im._graphs)[1]) and ('rescaled' not in list(im._graphs)[0])
    return x1, x2


@pytest.mark.parametrize("flavour", ["ddim", "dpmpp_2m"])
def test_captured_combined_cascade_is_the_eager_one_on_stand_ins(native, flavour):
    eager, graph = _standin_cascade(flavour, False), _standin_cascade(flavour, True)
    for i, (e, gr) in enumerate(zip(eager, graph), 1):
        print(f"{flavour} stage {i}: graph vs eager rel-L2 = {rel_l2(gr, e):.3e}")
        assert torch.isfinite(e).all() and torch.equal(gr, e)
