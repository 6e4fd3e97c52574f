"""Inpainting with RePaint resampling on the GPU: the three kernels (mi_inpaint_prologue / _advance / _finalize) against
their torch contracts, eagerly and under graph capture; the inpainting loop, captured and eager, against the plain loops,
the RePaint-form CPU restatement and the CPU emulation of the whole cascade; graph reuse and batch sharding."""
import pytest
import torch

import inpaint_restatement as P
from conftest import load_golden, rel_l2
from emu_ops import EmuOps, advance_ref, finalize_ref, prologue_ref
from test_inpaint import SHAPE, known_and_mask, restated_tiny
from test_respaced import _bank, _tiny_imagen

pytestmark = pytest.mark.gpu


def _inp(img, mask, R):
    """_p_sample_loop's `inpaint` argument from an image in [0, 1] and a bool mask."""
    b = img.shape[0]
    return ((img * 2 - 1).cuda().contiguous(), mask.float().reshape(b, -1).cuda().contiguous(), R)


def _loop(im, g, inpaint=None, sched=None, graph=True):
    im.use_cuda_graph = graph
    return im._p_sample_loop(im.unets[0], SHAPE, noise_scheduler=im.noise_schedulers[0],
                             text_embeds=g["text_embeds"].cuda(), text_mask=g["text_mask"].cuda(), cond_scale=3.,
                             schedule=sched, inpaint=inpaint)


def _capture(fn):
    """fn() captured in a CUDA graph after one warm-up call on a side stream."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph


# ------------------------------------------------------------------------------------------------ kernels
def test_prologue_and_finalize_kernels_bitwise(native):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    T, B, C, hw = 25, 6, 3, 40 * 40
    gd = GaussianDiffusion(timesteps=T).cuda()
    _, ra, rb = gd.inpaint_tables(gd.sampling_schedule(8, 0.5, "cuda"), "cuda")
    gen = torch.Generator(device="cuda").manual_seed(0)
    rn = lambda *s: torch.randn(*s, generator=gen, device="cuda")
    x, k, zr, zk = rn(B, C, 40, 40), rn(B, C, 40, 40), rn(B, C, 40, 40), rn(B, C, 40, 40)
    m = torch.rand(B, hw, generator=gen, device="cuda")                # fractional: the threshold is >= 0.5
    m[0, :8] = 0.5
    t = torch.tensor([24, 21, 0, -1, T, 10], dtype=torch.long, device="cuda")      # two out of range
    r = torch.tensor([0, 2, 0, 1, 1, 1], dtype=torch.long, device="cuda")
    args = (t, r, ra, rb, gd.sqrt_alphas_cumprod, gd.sqrt_one_minus_alphas_cumprod, k, m, zr, zk, T, B, C, hw)
    want = prologue_ref(x, *args)
    got = x.clone()
    native.inpaint_prologue(got, *args)
    assert torch.equal(got, want)
    assert torch.equal(got[3:5], x[3:5])                               # t outside [0, T): untouched
    # nothing known and r = 0: bitwise unchanged
    none = torch.zeros_like(m)
    z0 = torch.zeros_like(r)
    got = x.clone()
    native.inpaint_prologue(got, t, z0, ra, rb, gd.sqrt_alphas_cumprod, gd.sqrt_one_minus_alphas_cumprod, k, none,
                            zr, zk, T, B, C, hw)
    assert torch.equal(got, x)
    for unnorm in (0, 1):
        out = torch.empty_like(x)
        native.inpaint_finalize(x * 1.5, k, m, B, C, hw, unnorm, out)
        assert torch.equal(out, finalize_ref(x * 1.5, k, m, B, C, hw, unnorm))
    # captured: one replay = one prologue over the buffers' current contents
    buf = x.clone()
    graph = _capture(lambda: native.inpaint_prologue(buf, *args))
    buf.copy_(x)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(buf, want)


@pytest.mark.parametrize("walk", ["ddpm", "ddim"])
@pytest.mark.parametrize("R", [1, 3])
def test_advance_kernel_walk(native, walk, R):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    T, B = (25, 3) if walk == "ddpm" else (1000, 3)
    gd = GaussianDiffusion(timesteps=T)
    S = None if walk == "ddpm" else 8
    next_t = gd.inpaint_tables(None if S is None else gd.sampling_schedule(S, 0., "cuda"), "cuda")[0].cuda()
    Rt = torch.tensor([R], dtype=torch.long, device="cuda")
    plan = P.plan(T, R, S)
    assert len(plan) == (len(P.walk(T, S)) - 1) * R + 1
    t = torch.full((B,), T - 1, dtype=torch.long, device="cuda")
    r = torch.zeros_like(t)
    seen = []
    for _ in range(len(plan) + 2):
        seen.append((t.tolist(), r.tolist()))
        native.inpaint_advance(t, r, next_t, Rt, T, B)
    assert [(a[0], b[0]) for a, b in seen] == plan + [(0, 0), (0, 0)]
    assert all(len(set(a)) == 1 and len(set(b)) == 1 for a, b in seen)
    # out-of-range t goes to 0 with r = 0; a mid-repeat valid t repeats
    t = torch.tensor([-1, T, 1 << 40, -(1 << 40), T - 1, 0, T - 1], dtype=torch.long, device="cuda")
    r = torch.tensor([0, 0, 1, 0, 0, 0, R - 1], dtype=torch.long, device="cuda")
    want = advance_ref(t.clone(), r.clone(), next_t, Rt, T)
    native.inpaint_advance(t, r, next_t, Rt, T, t.numel())
    assert torch.equal(t, want[0]) and torch.equal(r, want[1])
    assert t.tolist()[:4] == [0, 0, 0, 0] and r.tolist()[:4] == [0, 0, 0, 0]
    # captured: one replay = one iteration of the plan
    t = torch.full((B,), T - 1, dtype=torch.long, device="cuda")
    r = torch.zeros_like(t)
    graph = _capture(lambda: native.inpaint_advance(t, r, next_t, Rt, T, B))
    t.fill_(T - 1)
    r.zero_()
    walked = []
    for _ in range(len(plan)):
        walked.append((int(t[0]), int(r[0])))
        graph.replay()
    torch.cuda.synchronize()
    assert walked == plan and int(t.max()) == 0 and int(r.max()) == 0


# ------------------------------------------------------------------------------------------------ the loop
@pytest.mark.parametrize("graph", [False, True])
def test_nothing_known_r1_equals_plain_loops(native, graph):
    """All-False mask, R = 1: the inpainting loop is the plain DDPM (T = 25) / DDIM (S = 8, eta 0.5) loop, same 'step' bank."""
    g = load_golden("sample_loop.pt")
    img, _ = known_and_mask(0)
    none = torch.zeros(2, 64, 64, dtype=torch.bool)
    for T, S in ((25, None), (1000, 8)):
        outs, banks = [], (_bank(11), _bank(12))
        for inpaint, bank in zip((None, _inp(img, none, 1)), banks):
            im = _tiny_imagen(g, T, "cuda")
            im.noise_fn = bank
            bank.bank.update(banks[0].bank)                  # the plain loop's 'init' and 'step' draws
            sched = None if S is None else im.noise_schedulers[0].sampling_schedule(S, 0.5, "cuda")
            outs.append(_loop(im, g, inpaint, sched, graph))
        assert [c for c in banks[1].calls if c[0] != "inpaint"] == banks[0].calls
        err = rel_l2(outs[1], outs[0])
        print(f"nothing known, R=1, T={T} S={S} (graph={graph}): rel-L2 vs plain loop = {err:.3e}")
        assert err <= 1e-6


@pytest.mark.parametrize("graph", [False, True])
def test_known_pixels_are_kept(native, graph):
    g = load_golden("sample_loop.pt")
    img, mask = known_and_mask(1)
    im = _tiny_imagen(g, 25, "cuda")
    for m in (torch.ones_like(mask), mask):
        im.noise_fn = _bank(12)
        out = _loop(im, g, _inp(img, m, 2), im.noise_schedulers[0].sampling_schedule(6, 0.5, "cuda"), graph).cpu()
        keep = m[:, None].expand(SHAPE)
        assert (out - img)[keep].abs().max() <= 1.2e-7
        if not bool(m.all()):
            assert (out - img)[~keep].abs().max() > 1e-2                # the rest is generated


@pytest.mark.parametrize("T,S,R", [(25, None, 3), (1000, 8, 2)])
def test_graph_eager_and_restatement(native, T, S, R):
    g = load_golden("sample_loop.pt")
    img, mask = known_and_mask(2)
    outs = {}
    for graph in (False, True):
        im = _tiny_imagen(g, T, "cuda")
        im.noise_fn = _bank(13)
        sched = None if S is None else im.noise_schedulers[0].sampling_schedule(S, 0.5, "cuda")
        outs[graph] = _loop(im, g, _inp(img, mask, R), sched, graph)
        if graph:
            assert len(im._graphs) == 1
    ref = restated_tiny(g, T, img, mask, R, _bank(13), steps=S, eta=0.5)
    e_ge, e_ref = rel_l2(outs[True], outs[False]), rel_l2(outs[True], ref)
    print(f"T={T} S={S} R={R}: graph vs eager {e_ge:.3e}; vs restated RePaint {e_ref:.3e}")
    assert e_ge <= 1e-5 and e_ref < 1e-3


def test_tensor_core_sr_config_vs_restatement(native):
    """The sr_d64 configuration of test_gpu_unet.CFGS (tensor-core convs, lowres conditioning) at 64x64, b = 2, CFG w = 3,
    S = 4, eta = 0, R = 2, random mask, against the restated RePaint loop.  fp16 operand budget: 2e-3."""
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import BaseTest, Unet
    from test_gpu_unet import CFGS
    _, cfg, s, lowres, b = next(c for c in CFGS if c[0] == "sr_d64")
    assert lowres and (s, b) == (64, 2)
    torch.manual_seed(0)
    im = Imagen(unets=(Unet(**BaseTest.defaults), Unet(**cfg)), text_encoder_name="t5_small", image_sizes=(16, s),
                timesteps=1000, cond_drop_prob=0.1).eval()
    sd = {k: v.clone() for k, v in im.unets[1].state_dict().items()}
    im = im.cuda()
    gen = torch.Generator().manual_seed(3)
    te = torch.randn(b, 20, 512, generator=gen)
    tm = torch.ones(b, 20, dtype=torch.bool)
    tm[-1, 5:] = False
    lowres_img = torch.rand(b, 3, s, s, generator=gen)
    lnt = torch.full((b,), 200)
    shape = (b, 3, s, s)
    img, mask = known_and_mask(4, shape)
    im.noise_fn = _bank(4, shape)
    sched = im.noise_schedulers[1].sampling_schedule(4, 0., "cuda")
    out = im._p_sample_loop(im.unets[1], shape, noise_scheduler=im.noise_schedulers[1], text_embeds=te.cuda(),
                            text_mask=tm.cuda(), lowres_cond_img=lowres_img.cuda(), lowres_noise_times=lnt.cuda(),
                            cond_scale=3., schedule=sched, inpaint=_inp(img, mask, 2))
    ref = P.inpaint_loop(sd, cfg, shape, 1000, img * 2 - 1, mask, 2, im.noise_fn, steps=4, eta=0., text_embeds=te,
                         text_mask=tm, lowres_cond_img=lowres_img * 2 - 1, lowres_noise_times=lnt)
    err = rel_l2(out, ref)
    print(f"sr_d64 S=4 R=2: rel-L2 vs restated RePaint = {err:.3e}")
    assert err < 2e-3


def test_graph_reused_across_mask_image_R_steps_eta(native):
    """One captured inpainting graph serves every mask, image, R, S and eta (and the DDPM walk); each loop equals eager.
    A text-only loop afterwards still equals its own eager run."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 25, "cuda")
    ref = _tiny_imagen(g, 25, "cuda")
    cases = ((8, 0.5, 2, 5), (None, 1., 2, 6), (5, 0., 3, 7), (12, 1., 1, 8))
    for S, eta, R, seed in cases:
        img, mask = known_and_mask(seed)
        outs = []
        for model, graph in ((im, True), (ref, False)):
            model.noise_fn = _bank(seed)
            sched = None if S is None else model.noise_schedulers[0].sampling_schedule(S, eta, "cuda")
            outs.append(_loop(model, g, _inp(img, mask, R), sched, graph))
        assert len(im._graphs) == 1
        err = rel_l2(outs[0], outs[1])
        print(f"reused inpainting graph S={S} eta={eta} R={R}: rel-L2 vs eager {err:.3e}")
        assert err <= 1e-5
    outs = []
    for model, graph in ((im, True), (ref, False)):
        model.noise_fn = _bank(9)
        outs.append(_loop(model, g, None, model.noise_schedulers[0].sampling_schedule(8, 0.5, "cuda"), graph))
    assert len(im._graphs) == 2
    assert rel_l2(outs[0], outs[1]) <= 1e-5


def test_cascade_vs_cpu_emulation(native):
    """The two-stage cascade of cascade_tiny.pt (16 -> 32, CFG w = 2, lowres augmentation) with inpainting at the final
    size, S = 8, R = 2: GPU sample vs the same call on the CPU emulation with the same draw bank; each stage pastes its
    resized known pixels into its output."""
    import minimagen_b200.ops as ops_mod
    from test_host_logic import _cascade_from_golden
    g = load_golden("cascade_tiny.pt")
    b = g["text_embeds"].shape[0]
    img, mask = known_and_mask(6, (b, 3, 32, 32))
    gen = torch.Generator().manual_seed(6)
    bank = {}

    def noise_fn(kind, shape, step):
        key = (kind, step, tuple(shape))
        if key not in bank:
            bank[key] = torch.randn(shape, generator=gen)
        return bank[key]

    outs, stages = {}, {}
    for dev in ("cuda", "cpu"):
        prev = ops_mod._OPS
        if dev == "cpu":
            ops_mod.set_ops(EmuOps())
        try:
            im, _ = _cascade_from_golden(g, dev)
            im.noise_fn = noise_fn
            im.use_cuda_graph = True
            loop, seen = im._p_sample_loop, []

            def spy(*a, **kw):
                out = loop(*a, **kw)
                seen.append((out.detach().cpu().clone(), kw["inpaint"]))
                return out
            im._p_sample_loop = spy
            outs[dev] = im.sample(text_embeds=g["text_embeds"].to(dev), text_masks=g["text_mask"].to(dev),
                                  cond_scale=g["cond_scale"], lowres_sample_noise_level=g["lowres_noise_level"],
                                  sampling_timesteps=8, inpaint_images=img.to(dev), inpaint_masks=mask.to(dev),
                                  inpaint_resample_times=2).cpu()
            stages[dev] = seen
        finally:
            ops_mod.set_ops(prev)
    err = rel_l2(outs["cuda"], outs["cpu"])
    print(f"cascade with inpainting, S=8 R=2: GPU vs CPU emulation rel-L2 = {err:.3e}")
    assert err < 1e-3
    assert len(stages["cuda"]) == 2
    for out, (k, m, R) in stages["cuda"]:
        assert R == 2
        known = (m.cpu() >= 0.5).reshape(b, 1, *out.shape[2:]).expand(out.shape)
        assert known.any()
        assert torch.equal(out[known], ((k.cpu().clamp(-1, 1) + 1) * 0.5)[known])
    keep = mask[:, None].expand(outs["cuda"].shape)
    assert (outs["cuda"] - img)[keep].abs().max() <= 1.2e-7


def test_inpaint_sample_sharding_invariance(native):
    """Imagen.sample with inpainting at b = 4 equals the same samples computed as two shards of 2 (what two ranks do)."""
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet
    g = load_golden("sample_loop.pt")
    u = Unet(**g["cfg"]).eval()
    u.load_state_dict(g["state_dict"])
    im = Imagen(unets=u.cuda(), text_encoder_name="t5_small", image_sizes=(64,), timesteps=25, cond_drop_prob=0.15).cuda()
    im.unets[0].load_state_dict(g["state_dict"])
    gen = torch.Generator().manual_seed(0)
    bank = {}

    def noise_fn(kind, shape, step):
        if (kind, step) not in bank:
            bank[(kind, step)] = torch.randn(4, *shape[1:], generator=gen)
        return bank[(kind, step)][noise_fn.lo:noise_fn.lo + shape[0]]
    noise_fn.lo = 0
    im.noise_fn = noise_fn
    te = torch.randn(4, 9, 512, generator=gen).cuda()
    tm = torch.ones(4, 9, dtype=torch.bool).cuda()
    img, mask = known_and_mask(7, (4, 3, 64, 64))
    img, mask = img.cuda(), mask.cuda()
    kw = dict(cond_scale=3., sampling_timesteps=6, ddim_eta=0.5, inpaint_resample_times=2)
    full = im.sample(text_embeds=te, text_masks=tm, inpaint_images=img, inpaint_masks=mask, **kw)
    assert full.shape == (4, 3, 64, 64) and torch.isfinite(full).all()
    parts = []
    for lo in (0, 2):
        noise_fn.lo = lo
        parts.append(im.sample(text_embeds=te[lo:lo + 2], text_masks=tm[lo:lo + 2], inpaint_images=img[lo:lo + 2],
                               inpaint_masks=mask[lo:lo + 2], **kw))
    err = rel_l2(torch.cat(parts), full)
    print(f"inpainting sample b=4 vs two shards of 2: rel-L2 = {err:.3e}")
    assert err <= 1e-5
