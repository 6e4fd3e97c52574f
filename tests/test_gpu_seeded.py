"""Per-image seeds on the GPU: mi_randn_keyed's bits independent of the batch and the launch, its normals against the
float64 restatement within a bound derived from CUDA's documented ulp errors, device labels against host labels; the
seeded sampler's batch invariance, captured against eager loops in the text, inpainting and multistep flavours and with
img2img, a split cascade, native against the CPU emulation, and seed=None left as it was."""
import numpy as np
import pytest
import torch

import keyed_noise_restatement as K
from conftest import load_golden, rel_l2
from emu_ops import EmuOps
from test_respaced import _tiny_imagen

pytestmark = pytest.mark.gpu
I64 = torch.int64
SEEDS = [7, 2 ** 40 + 3, 123456789012, 0, 2 ** 63 - 1]


def _draw(native, seeds, n, kind=1, stage=1, label=0, **dev_labels):
    s = torch.tensor(seeds, dtype=I64, device="cuda")
    out = torch.full((len(seeds), n), float("nan"), device="cuda")
    native.randn_keyed(out, s, len(seeds), n, kind, stage, label=label, **dev_labels)
    return out


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("n", [3 * 64 * 64, 1001])
def test_bits_independent_of_batch_and_launch(native, n):
    """An image's draws are bitwise the same at any batch position and batch size, and from two launches."""
    full = _draw(native, SEEDS, n, kind=4, stage=2, label=77)
    assert torch.isfinite(full).all()
    assert torch.equal(full, _draw(native, SEEDS, n, kind=4, stage=2, label=77))
    for i, s in enumerate(SEEDS):
        assert torch.equal(full[i], _draw(native, [s], n, kind=4, stage=2, label=77)[0])
    rev = _draw(native, SEEDS[::-1], n, kind=4, stage=2, label=77)
    assert torch.equal(rev, full.flip(0))
    # a different kind, stage or label is a different stream
    for other in (dict(kind=3, stage=2, label=77), dict(kind=4, stage=1, label=77), dict(kind=4, stage=2, label=78)):
        assert not torch.equal(_draw(native, SEEDS[:1], n, **other)[0], full[0])


@pytest.mark.parametrize("n", [3 * 64 * 64, 4099, 10])
@pytest.mark.parametrize("kind,stage,label", [(0, 1, -1), (1, 1, 999), (2, 2, 2), (3, 3, 4001), (4, 1, 2 ** 31 - 1)])
def test_normals_vs_float64(native, n, kind, stage, label):
    """|z - z64| <= 2^-20 |z64| element by element against the restatement from the same bits (n % 4 != 0 included:
    the tail lanes are the first lanes of the last quad)."""
    bound = K.ulp_bound()
    z = _draw(native, SEEDS, n, kind, stage, label).double().cpu().numpy()
    z64 = K.randn_keyed(SEEDS, n, kind, stage, label)
    err = np.abs(z - z64)
    worst = (err / np.maximum(np.abs(z64), 1e-300)).max()
    print(f"n={n} kind={kind}: max |z - z64| / |z64| = {worst:.2e} = 2^{np.log2(max(worst, 1e-300)):.1f}")
    assert (err <= bound * np.abs(z64) + 2.0 ** -126).all()
    assert np.abs(z).max() < 5.77


def test_device_labels_are_host_labels(native):
    """The label read on the device, t[b] * R[0] + r[b] (or t[b]), draws what the host label does."""
    n = 3 * 32 * 32
    t = torch.tensor([999, 5, 0, 17, 250], dtype=I64, device="cuda")
    r = torch.tensor([1, 0, 0, 2, 1], dtype=I64, device="cuda")
    R = torch.tensor([3], dtype=I64, device="cuda")
    for kind, kw, labels in ((1, dict(t=t), t.tolist()),
                             (3, dict(t=t, r=r, R=R), (t * 3 + r).tolist()),
                             (4, dict(t=t, r=r), (t + r).tolist())):
        dev = _draw(native, SEEDS, n, kind=kind, stage=2, **kw)
        for i, (s, lab) in enumerate(zip(SEEDS, labels)):
            assert torch.equal(dev[i], _draw(native, [s], n, kind=kind, stage=2, label=lab)[0]), (kind, i)


def test_checks(native):
    out = torch.zeros(2, 12, device="cuda")
    with pytest.raises(ValueError, match="seeds: expected at least 2 per-image seeds, got 1"):
        native.randn_keyed(out, torch.zeros(1, dtype=I64, device="cuda"), 2, 12, 1, 1)
    with pytest.raises(ValueError, match="contiguous"):
        native.randn_keyed(out, torch.zeros(4, dtype=I64, device="cuda")[::2], 2, 12, 1, 1)
    with pytest.raises(RuntimeError, match="unsupported"):
        native.randn_keyed(out, torch.zeros(2, dtype=I64, device="cuda"), 2, 12, 5, 1)


# ------------------------------------------------------------------------------------------------ the sampler
def _prompts(b=4, L=9, seed=21):
    gen = torch.Generator().manual_seed(seed)
    te = torch.randn(b, L, 512, generator=gen)
    tm = torch.ones(b, L, dtype=torch.bool)
    tm[1, 5:] = False
    tm[3, 2:] = False
    return te.cuda(), tm.cuda()


def test_batch_invariance(native):
    """sample(seed=[a, b, c, d]) on four random prompts: rows 2-3 are sample(seed=[c, d]) of those rows, row 1 is
    sample(seed=b) of row 1 alone (captured graphs at batch 4, 2 and 1)."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000, "cuda")
    te, tm = _prompts()
    seeds = [11, 2 ** 35, 3, 99]
    kw = dict(cond_scale=3., sampling_timesteps=8, ddim_eta=0.5)
    full = im.sample(text_embeds=te, text_masks=tm, seed=seeds, **kw)
    parts = [(slice(2, 4), seeds[2:]), (slice(1, 2), seeds[1:2])]
    for rows, s in parts:
        part = im.sample(text_embeds=te[rows], text_masks=tm[rows], seed=s, **kw)
        for i, j in enumerate(range(rows.start, rows.stop)):
            err = rel_l2(part[i], full[j])
            print(f"row {j} in a batch of {rows.stop - rows.start} vs of 4: rel-L2 {err:.3e}, bitwise "
                  f"{torch.equal(part[i], full[j])}")
            assert err <= 1e-5
    assert rel_l2(full[0], full[1]) > 0.1


def _sample(im, flavour, graph, seed):
    g = load_golden("sample_loop.pt")
    im.use_cuda_graph = graph
    gen = torch.Generator().manual_seed(5)
    kw = dict(text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda(), cond_scale=3.,
              sampling_timesteps=8, seed=seed)
    if flavour == "multistep":
        kw.update(sampler="dpmpp_2m")
    else:
        kw.update(ddim_eta=0.5)
    if flavour == "inpaint":
        mask = torch.zeros(2, 64, 64, dtype=torch.bool)
        mask[:, 16:48, 8:40] = True
        kw.update(inpaint_images=torch.rand(2, 3, 64, 64, generator=gen).cuda(), inpaint_masks=mask.cuda(),
                  inpaint_resample_times=2)
    if flavour == "img2img":
        kw.update(init_images=torch.rand(2, 3, 64, 64, generator=gen).cuda(), skip_steps=3)
    return im.sample(**kw)


@pytest.mark.parametrize("flavour", ["text", "inpaint", "multistep", "img2img"])
def test_graph_vs_eager_with_seed(native, flavour):
    g = load_golden("sample_loop.pt")
    outs = {}
    for graph in (False, True):
        im = _tiny_imagen(g, 1000, "cuda")
        outs[graph] = _sample(im, flavour, graph, [4, 2 ** 50])
        if graph:
            assert len(im._graphs) == 1 and ("seeded", 1) in next(iter(im._graphs))
    err = rel_l2(outs[True], outs[False])
    print(f"{flavour}: graph vs eager rel-L2 = {err:.3e}, bitwise {torch.equal(outs[True], outs[False])}")
    assert err <= 1e-5
    if flavour == "text":
        # the captured graph serves every seed: a second seed replays it and equals a fresh Imagen's eager loop
        other = _sample(im, flavour, True, 12345)
        assert len(im._graphs) == 1
        err2 = rel_l2(other, _sample(_tiny_imagen(g, 1000, "cuda"), flavour, False, [12345, 12346]))
        print(f"reused graph at another seed vs eager: rel-L2 = {err2:.3e}")
        assert err2 <= 1e-5 and rel_l2(other, outs[True]) > 0.1


def test_cascade_split(native):
    """A seeded two-stage cascade equals stage 1 alone (stop_at_unet_number=1), then stage 2 alone on its output."""
    from test_img2img import cascade
    im, g = cascade("cuda")
    im.noise_fn = None
    kw = dict(text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda(), cond_scale=2.,
              sampling_timesteps=(6, 5), ddim_eta=0.5, seed=77)
    both = im.sample(**kw)
    first = im.sample(stop_at_unet_number=1, **kw)
    second = im.sample(start_at_unet_number=2, start_images=first, **kw)
    err = rel_l2(second, both)
    print(f"split cascade vs whole: rel-L2 = {err:.3e}, bitwise {torch.equal(second, both)}")
    assert err <= 1e-5


def test_native_vs_emulated(native):
    """sample(seed=) on the tiny golden config: GPU (captured graph, keyed draws on the device) vs the CPU emulation
    (keyed draws from the restatement)."""
    import minimagen_b200.ops as ops_mod
    g = load_golden("sample_loop.pt")
    outs = {}
    for dev in ("cuda", "cpu"):
        prev = ops_mod._OPS
        if dev == "cpu":
            ops_mod.set_ops(EmuOps())
        try:
            im = _tiny_imagen(g, 1000, dev)
            outs[dev] = im.sample(text_embeds=g["text_embeds"].to(dev), text_masks=g["text_mask"].to(dev),
                                  cond_scale=3., sampling_timesteps=8, ddim_eta=0.5, seed=[6, 60]).cpu()
        finally:
            ops_mod.set_ops(prev)
    err = rel_l2(outs["cuda"], outs["cpu"])
    print(f"native vs emulated: rel-L2 = {err:.3e}")
    assert err < 1e-3


def test_seed_none_is_untouched(native, monkeypatch):
    """Without a seed no mi_randn_keyed is launched and the captured graph's key is the unseeded one; with one it is."""
    from minimagen_b200 import _native
    names = []
    call = _native.call
    monkeypatch.setattr(_native, "call", lambda name, *a: names.append(name) or call(name, *a))
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000, "cuda")
    kw = dict(text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda(), cond_scale=3.,
              sampling_timesteps=8, ddim_eta=0.5)
    a = im.sample(**kw)
    assert torch.isfinite(a).all() and "mi_randn_keyed" not in names
    sch = im.noise_schedulers[0]
    key = im._graph_key(im.unets[0], (2, 3, 64, 64), sch, kw["text_embeds"], kw["text_masks"], None, None, 3.)
    assert list(im._graphs) == [key] and not any("seeded" in str(k) for k in key)
    im.sample(seed=3, **kw)
    assert "mi_randn_keyed" in names and len(im._graphs) == 2
