"""Per-image seeds (Imagen.sample(seed=)) on the CPU, through the torch emulation of the ops interface extended by
mi_randn_keyed (its draws come from keyed_noise_restatement.py).  Covers the restated generator against the Random123
known-answer vectors and the moments / KS statistic / cross-correlations of its normals, the seeded sampler taking exactly
the (kind, label) draws of a noise_fn run with the right stage (DDPM, DDIM, RePaint, 2M, img2img, a two-stage cascade),
int seeds against lists, an image regenerated alone, the argument checks, the graph keys, and two gloo ranks without
noise_fn.  (The kernel, the captured graphs and the native sampler are covered on the GPU in test_gpu_seeded.py.)"""
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import keyed_noise_restatement as K
from conftest import load_golden, rel_l2
from emu_ops import EmuOps
from test_respaced import _tiny_imagen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ the generator
@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    """Philox4x32-10 known-answer vectors of Random123 (kat_vectors)."""
    got = K.philox4x32_10([np.uint64(c) for c in ctr], [np.uint64(k) for k in key])
    assert tuple(int(w) for w in got) == want


def test_counter_layout():
    """Element j is lane j % 4 of quad j / 4 of the counter (q, label mod 2^32, kind, stage), keyed by (lo32, hi32)."""
    seed = (0x12345678 << 32) | 0x9abcdef0
    x = K.bits(seed, 10, 3, 2, -1)
    for q in range(3):
        want = K.philox4x32_10([np.uint64(v) for v in (q, 0xffffffff, 3, 2)],
                               [np.uint64(0x9abcdef0), np.uint64(0x12345678)])
        assert [int(w) for w in x[q]] == [int(w) for w in want]
    u, v = K.uv(x)
    assert u.min() > 0 and u.max() < 1 and v.min() >= 0 and v.max() < 1
    z = K.normals64(seed, 10, 3, 2, -1)
    assert z.shape == (10,)
    assert np.array_equal(z, K.normals64(seed, 12, 3, 2, -1)[:10])          # a longer row is the same prefix
    assert math.sqrt(-2 * math.log(2.0 ** -24)) < 5.77                      # |z| bound: u >= 2^-24


N_STATS = 32 * 3 * 256 * 256


def _stats_draw(seed0=0, kind=1, stage=1, label=999):
    return K.randn_keyed(list(range(seed0, seed0 + 32)), 3 * 256 * 256, kind, stage, label).reshape(-1)


def test_normal_statistics():
    """Over 32 x 3 x 256^2 draws: mean and variance within 5 sigma of N(0, 1)'s, the KS test at p = 1e-3, |z| < 5.77."""
    from scipy import stats
    z = _stats_draw()
    N = z.size
    assert N == N_STATS
    mean, var = z.mean(), z.var()
    ks = stats.kstest(z, "norm")
    print(f"mean {mean:.2e} (5 sigma {5 / math.sqrt(N):.2e}), var - 1 {var - 1:.2e} (5 sigma "
          f"{5 * math.sqrt(2 / N):.2e}), KS {ks.statistic:.2e} p = {ks.pvalue:.3f}, max |z| {np.abs(z).max():.3f}")
    assert abs(mean) < 5 / math.sqrt(N)
    assert abs(var - 1) < 5 * math.sqrt(2 / N)
    assert ks.pvalue > 1e-3
    assert np.abs(z).max() < 5.77


@pytest.mark.parametrize("other", ["seed", "label", "kind", "stage"])
def test_draws_are_uncorrelated(other):
    """Draws that differ only in the seed, the label, the kind or the stage: |corr| < 5 / sqrt(N)."""
    z = _stats_draw()
    w = _stats_draw(**{"seed": dict(seed0=32), "label": dict(label=998), "kind": dict(kind=4),
                       "stage": dict(stage=2)}[other])
    corr = np.corrcoef(z, w)[0, 1]
    print(f"{other}: corr = {corr:.2e} (bound {5 / math.sqrt(z.size):.2e})")
    assert abs(corr) < 5 / math.sqrt(z.size)


def test_native_ops_checks_seed_count():
    from minimagen_b200.ops import NativeOps
    out = torch.zeros(2, 12)
    with pytest.raises(ValueError, match="seeds: expected at least 2 per-image seeds, got 1"):
        NativeOps().randn_keyed(out, torch.zeros(1, dtype=torch.long), 2, 12, 1, 1)
    with pytest.raises(TypeError, match="seeds: expected torch.int64"):
        NativeOps().randn_keyed(out, torch.zeros(2, dtype=torch.int32), 2, 12, 1, 1)


# ------------------------------------------------------------------------------------------------ the sampler's draws
def _recorder(seed=3):
    gen = torch.Generator().manual_seed(seed)
    calls = []

    def noise_fn(kind, shape, step):
        calls.append((kind, step))
        return torch.randn(tuple(shape), generator=gen)
    noise_fn.calls = calls
    return noise_fn


def _plan_kwargs(case):
    gen = torch.Generator().manual_seed(4)
    if case == "ddpm":
        return 25, {}
    if case == "ddim_eta":
        return 1000, dict(sampling_timesteps=6, ddim_eta=0.5)
    if case == "inpaint":
        mask = torch.zeros(2, 64, 64, dtype=torch.bool)
        mask[:, 8:40, 16:48] = True
        return 1000, dict(sampling_timesteps=5, ddim_eta=0.5, inpaint_images=torch.rand(2, 3, 64, 64, generator=gen),
                          inpaint_masks=mask, inpaint_resample_times=2)
    if case == "dpmpp_2m":
        return 1000, dict(sampling_timesteps=6, sampler="dpmpp_2m")
    if case == "img2img":
        return 1000, dict(sampling_timesteps=8, init_images=torch.rand(2, 3, 64, 64, generator=gen), skip_steps=3)
    raise ValueError(case)


@pytest.mark.parametrize("case", ["ddpm", "ddim_eta", "inpaint", "dpmpp_2m", "img2img"])
def test_seeded_draws_follow_the_noise_fn_plan(emu, case):
    """A seeded sample takes exactly the (kind, label) draws a noise_fn run requests, in the same order, at stage 1, with
    one label for every image."""
    g = load_golden("sample_loop.pt")
    T, kw = _plan_kwargs(case)
    im = _tiny_imagen(g, T)
    im.noise_fn = rec = _recorder()
    cond = dict(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=1.)
    im.sample(**cond, **kw)
    im.noise_fn = None
    out = im.sample(**cond, seed=17, **kw)
    got = [(kind, labels[0]) for kind, labels, _ in emu.keyed]
    assert got == rec.calls
    assert all(len(set(labels)) == 1 and stage == 1 for _, labels, stage in emu.keyed)
    assert torch.isfinite(out).all()
    if case == "inpaint":
        assert ("renoise", 999 * 2 + 1) in got and ("inpaint", 0) in got


def test_cascade_draws_carry_the_stage(emu):
    """Two-stage cascade: the seeded draws are the noise_fn run's, stage 1's with stage 1, the low-res augmentation
    (label 2) and stage 2's with stage 2."""
    from test_host_logic import _cascade_from_golden
    g = load_golden("cascade_tiny.pt")
    im, _ = _cascade_from_golden(g, "cpu")
    im.noise_fn = rec = _recorder()
    kw = dict(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=2., sampling_timesteps=(5, 4),
              ddim_eta=0.5)
    im.sample(**kw)
    im.noise_fn = None
    im.sample(seed=[5, 9], **kw)
    got = [(kind, labels[0]) for kind, labels, _ in emu.keyed]
    assert got == rec.calls
    stages = [stage for _, _, stage in emu.keyed]
    lowres = got.index(("lowres", 2))
    assert stages[:lowres] == [1] * lowres and stages[lowres:] == [2] * (len(stages) - lowres)
    assert all(labels_ == [labels_[0]] * 2 for _, labels_, _ in emu.keyed)


def test_int_seed_is_the_list(emu):
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    kw = dict(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=3., sampling_timesteps=5,
              ddim_eta=0.5)
    a = im.sample(seed=41, **kw)
    assert torch.equal(a, im.sample(seed=[41, 42], **kw))
    assert torch.equal(a, im.sample(seed=torch.tensor([41, 42]), **kw))
    assert not torch.equal(a, im.sample(seed=42, **kw))
    assert emu.keyed[0] == ("init", [-1, -1], 1)


def test_an_image_regenerates_alone(emu):
    """Row 1 of a seed-[a, b] batch is the seed-[b] run of row 1 alone: its draws do not depend on the batch."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    kw = dict(cond_scale=3., sampling_timesteps=5, ddim_eta=0.5)
    both = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], seed=[8, 30], **kw)
    alone = im.sample(text_embeds=g["text_embeds"][1:], text_masks=g["text_mask"][1:], seed=30, **kw)
    err = rel_l2(alone[0], both[1])
    print(f"row 1 alone vs in the batch: rel-L2 = {err:.3e}, bitwise {torch.equal(alone[0], both[1])}")
    # the CPU convolutions and GEMMs round differently over 1 and 2 rows (5.5e-5 after 5 steps at w = 3); other draws
    # would be O(1) apart, like row 0's.  The GPU test holds the native sampler to 1e-5.
    assert err < 1e-3
    assert rel_l2(alone[0], both[0]) > 0.1


def test_seed_none_is_unchanged(emu):
    """No keyed draw without a seed, and the graph keys of unseeded loops are those of before."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 25)
    torch.manual_seed(0)
    a = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=3., sampling_timesteps=4)
    torch.manual_seed(0)
    b = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=3., sampling_timesteps=4)
    assert torch.equal(a, b) and "randn_keyed" not in emu.calls and not emu.keyed
    sch = im.noise_schedulers[0]
    key = lambda **kw: im._graph_key(im.unets[0], (2, 3, 64, 64), sch, g["text_embeds"], g["text_mask"], None, None,
                                     3., **kw)
    assert key() == key(seeded=False) and all("seeded" not in str(k) for k in key())
    assert key(seeded=True, stage=1) != key() and key(seeded=True, stage=1) != key(seeded=True, stage=2)
    assert key(seeded=True, stage=1)[:len(key())] == key()


def test_argument_checks(emu):
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet, BaseTest
    im = Imagen(unets=Unet(**BaseTest.defaults), text_encoder_name="t5_small", image_sizes=(16,), timesteps=25,
                cond_drop_prob=0.1)
    te = torch.zeros(2, 4, 512)
    im.noise_fn = lambda kind, shape, step: torch.zeros(shape)
    with pytest.raises(AssertionError, match="seed and noise_fn cannot both be given"):
        im.sample(text_embeds=te, seed=1)
    im.noise_fn = None
    with pytest.raises(AssertionError, match="seed must be >= 0, got -1"):
        im.sample(text_embeds=te, seed=-1)
    for bad in (True, 1.5, "3", [1, 2.0], [], torch.ones(2), torch.ones(2, 1, dtype=torch.long),
                torch.ones(2, dtype=torch.bool)):
        with pytest.raises(AssertionError, match="seed must be an int, or a list or 1-D integer tensor"):
            im.sample(text_embeds=te, seed=bad)
    with pytest.raises(AssertionError, match=r"per-image seeds must be between 0 and 2\^63 - 1, got \[1, -2\]"):
        im.sample(text_embeds=te, seed=[1, -2])
    with pytest.raises(AssertionError, match=r"per-image seeds must be between 0 and 2\^63 - 1"):
        im.sample(text_embeds=te, seed=[1, 2 ** 63])
    with pytest.raises(AssertionError, match=r"seed must have one entry per image \(b = 2\), got 3"):
        im.sample(text_embeds=te, seed=[1, 2, 3])
    with pytest.raises(AssertionError, match=r"seed \+ b - 1 must be below 2\^63"):
        im.sample(text_embeds=te, seed=2 ** 63 - 1)
    with pytest.raises(AssertionError, match=r"timesteps \* inpaint_resample_times must be below 2\^31"):
        im.sample(text_embeds=te, seed=1, inpaint_images=torch.zeros(2, 3, 16, 16),
                  inpaint_masks=torch.ones(2, 16, 16, dtype=torch.bool), inpaint_resample_times=2 ** 27)
    assert not emu.keyed


# ------------------------------------------------------------------------------------------------ two gloo ranks
def _dist_inputs(B):
    gen = torch.Generator().manual_seed(7)
    te = torch.randn(B, 9, 512, generator=gen)
    tm = torch.ones(B, 9, dtype=torch.bool)
    tm[1, 4:] = False
    return dict(text_embeds=te, text_masks=tm, cond_scale=3., sampling_timesteps=5, ddim_eta=0.5, seed=1234)


def _worker(rank, world, port, out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import minimagen_b200.ops as ops_mod
    from test_distributed_cpu import _build
    ops_mod.set_ops(EmuOps())
    g = torch.load(os.path.join(ROOT, "tests", "golden", "sample_loop.pt"), map_location="cpu", weights_only=False)
    im = _build(g)
    out = im.sample(distributed=True, **_dist_inputs(4))
    assert out.shape == (4, 3, 64, 64)
    if rank == 0:
        torch.save(out, out_path)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_rank_gloo_with_seed_only(tmp_path, emu):
    """distributed=True with a seed and no noise_fn: the gathered batch is the single-process one."""
    from test_distributed_cpu import _build
    port = 29800 + (os.getpid() % 150)
    out_path = str(tmp_path / "dist_out.pt")
    mp.spawn(_worker, args=(2, port, out_path), nprocs=2, join=True)
    dist_out = torch.load(out_path)
    full = _build(load_golden("sample_loop.pt")).sample(**_dist_inputs(4))
    print(f"two ranks vs one process: max abs {(dist_out - full).abs().max():.3e}")
    assert torch.allclose(dist_out, full, atol=1e-5)
