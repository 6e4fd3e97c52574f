"""Negative prompts and per-image, per-stage guidance weights (Imagen.sample(negative_texts= / negative_text_embeds=,
cond_scale=number, [b] tensor or one entry per U-Net)) on the CPU, through the torch emulation of the ops interface
extended by the per-image weight array of mi_step_epilogue_w / mi_step_epilogue_multistep_w.  Covers the loop against the
restatement (negprompt_restatement.py) over DDPM and DDIM, the bitwise identities (equal weights = the scalar, all ones =
one U-Net pass, no negative = the null guidance), the batched guidance pass, the per-U-Net tuple, the argument checks, the
graph keys and two gloo ranks.  (The kernels, the captured graphs and their reuse are covered on the GPU in
test_gpu_guidance.py.)"""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import load_golden, rel_l2
from negprompt_restatement import negprompt_loop
from emu_ops import EmuOps
from test_respaced import _bank, _tiny_imagen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPE = (2, 3, 64, 64)


def _negative(b=2, L=6, seed=11):
    gen = torch.Generator().manual_seed(seed)
    nte = torch.randn(b, L, 512, generator=gen)
    ntm = torch.ones(b, L, dtype=torch.bool)
    ntm[0, 3:] = False
    return nte, ntm


def _loop(im, g, steps=None, eta=0., cond_scale=3., nte=None, ntm=None, seed=7):
    im.use_cuda_graph = False
    im.noise_fn = _bank(seed)
    sch = im.noise_schedulers[0]
    return im._p_sample_loop(im.unets[0], SHAPE, noise_scheduler=sch, text_embeds=g["text_embeds"],
                             text_mask=g["text_mask"], cond_scale=cond_scale,
                             schedule=None if steps is None else sch.sampling_schedule(steps, eta, "cpu"),
                             negative_text_embeds=nte, negative_text_mask=ntm)


def _count_forwards(unet):
    calls = []
    fwd = unet.forward
    unet.forward = lambda *a, **kw: calls.append(kw) or fwd(*a, **kw)
    return calls


# ------------------------------------------------------------------------------------------------ against the restatement
@pytest.mark.parametrize("T,steps,eta", [(25, None, 0.), (1000, 8, 0.5)])
def test_emulated_loop_vs_restatement(emu, T, steps, eta):
    """Negative prompt (one row's mask partly False) and per-image weights (2, 4.5) on sample_loop.pt's tiny U-Net, DDPM
    over T = 25 and DDIM S = 8 over T = 1000, vs the restated loop over the restated U-Net."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, T)
    nte, ntm = _negative()
    w = torch.tensor([2., 4.5])
    out = _loop(im, g, steps, eta, w, nte, ntm)
    ref = negprompt_loop(g["state_dict"], g["cfg"], SHAPE, T, _bank(7), w, text_embeds=g["text_embeds"],
                         text_mask=g["text_mask"], negative_text_embeds=nte, negative_text_mask=ntm, steps=steps,
                         eta=eta)
    err = rel_l2(out, ref)
    print(f"T={T} steps={steps}: rel-L2 vs restated negative-prompt loop = {err:.3e}")
    assert err < 1e-3
    assert emu.calls.count("step_epilogue") == (T if steps is None else steps)


def test_equal_weights_vector_is_the_scalar(emu):
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    nte, ntm = _negative()
    for neg in ((None, None), (nte, ntm)):
        a = _loop(im, g, 6, 0.5, 3., *neg)
        b = _loop(im, g, 6, 0.5, torch.full((2,), 3.), *neg)
        assert torch.equal(a, b)


def test_all_ones_runs_one_pass_and_is_cond_scale_1(emu):
    """An all-ones weight vector runs one U-Net pass per step, whatever negative is given, and gives cond_scale=1's bits."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    calls = _count_forwards(im.unets[0])
    one = _loop(im, g, 6, 0., 1.)
    assert len(calls) == 6
    nte, ntm = _negative()
    del calls[:]
    ones = _loop(im, g, 6, 0., torch.ones(2), nte, ntm)
    assert len(calls) == 6 and torch.equal(ones, one)
    del calls[:]
    _loop(im, g, 6, 0., torch.tensor([1., 2.]), nte, ntm)           # one image guided: the guidance pass runs
    assert len(calls) == 12


def test_no_negative_is_the_null_guidance(emu):
    """Without a negative the guidance pass is the reference's null pass (cond_drop_prob 1): bit for bit the loop of
    Unet.forward_with_cond_scale's combine fed to the step as its model output."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    calls = _count_forwards(im.unets[0])
    out = _loop(im, g, 5, 0.5, 3.)
    assert [kw.get("cond_drop_prob", 0.) for kw in calls] == [0., 1.] * 5
    u, sch = im.unets[0], im.noise_schedulers[0]
    walk = sch.sampling_schedule(5, 0.5, "cpu")
    bank = _bank(7)
    x = bank("init", SHAPE, -1)
    with torch.no_grad():
        for t in walk.grid:
            times = torch.full((2,), t, dtype=torch.long)
            eps = u.forward_with_cond_scale(x, times, text_embeds=g["text_embeds"], text_mask=g["text_mask"],
                                            cond_scale=3.)
            x = im._step(u, x, times, bank("step", SHAPE, t), noise_scheduler=sch, text_embeds=None, text_mask=None,
                         lowres_cond_img=None, lowres_noise_times=None, cond_scale=1., model_output=eps, schedule=walk)
    assert torch.equal(out, (x.clamp(-1, 1) + 1) * 0.5)
    nte, ntm = _negative()
    neg = _loop(im, g, 5, 0.5, 3., nte, ntm)
    err = rel_l2(neg, out)
    print(f"negative prompt vs null guidance: rel-L2 = {err:.3e}")
    assert err > 1e-2                                                 # far beyond rounding


@pytest.mark.parametrize("case", ["equal", "padded", "no_mask", "no_masks_equal"])
def test_cfg_batched_with_negative(emu, case):
    """cfg_batched puts the negative pass in the 2B batch when padding is exact (both masks, any lengths; or no masks and
    equal lengths) and falls back to two passes otherwise; either way it matches the unbatched path."""
    g = load_golden("sample_loop.pt")
    te, tm = g["text_embeds"], g["text_mask"]
    nte, ntm = _negative(L={"equal": 9, "padded": 4, "no_mask": 4, "no_masks_equal": 9}[case])
    if case == "no_mask":
        ntm = None
    if case == "no_masks_equal":
        tm = ntm = None
    outs, batched = [], []
    for cfg_batched in (False, True):
        im = _tiny_imagen(g, 1000)
        im.cfg_batched = cfg_batched
        fwd = im.unets[0]._forward_impl
        im.unets[0]._forward_impl = lambda *a, **kw: batched.append(a[0].shape[0]) or fwd(*a, **kw)
        im.use_cuda_graph = False
        im.noise_fn = _bank(3)
        sch = im.noise_schedulers[0]
        outs.append(im._p_sample_loop(im.unets[0], SHAPE, noise_scheduler=sch, text_embeds=te, text_mask=tm,
                                      cond_scale=torch.tensor([3., 2.]), schedule=sch.sampling_schedule(4, 0., "cpu"),
                                      negative_text_embeds=nte, negative_text_mask=ntm))
    err = rel_l2(outs[1], outs[0])
    print(f"{case}: batched vs unbatched rel-L2 = {err:.3e}")
    # padding is exact up to rounding: the text projection runs over more rows (4.4e-5 after 4 steps at w = 3)
    assert err < 1e-4
    assert (4 in batched) == (case != "no_mask")


def test_cascade_per_unet_scales_equal_stage_by_stage(emu):
    """cond_scale=(w1, w2) on the tiny cascade == stage 1 alone at w1, then stage 2 alone at w2 from its output."""
    from test_host_logic import _cascade_from_golden
    g = load_golden("cascade_tiny.pt")
    gen = torch.Generator().manual_seed(6)
    bank = {}

    def noise_fn(kind, shape, step):
        key = (kind, step, tuple(shape))
        if key not in bank:
            bank[key] = torch.randn(shape, generator=gen)
        return bank[key]
    im, _ = _cascade_from_golden(g, "cpu")
    im.noise_fn = noise_fn
    nte, ntm = _negative(L=5)
    w1 = torch.tensor([1.5, 3.])
    kw = dict(text_embeds=g["text_embeds"], text_masks=g["text_mask"], sampling_timesteps=(5, 4),
              negative_text_embeds=nte[:1], negative_text_masks=ntm[:1])
    both = im.sample(cond_scale=(w1, 4.), **kw)
    first = im.sample(cond_scale=w1, stop_at_unet_number=1, **kw)
    second = im.sample(cond_scale=4., start_at_unet_number=2, start_images=first, **kw)
    assert torch.equal(both, second)
    other = im.sample(cond_scale=(w1, 2.), **kw)
    assert not torch.equal(other, both)


def test_negative_texts_are_encoded(emu, monkeypatch):
    """negative_texts go through t5_encode_text like texts; one str is used for every image."""
    import minimagen_b200.Imagen as I
    nte, ntm = _negative(b=1, L=5)
    seen = []

    def fake_encode(texts, name):
        seen.append(list(texts))
        return nte.clone(), ntm.clone()
    monkeypatch.setattr(I, "t5_encode_text", fake_encode)
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    im.use_cuda_graph = False
    outs = []
    for neg in (dict(negative_texts="blurry, low quality"), dict(negative_text_embeds=nte, negative_text_masks=ntm)):
        im.noise_fn = _bank(5)
        outs.append(im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=3.,
                              sampling_timesteps=4, **neg))
    assert seen == [["blurry, low quality"]]
    assert torch.equal(outs[0], outs[1])
    im.noise_fn = _bank(5)
    im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=3., sampling_timesteps=4,
              negative_texts=["a", "b"])
    assert seen[-1] == ["a", "b"]


def test_argument_checks(emu):
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet, BaseTest, SuperTest
    im = Imagen(unets=(Unet(**BaseTest.defaults), Unet(**SuperTest.defaults)), text_encoder_name="t5_small",
                image_sizes=(16, 32), timesteps=25, cond_drop_prob=0.1)
    te = torch.zeros(2, 4, 512)
    nte = torch.zeros(2, 3, 512)
    with pytest.raises(AssertionError, match="negative_texts and negative_text_embeds cannot both be given"):
        im.sample(text_embeds=te, negative_texts="x", negative_text_embeds=nte)
    with pytest.raises(AssertionError, match="negative_text_masks need negative_text_embeds"):
        im.sample(text_embeds=te, negative_text_masks=torch.ones(2, 3, dtype=torch.bool))
    with pytest.raises(AssertionError, match=r"negative_text_embeds must be \(1 or b, n, text_embed_dim\) = "
                                             r"\(1 or 2, n, 512\), got \(3, 3, 512\)"):
        im.sample(text_embeds=te, negative_text_embeds=torch.zeros(3, 3, 512))
    with pytest.raises(AssertionError, match=r"got \(2, 3, 7\)"):
        im.sample(text_embeds=te, negative_text_embeds=torch.zeros(2, 3, 7))
    with pytest.raises(AssertionError, match=r"negative_text_masks must be \(rows, n\) = \(2, 3\)"):
        im.sample(text_embeds=te, negative_text_embeds=nte, negative_text_masks=torch.ones(2, 4, dtype=torch.bool))
    with pytest.raises(AssertionError, match="negative_texts must be a str or a list of 1 or b = 2 str, got 3"):
        im.sample(text_embeds=te, negative_texts=["a", "b", "c"])
    with pytest.raises(AssertionError, match="cond_scale must have one entry per unet"):
        im.sample(text_embeds=te, cond_scale=(3.,))
    for bad in (float("nan"), float("inf"), "3", None):
        with pytest.raises(AssertionError, match="cond_scale of unet 1 must be a finite number or a 1-D float tensor"):
            im.sample(text_embeds=te, cond_scale=bad)
    with pytest.raises(AssertionError, match="cond_scale of unet 2 must be a finite number"):
        im.sample(text_embeds=te, cond_scale=(3., float("nan")))
    with pytest.raises(AssertionError, match=r"cond_scale of unet 1 must be a 1-D float tensor of b = 2 per-image "
                                             r"weights, got \(3,\)"):
        im.sample(text_embeds=te, cond_scale=torch.ones(3))
    for bad in (torch.ones(2, 1), torch.ones(2, dtype=torch.long)):
        with pytest.raises(AssertionError, match="cond_scale of unet 1 must be a 1-D float tensor of b = 2"):
            im.sample(text_embeds=te, cond_scale=bad)
    with pytest.raises(AssertionError, match=r"cond_scale of unet 2 must be finite, got \[3.0, nan\]"):
        im.sample(text_embeds=te, cond_scale=(2., torch.tensor([3., float("nan")])))
    plain = Imagen(unets=Unet(**BaseTest.defaults), text_encoder_name="t5_small", image_sizes=(16,), timesteps=25,
                   cond_drop_prob=0.)
    with pytest.raises(AssertionError, match="classifier free guidance"):
        plain.sample(text_embeds=te, cond_scale=torch.tensor([1., 2.]))


# ------------------------------------------------------------------------------------------------ graph keys
def test_graph_keys_serve_every_scale():
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 25)
    sch = im.noise_schedulers[0]
    nte, ntm = _negative()
    key = lambda w, **neg: im._graph_key(im.unets[0], SHAPE, sch, g["text_embeds"], g["text_mask"], None, None, w, **neg)
    assert key(3.) == key(5.) == key(torch.tensor([2., 7.])) == key(torch.tensor([1., 2.]))
    assert key(1.) == key(torch.ones(2)) != key(3.)
    assert key(3., negative_text_embeds=nte, negative_text_mask=ntm) == \
        key(torch.tensor([4., 1.]), negative_text_embeds=nte * 2, negative_text_mask=ntm)
    assert key(3., negative_text_embeds=nte, negative_text_mask=ntm) != key(3.)
    assert key(3., negative_text_embeds=nte, negative_text_mask=ntm) != \
        key(3., negative_text_embeds=nte[:, :4], negative_text_mask=ntm[:, :4])
    assert key(1., negative_text_embeds=nte, negative_text_mask=ntm) == key(1.)      # unguided: the negative is unused

    class Cached:
        def __init__(self):
            self.ws, self.conds = [], []

        def set_cond(self, w=None, **cond):
            self.ws.append(w)
            self.conds.append(cond)

        def set_schedule(self, sched):
            pass

    guided, neg = Cached(), Cached()
    im._graphs = {key(3.): guided, key(3., negative_text_embeds=nte, negative_text_mask=ntm): neg}
    kw = dict(noise_scheduler=sch, text_embeds=g["text_embeds"], text_mask=g["text_mask"], lowres_cond_img=None,
              lowres_noise_times=None)
    assert im._step_graph(im.unets[0], SHAPE, cond_scale=5., **kw) is guided
    assert im._step_graph(im.unets[0], SHAPE, cond_scale=torch.tensor([2., 6.]), **kw) is guided
    assert im._step_graph(im.unets[0], SHAPE, cond_scale=3., negative_text_embeds=nte, negative_text_mask=ntm,
                          **kw) is neg
    assert [w.tolist() for w in guided.ws] == [[5., 5.], [2., 6.]] and neg.ws[0].tolist() == [3., 3.]
    assert neg.conds[0]["negative_text_embeds"] is nte and guided.conds[0]["negative_text_embeds"] is None
    assert len(im._graphs) == 2


# ------------------------------------------------------------------------------------------------ two gloo ranks
def _dist_inputs(B):
    gen = torch.Generator().manual_seed(7)
    te = torch.randn(B, 9, 512, generator=gen)
    tm = torch.ones(B, 9, dtype=torch.bool)
    tm[1, 4:] = False
    nte = torch.randn(B, 5, 512, generator=gen)
    ntm = torch.ones(B, 5, dtype=torch.bool)
    ntm[2, 2:] = False
    return dict(text_embeds=te, text_masks=tm, negative_text_embeds=nte, negative_text_masks=ntm,
                cond_scale=torch.tensor([1., 2., 3.5, 5.]), sampling_timesteps=5)


def _worker(rank, world, port, out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import minimagen_b200.ops as ops_mod
    from test_distributed_cpu import _build, _noise_bank
    ops_mod.set_ops(EmuOps())
    g = torch.load(os.path.join(ROOT, "tests", "golden", "sample_loop.pt"), map_location="cpu", weights_only=False)
    im = _build(g)
    B = 4
    bank = _noise_bank(B)
    per = B // world
    im.noise_fn = lambda kind, shape, step: bank[(kind, step)][rank * per:(rank + 1) * per]
    out = im.sample(distributed=True, **_dist_inputs(B))
    assert out.shape == (B, 3, 64, 64)
    if rank == 0:
        torch.save(out, out_path)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_rank_gloo_with_negative_and_per_image_scales(tmp_path, emu):
    from test_distributed_cpu import _build, _noise_bank
    port = 29400 + (os.getpid() % 200)
    out_path = str(tmp_path / "dist_out.pt")
    mp.spawn(_worker, args=(2, port, out_path), nprocs=2, join=True)
    dist_out = torch.load(out_path)
    g = load_golden("sample_loop.pt")
    im = _build(g)
    bank = _noise_bank(4)
    im.noise_fn = lambda kind, shape, step: bank[(kind, step)]
    full = im.sample(**_dist_inputs(4))
    err = rel_l2(dist_out, full)
    print(f"two ranks vs one process: rel-L2 = {err:.3e}, max abs {(dist_out - full).abs().max():.3e}")
    # the CPU GEMM of the negative prompt's projection rounds differently over 10 and 20 rows (7.7e-7), amplified by
    # the weights up to 5 to 5.5e-5; without a negative the two runs are bitwise equal.  A wrong shard would be O(1).
    assert err < 2e-4
