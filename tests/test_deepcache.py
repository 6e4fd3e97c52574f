"""DeepCache feature reuse (`Imagen.sample(..., cache_interval=N)`) on a machine without a GPU:

  * argument validation and its messages;
  * `deepcache_plan` against a hand-written table (intervals 1-5, guidance switching on and off mid-walk), and the plan a
    whole sample follows over its actual loop (RePaint iterations, skip_steps);
  * the U-Net's store and read passes as exact dataflow: the product's host code in float64 on the no-rounding backend
    (tests/test_lowering_exact.py's `exact` fixture) against tests/deepcache_restatement.py's split of the restatement,
    per element to 1e-12;
  * the sequence of U-Net passes whole emulated two-stage samples run, recorded by a spy on Unet._forward_dev: full or
    cached, which pass (rows of the cache), and which iteration stored what each read pass reads;
  * the same kind of samples with every kernel call checked against float64 (tests/checking_ops.py).
"""
import pytest
import torch

import deepcache_restatement as D
from checking_ops import ALLOWED, CheckingOps
from conftest import load_golden
from oracle import restatement as R
from test_host_logic import _cascade_from_golden
from test_lowering_exact import BIG, _arena, _exact, _inputs, _unet, exact  # noqa: F401  (exact: fixture)
from test_respaced import _tiny_imagen
from test_sampling_feature_calls import SMS, cascade_case, reached

T_, F_ = True, False


# ------------------------------------------------------------------------------------------------ validation
@pytest.mark.parametrize("value,msg", [
    (True, "cache_interval of unet 1 must be None or an int >= 1, got True"),
    (0, "cache_interval of unet 1 must be None or an int >= 1, got 0"),
    (-3, "cache_interval of unet 1 must be None or an int >= 1, got -3"),
    (2.0, "cache_interval of unet 1 must be None or an int >= 1, got 2.0"),
    ((2, 3), "cache_interval must have one entry per unet (1), got 2"),
    ([False], "cache_interval of unet 1 must be None or an int >= 1, got False"),
])
def test_cache_interval_validation(value, msg):
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 25)
    with pytest.raises(AssertionError) as e:
        im.sample(text_embeds=g["text_embeds"], cache_interval=value)
    assert str(e.value) == msg


# ------------------------------------------------------------------------------------------------ the plan
PLANS = [   # (on, N, full)
    ([T_] * 7, None, [T_] * 7),
    ([T_] * 7, 1, [T_] * 7),
    ([T_] * 7, 2, [T_, F_, T_, F_, T_, F_, T_]),
    ([T_] * 7, 3, [T_, F_, F_, T_, F_, F_, T_]),
    ([T_] * 7, 4, [T_, F_, F_, F_, T_, F_, F_]),
    ([F_] * 7, 5, [T_, F_, F_, F_, F_, T_, F_]),
    # guidance switched on mid-walk: the first guided iteration after an unguided full one is full
    ([F_, F_, T_, T_, T_, F_, F_, T_], 3, [T_, F_, T_, F_, F_, T_, F_, T_]),
    ([F_, F_, T_, T_, T_, F_, F_, T_], 2, [T_, F_, T_, F_, T_, F_, T_, T_]),
    ([F_, F_, T_, T_, T_, F_, F_, T_], 5, [T_, F_, T_, F_, F_, F_, F_, T_]),
    # switched off: an unguided iteration reads the conditional feature of a guided full one
    ([T_, T_, F_, F_, F_, T_], 4, [T_, F_, F_, F_, T_, T_]),
    ([T_, F_, T_, F_, T_, F_], 3, [T_, F_, F_, T_, T_, F_]),
    # a RePaint walk of S = 4 grid points at R = 2 is 7 iterations; guided at the first 4 (an interval)
    ([T_, T_, T_, T_, F_, F_, F_], 2, [T_, F_, T_, F_, T_, F_, T_]),
    # a walk shortened by skip_steps / max_steps is a shorter `on`: the plan restarts with it
    ([T_, T_, T_], 5, [T_, F_, F_]),
    ([T_], 3, [T_]),
    ([], 3, []),
]


@pytest.mark.parametrize("on,N,full", PLANS)
def test_deepcache_plan_table(on, N, full):
    from minimagen_b200.Imagen import deepcache_plan
    assert deepcache_plan(on, N) == full


# ------------------------------------------------------------------------------------------------ exact dataflow
_GOLD = load_golden("cascade_tiny.pt")["cfgs"]
SPLIT_CFGS = {
    "tiny_base": (dict(_GOLD[0]), 16, 2),                                   # not memory-efficient: Downsample after level 0
    "tiny_sr": (dict(_GOLD[1], lowres_cond=True), 32, 2),                   # memory-efficient: level 0 at half size
    # attention and cross-attention at level 0, three ResnetBlocks there, tensor-core shaped
    "attn_level0": (dict(dim=64, dim_mults=(1, 2), num_resnet_blocks=(3, 1), layer_attns=(True, False),
                         layer_cross_attns=(True, False), text_embed_dim=768), 32, 2),
    # one resolution: the kept feature is mid_block2's output
    "one_level": (dict(dim=64, dim_mults=(1,), num_resnet_blocks=2, layer_attns=True, layer_cross_attns=True,
                       text_embed_dim=768), 16, 2),
}


@pytest.mark.parametrize("name", list(SPLIT_CFGS))
def test_store_and_read_passes_exact(exact, name):
    from minimagen_b200.Unet import DeepCache
    cfg, s, b = SPLIT_CFGS[name]
    u, sd = _unet(cfg)
    x, t, kw = _inputs(cfg, s, b)
    x2, _, _ = _inputs(cfg, s, b, seed=8)
    t2 = torch.tensor([998, 1, 400][:b])
    cache = DeepCache(2 * b)
    with torch.no_grad(), _arena(BIG):
        for row0, drop in ((0, 0.), (b, 1.)):           # the conditional and the guidance pass, each in its rows
            what = f"{name} cond_drop_prob={drop}"
            ref = R.unet_forward(sd, cfg, x, t, cond_drop_prob=drop, **kw)
            feat = D.deep(sd, cfg, x, t, cond_drop_prob=drop, **kw)
            _exact(D.shallow(sd, cfg, feat, x, t, cond_drop_prob=drop, **kw), ref, f"{what}: deep + shallow")
            stored = u._forward_impl(x, t, cond_drop_prob=drop, deepcache=('store', cache, row0), **kw)
            _exact(stored, ref, f"{what}: store pass")
            same = u._forward_impl(x, t, cond_drop_prob=drop, deepcache=('read', cache, row0), **kw)
            assert torch.equal(same, stored), f"{what}: a read at the store's inputs differs from the store pass"
            read = u._forward_impl(x2, t2, cond_drop_prob=drop, deepcache=('read', cache, row0), **kw)
            _exact(read, D.shallow(sd, cfg, feat, x2, t2, cond_drop_prob=drop, **kw), f"{what}: read pass at (x2, t2)")


def test_read_pass_skips_the_deep_levels(exact):
    """A read pass runs no kernel of the levels below 0: fewer conv launches than a full pass, and no mid block GEMMs."""
    from minimagen_b200.Unet import DeepCache
    cfg, s, b = SPLIT_CFGS["attn_level0"]
    u, _ = _unet(cfg)
    x, t, kw = _inputs(cfg, s, b)
    cache = DeepCache(b)
    with torch.no_grad(), _arena(BIG):
        exact.conv_log.clear()
        u._forward_impl(x, t, deepcache=('store', cache, 0), **kw)
        full = len(exact.conv_log)
        exact.conv_log.clear()
        u._forward_impl(x, t, deepcache=('read', cache, 0), **kw)
        read = len(exact.conv_log)
    print(f"attn_level0: {full} conv launches in a full pass, {read} in a read pass")
    assert 0 < read < full


def test_caching_needs_no_grad_and_a_stored_feature(emu):
    from minimagen_b200.Unet import DeepCache
    cfg, s, b = SPLIT_CFGS["tiny_base"]
    u, _ = _unet(cfg)
    u.float()
    x, t, kw = _inputs(cfg, s, b)
    x, kw = x.float(), {k: (v.float() if v.is_floating_point() else v) for k, v in kw.items()}
    with pytest.raises(AssertionError, match="feature caching is for sampling"):
        u._forward_dev(x, t, deepcache=('store', DeepCache(b), 0), **kw)
    with torch.no_grad(), pytest.raises(AssertionError, match="a read pass needs a feature stored before it"):
        u._forward_dev(x, t, deepcache=('read', DeepCache(b), 0), **kw)


# ------------------------------------------------------------------------------------------------ the passes of a sample
class PassSpy:
    """Records every U-Net pass: (mode, row0, batch, t of the pass, t the read rows were stored at)."""

    def __init__(self, monkeypatch):
        from minimagen_b200.Unet import Unet
        self.passes, self.stored = [], {}
        orig = Unet._forward_dev

        def spy(unet, x, time, *a, deepcache=None, **k):
            mode, cache, row0 = deepcache if deepcache is not None else (None, None, 0)
            t, B = int(time[0]), x.shape[0]
            src = None
            if mode == 'store':
                for r in range(row0, row0 + B):
                    self.stored[id(cache), r] = t
            elif mode == 'read':
                srcs = {self.stored.get((id(cache), r)) for r in range(row0, row0 + B)}
                assert len(srcs) == 1, srcs
                src = srcs.pop()
            self.passes.append((id(unet), mode, row0, B, t, src))
            return orig(unet, x, time, *a, deepcache=deepcache, **k)
        monkeypatch.setattr(Unet, "_forward_dev", spy)


def _expected(passes, b, N):
    """Group one stage's passes into iterations (a pass at row 0 starts one) and check them against the plan."""
    from minimagen_b200.Imagen import deepcache_plan
    its = []
    for p in passes:
        if p[2] == 0:
            its.append([])
        its[-1].append(p)
    on = [any(p[3] == 2 * b or p[2] == b for p in it) for it in its]
    full = deepcache_plan(on, N)
    j = None
    for i, (it, f) in enumerate(zip(its, full)):
        assert {p[1] for p in it} == {'store' if f else 'read'}, (i, it, full)
        rows = sorted((p[2], p[3]) for p in it)
        assert rows in ([(0, b)], [(0, b), (b, b)], [(0, 2 * b)]), rows
        if f:
            j = it[0][4]
        else:
            assert all(p[5] == j for p in it), (i, it, j)        # reads what the same passes stored at the last full one
    return on, full


def _stages(passes):
    out = {}
    for p in passes:
        out.setdefault(p[0], []).append(p)
    return list(out.values())


@pytest.mark.parametrize("case", ["unbatched", "batched", "interval", "repaint", "dpmpp_2m"])
def test_sample_passes_follow_the_plan(emu, monkeypatch, case):
    g = load_golden("cascade_tiny.pt")
    im, _ = _cascade_from_golden(g, "cpu")
    im.noise_fn, im.use_cuda_graph = None, False
    b = 2
    kw = dict(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=3., seed=[3, 4],
              sampling_timesteps=(7, 6), cache_interval=(3, 2))
    if case == "batched":
        im.cfg_batched = True
    if case == "interval":
        kw.update(guidance_interval=(None, (0.3, 2.)), cond_scale=(3., 2.), cache_interval=3,
                  init_images=(None, torch.rand(b, 3, 16, 16)), skip_steps=(0, 1))
    if case == "repaint":
        mask = torch.zeros(b, 32, 32, dtype=torch.bool)
        mask[:, :, :12] = True
        kw.update(inpaint_images=torch.rand(b, 3, 32, 32), inpaint_masks=mask, inpaint_resample_times=2,
                  guidance_interval=((0.5, float("inf")), None))
    if case == "dpmpp_2m":
        kw.update(sampler="dpmpp_2m")
    spy = PassSpy(monkeypatch)
    out = im.sample(**kw)
    assert torch.isfinite(out).all()
    stages = _stages(spy.passes)
    assert len(stages) == 2
    N = (3, 3) if case == "interval" else (3, 2)
    walks = (7 if case != "repaint" else (7 - 1) * 2 + 1, 6 - (case == "interval") if case != "repaint" else 11)
    for stage, n, walk in zip(stages, N, walks):
        on, full = _expected(stage, b, n)
        print(f"{case}: guided {''.join('G' if v else '.' for v in on)}  full {''.join('F' if v else 'c' for v in full)}")
        assert len(full) == walk and not all(full)
    if case == "interval":
        on, _ = _expected(stages[1], b, 3)
        assert any(on) and not all(on)
    if case == "repaint":
        on, _ = _expected(stages[0], b, 3)
        assert any(on) and not all(on)


def test_noise_draws_do_not_depend_on_caching(emu):
    g = load_golden("cascade_tiny.pt")
    seqs = []
    for ci in (None, 3):
        im, _ = _cascade_from_golden(g, "cpu")
        im.use_cuda_graph = False
        calls, gen = [], torch.Generator().manual_seed(5)

        def noise_fn(kind, shape, step):
            calls.append((kind, tuple(shape), step))
            return torch.randn(shape, generator=gen)
        im.noise_fn = noise_fn
        im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=3., sampling_timesteps=(5, 4),
                  cache_interval=ci)
        seqs.append(calls)
    assert seqs[0] == seqs[1] and len(seqs[0]) > 0


# ------------------------------------------------------------------------------------------------ every call checked
@pytest.mark.parametrize("flavour,cfg_batched", [("ddim", False), ("ddim", True), ("dpmpp_2m", False)])
def test_emulated_cached_cascade_passes_every_call_check(emu, flavour, cfg_batched):
    import minimagen_b200.ops as ops_mod
    g = load_golden("cascade_tiny.pt")
    im, _ = _cascade_from_golden(g, "cpu")
    kw = cascade_case(im, flavour, 2, ((32, 48), (64, 96)), g["text_embeds"].shape[-1], "cpu", cfg_batched)
    proxy = CheckingOps(emu, sms=SMS)
    ops_mod.set_ops(proxy)
    out = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cache_interval=2, **kw)
    print(f"\n{flavour} cascade, cfg_batched={cfg_batched}, cache_interval=2 (emulated)")
    proxy.report()
    assert out.shape == (2, 3, 64, 96) and torch.isfinite(out).all()
    unchecked = proxy.called - proxy.checked - ALLOWED
    assert not unchecked, f"kernels that ran without a float64 check: {sorted(unchecked)}"
    assert {"step_epilogue_rescaled", "randn_keyed"} <= reached(proxy)
