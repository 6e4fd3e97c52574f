"""DeepCache feature reuse (`Imagen.sample(..., cache_interval=N)`) on the GPU:

  * caching off (None or 1) is the sample without the argument: the same bits and the same graph keys;
  * a read pass after a store at the same inputs returns the store pass's output bit for bit (tiny base and SR U-Nets,
    a Super-shaped U-Net at 256 x 256, a cfg_batched 2B pass), and the store pass is the plain forward;
  * the captured loop equals the eager loop bit for bit at N = 3 on the tiny golden cascade across the sampling features
    (DDPM with injected noise, DDIM at eta 0.5 with RePaint, seeds, per-image weights, a negative prompt, schedules and an
    interval, v-prediction with rescale, img2img; the same on DPM-Solver++(2M); cfg_batched; a partial cascade), and the
    replayed (guided, full) sequence is the plan's;
  * the kernel calls recorded while the cached graph is captured are the read pass's: fewer convolutions than the full
    graph's;
  * every kernel call checked against float64: an eager two-stage tiny cascade at cache_interval = 2, and the guided cfg-3
    loop at 256 x 256 with b = 32 over two steps, the second cached;
  * `noise_fn` sees the same (kind, shape, label) sequence with and without caching.
"""
import collections
import time

import pytest
import torch

from checking_ops import ALLOWED, CheckingOps
from conftest import load_golden, rel_l2
from test_host_logic import _cascade_from_golden
from test_respaced import _tiny_imagen
from test_sampling_feature_calls import cascade_case

pytestmark = pytest.mark.gpu


def _cascade():
    g = load_golden("cascade_tiny.pt")
    im, _ = _cascade_from_golden(g, "cuda")
    im.noise_fn = None
    return im, g


# ------------------------------------------------------------------------------------------------ off is off
def test_off_is_the_sample_without_the_argument(native):
    g = load_golden("sample_loop.pt")
    kw = dict(text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda(), cond_scale=3., seed=[4, 9],
              sampling_timesteps=8)
    im = _tiny_imagen(g, 1000, "cuda")
    outs, keys = [], []
    for extra in ({}, dict(cache_interval=None), dict(cache_interval=1), dict(cache_interval=[1])):
        outs.append(im.sample(**kw, **extra))
        keys.append(list(im._graphs))
    assert all(torch.equal(o, outs[0]) for o in outs) and all(k == keys[0] for k in keys)
    assert len(keys[0]) == 1 and 'deepcache' not in keys[0][0]


# ------------------------------------------------------------------------------------------------ read after store
def _net(name):
    from minimagen_b200.Unet import Super, Unet
    g = load_golden("cascade_tiny.pt")
    torch.manual_seed(0)
    if name == "tiny_base":
        u, s, E = Unet(**g["cfgs"][0]), 16, 512
        u.load_state_dict(g["state_dicts"][0])
    elif name == "tiny_sr":
        u, s, E = Unet(**dict(g["cfgs"][1], lowres_cond=True)), 32, 512
    else:
        u, s, E = Unet(**dict(Super.defaults, lowres_cond=True, text_embed_dim=768)), 256, 768
    return u.eval().cuda(), s, E


@pytest.mark.parametrize("name,batched", [("tiny_base", False), ("tiny_sr", False), ("super_256", False),
                                          ("super_256", True)])
def test_read_after_store_is_the_full_pass(native, name, batched):
    from minimagen_b200.Unet import DeepCache
    u, s, E = _net(name)
    b = 2
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(b, 3, s, s, generator=gen).cuda()
    t = torch.tensor([700, 30]).cuda()
    kw = dict(text_embeds=torch.randn(b, 12, E, generator=gen).cuda(), text_mask=torch.ones(b, 12, dtype=torch.bool).cuda())
    kw["text_mask"][1, 7:] = False
    if u.lowres_cond:
        kw.update(lowres_cond_img=torch.randn(b, 3, s, s, generator=gen).cuda(), lowres_noise_times=torch.tensor([5, 90]).cuda())
    if batched:      # the cfg_batched pass: conditional and null rows in one 2B batch
        two = lambda v: torch.cat((v, v))
        x, t, kw = two(x), two(t), {k: two(v) for k, v in kw.items()}
        kw["cond_keep"] = torch.cat((torch.ones(b, dtype=torch.uint8), torch.zeros(b, dtype=torch.uint8))).cuda()
        b *= 2
    cache = DeepCache(2 * b)
    with torch.no_grad():
        plain = u._forward_impl(x, t, **kw)
        store = u._forward_impl(x, t, deepcache=('store', cache, b), **kw)
        read = u._forward_impl(x, t, deepcache=('read', cache, b), **kw)
        other = u._forward_impl(x * 0.5, t // 2, deepcache=('read', cache, b), **kw)
    torch.cuda.synchronize()
    print(f"{name} b = {b}: store vs plain {rel_l2(store, plain):.3e}, read vs store {rel_l2(read, store):.3e}, "
          f"read at other (x, t) vs store {rel_l2(other, store):.3e}")
    assert torch.equal(store, plain) and torch.equal(read, store)
    assert torch.isfinite(other).all() and not torch.equal(other, store)


# ------------------------------------------------------------------------------------------------ captured vs eager
def _case(im, g, case):
    D = g["text_embeds"].shape[-1]
    kw = dict(text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda())
    if case in ("ddim", "dpmpp_2m", "ddim_batched"):
        kw.update(cascade_case(im, "dpmpp_2m" if case == "dpmpp_2m" else "ddim", 2, ((16, 24), (32, 48)), D, "cuda",
                               case == "ddim_batched"))
        kw["sampling_timesteps"] = (7, 6)
    elif case == "ddpm_noise_fn":
        im.noise_fn = _bank_any(3)
        kw.update(cond_scale=3.)
    elif case == "partial":
        gen = torch.Generator().manual_seed(5)
        kw.update(cond_scale=(3., torch.tensor([2., 4.]).cuda()), start_at_unet_number=2, seed=7,
                  start_images=torch.rand(2, 3, 16, 16, generator=gen).cuda(), sampling_timesteps=(None, 9),
                  ddim_eta=1.)
    return kw


def _bank_any(seed):
    """noise_fn over a seeded bank: one tensor per (kind, shape, label)."""
    gen, bank = torch.Generator().manual_seed(seed), {}

    def noise_fn(kind, shape, step):
        key = (kind, tuple(shape), step)
        if key not in bank:
            bank[key] = torch.randn(shape, generator=gen)
        return bank[key]
    return noise_fn


class _Spy:
    """Per stage: the eager loop's (guided, full) per iteration (Imagen._step), the captured loop's replays."""

    def __init__(self, monkeypatch):
        from minimagen_b200.Imagen import Imagen, _StepGraph
        self.steps, self.replays = collections.defaultdict(list), collections.defaultdict(list)
        step, replay = Imagen._step, _StepGraph.replay

        def spy_step(im, unet, *a, guided=None, deepcache=None, **k):
            self.steps[id(unet)].append((guided, deepcache is None or deepcache[0] == 'store'))
            return step(im, unet, *a, guided=guided, deepcache=deepcache, **k)

        def spy_replay(g, guided=True, full=True):
            self.replays[id(g.unet)].append((guided, full))
            return replay(g, guided, full)
        monkeypatch.setattr(Imagen, "_step", spy_step)
        monkeypatch.setattr(_StepGraph, "replay", spy_replay)


@pytest.mark.parametrize("case", ["ddpm_noise_fn", "ddim", "ddim_batched", "dpmpp_2m", "partial"])
def test_captured_loop_is_the_eager_loop(native, monkeypatch, case):
    from minimagen_b200.Imagen import deepcache_plan
    outs, spies = {}, {}
    for graph in (False, True):
        im, g = _cascade()
        kw = _case(im, g, case)
        im.use_cuda_graph = graph
        spies[graph] = spy = _Spy(monkeypatch)
        outs[graph] = im.sample(cache_interval=3, **kw)
        monkeypatch.undo()
        if graph:
            assert im._graphs and all('deepcache' in k for k in im._graphs)
            assert len(im._graphs) <= im.max_cached_graphs
            entries = list(im._graphs.values())
    print(f"{case}: captured vs eager rel-L2 {rel_l2(outs[True], outs[False]):.3e}")
    assert torch.equal(outs[True], outs[False])
    eager, captured = list(spies[False].steps.values()), list(spies[True].replays.values())
    assert len(eager) == len(captured) >= 1
    for steps, replays in zip(eager, captured):
        on, full = [s[0] for s in steps], [s[1] for s in steps]
        assert full == deepcache_plan(on, 3) and not all(full)
        assert [r[1] for r in replays] == full
        print(f"  guided {''.join('G' if v else '.' for v in on)}  full {''.join('F' if v else 'c' for v in full)}")
    assert any(e.graph_cached is not None or e.graph_cached_unguided is not None for e in entries)


def test_one_entry_serves_every_interval(native):
    im, g = _cascade()
    kw = dict(text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda(), cond_scale=3., seed=[1, 2],
              sampling_timesteps=(8, 6))
    outs = {}
    for n in (2, 3, 5):
        outs[n] = im.sample(cache_interval=n, **kw)
        graphs = [(e.graph, e.graph_cached) for e in im._graphs.values()]
        if n == 2:
            first = graphs
        assert graphs == first and len(im._graphs) == 2
    im.clear_graphs()
    assert not im._graphs
    fresh, _ = _cascade()
    assert torch.equal(fresh.sample(cache_interval=5, **kw), outs[5])


# ------------------------------------------------------------------------------------------------ what a cached graph runs
class _Recorder:
    def __init__(self, inner):
        self.inner, self.log = inner, None

    def __getattr__(self, name):
        f = getattr(self.inner, name)
        if not callable(f):
            return f

        def call(*a, **k):
            if self.log is not None:
                self.log.append(name)
            return f(*a, **k)
        return call


def test_cached_graph_runs_the_read_pass(native, monkeypatch):
    """The calls recorded while each graph of the entry is captured: the cached graph's are those of the store graph with
    the deep levels' launches removed -- fewer convolutions, the same step epilogue and draws."""
    import minimagen_b200.ops as ops_mod
    from minimagen_b200.Imagen import Imagen
    rec = _Recorder(native)
    ops_mod.set_ops(rec)
    logs = []
    orig = Imagen._capture

    def capture(body, device, pool=None):
        def recorded():
            rec.log = []
            body()
            logs.append(rec.log)
            rec.log = None
        return orig(recorded, device, pool)
    monkeypatch.setattr(Imagen, "_capture", staticmethod(capture))
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000, "cuda")
    im.sample(text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda(), cond_scale=3., seed=[1, 2],
              sampling_timesteps=8, cache_interval=3)
    assert len(logs) == 4                                   # warm-up + capture, store graph then read graph
    store, read = logs[1], logs[3]
    convs = lambda log: sum(1 for n in log if n.startswith("conv"))
    cs, cr = collections.Counter(store), collections.Counter(read)
    print(f"store graph: {len(store)} calls, {convs(store)} conv; read graph: {len(read)} calls, {convs(read)} conv")
    assert convs(read) < convs(store)
    for n in ("step_epilogue", "randn_keyed", "step_advance_t_table"):
        assert cs[n] == cr[n] == 1
    # the read pass per U-Net pass: what a direct read pass on the same shapes launches
    from minimagen_b200.Unet import DeepCache
    u = im.unets[0]
    x = torch.randn(2, 3, 64, 64, device="cuda")
    cache = DeepCache(2)
    rec.log = []
    with torch.no_grad():
        u._forward_impl(x, torch.tensor([5, 5]).cuda(), deepcache=('store', cache, 0), text_embeds=g["text_embeds"].cuda(),
                        text_mask=g["text_mask"].cuda())
        full_pass, rec.log = rec.log, []
        u._forward_impl(x, torch.tensor([5, 5]).cuda(), deepcache=('read', cache, 0), text_embeds=g["text_embeds"].cuda(),
                        text_mask=g["text_mask"].cuda())
        read_pass, rec.log = rec.log, None
    # two U-Net passes per guided step: the graphs save twice the per-pass difference
    assert convs(store) - convs(read) == 2 * (convs(full_pass) - convs(read_pass)) > 0


# ------------------------------------------------------------------------------------------------ every call checked
def _checked(native, fn):
    import minimagen_b200.ops as ops_mod
    proxy = CheckingOps(native)
    ops_mod.set_ops(proxy)                              # the `native` fixture restores the previous backend afterwards
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    print(f"\n{time.perf_counter() - t0:.1f} s, peak memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    proxy.report()
    assert torch.isfinite(out).all()
    unchecked = proxy.called - proxy.checked - ALLOWED
    assert not unchecked, f"kernels that ran without a float64 check: {sorted(unchecked)}"
    return proxy, out


def test_every_call_of_a_cached_tiny_cascade(native):
    im, g = _cascade()
    kw = _case(im, g, "ddim")
    im.use_cuda_graph = False
    proxy, out = _checked(native, lambda: im.sample(cache_interval=2, **kw))
    assert {"step_epilogue_rescaled", "inpaint_prologue", "randn_keyed"} <= proxy.checked


def test_every_call_of_a_cached_cfg3_step_at_benchmark_size(native):
    """The flagship U-Net (`Unet(**Super.defaults, lowres_cond=True, text_embed_dim=768)`) as the second stage, 64 -> 256
    px at b = 32, w = 3, two eager DDIM steps at cache_interval = 2: the first stores, the second reads."""
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import BaseTest, Super, Unet
    torch.manual_seed(0)
    b = 32
    u = Unet(**dict(Super.defaults, lowres_cond=True, text_embed_dim=768)).eval()
    first = Unet(**dict(BaseTest.defaults, text_embed_dim=768)).eval()
    im = Imagen(unets=(first, u), text_encoder_name="t5_base", image_sizes=(64, 256), timesteps=1000,
                cond_drop_prob=0.1).eval().cuda()
    im.use_cuda_graph = False
    gen = torch.Generator().manual_seed(11)
    te = torch.randn(b, 20, 768, generator=gen).cuda()
    tm = torch.ones(b, 20, dtype=torch.bool)
    tm[-1, 5:] = False
    start = torch.rand(b, 3, 64, 64, generator=gen).cuda()
    modes = []
    orig = u._forward_dev

    def spy(*a, deepcache=None, **k):
        modes.append(deepcache[0])
        return orig(*a, deepcache=deepcache, **k)
    u._forward_dev = spy
    proxy, out = _checked(native, lambda: im.sample(text_embeds=te, text_masks=tm.cuda(), cond_scale=3.,
                                                    sampling_timesteps=2, start_at_unet_number=2, start_images=start,
                                                    cache_interval=2))
    assert modes == ['store', 'store', 'read', 'read']
    assert tuple(out.shape) == (b, 3, 256, 256)
    assert {"conv_igemm", "gn_apply_silu", "attention", "step_epilogue"} <= proxy.checked


# ------------------------------------------------------------------------------------------------ draws
def test_noise_fn_sees_the_same_draws(native):
    seqs = []
    for ci in (None, 3):
        im, g = _cascade()
        calls, gen = [], torch.Generator().manual_seed(5)

        def noise_fn(kind, shape, step):
            calls.append((kind, tuple(shape), step))
            return torch.randn(shape, generator=gen)
        im.noise_fn = noise_fn
        im.sample(text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda(), cond_scale=3.,
                  sampling_timesteps=(6, 5), cache_interval=ci)
        seqs.append(calls)
    assert seqs[0] == seqs[1] and len(seqs[0]) > 0
