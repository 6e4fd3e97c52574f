"""Guidance intervals and guidance-weight schedules (Imagen.sample(guidance_interval=, guidance_schedule=)) on the CPU,
through the torch emulation of the ops interface extended by the scheduled step epilogues (mi_step_epilogue_ws /
mi_step_epilogue_multistep_ws).  Covers the table against the restatement (guidance_interval_restatement.py), the loop
against the restated loop for DDPM, DDIM and DPM-Solver++(2M), the three identities (a table of ones is the loop without
it, a table of zeros the cond_scale = 1 loop, unguided stages ignore it), the U-Net evaluation count, the draws, the
batched guidance pass, inpainting, skip_steps, per-U-Net tuples, the argument checks, the graph keys and two gloo ranks.
(The kernels and the captured graph pair are covered on the GPU in test_gpu_guidance_interval.py.)"""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import guidance_interval_restatement as G
from conftest import load_golden, rel_l2
from emu_ops import EmuOps
from test_guidance import _count_forwards, _negative
from test_respaced import _bank, _tiny_imagen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = torch.float32
SHAPE = (2, 3, 64, 64)
INF = float("inf")


def _walk(sch, sampler, steps, eta=0.):
    if sampler == "ddpm":
        return None
    if sampler == "dpmpp_2m":
        return sch.dpm_solver_schedule(steps, "cpu")
    return sch.sampling_schedule(steps, eta, "cpu")


def _loop(im, g, sampler="ddim", steps=8, eta=0.5, cond_scale=3., interval=None, schedule=None, nte=None, ntm=None,
          seed=7, inpaint=None):
    """_p_sample_loop on the tiny U-Net with the stage table of (interval, schedule) (none when both are None)."""
    im.use_cuda_graph = False
    im.noise_fn = _bank(seed)
    sch = im.noise_schedulers[0]
    tab = None if interval is None and schedule is None else sch.guidance_table(interval, schedule, "cpu")
    out = im._p_sample_loop(im.unets[0], SHAPE, noise_scheduler=sch, text_embeds=g["text_embeds"],
                            text_mask=g["text_mask"], cond_scale=cond_scale, schedule=_walk(sch, sampler, steps, eta),
                            negative_text_embeds=nte, negative_text_mask=ntm, guidance_table=tab, inpaint=inpaint)
    return out, im.noise_fn.calls


# ------------------------------------------------------------------------------------------------ the table
@pytest.mark.parametrize("T", [20, 25, 1000])
@pytest.mark.parametrize("interval", [None, (0.3, 5.), (0., INF), (2., INF), (0.5, 0.6)])
@pytest.mark.parametrize("schedule", [None, "linear", "cosine"])
def test_table_is_the_restatement(T, interval, schedule):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    gd = GaussianDiffusion(timesteps=T)
    tab = gd.guidance_table(interval, schedule, "cpu")
    assert tab.dtype == F32 and tab.shape == (T,)
    assert tab.tolist() == G.table(T, interval, schedule)
    assert gd.guidance_table(interval, schedule, "cpu") is tab                       # cached
    if schedule is not None:
        assert tab[T - 1] == 0                                                       # the ramps end at 0
    if T == 20 and interval is not None:
        assert (tab[T - 1] != 0) == (interval[1] == INF and schedule is None)        # sigma = inf at T = 20's last t


def test_ramps_average_one():
    T = 100000
    for schedule in ("linear", "cosine"):
        s = G.table(T, None, schedule)
        assert abs(sum(s) / T - 1.) < 1e-4
    assert G.weights([3., 1., 0.3], 1.) == [3., 1., 0.3]
    assert G.weights([3., 1.], 0.) == [1., 1.]


# ------------------------------------------------------------------------------------------------ against the restatement
LOOPS = [("ddpm", 25, None, 0., (0.5, 10.)), ("ddim", 1000, 8, 0.5, (0.4, 20.)), ("dpmpp_2m", 1000, 6, 0., (0.4, 20.))]


@pytest.mark.parametrize("sampler,T,steps,eta,interval", LOOPS, ids=[c[0] for c in LOOPS])
@pytest.mark.parametrize("schedule", [None, "linear", "cosine"])
def test_emulated_loop_vs_restatement(emu, sampler, T, steps, eta, interval, schedule):
    """Interval and schedule with a negative prompt and per-image weights (2, 4.5), against the restated loop over the
    restated U-Net; the U-Net runs S + k times for k guided points, the scheduled epilogue k times."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, T)
    nte, ntm = _negative()
    w = torch.tensor([2., 4.5])
    calls = _count_forwards(im.unets[0])
    out, _ = _loop(im, g, sampler, steps, eta, w, interval, schedule, nte, ntm)
    ref, guided = G.interval_loop(g["state_dict"], g["cfg"], SHAPE, T, _bank(7), [2., 4.5], interval=interval,
                                  schedule=schedule, sampler=sampler, steps=steps, eta=eta, text_embeds=g["text_embeds"],
                                  text_mask=g["text_mask"], negative_text_embeds=nte, negative_text_mask=ntm)
    S = T if steps is None else steps
    err = rel_l2(out, ref)
    print(f"{sampler} {schedule}: {len(guided)} of {S} points guided, rel-L2 vs restated loop = {err:.3e}")
    assert err < 1e-3
    assert 0 < len(guided) < S
    assert len(calls) == S + len(guided)
    step = "step_epilogue_multistep" if sampler == "dpmpp_2m" else "step_epilogue"
    assert emu.calls.count(step + "_scheduled") == len(guided)
    assert emu.calls.count(step) == S - len(guided)


# ------------------------------------------------------------------------------------------------ identities
@pytest.mark.parametrize("sampler", ["ddpm", "ddim", "dpmpp_2m"])
def test_ones_table_is_the_loop_without_it(emu, sampler):
    """A covering interval (no schedule) is bit for bit the loop without arguments, through the same entry points."""
    g = load_golden("sample_loop.pt")
    nte, ntm = _negative()
    outs, logs = [], []
    for interval in (None, (0., INF)):
        im = _tiny_imagen(g, 25)
        del emu.calls[:]
        outs.append(_loop(im, g, sampler, 6, 0.5, torch.tensor([2., 4.5]), interval, None, nte, ntm)[0])
        logs.append(list(emu.calls))
    assert torch.equal(outs[0], outs[1]) and logs[0] == logs[1]
    assert not any(c.endswith("_scheduled") for c in logs[1])


def test_skipped_points_do_not_count(emu):
    """A table that is 1 on the points a shortened walk visits (and 0 at the first one it skips) runs the loop without
    it, the same entry points and bits; so does one that is 1 at every point but not on all timesteps."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    sch = im.noise_schedulers[0]
    walk = sch.sampling_schedule(8, 0.5, "cpu")
    short = walk._replace(grid=walk.grid[2:])
    sig = G.sigmas(1000)
    interval = (0., sig[walk.grid[2]])                              # excludes grid[0] and grid[1] only
    tab = sch.guidance_table(interval, None, "cpu")
    assert tab[walk.grid[1]] == 0 and all(tab[t] == 1 for t in short.grid)
    outs, logs = [], []
    init = torch.rand(SHAPE, generator=torch.Generator().manual_seed(3)) * 2 - 1
    for table in (None, tab):
        im.noise_fn = _bank(7)
        del emu.calls[:]
        outs.append(im._p_sample_loop(im.unets[0], SHAPE, noise_scheduler=sch, text_embeds=g["text_embeds"],
                                      text_mask=g["text_mask"], cond_scale=3., schedule=short, init_image=init,
                                      guidance_table=table))
        logs.append([c for c in emu.calls if c.startswith("step")])     # (the first run also packs the weights)
    assert torch.equal(outs[0], outs[1]) and logs[0] == logs[1]


@pytest.mark.parametrize("sampler", ["ddim", "dpmpp_2m"])
def test_zeros_table_is_the_unguided_loop(emu, sampler):
    """An interval that holds no point of the walk runs the cond_scale = 1 loop bit for bit, one U-Net pass per point,
    and never conditions on the negative prompt."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    nte, ntm = _negative()
    calls = _count_forwards(im.unets[0])
    one, _ = _loop(im, g, sampler, 6, 0.5, 1.)
    del calls[:]
    empty, _ = _loop(im, g, sampler, 6, 0.5, torch.tensor([2., 4.5]), (1000., 2000.), "linear", nte, ntm)
    assert torch.equal(one, empty)
    assert len(calls) == 6 and all(kw.get("text_embeds") is g["text_embeds"] for kw in calls)


def test_unguided_stage_ignores_the_table(emu):
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    calls = _count_forwards(im.unets[0])
    a, _ = _loop(im, g, "ddim", 6, 0.5, 1.)
    b, _ = _loop(im, g, "ddim", 6, 0.5, torch.ones(2), (0.4, 20.), "cosine")
    assert torch.equal(a, b) and len(calls) == 12
    assert "step_epilogue_scheduled" not in emu.calls


def test_draws_do_not_change(emu):
    """The same noise_fn calls, in the same order, with and without an interval and a schedule (DDIM eta > 0, RePaint)."""
    g = load_golden("sample_loop.pt")
    gen = torch.Generator().manual_seed(2)
    mask = torch.zeros(2, 64, 64, dtype=torch.bool)
    mask[:, 16:48, 8:40] = True
    inpaint = ((torch.rand(SHAPE, generator=gen) * 2 - 1), mask.float().reshape(2, -1), 2)
    for inp in (None, inpaint):
        seqs = []
        for interval, schedule in ((None, None), ((0.4, 20.), "linear")):
            im = _tiny_imagen(g, 1000)
            seqs.append(_loop(im, g, "ddim", 6, 0.5, 3., interval, schedule, inpaint=inp)[1])
        assert seqs[0] == seqs[1] and len(seqs[0]) > 6


def test_inpainting_iterations_follow_their_t(emu):
    """RePaint with R = 2: each iteration (t, r) runs the guidance pass iff t is guided; a covering interval is the loop
    without it."""
    g = load_golden("sample_loop.pt")
    gen = torch.Generator().manual_seed(2)
    mask = torch.zeros(2, 64, 64, dtype=torch.bool)
    mask[:, 16:48, 8:40] = True
    inpaint = ((torch.rand(SHAPE, generator=gen) * 2 - 1), mask.float().reshape(2, -1), 2)
    im = _tiny_imagen(g, 1000)
    sch = im.noise_schedulers[0]
    grid = list(sch.sampling_schedule(6, 0.5, "cpu").grid)
    tab = G.table(1000, (0.4, 20.), "cosine")
    calls = _count_forwards(im.unets[0])
    out, _ = _loop(im, g, "ddim", 6, 0.5, 3., (0.4, 20.), "cosine", inpaint=inpaint)
    iters = [t for t in grid for _ in range(2 if t > 0 else 1)]
    want = []
    for t in iters:
        want += [0.] + ([1.] if tab[t] != 0 else [])
    assert [kw.get("cond_drop_prob", 0.) for kw in calls] == want
    plain, _ = _loop(im, g, "ddim", 6, 0.5, 3., inpaint=inpaint)
    cover, _ = _loop(im, g, "ddim", 6, 0.5, 3., (0., INF), None, inpaint=inpaint)
    assert torch.equal(plain, cover) and rel_l2(out, plain) > 1e-3


def test_cfg_batched(emu):
    """cfg_batched runs the guidance pass in the 2B batch at the guided points only, and matches the unbatched loop."""
    g = load_golden("sample_loop.pt")
    nte, ntm = _negative(L=9)
    outs, batched = [], []
    for cfg_batched in (False, True):
        im = _tiny_imagen(g, 1000)
        im.cfg_batched = cfg_batched
        fwd = im.unets[0]._forward_impl
        im.unets[0]._forward_impl = lambda *a, **kw: batched.append(a[0].shape[0]) or fwd(*a, **kw)
        outs.append(_loop(im, g, "ddim", 8, 0., torch.tensor([3., 2.]), (0.4, 20.), "linear", nte, ntm)[0])
    err = rel_l2(outs[1], outs[0])
    print(f"batched vs unbatched rel-L2 = {err:.3e}")
    assert err < 1e-4
    k = len(G.guided_points(G.D.ddim_grid(1000, 8), G.table(1000, (0.4, 20.), "linear")))
    assert 0 < k < 8 and batched.count(4) == k


def test_cascade_per_unet_entries_equal_stage_by_stage(emu):
    """guidance_interval=(None, pair) and guidance_schedule=('linear', None) on the tiny cascade == stage 1 alone with
    'linear', then stage 2 alone with the pair."""
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
    T = im.noise_schedulers[1].num_timesteps
    sig = G.sigmas(T)
    grid = G.D.ddim_grid(T, 4)
    pair = (sig[grid[-2]] - 1e-9, sig[grid[1]])                     # the two middle points of stage 2's walk
    kw = dict(text_embeds=g["text_embeds"], text_masks=g["text_mask"], sampling_timesteps=(5, 4), cond_scale=(2., 4.))
    both = im.sample(guidance_interval=(None, pair), guidance_schedule=("linear", None), **kw)
    first = im.sample(guidance_schedule="linear", stop_at_unet_number=1, **kw)
    second = im.sample(guidance_interval=pair, start_at_unet_number=2, start_images=first, **kw)
    assert torch.equal(both, second)
    assert not torch.equal(im.sample(**kw), both)


def test_argument_checks(emu):
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet, BaseTest, SuperTest
    im = Imagen(unets=(Unet(**BaseTest.defaults), Unet(**SuperTest.defaults)), text_encoder_name="t5_small",
                image_sizes=(16, 32), timesteps=25, cond_drop_prob=0.1)
    te = torch.zeros(2, 4, 512)
    for bad in ((1., 0.5), (0.5, 0.5), (-1., 2.), (INF, INF), (float("nan"), 1.), (0., float("nan"))):
        with pytest.raises(AssertionError, match=r"guidance_interval of unet 1 must have 0 <= sigma_lo < sigma_hi with "
                                                 r"a finite sigma_lo"):
            im.sample(text_embeds=te, guidance_interval=bad)
    with pytest.raises(AssertionError, match=r"guidance_interval of unet 2 must have 0 <= sigma_lo < sigma_hi"):
        im.sample(text_embeds=te, guidance_interval=(None, (3., 2.)))
    for bad in ((1., 2., 3.), ((1., 2.),)):
        with pytest.raises(AssertionError, match=r"guidance_interval must have one entry per unet \(2\)"):
            im.sample(text_embeds=te, guidance_interval=bad)
    for bad in ("wide", (None, (1., 2., 3.)), (None, "x"), (None, (True, 2.))):
        with pytest.raises(AssertionError, match=r"guidance_interval of unet \d must be None or a pair \(sigma_lo, "
                                                 r"sigma_hi\)"):
            im.sample(text_embeds=te, guidance_interval=bad)
    for bad in ("quadratic", 1, (None, "Linear")):
        with pytest.raises(AssertionError, match=r"guidance_schedule of unet \d must be None, 'linear' or 'cosine'"):
            im.sample(text_embeds=te, guidance_schedule=bad)
    with pytest.raises(AssertionError, match=r"guidance_schedule must have one entry per unet \(2\), got 3"):
        im.sample(text_embeds=te, guidance_schedule=("linear",) * 3)


# ------------------------------------------------------------------------------------------------ graph keys
def test_graph_keys():
    """A guidance-table pair is keyed apart, with a 'guidance_table' suffix, and serves every table; without a table, or
    unguided, the key is unchanged."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 25)
    sch = im.noise_schedulers[0]
    key = lambda w, *a, **kw: im._graph_key(im.unets[0], SHAPE, sch, g["text_embeds"], g["text_mask"], None, None, w,
                                            *a, **kw)
    assert key(3., scheduled=True) == key(3.) + ("guidance_table",)
    assert key(3., True, scheduled=True) == key(3., True)[:-1] + ("guidance_table", "inpaint")
    assert key(3., False, True, scheduled=True)[-2:] == ("guidance_table", "multistep")

    class Cached:
        def __init__(self):
            self.tables = []
            self.graph_unguided = "captured"

        def set_cond(self, **cond):
            pass

        def set_schedule(self, sched):
            pass

        def set_guidance(self, table):
            self.tables.append(table)

    plain, pair = Cached(), Cached()
    im._graphs = {key(3.): plain, key(3., scheduled=True): pair}
    kw = dict(noise_scheduler=sch, text_embeds=g["text_embeds"], text_mask=g["text_mask"], lowres_cond_img=None,
              lowres_noise_times=None)
    t1, t2 = sch.guidance_table((0.5, 10.), None, "cpu"), sch.guidance_table(None, "cosine", "cpu")
    assert im._step_graph(im.unets[0], SHAPE, cond_scale=3., **kw) is plain
    assert im._step_graph(im.unets[0], SHAPE, cond_scale=5., guidance_table=t1, unguided=True, **kw) is pair
    assert im._step_graph(im.unets[0], SHAPE, cond_scale=torch.tensor([2., 3.]), guidance_table=t2, **kw) is pair
    assert pair.tables == [t1, t2] and plain.tables == [] and len(im._graphs) == 2


# ------------------------------------------------------------------------------------------------ two gloo ranks
def _dist_inputs(B):
    gen = torch.Generator().manual_seed(7)
    te = torch.randn(B, 9, 512, generator=gen)
    tm = torch.ones(B, 9, dtype=torch.bool)
    tm[1, 4:] = False
    return dict(text_embeds=te, text_masks=tm, cond_scale=torch.tensor([1., 2., 3.5, 5.]), sampling_timesteps=5,
                guidance_interval=(0.5, 10.), guidance_schedule="linear")


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
def test_two_rank_gloo(tmp_path, emu):
    from test_distributed_cpu import _build, _noise_bank
    port = 29600 + (os.getpid() % 200)
    out_path = str(tmp_path / "dist_out.pt")
    mp.spawn(_worker, args=(2, port, out_path), nprocs=2, join=True)
    dist_out = torch.load(out_path)
    g = load_golden("sample_loop.pt")
    im = _build(g)
    bank = _noise_bank(4)
    im.noise_fn = lambda kind, shape, step: bank[(kind, step)]
    full = im.sample(**_dist_inputs(4))
    err = rel_l2(dist_out, full)
    print(f"two ranks vs one process: rel-L2 = {err:.3e}")
    tab = G.table(25, (0.5, 10.), "linear")
    assert 0 < len(G.guided_points(G.D.ddim_grid(25, 5), tab)) < 5
    assert err < 2e-4
