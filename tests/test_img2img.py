"""Image-to-image sampling and partial cascades (Imagen.sample(init_images=, skip_steps=, start_at_unet_number=,
start_images=, stop_at_unet_number=)) on the CPU, through the torch emulation of the ops interface.  Covers the 2M
schedule's first-order restart, the emulated sampler against the SDEdit restatement (img2img_restatement.py) on the tiny
golden U-Net and the tiny cascade, convergence on the analytic denoiser from a noised init image, cascade entry and exit
bit for bit, the defaults, the argument checks and two gloo ranks.  (The captured graph and the native path are covered on
the GPU in test_gpu_img2img.py.)"""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import ddim_restatement as D
import img2img_restatement as S
from conftest import load_golden, rel_l2
from test_dpmpp import MU, SD, SHAPE, AnalyticEps
from test_respaced import _bank, _tiny_imagen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def init_image(seed, shape=SHAPE):
    """An init image in [0, 1]."""
    return torch.rand(shape, generator=torch.Generator().manual_seed(seed))


def shape_bank(seed):
    """noise_fn over a seeded bank keyed by (kind, step, shape), for cascades whose stages draw at several sizes."""
    gen = torch.Generator().manual_seed(seed)
    bank, calls = {}, []

    def noise_fn(kind, shape, step):
        key = (kind, step, tuple(shape))
        calls.append(key)
        if key not in bank:
            bank[key] = torch.randn(shape, generator=gen)
        return bank[key]
    noise_fn.calls = calls
    return noise_fn


def cascade(device="cpu"):
    from test_host_logic import _cascade_from_golden
    g = load_golden("cascade_tiny.pt")
    im, _ = _cascade_from_golden(g, device)
    return im, g


def spy_stages(im):
    """Record each stage's _p_sample_loop keyword arguments and output."""
    loop, seen = im._p_sample_loop, []

    def spy(*a, **kw):
        out = loop(*a, **kw)
        seen.append((kw, out.detach().cpu().clone()))
        return out
    im._p_sample_loop = spy
    return seen


# ------------------------------------------------------------------------------------------------ 2M schedule
@pytest.mark.parametrize("T,S_", [(25, 7), (1000, 10), (1000, 50)])
def test_dpm_schedule_skip_restarts_at_first_order(T, S_):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    from test_dpmpp import first_order_walk
    gd = GaussianDiffusion(timesteps=T)
    full = gd.dpm_solver_schedule(S_, "cpu")
    first = first_order_walk(gd, S_, "cpu")
    assert gd.dpm_solver_schedule(S_, "cpu", skip=0) is full
    for k in range(S_):
        sch = gd.dpm_solver_schedule(S_, "cpu", skip=k)
        assert sch.grid == full.grid[k:]
        t0 = full.grid[k]
        assert sch.c3[t0] == 0 and sch.c1[t0] == first.c1[t0]              # first order: c1 = phi, no history term
        others = torch.ones(T, dtype=torch.bool)
        others[t0] = False
        assert torch.equal(sch.c1[others], full.c1[others]) and torch.equal(sch.c3[others], full.c3[others])
        for name in ("c2", "sigma", "next_t"):
            assert torch.equal(getattr(sch, name), getattr(full, name)), name
        assert gd.dpm_solver_schedule(S_, "cpu", skip=k) is sch            # cached per (steps, skip, device)
    with pytest.raises(AssertionError, match=f"skip must be between 0 and {S_ - 1}, got {S_}"):
        gd.dpm_solver_schedule(S_, "cpu", skip=S_)


# ------------------------------------------------------------------------------------------------ emulated sampler
CASES = [(25, None, 0., "ddim", 10), (1000, 8, 0., "ddim", 3), (1000, 8, 0.5, "ddim", 3), (1000, 8, 0., "dpmpp_2m", 3),
         (1000, 8, 0.5, "ddim", 0)]


@pytest.mark.parametrize("T,S_,eta,sampler,skip", CASES)
def test_emulated_sample_vs_restatement(emu, T, S_, eta, sampler, skip):
    """Imagen.sample(init_images=, skip_steps=) on sample_loop.pt's tiny U-Net (CFG w = 3) against the SDEdit
    restatement: DDPM, DDIM (eta 0, 0.5) and 2M; the draws are 'init', then one 'step' per point from grid[skip] on."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, T)
    im.noise_fn = _bank(20 + skip)
    img = init_image(skip)
    out = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=3., sampling_timesteps=S_,
                    ddim_eta=eta, sampler=sampler, init_images=img, skip_steps=skip)
    grid = S.walk(T, S_, sampler)[skip:]
    assert im.noise_fn.calls == [("init", -1)] + [("step", t) for t in grid]
    ref = S.sdedit_loop(g["state_dict"], g["cfg"], SHAPE, T, img * 2 - 1, skip, im.noise_fn, steps=S_, eta=eta,
                        sampler=sampler, text_embeds=g["text_embeds"], text_mask=g["text_mask"])
    err = rel_l2(out, ref)
    print(f"T={T} S={S_} eta={eta} {sampler} skip={skip}: rel-L2 vs restated SDEdit = {err:.3e}")
    assert err < 1e-3


def test_cascade_stages_vs_restatement(emu):
    """The two-stage cascade of cascade_tiny.pt (16 -> 32, CFG w = 2) with one init image at 32x32 for both stages: the
    base stage on DDPM skipping 10 points, the SR stage on 2M (S = 8) skipping 3.  Each stage against the SDEdit
    restatement on the inputs the product gave it (its resized init image and its low-res conditioning)."""
    im, g = cascade()
    im.noise_fn = shape_bank(3)
    seen = spy_stages(im)
    img = init_image(4, (2, 3, 32, 32))
    im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=2., sampling_timesteps=(None, 8),
              sampler="dpmpp_2m", init_images=img, skip_steps=(10, 3))
    assert len(seen) == 2
    assert torch.equal(seen[1][0]["init_image"], img * 2 - 1)             # already at the SR stage's size
    assert seen[0][0]["init_image"].shape == (2, 3, 16, 16)
    for (kw, out), cfg, sd, steps, sampler, skip, size in zip(seen, g["cfgs"], g["state_dicts"], (None, 8),
                                                               ("ddim", "dpmpp_2m"), (10, 3), g["image_sizes"]):
        shape = (2, 3, size, size)
        lowres = {} if kw["lowres_cond_img"] is None else dict(lowres_cond_img=kw["lowres_cond_img"] * 2 - 1,
                                                                 lowres_noise_times=kw["lowres_noise_times"])
        cfg = dict(cfg, lowres_cond=bool(lowres))                        # Imagen makes every U-Net after the first an SR one
        ref = S.sdedit_loop(sd, cfg, shape, 25, kw["init_image"], skip, im.noise_fn, steps=steps, sampler=sampler,
                            cond_scale=2., text_embeds=g["text_embeds"], text_mask=g["text_mask"], **lowres)
        err = rel_l2(out, ref)
        print(f"cascade stage {size}x{size} {sampler} skip={skip}: rel-L2 vs restated SDEdit = {err:.3e}")
        assert err < 1e-3


# ------------------------------------------------------------------------------------------------ analytic convergence
def exact_end_from(x_t0, t0, timesteps):
    """test_dpmpp.exact_end from any start t0: the probability-flow ODE keeps z = (x_t - sqrt(a_t) MU) /
    sqrt(a_t SD^2 + 1 - a_t) fixed, and E[x0 | x_0] = MU + sqrt(a_0) SD^2 / sqrt(a_0 SD^2 + 1 - a_0) z."""
    acp = D.alphas_cumprod_fp64(timesteps)
    a, a0 = acp[t0], acp[0]
    z = (x_t0.double() - a.sqrt() * MU) / (a * SD ** 2 + 1. - a).sqrt()
    return MU + a0.sqrt() * SD ** 2 / (a0 * SD ** 2 + 1. - a0).sqrt() * z


def analytic_img2img_errors(device, steps, graph):
    """rel-L2 of the final x0 against the exact end point, started at grid[steps // 2] from a noised init image drawn from
    the data distribution: DDIM eta = 0, 2M (first-order restart) and 2M's tables on grid[k:] without the restart."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000, device)
    im.use_cuda_graph = graph
    gd = im.noise_schedulers[0]
    standin = AnalyticEps(1000).to(device)
    te = g["text_embeds"].to(device)
    k = steps // 2
    init = (MU + SD * torch.randn(SHAPE, generator=torch.Generator().manual_seed(steps))).to(device)
    ddim = gd.sampling_schedule(steps, 0., device)
    full = gd.dpm_solver_schedule(steps, device)
    walks = {"ddim": ddim._replace(grid=ddim.grid[k:]), "2m": gd.dpm_solver_schedule(steps, device, skip=k),
             "no_restart": full._replace(grid=full.grid[k:])}
    errs, outs = {}, {}
    for name, sched in walks.items():
        im.noise_fn = _bank(22)
        out = im._p_sample_loop(standin, SHAPE, noise_scheduler=gd, text_embeds=te, cond_scale=1., schedule=sched,
                                init_image=init)
        t0 = sched.grid[0]
        # the start exactly as mi_q_sample forms it from the fp32 tables
        x_t0 = gd.sqrt_alphas_cumprod[t0] * init.cpu() + gd.sqrt_one_minus_alphas_cumprod[t0] * \
            im.noise_fn.bank[("init", -1)]
        outs[name] = out
        errs[name] = rel_l2(out.double() * 2 - 1, exact_end_from(x_t0, t0, 1000))
    return errs, outs


def test_analytic_convergence_from_init_image(emu):
    """From grid[S // 2], 2M's final x0 is at least 10x closer to the exact end point than DDIM eta = 0's and 2x closer
    than 2M's tables without the first-order restart (fp64 ratios: 106 / 27 / 75 and 24 / 3.0 / 5.1 at S = 10 / 20 / 50);
    DDIM and 2M are closer at S = 50 than at S = 10."""
    errs = {}
    for S_ in (10, 20, 50):
        errs[S_], _ = analytic_img2img_errors("cpu", S_, graph=False)
        e = errs[S_]
        print(f"S={S_}, skip {S_ // 2}: rel-L2 vs exact end point: DDIM {e['ddim']:.3e}, 2M {e['2m']:.3e}, "
              f"2M without restart {e['no_restart']:.3e}")
        assert e["2m"] * 10 <= e["ddim"]
        assert e["2m"] * 2 <= e["no_restart"]
    assert errs[50]["ddim"] < errs[10]["ddim"] and errs[50]["2m"] < errs[10]["2m"]


# ------------------------------------------------------------------------------------------------ cascade entry and exit
def test_cascade_entry_and_exit_bitwise(emu):
    """stop_at_unet_number=1 returns the first stage's output of a full run; start_at_unet_number=2 from that output
    returns the full run's output bit for bit, with the SR stage's draws only."""
    im, g = cascade()
    kw = dict(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=2., sampling_timesteps=(None, 6),
              ddim_eta=0.5)
    im.noise_fn = shape_bank(5)
    seen = spy_stages(im)
    full = im.sample(**kw)
    full_calls = list(im.noise_fn.calls)
    del im._p_sample_loop                                                   # the spy
    im.noise_fn = shape_bank(5)
    first = im.sample(stop_at_unet_number=1, **kw)
    assert torch.equal(first, seen[0][1]) and first.shape == (2, 3, 16, 16)
    n_first = len(im.noise_fn.calls)
    assert im.noise_fn.calls == full_calls[:n_first]
    bank = im.noise_fn
    bank.calls.clear()
    second = im.sample(start_at_unet_number=2, start_images=first, **kw)
    assert torch.equal(second, full)
    assert bank.calls == full_calls[n_first:] and bank.calls[0] == ("lowres", 2, (2, 3, 32, 32))


@pytest.mark.parametrize("sampler", ["ddim", "dpmpp_2m"])
def test_neutral_arguments_change_nothing(emu, sampler):
    """skip_steps 0, no init or start images and the full stage range give the default call's output bit for bit."""
    outs = []
    for extra in ({}, dict(init_images=None, skip_steps=0, start_at_unet_number=1, start_images=None,
                           stop_at_unet_number=2), dict(init_images=(None, None), skip_steps=(0, None))):
        im, g = cascade()
        im.noise_fn = shape_bank(6)
        outs.append(im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=2.,
                              sampling_timesteps=5, sampler=sampler, **extra))
    assert torch.equal(outs[1], outs[0]) and torch.equal(outs[2], outs[0])


# ------------------------------------------------------------------------------------------------ argument checks
def test_img2img_asserts(emu):
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet, BaseTest, SuperTest
    im = Imagen(unets=(Unet(**BaseTest.defaults), Unet(**SuperTest.defaults)), text_encoder_name="t5_small",
                image_sizes=(16, 32), timesteps=25, cond_drop_prob=0.1)
    te = torch.zeros(2, 4, 512)
    img = torch.rand(2, 3, 32, 32)
    for bad in (0, 3, 1.0, True):
        with pytest.raises(AssertionError, match="start_at_unet_number must be between 1 and 2, got"):
            im.sample(text_embeds=te, start_at_unet_number=bad, start_images=img)
    for bad in (0, 3, 2.0):
        with pytest.raises(AssertionError, match=r"stop_at_unet_number must be between start_at_unet_number \(1\) and 2"):
            im.sample(text_embeds=te, stop_at_unet_number=bad)
    with pytest.raises(AssertionError, match=r"stop_at_unet_number must be between start_at_unet_number \(2\) and 2, "
                                             r"got 1"):
        im.sample(text_embeds=te, start_at_unet_number=2, start_images=img, stop_at_unet_number=1)
    with pytest.raises(AssertionError, match="start_images are required to start at unet 2"):
        im.sample(text_embeds=te, start_at_unet_number=2)
    with pytest.raises(AssertionError, match="start_images need start_at_unet_number > 1"):
        im.sample(text_embeds=te, start_images=img)
    for name in ("init_images", "skip_steps"):
        with pytest.raises(AssertionError, match=f"{name} must have one entry per unet \\(2\\), got 3"):
            im.sample(text_embeds=te, **{name: (None, None, None)})
    for bad, n in ((25, 25), (-1, 25), (1.5, 25), (True, 25)):
        with pytest.raises(AssertionError, match=f"skip_steps of unet 1 must be an int between 0 and {n - 1} "
                                                 f"\\(its walk has {n} points\\), got"):
            im.sample(text_embeds=te, init_images=img, skip_steps=bad)
    with pytest.raises(AssertionError, match=r"skip_steps of unet 2 must be an int between 0 and 4 \(its walk has 5 "
                                             r"points\), got 5"):
        im.sample(text_embeds=te, init_images=img, skip_steps=(0, 5), sampling_timesteps=5, sampler="dpmpp_2m")
    with pytest.raises(AssertionError, match="skip_steps > 0 needs an init image, and unet 2 has none"):
        im.sample(text_embeds=te, init_images=(img, None), skip_steps=3)
    with pytest.raises(AssertionError, match="init_images of unet 1 must be a float tensor"):
        im.sample(text_embeds=te, init_images=(img * 255).to(torch.uint8))
    for bad in (torch.rand(3, 3, 32, 32), torch.rand(2, 1, 32, 32), torch.rand(2, 3, 32, 16), torch.rand(2, 3, 32)):
        with pytest.raises(AssertionError, match=r"init_images of unet 2 must be \(b, channels, s, s\) = \(2, 3, s, s\)"):
            im.sample(text_embeds=te, init_images=(None, bad))
        with pytest.raises(AssertionError, match=r"start_images must be \(b, channels, s, s\) = \(2, 3, s, s\), got"):
            im.sample(text_embeds=te, start_at_unet_number=2, start_images=bad)
    with pytest.raises(AssertionError, match="start_images must be a float tensor"):
        im.sample(text_embeds=te, start_at_unet_number=2, start_images=(img * 255).to(torch.uint8))


# ------------------------------------------------------------------------------------------------ two gloo ranks
def _worker(rank, world, port, out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import minimagen_b200.ops as ops_mod
    from emu_ops import EmuOps
    ops_mod.set_ops(EmuOps())
    outs = _gloo_case(lambda v: v[rank * 2 // world:(rank + 1) * 2 // world], distributed=True)
    if rank == 0:
        torch.save(outs, out_path)
    dist.barrier()
    dist.destroy_process_group()


def _gloo_case(rows, distributed=False):
    """Two calls on the tiny cascade: the base stage alone from an init image (stop_at_unet_number=1), and the SR stage
    alone from start images with an init image.  Draws are a function of the global sample index."""
    im, g = cascade()
    im.use_cuda_graph = False
    gen = torch.Generator().manual_seed(9)
    bank = {}

    def noise_fn(kind, shape, step):
        key = (kind, step, tuple(shape[1:]))
        if key not in bank:
            bank[key] = torch.randn(2, *shape[1:], generator=gen)
        return rows(bank[key])
    im.noise_fn = noise_fn
    img = torch.rand(2, 3, 32, 32, generator=torch.Generator().manual_seed(10))
    start = torch.rand(2, 3, 16, 16, generator=torch.Generator().manual_seed(11))
    kw = dict(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=2., sampling_timesteps=6,
              distributed=distributed)
    base = im.sample(init_images=img, skip_steps=2, stop_at_unet_number=1, **kw)
    sr = im.sample(init_images=(None, img), skip_steps=(None, 3), start_at_unet_number=2, start_images=start, **kw)
    return base, sr


@pytest.mark.timeout(600)
def test_two_rank_gloo_matches_single_process(tmp_path, emu):
    port = 29800 + (os.getpid() % 200)
    out_path = str(tmp_path / "img2img_dist.pt")
    mp.spawn(_worker, args=(2, port, out_path), nprocs=2, join=True)
    dist_outs = torch.load(out_path)
    full = _gloo_case(lambda v: v)
    assert dist_outs[0].shape == (2, 3, 16, 16) and dist_outs[1].shape == (2, 3, 32, 32)
    # the CPU convolutions round differently at batch 1 and 2: the plain cascade's shards differ by 1.4e-5 rel-L2 too
    for got, want in zip(dist_outs, full):
        assert rel_l2(got, want) <= 1e-4
