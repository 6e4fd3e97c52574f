"""Image-to-image sampling and partial cascades on the GPU: the captured loop against the eager one bit for bit (DDPM,
DDIM, 2M and inpainting, each from an init image with skipped points), one cached graph serving every skip count and
init image, the tensor-core SR configuration against the SDEdit restatement, cascade entry and exit on the native path,
and batch sharding with init and start images."""
import pytest
import torch

import img2img_restatement as S
from conftest import load_golden, rel_l2
from test_dpmpp import SHAPE, AnalyticEps
from test_img2img import cascade, init_image, spy_stages
from test_inpaint import known_and_mask
from test_respaced import _bank, _tiny_imagen

pytestmark = pytest.mark.gpu


def _walk(gd, kind, skip):
    """The shortened walk Imagen.sample builds for `skip_steps=skip`."""
    if kind == "2m":
        return gd.dpm_solver_schedule(12, "cuda", skip=skip)
    sched = gd.ddpm_schedule("cuda") if kind == "ddpm" else gd.sampling_schedule(12, 0.5, "cuda")
    return sched._replace(grid=sched.grid[skip:])


@pytest.mark.parametrize("kind,skip", [("ddpm", 990), ("ddim", 4), ("2m", 5), ("inpaint", 3)])
def test_graph_vs_eager_bitwise(native, kind, skip):
    """With the analytic stand-in (no atomics) the captured loop from a noised init image equals the eager one."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000, "cuda")
    standin = AnalyticEps(1000).cuda()
    gd = im.noise_schedulers[0]
    init = (init_image(skip) * 2 - 1).cuda()
    inpaint = None
    if kind == "inpaint":
        img, mask = known_and_mask(skip)
        inpaint = ((img * 2 - 1).cuda(), mask.float().reshape(2, -1).cuda(), 2)
    sched = _walk(gd, "ddim" if kind == "inpaint" else kind, skip)
    outs = []
    for graph in (False, True):
        im.use_cuda_graph = graph
        im.noise_fn = _bank(skip)
        outs.append(im._p_sample_loop(standin, SHAPE, noise_scheduler=gd, text_embeds=g["text_embeds"].cuda(),
                                      cond_scale=1., schedule=sched, inpaint=inpaint, init_image=init))
    assert torch.equal(outs[0], outs[1])
    assert len(im._graphs) == 1
    if kind == "inpaint":
        assert next(iter(im._graphs))[-1] == "inpaint"


def test_one_graph_serves_every_skip_and_init_image(native):
    """DDIM calls of Imagen.sample with and without init images and with several skip counts share one captured graph
    (2M ones one more); each equals the same call on the eager loop."""
    g = load_golden("sample_loop.pt")
    im, ref = _tiny_imagen(g, 1000, "cuda"), _tiny_imagen(g, 1000, "cuda")
    ref.use_cuda_graph = False
    cases = ((None, 0, "ddim", 1), (init_image(1), 3, "ddim", 1), (init_image(2), 6, "ddim", 1), (init_image(1), 0, "ddim", 1),
             (init_image(3), 2, "dpmpp_2m", 2), (init_image(4), 5, "dpmpp_2m", 2))
    for seed, (img, skip, sampler, n_graphs) in enumerate(cases):
        outs = []
        for model in (im, ref):
            model.noise_fn = _bank(30 + seed)
            outs.append(model.sample(text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda(),
                                     cond_scale=3., sampling_timesteps=10, ddim_eta=0.5 if sampler == "ddim" else 0.,
                                     sampler=sampler, init_images=None if img is None else img.cuda(),
                                     skip_steps=skip))
        err = rel_l2(outs[0], outs[1])
        print(f"{sampler} skip={skip} init={img is not None}: graph vs eager rel-L2 {err:.3e}")
        assert err <= 1e-5
        assert len(im._graphs) == n_graphs


@pytest.mark.parametrize("sampler,skip", [("ddim", 2), ("dpmpp_2m", 2)])
def test_tensor_core_sr_config_vs_restatement(native, sampler, skip):
    """The sr_d64 configuration of test_gpu_unet.CFGS (tensor-core convs, lowres conditioning) at 64x64, b = 2, CFG w = 3,
    S = 6 from a noised init image, against the restated SDEdit loop.  fp16 operand budget: 2e-3."""
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import BaseTest, Unet
    from test_gpu_unet import CFGS
    _, cfg, s, lowres, b = next(c for c in CFGS if c[0] == "sr_d64")
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
    init = init_image(5, shape) * 2 - 1
    im.noise_fn = _bank(4, shape)
    gd = im.noise_schedulers[1]
    if sampler == "dpmpp_2m":
        sched = gd.dpm_solver_schedule(6, "cuda", skip=skip)
    else:
        sched = gd.sampling_schedule(6, 0., "cuda")
        sched = sched._replace(grid=sched.grid[skip:])
    out = im._p_sample_loop(im.unets[1], shape, noise_scheduler=gd, text_embeds=te.cuda(), text_mask=tm.cuda(),
                            lowres_cond_img=lowres_img.cuda(), lowres_noise_times=lnt.cuda(), cond_scale=3.,
                            schedule=sched, init_image=init.cuda())
    ref = S.sdedit_loop(sd, cfg, shape, 1000, init, skip, im.noise_fn, steps=6, sampler=sampler, text_embeds=te,
                        text_mask=tm, lowres_cond_img=lowres_img * 2 - 1, lowres_noise_times=lnt)
    err = rel_l2(out, ref)
    print(f"sr_d64 {sampler} S=6 skip={skip}: rel-L2 vs restated SDEdit = {err:.3e}")
    assert err < 2e-3


def test_cascade_entry_and_exit_bitwise(native):
    """On the native path with captured graphs: stop_at_unet_number=1 returns the first stage's output of a full run, and
    start_at_unet_number=2 from it returns the full run's output bit for bit."""
    im, g = cascade("cuda")
    gen = torch.Generator().manual_seed(7)
    bank = {}

    def noise_fn(kind, shape, step):
        key = (kind, step, tuple(shape))
        if key not in bank:
            bank[key] = torch.randn(shape, generator=gen)
        return bank[key]
    im.noise_fn = noise_fn
    im.use_cuda_graph = True
    kw = dict(text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda(), cond_scale=2.,
              sampling_timesteps=(None, 6), ddim_eta=0.5)
    seen = spy_stages(im)
    full = im.sample(**kw)
    del im._p_sample_loop                                                   # the spy
    first = im.sample(stop_at_unet_number=1, **kw)
    assert torch.equal(first.cpu(), seen[0][1])
    second = im.sample(start_at_unet_number=2, start_images=first, **kw)
    assert torch.equal(second, full)


def test_sharding_invariance_with_init_and_start_images(native):
    """b = 4 equals two shards of 2 (what two ranks do), for the base stage alone from init images and the SR stage alone
    from start images with init images, on the tiny cascade."""
    im, g = cascade("cuda")
    gen = torch.Generator().manual_seed(0)
    bank = {}

    def noise_fn(kind, shape, step):
        key = (kind, step, tuple(shape[1:]))
        if key not in bank:
            bank[key] = torch.randn(4, *shape[1:], generator=gen)
        return bank[key][noise_fn.lo:noise_fn.lo + shape[0]]
    noise_fn.lo = 0
    im.noise_fn = noise_fn
    te = torch.randn(4, 9, 512, generator=gen).cuda()
    tm = torch.ones(4, 9, dtype=torch.bool).cuda()
    img = init_image(8, (4, 3, 32, 32)).cuda()
    start = init_image(9, (4, 3, 16, 16)).cuda()
    calls = (lambda lo, n: dict(init_images=img[lo:lo + n], skip_steps=2, stop_at_unet_number=1),
             lambda lo, n: dict(init_images=(None, img[lo:lo + n]), skip_steps=(None, 3), start_at_unet_number=2,
                                start_images=start[lo:lo + n]))
    for call in calls:
        noise_fn.lo = 0
        full = im.sample(text_embeds=te, text_masks=tm, cond_scale=2., sampling_timesteps=6, **call(0, 4))
        parts = []
        for lo in (0, 2):
            noise_fn.lo = lo
            parts.append(im.sample(text_embeds=te[lo:lo + 2], text_masks=tm[lo:lo + 2], cond_scale=2.,
                                   sampling_timesteps=6, **call(lo, 2)))
        err = rel_l2(torch.cat(parts), full)
        print(f"b=4 vs two shards of 2: rel-L2 = {err:.3e}")
        assert torch.isfinite(full).all() and err <= 1e-5
