"""Fewer-step DDIM sampling on the GPU: the timestep-table kernel (mi_step_advance_t_table), the respaced loop through the
captured step graph and eagerly, against the DDPM path (S = T, eta = 1), the paper-form CPU restatement and the
reference's cascade golden; one captured graph serving DDPM and DDIM loops in turn."""
import pytest
import torch

import ddim_restatement as D
from conftest import load_golden, rel_l2
from test_respaced import _bank, _tiny_imagen, restated_tiny_loop

pytestmark = pytest.mark.gpu

SHAPE = (2, 3, 64, 64)


def _loop(im, g, sched=None, graph=True, max_steps=None):
    im.use_cuda_graph = graph
    return im._p_sample_loop(im.unets[0], SHAPE, noise_scheduler=im.noise_schedulers[0],
                             text_embeds=g["text_embeds"].cuda(), text_mask=g["text_mask"].cuda(), cond_scale=3.,
                             schedule=sched, max_steps=max_steps)


def test_advance_t_table_kernel(native):
    from minimagen_b200.diffusion_model import GaussianDiffusion
    T, B = 1000, 5
    sched = GaussianDiffusion(timesteps=T).sampling_schedule(10, 0., "cuda")
    t = torch.full((B,), T - 1, dtype=torch.long, device="cuda")
    seen = []
    for _ in range(len(sched.grid) + 2):
        seen.append(t.tolist())
        native.step_advance_t_table(t, sched.next_t, T, B)
    assert [row[0] for row in seen] == list(sched.grid) + [0, 0]          # walks T-1 .. 0 exactly, then stays at 0
    assert all(len(set(row)) == 1 for row in seen)
    # out-of-range timesteps go to 0 (no read outside the table)
    t = torch.tensor([-1, T, 1 << 40, -(1 << 40), 999, 0], dtype=torch.long, device="cuda")
    native.step_advance_t_table(t, sched.next_t, T, t.numel())
    assert t.tolist() == [0, 0, 0, 0, 888, 0]
    # captured in a CUDA graph: one replay = one step of the walk
    t = torch.full((B,), T - 1, dtype=torch.long, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        native.step_advance_t_table(t, sched.next_t, T, B)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        native.step_advance_t_table(t, sched.next_t, T, B)
    t.fill_(T - 1)
    walk = []
    for _ in range(len(sched.grid)):
        graph.replay()
        walk.append(t.tolist())
    torch.cuda.synchronize()
    assert [row[0] for row in walk] == list(sched.grid[1:]) + [0] and all(len(set(r)) == 1 for r in walk)


@pytest.mark.parametrize("graph", [False, True])
def test_full_steps_equal_ddpm_loop(native, graph):
    """S = T = 25, eta = 1 is the DDPM sampler.  Both loops on the same kernels; the U-Net's double-atomic GroupNorm sums
    may reorder between runs, so the bound is 1e-6 rather than bitwise."""
    g = load_golden("sample_loop.pt")
    outs = []
    for respaced in (False, True):
        im = _tiny_imagen(g, 25, "cuda")
        im.noise_fn = _bank(5)
        sched = im.noise_schedulers[0].sampling_schedule(25, 1., "cuda") if respaced else None
        outs.append(_loop(im, g, sched, graph))
        assert im.noise_fn.calls == [("init", -1)] + [("step", t) for t in range(24, -1, -1)]
    err = rel_l2(outs[1], outs[0])
    print(f"S=T=25 eta=1 (graph={graph}): rel-L2 vs DDPM loop = {err:.3e}")
    assert err <= 1e-6


@pytest.mark.parametrize("eta", [0., 0.5])
def test_respaced_graph_eager_and_restatement(native, eta):
    g = load_golden("sample_loop.pt")
    outs = {}
    for graph in (False, True):
        im = _tiny_imagen(g, 1000, "cuda")
        im.noise_fn = _bank(7)
        outs[graph] = _loop(im, g, im.noise_schedulers[0].sampling_schedule(8, eta, "cuda"), graph)
        if graph:
            assert len(im._graphs) == 1
    ref = restated_tiny_loop(g, 1000, 8, eta, _bank(7))
    e_ge, e_ref = rel_l2(outs[True], outs[False]), rel_l2(outs[True], ref)
    print(f"S=8 eta={eta}: graph vs eager {e_ge:.3e}; vs restated DDIM {e_ref:.3e}")
    assert e_ge <= 1e-5 and e_ref < 1e-3


def test_respaced_graph_reused_across_steps_and_eta(native):
    """Changing S or eta reuses the one captured respaced graph (tables refreshed in place); each loop equals eager."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000, "cuda")
    ref = _tiny_imagen(g, 1000, "cuda")
    for S, eta in ((8, 0.5), (5, 0.), (12, 1.)):
        im.noise_fn, ref.noise_fn = _bank(S), _bank(S)
        out = _loop(im, g, im.noise_schedulers[0].sampling_schedule(S, eta, "cuda"), True)
        want = _loop(ref, g, ref.noise_schedulers[0].sampling_schedule(S, eta, "cuda"), False)
        assert len(im._graphs) == 1
        err = rel_l2(out, want)
        print(f"reused graph S={S} eta={eta}: rel-L2 vs eager {err:.3e}")
        assert err <= 1e-5
    # max_steps: the first iterations of the grid, through the same graph
    im.noise_fn, ref.noise_fn = _bank(3), _bank(3)
    out = _loop(im, g, im.noise_schedulers[0].sampling_schedule(10, 0.5, "cuda"), True, max_steps=4)
    want = _loop(ref, g, ref.noise_schedulers[0].sampling_schedule(10, 0.5, "cuda"), False, max_steps=4)
    assert len(im._graphs) == 1 and rel_l2(out, want) <= 1e-5
    assert im.noise_fn.calls == [("init", -1), ("step", 999), ("step", 888), ("step", 777), ("step", 666)]


def test_one_graph_serves_ddpm_and_ddim(native):
    """DDPM, then DDIM (S = 8, eta = 0.5), then DDPM again on one Imagen run through one captured graph; each loop equals
    its own eager run, and the last DDPM loop equals the first (the DDIM tables were replaced)."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 25, "cuda")
    ref = _tiny_imagen(g, 25, "cuda")
    outs = []
    for S in (None, 8, None):
        im.noise_fn, ref.noise_fn = _bank(11), _bank(11)
        out = _loop(im, g, None if S is None else im.noise_schedulers[0].sampling_schedule(S, 0.5, "cuda"), True)
        want = _loop(ref, g, None if S is None else ref.noise_schedulers[0].sampling_schedule(S, 0.5, "cuda"), False)
        err = rel_l2(out, want)
        print(f"S={S}: graph vs eager {err:.3e}")
        assert err <= 1e-5
        outs.append(out)
    assert len(im._graphs) == 1
    assert rel_l2(outs[2], outs[0]) <= 1e-5


def test_cascade_full_steps_vs_reference_golden(native):
    from test_host_logic import _cascade_from_golden
    g = load_golden("cascade_tiny.pt")
    im, it = _cascade_from_golden(g, "cuda")
    im.use_cuda_graph = True
    out = im.sample(text_embeds=g["text_embeds"].cuda(), text_masks=g["text_mask"].cuda(), cond_scale=g["cond_scale"],
                    lowres_sample_noise_level=g["lowres_noise_level"], sampling_timesteps=25, ddim_eta=1.)
    assert next(it, None) is None
    err = rel_l2(out, g["out"])
    print(f"cascade S=T=25 eta=1 (graph): rel-L2 vs reference = {err:.3e}")
    assert err < 1e-3


def test_tensor_core_sr_config_vs_restatement(native):
    """The sr_d64 configuration of test_gpu_unet.CFGS (tensor-core convs, lowres conditioning) at 64x64, b = 2, CFG w = 3,
    S = 4, eta = 0, against the restated DDIM loop.  fp16 operand budget: 2e-3."""
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
    lowres_img = torch.rand(b, 3, s, s, generator=gen)                # [0, 1]; the loop normalises it
    lnt = torch.full((b,), 200)
    shape = (b, 3, s, s)
    im.noise_fn = _bank(4, shape)
    sched = im.noise_schedulers[1].sampling_schedule(4, 0., "cuda")
    out = im._p_sample_loop(im.unets[1], shape, noise_scheduler=im.noise_schedulers[1], text_embeds=te.cuda(),
                            text_mask=tm.cuda(), lowres_cond_img=lowres_img.cuda(), lowres_noise_times=lnt.cuda(),
                            cond_scale=3., schedule=sched)
    ref = D.ddim_loop(sd, cfg, shape, 1000, 4, 0., im.noise_fn, text_embeds=te, text_mask=tm,
                      lowres_cond_img=lowres_img * 2 - 1, lowres_noise_times=lnt)
    err = rel_l2(out, ref)
    print(f"sr_d64 S=4 eta=0: rel-L2 vs restated DDIM = {err:.3e}")
    assert err < 2e-3


def test_respaced_sample_sharding_invariance(native):
    """A respaced Imagen.sample at b = 4 equals the same samples computed as two shards of 2 (what two ranks do)."""
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
    kw = dict(cond_scale=3., sampling_timesteps=6, ddim_eta=0.5)
    full = im.sample(text_embeds=te, text_masks=tm, **kw)
    assert full.shape == (4, 3, 64, 64) and torch.isfinite(full).all()
    assert sorted(k[1] for k in bank if k[0] == "step") == sorted(D.ddim_grid(25, 6))
    parts = []
    for lo in (0, 2):
        noise_fn.lo = lo
        parts.append(im.sample(text_embeds=te[lo:lo + 2], text_masks=tm[lo:lo + 2], **kw))
    err = rel_l2(torch.cat(parts), full)
    print(f"respaced sample b=4 vs two shards of 2: rel-L2 = {err:.3e}")
    assert err <= 1e-5
