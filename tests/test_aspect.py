"""Non-square sampling (Imagen.sample(image_sizes=)) and the implicit-GEMM convolution's tiling of widths that are not
powers of two, on the CPU.

  * `tile_box` / `conv_schedule` restate the tile geometry and schedule choice of conv_tc_launch (csrc/conv_tc.cu): the
    parent rule (tests/test_gpu_flagship_calls.py) on every shape it tiled exactly, and exact BW x BH one-image boxes for
    widths that are multiples of 8 but not powers of two (96: 32 x 4, 48: 16 x 8, 24: 8 x 16 at 128 pixels);
  * the U-Net lowering in float64 on the no-rounding backend (the `exact` fixture of test_lowering_exact.py) at 64 x 96
    and 128 x 192, with `RectEmuOps` answering the predicates by the new rule: every 3x3 / 1x1 / sub-pixel / in-place
    Downsample / stem conv goes to the tensor-core entry points, never to conv_direct, and the output equals the float64
    restatement to 1e-12 (1 + max|ref|);
  * the sampler at (32, 48) and the cascade (32, 48) -> (64, 96) on the emulated backend against the DDIM, 2M, RePaint
    and SDEdit restatements, image_sizes=None against explicit squares bit for bit, the argument checks, and two gloo
    ranks against one process.
"""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import ddim_restatement as D
import dpmpp_restatement as P
import img2img_restatement as S
import inpaint_restatement as IR
import test_lowering_exact as LX
from test_lowering_exact import exact  # noqa: F401  (the float64 host-code fixture)
from conftest import load_golden, rel_l2
from emu_ops import EmuOps
from oracle import restatement as R
from test_gpu_flagship_calls import pick_block_n
from test_gpu_flagship_calls import tile_geometry as old_tile_geometry
from test_gpu_flagship_calls import transposed_ok as old_transposed_ok
from test_img2img import cascade, shape_bank, spy_stages
from test_respaced import _tiny_imagen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT32_MAX = 2 ** 31 - 1
TRANSPOSED = (256, False, True)


# ------------------------------------------------------------------------------------------------ tile geometry
def tile_box(H, W, tile_pix):
    """(BW, BH) of conv_tc.cu's tile_box: exact one-image boxes for a width that is a multiple of 8 but neither a power of
    two nor a multiple of tile_pix, where BH = tile_pix / (W & -W) divides H; otherwise the parent rule."""
    low = W & -W
    if low != W and W % tile_pix and low >= 8 and H % (tile_pix // low) == 0:
        return low, tile_pix // low
    BW = tile_pix if W >= tile_pix else W
    return BW, min(tile_pix // BW, H)


def tile_geometry(H, W, B, tile_pix):
    """(BW, BH, tiles_w * tiles_h * tiles_b) as test_gpu_flagship_calls.tile_geometry, on tile_box."""
    BW, BH = tile_box(H, W, tile_pix)
    BB = tile_pix // (BW * BH)
    return BW, BH, -(-W // BW) * (H // BH) * -(-B // BB)


def _pow2(v):
    return v > 0 and v & (v - 1) == 0


def conv_supported(H, W):
    """conv_tc_supported's geometry part (channel conditions aside)."""
    if W >= 128:
        return True
    if not _pow2(W):
        low = W & -W
        return W > 0 and low >= 8 and H % (128 // low) == 0
    if W < 8:
        return False
    bh = 128 // W
    return H % bh == 0 if H >= bh else _pow2(H)


def transposed_ok(c_out, n_valid, out_sc, H, W, in_stride, out_sh, out_sw):
    if c_out != 128 or n_valid != c_out or out_sc != 1:
        return False
    BW, BH = tile_box(H, W, 256)
    if W % BW or not _pow2(BW) or BW < 8 or BW * in_stride > 256 or BW * BH != 256:
        return False
    if BH * out_sh + BW * out_sw + c_out > INT32_MAX:
        return False
    return H % BH == 0 and BH * in_stride <= 256


def conv_schedule(B, H, W, c_out, sms, hint=0, n_valid=0, out_sc=1, in_stride=1, out_sh=0, out_sw=0):
    """The (BLOCK_N, GN, transposed) instance conv_tc_launch launches (test_gpu_flagship_calls.conv_schedule on the new
    geometry)."""
    nv, sc, h = n_valid if n_valid > 0 else c_out, out_sc if out_sc > 0 else 1, abs(hint)
    ok = transposed_ok(c_out, nv, sc, H, W, in_stride, out_sh, out_sw)
    tr = ok if h == 256 else (h == 0 or c_out % h != 0) and ok and B * H * W // 256 >= sms
    if tr:
        return TRANSPOSED
    return pick_block_n(c_out, tile_geometry(H, W, B, 128)[2], hint, sms), False, False


def _old_supported(H, W):
    if W >= 128:
        return True
    if not _pow2(W) or W < 8:
        return False
    bh = 128 // W
    return H % bh == 0 if H >= bh else _pow2(H)


# every (H, W) an existing configuration, test or bench.py row runs a conv at: square powers of two from 1 to 1024 (with
# short images spanning several images per tile), the row GEMMs (H = 1), the ragged 136 / 520 widths and the 40 x 40 net
EXISTING = ([(s, s) for s in (1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024)] + [(40, 40), (20, 20), (10, 10)] +
            [(1, m) for m in (128, 256, 520, 1024, 2048, 4096, 8320, 16384)] + [(4, 136), (1, 136), (3, 136)] +
            [(2, 8), (4, 8), (8, 16), (1, 64), (2, 64)])


@pytest.mark.parametrize("H,W", EXISTING)
def test_existing_shapes_keep_their_geometry_and_schedule(H, W):
    for tp in (128, 256):
        for B in (1, 2, 32):
            if W % 8 == 0 or W >= tp or _pow2(W):
                assert tile_geometry(H, W, B, tp) == old_tile_geometry(H, W, B, tp)
    assert conv_supported(H, W) == _old_supported(H, W)
    for stride in (1, 2):
        assert transposed_ok(128, 128, 1, H, W, stride, W * 128, 128) == \
            old_transposed_ok(128, 128, 1, H, W, stride, W * 128, 128)
    for c_out in (16, 64, 128, 256, 384, 512):
        for B in (2, 32):
            assert conv_schedule(B, H, W, c_out, 132) == __import__("test_gpu_flagship_calls").conv_schedule(
                B, H, W, c_out, 132)


@pytest.mark.parametrize("W,box128,box256", [(24, (8, 16), (8, 32)), (48, (16, 8), (16, 16)), (96, (32, 4), (32, 8)),
                                             (192, (64, 2), (64, 4)), (384, (128, 1), (128, 2))])
def test_documented_boxes(W, box128, box256):
    assert tile_box(64, W, 128) == box128 and tile_box(64, W, 256) == box256
    for stride in (1, 2):
        assert transposed_ok(128, 128, 1, 64, W, stride, W * 128, 128) == (box256[0] * stride <= 256)
    H = 2 * W // 3                              # the 2:3 levels: 16 x 24 .. 256 x 384, on exact one-image tiles
    assert conv_supported(H, W) and tile_box(H, W, 128) == box128
    bw, bh = box128
    assert tile_geometry(H, W, 2, 128)[2] == (W // bw) * (H // bh) * 2
    # the 256-pixel box needs twice the rows: 16 x 24 has no transposed schedule
    assert transposed_ok(128, 128, 1, H, W, 1, W * 128, 128) == (H % box256[1] == 0) == (W != 24)


def test_widths_the_rule_rejects():
    assert not conv_supported(40, 40) and not conv_supported(12, 12) and not conv_supported(8, 12)
    assert not conv_supported(20, 24)                   # 20 % 16 != 0
    assert conv_supported(4, 136) and tile_box(4, 136, 128) == (128, 1)   # ragged tail as before (4 % 16 != 0)
    assert tile_box(128, 192, 128) == (64, 2)           # the one accepted class that changes: masked -> exact tiles


# ------------------------------------------------------------------------------------------------ exact lowering
class RectEmuOps(EmuOps):
    """EmuOps whose predicates follow the new width rule (conv_tc_supported, and through it the folded res_conv and the
    fused GroupNorm conv)."""

    def igemm_supported(self, H, W, c_in, c_out):
        if c_in <= 0 or c_in % 64 or c_out <= 0 or c_out % 16:
            return False
        return conv_supported(H, W)

    def conv_res1x1_supported(self, H, W, c_in, c_out, x_cin):
        return super().conv_res1x1_supported(H, W, c_in, c_out, x_cin) and self.igemm_supported(H, W, c_in, c_out)

    def conv_gn_supported(self, H, W, c0, c1, c_out, groups):
        return super().conv_gn_supported(H, W, c0, c1, c_out, groups) and self.igemm_supported(H, W, c0 + c1, c_out) \
            and H * W >= 128


@pytest.fixture
def rect_exact(exact):
    import minimagen_b200.ops as ops_mod
    e = RectEmuOps(lo=LX.F64, hi=LX.F64)
    ops_mod.set_ops(e)
    yield e


BASE_RECT = dict(dim=64, dim_mults=(1, 2, 4), layer_attns=(False, True, True), layer_cross_attns=(False, True, True),
                 text_embed_dim=768)
SR_RECT = dict(dim=64, dim_mults=(1, 2, 4), num_resnet_blocks=(1, 2, 2), layer_attns=(False, False, True),
               layer_cross_attns=(False, True, True), lowres_cond=True, memory_efficient=True, text_embed_dim=768)
RECT_CASES = {"base_64x96": (BASE_RECT, 64, 96), "sr_128x192": (SR_RECT, 128, 192)}


def _rect_forward(e, cfg, H, W, b=2):
    u, sd = LX._unet(cfg)
    g = torch.Generator().manual_seed(1)
    r = lambda *sh: torch.randn(*sh, generator=g, dtype=LX.F64)
    x = r(b, 3, H, W)
    kw = dict(text_embeds=r(b, 7, 768))
    if cfg.get("lowres_cond"):
        kw.update(lowres_cond_img=r(b, 3, H, W), lowres_noise_times=torch.tensor([200, 3][:b]))
    t = torch.tensor([999, 3][:b])
    out = {}
    e.calls.clear(), e.conv_log.clear()
    with torch.no_grad(), LX._arena(LX.BIG):
        for name, drop in (("cond", 0.), ("null", 1.)):
            out[name] = (u(x, t, cond_drop_prob=drop, **kw), R.unet_forward(sd, cfg, x, t, cond_drop_prob=drop, **kw))
    return out


@pytest.mark.parametrize("case", sorted(RECT_CASES))
def test_rectangular_lowering_exact(rect_exact, case):
    cfg, H, W = RECT_CASES[case]
    out = _rect_forward(rect_exact, cfg, H, W)
    for name, (got, ref) in out.items():
        ratio = LX._ratio(got, ref)
        print(f"{case} {name}: worst |out - ref| / (1e-12 (1 + max|ref|)) = {ratio:.2e}")
        assert ratio <= 1.
    calls = rect_exact.calls
    modes = {m[0] for m in rect_exact.conv_log if not isinstance(m[0], str)}
    assert "conv_direct" not in calls
    assert "stem_unroll" in calls and {2, 3, 4, 5, 6} <= modes
    assert any(m[0] == "res1x1" for m in rect_exact.conv_log)


def test_rectangular_lowering_exact_fused_gn(rect_exact, monkeypatch):
    """The fused GroupNorm conv (off by default) switched on everywhere it applies, at 64 x 96."""
    layers = LX._mods()[0]
    monkeypatch.setattr(layers, "FUSE_GN_CONV", "all")
    out = _rect_forward(rect_exact, BASE_RECT, 64, 96)
    for name, (got, ref) in out.items():
        assert LX._ratio(got, ref) <= 1., name
    assert "conv_gn" in rect_exact.calls and "conv_direct" not in rect_exact.calls


# ------------------------------------------------------------------------------------------------ emulated sampling
SHAPE = (2, 3, 32, 48)


def _bank(seed, shape=SHAPE):
    gen = torch.Generator().manual_seed(seed)
    bank, calls = {}, []

    def noise_fn(kind, shp, step):
        assert tuple(shp) == tuple(shape), (kind, shp)
        calls.append((kind, step))
        if (kind, step) not in bank:
            bank[(kind, step)] = torch.randn(shape, generator=gen)
        return bank[(kind, step)]
    noise_fn.calls = calls
    return noise_fn


def _ops(cls):
    import minimagen_b200.ops as ops_mod
    prev = ops_mod._OPS
    e = cls()
    ops_mod.set_ops(e)
    return e, prev


def _unet_kw(g):
    return dict(text_embeds=g["text_embeds"].cpu(), text_mask=g["text_mask"].cpu())


@pytest.mark.parametrize("sampler", ["ddim", "dpmpp_2m"])
def test_rectangular_sample_vs_restatement(emu, sampler):
    """Imagen.sample(image_sizes=((32, 48),)) on sample_loop.pt's tiny U-Net (CFG w = 3, S = 8 of T = 1000) against the
    DDIM (eta 0.5) and DPM-Solver++(2M) restatements, at the tolerance of their square tests."""
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    im.use_cuda_graph = False
    im.noise_fn = _bank(7)
    eta = 0.5 if sampler == "ddim" else 0.
    out = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=3., sampling_timesteps=8,
                    ddim_eta=eta, sampler=sampler, image_sizes=((32, 48),))
    assert out.shape == SHAPE
    if sampler == "ddim":
        ref = D.ddim_loop(g["state_dict"], g["cfg"], SHAPE, 1000, 8, eta, im.noise_fn, **_unet_kw(g))
    else:
        ref = P.dpmpp_loop(g["state_dict"], g["cfg"], SHAPE, 1000, 8, im.noise_fn, **_unet_kw(g))
    err = rel_l2(out, ref)
    print(f"{sampler} 32x48: rel-L2 vs restatement = {err:.3e}")
    assert err < 1e-3


@pytest.mark.parametrize("T,S_,R_", [(25, None, 2), (25, 5, 3)])
def test_rectangular_inpaint_vs_restatement(emu, T, S_, R_):
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, T)
    im.use_cuda_graph = False
    im.noise_fn = _bank(10 + R_)
    gen = torch.Generator().manual_seed(5)
    img = torch.rand(SHAPE, generator=gen)
    mask = torch.rand((2, 32, 48), generator=gen) < 0.5
    out = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=3., inpaint_images=img,
                    inpaint_masks=mask, inpaint_resample_times=R_, sampling_timesteps=S_, ddim_eta=0.5,
                    image_sizes=((32, 48),))
    ref = IR.inpaint_loop(g["state_dict"], g["cfg"], SHAPE, T, img * 2 - 1, mask, R_, im.noise_fn, steps=S_, eta=0.5,
                          **_unet_kw(g))
    err = rel_l2(out, ref)
    print(f"inpaint 32x48 T={T} S={S_} R={R_}: rel-L2 vs restated RePaint = {err:.3e}")
    assert err < 1e-3
    keep = mask[:, None].expand(SHAPE)
    assert (out - img)[keep].abs().max() <= 1.2e-7


def test_rectangular_cascade_vs_restatement(emu):
    """The tiny cascade of cascade_tiny.pt at (32, 48) -> (64, 96), CFG w = 2, with one init image at 16 x 24 for both
    stages (base on DDPM skipping 10 points, SR on 2M with S = 8 skipping 3); then the SR stage alone from start images at
    48 x 72.  Each stage against the SDEdit restatement on the inputs the product gave it."""
    im, g = cascade()
    sizes = ((32, 48), (64, 96))
    gen = torch.Generator().manual_seed(4)
    img = torch.rand(2, 3, 16, 24, generator=gen)
    start = torch.rand(2, 3, 48, 72, generator=gen)
    runs = (dict(init_images=img, skip_steps=(10, 3), sampling_timesteps=(None, 8)),
            dict(init_images=(None, img), skip_steps=(0, 3), sampling_timesteps=(None, 8), start_at_unet_number=2,
                 start_images=start))
    for run in runs:
        im.noise_fn = shape_bank(3)
        seen = spy_stages(im)
        final = im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=2., sampler="dpmpp_2m",
                          image_sizes=sizes, **run)
        del im._p_sample_loop
        first = run.get("start_at_unet_number", 1)
        assert len(seen) == 3 - first and final.shape == (2, 3, 64, 96)
        for (kw, out), i in zip(seen, range(first, 3)):
            shape = (2, 3, *sizes[i - 1])
            assert out.shape == shape and kw["init_image"].shape == shape
            cfg, sd = g["cfgs"][i - 1], g["state_dicts"][i - 1]
            lowres = {} if kw["lowres_cond_img"] is None else dict(lowres_cond_img=kw["lowres_cond_img"] * 2 - 1,
                                                                     lowres_noise_times=kw["lowres_noise_times"])
            assert (i == 2) == bool(lowres) and (not lowres or kw["lowres_cond_img"].shape == shape)
            cfg = dict(cfg, lowres_cond=bool(lowres))
            steps, sampler, skip = ((None, "ddim", 10), (8, "dpmpp_2m", 3))[i - 1]
            ref = S.sdedit_loop(sd, cfg, shape, 25, kw["init_image"], skip, im.noise_fn, steps=steps, sampler=sampler,
                                cond_scale=2., text_embeds=g["text_embeds"], text_mask=g["text_mask"], **lowres)
            err = rel_l2(out, ref)
            print(f"cascade stage {shape[2]}x{shape[3]} {sampler} skip={skip}: rel-L2 vs restated SDEdit = {err:.3e}")
            assert err < 1e-3


def test_rectangular_resize_axes():
    """resize_image_to with a pair scales each axis by its own factor; an int keeps the square path."""
    from minimagen_b200.helpers import resize_image_to
    import minimagen_b200.ops as ops_mod
    e, prev = _ops(EmuOps)
    try:
        x = torch.rand(2, 3, 16, 24, generator=torch.Generator().manual_seed(0))
        y = resize_image_to(x, (32, 48))
        assert y.shape == (2, 3, 32, 48)
        assert resize_image_to(x, (16, 24)) is x
        sq = torch.rand(2, 3, 16, 16, generator=torch.Generator().manual_seed(1))
        assert torch.equal(resize_image_to(sq, (32, 32)), resize_image_to(sq, 32))
        # a separable resize of a constant-per-axis image: rows of x stay rows of y
        col = torch.linspace(0, 1, 24).expand(2, 3, 16, 24).contiguous()
        yc = resize_image_to(col, (32, 48))
        assert (yc - yc[:, :, :1]).abs().max() < 1e-6
    finally:
        ops_mod.set_ops(prev)


@pytest.mark.parametrize("sampler", ["ddim", "dpmpp_2m"])
def test_explicit_squares_are_the_default(emu, sampler):
    """image_sizes=None, the constructor's sizes as ints and as (s, s) pairs give the same output bit for bit."""
    outs = []
    for sizes in (None, (16, 32), ((16, 16), [32, 32])):
        im, g = cascade()
        im.noise_fn = shape_bank(6)
        outs.append(im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=2.,
                              sampling_timesteps=5, sampler=sampler, image_sizes=sizes))
    assert torch.equal(outs[1], outs[0]) and torch.equal(outs[2], outs[0])


def test_rectangular_asserts(emu):
    im, g = cascade()
    kw = dict(text_embeds=g["text_embeds"], text_masks=g["text_mask"], sampling_timesteps=3)
    assert im.downsample_factor(im.unets[0]) == 2 and im.downsample_factor(im.unets[1]) == 4
    with pytest.raises(AssertionError, match=r"image_sizes must have one entry per unet \(2\), got"):
        im.sample(image_sizes=((32, 48),), **kw)
    for bad in ((32, 48, 1), "32", 32.0, (32, None)):
        with pytest.raises(AssertionError, match=r"image size of unet 1 must be an int or a pair \(h, w\), got"):
            im.sample(image_sizes=(bad, (64, 96)), **kw)
    with pytest.raises(AssertionError, match="image size of unet 1 must be positive multiples of its downsampling "
                                             "factor 2, got 31 x 48"):
        im.sample(image_sizes=((31, 48), (64, 96)), **kw)
    with pytest.raises(AssertionError, match="image size of unet 2 must be positive multiples of its downsampling "
                                             "factor 4, got 64 x 94"):
        im.sample(image_sizes=((32, 48), (64, 94)), **kw)
    with pytest.raises(AssertionError, match="factor 2, got 0 x 0"):
        im.sample(image_sizes=(0, 32), **kw)
    with pytest.raises(AssertionError, match=r"the unets that run must share one aspect ratio: unet 2 samples 64 x 64, "
                                             r"unet 1 32 x 48"):
        im.sample(image_sizes=((32, 48), 64), **kw)
    # only the stages that run are read
    im.noise_fn = shape_bank(1)
    out = im.sample(image_sizes=("unused", (32, 48)), start_at_unet_number=2, start_images=torch.rand(2, 3, 8, 12), **kw)
    assert out.shape == (2, 3, 32, 48)
    sizes = ((32, 48), (64, 96))
    for bad in (torch.rand(2, 3, 32, 32), torch.rand(2, 3, 48, 32), torch.rand(2, 1, 32, 48), torch.rand(2, 3, 48)):
        with pytest.raises(AssertionError, match=r"init_images of unet 2 must be \(b, channels, h, w\) = \(2, 3, h, w\) "
                                                 r"with h:w = 2:3"):
            im.sample(image_sizes=sizes, init_images=(None, bad), **kw)
        with pytest.raises(AssertionError, match=r"start_images must be \(b, channels, h, w\) = \(2, 3, h, w\) with "
                                                 r"h:w = 2:3"):
            im.sample(image_sizes=sizes, start_at_unet_number=2, start_images=bad, **kw)
        with pytest.raises(AssertionError, match=r"inpaint_images must be \(b, channels, h, w\) = \(2, 3, h, w\) with "
                                                 r"h:w = 2:3"):
            im.sample(image_sizes=sizes, inpaint_images=bad, inpaint_masks=torch.ones(2, 32, 48, dtype=torch.bool), **kw)
    img = torch.rand(2, 3, 32, 48)
    for bad in (torch.ones(2, 32, 32, dtype=torch.bool), torch.ones(2, 48, 32, dtype=torch.bool),
                torch.ones(2, 1, 32, 48, dtype=torch.bool)):
        with pytest.raises(AssertionError, match=r"inpaint_masks must be \(b, h, w\) = \(2, 32, 48\) like inpaint_images"):
            im.sample(image_sizes=sizes, inpaint_images=img, inpaint_masks=bad, **kw)
    # square runs keep the square messages
    with pytest.raises(AssertionError, match=r"init_images of unet 2 must be \(b, channels, s, s\) = \(2, 3, s, s\)"):
        im.sample(init_images=(None, img), **kw)


# ------------------------------------------------------------------------------------------------ two gloo ranks
def _gloo_case(rows, distributed=False):
    """The tiny cascade at (32, 48) -> (64, 96) with an init image for the SR stage; draws are a function of the global
    sample index."""
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
    img = torch.rand(2, 3, 32, 48, generator=torch.Generator().manual_seed(10))
    return im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=2., sampling_timesteps=6,
                     init_images=(None, img), skip_steps=(0, 2), image_sizes=((32, 48), (64, 96)),
                     distributed=distributed)


def _worker(rank, world, port, out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import minimagen_b200.ops as ops_mod
    ops_mod.set_ops(EmuOps())
    out = _gloo_case(lambda v: v[rank * 2 // world:(rank + 1) * 2 // world], distributed=True)
    if rank == 0:
        torch.save(out, out_path)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_rank_gloo_rectangular_matches_single_process(tmp_path, emu):
    port = 30000 + (os.getpid() % 200)
    out_path = str(tmp_path / "aspect_dist.pt")
    mp.spawn(_worker, args=(2, port, out_path), nprocs=2, join=True)
    got = torch.load(out_path)
    want = _gloo_case(lambda v: v)
    assert got.shape == want.shape == (2, 3, 64, 96)
    # the CPU convolutions round differently at batch 1 and 2 (test_img2img's gloo test: 1.4e-5 rel-L2)
    assert rel_l2(got, want) <= 1e-4
