"""Every kernel call writes only its outputs, on the native kernels (FootprintOps, tests/footprint_ops.py): each call's
arguments relocated between guard bands, and after the call every guard byte and every byte outside the call's write
footprint bitwise unchanged.

  * real runs, every call footprint-checked (and, but for the cfg-3 pass, float64-checked by CheckingOps around it): every
    forward case of test_gpu_lowering_calls (batch16_two_chunks and cfg_batched among them), every training step of
    checking_ops.train_cases(), the cfg-batched DDIM cascade of test_every_call_of_a_combined_cascade, DeepCache's cached
    tiny cascade, the rectangular 64 x 96 base forward, a B = 1 eager sample of cfg 2b's U-Net (Base at dim 128) at 64 px
    (8 x 8 levels: a conv tile covers image 1, which does not exist), and one conditional pass of the cfg-3 U-Net at the
    benchmark's size (b = 32, 256 x 256) with FootprintOps alone (test_gpu_flagship_calls checks that call list in float64);
  * the boundary calls of test_footprint.boundary_calls, outputs sized exactly so that a first stray element lands in a
    guard: partial multi-image tiles, ragged widths, every conv schedule, the NCHW final conv, a concat slice, the four
    sub-pixel phases, adjacent accumulators, attention on both paths, the step-epilogue family, ...;
  * negative controls: for conv_igemm at a ragged width, the strided attention output and step_epilogue a footprint one
    pixel column, row or element smaller than the real one must fail and name that element (every store still lands in
    memory the test allocated), which shows the check sees the native kernels' writes.

Each case prints its calls, methods, bytes relocated, wall time and peak memory; the last test asserts that every
kernel-launching method of NativeOps was footprint-checked by the file's cases.  Eager runs only.
"""
import inspect
import time

import pytest
import torch

from checking_ops import ALLOWED, CheckingOps, run_training_step, train_cases
from footprint_ops import FootprintOps, _view, installed, unchecked
from test_gpu_lowering_calls import CASES

pytestmark = pytest.mark.gpu
COVERED = set()


def _run(native, name, fn, checking=True, fp=None, fresh=False):
    fp = fp or FootprintOps(native)
    proxy = CheckingOps(fp, fresh_accumulators=fresh) if checking else fp
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    with installed(proxy):
        out = fn(proxy)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    print(f"\n{name} on {torch.cuda.get_device_name(0)}: {fp.calls} calls of {len(fp.checked)} methods, "
          f"{fp.relocated / 2 ** 30:.2f} GiB relocated, {wall:.1f} s, peak memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    assert not unchecked(fp), f"kernels that ran without a footprint check: {sorted(unchecked(fp))}"
    if checking:
        assert not proxy.called - proxy.checked - ALLOWED
    COVERED.update(fp.checked)
    return out


# ------------------------------------------------------------------------------------------------ real runs
@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_forward(native, name):
    from test_gpu_lowering_calls import forward_case, run_forward
    case = forward_case(name)
    out = _run(native, name, lambda ops: run_forward(ops, *case))
    assert torch.isfinite(out).all()


@pytest.mark.parametrize("name", list(train_cases()))
def test_training_step(native, name):
    spec = train_cases()[name][0]
    grads = _run(native, f"{name} training step", lambda ops: run_training_step(spec, "cuda"), fresh=True)
    assert all(torch.isfinite(g).all() for g in grads.values())


def test_combined_cascade(native):
    from test_gpu_aspect import _imagen, _prompts
    from test_gpu_sampling_feature_calls import SIZES
    from test_sampling_feature_calls import cascade_case
    im = _imagen(True)
    te, tm = _prompts(4)
    kw = cascade_case(im, "ddim", 4, SIZES, 512, "cuda", True)
    out = _run(native, "DDIM cascade, cfg_batched", lambda ops: im.sample(text_embeds=te, text_masks=tm, **kw))
    assert torch.isfinite(out).all()


def test_cached_tiny_cascade(native):
    from test_gpu_deepcache import _cascade, _case
    im, g = _cascade()
    kw = _case(im, g, "ddim")
    im.use_cuda_graph = False
    out = _run(native, "DeepCache tiny cascade", lambda ops: im.sample(cache_interval=2, **kw))
    assert torch.isfinite(out).all()


def test_rectangular_base_forward(native):
    from test_gpu_aspect import _forward_case, _run_forward
    _, u, _, x, t, kw = _forward_case("base_64x96")
    outs = _run(native, "base 64 x 96", lambda ops: _run_forward("base_64x96", ops, u, x, t, kw)[0])
    assert all(torch.isfinite(o).all() for o in outs)


def test_b1_sample_of_cfg2b_base(native):
    """cfg 2b's U-Net at 64 px, B = 1, the conditional and null passes separate (no cfg_batched): its 8 x 8 convs run
    tiles that cover image 1."""
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Base, Unet
    torch.manual_seed(0)
    u = Unet(**{**Base.defaults, "dim": 128}, text_embed_dim=768)
    im = Imagen(unets=(u,), text_encoder_name="t5_base", image_sizes=(64,), timesteps=1000, cond_drop_prob=0.1).eval().cuda()
    im.use_cuda_graph = False
    im.cfg_batched = False
    gen = torch.Generator().manual_seed(2)
    te, tm = torch.randn(1, 12, 768, generator=gen).cuda(), torch.ones(1, 12, dtype=torch.bool).cuda()
    out = _run(native, "cfg 2b base, B = 1, 64 px", lambda ops: im.sample(text_embeds=te, text_masks=tm, cond_scale=3.,
                                                                           sampling_timesteps=2))
    assert out.shape == (1, 3, 64, 64) and torch.isfinite(out).all()


def test_cfg3_conditional_pass_at_benchmark_size(native):
    from minimagen_b200.Unet import Super, Unet
    torch.manual_seed(0)
    b = 32
    u = Unet(**dict(Super.defaults, lowres_cond=True, text_embed_dim=768)).eval().cuda()
    gen = torch.Generator().manual_seed(11)
    x, low = (torch.randn(b, 3, 256, 256, generator=gen).cuda() for _ in range(2))
    tm = torch.ones(b, 20, dtype=torch.bool)
    tm[-1, 5:] = False
    kw = dict(text_embeds=torch.randn(b, 20, 768, generator=gen).cuda(), text_mask=tm.cuda(), lowres_cond_img=low,
              lowres_noise_times=torch.full((b,), 200).cuda())
    t = torch.randint(0, 1000, (b,), generator=gen).cuda()

    def fwd(ops):
        with torch.no_grad():
            return u(x, t, **kw)
    out = _run(native, "cfg 3 conditional pass, b = 32, 256 x 256", fwd, checking=False)
    assert torch.isfinite(out).all()


# ------------------------------------------------------------------------------------------------ boundary calls
def test_boundary_calls(native):
    from test_footprint import boundary_calls
    _run(native, "boundary calls", lambda ops: boundary_calls(ops, "cuda"))


# ------------------------------------------------------------------------------------------------ negative controls
class _Narrow(FootprintOps):
    """Declares conv_igemm one pixel column, attention one query row and step_epilogue one element short."""

    def _writes_conv_igemm(self, act, B, H, W, lda, c_off, c_in, wp, c_out, kh, kw, mode, bias, residual, out_f32,
                           out_f16, out_strides, block_n=0, out_sc=1, n_valid=0, act2=None, lda2=0, c_off2=0, c_in1=0,
                           out_stats=None):
        sb, sh, sw = out_strides
        return [_view(out_f16, (B, H, W - 1, c_out), (sb, sh, sw, 1)), _view(out_stats, (B * c_out // 8,), (1,))]

    def _writes_attention(self, q, q_bs, ldq, k, v, kv_bs, ldkv, kv_hs, null_kv, mask, B, heads, n, m, out, o_bs, ldo):
        return [_view(out, (B, heads, n - 1, 64), (o_bs, 64, ldo, 1))]

    def _writes_step_epilogue(self, x_t, eps_cond, eps_null, cond_scale, t, tab_a, tab_b, c1, c2, sigma, noise, B, n,
                              rank_lo, rank_hi, weight, min_s, out, s_out=None):
        return [_view(out, (B * n - 1,), (1,)), _view(s_out, (B,), (1,))]


def test_a_narrower_footprint_fails_on_the_native_writes(native):
    fp = _Narrow(native, strict=False)
    g = torch.Generator().manual_seed(1)
    rn = lambda *s, dt=torch.float32: torch.randn(*s, generator=g).to(dt).cuda()
    F16 = torch.float16
    B, H, W, C = 2, 8, 200, 64
    fp.conv_igemm(rn(B, H, W, C, dt=F16), B, H, W, C, 0, C, rn(C, 9 * C, dt=F16), C, 3, 3, 0, rn(C), rn(B, H, W, C), None,
                  torch.empty(B, H, W, C, dtype=F16, device="cuda"), (H * W * C, W * C, C),
                  out_stats=torch.zeros(B, C // 16, 2, dtype=torch.float64, device="cuda"))
    B, heads, n, m = 2, 2, 70, 77
    ldo = heads * 64 + 64
    o_bs = n * ldo + 192
    kv = rn(B, m, 2 * heads * 64, dt=F16)
    out = torch.empty((B - 1) * o_bs + (heads - 1) * 64 + (n - 1) * ldo + 64, dtype=F16, device="cuda")
    fp.attention(rn(B, n, heads * 64, dt=F16), n * heads * 64, heads * 64, kv, kv[..., heads * 64:], m * 2 * heads * 64,
                 2 * heads * 64, 64, rn(2, 64), None, B, heads, n, m, out, o_bs, ldo)
    from minimagen_b200.Imagen import quantile_rank
    from minimagen_b200.diffusion_model import GaussianDiffusion
    gd = GaussianDiffusion(timesteps=50)
    sch = gd.sampling_schedule(10, 0.5, "cuda")
    B, n = 3, 3 * 17 * 17
    lo, hi, wq = quantile_rank(n, 0.9)
    fp.step_epilogue(rn(B, n), rn(B, n), rn(B, n), 3., torch.tensor([sch.grid[1], sch.grid[4], 0]).cuda(),
                     gd.sqrt_recip_alphas_cumprod.cuda(), gd.sqrt_recipm1_alphas_cumprod.cuda(), sch.c1, sch.c2, sch.sigma,
                     rn(B, n), B, n, lo, hi, wq, 1.0, torch.empty(B, n, device="cuda"),
                     s_out=torch.empty(B, device="cuda"))
    print("\n" + "\n".join(fp.failures))
    want = {"conv_igemm": "element [0, 0, 199, 0] of `out_f16`",      # column W - 1 of image 0's first row
            "attention": f"element [{69 * ldo}] of `out`",              # query row n - 1 of image 0, head 0
            "step_epilogue": f"element [{B - 1}, {n - 1}] of `out`"}   # the last element
    for method, element in want.items():
        hits = [f for f in fp.failures if f.startswith(method + ":")]
        assert len(hits) == 1 and "storage outside the footprint" in hits[0] and element in hits[0], (method, hits)
    assert len(fp.failures) == 3


# ------------------------------------------------------------------------------------------------ coverage
def test_every_kernel_method_was_footprint_checked():
    """Runs last: across this file's cases, every kernel-launching method of NativeOps was footprint-checked."""
    from minimagen_b200.ops import NativeOps
    methods = {n for n, _ in inspect.getmembers(NativeOps, inspect.isfunction) if not n.startswith("_")} - ALLOWED
    missing = sorted(methods - COVERED)
    print(f"\n{len(COVERED & methods)} of {len(methods)} kernel-launching methods footprint-checked")
    assert not missing, f"kernel methods no case of this file footprint-checked: {missing}"
