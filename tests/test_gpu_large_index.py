"""Every kernel that touches a cfg-5 1024 x 1024 activation, past 2^31 elements, against float64.

Nothing limits the batch of a 1024-px stage.  One cfg-5 activation at 1024^2 x 256 channels has 2^28 elements per image, so
image 8 starts at element 2^31 (byte 2^32 in fp16): `Imagen.sample` reaches it with 9 images, or 5 under `cfg_batched`
guidance.  test_kernels_past_2_31_elements calls each such kernel once, directly, at B = 9 x 1024^2 x 256 (2.42 G elements:
4.5 GiB in fp16, 9 GiB in fp32), and compares images 0 (a 32-bit wrap writes there), 7 and 8 (either side of element
2^31; 8 is also the last) with their float64 references, computed in bands of rows (checking_ops._bands).

Where each kernel's index arithmetic widens to 64 bits (read before this test first ran on a GPU):
  * nchw_to_nhwc_kernel (csrc/elementwise.cu): the flat index i is long long from `(long long)blockIdx.x * blockDim.x`;
    pix, b and p are long long, so `(b * Ca + c) * HW + p` is 64-bit.
  * stem_unroll_kernel: b = blockIdx.z is long long, so both the NCHW reads `((b * Ca + c) * H + h) * W + ws` and the store
    offset `(((b * H + h) * W + w) * 16 + j) * 8` are 64-bit.
  * conv_wg_kernel (csrc/conv_tc.cu; the 3 x 3, the 15 x 1 stem conv, the stride-2 conv read in place (mode 6) or from
    phases (mode 1), the sub-pixel phases, the NCHW final conv): operands are read by TMA, whose tensor maps
    (encode_act) take cuuint64_t dimensions and byte strides, with the image as its own coordinate; the row-major epilogue
    forms `pix = (long long)b * out_sb + (long long)h * out_sh + (long long)w * out_sw` and adds `(long long)(n + e) *
    out_sc` for the strided (NCHW) store; the transposed epilogue's tile base is long long and only the offsets inside a
    tile are int, which transposed_ok bounds by INT32_MAX; statistics rows are `(long long)b_img * stats_blocks`.  The
    strides are long long from the C entry point (igemm_common) down.
  * cast_kernel: the flat index, pix, b and all four output pixel offsets opix are long long (the x2 upsample's base uses
    2LL * W); load_cat8 takes the pixel as long long.
  * gn_stats_kernel / gn_apply_silu_kernel: one CTA covers a chunk of one image's pixels (grid.y = image), and
    `pix_base = (long long)b * HW + p0` carries the image offset; the index inside a chunk is int (at most 16 K elements).
So no kernel here needed a fix; this test confirms the reading.  test_planted_wrap_fails_the_boundary_images shows on the
CPU, at a reduced size, that a kernel storing image 8 over image 0 fails these checks.
"""
import gc
import time

import pytest
import torch

from checking_ops import CheckingOps
from emu_ops import EmuOps

F16, F32, F64 = torch.float16, torch.float32, torch.float64
FREE_BYTES = 36 << 30           # the largest call (the 3x3 conv: fp16 input, fp32 residual, fp32 + fp16 outputs) holds
                                # 27 GiB at full size, the float64 references a few more (28 GiB peak on an H100)


def _run_calls(ops, B, H, W, C, dev, seed=0):
    """The calls, with activations [B, H, W, C] (H x W the 1024^2 level, C its channels)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *s, dtype=F32, scale=1.0: (torch.randn(*s, generator=g, device=dev) * scale).to(dtype)
    x32 = rnd(B, H, W, C)
    x16 = rnd(B, H, W, C, dtype=F16)
    w = lambda taps, c_out=C: rnd(c_out, taps * (C if taps != 15 else 128), dtype=F16, scale=0.03)
    bias = rnd(C)
    st = (H * W * C, W * C, C)
    zeros = lambda n: torch.zeros(B, n, 2, dtype=F64, device=dev)
    h2, w2 = H // 2, W // 2

    # NCHW fp32 -> NHWC (the x32 buffer read as [B, C, H W])
    out = torch.empty(B, H * W, C, device=dev)
    ops.nchw_to_nhwc(x32.view(B, C, H * W), C, None, 0, B, H * W, C, out)
    del out
    # the stem: unrolled 15-tap operand, then the 15 x 1 conv over its 128 channels
    img, low = rnd(B, 3, H, W), rnd(B, 3, H, W)
    a = torch.empty(B, H, W, 128, dtype=F16, device=dev)
    ops.stem_unroll(img, 3, low, 3, B, H, W, a)
    del img, low
    o32 = torch.empty(B, H, W, C, device=dev)
    ops.conv_igemm(a, B, H, W, 128, 0, 128, w(15), C, 15, 1, 0, bias, None, o32, None, st)
    del a
    # 3 x 3 C -> C with bias, residual, fp32 and fp16 outputs and statistics
    o16 = torch.empty(B, H, W, C, dtype=F16, device=dev)
    ops.conv_igemm(x16, B, H, W, C, 0, C, w(9), C, 3, 3, 0, bias, x32, o32, o16, st, out_stats=zeros(C // 16))
    del o32, o16
    # the stride-2 Downsample from 1024^2: read in place (mode 6), and from the four phases cast_act mode 2 writes (mode 1)
    sd = (h2 * w2 * C, w2 * C, C)
    d32 = torch.empty(B, h2, w2, C, device=dev)
    ops.conv_igemm(x16, B, h2, w2, C, 0, C, w(16), C, 4, 4, 6, bias, None, d32, None, sd, out_stats=zeros(C // 16))
    ph = torch.empty(B, 4, h2, w2, C, dtype=F16, device=dev)
    ops.cast_act(x32, C, None, 0, 1.0, B, H, W, 2, ph)
    ops.conv_igemm(ph, B, h2, w2, C, 0, C, w(16), C, 4, 4, 1, bias, None, d32, None, sd)
    del ph, d32
    # the Upsample onto 1024^2: four sub-pixel phases of a 512^2 operand into one interleaved output, shared statistics
    lo16 = x16.view(-1)[:B * h2 * w2 * C].view(B, h2, w2, C)
    o32 = torch.empty(B, H, W, C, device=dev)
    o16 = torch.empty(B, H, W, C, dtype=F16, device=dev)
    stats = zeros(C // 16)
    for p in range(4):
        off = ((p >> 1) * W + (p & 1)) * C
        ops.conv_igemm(lo16, B, h2, w2, C, 0, C, w(4), C, 2, 2, 2 + p, bias, None, o32.view(-1)[off:], o16.view(-1)[off:],
                       (H * W * C, 2 * W * C, 2 * C), out_stats=stats)
    del o32
    # the final conv C -> 3 (packed to 16 output channels), stored NCHW
    wf = w(9, 16)
    wf[3:] = 0
    fin = torch.empty(B, 3, H, W, device=dev)
    ops.conv_igemm(x16, B, H, W, C, 0, C, wf, 16, 3, 3, 0, torch.zeros(16, device=dev), None, fin, None, (3 * H * W, W, 1),
                   out_sc=H * W, n_valid=3)
    del fin
    # cast_act: fp32 -> fp16 (mode 0), the nearest x2 upsample of a 512^2 operand onto 1024^2 (mode 1)
    ops.cast_act(x32, C, None, 0, 1.0, B, H, W, 0, o16)
    ops.cast_act(x32.view(-1)[:B * h2 * w2 * C], C, None, 0, 1.0, B, h2, w2, 1, o16)
    del o16
    # GroupNorm: statistics of the fp32 activation, then the apply with FiLM, fp32 -> fp16 and fp16 -> fp32
    G = 8
    sums = zeros(G)
    ops.gn_stats(x32, C, None, 0, 1.0, B, H * W, G, sums)
    gamma, beta, ss = 1 + rnd(C, scale=0.1), rnd(C, scale=0.1), rnd(B, 2 * C, scale=0.1)
    y16 = torch.empty(B, H * W, C, dtype=F16, device=dev)
    ops.gn_apply_silu(x32, C, None, 0, 1.0, B, H * W, G, sums, 0, None, 0, gamma, beta, ss, 2 * C, 1e-5, y16)
    del y16
    s16 = zeros(G)
    ops.gn_stats(x16, C, None, 0, 1.0, B, H * W, G, s16)
    del x32
    y32 = torch.empty(B, H * W, C, device=dev)
    ops.gn_apply_silu(x16, C, None, 0, 1.0, B, H * W, G, s16, 0, None, 0, gamma, beta, ss, 2 * C, 1e-5, y32)


METHODS = {"nchw_to_nhwc", "stem_unroll", "conv_igemm", "cast_act", "gn_stats", "gn_apply_silu"}


def _images(B):
    return sorted({0, 7, 8, B - 1})


@pytest.mark.gpu
def test_kernels_past_2_31_elements(native):
    B, H, W, C = 9, 1024, 1024, 256
    assert B * H * W * C > 2 ** 31 and 8 * H * W * C == 2 ** 31
    gc.collect()
    torch.cuda.empty_cache()                                # what earlier tests left in the caching allocator is free
    free, total = torch.cuda.mem_get_info()
    if free < FREE_BYTES:
        reason = f"needs {FREE_BYTES / 2 ** 30:.0f} GiB free on the device, {free / 2 ** 30:.1f} of {total / 2 ** 30:.1f} GiB are"
        print(reason)
        pytest.skip(reason)
    props = torch.cuda.get_device_properties(0)
    proxy = CheckingOps(native, images=_images(B))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    _run_calls(proxy, B, H, W, C, "cuda")
    torch.cuda.synchronize()
    print(f"\nB = {B} x {H}x{W} x {C} ({B * H * W * C / 2 ** 30:.2f} Gi elements) on {props.name}: {time.time() - t0:.1f} s, "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB allocated; images {_images(B)} checked")
    proxy.report()
    for (name, b), r in sorted(proxy.per_image.items()):
        print(f"  {name:28s} image {b}   worst |err|/bound {r:.3g}")
    assert proxy.called == proxy.checked == METHODS
    assert {b for _, b in proxy.per_image} == set(_images(B))


# ------------------------------------------------------------------------------------------------ on the CPU
SMALL = (9, 32, 32, 64)         # B, H, W, C: the same calls, image 8 the last


def test_boundary_image_checks_pass_on_the_emulation():
    """The call list above, on the emulated backend at a reduced size: every call passes its checks."""
    B, H, W, C = SMALL
    proxy = CheckingOps(EmuOps(), sms=132, images=_images(B))
    _run_calls(proxy, B, H, W, C, "cpu")
    proxy.report()
    assert proxy.called == proxy.checked == METHODS
    assert {b for _, b in proxy.per_image} == set(_images(B))


def _wrap_image8(emu, method):
    """`method` storing image 8 over image 0 (what a 32-bit image offset that wraps at 2^31 does): image 0's output holds
    image 8's values and image 8's is never written.  Applied to every output of the method that is a whole contiguous
    [B, ...] tensor."""
    import inspect
    orig = getattr(emu, method)
    sig = inspect.signature(orig)
    B = SMALL[0]

    def f(*args, **kwargs):
        p = sig.bind(*args, **kwargs).arguments
        outs = [p[k] for k in ("out", "out_f32", "out_f16", "sums", "out_stats")
                if torch.is_tensor(p.get(k)) and p[k].is_contiguous() and p[k].numel() % B == 0
                and p[k].data_ptr() == p[k].untyped_storage().data_ptr()]
        kept = [o.reshape(B, -1)[8].clone() for o in outs]
        orig(*args, **kwargs)
        for o, k in zip(outs, kept):
            v = o.reshape(B, -1)
            v[0] = v[8]
            v[8] = k
    return f


@pytest.mark.parametrize("method", ["nchw_to_nhwc", "stem_unroll", "conv_igemm", "cast_act", "gn_stats", "gn_apply_silu"])
def test_planted_wrap_fails_the_boundary_images(method):
    B, H, W, C = SMALL
    emu = EmuOps()
    setattr(emu, method, _wrap_image8(emu, method))
    proxy = CheckingOps(emu, sms=132, images=_images(B), only={method}, strict=False)
    _run_calls(proxy, B, H, W, C, "cpu")
    with pytest.raises(AssertionError) as e:
        proxy.raise_failures()
    print(f"\n{method}: {len(proxy.failures)} failed calls: {str(e.value)[:200]}")
    assert all(f.startswith(method + "(") for f in proxy.failures)
