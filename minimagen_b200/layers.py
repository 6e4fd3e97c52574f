"""Building blocks of the U-Net, H100-native.

Every class keeps the NAME, constructor signature, sub-module attribute names and parameter shapes of its counterpart
in the reference's `minimagen/layers.py` (so `state_dict()` keys are identical -- the checkpoint ABI), but none of the
reference's torch forward code: each module lowers itself onto the sm_90a kernels through `run(...)`, which works on
NHWC fp32 activations `[B, H, W, C]` and makes C-ABI calls via `minimagen_b200.ops`.

`forward(...)` keeps the reference's NCHW (or `[b, n, c]` for attention) calling convention for stand-alone use and
simply wraps `run`.  Inference only: there is no autograd through the kernels (training is SURVEY.md 8f-2, "next").
"""
import math
import os

import torch
from torch import nn

from .helpers import default, exists
from .ops import get_ops

F16, F32, F64 = torch.float16, torch.float32, torch.float64


# ------------------------------------------------------------------------------------------------ plumbing
STATS_BLOCK = 16   # channels per GroupNorm block-statistics entry written by the conv epilogues

# GroupNorm INPUT precision on the tensor-core path.  True (default): GroupNorm reads the fp32 copy of its input, so the
# only fp16 roundings are the tensor-core operands themselves (measured 9e-4 rel-L2 on the cfg-3 network, inside the
# north star's 1e-3).  False: conv outputs that only feed a GroupNorm are kept in fp16 only (2 B instead of 4 B per
# element written and re-read; ~5 % faster steps) at 1.05e-3 rel-L2.
GN_INPUT_F32 = True

# Block.forward as ONE kernel (GroupNorm/FiLM/SiLU as the conv's prologue: mi_conv3x3_gn_silu_f16) where the geometry allows
# (3x3, H % 32 == 0, W % 8 == 0, channels % 64, C_out % 128, fp32 sources with epilogue block statistics)
# 'pair' : only the layers with C_out % 256 == 0 (the name is historical: every mode runs the same fused kernel, conv_tc.cu);
# True   : 'pair' plus the C_out == 128 layers;
# 'all'  : wherever supported; False: never.
FUSE_GN_CONV = {"0": False, "1": True, "pair": "pair", "all": "all"}.get(os.environ.get("MI_FUSE_GN_CONV", "0"), False)
# a ResnetBlock tail can either fold res_conv into block2's conv (FOLD_RES_CONV) or run block2 on the fused kernel; which wins
FUSE_OVER_FOLD = os.environ.get("MI_FUSE_OVER_FOLD", "1") == "1"


def fuse_block_ok(c_out):
    """Does the FUSE_GN_CONV policy select the fused kernel for a Block whose conv has `c_out` output channels?"""
    if not FUSE_GN_CONV:
        return False
    if FUSE_GN_CONV == 'all':
        return True
    return c_out % 256 == 0 or (FUSE_GN_CONV is True and c_out == 128)


# ResnetBlock tail  block2.project(h) + res_conv(x)  as ONE launch (mi_conv3x3_res1x1_f16: the 1x1 conv rides the 3x3 conv's
# accumulator as extra K chunks) where the geometry allows (mi_conv3x3_res1x1_supported)
FOLD_RES_CONV = os.environ.get("MI_FOLD_RES_CONV", "1") == "1"

# nearest-x2 upsample + 3x3 conv as four 2x2 sub-pixel convs on the low-res tensor (4/9 of the FLOPs, no upsampled copy)
SUBPIXEL_UPSAMPLE = True

# Downsample (4x4 stride 2) reads the producer's fp16 copy in place (TMA element strides) instead of a phase-split copy
INPLACE_DOWNSAMPLE = True


class ZeroArena:
    """One zero-filled fp64 buffer per forward pass from which the (many, tiny) GroupNorm statistics accumulators are
    carved, instead of one fill kernel per accumulator."""

    def __init__(self, device, n_doubles):
        self.buf = torch.zeros((n_doubles,), dtype=F64, device=device)
        self.off = 0

    def take(self, shape):
        n = 1
        for d in shape:
            n *= d
        if self.off + n > self.buf.numel():
            return None
        out = self.buf[self.off:self.off + n].view(shape)
        self.off += (n + 1) // 2 * 2      # keep 16-byte alignment
        return out


_ARENA = None


def stats_zeros(shape, device):
    if _ARENA is not None and _ARENA.buf.device == device:
        t = _ARENA.take(shape)
        if t is not None:
            return t
    return torch.zeros(shape, dtype=F64, device=device)


class Act:
    """One NHWC activation [B, H, W, C] of the U-Net: an fp32 copy (residual stream precision, only kept where an
    identity residual or a LayerNorm needs it), an fp16 copy (tensor-core / GroupNorm-apply operand) -- at least one of
    the two -- and optionally the GroupNorm block statistics [B, C/16, 2] (sum, sum of squares per 16 channels) that
    the producing conv epilogue accumulated."""
    __slots__ = ("f32", "f16", "stats")

    def __init__(self, f32=None, f16=None, stats=None):
        assert f32 is not None or f16 is not None
        self.f32, self.f16, self.stats = f32, f16, stats

    @property
    def any(self):
        return self.f32 if self.f32 is not None else self.f16

    @property
    def shape(self):
        sh = self.any.shape
        return (sh[0], sh[-3], sh[-2], sh[-1])

    @property
    def device(self):
        return self.any.device

    def need_f32(self):
        if self.f32 is None:
            B, H, W, C = self.shape
            self.f32 = torch.empty((B, H, W, C), dtype=F32, device=self.device)
            get_ops().cast_act(self.f16, C, None, 0, 1.0, B, H, W, 0, self.f32)
        return self.f32

    def need_f16(self):
        if self.f16 is None:
            B, H, W, C = self.shape
            self.f16 = torch.empty((B, 1, H, W, C), dtype=F16, device=self.device)
            get_ops().cast_act(self.f32, C, None, 0, 1.0, B, H, W, 0, self.f16)
        return self.f16

    def need_stats(self):
        """Block statistics by a stand-alone pass (tensors not produced by a conv epilogue, e.g. attention outputs)."""
        if self.stats is None:
            B, H, W, C = self.shape
            self.stats = stats_zeros((B, C // STATS_BLOCK, 2), self.device)
            get_ops().gn_stats(self.any, C, None, 0, 1.0, B, H * W, C // STATS_BLOCK, self.stats)
        return self.stats


def as_act(x):
    return x if isinstance(x, (Act, Cat)) else Act(f32=x)


class Cat:
    """Virtual channel concatenation cat(a, b * scale) of two activations (the up-path skip connection, reference
    Unet.py:445).  Never materialised in fp32: GroupNorm statistics combine the two sources' block statistics, the
    GroupNorm-apply / cast kernels read both sources, and 1x1 / 3x3 convs read them as two TMA sources."""

    def __init__(self, a, b, scale):
        a, b = as_act(a), as_act(b)
        assert a.shape[:3] == b.shape[:3]
        self.a, self.b, self.scale = a, b, float(scale)

    @property
    def shape(self):
        return (*self.a.shape[:3], self.a.shape[3] + self.b.shape[3])

    @property
    def device(self):
        return self.a.device


def _srcs(x, prefer_f16):
    """-> (src0, C0, src1, C1, scale1) with both sources in ONE dtype (fp16 if every source has it and it is preferred)"""
    parts = [x.a, x.b] if isinstance(x, Cat) else [x]
    use16 = prefer_f16 and all(p.f16 is not None for p in parts)
    if not use16 and not all(p.f32 is not None for p in parts):
        use16 = all(p.f16 is not None for p in parts)
        if not use16:
            for p in parts:
                p.need_f32()
    t = [(p.f16 if use16 else p.f32) for p in parts]
    if isinstance(x, Cat):
        return t[0], x.a.shape[3], t[1], x.b.shape[3], x.scale
    return t[0], x.shape[3], None, 0, 1.0


def _no_grad_check(*tensors):
    if torch.is_grad_enabled() and any(exists(t) and t.requires_grad for t in tensors):
        raise NotImplementedError(
            "minimagen_b200 implements the inference (sampling) hot path only; autograd through the sm_90a kernels "
            "(training, SURVEY.md 8f-2) is not built yet. Call under torch.no_grad().")


def to_nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def to_nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


class _PackCache:
    """fp16 tensor-core copy of a weight, rebuilt when the parameter changes (load_state_dict bumps `_version`)."""

    def __init__(self):
        self._key = None
        self._val = None

    def get(self, param, scale=1.0):
        key = (param.data_ptr(), param._version, str(param.device), float(scale))
        if key != self._key:
            self._val = get_ops().pack_conv_weight(param, scale)
            self._key = key
        return self._val


def _linear_rows(x_f32, x_f16, M, K, weight, pack, Nout, bias=None, residual=None, want_f16=False, scale=1.0):
    """Row-major linear layer out[M][Nout] = x[M][K] @ weight[Nout][K]^T (+bias)(+residual), `scale` folded into the
    weight.  Tensor-core implicit GEMM when (K, Nout) are tensor-core shaped, fp32 CUDA-core kernel otherwise.
    Exactly one of x_f32 / x_f16 is needed (the one matching the chosen path).  Returns fp16 if want_f16 else fp32."""
    ops = get_ops()
    dev = (x_f32 if x_f32 is not None else x_f16).device
    out = torch.empty((M, Nout), dtype=F16 if want_f16 else F32, device=dev)
    if x_f16 is not None:
        ops.conv_igemm(x_f16, 1, 1, M, K, 0, K, pack.get(weight, scale), Nout, 1, 1, 0, bias, residual,
                       None if want_f16 else out, out if want_f16 else None, (0, 0, Nout))
    else:
        w2 = weight.detach().reshape(Nout, K)
        ops.linear_f32(x_f32, M, K, w2, bias, Nout, 0, 0, residual, None if want_f16 else out,
                       out if want_f16 else None, scale)
    return out


def _tc_linear_ok(M, K, Nout):
    return get_ops().igemm_supported(1, M, K, Nout) and M >= 128


# ------------------------------------------------------------------------------------------------ simple modules
class Identity(nn.Module):
    """reference: layers.py:322-330"""

    def __init__(self, *args, **kwargs):
        super().__init__()

    def forward(self, x, *args, **kwargs):
        return x

    def run(self, x, *args, **kwargs):
        return x


class LayerNorm(nn.Module):
    """reference: layers.py:333-343 -- learnable gamma, beta is a zero *buffer* (part of the checkpoint)."""

    def __init__(self, dim):
        super().__init__()
        self.gamma = nn.Parameter(torch.ones(dim))
        self.register_buffer('beta', torch.zeros(dim))

    def run_rows(self, rows_f32, R, C, residual=None, out_dtype=F32, pre_gelu=False, both=False):
        """-> fp32 or fp16 [R, C]; with `both` -> (fp32, fp16)."""
        o32 = torch.empty((R, C), dtype=F32, device=rows_f32.device) if (both or out_dtype == F32) else None
        o16 = torch.empty((R, C), dtype=F16, device=rows_f32.device) if (both or out_dtype == F16) else None
        get_ops().ln_rows(rows_f32, R, C, self.gamma, self.beta, 1e-5, pre_gelu, residual, o32, o16)
        return (o32, o16) if both else (o32 if out_dtype == F32 else o16)

    def forward(self, x):
        _no_grad_check(x, self.gamma)
        C = x.shape[-1]
        return self.run_rows(x.reshape(-1, C).contiguous(), x.numel() // C, C).reshape(x.shape)


class ChanLayerNorm(nn.Module):
    """reference: layers.py:164-177 -- LayerNorm over the channel dim of an image == row LN in NHWC."""

    def __init__(self, dim, eps=1e-5):
        super().__init__()
        self.eps = eps
        self.g = nn.Parameter(torch.ones(1, dim, 1, 1))

    def run_rows(self, rows_f32, R, C, out_dtype=F32, pre_gelu=False):
        out = torch.empty((R, C), dtype=out_dtype, device=rows_f32.device)
        get_ops().ln_rows(rows_f32, R, C, self.g.detach().reshape(C), None, self.eps, pre_gelu, None,
                          out if out_dtype == F32 else None, out if out_dtype == F16 else None)
        return out

    def forward(self, x):
        _no_grad_check(x, self.g)
        B, C, H, W = x.shape
        return to_nchw(self.run_rows(to_nhwc(x).reshape(-1, C), B * H * W, C).reshape(B, H, W, C))


class SinusoidalPosEmb(nn.Module):
    """reference: layers.py:442-465"""

    def __init__(self, dim):
        super().__init__()
        self.dim = dim

    def forward(self, x):
        B = x.shape[0]
        out = torch.empty((B, self.dim), dtype=F32, device=x.device)
        get_ops().posemb(x.to(torch.int64).contiguous(), B, self.dim, out)
        return out


class Residual(nn.Module):
    """reference: layers.py:359-368"""

    def __init__(self, fn):
        super().__init__()
        self.fn = fn

    def forward(self, x, **kwargs):
        return self.fn(x, **kwargs) + x


class Parallel(nn.Module):
    """reference: layers.py:346-356 -- sum of parallel branches (last non-memory-efficient down layer,
    Unet.py:233-234: conv3x3(x) + conv1x1(x)).  Lowered as: second conv accumulates onto the first via the
    residual input of the conv epilogue."""

    def __init__(self, *fns):
        super().__init__()
        self.fns = nn.ModuleList(fns)

    def run(self, x):
        x = as_act(x)
        out = None
        for i, fn in enumerate(self.fns):
            last = i == len(self.fns) - 1
            out = fn.run(x, residual=out.f32 if exists(out) else None, f32=True, f16=last, stats=last)
        return out

    def forward(self, x):
        _no_grad_check(x)
        return to_nchw(self.run(to_nhwc(x)).need_f32())


class TokenView(nn.Module):
    """Stand-in for einops_exts.torch.EinopsToAndFrom('b c h w', 'b (h w) c', fn) (reference layers.py:403, :492,
    Unet.py:272).  In NHWC the rearrangement is a free view, so this only keeps the `fn` attribute name that the
    checkpoint keys (`...cross_attn.fn.*`, `...attn.fn.*`, `mid_attn.fn.fn.*`) depend on."""

    def __init__(self, fn):
        super().__init__()
        self.fn = fn

    def run(self, x, **kwargs):
        return self.fn.run(x, **kwargs)

    def forward(self, x, **kwargs):
        _no_grad_check(x)
        if "context" in kwargs and not isinstance(kwargs["context"], Context):
            kwargs["context"] = Context(kwargs["context"])
        return to_nchw(self.run(as_act(to_nhwc(x)), **kwargs).need_f32())


# ------------------------------------------------------------------------------------------------ convolutions
class Conv2d(nn.Conv2d):
    """nn.Conv2d parameter container (same keys / shapes) lowered onto the wgmma implicit GEMM
    (mi_conv2d_igemm_f16) or, for non-tensor-core shapes, the direct fp32 kernel (mi_conv2d_direct_f32).

    Supported geometries = the ones the reference U-Net uses: k x k stride 1 'same' padding (k odd), and the
    Downsample conv 4x4 / stride 2 / pad 1 (layers.py:319)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._pack = _PackCache()

    @property
    def _geom(self):
        kh, kw = self.kernel_size
        s, p = self.stride[0], self.padding[0]
        if s == 1 and kh == kw and kh % 2 == 1 and p == kh // 2:
            return 'same'
        if s == 2 and kh == 4 and kw == 4 and p == 1:
            return 'down'
        raise NotImplementedError(f"conv geometry k={self.kernel_size} s={self.stride} p={self.padding}")

    def tc_ok(self, H, W):
        """(H, W) = OUTPUT grid."""
        kh, kw = self.kernel_size
        return kh * kw <= 16 and get_ops().igemm_supported(H, W, self.in_channels, self.out_channels)

    def _pack_fold(self, rc, c0, scale):
        """[C_out][9*C_in + C_x] fp16: this 3x3 conv's packed weight followed by the 1x1 conv `rc`'s (input channels >= c0 of
        rc carry the skip-connection scale), and the summed bias -- the operands of mi_conv3x3_res1x1_f16."""
        key = (self.weight.data_ptr(), self.weight._version, rc.weight.data_ptr(), rc.weight._version, c0, float(scale),
               self.bias._version if exists(self.bias) else -1, rc.bias._version if exists(rc.bias) else -1)
        if getattr(self, "_fold_key", None) != key:
            ops = get_ops()
            w1 = rc.weight.detach().clone()
            if c0 is not None:
                w1[:, c0:] *= scale
            self._fold_w = torch.cat((ops.pack_conv_weight(self.weight), ops.pack_conv_weight(w1)), dim=1).contiguous()
            b = torch.zeros((self.out_channels,), dtype=F32, device=self.weight.device)
            if exists(self.bias):
                b = b + self.bias.detach()
            if exists(rc.bias):
                b = b + rc.bias.detach()
            self._fold_b = b.contiguous()
            self._fold_key = key
        return self._fold_w, self._fold_b

    def run_folded(self, a, B, H, W, xsrc, rc, residual=None, f32=True, f16=False, stats=False):
        """conv3x3(a) + rc(xsrc) in one launch (see FOLD_RES_CONV); a: fp16 [B,1,H,W,C_in]; xsrc: Act / Cat; rc: 1x1 Conv2d."""
        ops = get_ops()
        Cin, Cout = self.in_channels, self.out_channels
        dev = a.device
        cat = isinstance(xsrc, Cat)
        parts = [xsrc.a, xsrc.b] if cat else [xsrc]
        x0 = parts[0].need_f16()
        x1 = parts[1].need_f16() if cat else None
        c0 = parts[0].shape[3] if cat else None
        wp, bias = self._pack_fold(rc, c0, xsrc.scale if cat else 1.0)
        st = stats_zeros((B, Cout // STATS_BLOCK, 2), dev) if (stats and Cout % 32 == 0 and (H * W) % 32 == 0) else None
        if not f32 and not f16:
            f32 = True
        o32 = torch.empty((B, H, W, Cout), dtype=F32, device=dev) if f32 else None
        o16 = torch.empty((B, 1, H, W, Cout), dtype=F16, device=dev) if f16 else None
        ops.conv_res1x1(a, B, H, W, a.shape[-1], Cin, None, 0, 0, x0, x0.shape[-1], rc.in_channels, x1,
                        x1.shape[-1] if cat else 0, c0 if cat else 0, wp, Cout, bias, residual, o32, o16, st)
        return Act(o32, o16, st)

    def run_prepared(self, a, B, H, W, residual=None, f32=True, f16=False, stats=False, a2=None, c_in1=0, wp=None,
                     in_place_s2=False):
        """Conv over an already prepared operand `a`:
           tensor-core path: fp16 [B, P, H, W, C] (P = 4 phases for the stride-2 geometry), (H, W) = output grid;
                             optional second source `a2` (virtual concat: channels [c_in1, C_in) come from it);
           direct path:      fp32 [B, H_in, W_in, C_in].
        Returns an Act [B, H, W, C_out] (bias added, fp32 NHWC `residual` added) holding the requested copies; `stats`
        additionally accumulates the output's GroupNorm block statistics in the epilogue (tensor-core path only)."""
        ops = get_ops()
        Cin, Cout = self.in_channels, self.out_channels
        kh, kw = self.kernel_size
        strides = (H * W * Cout, W * Cout, Cout)
        dev = a.device
        if a.dim() == 5:      # the operand's layout, not its dtype, names the path
            assert a.dtype == F16
            # Downsample: 4-phase split operand (mode 1) or the fp16 activation read in place with TMA element strides (6)
            mode = (6 if in_place_s2 else 1) if self._geom == 'down' else 0
            # epilogue statistics credit a warp's 32 pixel rows to ONE image: needs whole images per 32-row slab
            st = stats_zeros((B, Cout // STATS_BLOCK, 2), dev) if (stats and Cout % 32 == 0 and (H * W) % 32 == 0) else None
            if not f32 and not f16:
                f32 = True
            o32 = torch.empty((B, H, W, Cout), dtype=F32, device=dev) if f32 else None
            o16 = torch.empty((B, 1, H, W, Cout), dtype=F16, device=dev) if f16 else None
            lda = a.shape[-1]
            ops.conv_igemm(a, B, H, W, lda, 0, Cin, wp if exists(wp) else self._pack.get(self.weight), Cout, kh, kw, mode,
                           self.bias, residual, o32, o16, strides, act2=a2, lda2=a2.shape[-1] if exists(a2) else 0,
                           c_in1=c_in1, out_stats=st)
            return Act(o32, o16, st)
        assert a.dtype == F32
        out = torch.empty((B, H, W, Cout), dtype=F32, device=dev)
        Hin, Win = a.shape[1], a.shape[2]
        ops.conv_direct(a, B, Hin, Win, Cin, a.shape[3], self.weight.detach(), Cout, kh, kw, self.stride[0],
                        self.padding[0], self.bias, residual, out, H, W, (*strides, 1))
        return Act(f32=out)

    def _run_subpixel(self, x, B, H, W, f32, f16, stats):
        """nn.Upsample(x2, nearest) + 3x3 conv (layers.py:513-514) as four 2x2 convs on the LOW-RES tensor: output pixel
        (2y+a, 2x+b) sees each low-res neighbour through the sum of the 3x3 taps that land on it.  No upsampled copy is
        ever written and the GEMM shrinks to 4/9 of the FLOPs; the four launches write the interleaved output directly."""
        ops = get_ops()
        Cin, Cout = self.in_channels, self.out_channels
        key = (self.weight.data_ptr(), self.weight._version)
        if getattr(self, "_sub_key", None) != key:
            w = self.weight.detach().to(F32)                                   # (O, I, 3, 3)
            rows = ((slice(0, 1), slice(1, 3)), (slice(0, 2), slice(2, 3)))    # phase a -> 3x3 rows folded onto r = 0 / 1
            self._sub_w = []
            for a in range(2):
                for b in range(2):
                    k = torch.stack([torch.stack([w[:, :, rows[a][r], rows[b][s]].sum(dim=(2, 3)) for s in range(2)], dim=-1)
                                     for r in range(2)], dim=-2)              # (O, I, 2, 2)
                    self._sub_w.append(ops.pack_conv_weight(k))
            self._sub_key = key
        dev = x.device
        Ho, Wo = 2 * H, 2 * W
        if not f32 and not f16:
            f32 = True
        st = stats_zeros((B, Cout // STATS_BLOCK, 2), dev) if (stats and Cout % 32 == 0 and (H * W) % 32 == 0) else None
        o32 = torch.empty((B, Ho, Wo, Cout), dtype=F32, device=dev) if f32 else None
        o16 = torch.empty((B, 1, Ho, Wo, Cout), dtype=F16, device=dev) if f16 else None
        a16 = x.need_f16()
        strides = (Ho * Wo * Cout, 2 * Wo * Cout, 2 * Cout)
        for p in range(4):
            off = ((p >> 1) * Wo + (p & 1)) * Cout
            ops.conv_igemm(a16, B, H, W, a16.shape[-1], 0, Cin, self._sub_w[p], Cout, 2, 2, 2 + p, self.bias, None,
                           o32.reshape(-1)[off:] if f32 else None, o16.reshape(-1)[off:] if f16 else None, strides,
                           out_stats=st)
        return Act(o32, o16, st)

    def _pack_cat(self, c0, scale):
        """Packed weight whose input-channel columns >= c0 (of every tap) carry the skip-connection scale."""
        key = (self.weight.data_ptr(), self.weight._version, c0, float(scale))
        if getattr(self, "_cat_key", None) != key:
            w = self.weight.detach().clone()
            w[:, c0:] *= scale
            self._cat_w = get_ops().pack_conv_weight(w)
            self._cat_key = key
        return self._cat_w

    def run_prepared_nchw(self, a, B, H, W, out=None):
        """Same-padding conv whose result is written straight to an NCHW fp32 tensor [B, C_out, H, W] (the U-Net's
        final_conv, Unet.py:327/:472).  Tensor-core path: C_out is zero-padded to a multiple of 16 in the packed
        weight and only the real channels are stored (n_valid)."""
        ops = get_ops()
        Cin, Cout = self.in_channels, self.out_channels
        kh, kw = self.kernel_size
        if out is None:
            out = torch.empty((B, Cout, H, W), dtype=F32, device=a.device)
        if a.dim() == 5:
            assert a.dtype == F16
            Np = (Cout + 15) // 16 * 16
            key = (self.weight.data_ptr(), self.weight._version, self.bias._version if exists(self.bias) else -1)
            if getattr(self, "_nchw_key", None) != key:
                wp = torch.zeros((Np, kh * kw * Cin), dtype=F16, device=a.device)
                wp[:Cout] = ops.pack_conv_weight(self.weight)
                bp = torch.zeros((Np,), dtype=F32, device=a.device)
                if exists(self.bias):
                    bp[:Cout] = self.bias.detach()
                self._nchw_w, self._nchw_b, self._nchw_key = wp, bp, key
            ops.conv_igemm(a, B, H, W, Cin, 0, Cin, self._nchw_w, Np, kh, kw, 0, self._nchw_b, None, out, None,
                           (Cout * H * W, W, 1), out_sc=H * W, n_valid=Cout)
        else:
            ops.conv_direct(a, B, H, W, Cin, a.shape[3], self.weight.detach(), Cout, kh, kw, 1, self.padding[0],
                            self.bias, None, out, H, W, (Cout * H * W, W, 1, H * W))
        return out

    def run(self, x, residual=None, upsample=False, f32=True, f16=False, stats=False):
        """x: Act / Cat (or a bare fp32 NHWC tensor).  `upsample` applies nn.Upsample(scale_factor=2, 'nearest') first
        (layers.py:513).  Returns an Act."""
        ops = get_ops()
        x = as_act(x)
        B, H, W, C = x.shape
        assert C == self.in_channels, (C, self.in_channels)
        geom = self._geom
        if upsample:
            assert geom == 'same'
            Ho, Wo = 2 * H, 2 * W
        elif geom == 'down':
            Ho, Wo = H // 2, W // 2
        else:
            Ho, Wo = H, W
        kw = dict(residual=residual, f32=f32, f16=f16, stats=stats)
        if upsample and SUBPIXEL_UPSAMPLE and not isinstance(x, Cat) and residual is None and self.kernel_size == (3, 3) \
                and get_ops().igemm_supported(H, W, C, self.out_channels):
            return self._run_subpixel(x, B, H, W, f32=f32, f16=f16, stats=stats)
        if self.tc_ok(Ho, Wo):
            if not upsample and geom == 'same':
                if isinstance(x, Cat):
                    c0 = x.a.shape[3]
                    if c0 % 64 == 0:      # two TMA sources, skip scale folded into the packed weight
                        return self.run_prepared(x.a.need_f16(), B, H, W, a2=x.b.need_f16(), c_in1=c0,
                                                 wp=self._pack_cat(c0, x.scale), **kw)
                else:
                    return self.run_prepared(x.need_f16(), B, H, W, **kw)
            if geom == 'down' and INPLACE_DOWNSAMPLE and not isinstance(x, Cat) and x.f16 is not None:
                return self.run_prepared(x.f16, B, Ho, Wo, in_place_s2=True, **kw)
            s0, C0, s1, C1, sc = _srcs(x, True)
            mode = 1 if upsample else (2 if geom == 'down' else 0)
            a = torch.empty((B, 4 if mode == 2 else 1, Ho, Wo, C), dtype=F16, device=x.device)
            ops.cast_act(s0, C0, s1, C1, sc, B, H, W, mode, a)
            return self.run_prepared(a, B, Ho, Wo, **kw)
        if upsample or isinstance(x, Cat):
            s0, C0, s1, C1, sc = _srcs(x, False)
            a = torch.empty((B, Ho if upsample else H, Wo if upsample else W, C), dtype=F32, device=x.device)
            ops.cast_act(s0, C0, s1, C1, sc, B, H, W, 1 if upsample else 0, a)
        else:
            a = x.need_f32()
        return self.run_prepared(a, B, Ho, Wo, **kw)

    def forward(self, x):
        _no_grad_check(x, self.weight)
        return to_nchw(self.run(to_nhwc(x)).need_f32())


def Downsample(dim, dim_out=None):
    """reference: layers.py:308-319 -- 4x4 stride-2 pad-1 conv."""
    return Conv2d(dim, default(dim_out, dim), kernel_size=4, stride=2, padding=1)


class _UpsampleSeq(nn.Sequential):
    """nn.Sequential(nn.Upsample(x2, nearest), Conv2d 3x3) with the reference's key layout ('1.weight', '1.bias');
    lowered as ONE cast kernel (nearest x2 fused into the operand preparation) + one conv."""

    def run(self, x):
        # consumed only through the next up block's virtual concat: fp16 + statistics suffice on the tensor-core path
        return self[1].run(x, upsample=True, f32=GN_INPUT_F32, f16=True, stats=True)

    def forward(self, x):
        _no_grad_check(x)
        return to_nchw(self.run(to_nhwc(x)).need_f32())


def Upsample(dim, dim_out=None):
    """reference: layers.py:502-515"""
    return _UpsampleSeq(nn.Upsample(scale_factor=2, mode='nearest'), Conv2d(dim, default(dim_out, dim), 3, padding=1))


class CrossEmbedLayer(nn.Module):
    """reference: layers.py:254-305 -- parallel convs (k = 3/7/15 for the U-Net stem) whose outputs are channel
    concatenated.  Each conv writes straight into its channel slice of one NHWC buffer (no torch.cat)."""

    def __init__(self, dim_in, kernel_sizes, dim_out=None, stride=2):
        super().__init__()
        assert all((k % 2) == (stride % 2) for k in kernel_sizes)
        dim_out = default(dim_out, dim_in)
        kernel_sizes = sorted(kernel_sizes)
        num_scales = len(kernel_sizes)
        dim_scales = [int(dim_out / (2 ** i)) for i in range(1, num_scales)]
        dim_scales = [*dim_scales, dim_out - sum(dim_scales)]
        self.dim_in, self.dim_out, self.stride = dim_in, dim_out, stride
        self.convs = nn.ModuleList([
            Conv2d(dim_in, ds, k, stride=stride, padding=(k - stride) // 2) for k, ds in zip(kernel_sizes, dim_scales)])

    def stem_tc_ok(self, H, W):
        ks = [c.kernel_size[0] for c in self.convs]
        return (self.stride == 1 and self.dim_in <= 8 and max(ks) <= 15 and all(k % 2 == 1 for k in ks)
                and get_ops().igemm_supported(H, W, 128, self.dim_out))

    def _stem_weights(self):
        """All convs zero-embedded in one 15x15 window over 8 (zero-padded) channels, laid out for the 15-tap vertical
        implicit GEMM over the horizontally unrolled operand (see mi_stem_unroll_f16): [dim_out][r*128 + j*8 + c]."""
        key = tuple((c.weight.data_ptr(), c.weight._version, c.bias._version) for c in self.convs)
        if getattr(self, "_stem_key", None) != key:
            dev = self.convs[0].weight.device
            wm = torch.zeros((self.dim_out, 15, 16, 8), dtype=F32, device=dev)
            off = 0
            for conv in self.convs:
                k, n = conv.kernel_size[0], conv.out_channels
                lo = 7 - k // 2
                wm[off:off + n, lo:lo + k, lo:lo + k, :self.dim_in] = conv.weight.detach().permute(0, 2, 3, 1)
                off += n
            self._stem_w = wm.reshape(self.dim_out, 15 * 128).to(F16).contiguous()
            self._stem_b = torch.cat([c.bias.detach() for c in self.convs]).contiguous()
            self._stem_key = key
        return self._stem_w, self._stem_b

    def run_stem(self, x, lowres=None):
        """x (and optionally lowres_cond_img): NCHW fp32.  Returns NHWC fp32 [B, H, W, dim_out]."""
        ops = get_ops()
        B, Cx, H, W = x.shape
        Cl = lowres.shape[1] if exists(lowres) else 0
        assert Cx + Cl == self.dim_in
        x = x.to(F32).contiguous()
        lowres = lowres.to(F32).contiguous() if exists(lowres) else None
        if self.stem_tc_ok(H, W):
            a = torch.empty((B, 1, H, W, 128), dtype=F16, device=x.device)
            ops.stem_unroll(x, Cx, lowres, Cl, B, H, W, a)
            wp, bias = self._stem_weights()
            C = self.dim_out
            out = torch.empty((B, H, W, C), dtype=F32, device=x.device)
            out16 = torch.empty((B, 1, H, W, C), dtype=F16, device=x.device)
            st = stats_zeros((B, C // STATS_BLOCK, 2), x.device) if (C % 32 == 0 and (H * W) % 32 == 0) else None
            ops.conv_igemm(a, B, H, W, 128, 0, 128, wp, C, 15, 1, 0, bias, None, out, out16, (H * W * C, W * C, C),
                           out_stats=st)
            return Act(out, out16, st)
        cp = (self.dim_in + 3) // 4 * 4
        x_pad = torch.empty((B, H, W, cp), dtype=F32, device=x.device)
        ops.nchw_to_nhwc(x, Cx, lowres, Cl, B, H * W, cp, x_pad)
        return Act(f32=self.run_padded(x_pad, B, H, W))

    def run_padded(self, x_pad, B, H, W):
        """x_pad: fp32 NHWC [B, H, W, ld] holding dim_in channels (zero padded to ld). stride must be 1."""
        assert self.stride == 1
        ops = get_ops()
        out = torch.empty((B, H, W, self.dim_out), dtype=F32, device=x_pad.device)
        C = self.dim_out
        off = 0
        for conv in self.convs:
            k = conv.kernel_size[0]
            ops.conv_direct(x_pad, B, H, W, self.dim_in, x_pad.shape[3], conv.weight.detach(), conv.out_channels, k, k,
                            1, conv.padding[0], conv.bias, None, out[..., off:], H, W, (H * W * C, W * C, C, 1))
            off += conv.out_channels
        return out

    def forward(self, x):
        _no_grad_check(x)
        return to_nchw(self.run_stem(x).need_f32())


# ------------------------------------------------------------------------------------------------ ResNet
class Block(nn.Module):
    """reference: layers.py:107-145 -- GroupNorm -> (scale+1, shift) -> SiLU -> Conv2d 3x3.
    Lowered as: mi_gn_stats, mi_gn_apply_silu (writes the conv operand), conv with bias/residual epilogue."""

    def __init__(self, dim, dim_out, groups=8, norm=True):
        super().__init__()
        self.groupnorm = nn.GroupNorm(groups, dim) if norm else Identity()
        self.activation = nn.SiLU()
        self.project = Conv2d(dim, dim_out, 3, padding=1)

    def run(self, x, scale_shift=None, residual=None, f32=True, f16=False, stats=False, fold=None):
        """x: Act / Cat.  `fold` = (xsrc, res_conv): add res_conv(xsrc) inside the conv launch (ResnetBlock tail), or None.
        GroupNorm statistics come from the producers' epilogue block statistics when every source has
        (or can cheaply get) them and the groups are unions of 16-channel blocks; otherwise from one mi_gn_stats pass."""
        ops = get_ops()
        x = as_act(x)
        B, H, W, C = x.shape
        gn = self.groupnorm
        assert isinstance(gn, nn.GroupNorm), "Block(norm=False) is never instantiated by the U-Net"
        G = gn.num_groups
        Cg = C // G
        tc = self.project.tc_ok(H, W)
        parts = [x.a, x.b] if isinstance(x, Cat) else [x]
        block_mode = tc and Cg % STATS_BLOCK == 0 and all(p.shape[3] % STATS_BLOCK == 0 for p in parts)
        if (fold is None and block_mode and fuse_block_ok(self.project.out_channels)
                and all(p.f32 is not None for p in parts)
                and ops.conv_gn_supported(H, W, parts[0].shape[3], parts[1].shape[3] if len(parts) > 1 else 0,
                                          self.project.out_channels, G)):
            # one kernel: GroupNorm/FiLM/SiLU as the conv's shared-memory prologue (mi_conv3x3_gn_silu_f16)
            conv = self.project
            Cout = conv.out_channels
            dev = x.device
            if not f32 and not f16:
                f32 = True
            o32 = torch.empty((B, H, W, Cout), dtype=F32, device=dev) if f32 else None
            o16 = torch.empty((B, 1, H, W, Cout), dtype=F16, device=dev) if f16 else None
            st = stats_zeros((B, Cout // STATS_BLOCK, 2), dev) if stats else None
            p1 = parts[1] if len(parts) > 1 else None
            ops.conv_gn(parts[0].f32, parts[0].shape[3], p1.f32 if p1 else None, p1.shape[3] if p1 else 0,
                        x.scale if p1 else 1.0, B, H, W, G, parts[0].need_stats(), p1.need_stats() if p1 else None,
                        gn.weight, gn.bias, scale_shift, scale_shift.stride(0) if exists(scale_shift) else 0, gn.eps,
                        conv._pack.get(conv.weight), Cout, conv.bias, residual, o32, o16, st)
            return Act(o32, o16, st)
        s0, C0, s1, C1, sc = _srcs(x, tc and not GN_INPUT_F32)
        if block_mode:
            st0, sb0 = parts[0].need_stats(), STATS_BLOCK
            st1, sb1 = (parts[1].need_stats(), STATS_BLOCK) if len(parts) > 1 else (None, 0)
        else:
            st0 = stats_zeros((B, G, 2), x.device)
            ops.gn_stats(s0, C0, s1, C1, sc, B, H * W, G, st0)
            sb0, st1, sb1 = 0, None, 0
        a = torch.empty((B, 1, H, W, C) if tc else (B, H, W, C), dtype=F16 if tc else F32, device=x.device)
        ss_ld = scale_shift.stride(0) if exists(scale_shift) else 0
        ops.gn_apply_silu(s0, C0, s1, C1, sc, B, H * W, G, st0, sb0, st1, sb1, gn.weight, gn.bias, scale_shift, ss_ld,
                          gn.eps, a)
        if fold is not None:
            return self.project.run_folded(a, B, H, W, fold[0], fold[1], residual, f32=f32, f16=f16, stats=stats)
        return self.project.run_prepared(a, B, H, W, residual, f32=f32, f16=f16, stats=stats)

    def forward(self, x, scale_shift=None):
        _no_grad_check(x)
        ss = None
        if exists(scale_shift):
            scale, shift = scale_shift
            ss = torch.cat((scale.reshape(x.shape[0], -1), shift.reshape(x.shape[0], -1)), dim=1).contiguous()
        return to_nchw(self.run(to_nhwc(x), ss).need_f32())


class ResnetBlock(nn.Module):
    """reference: layers.py:371-439"""

    def __init__(self, dim, dim_out, *, cond_dim=None, time_cond_dim=None, groups=8):
        super().__init__()
        self.time_mlp = None
        if exists(time_cond_dim):
            self.time_mlp = nn.Sequential(nn.SiLU(), nn.Linear(time_cond_dim, dim_out * 2))
        self.cross_attn = None
        if exists(cond_dim):
            self.cross_attn = TokenView(CrossAttention(dim=dim_out, context_dim=cond_dim))
        self.block1 = Block(dim, dim_out, groups=groups)
        self.block2 = Block(dim_out, dim_out, groups=groups)
        self.res_conv = Conv2d(dim, dim_out, 1) if dim != dim_out else Identity()

    def run(self, x, time_emb=None, cond=None, scale_shift=None, out_f32=True):
        """x: Act / Cat; returns an Act (fp32 copy only if `out_f32`, needed when the consumer adds it as an identity
        residual or runs a LayerNorm on it); time_emb: [B, time_cond_dim] fp32; cond: conditioning context (see CrossAttention.run).
        `scale_shift`: this block's time_mlp output [B, 2*dim_out] if the caller already computed it (the U-Net batches
        the time_mlps of all its ResnetBlocks into one GEMM per step); otherwise it is computed here from `time_emb`."""
        ops = get_ops()
        B = x.shape[0]
        if not exists(scale_shift) and exists(self.time_mlp) and exists(time_emb):
            lin = self.time_mlp[1]
            scale_shift = torch.empty((B, lin.out_features), dtype=F32, device=time_emb.device)
            # SiLU -> Linear (layers.py:396-399); chunk(2, dim=1) = (scale, shift) is read in place by gn_apply
            ops.linear_f32(time_emb, B, lin.in_features, lin.weight, lin.bias, lin.out_features, 1, 0, None,
                           scale_shift, None)
        x = as_act(x)
        tc = self.block1.project.tc_ok(x.shape[1], x.shape[2]) and self.block2.project.tc_ok(x.shape[1], x.shape[2])
        attn = exists(self.cross_attn)
        # conv1's output feeds only GroupNorm 2 (fp16 + epilogue statistics) unless cross-attention reads it (fp32)
        keep32 = attn or not tc or GN_INPUT_F32
        h = self.block1.run(x, f32=keep32, f16=not keep32, stats=tc and not attn)
        if attn:
            assert exists(cond)
            h = self.cross_attn.run(h, context=cond)      # attn(h) + h
        if isinstance(self.res_conv, Identity):
            assert not isinstance(x, Cat)
            res = x.need_f32()
        else:
            _, H, W, _ = x.shape
            c2 = self.block2.project
            xparts = [x.a, x.b] if isinstance(x, Cat) else [x]
            fused_gn = FUSE_OVER_FOLD and fuse_block_ok(c2.out_channels) and ops.conv_gn_supported(
                H, W, c2.in_channels, 0, c2.out_channels, self.block2.groupnorm.num_groups)
            if (FOLD_RES_CONV and tc and not fused_gn and self.res_conv.kernel_size == (1, 1)
                    and all(p.shape[3] % 64 == 0 for p in xparts)
                    and ops.conv_res1x1_supported(H, W, c2.in_channels, c2.out_channels, self.res_conv.in_channels)):
                # res_conv(x) rides block2's conv launch: no separate 1x1 kernel, no fp32 round trip of the residual branch
                return self.block2.run(h, scale_shift, residual=None, f32=out_f32 or not tc, f16=tc, stats=tc,
                                       fold=(x, self.res_conv))
            res = self.res_conv.run(x, f32=True).f32
        return self.block2.run(h, scale_shift, residual=res, f32=out_f32 or not tc, f16=tc, stats=tc)

    def forward(self, x, time_emb=None, cond=None):
        _no_grad_check(x)
        ctx = Context(cond) if exists(cond) else None
        return to_nchw(self.run(to_nhwc(x), time_emb, ctx).need_f32())


# ------------------------------------------------------------------------------------------------ attention
class Context:
    """Conditioning tokens c [B, m, D] (fp32) plus lazily created fp16 copy for the tensor-core k/v projections."""

    def __init__(self, c_f32):
        self.f32 = c_f32.contiguous()
        self._f16 = None

    @property
    def f16(self):
        if self._f16 is None:
            B, m, D = self.f32.shape
            self._f16 = torch.empty((B * m, D), dtype=F16, device=self.f32.device)
            get_ops().cast_act(self.f32, D, None, 0, 1.0, 1, 1, B * m, 0, self._f16)
        return self._f16


class CrossAttention(nn.Module):
    """reference: layers.py:180-251.  8 heads x 64 (defaults; the U-Net never overrides them), context is NOT normed,
    a learned null key/value is prepended, q is scaled by dim_head**-0.5 (folded into the packed to_q weight)."""

    def __init__(self, dim, *, context_dim=None, dim_head=64, heads=8, norm_context=False):
        super().__init__()
        assert dim_head == 64, "the fused attention kernel is specialised for dim_head = 64 (the reference's constant)"
        self.scale = dim_head ** -0.5
        self.heads = heads
        inner_dim = dim_head * heads
        context_dim = default(context_dim, dim)
        self.norm = LayerNorm(dim)
        self.norm_context = LayerNorm(context_dim) if norm_context else Identity()
        self.null_kv = nn.Parameter(torch.randn(2, dim_head))
        self.to_q = nn.Linear(dim, inner_dim, bias=False)
        self.to_kv = nn.Linear(context_dim, inner_dim * 2, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim, bias=False), LayerNorm(dim))
        self._pq, self._pkv, self._po = _PackCache(), _PackCache(), _PackCache()

    def run(self, x, context, mask=None, residual=True):
        """x: NHWC [B, H, W, C] (tokens = pixels); context: Context; mask: uint8 [B, m] or None.  Returns attn(x) + x
        when `residual` (the `+ h` of ResnetBlock.forward, layers.py:435, is fused into the output LayerNorm kernel)."""
        ops = get_ops()
        x = as_act(x)
        B, H, W, C = x.shape
        n = H * W
        m, D = context.f32.shape[1], context.f32.shape[2]
        inner = self.heads * 64
        rows = x.need_f32().reshape(B * n, C)
        assert isinstance(self.norm_context, Identity)
        # q projection
        tc_q = _tc_linear_ok(B * n, C, inner)
        xn = self.norm.run_rows(rows, B * n, C, out_dtype=F16 if tc_q else F32)
        q = _linear_rows(None if tc_q else xn, xn if tc_q else None, B * n, C, self.to_q.weight, self._pq, inner,
                         want_f16=True, scale=self.scale)
        # k/v projection of the (un-normed) context
        tc_kv = _tc_linear_ok(B * m, D, 2 * inner)
        kv = _linear_rows(None if tc_kv else context.f32.reshape(B * m, D), context.f16 if tc_kv else None, B * m, D,
                          self.to_kv.weight, self._pkv, 2 * inner, want_f16=True)
        o = torch.empty((B * n, inner), dtype=F16, device=x.device)
        ops.attention(q, n * inner, inner, kv, kv[:, inner:], m * 2 * inner, 2 * inner, 64, self.null_kv, mask, B,
                      self.heads, n, m, o, n * inner, inner)
        # output projection (K = 512 is always tensor-core shaped) + LayerNorm + residual
        tc_o = _tc_linear_ok(B * n, inner, C)
        if tc_o:
            y = _linear_rows(None, o, B * n, inner, self.to_out[0].weight, self._po, C)
        else:
            y = _linear_rows(o.to(F32), None, B * n, inner, self.to_out[0].weight, self._po, C)
        o32, o16 = self.to_out[1].run_rows(y, B * n, C, residual=rows if residual else None, both=True)
        return Act(o32.reshape(B, H, W, C), o16.reshape(B, 1, H, W, C))

    def forward(self, x, context, mask=None):
        """Reference calling convention: x [b, n, dim], context [b, m, context_dim] -> [b, n, dim] (no residual)."""
        _no_grad_check(x, context)
        B, n, C = x.shape
        xx = x.contiguous().reshape(B, 1, n, C)
        mk = mask.to(torch.uint8).contiguous() if exists(mask) else None
        return self.run(xx, Context(context), mk, residual=False).f32.reshape(B, n, C)


class Attention(nn.Module):
    """reference: layers.py:14-104 -- multi-query self attention: `heads` query heads share ONE key/value head
    (to_kv: dim -> 2*64), learned null kv prepended.  `context` / `attn_bias` are never used by the U-Net."""

    def __init__(self, dim, *, dim_head=64, heads=8, context_dim=None):
        super().__init__()
        assert dim_head == 64, "the fused attention kernel is specialised for dim_head = 64 (Unet.py:86 ATTN_DIM_HEAD)"
        assert not exists(context_dim), "Attention(context_dim=...) is never instantiated by the U-Net"
        self.scale = dim_head ** -0.5
        self.heads = heads
        inner_dim = dim_head * heads
        self.norm = LayerNorm(dim)
        self.null_kv = nn.Parameter(torch.randn(2, dim_head))
        self.to_q = nn.Linear(dim, inner_dim, bias=False)
        self.to_kv = nn.Linear(dim, dim_head * 2, bias=False)
        self.to_context = None
        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim, bias=False), LayerNorm(dim))
        self._pq, self._pkv, self._po = _PackCache(), _PackCache(), _PackCache()

    def run(self, x, context=None, mask=None, residual=True):
        """x: NHWC [B, H, W, C].  Returns attn(x) (+ x when `residual`: TransformerBlock.forward layers.py:497 and the
        mid Residual(Attention), Unet.py:273)."""
        assert context is None
        ops = get_ops()
        x = as_act(x)
        B, H, W, C = x.shape
        n = H * W
        inner = self.heads * 64
        rows = x.need_f32().reshape(B * n, C)
        tc = _tc_linear_ok(B * n, C, inner) and _tc_linear_ok(B * n, C, 128)
        xn = self.norm.run_rows(rows, B * n, C, out_dtype=F16 if tc else F32)
        q = _linear_rows(None if tc else xn, xn if tc else None, B * n, C, self.to_q.weight, self._pq, inner,
                         want_f16=True, scale=self.scale)
        kv = _linear_rows(None if tc else xn, xn if tc else None, B * n, C, self.to_kv.weight, self._pkv, 128,
                          want_f16=True)
        o = torch.empty((B * n, inner), dtype=F16, device=x.device)
        ops.attention(q, n * inner, inner, kv, kv[:, 64:], n * 128, 128, 0, self.null_kv, mask, B, self.heads, n, n, o,
                      n * inner, inner)
        if _tc_linear_ok(B * n, inner, C):
            y = _linear_rows(None, o, B * n, inner, self.to_out[0].weight, self._po, C)
        else:
            y = _linear_rows(o.to(F32), None, B * n, inner, self.to_out[0].weight, self._po, C)
        o32, o16 = self.to_out[1].run_rows(y, B * n, C, residual=rows if residual else None, both=True)
        return Act(o32.reshape(B, H, W, C), o16.reshape(B, 1, H, W, C))

    def forward(self, x, context=None, mask=None, attn_bias=None):
        _no_grad_check(x)
        assert context is None and attn_bias is None
        B, n, C = x.shape
        mk = mask.to(torch.uint8).contiguous() if exists(mask) else None
        return self.run(x.contiguous().reshape(B, 1, n, C), mask=mk, residual=False).f32.reshape(B, n, C)


class _ResidualAttention(Residual):
    """Residual(Attention) for the optional mid attention (Unet.py:272-274); keeps the `fn` key."""

    def run(self, x):
        return self.fn.run(x, residual=True)


def ChanFeedForward(dim, mult=2):
    """reference: layers.py:148-161 (parameter container; lowered inside TransformerBlock.run)."""
    hidden_dim = int(dim * mult)
    return nn.Sequential(
        ChanLayerNorm(dim),
        Conv2d(dim, hidden_dim, 1, bias=False),
        nn.GELU(),
        ChanLayerNorm(hidden_dim),
        Conv2d(hidden_dim, dim, 1, bias=False))


class TransformerBlock(nn.Module):
    """reference: layers.py:468-499 -- x = attn(x) + x ; x = ff(x) + x"""

    def __init__(self, dim, *, heads=8, dim_head=32, ff_mult=2, context_dim=None):
        super().__init__()
        self.attn = TokenView(Attention(dim=dim, heads=heads, dim_head=dim_head, context_dim=context_dim))
        self.ff = ChanFeedForward(dim=dim, mult=ff_mult)

    def run(self, x, context=None):
        x = as_act(x)
        B, H, W, C = x.shape
        R = B * H * W
        x = self.attn.run(x, residual=True)
        ln1, conv1, _, ln2, conv2 = self.ff
        hid = conv1.out_channels
        rows = x.f32.reshape(R, C)
        tc1 = _tc_linear_ok(R, C, hid)
        y = ln1.run_rows(rows, R, C, out_dtype=F16 if tc1 else F32)
        h = _linear_rows(None if tc1 else y, y if tc1 else None, R, C, conv1.weight, conv1._pack, hid)
        tc2 = _tc_linear_ok(R, hid, C) and conv2.tc_ok(H, W)
        z = ln2.run_rows(h, R, hid, out_dtype=F16 if tc2 else F32, pre_gelu=True)       # GELU(erf) -> ChanLayerNorm
        if tc2:   # 1x1 conv in image geometry: fp32 + fp16 copies and GroupNorm statistics from the epilogue
            return conv2.run_prepared(z.reshape(B, 1, H, W, hid), B, H, W, residual=x.f32, f32=True, f16=True, stats=True)
        out = _linear_rows(z, None, R, hid, conv2.weight, conv2._pack, C, residual=rows)
        return Act(f32=out.reshape(B, H, W, C))

    def forward(self, x, context=None):
        _no_grad_check(x)
        return to_nchw(self.run(to_nhwc(x)).need_f32())
