"""torch.autograd.Function wrappers of the C-ABI ops: the TRAINING side of the hot path (SURVEY.md 8f-2).

`Imagen.forward` / `_p_losses` (reference Imagen.py:512-650) back-propagate through `Unet.forward`; under grad mode the
U-Net runs `minimagen_b200.train_path.unet_forward_train`, which is built from the Functions below.  Each Function's forward
is the same kernel the sampling path uses (tensor-core implicit GEMM for tensor-core-shaped convs, fp32 kernels otherwise);
each backward calls the backward entry points of the ABI (csrc/backward.cu) -- or, for the data gradient of a tensor-core-
shaped 3x3 / 1x1 conv, the forward wgmma kernel itself on the flipped, in/out-transposed packed weight.

Activations here are plain fp32 NHWC tensors `[B, H, W, C]` (rows `[R, C]` for token ops); torch is only the tape.
"""
import torch

from .ops import get_ops

F16, F32, F64 = torch.float16, torch.float32, torch.float64

# The tensor-core routes are taken for CUDA tensors only; tests/test_training.py sets this to walk the same host logic
# (sub-pixel Downsample data gradient, padded Linear rows, weight-gradient geometry) through the emulated ops on the CPU.
ROUTE_TC_ON_CPU = False


def _c(t):
    return t.contiguous()


# Gradient operands of the fp16 backward routes.  An MSE-mean loss over b * 3 * H * W elements makes dL/dpred ~1e-5 and the
# gradients deeper in the network smaller still: below fp16's smallest normal (6.1e-5) a plain cast keeps a bit or two of
# each element.  So a gradient is cast as g * 2^k, with k chosen on the device from its amax (no host sync: the step stays
# capturable) so that the scaled amax lies in [2^13, 2^14), and the kernels' fp32 outputs (dx, dw) are multiplied by 2^-k.
# Powers of two are exact both ways.  _SCALES[device][e] = (2^k, 2^-k) for the biased fp32 exponent e of the amax, k =
# 140 - e clamped to [-126, 126] (both stay normal fp32).
_SCALES = {}


def _grad_scales(g):
    """(2^k, 2^-k) as a 2-element fp32 device tensor for the gradient g (see above)."""
    tab = _SCALES.get(g.device)
    if tab is None:
        ks = [min(126, max(-126, 140 - e)) for e in range(256)]
        tab = _SCALES[g.device] = torch.tensor([[2.0 ** k, 2.0 ** -k] for k in ks], dtype=torch.float32, device=g.device)
    amax = torch.linalg.vector_norm(g, float("inf")).float().reshape(1)
    return torch.index_select(tab, 0, (amax.view(torch.int32) >> 23) & 255)[0]


def _cast_grad16(ops, g, C, B, H, W, out):
    """out <- fp16(g * 2^k) through cast_act (mode 0); returns 2^-k, the factor of the outputs computed from `out`."""
    s = _grad_scales(g)
    ops.cast_act(g * s[0], C, None, 0, 1.0, B, H, W, 0, out)
    return s[1]


class Conv2dFn(torch.autograd.Function):
    """y = conv2d(x, weight, bias) for the reference's geometries: k x k stride 1 'same' (k odd), and any (k, stride, pad)
    on the fp32 path.  x: [B, H, W, C_in] fp32 NHWC; weight: (C_out, C_in, kh, kw); returns [B, Ho, Wo, C_out]."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, pad):
        ops = get_ops()
        x = _c(x)
        B, H, W, Cin = x.shape
        Cout, _, kh, kw = weight.shape
        Ho = (H + 2 * pad - kh) // stride + 1
        Wo = (W + 2 * pad - kw) // stride + 1
        same = stride == 1 and kh == kw and kh % 2 == 1 and pad == kh // 2
        down = stride == 2 and kh == 4 and kw == 4 and pad == 1
        tc = (same or down) and kh * kw <= 16 and ops.igemm_supported(Ho, Wo, Cin, Cout) and (x.is_cuda or ROUTE_TC_ON_CPU)
        y = torch.empty((B, Ho, Wo, Cout), dtype=F32, device=x.device)
        strides = (Ho * Wo * Cout, Wo * Cout, Cout)
        w = weight.detach()
        b = bias.detach() if bias is not None else None
        if tc:
            a16 = torch.empty((B, 1, H, W, Cin), dtype=F16, device=x.device)
            ops.cast_act(x, Cin, None, 0, 1.0, B, H, W, 0, a16)
            ops.conv_igemm(a16, B, Ho, Wo, Cin, 0, Cin, ops.pack_conv_weight(w), Cout, kh, kw, 6 if down else 0, b, None, y, None,
                           strides)
        else:
            xp, ld = x, Cin
            if Cin % 4:                                   # the direct kernel reads channel quads
                ld = (Cin + 3) // 4 * 4
                xp = torch.zeros((B, H, W, ld), dtype=F32, device=x.device)
                xp[..., :Cin] = x
            ops.conv_direct(xp, B, H, W, Cin, ld, _c(w), Cout, kh, kw, stride, pad, b, None, y, Ho, Wo, (*strides, 1))
        ctx.save_for_backward(x, weight)
        ctx.geom = (stride, pad, same, down, tc, bias is not None)
        # the fp16 copy of x is the weight-gradient kernel's operand too: keep it instead of casting x again in backward
        ctx.x16 = a16 if tc and ops.conv_wgrad_tc_supported(Ho, Wo, Cin, Cout, kh, kw, stride) else None
        return y

    @staticmethod
    def backward(ctx, dy):
        ops = get_ops()
        x, weight = ctx.saved_tensors
        stride, pad, same, down, tc, has_bias = ctx.geom
        dy = _c(dy)
        B, H, W, Cin = x.shape
        _, Ho, Wo, Cout = dy.shape
        kh, kw = weight.shape[2], weight.shape[3]
        w = weight.detach()
        dx = dw = db = None
        g16 = inv = None

        def dy16():
            nonlocal g16, inv
            if g16 is None:
                g16 = torch.empty((B, 1, Ho, Wo, Cout), dtype=F16, device=dy.device)
                inv = _cast_grad16(ops, dy, Cout, B, Ho, Wo, g16)
            return g16

        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            if tc and same and Cout % 64 == 0 and Cin % 16 == 0 and ops.igemm_supported(H, W, Cout, Cin):
                # data gradient of a 'same' conv = the same conv of dy with the taps flipped and in/out channels swapped:
                # runs on the forward wgmma implicit-GEMM kernel
                g16 = dy16()
                ops.conv_igemm(g16, B, H, W, Cout, 0, Cout, ops.pack_conv_weight_dgrad(w), Cin, kh, kw, 0, None, None, dx, None,
                               (H * W * Cin, W * Cin, Cin))
                dx.mul_(inv)
            elif tc and down and Cout % 64 == 0 and Cin % 16 == 0 and ops.igemm_supported(Ho, Wo, Cout, Cin):
                # transposed 4x4 stride-2 conv = four 2x2 convs of dy, one per output parity (a, b): input pixel 2v + a sees
                # dy[v - 1], dy[v] through kernel rows 3, 1 (a = 0) or dy[v], dy[v + 1] through rows 2, 0 (a = 1) -- the tap
                # geometry of the sub-pixel phases of the forward kernel (modes 2..5), which write the interleaved dx in place
                taps = ((3, 1), (2, 0))
                g16 = dy16()
                for ph in range(4):
                    a, b = ph >> 1, ph & 1
                    # integer indexing only (an index list would build a CPU index tensor: not capturable in a CUDA graph)
                    k = torch.stack([torch.stack([w[:, :, ra, cb] for cb in taps[b]], dim=-1) for ra in taps[a]], dim=-2)
                    k = k.transpose(0, 1)                                                # (C_in, C_out, 2, 2)
                    off = (a * W + b) * Cin
                    ops.conv_igemm(g16, B, Ho, Wo, Cout, 0, Cout, ops.pack_conv_weight(_c(k)), Cin, 2, 2, 2 + ph, None, None,
                                   dx.reshape(-1)[off:], None, (H * W * Cin, 2 * W * Cin, 2 * Cin))
                dx.mul_(inv)
            else:
                ops.conv_dgrad(dy, B, Ho, Wo, Cout, _c(w), Cin, kh, kw, stride, pad, dx, H, W)
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(w, memory_format=torch.contiguous_format)
            if tc and (same or down) and ops.conv_wgrad_tc_supported(Ho, Wo, Cin, Cout, kh, kw, stride):
                # contraction over the pixels on wgmma: fp16 NHWC dy and x are both MN-major operands (csrc/wgrad_tc.cu)
                x16 = ctx.x16
                if x16 is None:
                    x16 = torch.empty((B, 1, H, W, Cin), dtype=F16, device=x.device)
                    ops.cast_act(x, Cin, None, 0, 1.0, B, H, W, 0, x16)
                ops.conv_wgrad_tc(dy16(), x16, B, Ho, Wo, Cin, Cout, kh, kw, dw, stride)
                dw.mul_(inv)
            elif same and Cout < 32 <= Cin:
                # few OUTPUT channels (the 3-channel final conv): sum over input pixels q instead,
                # dW[co][ci][t] = sum_q x[q][ci] * dy[q - (t - pad)][co] -- the same kernel with x and dy swapped computes
                # dW'[ci][co][t'] with t' the flipped tap, so its 32-wide tile axis is C_in (full) and the ragged 3-channel axis is
                # flattened with the taps instead of wasting 29/32 of a C_out tile
                dwt = torch.empty((Cin, Cout, kh, kw), dtype=F32, device=dy.device)
                ops.conv_wgrad(x, dy, B, H, W, Cout, H, W, Cin, kh, kw, 1, pad, dwt)
                dw = _c(dwt.flip(2, 3).transpose(0, 1))
            else:
                ops.conv_wgrad(dy, x, B, H, W, Cin, Ho, Wo, Cout, kh, kw, stride, pad, dw)
        if has_bias and ctx.needs_input_grad[2]:
            db = torch.empty((Cout,), dtype=F32, device=dy.device)
            ops.colsum(dy, B * Ho * Wo, Cout, db)
        return dx, dw, db, None, None


class GroupNormSiluFn(torch.autograd.Function):
    """Block.forward's front half (layers.py:136-144): SiLU(GroupNorm(x) * (scale + 1) + shift); x [B, H, W, C] fp32,
    scale_shift [B, 2C] = [scale | shift] or None."""

    @staticmethod
    def forward(ctx, x, gamma, beta, scale_shift, groups, eps):
        ops = get_ops()
        x = _c(x)
        B, H, W, C = x.shape
        sums = torch.zeros((B, groups, 2), dtype=F64, device=x.device)
        ops.gn_stats(x, C, None, 0, 1.0, B, H * W, groups, sums)
        y = torch.empty_like(x)
        ss = _c(scale_shift.detach()) if scale_shift is not None else None
        ops.gn_apply_silu(x, C, None, 0, 1.0, B, H * W, groups, sums, 0, None, 0, gamma.detach(), beta.detach(), ss,
                          2 * C if ss is not None else 0, eps, y)
        ctx.save_for_backward(x, sums, gamma, beta, ss if ss is not None else torch.empty(0, device=x.device))
        ctx.cfg = (groups, eps, ss is not None)
        return y

    @staticmethod
    def backward(ctx, dy):
        ops = get_ops()
        x, sums, gamma, beta, ss = ctx.saved_tensors
        groups, eps, has_ss = ctx.cfg
        B, H, W, C = x.shape
        dy = _c(dy)
        dx = torch.empty_like(x)
        dgamma = torch.zeros_like(gamma)
        dbeta = torch.zeros_like(beta)
        dss = torch.empty((B, 2 * C), dtype=F32, device=x.device) if has_ss else None
        ops.gn_silu_bwd(x, dy, sums, B, H * W, C, groups, gamma.detach(), beta.detach(), ss if has_ss else None,
                        2 * C if has_ss else 0, eps, dx, dgamma, dbeta, dss, 2 * C if has_ss else 0)
        return dx, dgamma, dbeta, dss, None, None


class LayerNormFn(torch.autograd.Function):
    """Row LayerNorm over the last dim (+ optional exact-erf GELU in front): layers.LayerNorm / ChanLayerNorm / nn.LayerNorm.
    beta may be None or a tensor (parameter or zero buffer)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps, pre_gelu):
        ops = get_ops()
        shp = x.shape
        C = shp[-1]
        rows = _c(x).reshape(-1, C)
        R = rows.shape[0]
        y = torch.empty_like(rows)
        g = _c(gamma.detach().reshape(C))
        ops.ln_rows(rows, R, C, g, _c(beta.detach()) if beta is not None else None, eps, bool(pre_gelu), None, y, None)
        ctx.save_for_backward(rows, g)
        ctx.cfg = (eps, bool(pre_gelu), shp, gamma.shape, beta is not None)
        return y.reshape(shp)

    @staticmethod
    def backward(ctx, dy):
        ops = get_ops()
        rows, g = ctx.saved_tensors
        eps, pre_gelu, shp, gshape, has_beta = ctx.cfg
        R, C = rows.shape
        dyr = _c(dy).reshape(R, C)
        dx = torch.empty_like(rows)
        dgamma = torch.zeros((C,), dtype=F32, device=rows.device) if ctx.needs_input_grad[1] else None
        dbeta = torch.zeros((C,), dtype=F32, device=rows.device) if (has_beta and ctx.needs_input_grad[2]) else None
        ops.ln_rows_bwd(rows, dyr, R, C, g, eps, pre_gelu, dx, dgamma, dbeta)
        return dx.reshape(shp), (dgamma.reshape(gshape) if dgamma is not None else None), dbeta, None, None


class LinearFn(torch.autograd.Function):
    """y = x @ W^T + b on rows; x [M, K] fp32, W the nn.Linear weight [N, K].  Tensor-core-shaped problems (M >= 256, K % 64 == 0,
    N % 16 == 0: the attention projections over image tokens and over the text / time context) run as 1x1 convs of a
    (Mp/128) x 128 "image" (Mp = M rounded up to 128 with zero rows) on the wgmma implicit-GEMM kernel with fp16 operands --
    forward, dX (transposed packed weight) and dW (contraction over the rows on the weight-gradient kernel, csrc/wgrad_tc.cu);
    everything else (time / text MLPs on B rows, ragged widths) stays fp32."""

    @staticmethod
    def _buf16(t, Mp, C):
        """the fp16 operand of M rows of t, zero-padded to Mp rows"""
        return (torch.empty if Mp == t.shape[0] else torch.zeros)((1, 1, Mp // 128, 128, C), dtype=F16, device=t.device)

    @staticmethod
    def _rows16(ops, t, M, Mp, C):
        a = LinearFn._buf16(t, Mp, C)
        ops.cast_act(t, C, None, 0, 1.0, 1, 1, M, 0, a)
        return a

    @staticmethod
    def forward(ctx, x, weight, bias):
        ops = get_ops()
        x = _c(x)
        M, K = x.shape
        Nn = weight.shape[0]
        Mp = (M + 127) // 128 * 128
        w = _c(weight.detach().reshape(Nn, K))
        b = bias.detach() if bias is not None else None
        tc = (x.is_cuda or ROUTE_TC_ON_CPU) and M >= 256 and K % 64 == 0 and Nn % 16 == 0 and ops.igemm_supported(Mp // 128, 128, K, Nn)
        if tc:
            y = torch.empty((Mp, Nn), dtype=F32, device=x.device)
            a16 = LinearFn._rows16(ops, x, M, Mp, K)
            ops.conv_igemm(a16, 1, Mp // 128, 128, K, 0, K, ops.pack_conv_weight(w), Nn, 1, 1, 0, b, None, y, None,
                           (Mp * Nn, 128 * Nn, Nn))
            y = y[:M]
            ctx.x16 = a16
        else:
            y = torch.empty((M, Nn), dtype=F32, device=x.device)
            ops.linear_f32(x, M, K, w, b, Nn, 0, 0, None, y, None)
        ctx.save_for_backward(x, w)
        ctx.cfg = (weight.shape, bias is not None, tc)
        return y

    @staticmethod
    def backward(ctx, dy):
        ops = get_ops()
        x, w = ctx.saved_tensors
        wshape, has_bias, tc = ctx.cfg
        dy = _c(dy)
        M, K = x.shape
        Nn = w.shape[0]
        Mp = (M + 127) // 128 * 128
        dx = dw = db = None
        g16 = inv = None
        if tc:
            g16 = LinearFn._buf16(dy, Mp, Nn)
            inv = _cast_grad16(ops, dy, Nn, 1, 1, M, g16)
        if ctx.needs_input_grad[0]:
            if g16 is not None and Nn % 64 == 0 and K % 16 == 0 and ops.igemm_supported(Mp // 128, 128, Nn, K):
                dx = torch.empty((Mp, K), dtype=F32, device=x.device)          # dX[M,K] = dY[M,N] W[N,K]
                ops.conv_igemm(g16, 1, Mp // 128, 128, Nn, 0, Nn, ops.pack_conv_weight_dgrad(w), K, 1, 1, 0, None, None, dx, None,
                               (Mp * K, 128 * K, K))
                dx = dx[:M].mul_(inv)
            else:
                dx = torch.empty_like(x)
                ops.gemm_f32(dy, w, dx, M, K, Nn, (Nn, 1), (K, 1), (K, 1))
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(w)                       # dW[N,K] = dY^T[N,M] X[M,K]
            if g16 is not None and ops.conv_wgrad_tc_supported(8, 8, K, Nn, 1, 1):
                ops.conv_wgrad_tc(g16, ctx.x16, Mp // 64, 8, 8, K, Nn, 1, 1, dw)
                dw.mul_(inv)
            else:
                ops.gemm_f32(dy, x, dw, Nn, K, M, (1, Nn), (K, 1), (K, 1))
            dw = dw.reshape(wshape)
        if has_bias and ctx.needs_input_grad[2]:
            db = torch.empty((Nn,), dtype=F32, device=dy.device)
            ops.colsum(dy, M, Nn, db)
        return dx, dw, db


class AttentionFn(torch.autograd.Function):
    """softmax(q k^T) v with the learned null key/value prepended (layers.py:65-99 multi-query, :228-248 cross attention).
    q [B, n, h*64] (already scaled by dim_head**-0.5); k, v [B, m, hk*64] with hk = h (cross) or 1 (multi-query);
    null_kv [2, 64].  fp32 throughout (scores materialised per (batch, head) by strided batched GEMMs)."""

    @staticmethod
    def forward(ctx, q, k, v, null_kv, heads):
        ops = get_ops()
        q, k, v = _c(q), _c(k), _c(v)
        B, n, inner = q.shape
        D = 64
        m = k.shape[1]
        hk = k.shape[2] // D
        L = m + 1
        nk = null_kv.detach()
        ke = torch.cat((nk[0].expand(B, hk, 1, D), k.reshape(B, m, hk, D).permute(0, 2, 1, 3)), dim=2).contiguous()
        ve = torch.cat((nk[1].expand(B, hk, 1, D), v.reshape(B, m, hk, D).permute(0, 2, 1, 3)), dim=2).contiguous()
        kb = (hk * L * D, L * D if hk > 1 else 0)
        P = torch.empty((B, heads, n, L), dtype=F32, device=q.device)
        ops.gemm_f32(q, ke, P, n, L, D, (inner, 1), (1, D), (L, 1), B, heads, (n * inner, D), kb, (heads * n * L, n * L))
        ops.softmax_rows(P, B * heads * n, L)
        o = torch.empty_like(q)
        ops.gemm_f32(P, ve, o, n, D, L, (L, 1), (D, 1), (inner, 1), B, heads, (heads * n * L, n * L), kb, (n * inner, D))
        ctx.save_for_backward(q, ke, ve, P)
        ctx.cfg = (heads, hk, m)
        return o

    @staticmethod
    def backward(ctx, do):
        ops = get_ops()
        q, ke, ve, P = ctx.saved_tensors
        heads, hk, m = ctx.cfg
        do = _c(do)
        B, n, inner = q.shape
        D, L = 64, m + 1
        kb = (hk * L * D, L * D if hk > 1 else 0)
        pb = (heads * n * L, n * L)
        qb = (n * inner, D)
        dP = torch.empty_like(P)                           # dP = dO V^T, then dS in place
        ops.gemm_f32(do, ve, dP, n, L, D, (inner, 1), (1, D), (L, 1), B, heads, qb, kb, pb)
        ops.softmax_rows_bwd(P, dP, B * heads * n, L)
        dq = torch.empty_like(q)                           # dq = dS K
        ops.gemm_f32(dP, ke, dq, n, D, L, (L, 1), (D, 1), (inner, 1), B, heads, pb, kb, qb)
        dke = torch.empty((B, heads, L, D), dtype=F32, device=q.device)      # per query head; summed below for multi-query
        dve = torch.empty_like(dke)
        hb = (heads * L * D, L * D)
        ops.gemm_f32(dP, q, dke, L, D, n, (1, L), (inner, 1), (D, 1), B, heads, pb, qb, hb)       # dK = dS^T q
        ops.gemm_f32(P, do, dve, L, D, n, (1, L), (inner, 1), (D, 1), B, heads, pb, qb, hb)       # dV = P^T dO
        if hk == 1:
            dke, dve = dke.sum(dim=1, keepdim=True), dve.sum(dim=1, keepdim=True)
        dnull = torch.stack((dke[:, :, 0].sum(dim=(0, 1)), dve[:, :, 0].sum(dim=(0, 1))))
        dk = dke[:, :, 1:].permute(0, 2, 1, 3).reshape(B, m, hk * D)
        dv = dve[:, :, 1:].permute(0, 2, 1, 3).reshape(B, m, hk * D)
        return dq, dk, dv, dnull, None


class Upsample2xFn(torch.autograd.Function):
    """nn.Upsample(scale_factor=2, mode='nearest') on NHWC (layers.py:513)."""

    @staticmethod
    def forward(ctx, x):
        ops = get_ops()
        x = _c(x)
        B, H, W, C = x.shape
        y = torch.empty((B, 2 * H, 2 * W, C), dtype=F32, device=x.device)
        ops.cast_act(x, C, None, 0, 1.0, B, H, W, 1, y)
        return y

    @staticmethod
    def backward(ctx, dy):
        ops = get_ops()
        dy = _c(dy)
        B, H2, W2, C = dy.shape
        dx = torch.empty((B, H2 // 2, W2 // 2, C), dtype=F32, device=dy.device)
        ops.upsample2x_bwd(dy, B, H2 // 2, W2 // 2, C, dx)
        return dx
