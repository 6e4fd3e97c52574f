"""TEST INFRASTRUCTURE ONLY: a torch (CPU) emulation of the `minimagen_b200.ops` interface.

It mirrors the CONTRACT of every C-ABI entry point (layouts, packing order, strides, fp16 operand rounding, in-place
output semantics) with plain torch ops, so that the host-side orchestration in minimagen_b200/{layers,Unet,Imagen}.py
can be executed -- and compared against the real reference -- on a box without a GPU.  The product never imports this
file; on a GPU box the native library is the only backend.  EmuOps has every public method of NativeOps, with the same
parameters; the module's `*_ref` functions are contracts the GPU tests also compare the native kernels against.

Two modes, chosen by the storage-dtype pair of the U-Net ops (the sampler's step ops are fp32 in both):

  EmuOps()                                       lo = fp16, hi = fp32: the kernels' storage types.  Tensor-core operands and
                                                 fp16 outputs are rounded (saturating) to fp16 like the kernels do, so a
                                                 network agrees with the fp32 reference at the operand-rounding level (~1e-3).
  EmuOps(lo=torch.float64, hi=torch.float64)     exact mode: no rounding and no saturation anywhere.  Together with the host
                                                 modules' dtype constants set to float64 (tests/test_lowering_exact.py) the
                                                 orchestration becomes a pure DATAFLOW: it must agree with a float64 run of the
                                                 reference restatement to ~1e-10 per element, whatever the network amplifies.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

import fp64_ref
import keyed_noise_restatement as K

F16, F32, F64 = torch.float16, torch.float32, torch.float64
KIND_NAMES = {v: k for k, v in K.KINDS.items()}


def _strided(out, shape, strides):
    return out.as_strided(shape, strides, out.storage_offset())


def _cat_src(src0, c0, src1, c1, scale1, lead_shape):
    a = src0.reshape(*lead_shape, c0)
    if src1 is None or c1 == 0:
        return a
    return torch.cat((a, src1.reshape(*lead_shape, c1) * scale1), dim=-1)


# ------------------------------------------------------------------------------------------------ step contracts
def _guided(eps_cond, eps_null, w, B, n):
    """The prediction [B, n] the step uses: eps_cond, or null + (cond - null) * w for a number or [B] fp32 weights."""
    e = eps_cond.reshape(B, n)
    if eps_null is None:
        return e
    if torch.is_tensor(w):
        assert w.dtype == F32 and w.numel() == B
        w = w.reshape(B, 1)
    nl = eps_null.reshape(B, n)
    return nl + (e - nl) * w


def _scheduled(eps_cond, eps_null, cond_scale, w_sched, t, B, n):
    """_guided at the weights w_b(t[b]) of the guidance table w_sched (None: w_b), formed by fp64_ref.scheduled_weights."""
    return _guided(eps_cond, eps_null, fp64_ref.scheduled_weights(cond_scale, w_sched, t, B).to(eps_cond.device), B, n)


def _x0(x_t, e, t, tab_a, tab_b, B, n):
    return tab_a[t][:, None] * x_t.reshape(B, n) - tab_b[t][:, None] * e


def _quantile(x0, B, n, rank_lo, rank_hi, weight, min_s):
    srt = x0.reshape(B, n).abs().sort(dim=-1).values
    # torch.quantile: a row containing NaN (sorted last) takes both order statistics from its last element -> NaN
    nan = srt[:, -1].isnan()
    lo = torch.where(nan, srt[:, -1], srt[:, rank_lo])
    hi = torch.where(nan, srt[:, -1], srt[:, rank_hi])
    return torch.lerp(lo, hi, torch.tensor(weight, dtype=F32)).clamp(min=min_s)


def _posterior(x0, s, x_t, noise, t, c1, c2, sigma, c3, hist, B, n):
    """(out, clamped x0) [B, n] from x0 [B, n] unclamped and the thresholds s [B]; with c3 and hist the multistep mean, whose
    c3 term is selected away, not multiplied, where c3[t] == 0."""
    sb = s[:, None]
    xs = x0.reshape(B, n).clamp(-sb, sb) / sb
    mean = c1[t][:, None] * xs + c2[t][:, None] * x_t.reshape(B, n)
    if c3 is not None:
        c3t = c3[t][:, None]
        mean = torch.where(c3t != 0, mean + c3t * hist.reshape(B, n), mean)
    sig = torch.where(t == 0, torch.zeros_like(sigma[t]), sigma[t])[:, None]
    return mean + sig * noise.reshape(B, n), xs


def _step(x_t, e, t, tab_a, tab_b, c1, c2, sigma, c3, noise, hist, B, n, rank_lo, rank_hi, weight, min_s, out, s_out):
    """The step epilogue from the prediction e [B, n]: x0 -> quantile -> posterior (out may alias x_t); with c3 and hist
    the multistep form, hist <- the clamped x0."""
    x0 = _x0(x_t, e, t, tab_a, tab_b, B, n)
    s = _quantile(x0, B, n, rank_lo, rank_hi, weight, min_s)
    res, xs = _posterior(x0, s, x_t, noise, t, c1, c2, sigma, c3, hist, B, n)
    if hist is not None:
        hist.copy_(xs.reshape(hist.shape))
    out.copy_(res.reshape(out.shape))
    if s_out is not None:
        s_out.copy_(s)


def multistep_ref(x0, s, x_t, noise, hist, t, c1, c2, sigma, c3, B, n):
    """Contract of mi_step_epilogue_multistep after the x0 prediction (x0 [B, n] unclamped) and the threshold s [B]:
    (out, new hist), op by op."""
    out, xs = _posterior(x0, s, x_t, noise, t, c1, c2, sigma, c3, hist, B, n)
    return out.reshape(x_t.shape), xs.reshape(hist.shape)


def prologue_ref(x, t, r, ra, rb, sqrt_acp, sqrt_1m_acp, k, m, z_renoise, z_known, T, B, C, hw):
    """Contract of mi_inpaint_prologue, op for op (x is returned, not modified)."""
    xv = x.reshape(B, C, hw)
    valid = ((t >= 0) & (t < T))[:, None, None]
    tc = t.clamp(0, T - 1)
    col = lambda tab: tab[tc][:, None, None]
    v = torch.where((r > 0)[:, None, None], col(ra) * xv + col(rb) * z_renoise.reshape(B, C, hw), xv)
    v = torch.where(m.reshape(B, 1, hw) >= 0.5, col(sqrt_acp) * k.reshape(B, C, hw) + col(sqrt_1m_acp) *
                    z_known.reshape(B, C, hw), v)
    return torch.where(valid, v, xv).reshape(x.shape)


def advance_ref(t, r, next_t, R, T):
    """Contract of mi_inpaint_advance: the new (t, r)."""
    valid = (t >= 0) & (t < T)
    rep = valid & (t > 0) & (r + 1 < R.reshape(-1)[0])
    nt = torch.where(valid, next_t[t.clamp(0, T - 1)], torch.zeros_like(t))
    return torch.where(rep, t, nt), torch.where(rep, r + 1, torch.zeros_like(r))


def finalize_ref(x, k, m, B, C, hw, unnormalize):
    v = torch.where(m.reshape(B, 1, hw) >= 0.5, k.reshape(B, C, hw), x.reshape(B, C, hw)).clamp(-1., 1.)
    return ((v + 1) * 0.5 if unnormalize else v).reshape(x.shape)


class EmuOps:
    name = "torch-emulation (tests only)"

    def __init__(self, lo=F16, hi=F32):
        self.lo, self.hi = lo, hi
        self.calls = []
        self.conv_log = []      # per host call: conv_igemm (mode, kh, kw, c_in, c_out); conv_res1x1 ('res1x1', two x sources, x_cin, c_in, c_out)
        self.keyed = []         # per randn_keyed call: (kind name, per-image labels, stage)

    def _sat16(self, y):
        """hi -> lo; fp32 -> fp16 saturates (csrc/sat_half.cuh): beyond +-65504 -> +-65504, not inf."""
        return y.clamp(-65504.0, 65504.0).to(F16) if self.lo == F16 else y.to(self.lo)

    def _log(self, name):
        self.calls.append(name)

    def set_launch_mode(self, pdl):
        """Launch modes are a property of the native kernels: nothing to emulate."""

    # ---------------------------------------------------------------- capability / weights
    def igemm_supported(self, H, W, c_in, c_out):
        def ilog2(v):
            l = int(math.log2(v)) if v > 0 else -1
            return l if (1 << l) == v else -1
        if c_in <= 0 or c_in % 64 or c_out <= 0 or c_out % 16:
            return False
        if W >= 128:
            return True
        if ilog2(W) < 3:
            return False
        bh = 128 // W
        if H >= bh:
            return H % bh == 0
        return ilog2(H) >= 0

    def pack_conv_weight(self, w, scale=1.0):
        self._log("pack")
        if w.dim() == 2:
            w = w[:, :, None, None]
        O, I, KH, KW = w.shape
        return (w.detach().to(self.hi) * scale).permute(0, 2, 3, 1).reshape(O, KH * KW * I).to(self.lo).contiguous()

    def pack_conv_weight_dgrad(self, w):
        if w.dim() == 2:
            w = w[:, :, None, None]
        return self.pack_conv_weight(w.detach().flip(2, 3).transpose(0, 1).contiguous())

    # ---------------------------------------------------------------- convolutions
    def conv_igemm(self, act, B, H, W, lda, c_off, c_in, wp, c_out, kh, kw, mode, bias, residual, out_f32, out_f16,
                   out_strides, block_n=0, out_sc=1, n_valid=0, act2=None, lda2=0, c_off2=0, c_in1=0, out_stats=None):
        self._log("conv_igemm")
        self.conv_log.append((mode, kh, kw, c_in, c_out))
        assert act.dtype == self.lo and wp.dtype == self.lo
        P = 4 if mode == 1 else 1
        if mode == 6:
            a = act.reshape(B, 2 * H, 2 * W, lda)[..., c_off:c_off + c_in].to(self.hi)
            w = wp.to(self.hi).reshape(c_out, kh, kw, c_in).permute(0, 3, 1, 2)
            y = F.conv2d(a.permute(0, 3, 1, 2), w, None, stride=2, padding=1).permute(0, 2, 3, 1)
            return self._conv_finish(y, B, H, W, c_out, bias, residual, out_f32, out_f16, out_strides, out_sc, n_valid,
                                     out_stats)
        if act2 is None:
            a = act.reshape(B, P, H, W, lda)[..., c_off:c_off + c_in].to(self.hi)
        else:
            a = torch.cat((act.reshape(B, P, H, W, lda)[..., c_off:c_off + c_in1].to(self.hi),
                           act2.reshape(B, P, H, W, lda2)[..., c_off2:c_off2 + (c_in - c_in1)].to(self.hi)), dim=-1)
        w = wp.to(self.hi).reshape(c_out, kh, kw, c_in).permute(0, 3, 1, 2)           # OIHW
        if mode == 0:
            y = F.conv2d(a[:, 0].permute(0, 3, 1, 2), w, None, stride=1, padding=(kh // 2, kw // 2))
        elif mode >= 2:
            # sub-pixel phase (pa, pb): taps (r, s) read low-res pixel (y + pa-1+r, x + pb-1+s)
            pa, pb = (mode - 2) >> 1, (mode - 2) & 1
            x = F.pad(a[:, 0].permute(0, 3, 1, 2), (1, 1, 1, 1))
            y = F.conv2d(x[:, :, pa:pa + H + 1, pb:pb + W + 1], w, None)
        else:
            # un-split the 4 phases back to the (2H, 2W) input: phase p = (h&1)*2 + (w&1)
            full = torch.zeros((B, 2 * H, 2 * W, c_in), dtype=self.hi)
            for p in range(4):
                full[:, (p >> 1)::2, (p & 1)::2] = a[:, p]
            y = F.conv2d(full.permute(0, 3, 1, 2), w, None, stride=2, padding=1)
        y = y.permute(0, 2, 3, 1)                                                 # B,H,W,Cout
        self._conv_finish(y, B, H, W, c_out, bias, residual, out_f32, out_f16, out_strides, out_sc, n_valid, out_stats)

    def _conv_finish(self, y, B, H, W, c_out, bias, residual, out_f32, out_f16, out_strides, out_sc, n_valid, out_stats):
        if bias is not None:
            y = y + bias
        sb, sh, sw = out_strides
        nv = n_valid if n_valid else c_out
        if residual is not None:
            assert out_sc == 1
            y = y + _strided(residual, (B, H, W, c_out), (sb, sh, sw, 1))
        if out_stats is not None:
            yb = y.double().reshape(B, H * W, c_out // 16, 16)
            out_stats[:, :, 0] += yb.sum(dim=(1, 3))
            out_stats[:, :, 1] += (yb * yb).sum(dim=(1, 3))
        y = y[..., :nv]
        if out_f32 is not None:
            _strided(out_f32, (B, H, W, nv), (sb, sh, sw, out_sc)).copy_(y)
        if out_f16 is not None:
            _strided(out_f16, (B, H, W, nv), (sb, sh, sw, out_sc)).copy_(self._sat16(y))

    def conv_res1x1_supported(self, H, W, c_in, c_out, x_cin):
        t16 = W == 16 and H % 16 == 0
        t32 = (not t16) and H % 32 == 0 and W % 8 == 0
        return (t16 or t32) and c_in > 0 and c_in % 64 == 0 and x_cin > 0 and x_cin % 64 == 0 and c_out % 128 == 0

    def conv_res1x1(self, act, B, H, W, lda, c_in, act2, lda2, c_in1, x, ldx, x_cin, x2, ldx2, x_cin1, wp, c_out, bias,
                    residual, out_f32, out_f16, out_stats):
        self._log("conv_res1x1")
        self.conv_log.append(("res1x1", x2 is not None, x_cin, c_in, c_out))
        K3 = 9 * c_in
        y = torch.zeros((B, H, W, c_out), dtype=self.hi)
        st = (H * W * c_out, W * c_out, c_out)
        self.conv_igemm(act, B, H, W, lda, 0, c_in, wp[:, :K3].contiguous(), c_out, 3, 3, 0, None, None, y, None, st,
                        act2=act2, lda2=lda2, c_in1=c_in1)
        self.calls.pop(), self.conv_log.pop()
        y1 = torch.zeros((B, H, W, c_out), dtype=self.hi)
        self.conv_igemm(x, B, H, W, ldx, 0, x_cin, wp[:, K3:].contiguous(), c_out, 1, 1, 0, None, None, y1, None, st,
                        act2=x2, lda2=ldx2, c_in1=x_cin1)
        self.calls.pop(), self.conv_log.pop()
        self._conv_finish(y + y1, B, H, W, c_out, bias, residual, out_f32, out_f16, st, 1, 0, out_stats)

    def conv_gn_supported(self, H, W, c0, c1, c_out, groups):
        C = c0 + c1
        return (H % 32 == 0 and W % 8 == 0 and c0 > 0 and c0 % 64 == 0 and c1 % 64 == 0 and C > 0 and c_out % 128 == 0
                and 1 <= groups <= 32 and C % groups == 0 and (C // groups) % 16 == 0)

    def conv_gn(self, src0, c0, src1, c1, scale1, B, H, W, groups, stats0, stats1, gamma, beta, scale_shift, ss_ld, eps,
                wp, c_out, bias, residual, out_f32, out_f16, out_stats):
        self._log("conv_gn")
        C = c0 + c1
        a = torch.zeros((B, 1, H, W, C), dtype=self.lo)
        self.gn_apply_silu(src0, c0, src1, c1, scale1, B, H * W, groups, stats0, 16, stats1, 16, gamma, beta, scale_shift,
                           ss_ld, eps, a)
        self.calls.pop()
        self.conv_igemm(a, B, H, W, C, 0, C, wp, c_out, 3, 3, 0, bias, residual, out_f32, out_f16,
                        (H * W * c_out, W * c_out, c_out), out_stats=out_stats)
        self.calls.pop(), self.conv_log.pop()

    def conv_direct(self, inp, B, Hin, Win, c_in, ldi, w, c_out, kh, kw, stride, pad, bias, residual, out, Hout, Wout,
                    out_strides):
        self._log("conv_direct")
        a = inp.reshape(B, Hin, Win, ldi)[..., :c_in].permute(0, 3, 1, 2)
        y = F.conv2d(a, w.detach().reshape(c_out, c_in, kh, kw), None, stride=stride, padding=pad).permute(0, 2, 3, 1)
        assert y.shape[1] == Hout and y.shape[2] == Wout
        if bias is not None:
            y = y + bias.detach()
        if residual is not None:
            y = y + _strided(residual, (B, Hout, Wout, c_out), out_strides)
        _strided(out, (B, Hout, Wout, c_out), out_strides).copy_(y)

    # ---------------------------------------------------------------- normalisation / casts
    def gn_stats(self, src0, c0, src1, c1, scale1, B, hw, groups, sums):
        self._log("gn_stats")
        x = _cat_src(src0.to(self.hi), c0, src1.to(self.hi) if src1 is not None else None, c1, scale1, (B, hw)).double()
        C = c0 + c1
        xg = x.reshape(B, hw, groups, C // groups)
        sums[:, :, 0] += xg.sum(dim=(1, 3))
        sums[:, :, 1] += (xg * xg).sum(dim=(1, 3))

    def gn_apply_silu(self, src0, c0, src1, c1, scale1, B, hw, groups, stats0, sb0, stats1, sb1, gamma, beta,
                      scale_shift, ss_ld, eps, out):
        self._log("gn_apply_silu")
        x = _cat_src(src0.to(self.hi), c0, src1.to(self.hi) if src1 is not None else None, c1, scale1, (B, hw))
        C = c0 + c1
        n = (C // groups) * hw
        if sb0 == 0:
            sums = stats0
        else:
            # per-channel-block sums of both sources -> per-channel-range sums of the concat -> groups
            parts = [stats0.reshape(B, c0 // sb0, 1, 2).expand(B, c0 // sb0, sb0, 2).reshape(B, c0, 2) / sb0]
            if c1:
                s1 = stats1.clone().reshape(B, c1 // sb1, 2)
                s1[..., 0] *= scale1
                s1[..., 1] *= scale1 * scale1
                parts.append(s1.reshape(B, c1 // sb1, 1, 2).expand(B, c1 // sb1, sb1, 2).reshape(B, c1, 2) / sb1)
            per_ch = torch.cat(parts, dim=1)                               # [B, C, 2] (block sums spread evenly)
            sums = per_ch.reshape(B, groups, C // groups, 2).sum(dim=2)
        mean = sums[:, :, 0] / n
        var = (sums[:, :, 1] / n - mean * mean).clamp(min=0)
        rstd = 1.0 / torch.sqrt(var + eps)
        mean_c = mean.to(self.hi).repeat_interleave(C // groups, dim=1)[:, None, :]
        rstd_c = rstd.to(self.hi).repeat_interleave(C // groups, dim=1)[:, None, :]
        y = (x - mean_c) * rstd_c * gamma.detach() + beta.detach()
        if scale_shift is not None:
            ss = scale_shift.as_strided((B, 2 * C), (ss_ld, 1), scale_shift.storage_offset())
            y = y * (ss[:, None, :C] + 1.0) + ss[:, None, C:]
        y = y * torch.sigmoid(y)
        out.reshape(B, hw, C).copy_(self._sat16(y) if out.dtype == self.lo else y)

    def cast_act(self, src0, c0, src1, c1, scale1, B, H, W, mode, out):
        self._log("cast_act")
        x = _cat_src(src0.to(self.hi), c0, src1.to(self.hi) if src1 is not None else None, c1, scale1, (B, H, W))
        C = c0 + c1
        if mode == 0:
            out.reshape(-1)[:B * H * W * C].reshape(B, H, W, C).copy_(x.to(out.dtype))     # the kernel writes the first B*H*W rows
        elif mode == 1:
            out.reshape(-1)[:4 * B * H * W * C].reshape(B, 2 * H, 2 * W, C).copy_(
                x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).to(out.dtype))
        else:
            o = out.reshape(-1)[:B * H * W * C].reshape(B, 4, H // 2, W // 2, C)
            for p in range(4):
                o[:, p].copy_(x[:, (p >> 1)::2, (p & 1)::2].to(out.dtype))

    def ln_rows(self, inp, rows, C, gamma, beta, eps, pre_gelu, residual, out_f32, out_f16):
        self._log("ln_rows")
        x = inp.reshape(rows, C)
        if pre_gelu:
            x = F.gelu(x)
        y = F.layer_norm(x, (C,), gamma.detach().reshape(C), beta.detach().reshape(C) if beta is not None else None, eps)
        if residual is not None:
            y = y + residual.reshape(rows, C)
        if out_f32 is not None:
            out_f32.reshape(rows, C).copy_(y)
        if out_f16 is not None:
            out_f16.reshape(rows, C).copy_(y.to(self.lo))

    # ---------------------------------------------------------------- conditioning
    def linear_f32(self, inp, M, K, W, bias, Nout, in_act, out_act, addend, out_f32, out_f16, out_scale=1.0):
        self._log("linear_f32")
        x = inp.reshape(M, K)
        if in_act == 1:
            x = F.silu(x)
        y = F.linear(x, W.detach().reshape(Nout, K), bias.detach() if bias is not None else None)
        if addend is not None:
            y = y + addend.reshape(M, Nout)
        if out_act == 1:
            y = F.silu(y)
        y = y * out_scale
        if out_f32 is not None:
            out_f32.reshape(M, Nout).copy_(y)
        if out_f16 is not None:
            out_f16.reshape(M, Nout).copy_(y.to(self.lo))

    def posemb(self, t, B, dim, out):
        self._log("posemb")
        half = dim // 2
        step = math.log(10000) / (half - 1)
        emb = torch.exp(torch.arange(half).to(self.hi) * -step)
        arg = t[:, None] * emb[None, :]
        out.copy_(torch.cat((arg.sin(), arg.cos()), dim=-1))

    def text_tokens(self, proj, B, L, D, mask, keep, null_embed, max_len, c_out, m, row_off, pooled):
        self._log("text_tokens")
        Lc = min(L, max_len)
        tok = torch.zeros((B, max_len, D), dtype=self.hi)
        tok[:, :Lc] = proj.reshape(B, L, D)[:, :Lc]
        cond = keep.bool()[:, None].expand(B, max_len).clone()
        if mask is not None:
            mk = torch.zeros((B, max_len), dtype=torch.bool)
            mk[:, :Lc] = mask.bool()[:, :Lc]
            cond = cond & mk
        o = torch.where(cond[:, :, None], tok, null_embed.detach().reshape(1, max_len, D))
        c_out.reshape(B, m, D)[:, row_off:row_off + max_len] = o
        pooled.copy_(o.mean(dim=1))

    def place_rows(self, src, B, r, D, dst, m, row_off):
        self._log("place_rows")
        dst.reshape(B, m, D)[:, row_off:row_off + r] = src.reshape(B, r, D)

    def select_rows(self, a, null_row, keep, addend, B, Nn, out):
        self._log("select_rows")
        y = torch.where(keep.bool()[:, None], a.reshape(B, Nn), null_row.detach().reshape(1, Nn))
        if addend is not None:
            y = y + addend.reshape(B, Nn)
        out.copy_(y)

    def nchw_to_nhwc(self, a, ca, b, cb, B, hw, c_pad, out):
        self._log("nchw_to_nhwc")
        o = out.reshape(B, hw, c_pad)
        o.zero_()
        o[:, :, :ca] = a.reshape(B, ca, hw).permute(0, 2, 1)
        if b is not None and cb:
            o[:, :, ca:ca + cb] = b.reshape(B, cb, hw).permute(0, 2, 1)

    def stem_unroll(self, a, ca, b, cb, B, H, W, out):
        self._log("stem_unroll")
        x = a if b is None or cb == 0 else torch.cat((a, b), dim=1)            # B,C,H,W
        C = x.shape[1]
        xp = F.pad(x, (7, 8))                                                   # w + j - 7, j in [0,16)
        o = torch.zeros((B, H, W, 16, 8), dtype=self.hi)
        for j in range(15):
            o[:, :, :, j, :C] = xp[:, :, :, j:j + W].permute(0, 2, 3, 1)
        out.reshape(B, H, W, 128).copy_(o.reshape(B, H, W, 128).to(self.lo))

    def resize_separable(self, inp, planes, hin, win, out, hout, wout, iy, wy, ix, wx, clamp=None):
        self._log("resize_separable")
        x = inp.reshape(planes, hin, win)
        rows = (x[:, iy.long(), :] * wy[None, :, :, None]).sum(2)            # planes, hout, win
        res = (rows[:, :, ix.long()] * wx[None, None, :, :]).sum(3)          # planes, hout, wout
        if clamp is not None:
            res = res.clamp(*clamp)
        out.reshape(planes, hout, wout).copy_(res)

    def silu(self, inp, out):
        self._log("silu")
        out.copy_(F.silu(inp))

    # ---------------------------------------------------------------- attention
    def attention(self, q, q_bs, ldq, k, v, kv_bs, ldkv, kv_hs, null_kv, mask, B, heads, n, m, out, o_bs, ldo):
        self._log("attention")
        qq = q.as_strided((B, heads, n, 64), (q_bs, 64, ldq, 1), q.storage_offset()).to(self.hi)
        kk = k.as_strided((B, heads, m, 64), (kv_bs, kv_hs, ldkv, 1), k.storage_offset()).to(self.hi)
        vv = v.as_strided((B, heads, m, 64), (kv_bs, kv_hs, ldkv, 1), v.storage_offset()).to(self.hi)
        nk = null_kv.detach()[0].to(self.lo).to(self.hi).reshape(1, 1, 1, 64).expand(B, heads, 1, 64)
        nv = null_kv.detach()[1].to(self.lo).to(self.hi).reshape(1, 1, 1, 64).expand(B, heads, 1, 64)
        kk = torch.cat((nk, kk), dim=2)
        vv = torch.cat((nv, vv), dim=2)
        sim = qq @ kk.transpose(-1, -2)
        if mask is not None:
            mk = F.pad(mask.bool(), (1, 0), value=True)[:, None, None, :]
            sim = sim.masked_fill(~mk, -torch.finfo(sim.dtype).max)
        attn = sim.softmax(dim=-1)
        o = attn @ vv                                                       # B,h,n,64
        out.as_strided((B, heads, n, 64), (o_bs, 64, ldo, 1), out.storage_offset()).copy_(o.to(self.lo))

    # ---------------------------------------------------------------- sampling step
    def step_x0(self, x_t, eps_cond, eps_null, cond_scale, t, tab_a, tab_b, B, n, x0):
        self._log("step_x0")
        x0.reshape(B, n).copy_(_x0(x_t, _guided(eps_cond, eps_null, cond_scale, B, n), t, tab_a, tab_b, B, n))

    def step_quantile(self, x0, B, n, rank_lo, rank_hi, weight, min_s, s):
        self._log("step_quantile")
        s.copy_(_quantile(x0, B, n, rank_lo, rank_hi, weight, min_s))

    def step_posterior(self, x0, x_t, noise, s, t, c1, c2, sigma, B, n, out):
        self._log("step_posterior")
        out.reshape(B, n).copy_(_posterior(x0, s, x_t, noise, t, c1, c2, sigma, None, None, B, n)[0])

    def step_epilogue(self, x_t, eps_cond, eps_null, cond_scale, t, tab_a, tab_b, c1, c2, sigma, noise, B, n, rank_lo,
                      rank_hi, weight, min_s, out, s_out=None):
        """contract of mi_step_epilogue (cond_scale a number) and mi_step_epilogue_w (a [B] tensor of per-image weights)"""
        self._log("step_epilogue")
        _step(x_t, _guided(eps_cond, eps_null, cond_scale, B, n), t, tab_a, tab_b, c1, c2, sigma, None, noise, None, B, n,
              rank_lo, rank_hi, weight, min_s, out, s_out)

    def step_epilogue_multistep(self, x_t, eps_cond, eps_null, cond_scale, t, tab_a, tab_b, c1, c2, sigma, c3, noise, hist,
                                B, n, rank_lo, rank_hi, weight, min_s, out, s_out=None):
        """contract of mi_step_epilogue_multistep(_w)"""
        self._log("step_epilogue_multistep")
        _step(x_t, _guided(eps_cond, eps_null, cond_scale, B, n), t, tab_a, tab_b, c1, c2, sigma, c3, noise, hist, B, n,
              rank_lo, rank_hi, weight, min_s, out, s_out)

    def step_epilogue_scheduled(self, x_t, eps_cond, eps_null, cond_scale, w_sched, t, tab_a, tab_b, c1, c2, sigma, noise, B,
                                n, rank_lo, rank_hi, weight, min_s, out, s_out=None):
        """contract of mi_step_epilogue_ws: step_epilogue at the weights w_b(t[b])"""
        self._log("step_epilogue_scheduled")
        _step(x_t, _scheduled(eps_cond, eps_null, cond_scale, w_sched, t, B, n), t, tab_a, tab_b, c1, c2, sigma, None,
              noise, None, B, n, rank_lo, rank_hi, weight, min_s, out, s_out)

    def step_epilogue_multistep_scheduled(self, x_t, eps_cond, eps_null, cond_scale, w_sched, t, tab_a, tab_b, c1, c2,
                                          sigma, c3, noise, hist, B, n, rank_lo, rank_hi, weight, min_s, out, s_out=None):
        """contract of mi_step_epilogue_multistep_ws: step_epilogue_multistep at the weights w_b(t[b])"""
        self._log("step_epilogue_multistep_scheduled")
        _step(x_t, _scheduled(eps_cond, eps_null, cond_scale, w_sched, t, B, n), t, tab_a, tab_b, c1, c2, sigma, c3,
              noise, hist, B, n, rank_lo, rank_hi, weight, min_s, out, s_out)

    def guidance_rescale_factor(self, eps_cond, eps_null, cond_scale, w_sched, t, phi, B, n, f):
        """contract of mi_guidance_rescale_factor: fp64 sums of squares about the mean, f rounded once to fp32"""
        self._log("guidance_rescale_factor")
        c = eps_cond.reshape(B, n).double()
        g = _scheduled(eps_cond, eps_null, cond_scale, w_sched, t, B, n).double()
        ssc = ((c - c.mean(dim=1, keepdim=True)) ** 2).sum(dim=1)
        ssg = ((g - g.mean(dim=1, keepdim=True)) ** 2).sum(dim=1)
        ph = phi.double()
        f.copy_(torch.where(ssg == 0, torch.ones_like(ssg), ph * (ssc / ssg).sqrt() + (1. - ph)).to(F32))

    def step_epilogue_rescaled(self, x_t, eps_cond, eps_null, cond_scale, w_sched, f, t, tab_a, tab_b, c1, c2, sigma, c3,
                               noise, hist, B, n, rank_lo, rank_hi, weight, min_s, out, s_out=None):
        """contract of mi_step_epilogue_rescaled: the step of fp32(g * f) without a guidance pass, g the guided prediction
        at w_b(t[b]); with c3 and hist the multistep form"""
        self._log("step_epilogue_rescaled")
        e = _scheduled(eps_cond, eps_null, cond_scale, w_sched, t, B, n) * f[:, None]
        _step(x_t, e, t, tab_a, tab_b, c1, c2, sigma, c3, noise, hist, B, n, rank_lo, rank_hi, weight, min_s, out, s_out)

    def step_advance_t(self, t, B):
        self._log("step_advance_t")
        t[:B] = (t[:B] - 1).clamp(min=0)                                   # the kernel advances t[:B] only

    def step_advance_t_table(self, t, next_t, T, B):
        self._log("step_advance_t_table")
        tb = t[:B]
        inside = (tb >= 0) & (tb < T)
        tb.copy_(torch.where(inside, next_t[tb.clamp(0, T - 1)], torch.zeros_like(tb)))

    def step_finalize(self, x, n, unnormalize, out):
        self._log("step_finalize")
        v = x.clamp(-1., 1.)
        out.copy_((v + 1) * 0.5 if unnormalize else v)

    def inpaint_prologue(self, x, t, r, ra, rb, sqrt_acp, sqrt_1m_acp, k, m, z_renoise, z_known, T, B, C, hw):
        self._log("inpaint_prologue")
        x.copy_(prologue_ref(x, t, r, ra, rb, sqrt_acp, sqrt_1m_acp, k, m, z_renoise, z_known, T, B, C, hw))

    def inpaint_advance(self, t, r, next_t, R, T, B):
        self._log("inpaint_advance")
        nt, nr = advance_ref(t[:B], r[:B], next_t, R, T)
        t[:B] = nt
        r[:B] = nr

    def inpaint_finalize(self, x, k, m, B, C, hw, unnormalize, out):
        self._log("inpaint_finalize")
        out.copy_(finalize_ref(x, k, m, B, C, hw, unnormalize))

    def q_sample(self, x0, noise, t, tab_a, tab_b, B, n, post_scale, post_shift, out):
        self._log("q_sample")
        v = tab_a[t][:, None] * x0.reshape(B, n) + tab_b[t][:, None] * noise.reshape(B, n)
        out.reshape(B, n).copy_(v * post_scale + post_shift)

    def randn_keyed(self, out, seeds, B, n, kind, stage, t=None, r=None, R=None, label=0):
        """contract of mi_randn_keyed: the restated generator (keyed_noise_restatement.py), rounded to fp32"""
        self._log("randn_keyed")
        assert seeds.dtype == torch.int64 and seeds.numel() >= B and out.dtype == torch.float32 and out.numel() == B * n
        if t is None:
            labels = [int(label)] * B
        else:
            labels = (t[:B] * (int(R[0]) if R is not None else 1) + (r[:B] if r is not None else 0)).tolist()
        self.keyed.append((KIND_NAMES[kind], labels, stage))
        z = K.randn_keyed(seeds.tolist()[:B], n, kind, stage, labels, np.float32)
        out.reshape(B, n).copy_(torch.from_numpy(z))


    # ---------------------------------------------------------------- training side (contracts of the backward entry points)
    def gemm_f32(self, A, B, C, M, N, K, a_str, b_str, c_str, Z1=1, Z2=1, a_b=(0, 0), b_b=(0, 0), c_b=(0, 0), alpha=1.0,
                 accumulate=False):
        self._log("gemm_f32")
        Av = A.as_strided((Z1, Z2, M, K), (a_b[0], a_b[1], a_str[0], a_str[1]), A.storage_offset())
        Bv = B.as_strided((Z1, Z2, K, N), (b_b[0], b_b[1], b_str[0], b_str[1]), B.storage_offset())
        Cv = C.as_strided((Z1, Z2, M, N), (c_b[0], c_b[1], c_str[0], c_str[1]), C.storage_offset())
        R = alpha * torch.matmul(Av, Bv)
        Cv.copy_(Cv + R if accumulate else R)

    def colsum(self, x, M, Nc, out, accumulate=False):
        self._log("colsum")
        r = x.reshape(M, Nc).sum(dim=0)
        out.copy_(out + r if accumulate else r)

    def conv_dgrad(self, dy, B, Ho, Wo, c_out, w, c_in, kh, kw, stride, pad, dx, Hi, Wi):
        self._log("conv_dgrad")
        g = torch.nn.grad.conv2d_input((B, c_in, Hi, Wi), w.detach().reshape(c_out, c_in, kh, kw),
                                       dy.reshape(B, Ho, Wo, c_out).permute(0, 3, 1, 2), stride=stride, padding=pad)
        dx.reshape(B, Hi, Wi, c_in).copy_(g.permute(0, 2, 3, 1))

    def conv_wgrad(self, dy, x, B, Hi, Wi, c_in, Ho, Wo, c_out, kh, kw, stride, pad, dw):
        self._log("conv_wgrad")
        g = torch.nn.grad.conv2d_weight(x.reshape(B, Hi, Wi, c_in).permute(0, 3, 1, 2), (c_out, c_in, kh, kw),
                                        dy.reshape(B, Ho, Wo, c_out).permute(0, 3, 1, 2), stride=stride, padding=pad)
        dw.reshape(c_out, c_in, kh, kw).copy_(g)

    def conv_wgrad_tc_supported(self, Ho, Wo, c_in, c_out, kh, kw, stride=1):
        geom = (stride == 1 and kh == kw and kh in (1, 3)) or (stride == 2 and kh == 4 and kw == 4)
        return Ho % 8 == 0 and Wo % 8 == 0 and c_in % 64 == 0 and c_out % 128 == 0 and geom

    def conv_wgrad_tc(self, dy16, x16, B, Ho, Wo, c_in, c_out, kh, kw, dw, stride=1):
        self._log("conv_wgrad_tc")
        pad = 1 if stride == 2 else kh // 2
        g = torch.nn.grad.conv2d_weight(x16.to(self.hi).reshape(B, stride * Ho, stride * Wo, c_in).permute(0, 3, 1, 2),
                                        (c_out, c_in, kh, kw), dy16.to(self.hi).reshape(B, Ho, Wo, c_out).permute(0, 3, 1, 2),
                                        stride=stride, padding=pad)
        dw.reshape(c_out, c_in, kh, kw).copy_(g)

    def gn_silu_bwd(self, x, dy, sums, B, hw, C, groups, gamma, beta, scale_shift, ss_ld, eps, dx, dgamma, dbeta, dss, dss_ld):
        self._log("gn_silu_bwd")
        with torch.enable_grad():
            x_ = x.detach().reshape(B, hw, C).clone().requires_grad_(True)
            g_ = gamma.detach().clone().requires_grad_(True)
            b_ = beta.detach().clone().requires_grad_(True)
            y = F.group_norm(x_.transpose(1, 2), groups, g_, b_, eps).transpose(1, 2)
            leaves = [x_, g_, b_]
            if scale_shift is not None:
                ss_ = torch.as_strided(scale_shift, (B, 2 * C), (ss_ld, 1), scale_shift.storage_offset()).detach().clone()
                ss_.requires_grad_(True)
                y = y * (ss_[:, None, :C] + 1) + ss_[:, None, C:]
                leaves.append(ss_)
            y = F.silu(y)
            grads = torch.autograd.grad(y, leaves, dy.reshape(B, hw, C))
        dx.reshape(B, hw, C).copy_(grads[0])
        dgamma.add_(grads[1])
        dbeta.add_(grads[2])
        if dss is not None:
            torch.as_strided(dss, (B, 2 * C), (dss_ld, 1), dss.storage_offset()).copy_(grads[3])

    def ln_rows_bwd(self, inp, dy, R, C, gamma, eps, pre_gelu, dx, dgamma, dbeta):
        self._log("ln_rows_bwd")
        with torch.enable_grad():
            x_ = inp.detach().reshape(R, C).clone().requires_grad_(True)
            g_ = gamma.detach().reshape(C).clone().requires_grad_(True)
            v = F.gelu(x_) if pre_gelu else x_
            y = F.layer_norm(v, (C,), None, None, eps) * g_
            gx, gg = torch.autograd.grad(y, [x_, g_], dy.reshape(R, C))
        dx.reshape(R, C).copy_(gx)
        if dgamma is not None:
            dgamma.reshape(C).add_(gg)
        if dbeta is not None:
            dbeta.reshape(C).add_(dy.reshape(R, C).sum(dim=0))

    def softmax_rows(self, s, R, L):
        self._log("softmax_rows")
        v = s.reshape(R, L)
        v.copy_(torch.softmax(v, dim=-1))

    def softmax_rows_bwd(self, P, dP, R, L):
        self._log("softmax_rows_bwd")
        p, d = P.reshape(R, L), dP.reshape(R, L)
        d.copy_(p * (d - (p * d).sum(dim=-1, keepdim=True)))

    def upsample2x_bwd(self, dy, B, H, W, C, dx):
        self._log("upsample2x_bwd")
        q = dy.reshape(B, H, 2, W, 2, C)
        dx.reshape(B, H, W, C).copy_((q[:, :, 0, :, 0] + q[:, :, 0, :, 1]) + (q[:, :, 1, :, 0] + q[:, :, 1, :, 1]))
