"""TEST INFRASTRUCTURE ONLY: float64 references of the token-side kernels, of the image-side forward kernels (implicit-GEMM,
direct and stem convolutions, the conv epilogue's GroupNorm statistics, GroupNorm statistics and GroupNorm/FiLM/SiLU, the
fused GroupNorm conv), of the image-side training kernels (GroupNorm/SiLU backward, convolution weight and data
gradients, upsample backward) and of the sampling loop's kernels outside the U-Net (the step epilogue's x0, threshold and
posterior, q_sample, the RePaint prologue, the scheduled guidance weights and the guidance-rescale factor, the cascade
resize, the timestep embedding and the text-token pooling) with elementwise error bounds.

Every reference takes the operands exactly as the kernel reads them (fp16-rounded where the kernel reads fp16, the null
key/value included), computes in float64 on the operands' device, and returns (reference, bound): |kernel - reference| <=
bound must hold for EVERY element.  A bound is derived from the kernel's own rounding steps (the derivation is in each
docstring) and has the general form

    c * n * u * twin + u_out * |ref|,        c <= 4,

with n the accumulation length (it may follow the kernel's documented summation structure), u the unit roundoff of the
accumulation (U32) or of an fp16 operand (U16), and `twin` the same expression evaluated on absolute values.  The
constants are fixed here and not tuned per test.  tests/test_error_bounds.py shows on the CPU that the torch emulation of
the kernels' contract passes every bound and that planted defects fail it.
"""
import math

import torch

U16 = 2.0 ** -11            # unit roundoff of fp16
U32 = 2.0 ** -24            # unit roundoff of fp32
ETA32 = 2.0 ** -147         # four fp32 subnormal spacings: absolute error of a few roundings in the underflow range
HALF_MAX = 65504.0
F64 = torch.float64


def _d(t):
    return None if t is None else t.detach().to(F64)


def _abs(t):
    return 0.0 if t is None else t.abs()


def check(out, ref, bound, what, sentinel=None):
    """Assert that `out` is finite, that |out - ref| <= bound elementwise and that the sentinel elements of the output
    buffer (bool mask of `out`'s shape, True = must still be NaN) were not written.  Prints -- and on failure reports --
    the worst element and its ratio |out - ref| / bound.  Returns that ratio."""
    o = out.detach().to(F64)
    ref = ref.to(o.device, F64).expand(o.shape)
    bound = torch.as_tensor(bound, dtype=F64, device=o.device).expand(o.shape)
    live = torch.ones(o.shape, dtype=torch.bool, device=o.device)
    if sentinel is not None:
        sentinel = sentinel.to(o.device)
        touched = int((~torch.isnan(o[sentinel])).sum())
        assert touched == 0, f"{what}: {touched} sentinel elements were overwritten"
        live = ~sentinel
    bad = live & ~torch.isfinite(o)
    assert not bad.any(), f"{what}: {int(bad.sum())} non-finite elements, first at {tuple(bad.nonzero()[0].tolist())}"
    err = torch.where(live, (o - ref).abs(), torch.zeros((), dtype=F64, device=o.device))
    ratio = err / bound.clamp(min=1e-300)
    worst = int(ratio.reshape(-1).argmax())
    idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), o.shape))
    r = float(ratio.reshape(-1)[worst])
    msg = (f"{what}: worst |err|/bound = {r:.3g} at {idx} (out {float(o[idx]):.9g}, ref {float(ref[idx]):.9g}, "
           f"bound {float(bound[idx]):.3g})")
    print(msg)
    assert r <= 1.0, msg
    return r


def check_rel_l2(out, ref, limit, what):
    """Assert ||out - ref|| / ||ref|| < limit over the whole tensor.  The elementwise bounds are worst cases: at long
    accumulations they leave room for a small error that is the same in every element (fp16 operands in an fp32 GEMM, a
    1e-4 relative scale error, a 1 % error over a whole attention output with zero-mean values), which rounding noise
    never produces.  This aggregate check sees such an error; it uses the limits the op tests have always used.  Prints
    and returns the value."""
    o = out.detach().to(F64)
    ref = ref.to(o.device, F64)
    r = float((o - ref).norm() / ref.norm().clamp(min=1e-300))
    msg = f"{what}: rel-L2 = {r:.3g} (limit {limit:.3g})"
    print(msg)
    assert r < limit, msg
    return r


def half_out(ref, bound):
    """Reference and bound of an fp16 output whose fp32 value (before rounding) has reference `ref` and bound `bound`.
    The kernels convert with saturation (csrc/sat_half.cuh: beyond +-65504 -> +-65504), so the reference is clamped to
    +-65504 and then rounded.  Clamping is 1-Lipschitz and each of the two roundings (kernel value, reference) is off by
    at most U16 relative or, among subnormals, 2^-25 absolute:
        |fp16(clamp(y)) - fp16(clamp(r))| <= (1 + U16) bound + 2 U16 |clamp(r)| + 2^-24."""
    rc = ref.clamp(-HALF_MAX, HALF_MAX)
    return rc.to(torch.float16).to(F64), (1 + U16) * bound + 2 * U16 * rc.abs() + 2.0 ** -24


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x * (0.5 ** 0.5)))


def _silu(x):
    return x * torch.sigmoid(x)


# ---------------------------------------------------------------------------------------------- attention
def attention_views(q, q_bs, ldq, k, v, kv_bs, ldkv, kv_hs, B, heads, n, m):
    """The [B, h, n, 64] query and [B, hk, m, 64] key / value views that mi_attention_fwd reads (hk = 1: kv_hs == 0)."""
    hk = heads if kv_hs else 1
    qv = q.as_strided((B, heads, n, 64), (q_bs, 64, ldq, 1), q.storage_offset())
    kv = k.as_strided((B, hk, m, 64), (kv_bs, kv_hs, ldkv, 1), k.storage_offset())
    vv = v.as_strided((B, hk, m, 64), (kv_bs, kv_hs, ldkv, 1), v.storage_offset())
    return qv, kv, vv


def attention_ref(q, k, v, null_kv, mask=None, p16=True, out16=True):
    """softmax([null_k, k] q^T) [null_v, v] per (batch, head, query row) -- mi_attention_fwd and AttentionFn.forward.

    q [B, h, n, 64]; k, v [B, hk, m, 64] with hk = h or 1 (multi-query); null_kv [2, 64]; mask [B, m] (nonzero = key
    takes part; the null key always does).  Pass the values the kernel reads: fp16-rounded q / k / v / null_kv for the
    fused kernels, the fp32 values for AttentionFn.  Keys that are masked out get probability 0 in the reference, as in
    both kernels (-FLT_MAX scores underflow exp to exactly 0).

    Bound, per element, with A = sum_j p_j |v_j| over the unmasked keys, L = m + 1 keys and
    ds = 64 U32 max_j sum_d |q_d k_jd| the row's fp32 score error (64-term fp32 dot products):
        2 (U16 |o| + (U16 + 4 ds + (L + 8) U32) A)
      * U16 A      : P is rounded to fp16 before the P V product (p16; 0 for the fp32 path);
      * 4 ds A     : a score error ds moves exp(s - max) by e^ds and the row sum l by as much: p_j / l off by <= 2 ds
                     relative, and sum_j dp_j |v_j - o| <= 2 ds 2 A;
      * (L+8) U32 A: fp32 exp (a few ulp), the L-term sums of l and of P V, the final division;
      * U16 |o|    : fp16 output rounding (out16; U32 |o| for an fp32 output);
    doubled for second-order terms.  Chunked per image so that the float64 scores of one image only are live."""
    B, h, n, D = q.shape
    m, hk = k.shape[2], k.shape[1]
    L = m + 1
    nk = null_kv.detach().to(F64, copy=True).to(q.device)
    o = torch.empty((B, h, n, D), dtype=F64, device=q.device)
    bound = torch.empty_like(o)
    up, uo = (U16 if p16 else 0.0), (U16 if out16 else U32)
    for b in range(B):
        kk = torch.cat((nk[0].expand(hk, 1, D), _d(k[b])), dim=1)
        vv = torch.cat((nk[1].expand(hk, 1, D), _d(v[b])), dim=1)
        qb = _d(q[b])
        s = qb @ kk.transpose(-1, -2)                                   # [h, n, L]
        qk = qb.abs() @ kk.abs().transpose(-1, -2)
        if mask is not None:
            valid = torch.cat((torch.ones(1, dtype=torch.bool, device=q.device), mask[b].to(q.device) != 0))
            s = s.masked_fill(~valid, -math.inf)
            qk = qk.masked_fill(~valid, 0.0)
        p = torch.softmax(s, dim=-1)
        o[b] = p @ vv
        A = p @ vv.abs()
        ds = 64 * U32 * qk.amax(dim=-1, keepdim=True)
        bound[b] = 2 * (uo * o[b].abs() + (up + 4 * ds + (L + 8) * U32) * A)
    return o, bound


def attention_fn_ref(q, k, v, null_kv, heads, do):
    """AttentionFn (minimagen_b200/autograd.py) forward and backward in float64 autograd: q [B, n, h*64], k / v
    [B, m, hk*64], null_kv [2, 64], upstream gradient do [B, n, h*64].  Returns {name: (reference, bound)} for
    o, dq, dk, dv, dnull.

    The fp32 chain is S = q K^T (64-term fma GEMM), P = softmax(S), o = P V (L terms); dP = dO V^T (64 terms),
    dS = P (dP - sum P dP) (L terms), dq = dS K (L terms), dK = dS^T q and dV = P^T dO (n terms), the multi-query head sum
    (h terms) and the null key's batch sum (B h terms).  To first order every rounding adds at most U32 times the
    magnitude of its operands, and every intermediate is dominated by the chain evaluated on absolute values (`twin`:
    |dP| <= |dO| |V|^T, |dS| <= P (|dP| + sum P |dP|), ...).  The score error ds (see attention_ref) moves P by <= 4 ds
    relative.  So each gradient is bounded by 2 N U32 twin with N = n + L + 64 + h + B h + 16 + 4 max(ds) / U32; the
    output uses attention_ref's bound for fp32 P and an fp32 result."""
    B, n, inner = q.shape
    m, D = k.shape[1], 64
    hk = k.shape[2] // D
    L = m + 1
    q_, k_, v_, nk_ = (_d(t).requires_grad_(True) for t in (q, k, v, null_kv))
    with torch.enable_grad():
        qh = q_.reshape(B, n, heads, D).permute(0, 2, 1, 3)
        kh = torch.cat((nk_[0].expand(B, hk, 1, D), k_.reshape(B, m, hk, D).permute(0, 2, 1, 3)), dim=2)
        vh = torch.cat((nk_[1].expand(B, hk, 1, D), v_.reshape(B, m, hk, D).permute(0, 2, 1, 3)), dim=2)
        p = torch.softmax(qh @ kh.transpose(-1, -2), dim=-1)                           # [B, h, n, L]
        o = (p @ vh).permute(0, 2, 1, 3).reshape(B, n, inner)
        grads = torch.autograd.grad(o, (q_, k_, v_, nk_), _d(do))
    o = o.detach()
    p = p.detach()
    qa, ka, va, doa = qh.detach().abs(), kh.detach().abs(), vh.detach().abs(), _d(do).reshape(B, n, heads, D).permute(0, 2, 1, 3).abs()
    ds = 64 * U32 * (qa @ ka.transpose(-1, -2)).amax()
    # forward
    A = (p @ va).permute(0, 2, 1, 3).reshape(B, n, inner)
    bo = 2 * (U32 * o.abs() + (4 * ds + (L + 8) * U32) * A)
    # backward twins
    dPt = doa @ va.transpose(-1, -2)
    dSt = p * (dPt + (p * dPt).sum(dim=-1, keepdim=True))
    dqt = (dSt @ ka).permute(0, 2, 1, 3).reshape(B, n, inner)
    dkt = dSt.transpose(-1, -2) @ qa                                                   # [B, h, L, D]
    dvt = p.transpose(-1, -2) @ doa
    if hk == 1:
        dkt, dvt = dkt.sum(dim=1, keepdim=True), dvt.sum(dim=1, keepdim=True)
    dnt = torch.stack((dkt[:, :, 0].sum(dim=(0, 1)), dvt[:, :, 0].sum(dim=(0, 1))))
    dkt = dkt[:, :, 1:].permute(0, 2, 1, 3).reshape(B, m, hk * D)
    dvt = dvt[:, :, 1:].permute(0, 2, 1, 3).reshape(B, m, hk * D)
    N = n + L + 64 + heads + B * heads + 16 + 4 * float(ds) / U32
    out = {"o": (o, bo)}
    for name, g, t in zip(("dq", "dk", "dv", "dnull"), grads, (dqt, dkt, dvt, dnt)):
        out[name] = (g.detach(), 2 * N * U32 * t)
    return out


# ---------------------------------------------------------------------------------------------- LayerNorm
def ln_ref(x, gamma, beta, eps, pre_gelu, residual):
    """mi_ln_rows: y = (v - mean) rstd gamma + beta + residual over the last dim, v = gelu_erf(x) if pre_gelu else x,
    rstd = 1 / sqrt(mean((v - mean)^2) + eps).  Reference y and the bound of the fp32 output (half_out for the fp16 one).

    The fp32 mean (a C-term sum) is off by <= C U32 max|v|, the centred value v_c - mean by that plus U32 |v_c - mean|,
    the variance (C positive terms) and rsqrtf by <= (C + 4) U32 relative.  Scaled by |gamma_c| rstd this is the
    cancellation term
        |gamma_c| rstd (C + 16) U32 (max_row |v| + |v_c - mean|),
    which also holds for near-constant rows (variance << eps), where rstd ~ eps^-1/2 magnifies the mean's error.  The
    fp32 GELU (erff, a few ulp) is off by <= 4 U32 (|v| + |x|) absolute (1 + erf cancels for negative x); an input error
    of at most G per element moves y_c by <= |gamma_c| rstd (2 + |xhat_c|) G.  The affine epilogue adds at most
    4 U32 (|gamma_c xhat_c| + |beta_c| + |residual_c|).  Bound = 2 x the first two terms + the third."""
    x64 = _d(x)
    C = x64.shape[-1]
    v = _gelu(x64) if pre_gelu else x64
    mu = v.mean(dim=-1, keepdim=True)
    dv = v - mu
    rstd = 1.0 / torch.sqrt((dv * dv).mean(dim=-1, keepdim=True) + eps)
    xh = dv * rstd
    g = _d(gamma)
    y = xh * g
    if beta is not None:
        y = y + _d(beta)
    if residual is not None:
        y = y + _d(residual)
    canc = (C + 16) * U32 * (v.abs().amax(dim=-1, keepdim=True) + dv.abs())
    if pre_gelu:
        canc = canc + (2 + xh.abs()) * 4 * U32 * (v.abs() + x64.abs()).amax(dim=-1, keepdim=True)
    bound = 2 * g.abs() * rstd * canc + 4 * U32 * ((g * xh).abs() + _abs(_d(beta)) + _abs(_d(residual)))
    return y, bound


def ln_bwd_acc_len(R, sms):
    """Summation length behind one dgamma / dbeta element of ln_bwd_kernel (csrc/backward.cu): min(ceil(R / 8), 2 sms)
    blocks of 8 warps stride over the rows; each block accumulates its rows into shared memory, then adds the block's
    partial to the global accumulator (that already holds the caller's value)."""
    blocks = min(-(-R // 8), 2 * sms)
    return -(-R // (8 * blocks)) * 8 + blocks + 1


def ln_bwd_ref(x, dy, gamma, eps, pre_gelu, dgamma0, dbeta0, acc_len):
    """mi_ln_rows_bwd (LayerNorm without beta, optional exact-erf GELU in front): dx, and dgamma / dbeta accumulated
    onto dgamma0 / dbeta0.  Returns ((dx, bound), (dgamma, bound), (dbeta, bound)).

    With xhat = (v - mean) rstd, g = gamma dy: dx = rstd (g - mean(g) - xhat mean(g xhat)) [* gelu'(x)].  xhat_c is off
    by <= (C + 16) U32 e_c with e_c = rstd (max_row |v| + |v_c - mean|) (see ln_ref; e_c >= |xhat_c|), the two C-term
    means by C U32 times their absolute twins, so
        |d dx_c| <= 4 (C + 16) U32 rstd (|g_c| + mean|g| + e_c mean(|g| e))  (* |gelu'(x_c)|)
    plus, with GELU, 8 U32 |inner_c| for the fp32 gelu' (inner = dx / gelu') and 4 U32 (|v| + |x|) of GELU error in e.
    dgamma_c = dgamma0_c + sum_rows dy xhat: acc_len roundings (ln_bwd_acc_len) and the xhat errors:
        2 (acc_len + C + 16) U32 (sum_rows |dy_c| e_c + |dgamma0_c|);  dbeta likewise with sum_rows |dy_c|."""
    x64, d = _d(x), _d(dy)
    C = x64.shape[-1]
    with torch.enable_grad():
        x_ = x64.clone().requires_grad_(True)
        g_ = _d(gamma).clone().requires_grad_(True)
        v_ = _gelu(x_) if pre_gelu else x_
        y = torch.nn.functional.layer_norm(v_, (C,), None, None, eps) * g_
        gx, gg = torch.autograd.grad(y, (x_, g_), d)
    v = _gelu(x64) if pre_gelu else x64
    mu = v.mean(dim=-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((v - mu) ** 2).mean(dim=-1, keepdim=True) + eps)
    vmax = v.abs().amax(dim=-1, keepdim=True)
    if pre_gelu:
        vmax = vmax + 4 * (v.abs() + x64.abs()).amax(dim=-1, keepdim=True)
    e = rstd * (vmax + (v - mu).abs())
    ga = (_d(gamma) * d).abs()
    twin = ga + ga.mean(dim=-1, keepdim=True) + e * (ga * e).mean(dim=-1, keepdim=True)
    bdx = 4 * (C + 16) * U32 * rstd * twin
    if pre_gelu:       # dx = gelu'(x) inner; the fp32 gelu' (erff, expf) is off by <= 8 U32 absolute
        xh = (v - mu) * rstd
        g = _d(gamma) * d
        inner = rstd * (g - g.mean(dim=-1, keepdim=True) - xh * (g * xh).mean(dim=-1, keepdim=True))
        gp = 0.5 * (1 + torch.erf(x64 * 0.5 ** 0.5)) + x64 * torch.exp(-0.5 * x64 * x64) / math.sqrt(2 * math.pi)
        bdx = bdx * (gp.abs() + 8 * U32) + 8 * U32 * inner.abs()
    dg = gg + _d(dgamma0)
    db = d.sum(dim=0) + _d(dbeta0)
    bdg = 2 * (acc_len + C + 16) * U32 * ((d.abs() * e).sum(dim=0) + _d(dgamma0).abs())
    bdb = 2 * acc_len * U32 * (d.abs().sum(dim=0) + _d(dbeta0).abs())
    return (gx, bdx), (dg, bdg), (db, bdb)


# ---------------------------------------------------------------------------------------------- fp32 linear / GEMM
def linear_ref(x, w, bias, in_act, out_act, addend, out_scale):
    """mi_linear_f32: y = s * act_out(act_in(x) W^T + bias + addend), act = SiLU when the flag is 1.  Bound of the fp32
    output (half_out for the fp16 one).

    The K-term fp32 dot product (any order) and the two adds are off by <= (K + 2) U32 twin, twin = |act_in(x)| |W|^T +
    |bias| + |addend|; the fp32 SiLU of the input (x / (1 + expf(-x)), a few ulp) adds <= 4 U32 twin; SiLU at the output
    has slope <= 1.1 and rounds by <= 4 U32 |y|; the scale rounds once:
        |s| 2 (K + 8) U32 twin (x 1.1 with out_act) + 4 U32 |y|."""
    x64, w64 = _d(x), _d(w)
    K = x64.shape[-1]
    xa = _silu(x64) if in_act else x64
    pre = xa @ w64.t()
    twin = xa.abs() @ w64.abs().t()
    if bias is not None:
        pre, twin = pre + _d(bias), twin + _d(bias).abs()
    if addend is not None:
        pre, twin = pre + _d(addend), twin + _d(addend).abs()
    e = 2 * (K + 8) * U32 * twin
    y = pre
    if out_act:
        y, e = _silu(pre), 1.1 * e
    y = y * out_scale
    return y, abs(out_scale) * e + 4 * U32 * y.abs()


def gemm_ref(A, B, C0, alpha, accumulate):
    """mi_gemm_f32: C = alpha A B (+ C0), batched over leading dims.  The kernel accumulates K fused multiply-adds in
    fp32, scales once and adds once:  2 (K + 2) U32 (|alpha| |A| |B| + |C0|)."""
    A64, B64 = _d(A), _d(B)
    K = A64.shape[-1]
    r = alpha * (A64 @ B64)
    twin = abs(alpha) * (A64.abs() @ B64.abs())
    if accumulate:
        r, twin = r + _d(C0), twin + _d(C0).abs()
    return r, 2 * (K + 2) * U32 * twin


def colsum_acc_len(M):
    """Summation length behind one column of colsum_kernel (csrc/backward.cu): min(ceil(M / 1024), 512) row splits of
    rpb rows; a thread sums every 8th row of its split, 8 partials are added, then one atomicAdd per split onto out."""
    splits = min(-(-M // 1024), 512)
    rpb = -(-M // splits)
    return -(-rpb // 8) + 8 + splits + 1


def colsum_ref(x, out0, acc_len):
    """mi_colsum_f32: out = sum_rows x (+ out0):  2 acc_len U32 (sum_rows |x| + |out0|)."""
    x64 = _d(x)
    s, twin = x64.sum(dim=0), x64.abs().sum(dim=0)
    if out0 is not None:
        s, twin = s + _d(out0), twin + _d(out0).abs()
    return s, 2 * acc_len * U32 * twin


# ---------------------------------------------------------------------------------------------- softmax rows
def softmax_ref(s):
    """mi_softmax_rows: p = exp(s - max) / sum.  The fp32 difference s - max rounds by U32 |s - max| (an exponent error:
    relative error of the same size in p), expf is good to a few ulp, the sum of L positive terms to L U32 relative,
    the reciprocal and the product to an ulp each; probabilities below 2^-126 are subnormal, where expf and the product
    round to absolute steps of 2^-149:  2 p ((L + 8) U32 + U32 |s - max|) + ETA32."""
    s64 = _d(s)
    L = s64.shape[-1]
    p = torch.softmax(s64, dim=-1)
    return p, 2 * p * ((L + 8) * U32 + U32 * (s64 - s64.amax(dim=-1, keepdim=True)).abs()) + ETA32


def softmax_bwd_ref(P, dP):
    """mi_softmax_rows_bwd: dS = P (dP - sum_j P_j dP_j) with the kernel's own (fp32) P.  The dot product is an L-term
    fma sum, the difference and the product round once (the product by up to 2^-149 absolute among subnormals):
        2 (L + 4) U32 P (|dP| + sum_j |P_j dP_j|) + ETA32."""
    P64, d64 = _d(P), _d(dP)
    L = P64.shape[-1]
    dot = (P64 * d64).sum(dim=-1, keepdim=True)
    twin = P64 * (d64.abs() + (P64 * d64).abs().sum(dim=-1, keepdim=True))
    return P64 * (d64 - dot), 2 * (L + 4) * U32 * twin + ETA32


# ---------------------------------------------------------------------------------------------- GroupNorm/FiLM/SiLU backward
def gn_bwd_splits(B, HW, C, sms):
    """Pixel splits Z of gn_bwd_sums_kernel (csrc/backward.cu, gn_silu_bwd): about 8 blocks per SM over the (C/32, B, Z)
    grid, at most one split per 64 pixels."""
    blocks_xy = -(-C // 32) * B
    return max(min(-(-8 * sms // blocks_xy), HW // 64), 1)


def gn_bwd_acc_len(B, HW, C, sms):
    """Summation length behind one pixel sum A[b][c] of gn_bwd_sums_kernel: a thread sums every 8th pixel of its chunk
    (chunk = ceil(HW / Z)), the 8 partials are added, then one atomicAdd per split onto the zeroed A."""
    Z = gn_bwd_splits(B, HW, C, sms)
    return -(-(-(-HW // Z)) // 8) + 8 + Z


def gn_silu_bwd_ref(x, dy, gamma, beta, ss, groups, eps, dgamma0, dbeta0, acc_len):
    """mi_gn_silu_bwd: the gradients of y = SiLU(v), v = (xhat gamma + beta) (scale + 1) + shift, xhat the GroupNorm of x
    over (pixels, Cg = C / groups channels) per image.  x, dy [B, HW, C] fp32; ss [B, 2C] = [scale | shift] (a strided view
    is fine) or None.  Returns ((dx, bound), (dgamma, bound), (dbeta, bound), (dscale, bound), (dshift, bound)); dgamma /
    dbeta accumulate onto dgamma0 / dbeta0.

    With sc = scale + 1, dv = dy silu'(v), A1 = sum_p dv, A2 = sum_p dv xhat (per image and channel), N = Cg HW:
        dgamma = dgamma0 + sum_b sc A2,  dbeta = dbeta0 + sum_b sc A1,  dscale = gamma A2 + beta A1,  dshift = A1,
        m1 = sum_{c in g} gamma sc A1 / N,  m2 = sum_{c in g} gamma sc A2 / N,  dx = rstd (gamma sc dv - m1 - xhat m2).
    Kernel rounding, first order:
      * xhat: the fp32 mean (off by U32 |mean|), the difference, the fp32 rstd and the product give
            |d xhat| <= 3 U32 e,   e = rstd (|mean| + |x - mean|):  the cancellation term, e / |xhat| grows with |mean| / std
            (and with rstd ~ eps^-1/2 on a near-constant group);
      * v: xhat's error and four roundings (sc = ss + 1 included):  |d v| <= 3 U32 |gamma sc| e + 4 U32 V,
            V = |gamma sc xhat| + |beta sc| + |shift|;
      * dv: silu' has slope <= 0.5; the fp32 silu' (expf, a division, 1 - sigmoid times v) is off by <= 8 U32 (1 + |v|);
            the product rounds once:  Ddv = U32 |dy| (10 (1 + V) + 2 |gamma sc| e);
      * A1 / A2: acc_len roundings (gn_bwd_acc_len) of the pixel sums plus the summed input errors:
            dA1 = acc_len U32 T1 + sum_p Ddv,  dA2 = acc_len U32 T2 + sum_p (Ddv |xhat| + 3 U32 |dv| e),
            T1 = sum_p |dv|,  T2 = sum_p |dv xhat|;
      * dgamma / dbeta: B atomics onto the caller's value and the product sc A:  (B + 2) U32 (sum_b |sc| T + |d0|);
      * m1 / m2: a Cg-term shared-memory sum, the products gamma sc A and the multiply by 1 / N:  (Cg + 4) U32 M1t plus
            sum_c |gamma sc| dA / N, with M1t = sum_{c in g} |gamma sc| T1 / N (M2t likewise with T2);
      * dx: rstd (|gamma sc| Ddv + dm1 + |xhat| dm2 + 3 U32 e M2t + 8 U32 (|gamma sc dv| + M1t + |xhat| M2t)) -- the
            errors of the three terms, the difference, the products and rstd's rounding;
    every bound doubled for second-order terms."""
    x64, d = _d(x), _d(dy)
    B, HW, C = x64.shape
    Cg = C // groups
    N = Cg * HW
    dev = x64.device
    xg = x64.reshape(B, HW, groups, Cg)
    mu = xg.mean(dim=(1, 3))                                                       # [B, G]
    rstd = 1.0 / torch.sqrt(((xg - mu[:, None, :, None]) ** 2).mean(dim=(1, 3)) + eps)
    mu_c = mu.repeat_interleave(Cg, dim=1)[:, None, :]                             # [B, 1, C]
    rs_c = rstd.repeat_interleave(Cg, dim=1)[:, None, :]
    g64, b64 = _d(gamma).to(dev), _d(beta).to(dev)
    if ss is not None:
        s64 = _d(ss).to(dev)
        sc, sh = s64[:, :C] + 1.0, s64[:, C:2 * C]
    else:
        sc, sh = torch.ones(B, C, dtype=F64, device=dev), torch.zeros(B, C, dtype=F64, device=dev)
    xh = (x64 - mu_c) * rs_c
    v = (xh * g64 + b64) * sc[:, None] + sh[:, None]
    sg = torch.sigmoid(v)
    dv = d * (sg * (1 + v * (1 - sg)))
    del sg
    A1, A2 = dv.sum(dim=1), (dv * xh).sum(dim=1)                                   # [B, C]
    gs = (g64 * sc).abs()
    grp = lambda t: t.reshape(B, groups, Cg).sum(dim=2).repeat_interleave(Cg, dim=1)     # group sum, spread over channels
    m1, m2 = grp(g64 * sc * A1) / N, grp(g64 * sc * A2) / N
    dx = rs_c * (g64 * sc[:, None] * dv - m1[:, None] - xh * m2[:, None])
    # bounds
    e = rs_c * (mu_c.abs() + (x64 - mu_c).abs())
    ax = xh.abs()
    del xh, v
    gs_ = gs[:, None]
    V = gs_ * ax + (b64 * sc).abs()[:, None] + sh.abs()[:, None]
    Ddv = U32 * d.abs() * (10 * (1 + V) + 2 * gs_ * e)
    del V
    adv = dv.abs()
    T1, T2 = adv.sum(dim=1), (adv * ax).sum(dim=1)
    dA1 = acc_len * U32 * T1 + Ddv.sum(dim=1)
    dA2 = acc_len * U32 * T2 + (Ddv * ax + 3 * U32 * adv * e).sum(dim=1)
    M1t, M2t = grp(gs * T1) / N, grp(gs * T2) / N
    dm1 = grp(gs * dA1) / N + (Cg + 4) * U32 * M1t
    dm2 = grp(gs * dA2) / N + (Cg + 4) * U32 * M2t
    M1t, M2t, dm1, dm2 = M1t[:, None], M2t[:, None], dm1[:, None], dm2[:, None]
    bdx = 2 * rs_c * (gs_ * Ddv + dm1 + ax * dm2 + 3 * U32 * e * M2t + 8 * U32 * (gs_ * adv + M1t + ax * M2t))
    dg0, db0 = _d(dgamma0).to(dev), _d(dbeta0).to(dev)
    dg = dg0 + (sc * A2).sum(dim=0)
    db = db0 + (sc * A1).sum(dim=0)
    bdg = 2 * ((sc.abs() * dA2).sum(dim=0) + (B + 2) * U32 * ((sc.abs() * T2).sum(dim=0) + dg0.abs()))
    bdb = 2 * ((sc.abs() * dA1).sum(dim=0) + (B + 2) * U32 * ((sc.abs() * T1).sum(dim=0) + db0.abs()))
    dscale = g64 * A2 + b64 * A1
    bds = 2 * (g64.abs() * dA2 + b64.abs() * dA1 + 2 * U32 * (g64.abs() * T2 + b64.abs() * T1))
    return (dx, bdx), (dg, bdg), (db, bdb), (dscale, bds), (A1, 2 * dA1)


# ---------------------------------------------------------------------------------------------- convolution gradients
def wgrad_f32_plan(B, Ho, Wo, Cin, Cout, kh, kw, sms):
    """(pixels per block, pixel splits) of conv_wgrad_kernel (csrc/backward.cu, conv2d_wgrad_f32): the flat variant
    (C_in < 32 and more than one tap) tiles (C_out, C_in x taps) by 32 x 32, the tiled one (C_out, C_in) per tap; both aim
    at 16 blocks per SM, with at least 128 pixels per split, rounded to 32-pixel stages."""
    total = B * Ho * Wo
    taps = kh * kw
    flat = Cin < 32 and taps > 1
    tiles = -(-Cout // 32) * -(-(Cin * taps if flat else Cin) // 32)
    work = tiles if flat else tiles * taps
    splits = min(-(-16 * sms // work), -(-total // 128))
    splits = min(max(splits, 1), 65535)
    ppb = -(-(-(-total // splits)) // 32) * 32
    return ppb, -(-total // ppb)


def wgrad_f32_acc_len(B, Ho, Wo, Cin, Cout, kh, kw, sms):
    """Summation length behind one dW element of conv2d_wgrad_f32: an fma per pixel of the block's range, then one atomicAdd
    per split onto the zeroed dW."""
    ppb, splits = wgrad_f32_plan(B, Ho, Wo, Cin, Cout, kh, kw, sms)
    return ppb + splits


def wgrad_tc_plan(B, Ho, Wo, Cin, Cout, k, sms):
    """(8 x 8 pixel boxes per CTA, splits) of conv_wgrad_tc (csrc/wgrad_tc.cu, wgrad_plan): about two CTAs per SM over
    (C_out / 128) x (C_in / N) x taps tile groups, N = 128 when C_in % 128 == 0 else 64."""
    nb = 2 if Cin % 128 == 0 else 1
    total = B * (Ho // 8) * (Wo // 8)
    groups = (Cout // 128) * (Cin // (nb * 64)) * k * k
    splits = min(max(-(-2 * sms // groups), 1), total, 65535)
    per = -(-total // splits)
    return per, -(-total // per)


def wgrad_tc_acc_len(B, Ho, Wo, Cin, Cout, k, sms):
    """Summation length behind one dW element of conv_wgrad_tc: 64 pixels per box in the CTA's wgmma accumulators, then
    wgrad_reduce_kernel's sum over the splits."""
    per, splits = wgrad_tc_plan(B, Ho, Wo, Cin, Cout, k, sms)
    return 64 * per + splits


def _nchw(t):
    return _d(t).permute(0, 3, 1, 2)


FP16_MIN_NORMAL = 2.0 ** -14


def align_mag(t):
    """|t| as a wgmma k-group aligns it (float64): for an fp16 operand, a subnormal counts as 2^-14.

    The tensor cores align the 16 products of a k-group to the largest exponent e_a + e_b read from the operands' exponent
    fields.  An fp16 subnormal's exponent field reads as that of 2^-14 and its significand is not renormalised first, so its
    product is aligned as if it were up to 2^10 times larger than it is, and the truncation unit grows with it.  Measured on
    an H100: dW of a training step whose dy rounds to fp16 subnormals (~2^-24) was off by one unit of 2^-39 at x ~ 2^-2,
    i.e. 2^-23 relative to 2^-14 * 2^-2, not to the product's own 2^-26; and the same dy bits scaled by 2^16 into the
    normal range (an exact scaling, which leaves fp32 arithmetic's relative error unchanged) gave a 5 - 8 x smaller median
    relative error of dW.  fp32 operands (the CUDA-core kernels) are returned as |t|."""
    a = _d(t).abs()
    if t.dtype == torch.float16:
        a = torch.where((a > 0) & (a < FP16_MIN_NORMAL), torch.full_like(a, FP16_MIN_NORMAL), a)
    return a


def conv_wgrad_ref(dy, x, stride, pad, kh, kw, acc_len):
    """dW[co][ci][r][s] = sum over output pixels (b, h, w) of dy[b, h, w, co] x[b, stride h + r - pad, stride w + s - pad, ci]
    (zero outside the image): conv2d_wgrad_f32 and mi_conv2d_wgrad_f16.  dy [B, Ho, Wo, C_out] and x [B, Hi, Wi, C_in] NHWC
    as the kernel reads them (fp16 for the tensor-core kernel).  Returns (dW OIHW, bound).

    Bound 3 acc_len U32 twin, twin = the same sum over |dy| |x|; acc_len from wgrad_f32_acc_len / wgrad_tc_acc_len.  The fp32
    kernel is an fma chain per split plus one atomicAdd per split: acc_len roundings of a partial sum dominated by twin, so
    2 acc_len U32 twin.  On the tensor cores the products of fp16 operands are exact in fp32, but a wgmma k-group adds 16
    products to the accumulator by aligning them to the largest exponent and truncating, not rounding to nearest: each of
    the 17 terms loses less than one unit of 2^-23 relative to the group's largest term, and the normalised sum is
    truncated once more.  That is <= 17 x 2 U32 x (|accumulator| + sum |products|) <= 34 U32 twin per 16 products,
    2.125 U32 twin per product; the fp32 split reduction adds U32 twin per split.  Hence c = 3 for both kernels.  The
    largest term is the one the hardware aligns to, so for fp16 operands twin is taken over align_mag (an fp16 subnormal
    counts as 2^-14)."""
    g = torch.nn.grad.conv2d_weight
    Co, Ci = dy.shape[-1], x.shape[-1]
    shape = (Co, Ci, kh, kw)
    ref = g(_nchw(x), shape, _nchw(dy), stride=stride, padding=pad)
    mag = lambda t: align_mag(t).permute(0, 3, 1, 2)
    twin = g(mag(x), shape, mag(dy), stride=stride, padding=pad)
    return ref, 3 * acc_len * U32 * twin


def conv_dgrad_ref(dy, w, stride, pad, Hi, Wi):
    """dx[b, h, w, ci] = sum over taps (r, s) and co of dy[b, (h + pad - r) / stride, (w + pad - s) / stride, co] w[co][ci][r][s]
    where the division is exact and in range: conv2d_dgrad_f32 (general and small-C_out kernels, fp32 operands) and the
    tensor-core data gradients of Conv2dFn (fp16 dy and fp16 packed weights: pass those values).  dy [B, Ho, Wo, C_out]
    NHWC, w (C_out, C_in, kh, kw).  Returns (dx NHWC, bound).

    Every kernel sums at most n = taps x C_out products into one fp32 accumulator: an fma chain on the CUDA cores
    (2 n U32 twin), the wgmma K loop of the implicit GEMM on the tensor cores (see conv_wgrad_ref: 2.125 n U32 twin):
        3 n U32 twin + U32 |dx|,   twin = the same sum over |dy| |w| (align_mag for fp16 operands)."""
    B, Ci = dy.shape[0], w.shape[1]
    Co, kh, kw = w.shape[0], w.shape[2], w.shape[3]
    g = torch.nn.grad.conv2d_input
    w64 = _d(w).to(dy.device)
    ref = g((B, Ci, Hi, Wi), w64, _nchw(dy), stride=stride, padding=pad).permute(0, 2, 3, 1)
    twin = g((B, Ci, Hi, Wi), align_mag(w).to(dy.device), align_mag(dy).permute(0, 3, 1, 2), stride=stride,
             padding=pad).permute(0, 2, 3, 1)
    return ref, 3 * kh * kw * Co * U32 * twin + U32 * ref.abs()


def upsample2x_bwd_ref(dy):
    """mi_upsample2x_bwd: dx[b, h, w] = (dy[2h, 2w] + dy[2h, 2w + 1]) + (dy[2h + 1, 2w] + dy[2h + 1, 2w + 1]) in fp32, in
    this order: a fixed-order sum, so the kernel must match it bit for bit.  dy [B, 2H, 2W, C] fp32."""
    B, H2, W2, C = dy.shape
    q = dy.float().reshape(B, H2 // 2, 2, W2 // 2, 2, C)
    return (q[:, :, 0, :, 0] + q[:, :, 0, :, 1]) + (q[:, :, 1, :, 0] + q[:, :, 1, :, 1])


# ---------------------------------------------------------------------------------------------- convolution forward
U64 = 2.0 ** -53            # unit roundoff of fp64: the double sums and atomics of the statistics
ETA_SILU = 2.0 ** -118      # |SiLU(v)| where the fp32 SiLU flushes to 0 (v < -87: 1 + e^-v > 2^126)


def unpack_conv_weight(wp, kh, kw, c_in):
    """The first kh * kw * c_in columns of a packed [C_out][taps * C_in (+ C_x)] weight (tap-major, channel-minor, the
    layout of mi_pack_conv_weight_f16) as float64 OIHW."""
    return _d(wp[:, :kh * kw * c_in]).reshape(wp.shape[0], kh, kw, c_in).permute(0, 3, 1, 2)


def conv_nhwc(a, w, mode):
    """Float64 convolution of the NHWC operand `a` with OIHW `w` as mi_conv2d_igemm_f16 reads it in `mode`; NHWC result.
      mode 0: 'same' k x k conv of a [B, H, W, C];
      mode 1: the 4x4 stride-2 pad-1 conv of the phase-split a [B, 4, H, W, C] (phase p = (h & 1) * 2 + (w & 1));
      modes 2..5: sub-pixel phase (pa, pb) = ((mode - 2) >> 1, (mode - 2) & 1) of a [B, H, W, C]: the 2x2 taps of output
                  pixel (y, x) read the pixels (y + pa - 1 + r, x + pb - 1 + s);
      mode 6: the 4x4 stride-2 pad-1 conv of a [B, 2H, 2W, C] read in place."""
    F = torch.nn.functional
    if mode == 1:
        B, _, H, W, C = a.shape
        full = a.new_zeros(B, 2 * H, 2 * W, C)
        for p in range(4):
            full[:, (p >> 1)::2, (p & 1)::2] = a[:, p]
        a, mode = full, 6
    x = a.permute(0, 3, 1, 2)
    if mode == 6:
        y = F.conv2d(x, w, stride=2, padding=1)
    elif mode == 0:
        y = F.conv2d(x, w, padding=(w.shape[2] // 2, w.shape[3] // 2))
    else:
        pa, pb = (mode - 2) >> 1, (mode - 2) & 1
        H, W = x.shape[2], x.shape[3]
        y = F.conv2d(F.pad(x, (1, 1, 1, 1))[:, :, pa:pa + H + 1, pb:pb + W + 1], w)
    return y.permute(0, 2, 3, 1)


def conv_fwd_ref(a, wp, kh, kw, mode=0, bias=None, residual=None, x=None):
    """conv + bias + residual of mi_conv2d_igemm_f16 / mi_conv3x3_res1x1_f16 (and, with fp32 operands, mi_conv2d_direct_f32):
    a the fp16 operand as the kernel reads it (see conv_nhwc; a two-source virtual concat is the channel concat of both
    sources, the skip scale folded into the packed weight), wp the packed fp16 weight [C_out][kh kw C_in (+ C_x)], x the
    operand of the folded 1x1 conv [B, H, W, C_x] (columns kh kw C_in ... of wp, read at the centre tap), residual
    [B, H, W, C_out].  Returns (reference NHWC, bound of the fp32 output); half_out gives the fp16 output's.

    Every output element is one fp32 accumulation of n = taps C_in (+ C_x) exact fp16 products, then the bias and the
    residual adds.  The wgmma k-groups truncate instead of rounding (2.125 U32 twin per product, see conv_wgrad_ref), so
        3 (n + 2) U32 twin,   twin = sum |a| |w| + |bias| + |residual|.
    conv_direct_f32 is an fma chain over taps x ceil4(C_in) products (2 n U32 twin): the same form with that n; the stem's
    15-tap GEMM over 128 unrolled channels has n = 15 x 128.  For fp16 operands twin is taken over align_mag (an fp16
    subnormal counts as 2^-14, as the wgmma k-group aligns it)."""
    c_in = a.shape[-1]
    w = unpack_conv_weight(wp, kh, kw, c_in).to(a.device)
    wm = unpack_conv_weight(align_mag(wp), kh, kw, c_in).to(a.device)
    ref, twin = conv_nhwc(_d(a), w, mode), conv_nhwc(align_mag(a), wm, mode)
    n = kh * kw * c_in
    if x is not None:
        wx, x64 = _d(wp[:, n:]).to(a.device), _d(x)
        ref, twin = ref + x64 @ wx.t(), twin + align_mag(x) @ align_mag(wp[:, n:]).to(a.device).t()
        n += x.shape[-1]
    for t in (bias, residual):
        if t is not None:
            ref, twin = ref + _d(t), twin + _d(t).abs()
    return ref, 3 * (n + 2) * U32 * twin


def conv_stats_acc_len():
    """Rounding steps behind one (image, 16-channel block) statistic of the conv epilogue (csrc/conv_tc.cu): a thread adds
    its 8 values of the block (2 rows x 2 column pairs, each pair summed first; for the squares one product and one fma per
    pair) in fp32 -- at most 8 roundings on any value's path -- then 5 xor-shuffle levels add the warp's 32 partials in
    fp32; the rest (per warp or per warpgroup) is fp64."""
    return 8 + 5 + 1


def conv_stats_ref(out32, sb=16, P=None):
    """The epilogue's GroupNorm statistics, per (image, sb-channel block), of the kernel's OWN fp32 output out32
    [B, ..., C] (valid pixels only; the phases of modes 2..5 all in one tensor): float64 (sum, sum of squares) [B, C/sb, 2]
    and their bound
        2 acc_len U32 sum|f|  (resp. sum f^2)  +  P U64 (same),
    acc_len = conv_stats_acc_len(), P the pixel count (more than the fp64 adds of any reduction order).  Because it compares
    with the output the kernel wrote, not with reference statistics, the bound is tight enough to see one warp's 16 rows, a
    tile credited to the wrong image, or masked rows that were counted.  P (default: out32's pixels) is the image's pixel
    count when out32 is one band of rows: both results are then linear in the band's values and add up over the bands."""
    f = _d(out32)
    B, C = f.shape[0], f.shape[-1]
    fb = f.reshape(B, -1, C // sb, sb)
    P = fb.shape[1] if P is None else P
    s, q, t = fb.sum(dim=(1, 3)), (fb * fb).sum(dim=(1, 3)), fb.abs().sum(dim=(1, 3))
    c = 2 * conv_stats_acc_len() * U32 + P * U64
    return torch.stack((s, q), dim=-1), torch.stack((c * t, c * q), dim=-1)


# ---------------------------------------------------------------------------------------------- GroupNorm forward
def _f32(v):
    """A Python scale as the fp32 number the kernels multiply by."""
    return float(torch.tensor(float(v), dtype=torch.float32))


def gn_concat(src0, src1=None, scale1=1.0):
    """The virtual concat cat(src0, src1 * scale1) [B, HW, C] in float64, src1 scaled by the fp32 scale1 (exact here; the
    kernels' fp32 product rounds by U32 of it)."""
    x = _d(src0)
    if src1 is not None:
        x = torch.cat((x, _d(src1) * _f32(scale1)), dim=-1)
    return x


def gn_stats_plan(C, HW):
    """(chunk, planes, L) of gn_stats_kernel (csrc/elementwise.cu, gn_stats): the grid covers `chunk` = clamp(32768 / C, 4,
    HW) pixels per CTA; its 256 threads split into `planes` = 256 / (C / 8) pixel planes of C / 8 channel vectors (1 plane
    when C > 2048); a thread's fp32 chain adds every planes-th pixel of the chunk, L = ceil(chunk / planes) values."""
    chunk = min(max(32768 // C, 4), HW)
    V = C // 8
    planes = 256 // V if V <= 256 else 1
    return chunk, planes, -(-chunk // planes)


def gn_stats_ref(src0, groups, src1=None, scale1=1.0, L=None, HW=None):
    """mi_gn_stats: per (image, group) float64 (sum, sum of squares) [B, G, 2] of the virtual concat, and the bound
        (L + 3) U32 sum|x|  (resp. sum x^2)  +  (HW + 2048) U64 (same).
    A thread's fp32 chain of L values (gn_stats_plan) rounds at most L times on any value's path, the squares once more
    and the fp32 product x * scale1 once (U32 |x|, 2 U32 x^2); the 8 partials of a thread, the CTA's shared-memory sum and
    the atomics per chunk are fp64.  HW (default: the sources' pixels) is the image's pixel count when the sources are
    one band of its pixels: the results then add up over the bands."""
    x = gn_concat(src0, src1, scale1)
    B, _, C = x.shape
    HW = x.shape[1] if HW is None else HW
    if L is None:
        L = gn_stats_plan(C, HW)[2]
    xg = x.reshape(B, -1, groups, C // groups)
    s, q, t = xg.sum(dim=(1, 3)), (xg * xg).sum(dim=(1, 3)), xg.abs().sum(dim=(1, 3))
    c = (L + 3) * U32 + (HW + 2048) * U64
    return torch.stack((s, q), dim=-1), torch.stack((c * t, c * q), dim=-1)


def group_sums(stats0, C0, groups, stats1=None, C1=0, scale1=1.0, sb=16):
    """Per-source block statistics [B, C_s / sb, 2] (of a conv epilogue, or gn_stats with C_s / sb groups) gathered into
    the groups of the virtual concat, as gn_apply_silu_kernel and the fused GroupNorm conv gather them (the second source's
    sums times scale1, its squares times scale1^2).  Works for bounds too (they are non-negative)."""
    s1 = _f32(scale1)
    parts = [_d(stats0)]
    if stats1 is not None and C1:
        t = _d(stats1).clone()
        t[..., 0] *= s1
        t[..., 1] *= s1 * s1
        parts.append(t)
    blocks = torch.cat(parts, dim=1)                                   # [B, (C0 + C1) / sb, 2]
    B = blocks.shape[0]
    return blocks.reshape(B, groups, -1, 2).sum(dim=2)


def _gn_silu(x, groups, gamma, beta, ss, eps, sums, sums_err, fast, HW=None):
    """y = SiLU(((x - mean) rstd gamma + beta) (scale + 1) + shift) in float64 from the statistics `sums` [B, G, 2] over
    HW pixels per image (default: x's), and the bound of the kernel's fp32 y before any fp16 rounding.  See
    gn_apply_silu_ref."""
    B, _, C = x.shape
    HW = x.shape[1] if HW is None else HW
    Cg = C // groups
    n = Cg * HW
    dev = x.device
    sums = _d(sums).to(dev)
    mean = sums[..., 0] / n
    var = (sums[..., 1] / n - mean * mean).clamp(min=0)
    V = var + eps
    rstd = 1.0 / torch.sqrt(V)
    spread = lambda t: t.repeat_interleave(Cg, dim=1)[:, None, :]              # [B, G] -> [B, 1, C]
    g, be = _d(gamma).to(dev), _d(beta).to(dev)
    if ss is not None:
        s64 = _d(ss).to(dev)
        sc, sh = (s64[:, :C] + 1.0)[:, None], s64[:, C:2 * C][:, None]
    else:
        sc, sh = torch.ones((), dtype=F64, device=dev), torch.zeros((), dtype=F64, device=dev)
    m_c, r_c = spread(mean), spread(rstd)
    A = r_c * g * sc
    Bc = (be - m_c * r_c * g) * sc + sh
    v = x * A + Bc
    y = _silu(v)
    ev = U32 * (6 * (x * A).abs() + sc.abs() * (7 * (m_c * r_c * g).abs() + 3 * be.abs()) + Bc.abs() + v.abs())
    if sums_err is not None:
        e = _d(sums_err).to(dev)
        dm = e[..., 0] / n
        dvar = e[..., 1] / n + (2 * mean.abs() + dm) * dm + 4 * U64 * sums[..., 1].abs() / n
        lo = (V - dvar).clamp(min=eps)
        drs = dvar / (lo.sqrt() * V.sqrt() * (lo.sqrt() + V.sqrt()))
        ev = ev + (g * sc).abs() * ((x - m_c).abs() * spread(drs) + spread(rstd + drs) * spread(dm))
    if fast:
        rel = 2 * U32 * (2 + 1.16 * v.abs()) * torch.sigmoid(-v) + 8 * U32
    else:
        rel = 8 * U32
    return y, 2 * (1.1 * ev + rel * y.abs()) + ETA_SILU


def gn_apply_silu_ref(src0, groups, gamma, beta, ss, eps, sums, sums_err=None, src1=None, scale1=1.0, out16=False,
                      fast=None, HW=None):
    """mi_gn_apply_silu: y = SiLU(GroupNorm(x) (scale + 1) + shift) over the virtual concat x = cat(src0, src1 * scale1)
    [B, HW, C], ss [B, 2C] = [scale | shift] (a view without the row gaps) or None.  `sums` [B, G, 2] are the statistics the
    reference normalises with; `sums_err` (optional) bounds how far the kernel's statistics are from them.  Returns the
    reference and the bound of the output (fp16 when out16).  fast: the __expf / __fdividef SiLU the kernel uses for fp16
    outputs (default: out16).  HW: the image's pixel count when the sources are one band of its pixels (default: theirs).

    (a) Exact statistics (sums_err None): the kernel casts mean and rstd to fp32 and folds
            a = rstd gamma,  bb = beta - mean a,  a *= sc,  bb = bb sc + shift,  v = fmaf(x, a, bb),
        with sc = scale + 1 rounded once.  Each step rounds once: a is off by 4 U32 |a|, bb by 4 U32 |mean a| (the
        cancellation term) plus 3 U32 |beta - mean a| before the FiLM, so with A = rstd gamma sc, Bc the exact coefficients
            |dv| <= U32 (6 |x A| + |sc| (7 |mean rstd gamma| + 3 |beta|) + |Bc| + |v|)
        (6 |x A| includes the fp32 product x * scale1 of the second source).  SiLU has slope <= 1.1; silu_f (expf, a
        division) is good to 8 U32 |y|; on fp16 outputs __expf is off by (2 + 1.16 |v|) ulp of e^-v, weighted by
        e^-v / (1 + e^-v) in y, and __fdividef adds 2 ulp -- and returns 0 once 1 + e^-v > 2^126 (ETA_SILU absolute):
            2 (1.1 |dv| + rel |y|) + ETA_SILU,   then half_out for fp16.
    (b) Statistics a kernel produced (sums_err = their bound): mean is off by dm = e_sum / n, var = sq / n - mean^2 by
        dvar = e_sq / n + (2 |mean| + dm) dm -- relative to var that grows with (|mean| / std)^2 -- and rstd by
        |1/sqrt(V - dvar) - 1/sqrt(V)| (V = var + eps); v moves by |gamma sc| (|x - mean| drstd + (rstd + drstd) dm)."""
    x = gn_concat(src0, src1, scale1)
    y, bound = _gn_silu(x, groups, gamma, beta, ss, eps, sums, sums_err, out16 if fast is None else fast, HW)
    return half_out(y, bound) if out16 else (y, bound)


def conv_gn_ref(src0, groups, gamma, beta, ss, eps, sums, wp, bias=None, residual=None, src1=None, scale1=1.0):
    """mi_conv3x3_gn_silu_f16: GroupNorm -> FiLM -> SiLU (gn_apply_silu_ref (a), fast SiLU, statistics `sums` [B, G, 2]
    gathered with group_sums) in float64, then the 3x3 conv with the fp16 packed weight wp, + bias + residual.  src0 / src1
    [B, H, W, C_s].  Returns (reference NHWC, bound of the fp32 output).

    The kernel rounds the activated operand a to fp16 (sat_half: U16 |a|, 2^-25 among subnormals) after an fp32 error e_a
    (the bound of (a) before rounding), so
        3 (n + 2) U32 (conv(|a|, |w|) + |bias| + |residual|)  +  conv(U16 |a| + e_a + 2^-25, |w|),   n = 9 C."""
    B, H, W, _ = src0.shape
    x = gn_concat(src0.reshape(B, H * W, -1), None if src1 is None else src1.reshape(B, H * W, -1), scale1)
    C = x.shape[-1]
    a, ea = _gn_silu(x, groups, gamma, beta, ss, eps, sums, None, True)
    a, ea = a.reshape(B, H, W, C), ea.reshape(B, H, W, C)
    w = unpack_conv_weight(wp, 3, 3, C).to(x.device)
    ref, twin = conv_nhwc(a, w, 0), conv_nhwc(a.abs(), w.abs(), 0)
    for t in (bias, residual):
        if t is not None:
            ref, twin = ref + _d(t), twin + _d(t).abs()
    return ref, 3 * (9 * C + 2) * U32 * twin + conv_nhwc(U16 * a.abs() + ea + 2.0 ** -25, w.abs(), 0)


# ---------------------------------------------------------------------------------------------- sampling step
# Operands of the step kernels as they read them: per-image scalars gathered from the fp32 schedule tables at t [B], the
# guidance weight w (a number or [B]) as fp32, [B, n] images.  The elementwise bounds hold for finite data; NaN and inf
# are checked for parity with the torch restatement instead.
def _per_image(tab, t):
    return _d(tab.detach().cpu()[t.detach().cpu()])[:, None]


def _scale_col(w, B):
    if torch.is_tensor(w):
        return _d(w.detach().cpu()).reshape(B, 1)
    return torch.full((B, 1), _f32(w), dtype=F64)


def step_x0_ref(x_t, eps_cond, eps_null, w, t, tab_a, tab_b):
    """guided_x0 (csrc/step.cu): e = nl + (c - nl) w, x0 = a[t] x - b[t] e, every product and sum rounded on its own.
    First-order error: fl(c - nl) and the product w (c - nl) put 2 U32 |w| |c - nl| on p, the sum adds U32 |nl + p|, so
    e is off by U32 |nl| + 3 U32 |w| |c - nl|; b e adds U32 |b e|, a x one U32 |a x|, the subtraction U32 |x0|:
        |dx0| <= U32 (2 |a x| + |b| (3 |nl| + 5 |w| (|c| + |nl|)))  <=  5 U32 (|a x| + |b| (|nl| + |w| (|c| + |nl|)))
    (without eps_null: 2 U32 (|a x| + |b c|)), + ETA32 for products that underflow.  Returns (x0, bound) [B, n]."""
    x, c = _d(x_t).cpu(), _d(eps_cond).cpu()
    B = x.shape[0]
    a, b = _per_image(tab_a, t), _per_image(tab_b, t)
    if eps_null is None:
        e, te = c, c.abs()
    else:
        nl, wc = _d(eps_null).cpu(), _scale_col(w, B)
        e = nl + (c - nl) * wc
        te = nl.abs() + wc.abs() * (c.abs() + nl.abs())
    x0 = a * x - b * e
    return x0, 5 * U32 * ((a * x).abs() + b.abs() * te) + ETA32


def step_threshold_ref(x0, x0_bound, rank_lo, rank_hi, weight, min_s):
    """The dynamic threshold s [B] from the float64 x0 [B, n] and its bound: the order statistics lo, hi of |x0| at
    rank_lo / rank_hi, s = max(lo + w (hi - lo), min_s) with the fp32 weight w of quantile_rank.  Order statistics are
    1-Lipschitz in the sup norm, so the kernel's selected values (of its fp32 x0) are within D = max_i x0_bound_i of lo and
    hi -- per image, not per element; the lerp is a convex combination (1-Lipschitz too) rounded twice (hi - lo, then one
    fma), and the clamp is 1-Lipschitz:
        |s - s64| <= D (1 + 3 U32) + U32 (|hi - lo| + |s64|) + ETA32.
    Returns (s, bound) [B]."""
    srt = x0.abs().sort(dim=-1).values
    lo, hi = srt[:, rank_lo], srt[:, rank_hi]
    wt = _f32(weight)
    s = (lo + wt * (hi - lo)).clamp(min=_f32(min_s))
    D = x0_bound.amax(dim=-1)
    return s, D * (1 + 3 * U32) + U32 * ((hi - lo).abs() + s.abs()) + ETA32


def step_posterior_ref(x0, x0_bound, s, s_bound, x_t, noise, t, tab_c1, tab_c2, tab_sigma, tab_c3=None, hist=None):
    """posterior_elem: xs = clamp(x0, -s, s) / s, out = c1[t] xs + c2[t] x + c3[t] h + sigma[t] z with sigma = 0 at t = 0;
    the multistep form (tab_c3, hist given) also returns xs, the new history.  clamp(x, -s, s) is 1-Lipschitz in x and in
    s, and |clamp / s| <= 1, so with dx = x0_bound, ds = s_bound
        |xs - xs64| <= (dx + 2 ds) / (s64 - ds) + U32 (|xs64| + ...)  =: dxs,
    and the four products and three sums of the output put at most four roundings on each term:
        |out - out64| <= |c1| dxs (1 + 4 U32) + 4 U32 (|c1 xs| + |c2 x| + |c3 h| + |sigma z|) + ETA32.
    Returns (out, out_bound, xs, xs_bound) [B, n] (xs for the history)."""
    x, z = _d(x_t).cpu(), _d(noise).cpu()
    sc, ds = s[:, None], s_bound[:, None]
    xs = torch.minimum(torch.maximum(x0, -sc), sc) / sc
    dxs0 = (x0_bound + 2 * ds) / (sc - ds)
    dxs = dxs0 + U32 * (xs.abs() + dxs0) + ETA32
    c1, c2 = _per_image(tab_c1, t), _per_image(tab_c2, t)
    sig = torch.where(t.detach().cpu()[:, None] == 0, torch.zeros((), dtype=F64), _per_image(tab_sigma, t))
    out = c1 * xs + c2 * x + sig * z
    twin = (c1 * xs).abs() + (c2 * x).abs() + (sig * z).abs()
    if tab_c3 is not None:
        c3, h = _per_image(tab_c3, t), _d(hist).cpu()
        out = out + c3 * h
        twin = twin + (c3 * h).abs()
    return out, c1.abs() * dxs * (1 + 4 * U32) + 4 * U32 * twin + ETA32, xs, dxs


def q_sample_ref(x0, noise, t, tab_a, tab_b, post_scale, post_shift):
    """q_sample_kernel: v = a[t] x0 + b[t] z (three roundings), then v * post_scale + post_shift (two more):
        |out - out64| <= 4 U32 (|post_scale| (|a x0| + |b z|) + |post_shift|) + ETA32."""
    x, z = _d(x0).cpu(), _d(noise).cpu()
    a, b = _per_image(tab_a, t), _per_image(tab_b, t)
    ps, sh = _f32(post_scale), _f32(post_shift)
    ref = (a * x + b * z) * ps + sh
    return ref, 4 * U32 * (abs(ps) * ((a * x).abs() + (b * z).abs()) + abs(sh)) + ETA32


def inpaint_prologue_ref(x, t, r, ra, rb, sqrt_acp, sqrt_1m_acp, k, m, z_renoise, z_known, T):
    """inpaint_prologue_kernel on x [B, C, hw] (m [B, 1, hw], t and r [B] as the kernel read them): where r > 0,
    v = ra[t] x + rb[t] z_renoise; then where m >= 0.5, v = sqrt_acp[t] k + sqrt_1m_acp[t] z_known; images with t outside
    [0, T) and the pixels neither branch takes are left alone.  Each branch is two fp32 products and one sum, so with
    twin = |p| + |q| for its two products p, q:  |v - v64| <= U32 twin + U32 |fl(p) + fl(q)| <= 2 U32 (1 + U32) twin,
    + ETA32 for products that underflow.  Returns (ref, bound, touched) [B, C, hw]; the bound is 0 where not touched and
    z_renoise is not read there (nor where r == 0)."""
    B = x.shape[0]
    tt, rr = t.detach()[:B], r.detach()[:B]
    valid = ((tt >= 0) & (tt < T)).reshape(B, 1, 1)
    tc = tt.clamp(0, T - 1)
    col = lambda tab: _d(tab)[tc].reshape(B, 1, 1)
    xd = _d(x)
    ren = valid & (rr > 0).reshape(B, 1, 1)
    paste = valid & (_d(m) >= 0.5)
    zr = torch.where(ren, _d(z_renoise), torch.zeros((), dtype=F64, device=xd.device))   # NaN where not read is allowed
    p, q = col(ra) * xd, col(rb) * zr
    pk, qk = col(sqrt_acp) * _d(k), col(sqrt_1m_acp) * _d(z_known)
    c = 2 * U32 * (1 + U32)
    ref = torch.where(paste, pk + qk, torch.where(ren, p + q, xd))
    zero = torch.zeros((), dtype=F64, device=xd.device)
    bound = torch.where(paste, c * (pk.abs() + qk.abs()) + ETA32, torch.where(ren, c * (p.abs() + q.abs()) + ETA32, zero))
    return ref, bound, (paste | ren).expand(xd.shape)


# ---------------------------------------------------------------------------------------------- guidance weights
def scheduled_weights(w, w_sched, t, B):
    """image_scale (csrc/step.cu) as fp32 [B] on the CPU: w_b, or 1 + (w_b - 1) * w_sched[t_b] rounded op by op where the
    guidance table is not 1."""
    wt = w.detach().cpu().to(torch.float32) if torch.is_tensor(w) else torch.full((B,), _f32(w), dtype=torch.float32)
    if w_sched is None:
        return wt
    s = w_sched.detach().cpu()[t.detach().cpu()[:B]]
    return torch.where(s == 1, wt, 1 + (wt - 1) * s)


def guided_fp32(eps_cond, eps_null, w, w_sched, t, B, n):
    """The guided prediction g = null + (cond - null) * w_b(t) [B, n] exactly as the kernels form it in fp32 (three
    roundings, op by op), on the CPU."""
    c, nl = eps_cond.detach().cpu().reshape(B, n), eps_null.detach().cpu().reshape(B, n)
    return nl + (c - nl) * scheduled_weights(w, w_sched, t, B)[:, None]


def rescale_factor_ref(eps_cond, eps_null, w, w_sched, t, phi, B, n):
    """rescale_factor_kernel: f_b = phi_b sqrt(SS_c / SS_g) + (1 - phi_b) (1 where SS_g == 0), SS the sum of squares about
    the image mean, from the fp32 g the kernel forms (guided_fp32).  The kernel sums in fp64 over at most ~2^22 values per
    image and takes a chunked two-pass variance (Chan et al.), relative error ~ n U64 ~ 2^-31 on SS, so f is within its
    final rounding of the fp64 value plus a margin far below it: |f - f64| <= 2 U32 |f64| (one fp32 ulp).  Returns (f, bound)
    [B] in float64."""
    c = eps_cond.detach().cpu().reshape(B, n).to(F64)
    g = guided_fp32(eps_cond, eps_null, w, w_sched, t, B, n).to(F64)
    ssc = ((c - c.mean(dim=1, keepdim=True)) ** 2).sum(dim=1)
    ssg = ((g - g.mean(dim=1, keepdim=True)) ** 2).sum(dim=1)
    ph = phi.detach().cpu().to(F64).reshape(-1)[:B]
    f = torch.where(ssg == 0, torch.ones((), dtype=F64), ph * (ssc / ssg).sqrt() + (1. - ph))
    return f, 2 * U32 * f.abs() + ETA32


def rescaled_eps_fp32(eps_cond, eps_null, w, w_sched, t, f, B, n):
    """The prediction the rescaled step uses in place of g: fp32(g * f_b) [B, n] (g from guided_fp32), on the CPU."""
    return guided_fp32(eps_cond, eps_null, w, w_sched, t, B, n) * f.detach().cpu().reshape(-1)[:B, None]


def resize_ref(x, iy, wy, ix, wx, clamp=None):
    """resize_sep_kernel: out[p, y, x] = clamp(sum_j wx[x, j] sum_i wy[y, i] in[p, iy[y, i], ix[x, j]]) over the fp32 tap
    tables, x [P, Hin, Win].  The kernel's inner chain (ty products and sums from 0) and outer chain (one product, tx sums)
    round at most ty + tx + 1 times on any term's path; the clamp is 1-Lipschitz:
        |out - out64| <= (ty + tx + 2) U32 * twin + ETA32,   twin = the same sums over |w| and |in|.
    Returns (out, bound) [P, Hout, Wout]."""
    xd = _d(x).cpu()
    iy, ix = iy.detach().cpu().long(), ix.detach().cpu().long()
    wy, wx = _d(wy).cpu(), _d(wx).cpu()

    def sep(v, wyv, wxv):
        rows = (v[:, iy, :] * wyv[None, :, :, None]).sum(2)                 # [P, Hout, Win]
        return (rows[:, :, ix] * wxv[None, None, :, :]).sum(3)              # [P, Hout, Wout]
    ref, twin = sep(xd, wy, wx), sep(xd.abs(), wy.abs(), wx.abs())
    if clamp is not None:
        ref = ref.clamp(_f32(clamp[0]), _f32(clamp[1]))
    return ref, (iy.shape[1] + ix.shape[1] + 2) * U32 * twin + ETA32


def posemb_ref(t, dim):
    """posemb_kernel: out = cat(sin(arg), cos(arg)), arg_j = t exp(-j ln(1e4) / (half - 1)), half = dim / 2.  The kernel
    rounds the step ln(1e4) / (half - 1) to fp32 (U32), j * step once more (U32), then expf (2 ulp, 4 U32) and the product
    with t (U32): with e_j = j ln(1e4) / (half - 1) <= ln(1e4) the argument is off by
        |d arg| <= |arg| (2 U32 e_j + 6 U32),
    and sin / cos (1-Lipschitz) add their own 2 ulp (4 U32 |out|):
        |out - out64| <= |arg| (2 e_j + 6) U32 + 4 U32 |out64| + ETA32.     Returns (out, bound) [B, dim]."""
    half = dim // 2
    j = torch.arange(half, dtype=F64)
    e = j * (math.log(10000.0) / (half - 1))
    arg = _d(t).cpu()[:, None] * torch.exp(-e)[None, :]
    ref = torch.cat((arg.sin(), arg.cos()), dim=-1)
    darg = arg.abs() * (2 * e + 6) * U32
    return ref, torch.cat((darg, darg), dim=-1) + 4 * U32 * ref.abs() + ETA32


def text_pool_ref(rows):
    """text_tokens_kernel's pooled mean of the max_len conditioning rows it wrote, rows [B, max_len, D]: the kernel adds
    them one by one in fp32 from 0 (max_len - 1 roundings on the first row's path) and divides by max_len (one more):
        |pooled - mean64| <= max_len U32 mean(|rows|) + ETA32.
    Returns (mean, bound) [B, D]; `text_pool_fp32` is the same sum in the kernel's own order."""
    r = _d(rows).cpu()
    L = r.shape[1]
    return r.mean(dim=1), L * U32 * r.abs().mean(dim=1) + ETA32


def text_pool_fp32(rows):
    """The serial fp32 sum of the rows [B, max_len, D], then the division by max_len, in the kernel's order."""
    s = torch.zeros(rows.shape[0], rows.shape[2], dtype=torch.float32)
    for l in range(rows.shape[1]):
        s = s + rows[:, l].float().cpu()
    return s / float(rows.shape[1])
