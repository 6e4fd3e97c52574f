"""The float64 error bounds of tests/fp64_ref.py, proven on the CPU: the torch emulation of each kernel's contract
(tests/emu_ops.py) passes every bound, and each planted defect -- a kernel that is only subtly wrong -- fails it.  (The
fp16 saturation range is left to the GPU tests: the emulation converts with .to(float16), which gives inf there.)"""
import pytest
import torch

import fp64_ref as R
from emu_ops import EmuOps
from fp64_ref import check, check_rel_l2, half_out

F16 = torch.float16
EMU = EmuOps()


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _fails(out, ref, bound, what):
    with pytest.raises(AssertionError):
        check(out, ref, bound, what)


# ---------------------------------------------------------------------------------------------- attention
def _attention_case():
    B, heads, n, m = 2, 4, 256, 200                    # L = 201 keys: one key's probability is visible at fp16
    inner = heads * 64
    g = _g(1)
    q = (torch.randn(B * n, inner, generator=g) * 0.3).to(F16)
    kv = torch.randn(B * m, 2 * inner, generator=g)
    kv[:, inner:] += 2.0                               # values with a common offset: |o| ~ sum p |v|
    kv = kv.to(F16)
    null_kv = torch.randn(2, 64, generator=g)
    null_kv[1] -= 2.0
    mask = (torch.rand(B, m, generator=g) > 0.3).to(torch.uint8)
    args = (n * inner, inner, kv, kv[:, inner:], m * 2 * inner, 2 * inner, 64)
    return B, heads, n, m, inner, q, kv, null_kv, mask, args


def _emu_attention(q, args, null_kv, mask, B, heads, n, m, inner):
    o = torch.zeros(B * n, inner, dtype=F16)
    EMU.attention(q, *args, null_kv, mask, B, heads, n, m, o, n * inner, inner)
    return o


def test_attention_bound():
    B, heads, n, m, inner, q, kv, null_kv, mask, args = _attention_case()
    o = _emu_attention(q, args, null_kv, mask, B, heads, n, m, inner)
    qv, kk, vv = R.attention_views(q, *args, B, heads, n, m)
    nk16 = null_kv.to(F16).float()
    ref, bound = R.attention_ref(qv, kk, vv, nk16, mask)
    view = lambda t: t.reshape(B, n, heads, 64).permute(0, 2, 1, 3)
    check(view(o), ref, bound, "attention (emulation)")

    # 1. the highest-scoring masked key of (b, h) = (0, 1) takes part
    b, h = 0, 1
    s = qv[b, h].float() @ kk[b, h].float().t()                               # [n, m]
    s[:, mask[b] != 0] = -float("inf")
    j = int(s.amax(dim=0).argmax())
    mk = mask.clone()
    mk[b, j] = 1
    o2 = _emu_attention(q, args, null_kv, mk, B, heads, n, m, inner)
    d = o.clone()
    d[b * n:(b + 1) * n, h * 64:(h + 1) * 64] = o2[b * n:(b + 1) * n, h * 64:(h + 1) * 64]
    _fails(view(d), ref, bound, "masked key unmasked")

    # 2. the null key left out of the row where it weighs most
    sn = qv.float() @ nk16[0]                                                  # [B, h, n]
    b, h, r = (int(i) for i in torch.unravel_index(sn.reshape(-1).argmax(), sn.shape))
    s = qv[b, h, r].float() @ kk[b, h].float().t()
    s[mask[b] == 0] = -float("inf")
    d = o.clone()
    d[b * n + r, h * 64:(h + 1) * 64] = (torch.softmax(s, dim=0) @ vv[b, h].float()).to(F16)
    _fails(view(d), ref, bound, "null key dropped")

    # 3. another head's output in one query row
    d = o.clone()
    d[n + 5, 2 * 64:3 * 64] = o[n + 5, 3 * 64:4 * 64]
    _fails(view(d), ref, bound, "other head's row")

    # 4. a 1 % error confined to one 128-row query tile
    d = o.clone()
    d[128:256, 0:64] = (d[128:256, 0:64].float() * 1.01).to(F16)
    _fails(view(d), ref, bound, "1% error in one query tile")


def test_attention_fn_bound(emu):
    """AttentionFn (fp32 GEMMs + row softmax) forward and backward on the emulated ops vs float64 autograd."""
    from minimagen_b200.autograd import AttentionFn
    g = _g(2)
    for hk in (4, 1):
        B, heads, n, m = 2, 4, 40, 17
        q = (torch.randn(B, n, heads * 64, generator=g) * 0.125).requires_grad_(True)
        k = torch.randn(B, m, hk * 64, generator=g).requires_grad_(True)
        v = torch.randn(B, m, hk * 64, generator=g).requires_grad_(True)
        nk = torch.randn(2, 64, generator=g).requires_grad_(True)
        do = torch.randn(B, n, heads * 64, generator=g)
        o = AttentionFn.apply(q, k, v, nk, heads)
        got = dict(zip(("dq", "dk", "dv", "dnull"), torch.autograd.grad(o, (q, k, v, nk), do)), o=o)
        for name, (ref, bound) in R.attention_fn_ref(q, k, v, nk, heads, do).items():
            check(got[name], ref, bound, f"AttentionFn {name} (hk={hk}, emulation)")


# ---------------------------------------------------------------------------------------------- LayerNorm
def _ln_inputs(Rr, C, seed):
    g = _g(seed)
    x = torch.randn(Rr, C, generator=g) * 3 + 1
    x[3] = 2.5 + 1e-4 * torch.randn(C, generator=g)          # near-constant row: variance 1e-8 << eps
    return x, torch.randn(C, generator=g), torch.randn(C, generator=g), torch.randn(Rr, C, generator=g)


@pytest.mark.parametrize("pre_gelu", [0, 1])
def test_ln_rows_bound(pre_gelu):
    Rr, C, eps = 40, 256, 1e-5
    x, gamma, beta, res = _ln_inputs(Rr, C, 3)
    o, o16 = torch.zeros(Rr, C), torch.zeros(Rr, C, dtype=F16)
    EMU.ln_rows(x, Rr, C, gamma, beta, eps, pre_gelu, res, o, o16)
    ref, bound = R.ln_ref(x, gamma, beta, eps, pre_gelu, res)
    check(o, ref, bound, "ln_rows fp32 (emulation)")
    check(o16, *half_out(ref, bound), "ln_rows fp16 (emulation)")

    v = torch.nn.functional.gelu(x.double()) if pre_gelu else x.double()
    mu, var = v.mean(dim=1, keepdim=True), v.var(dim=1, unbiased=False, keepdim=True)
    g64, b64 = gamma.double(), beta.double() + res.double()

    def row(i, mean, denom, gam):
        d = o.clone()
        d[i] = ((v[i] - mean) / denom * gam + b64[i]).float()
        return d
    _fails(row(7, mu[8], (var[7] + eps).sqrt(), g64), ref, bound, "neighbouring row's mean")
    _fails(row(3, mu[3], var[3].sqrt(), g64), ref, bound, "eps ignored on a near-constant row")
    _fails(row(11, mu[11], (var[11] + eps).sqrt(), g64.roll(1)), ref, bound, "gamma shifted by one channel")


@pytest.mark.parametrize("pre_gelu", [0, 1])
def test_ln_rows_bwd_bound(pre_gelu):
    Rr, C, eps = 300, 48, 1e-5
    x, gamma, _, dy = _ln_inputs(Rr, C, 4)
    dg0, db0 = torch.randn(C, generator=_g(5)), torch.randn(C, generator=_g(6))
    dx, dg, db = torch.zeros(Rr, C), dg0.clone(), db0.clone()
    EMU.ln_rows_bwd(x, dy, Rr, C, gamma, eps, pre_gelu, dx, dg, db)
    (rx, bx), (rg, bg), (rb, bb) = R.ln_bwd_ref(x, dy, gamma, eps, pre_gelu, dg0, db0, R.ln_bwd_acc_len(Rr, 132))
    check(dx, rx, bx, "ln_rows_bwd dx (emulation)")
    check(dg, rg, bg, "ln_rows_bwd dgamma (emulation)")
    check(db, rb, bb, "ln_rows_bwd dbeta (emulation)")
    v = torch.nn.functional.gelu(x.double()) if pre_gelu else x.double()
    xh = (v - v.mean(dim=1, keepdim=True)) / (v.var(dim=1, unbiased=False, keepdim=True) + eps).sqrt()
    r = int((dy[:, 5] * xh[:, 5]).abs().argmax())
    d = dg.clone()
    d[5] -= float(dy[r, 5] * xh[r, 5])
    _fails(d, rg, bg, "one row missing from the dgamma sum")


# ---------------------------------------------------------------------------------------------- linear / GEMM
@pytest.mark.parametrize("M,K,N,in_act,out_act,add,scale", [(37, 36, 131, 1, 0, True, 0.5), (5, 1028, 77, 0, 1, False, 1.0),
                                                            (77, 4, 1001, 1, 1, True, -3.0)])
def test_linear_bound(M, K, N, in_act, out_act, add, scale):
    g = _g(M + K + N)
    x, w, b = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) * K ** -0.5, torch.randn(N, generator=g)
    a = torch.randn(M, N, generator=g) if add else None
    o, o16 = torch.zeros(M, N), torch.zeros(M, N, dtype=F16)
    EMU.linear_f32(x, M, K, w, b, N, in_act, out_act, a, o, o16, scale)
    ref, bound = R.linear_ref(x, w, b, in_act, out_act, a, scale)
    check(o, ref, bound, "linear_f32 fp32 (emulation)")
    check(o16, *half_out(ref, bound), "linear_f32 fp16 (emulation)")

    def col(j, kk, bias):
        xa = torch.nn.functional.silu(x) if in_act else x
        y = xa[:, :kk] @ w[j, :kk] + bias + (a[:, j] if add else 0)
        y = torch.nn.functional.silu(y) if out_act else y
        d = o.clone()
        d[:, j] = y * scale
        return d
    if K > 32:
        _fails(col(17, (K - 1) // 32 * 32, b[17]), ref, bound, "last partial K chunk dropped")
    _fails(col(5, K, 0.0), ref, bound, "bias dropped in one column")


LAYOUTS = [(True, True), (True, False), (False, True), (False, False)]


@pytest.mark.parametrize("a_kfast,b_nfast", LAYOUTS)
def test_gemm_bound(a_kfast, b_nfast):
    Z1, Z2, M, N, K, alpha = 2, 3, 65, 130, 17, 0.37
    g = _g(7)
    A = torch.randn(Z1 * Z2 * M * K + 5, generator=g)
    B = torch.randn(Z1 * Z2 * K * N + 3, generator=g)
    a_str = (K, 1) if a_kfast else (1, M)
    b_str = (N, 1) if b_nfast else (1, K)
    a_b, b_b, c_b = (Z2 * M * K, M * K), (Z2 * K * N, K * N), (Z2 * M * N, M * N)
    C = torch.randn(Z1 * Z2 * M * N, generator=g)
    view = lambda t, sh, st, bb: t.as_strided((Z1, Z2) + sh, bb + st)
    Av, Bv = view(A, (M, K), a_str, a_b), view(B, (K, N), b_str, b_b)
    C0 = view(C, (M, N), (N, 1), c_b).clone()
    EMU.gemm_f32(A, B, C, M, N, K, a_str, b_str, (N, 1), Z1, Z2, a_b, b_b, c_b, alpha=alpha, accumulate=True)
    out = view(C, (M, N), (N, 1), c_b)
    ref, bound = R.gemm_ref(Av, Bv, C0, alpha, True)
    check(out, ref, bound, "gemm_f32 (emulation)")
    d = out.clone()
    d[1, 2, :64, 64:128] = C0[1, 2, :64, 64:128] + Av[1, 2, :64] @ Bv[1, 2, :, 64:128]
    _fails(d, ref, bound, "alpha ignored in one 64x64 tile")
    _fails(out - C0, ref, bound, "overwrite instead of accumulate")


def test_colsum_bound():
    M, N = 5000, 37
    g = _g(8)
    x, out0 = torch.randn(M, N, generator=g), torch.randn(N, generator=g)
    out = out0.clone()
    EMU.colsum(x, M, N, out, accumulate=True)
    check(out, *R.colsum_ref(x, out0, R.colsum_acc_len(M)), "colsum (emulation)")


# ---------------------------------------------------------------------------------------------- softmax rows
@pytest.mark.parametrize("L", [18, 259])
def test_softmax_bounds(L):
    Rr = 50
    g = _g(L)
    s = torch.randn(Rr, L, generator=g) * 3
    p = s.clone()
    EMU.softmax_rows(p, Rr, L)
    check(p, *R.softmax_ref(s), "softmax_rows (emulation)")
    dP = torch.randn(Rr, L, generator=g) + 1.0
    dS = dP.clone()
    EMU.softmax_rows_bwd(p, dS, Rr, L)
    ref, bound = R.softmax_bwd_ref(p, dP)
    check(dS, ref, bound, "softmax_rows_bwd (emulation)")
    d = dS.clone()
    d[7] = p[7] * dP[7]
    _fails(d, ref, bound, "-sum P dP left out of one row")


# ---------------------------------------------------------------------------------------------- whole-tensor checks
def test_rel_l2_catches_uniform_errors():
    """Errors spread evenly over a whole tensor can stay inside the elementwise worst-case bounds at long accumulations
    and zero-mean values; the rel-L2 limits that sit next to them in the GPU tests (check_rel_l2) reject them, while the
    emulation passes those limits."""
    g = _g(11)
    # fp32 linear at K = 1024 computed from fp16-rounded operands
    M, K, N = 32, 1024, 2048
    x, w, b = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) * K ** -0.5, torch.randn(N, generator=g)
    ref, bound = R.linear_ref(x, w, b, 1, 0, None, 0.125)
    o = torch.zeros(M, N)
    EMU.linear_f32(x, M, K, w, b, N, 1, 0, None, o, None, 0.125)
    check_rel_l2(o, ref, 2e-6, "linear_f32 (emulation)")
    xh, wh = torch.nn.functional.silu(x).half().double(), w.half().double()
    d = ((xh @ wh.t() + b.double()) * 0.125).float()
    check(d, ref, bound, "linear_f32 with fp16 operands (inside the elementwise bound)")
    with pytest.raises(AssertionError):
        check_rel_l2(d, ref, 2e-6, "planted: linear_f32 with fp16 operands")
    # LayerNorm with a uniform 1e-4 relative error
    Rr, C = 513, 1024
    x, gamma = torch.randn(Rr, C, generator=g) * 3 + 1, torch.randn(C, generator=g)
    ref, bound = R.ln_ref(x, gamma, None, 1e-5, 1, None)
    o = torch.zeros(Rr, C)
    EMU.ln_rows(x, Rr, C, gamma, None, 1e-5, 1, None, o, None)
    check_rel_l2(o, ref, 3e-6, "ln_rows (emulation)")
    with pytest.raises(AssertionError):
        check_rel_l2(o * (1 + 1e-4), ref, 3e-6, "planted: ln_rows 1e-4 relative error")
    # attention with zero-mean values and a 1 % error over the whole output
    B, heads, n, m = 1, 2, 1024, 1024
    q = (torch.randn(B * n, heads * 64, generator=g) * 0.125).to(F16)
    kv = torch.randn(B * m, 128, generator=g).to(F16)
    null_kv = torch.randn(2, 64, generator=g)
    args = (n * heads * 64, heads * 64, kv, kv[:, 64:], m * 128, 128, 0)
    o = _emu_attention(q, args, null_kv, None, B, heads, n, m, heads * 64)
    ref, bound = R.attention_ref(*R.attention_views(q, *args, B, heads, n, m), null_kv.to(F16).float())
    view = lambda t: t.reshape(B, n, heads, 64).permute(0, 2, 1, 3)
    check_rel_l2(view(o), ref, 2e-3, "attention (emulation)")
    with pytest.raises(AssertionError):
        check_rel_l2(view(o).float() * 1.01, ref, 2e-3, "planted: attention 1% error over the whole output")
    # fp32 data gradient of a 3x3 conv over 128 output channels computed from fp16-rounded dy
    B, Ho, Wo, Co, Ci = 2, 16, 16, 128, 32
    dy, w = torch.randn(B, Ho, Wo, Co, generator=g), torch.randn(Co, Ci, 3, 3, generator=g) * 0.05
    ref, bound = R.conv_dgrad_ref(dy, w, 1, 1, Ho, Wo)
    dx = torch.zeros(B, Ho, Wo, Ci)
    EMU.conv_dgrad(dy, B, Ho, Wo, Co, w, Ci, 3, 3, 1, 1, dx, Ho, Wo)
    check_rel_l2(dx, ref, 2e-5, "conv_dgrad (emulation)")
    d = torch.zeros(B, Ho, Wo, Ci)
    EMU.conv_dgrad(dy.half().float(), B, Ho, Wo, Co, w, Ci, 3, 3, 1, 1, d, Ho, Wo)
    check(d, ref, bound, "conv_dgrad with fp16-rounded dy (inside the elementwise bound)")
    with pytest.raises(AssertionError):
        check_rel_l2(d, ref, 2e-5, "planted: conv_dgrad with fp16-rounded dy")


# ---------------------------------------------------------------------------------------------- GroupNorm/FiLM/SiLU backward
def _gn_case():
    B, H, W, C, G, eps = 2, 24, 20, 48, 8, 1e-5                  # Cg = 6: groups straddle the kernel's channel quads
    g = _g(12)
    x = torch.randn(B, H * W, C, generator=g) * 2 + 0.5
    x[0, :, 12:18] = 2.5 + 1e-4 * torch.randn(H * W, 6, generator=g)      # image 0, group 2: near-constant (var << eps)
    x[1, :, 30:36] = 100.0 + torch.randn(H * W, 6, generator=g)          # image 1, group 5: |mean| / std ~ 100
    dy = torch.randn(B, H * W, C, generator=g)
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    ss = torch.randn(B, 2 * C, generator=g) * 0.3
    dg0, db0 = torch.randn(C, generator=g), torch.randn(C, generator=g)
    xd = x.double().reshape(B, H * W, G, C // G)
    sums = torch.stack((xd.sum(dim=(1, 3)), (xd * xd).sum(dim=(1, 3))), dim=-1)          # [B, G, 2], as gn_stats makes them
    return B, H * W, C, G, eps, x, dy, gamma, beta, ss, dg0, db0, sums


def _gn_bwd_fp32(x, dy, sums, gamma, beta, ss, G, eps, dg0, db0, Z, defect=None):
    """The three passes of gn_silu_bwd (csrc/backward.cu) restated in fp32 torch, Z pixel splits; `defect` plants one
    subtle mistake.  Returns dx, dgamma, dbeta, dscale, dshift."""
    B, HW, C = x.shape
    Cg, n = C // G, (C // G) * HW
    m = sums[..., 0] / n
    var = (sums[..., 1] / n - m * m).clamp(min=0)
    rstd = 1.0 / torch.sqrt(var + eps)
    if defect == "eps ignored":                                             # on the near-constant group (image 0, group 2)
        rstd[0, 2] = 1.0 / torch.sqrt(var[0, 2])
    mean_c = m.float().repeat_interleave(Cg, dim=1)[:, None]
    rstd_c = rstd.float().repeat_interleave(Cg, dim=1)[:, None]
    sc, sh = (ss[:, None, :C] + 1.0), ss[:, None, C:]
    xn = (x - mean_c) * rstd_c
    v = (xn * gamma + beta) * sc + sh
    if defect == "silu' before FiLM":                                       # in channel 7
        v[..., 7] = xn[..., 7] * gamma[7] + beta[7]
    sg = torch.sigmoid(v)
    dv = dy * (sg * (1.0 + v * (1.0 - sg)))
    chunk = -(-HW // Z)
    A1 = sum(dv[:, z * chunk:(z + 1) * chunk].sum(dim=1) for z in range(Z))
    A2 = sum((dv * xn)[:, z * chunk:(z + 1) * chunk].sum(dim=1) for z in range(Z))
    if defect == "split missing":                                           # the second split of (b, c) = (1, 20)
        A1[1, 20] -= dv[1, chunk:2 * chunk, 20].sum()
        A2[1, 20] -= (dv * xn)[1, chunk:2 * chunk, 20].sum()
    sc, sh = sc[:, 0], sh[:, 0]
    dscale, dshift = gamma * A2 + beta * A1, A1.clone()
    if defect == "dss swapped":                                             # in image 1
        dscale[1], dshift[1] = A1[1], gamma * A2[1] + beta * A1[1]
    dg, db = dg0 + (sc * A2).sum(dim=0), db0 + (sc * A1).sum(dim=0)
    grp = lambda t: t.reshape(B, G, Cg).sum(dim=2) / n
    m1, m2 = grp(gamma * sc * A1), grp(gamma * sc * A2)
    if defect == "neighbour's m1":                                          # image 1, group 3 takes group 4's m1
        m1[1, 3] = m1[1, 4]
    m1c, m2c = m1.repeat_interleave(Cg, dim=1)[:, None], m2.repeat_interleave(Cg, dim=1)[:, None]
    dx = rstd_c * ((gamma * sc)[:, None] * dv - m1c - xn * m2c)
    return dx, dg, db, dscale, dshift


GN_OUTS = ("dx", "dgamma", "dbeta", "dscale", "dshift")


def test_gn_silu_bwd_bound():
    B, HW, C, G, eps, x, dy, gamma, beta, ss, dg0, db0, sums = _gn_case()
    Z = R.gn_bwd_splits(B, HW, C, 132)
    assert Z > 1
    refs = R.gn_silu_bwd_ref(x, dy, gamma, beta, ss, G, eps, dg0, db0, R.gn_bwd_acc_len(B, HW, C, 132))
    # the emulation (float32 autograd through F.group_norm); the near-constant group is left out of the aggregate: its
    # elementwise bound is large by nature (rstd ~ eps^-1/2 magnifies the fp32 mean's rounding)
    dx, dg, db, dss = torch.zeros(B, HW, C), dg0.clone(), db0.clone(), torch.zeros(B, 2 * C)
    EMU.gn_silu_bwd(x, dy, sums, B, HW, C, G, gamma, beta, ss, 2 * C, eps, dx, dg, db, dss, 2 * C)
    agg_x, agg_c, agg_bc = torch.ones(B, HW, C, dtype=torch.bool), torch.ones(C, dtype=torch.bool), torch.ones(B, C, dtype=torch.bool)
    agg_x[0, :, 12:18], agg_c[12:18], agg_bc[0, 12:18] = False, False, False
    for name, out, (ref, bound), agg in zip(GN_OUTS, (dx, dg, db, dss[:, :C], dss[:, C:]), refs,
                                            (agg_x, agg_c, agg_c, agg_bc, agg_bc)):
        check(out, ref, bound, f"gn_silu_bwd {name} (emulation)")
        check_rel_l2(out[agg], ref[agg], 5e-5, f"gn_silu_bwd {name} (emulation)")
    # the kernel's own three passes in fp32, then each planted defect
    outs = _gn_bwd_fp32(x, dy, sums, gamma, beta, ss, G, eps, dg0, db0, Z)
    for name, out, (ref, bound) in zip(GN_OUTS, outs, refs):
        check(out, ref, bound, f"gn_silu_bwd {name} (fp32 restatement)")
    for defect, which in (("split missing", "dbeta"), ("split missing", "dx"), ("neighbour's m1", "dx"),
                          ("silu' before FiLM", "dx"), ("silu' before FiLM", "dgamma"), ("dss swapped", "dscale"),
                          ("eps ignored", "dx")):
        i = GN_OUTS.index(which)
        out = _gn_bwd_fp32(x, dy, sums, gamma, beta, ss, G, eps, dg0, db0, Z, defect)[i]
        _fails(out, *refs[i], f"gn_silu_bwd {which}: {defect}")


# ---------------------------------------------------------------------------------------------- convolution gradients
def _wgrad_case(stride, k):
    B, Ho, Wo, Ci, Co = 2, 16, 24, 64, 128
    g = _g(13 + k)
    x16 = torch.randn(B, stride * Ho, stride * Wo, Ci, generator=g).to(F16)
    dy16 = torch.randn(B, Ho, Wo, Co, generator=g).to(F16)
    return B, Ho, Wo, Ci, Co, x16, dy16


@pytest.mark.parametrize("stride,k", [(1, 3), (2, 4)])
def test_conv_wgrad_bound(stride, k):
    """The weight-gradient bound at the tensor-core kernel's summation length, on the emulation of mi_conv2d_wgrad_f16."""
    B, Ho, Wo, Ci, Co, x16, dy16 = _wgrad_case(stride, k)
    pad = 1 if stride == 2 else k // 2
    per, splits = R.wgrad_tc_plan(B, Ho, Wo, Ci, Co, k, 132)
    assert splits > 1
    ref, bound = R.conv_wgrad_ref(dy16, x16, stride, pad, k, k, R.wgrad_tc_acc_len(B, Ho, Wo, Ci, Co, k, 132))
    dw = torch.zeros(Co, Ci, k, k)
    EMU.conv_wgrad_tc(dy16, x16, B, Ho, Wo, Ci, Co, k, k, dw, stride)
    check(dw, ref, bound, f"conv_wgrad_tc stride {stride} k {k} (emulation)")
    check_rel_l2(dw, ref, 1e-5, f"conv_wgrad_tc stride {stride} k {k} (emulation)")

    def without(keep):
        """dW of the pixels where `keep` [B, Ho, Wo] is True only"""
        return R.conv_wgrad_ref(dy16 * keep[..., None], x16, stride, pad, k, k, 1)[0].float()
    boxes = torch.zeros(B, Ho // 8, Wo // 8, dtype=torch.bool)
    boxes.view(-1)[per:2 * per] = True                                                # the second split's 8x8 boxes
    split = boxes.repeat_interleave(8, dim=1).repeat_interleave(8, dim=2)
    d = dw.clone()
    d[:, :, 0, 1] -= without(split)[:, :, 0, 1]
    _fails(d, ref, bound, "one split missing from tap (0, 1)")
    last = torch.zeros(B, Ho, Wo, dtype=torch.bool)
    last[1, -8:, -8:] = True
    _fails(dw - without(last), ref, bound, "last 8x8 box of image 1 dropped")
    # the zero padding above the image replaced by the first row (a tap shift that is wrong at the border only)
    xp = torch.nn.functional.pad(x16.float().permute(0, 3, 1, 2), (pad, pad, pad, pad))
    xp[:, :, 0] = xp[:, :, 1]
    d = torch.nn.grad.conv2d_weight(xp, (Co, Ci, k, k), dy16.float().permute(0, 3, 1, 2), stride=stride)
    _fails(d, ref, bound, "top border padding replaced by the neighbouring row")


@pytest.mark.parametrize("stride,k,Co", [(1, 3, 40), (2, 4, 40), (1, 3, 3)])
def test_conv_dgrad_bound(stride, k, Co):
    B, Ho, Wo, Ci = 2, 12, 10, 24
    pad = 1 if stride == 2 else k // 2
    Hi, Wi = stride * Ho, stride * Wo
    g = _g(14 + k + Co)
    dy = torch.randn(B, Ho, Wo, Co, generator=g)
    w = torch.randn(Co, Ci, k, k, generator=g) * 0.2
    dx = torch.zeros(B, Hi, Wi, Ci)
    EMU.conv_dgrad(dy, B, Ho, Wo, Co, w, Ci, k, k, stride, pad, dx, Hi, Wi)
    ref, bound = R.conv_dgrad_ref(dy, w, stride, pad, Hi, Wi)
    what = f"conv_dgrad stride {stride} k {k} C_out {Co}"
    check(dx, ref, bound, what + " (emulation)")
    check_rel_l2(dx, ref, 2e-5, what + " (emulation)")
    last = torch.zeros_like(dy)
    last[:, :, -1] = dy[:, :, -1]
    _fails(dx - R.conv_dgrad_ref(last, w, stride, pad, Hi, Wi)[0].float(), ref, bound, what + ": last dy column dropped")
    wf = w.clone()
    wf[:, 5] = w[:, 5].flip(1, 2)
    d = dx.clone()
    d[..., 5] = R.conv_dgrad_ref(dy, wf, stride, pad, Hi, Wi)[0][..., 5].float()
    _fails(d, ref, bound, what + ": taps of channel 5 not flipped")
    if stride == 2:
        d = dx.clone()
        d[1, 0::2, 0::2], d[1, 0::2, 1::2] = dx[1, 0::2, 1::2], dx[1, 0::2, 0::2]
        _fails(d, ref, bound, what + ": output parities (0, 0) and (0, 1) of image 1 swapped")


def test_upsample2x_bwd_order():
    """upsample2x_bwd is a fixed-order sum of four fp32 values: the emulation matches it bit for bit, another order does not."""
    B, H, W, C = 2, 5, 7, 64
    dy = torch.randn(B, 2 * H, 2 * W, C, generator=_g(15)) * 1e3
    dx = torch.zeros(B, H, W, C)
    EMU.upsample2x_bwd(dy, B, H, W, C, dx)
    ref = R.upsample2x_bwd_ref(dy)
    assert torch.equal(dx, ref)
    q = dy.reshape(B, H, 2, W, 2, C)
    assert not torch.equal((q[:, :, 0, :, 0] + q[:, :, 1, :, 0]) + (q[:, :, 0, :, 1] + q[:, :, 1, :, 1]), ref)
