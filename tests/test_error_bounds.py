"""The float64 error bounds of tests/fp64_ref.py, proven on the CPU: the torch emulation of each kernel's contract
(tests/emu_ops.py) passes every bound, and each planted defect -- a kernel that is only subtly wrong -- fails it.  Where the
emulation's arithmetic differs from the kernel's in structure (the conv epilogue's statistics, gn_stats's chains, the
GroupNorm coefficient fold), an fp32 restatement of the kernel's own order passes the bound too."""
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


# ---------------------------------------------------------------------------------------------- convolution forward
F64 = torch.float64


def _conv_operands(B, H, W, Cin, Cout, k, mode, seed, C1=0):
    """fp16 operand(s) in the layout of `mode`, the OIHW fp32 weight, bias, residual"""
    g = _g(seed)
    lead = (B, 2 * H, 2 * W) if mode == 6 else (B, 4, H, W) if mode == 1 else (B, H, W)
    a0 = torch.randn(*lead, Cin, generator=g).to(F16)
    a1 = torch.randn(*lead, C1, generator=g).to(F16) if C1 else None
    w = torch.randn(Cout, Cin + C1, k, k, generator=g) * (k * k * (Cin + C1)) ** -0.5
    return a0, a1, w, torch.randn(Cout, generator=g), torch.randn(B, H, W, Cout, generator=g)


def _emu_conv(a0, a1, wp, B, H, W, Cout, k, mode, bias, res, stats=True):
    o, o16 = torch.zeros(B, H, W, Cout), torch.zeros(B, H, W, Cout, dtype=F16)
    st = torch.zeros(B, Cout // 16, 2, dtype=F64) if stats else None
    kw = dict(act2=a1, lda2=a1.shape[-1], c_in1=a0.shape[-1]) if a1 is not None else {}
    Cin = a0.shape[-1] + (a1.shape[-1] if a1 is not None else 0)
    EMU.conv_igemm(a0, B, H, W, a0.shape[-1], 0, Cin, wp, Cout, k, k, mode, bias, res, o, o16,
                   (H * W * Cout, W * Cout, Cout), out_stats=st, **kw)
    return o, o16, st


def _epilogue_stats_fp32(out32):
    """The conv epilogue's statistics in the kernel's own order (csrc/conv_tc.cu): lane 4 rr + cc of a warp holds rows
    rr, rr + 8 of its 16 and columns 8 jj + 2 cc + e of each 16-channel block; it adds its two column pairs (j = 2q, 2q + 1)
    of both rows in fp32, pair sums first; five xor-shuffle levels add the 32 lanes in fp32; warps are added in fp64."""
    B, C = out32.shape[0], out32.shape[-1]
    f = out32.float().reshape(B, -1, 2, 8, C // 16, 2, 4, 2)          # [B, warp, r, rr, q, jj, cc, e]
    ps = f[..., 0] + f[..., 1]
    pq = f[..., 0] * f[..., 0] + f[..., 1] * f[..., 1]
    lanes = torch.arange(32)
    out = []
    for p in (ps, pq):
        t = ((p[:, :, 0, :, :, 0] + p[:, :, 1, :, :, 0]) + p[:, :, 0, :, :, 1]) + p[:, :, 1, :, :, 1]   # [B, warp, rr, q, cc]
        t = t.permute(0, 1, 3, 2, 4).reshape(B, -1, C // 16, 32)
        for o in (1, 2, 4, 8, 16):
            t = t + t[..., lanes ^ o]
        out.append(t[..., 0].double().sum(dim=1))
    return torch.stack(out, dim=-1)


CONV_FWD_CASES = [
    # B, H, W, C_in, C_out, k, mode
    (2, 16, 16, 128, 64, 3, 0), (3, 8, 8, 64, 32, 1, 0), (2, 8, 16, 64, 32, 4, 1), (2, 8, 8, 64, 32, 4, 6),
    (2, 8, 8, 64, 32, 2, 2), (1, 4, 136, 64, 32, 3, 0),
]


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,mode", CONV_FWD_CASES)
def test_conv_fwd_bound(B, H, W, Cin, Cout, k, mode):
    """The emulation of mi_conv2d_igemm_f16 (fp32 and fp16 outputs, block statistics) passes conv_fwd_ref / conv_stats_ref,
    and the kernel-ordered fp32 statistics of the same output pass conv_stats_ref.  Modes 2..5 write one interleaved
    2H x 2W output."""
    a0, _, w, bias, res = _conv_operands(B, H, W, Cin, Cout, k, mode, seed=20 + mode + k)
    what = f"conv mode {mode} k {k} {H}x{W}"
    if mode == 2:
        o, o16 = torch.zeros(B, 2 * H, 2 * W, Cout), torch.zeros(B, 2 * H, 2 * W, Cout, dtype=F16)
        ref, bound = torch.zeros(B, 2 * H, 2 * W, Cout, dtype=F64), torch.zeros(B, 2 * H, 2 * W, Cout, dtype=F64)
        st = torch.zeros(B, Cout // 16, 2, dtype=F64)
        strides = (4 * H * W * Cout, 4 * W * Cout, 2 * Cout)
        for p in range(4):
            wp = EMU.pack_conv_weight(w + 0.1 * p)
            off = ((p >> 1) * 2 * W + (p & 1)) * Cout
            EMU.conv_igemm(a0, B, H, W, Cin, 0, Cin, wp, Cout, 2, 2, 2 + p, bias, None, o.view(-1)[off:], o16.view(-1)[off:],
                           strides, out_stats=st)
            r, bd = R.conv_fwd_ref(a0, wp, 2, 2, 2 + p, bias)
            ref[:, p >> 1::2, p & 1::2], bound[:, p >> 1::2, p & 1::2] = r, bd
    else:
        wp = EMU.pack_conv_weight(w)
        o, o16, st = _emu_conv(a0, None, wp, B, H, W, Cout, k, mode, bias, res)
        ref, bound = R.conv_fwd_ref(a0, wp, k, k, mode, bias, res)
    check(o, ref, bound, what + " (emulation)")
    check_rel_l2(o, ref, 2e-5, what + " (emulation)")
    check(o16, *half_out(ref, bound), what + " fp16 (emulation)")
    check_rel_l2(o16, ref, 1e-3, what + " fp16 (emulation)")
    sref, sbound = R.conv_stats_ref(o)
    check(st, sref, sbound, what + " statistics (emulation)")
    check(_epilogue_stats_fp32(o), sref, sbound, what + " statistics (fp32 restatement)")
    if mode == 2:
        d = o.clone()
        d[1, 0::2, 1::2], d[1, 1::2, 0::2] = o[1, 1::2, 0::2], o[1, 0::2, 1::2]
        _fails(d, ref, bound, what + ": sub-pixel phases (0, 1) and (1, 0) of image 1 swapped")
    if W == 136:
        # the masked columns 136..255 of each row's second 128-pixel tile counted with their bias value (acc = 0)
        d = st.clone()
        nb = (256 - W) * H
        bb = bias.double().reshape(-1, 16)
        d[..., 0] += nb * bb.sum(dim=1)
        d[..., 1] += nb * (bb * bb).sum(dim=1)
        _fails(d, sref, sbound, what + ": masked ragged-W rows counted")


def test_conv_fwd_defects():
    """Planted defects of the implicit-GEMM conv and its statistics fail the bounds (3x3, C_in = 128: two 64-channel
    k-blocks per tap; 16 x 16 images: a 128-pixel tile is 8 rows of one image)."""
    B, H, W, Cin, Cout, k = 2, 16, 16, 128, 64, 3
    a0, _, w, bias, res = _conv_operands(B, H, W, Cin, Cout, k, 0, seed=30)
    wp = EMU.pack_conv_weight(w)
    o, _, st = _emu_conv(a0, None, wp, B, H, W, Cout, k, 0, bias, res)
    ref, bound = R.conv_fwd_ref(a0, wp, k, k, 0, bias, res)
    check(o, ref, bound, "conv 3x3 (emulation)")
    w64 = R.unpack_conv_weight(wp, k, k, Cin)
    a64 = a0.double()
    # 1. the second k-block (channels 64..127) of tap (1, 2) missing in the first tile of image 1
    wpart = torch.zeros_like(w64)
    wpart[:, 64:, 1, 2] = w64[:, 64:, 1, 2]
    d = o.clone()
    d[1, :8] -= R.conv_nhwc(a64, wpart, 0)[1, :8].float()
    _fails(d, ref, bound, "one k-block of one tap missing in one tile")
    # 2. the right-border taps read the first pixel of the next row instead of the zero padding
    xp = torch.nn.functional.pad(a64.permute(0, 3, 1, 2), (1, 1, 1, 1))
    xp[:, :, 1:H, W + 1] = xp[:, :, 2:H + 1, 1]
    d = (torch.nn.functional.conv2d(xp, w64).permute(0, 2, 3, 1) + bias.double() + res.double()).float()
    _fails(d, ref, bound, "right-border tap reads the next row")
    # 3. the bias shifted by one 16-channel block
    _fails(o - bias + bias.roll(16), ref, bound, "bias shifted by one 16-channel block")
    # statistics: 4. one warp's 16 rows missing from block 1 of image 0; 5. the first tile of image 0 credited to image 1
    sref, sbound = R.conv_stats_ref(o)
    f = o.double().reshape(B, H * W, Cout)
    d = st.clone()
    d[0, 1, 0] -= f[0, 16:32, 16:32].sum()
    d[0, 1, 1] -= (f[0, 16:32, 16:32] ** 2).sum()
    _fails(d, sref, sbound, "one warp's 16 rows missing from one statistics block")
    t = f[0, :128].reshape(128, Cout // 16, 16)
    ts = torch.stack((t.sum(dim=(0, 2)), (t * t).sum(dim=(0, 2))), dim=-1)
    d = st.clone()
    d[0] -= ts
    d[1] += ts
    _fails(d, sref, sbound, "a tile's statistics added to image b + 1")


def test_conv_fwd_concat_and_res1x1():
    """The two-source virtual concat (skip scale folded into the packed weight) and the folded res_conv 1x1: the emulation
    passes; the second source without its scale fails."""
    B, H, W, C0, C1, Cout = 2, 8, 16, 64, 64, 128
    a0, a1, w, bias, res = _conv_operands(B, H, W, C0, Cout, 3, 0, seed=31, C1=C1)
    wsc = w.clone()
    wsc[:, C0:] *= 0.7071
    wp = EMU.pack_conv_weight(wsc)
    o, _, _ = _emu_conv(a0, a1, wp, B, H, W, Cout, 3, 0, bias, res)
    a = torch.cat((a0, a1), dim=-1)
    ref, bound = R.conv_fwd_ref(a, wp, 3, 3, 0, bias, res)
    check(o, ref, bound, "conv concat (emulation)")
    d, _, _ = _emu_conv(a0, a1, EMU.pack_conv_weight(w), B, H, W, Cout, 3, 0, bias, res)
    _fails(d, ref, bound, "second source without its scale")
    # folded 1x1 over x = cat(x0, x1)
    g = _g(32)
    x0, x1 = torch.randn(B, H, W, 64, generator=g).to(F16), torch.randn(B, H, W, 64, generator=g).to(F16)
    w3 = torch.randn(Cout, C0, 3, 3, generator=g) * (9 * C0) ** -0.5
    w1 = torch.randn(Cout, 128, 1, 1, generator=g) * 128 ** -0.5
    wp = torch.cat((EMU.pack_conv_weight(w3), EMU.pack_conv_weight(w1)), dim=1).contiguous()
    o, st = torch.zeros(B, H, W, Cout), torch.zeros(B, Cout // 16, 2, dtype=F64)
    EMU.conv_res1x1(a0, B, H, W, C0, C0, None, 0, 0, x0, 64, 128, x1, 64, 64, wp, Cout, bias, res, o, None, st)
    ref, bound = R.conv_fwd_ref(a0, wp, 3, 3, 0, bias, res, x=torch.cat((x0, x1), dim=-1))
    check(o, ref, bound, "conv res1x1 (emulation)")
    check_rel_l2(o, ref, 2e-5, "conv res1x1 (emulation)")
    check(st, *R.conv_stats_ref(o), "conv res1x1 statistics (emulation)")
    d = o.clone()
    d[0] -= (x1[0].double() @ R._d(wp[:, 9 * C0 + 64:]).t()).float()
    _fails(d, ref, bound, "folded 1x1: second x source dropped in image 0")


def test_conv_direct_and_stem_bound():
    """conv_direct_f32 (fp32 operands, n = taps x ceil4(C_in)) and the stem's 15-tap GEMM over 128 unrolled channels
    (n = 15 x 128) have the conv_fwd_ref form."""
    g = _g(33)
    B, H, W, Cin, ldi, Cout, k = 2, 12, 12, 6, 8, 16, 7
    x = torch.zeros(B, H, W, ldi)
    x[..., :Cin] = torch.randn(B, H, W, Cin, generator=g)
    w, b = torch.randn(Cout, Cin, k, k, generator=g) * 0.1, torch.randn(Cout, generator=g)
    o = torch.zeros(B, H, W, Cout)
    EMU.conv_direct(x, B, H, W, Cin, ldi, w, Cout, k, k, 1, k // 2, b, None, o, H, W, (H * W * Cout, W * Cout, Cout, 1))
    wpad = torch.zeros(Cout, ldi, k, k)
    wpad[:, :Cin] = w
    wp = wpad.permute(0, 2, 3, 1).reshape(Cout, -1)
    ref, bound = R.conv_fwd_ref(x, wp, k, k, 0, b)
    check(o, ref, bound, "conv_direct (emulation)")
    d = o.clone()
    d[..., 3] -= R.conv_nhwc(x.double()[..., Cin - 1:Cin], w[3:4, Cin - 1:Cin].double(), 0)[..., 0].float()
    _fails(d, ref, bound, "conv_direct: last input channel dropped in output channel 3")
    # stem: unroll the (fp16) image, 15-tap vertical GEMM == the float64 k = 3 / 7 / 15 convs of the fp16 operands
    from minimagen_b200.layers import CrossEmbedLayer
    torch.manual_seed(0)
    layer = CrossEmbedLayer(6, (3, 7, 15), dim_out=64, stride=1)
    img = torch.randn(B, 6, 16, 16, generator=g)
    a = torch.zeros(B, 16, 16, 128, dtype=F16)
    EMU.stem_unroll(img[:, :3], 3, img[:, 3:], 3, B, 16, 16, a)
    wp16, sbias = layer._stem_weights()
    ref, bound = R.conv_fwd_ref(a, wp16, 15, 1, 0, sbias)
    x16 = img.half().double()
    direct = torch.cat([torch.nn.functional.conv2d(x16, c.weight.detach().half().double(), c.bias.detach().double(),
                                                   padding=c.padding) for c in layer.convs], dim=1).permute(0, 2, 3, 1)
    assert (direct - ref).abs().max() < 1e-12                  # the unrolled GEMM is the three convs
    o = torch.zeros(B, 16, 16, 64)
    EMU.conv_igemm(a, B, 16, 16, 128, 0, 128, wp16, 64, 15, 1, 0, sbias, None, o, None, (16 * 16 * 64, 16 * 64, 64))
    check(o, ref, bound, "stem 15-tap GEMM (emulation)")


# ---------------------------------------------------------------------------------------------- GroupNorm forward
def _gn_stats_fp32(x32, groups, chunk, planes, lost_chunk=None):
    """gn_stats_kernel in its own order: per chunk of pixels, per plane, an fp32 chain over every planes-th pixel, two
    values per step (s += v0 + v1, q += v0 v0 + v1 v1), a single value at the end; the per-(chunk, plane, channel) chains
    are added in fp64.  x32 [B, HW, C] is the fp32 concat the kernel loads (src1 * scale1 rounded)."""
    B, HW, C = x32.shape
    S = torch.zeros(B, C, dtype=F64)
    Q = torch.zeros(B, C, dtype=F64)
    for k, p0 in enumerate(range(0, HW, chunk)):
        if k == lost_chunk:
            continue
        xs = x32[:, p0:p0 + chunk]
        L = -(-xs.shape[1] // planes)
        xs = torch.cat((xs, xs.new_zeros(B, L * planes - xs.shape[1], C)), dim=1).reshape(B, L, planes, C)
        xs = torch.cat((xs, xs.new_zeros(B, L % 2, planes, C)), dim=1)        # zeros add exactly
        s, q = torch.zeros(B, planes, C), torch.zeros(B, planes, C)
        for i in range(0, xs.shape[1], 2):
            v0, v1 = xs[:, i], xs[:, i + 1]
            s = s + (v0 + v1)
            q = q + (v0 * v0 + v1 * v1)
        S += s.double().sum(dim=1)
        Q += q.double().sum(dim=1)
    return torch.stack((S.reshape(B, groups, -1).sum(dim=2), Q.reshape(B, groups, -1).sum(dim=2)), dim=-1)


@pytest.mark.parametrize("HW,C0,C1,groups", [(1000, 48, 0, 16), (1000, 48, 0, 8), (300, 256, 128, 8), (50, 4096, 0, 32)])
def test_gn_stats_bound(HW, C0, C1, groups):
    """gn_stats_ref on the emulation and on the kernel-ordered fp32 chains (gn_stats_plan); a lost chunk and the straddling
    8-channel vector credited to its first group (Cg = 3, 6) fail."""
    B, C = 2, C0 + C1
    g = _g(HW + C)
    s0 = torch.randn(B, HW, C0, generator=g) * 2 + 0.5
    s1 = torch.randn(B, HW, C1, generator=g) if C1 else None
    scale1 = 0.7071 if C1 else 1.0
    sums = torch.zeros(B, groups, 2, dtype=F64)
    EMU.gn_stats(s0, C0, s1, C1, scale1, B, HW, groups, sums)
    chunk, planes, L = R.gn_stats_plan(C, HW)
    ref, bound = R.gn_stats_ref(s0, groups, s1, scale1, L)
    what = f"gn_stats HW={HW} C={C} G={groups}"
    check(sums, ref, bound, what + " (emulation)")
    x32 = torch.cat((s0, s1 * scale1), dim=-1) if C1 else s0
    check(_gn_stats_fp32(x32, groups, chunk, planes), ref, bound, what + " (fp32 restatement)")
    if HW > chunk:
        _fails(_gn_stats_fp32(x32, groups, chunk, planes, lost_chunk=1), ref, bound, what + ": one chunk lost")
    Cg = C // groups
    if Cg in (3, 6):
        d = sums.clone()
        v = x32.double()[..., 8:16]                    # the vector straddling groups 8 // Cg and 15 // Cg
        for c in range(8):
            if (8 + c) // Cg != 8 // Cg:
                d[:, 8 // Cg, 0] += v[..., c].sum(dim=1)
                d[:, (8 + c) // Cg, 0] -= v[..., c].sum(dim=1)
        _fails(d, ref, bound, what + ": straddling vector's last channels credited to its first group")


def _gn_apply_fp32(x32, sums, groups, gamma, beta, ss, eps, out16, defect=None):
    """gn_apply_silu_kernel in its own order: fp64 mean / var / rstd cast to fp32; a = rstd gamma, bb = beta - mean a,
    FiLM a *= sc, bb = fma(bb, sc, shift); v = fma(x, a, bb) (an fma: exact product in fp64, one rounding); SiLU in fp32."""
    B, HW, C = x32.shape
    Cg, n = C // groups, (C // groups) * HW
    mean = sums[..., 0] / n
    var = (sums[..., 1] / n - mean * mean).clamp(min=0)
    rstd = 1.0 / torch.sqrt(var + eps)
    if defect == "eps ignored":                                  # on the near-constant group (image 0, group 2)
        rstd[0, 2] = 1.0 / torch.sqrt(var[0, 2])
    if defect == "neighbour's mean":                             # image 1, group 3 takes group 4's mean
        mean[1, 3] = mean[1, 4]
    m, r = mean.float().repeat_interleave(Cg, dim=1), rstd.float().repeat_interleave(Cg, dim=1)
    a = r * gamma
    bb = beta - m * a
    if ss is not None:
        sc = ss[:, :C] + 1.0
        if defect == "scale without +1":                         # image 0
            sc[0] = ss[0, :C]
        a = a * sc
        bb = (bb.double() * sc.double() + ss[:, C:2 * C].double()).float()
    v = (x32.double() * a.double()[:, None] + bb.double()[:, None]).float()
    y = v / (1.0 + torch.exp(-v))
    return y.clamp(-65504, 65504).half() if out16 else y


def _gn_apply_case():
    B, HW, C0, C1, G = 2, 96, 32, 16, 8                        # Cg = 6: groups straddle the two sources and 8-vectors
    C = C0 + C1
    g = _g(34)
    s0 = torch.randn(B, HW, C0, generator=g) * 2 + 0.5
    s1 = torch.randn(B, HW, C1, generator=g)
    s0[0, :, 12:18] = 2.5 + 1e-4 * torch.randn(HW, 6, generator=g)          # image 0, group 2: near-constant
    s1[1, :, 0:6] = 100.0 / 0.7071 + torch.randn(HW, 6, generator=g)         # image 1, group 5 (after the scale): |mean|/std ~ 100
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    gamma[45] = 3e4                                              # v beyond 65504 and below -88 in channel 45
    ss = torch.randn(B, 2 * C, generator=g) * 0.3
    return B, HW, C0, C1, G, C, s0, s1, gamma, beta, ss


@pytest.mark.parametrize("out16", [False, True])
def test_gn_apply_silu_bound(out16):
    """gn_apply_silu_ref (a) on the emulation and on the kernel's coefficient fold; (b) with the kernel-ordered gn_stats of
    the same input; planted defects fail."""
    B, HW, C0, C1, G, C, s0, s1, gamma, beta, ss = _gn_apply_case()
    sums, sums_err = R.gn_stats_ref(s0, G, s1, 0.7071)
    x32 = torch.cat((s0, s1 * 0.7071), dim=-1)
    out = torch.zeros(B, HW, C, dtype=F16 if out16 else torch.float32)
    EMU.gn_apply_silu(s0, C0, s1, C1, 0.7071, B, HW, G, sums, 0, None, 0, gamma, beta, ss, 2 * C, 1e-5, out)
    ref, bound = R.gn_apply_silu_ref(s0, G, gamma, beta, ss, 1e-5, sums, src1=s1, scale1=0.7071, out16=out16)
    what = f"gn_apply_silu out16={out16}"
    check(out, ref, bound, what + " (emulation)")
    assert (out.double().abs().max() == 65504.0) if out16 else (out.abs().max() > 65504.0)
    fold = _gn_apply_fp32(x32, sums, G, gamma, beta, ss, 1e-5, out16)
    check(fold, ref, bound, what + " (fp32 coefficient fold)")
    # the aggregate leaves out the saturating channel 45 and the near-constant and |mean|/std ~ 100 groups, whose elementwise
    # bounds are large by nature
    agg = torch.ones(B, HW, C, dtype=torch.bool)
    agg[..., 45], agg[0, :, 12:18], agg[1, :, 30:36] = False, False, False
    check_rel_l2(fold[agg], ref[agg], 1e-3 if out16 else 5e-6, what + " (fp32 coefficient fold)")
    for defect in ("eps ignored", "neighbour's mean", "scale without +1"):
        _fails(_gn_apply_fp32(x32, sums, G, gamma, beta, ss, 1e-5, out16, defect), ref, bound, f"{what}: {defect}")
    # (b): the statistics of the kernel-ordered gn_stats chains, the reference on the exact ones
    chunk, planes, L = R.gn_stats_plan(C, HW)
    ks = _gn_stats_fp32(x32, G, chunk, planes)
    fold = _gn_apply_fp32(x32, ks, G, gamma, beta, ss, 1e-5, out16)
    ref, bound = R.gn_apply_silu_ref(s0, G, gamma, beta, ss, 1e-5, sums, sums_err, src1=s1, scale1=0.7071, out16=out16)
    check(fold, ref, bound, what + " (b) with kernel-ordered statistics")
    check(fold[1, :, 30:36], ref[1, :, 30:36], bound[1, :, 30:36], what + " (b) the |mean|/std ~ 100 group")


def test_conv_gn_bound():
    """mi_conv3x3_gn_silu_f16's emulation (gn_apply_silu to fp16, then the conv) passes conv_gn_ref; the FiLM scale
    without +1 in image 0 fails."""
    B, H, W, C0, C1, Cout, G = 2, 32, 8, 64, 64, 128, 8
    C = C0 + C1
    g = _g(35)
    x0, x1 = torch.randn(B, H, W, C0, generator=g) * 1.5 + 0.3, torch.randn(B, H, W, C1, generator=g)
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    ss = torch.randn(B, 2 * C, generator=g) * 0.3
    w = torch.randn(Cout, C, 3, 3, generator=g) * (9 * C) ** -0.5
    bias, res = torch.randn(Cout, generator=g), torch.randn(B, H, W, Cout, generator=g)
    wp = EMU.pack_conv_weight(w)
    st = []
    for t, Cc in ((x0, C0), (x1, C1)):
        s = torch.zeros(B, Cc // 16, 2, dtype=F64)
        EMU.gn_stats(t, Cc, None, 0, 1.0, B, H * W, Cc // 16, s)
        st.append(s)
    o = torch.zeros(B, H, W, Cout)
    EMU.conv_gn(x0, C0, x1, C1, 0.7071, B, H, W, G, st[0], st[1], gamma, beta, ss, 2 * C, 1e-5, wp, Cout, bias, res, o,
                None, None)
    sums = R.group_sums(st[0], C0, G, st[1], C1, 0.7071)
    ref, bound = R.conv_gn_ref(x0, G, gamma, beta, ss, 1e-5, sums, wp, bias, res, src1=x1, scale1=0.7071)
    check(o, ref, bound, "conv_gn (emulation)")
    check_rel_l2(o, ref, 1.5e-3, "conv_gn (emulation)")
    ss2 = ss.clone()
    ss2[0, :C] -= 1.0
    d = o.clone()
    EMU.conv_gn(x0, C0, x1, C1, 0.7071, B, H, W, G, st[0], st[1], gamma, beta, ss2, 2 * C, 1e-5, wp, Cout, bias, res, d,
                None, None)
    _fails(d, ref, bound, "conv_gn: FiLM scale without +1 in image 0")


# ---------------------------------------------------------------------------------------------- sampling step
# The step kernels compute op by op in fp32 in the order torch evaluates the restatement (un-fused products and sums, an
# exact select, at::lerp), so the emulation below is also the fp32 restatement in the kernels' order.
def _schedule(kind, T=1000):
    """(a, b, c1, c2, sigma, c3) fp32 tables of GaussianDiffusion's DDPM, DDIM (eta 0.5) or DPM-Solver++(2M) walk.  The
    library's sigma[0] is 0 or 1e-10, where a kernel that forgot to zero the noise at t = 0 would stay below any bound; the
    tests give sigma[0] = 0.25 so that the zeroing shows."""
    from minimagen_b200.diffusion_model import GaussianDiffusion
    gd = GaussianDiffusion(timesteps=T)
    sch = {"ddpm": gd.ddpm_schedule, "ddim": lambda d: gd.sampling_schedule(50, 0.5, d),
           "dpmpp": lambda d: gd.dpm_solver_schedule(20, d)}[kind]("cpu")
    sigma = sch.sigma.clone()
    sigma[0] = 0.25
    return gd.sqrt_recip_alphas_cumprod, gd.sqrt_recipm1_alphas_cumprod, sch.c1, sch.c2, sigma, sch.c3, sch.grid


def _step_data(B, n, seed, grid):
    g = _g(seed)
    x = torch.randn(B, n, generator=g) * 1.3
    x[-1] *= 0.2                                       # the last image's |x0| quantile is below min_s = 1 at t = 0
    eps, eps0, noise = (torch.randn(B, n, generator=g) for _ in range(3))
    hist = torch.randn(B, n, generator=g)
    t = torch.tensor([grid[0], grid[len(grid) // 2], 0][:B])
    w = torch.tensor([7.0, 3.0, 1.5][:B])
    return x, eps, eps0, noise, hist, t, w


def step_fp32(x, eps, eps0, w, t, tabs, lo, hi, wt, min_s, noise, hist=None, defect=None):
    """The step epilogue in fp32, op by op in the kernels' order: (x0, s, out, new hist).  `defect` plants one error."""
    a, b, c1, c2, sigma, c3 = tabs
    B = x.shape[0]
    wc = w.reshape(B, 1) if torch.is_tensor(w) else w
    if defect == "w0":
        wc = w[0]
    e = eps if eps0 is None else eps0 + (eps - eps0) * wc
    x0 = a[t][:, None] * x - b[t][:, None] * e
    s = torch.empty(B)
    EMU.step_quantile(x0, B, x0.shape[1], lo + (defect == "rank"), hi, wt, min_s, s)
    if defect == "lerp":
        srt = x0.abs().sort(dim=-1).values
        s = torch.lerp(srt[:, lo], srt[:, hi], torch.tensor(1 - wt)).clamp(min=min_s)
    if defect == "min_s":
        EMU.step_quantile(x0, B, x0.shape[1], lo, hi, wt, 0.0, s)
    if defect == "neighbour":
        s = s.roll(1)
    sb = s[:, None]
    xs = x0.clamp(-sb, sb) / sb
    mean = c1[t][:, None] * xs + c2[t][:, None] * x
    if hist is not None:
        c3t = c3[t][:, None]
        mean = torch.where(c3t != 0, mean + c3t * hist, mean)
    sig = sigma[t] if defect == "sigma0" else torch.where(t == 0, torch.zeros(()), sigma[t])
    return x0, s, mean + sig[:, None] * noise, xs


def _step_refs(x, eps, eps0, w, t, tabs, lo, hi, wt, min_s, noise, hist):
    a, b, c1, c2, sigma, c3 = tabs
    x0r, bx0 = R.step_x0_ref(x, eps, eps0, w, t, a, b)
    sr, bs = R.step_threshold_ref(x0r, bx0, lo, hi, wt, min_s)
    o = R.step_posterior_ref(x0r, bx0, sr, bs, x, noise, t, c1, c2, sigma, c3 if hist is not None else None, hist)
    return (x0r, bx0), (sr, bs), o


@pytest.mark.parametrize("kind", ["ddpm", "ddim", "dpmpp"])
@pytest.mark.parametrize("cfg", [True, False])
def test_step_bounds(kind, cfg):
    from minimagen_b200.Imagen import quantile_rank
    *tabs, grid = _schedule(kind)
    B, n = 3, 3 * 64 * 64
    x, eps, eps0, noise, hist, t, w = _step_data(B, n, 5, grid)
    eps0 = eps0 if cfg else None
    hist = hist if kind == "dpmpp" else None
    lo, hi, wt = quantile_rank(n, 0.9)
    (x0r, bx0), (sr, bs), (outr, bo, xsr, bxs) = _step_refs(x, eps, eps0, w, t, tabs, lo, hi, wt, 1.0, noise, hist)
    x0, s, out, xs = step_fp32(x, eps, eps0, w, t, tabs, lo, hi, wt, 1.0, noise, hist)
    check(x0, x0r, bx0, f"{kind} x0")
    check(s, sr, bs, f"{kind} s")
    check(out, outr, bo, f"{kind} out")
    check_rel_l2(out, outr, 1e-6, f"{kind} out")
    if hist is not None:
        check(xs, xsr, bxs, f"{kind} hist")
    # the emulation of the ops interface, scalar weight (the library's own entry point)
    if kind != "dpmpp":
        o2, s2 = torch.empty_like(x), torch.empty(B)
        c1, c2, sigma = tabs[2], tabs[3], tabs[4]
        EMU.step_epilogue(x, eps, eps0, 3.0, t, tabs[0], tabs[1], c1, c2, sigma, noise, B, n, lo, hi, wt, 1.0, o2, s2)
        (_, bx2), (sr2, bs2), (or2, bo2, _, _) = _step_refs(x, eps, eps0, 3.0, t, tabs, lo, hi, wt, 1.0, noise, None)
        check(s2, sr2, bs2, f"{kind} emu s")
        check(o2, or2, bo2, f"{kind} emu out")


@pytest.mark.parametrize("defect", ["rank", "lerp", "min_s", "neighbour", "w0", "sigma0"])
def test_step_defects(defect):
    """Each planted defect of the select or the step fails the bound of s or of out (the last image's s is below min_s = 1,
    the three images have different t and guidance weights, t = 0 is one of them)."""
    from minimagen_b200.Imagen import quantile_rank
    *tabs, grid = _schedule("ddpm")
    B, n = 3, 3 * 64 * 64
    x, eps, eps0, noise, _, t, w = _step_data(B, n, 5, grid)
    lo, hi, wt = quantile_rank(n, 0.9)
    _, (sr, bs), (outr, bo, _, _) = _step_refs(x, eps, eps0, w, t, tabs, lo, hi, wt, 1.0, noise, None)
    _, s, out, _ = step_fp32(x, eps, eps0, w, t, tabs, lo, hi, wt, 1.0, noise, defect=defect)
    _fails(out, outr, bo, f"step defect {defect}")
    if defect in ("rank", "lerp", "min_s", "neighbour"):
        _fails(s, sr, bs, f"step defect {defect} (s)")


def test_step_quantile_nan_follows_torch():
    """The emulated select gives NaN for a row containing NaN, and NaN (lerp(inf, inf)) when both order statistics are inf,
    as torch.quantile; the restatement's clamp / divide then makes the whole image NaN."""
    from minimagen_b200.Imagen import quantile_rank
    from oracle import restatement as RS
    B, n = 3, 1000
    x0 = torch.randn(B, n, generator=_g(3))
    x0[0, 17] = float("nan")
    x0[1, :150] = float("inf")
    lo, hi, wt = quantile_rank(n, 0.9)
    s = torch.empty(B)
    EMU.step_quantile(x0, B, n, lo, hi, wt, 1.0, s)
    ref = torch.quantile(x0.abs(), 0.9, dim=-1).clamp(min=1.0)
    assert torch.equal(s.isnan(), torch.tensor([True, True, False])) and torch.equal(s[2], ref[2])
    tabs = RS.ddpm_tables(1000)
    t = torch.tensor([5, 5, 5])
    out = torch.empty(B, n)
    EMU.step_epilogue(x0, torch.zeros(B, n), None, 1.0, t, torch.ones(1000), torch.zeros(1000),
                      tabs["posterior_mean_coef1"], tabs["posterior_mean_coef2"], torch.zeros(1000), torch.zeros(B, n),
                      B, n, lo, hi, wt, 1.0, out)
    assert out[:2].isnan().all() and not out[2].isnan().any()


def test_q_sample_bound():
    from oracle import restatement as RS
    tabs = RS.ddpm_tables(1000)
    g = _g(8)
    x0, z = torch.rand(3, 5000, generator=g), torch.randn(3, 5000, generator=g)
    t = torch.tensor([0, 500, 999])
    a, b = tabs["sqrt_alphas_cumprod"], tabs["sqrt_one_minus_alphas_cumprod"]
    for ps, sh in ((1.0, 0.0), (2.0, -1.0)):
        o = torch.empty(3, 5000)
        EMU.q_sample(x0, z, t, a, b, 3, 5000, ps, sh, o)
        ref, bound = R.q_sample_ref(x0, z, t, a, b, ps, sh)
        check(o, ref, bound, f"q_sample ({ps}, {sh})")
        if sh:
            EMU.q_sample(x0, z, t, a, b, 3, 5000, ps, 0.0, o)        # post_shift dropped
            _fails(o, ref, bound, "q_sample without post_shift")


def resize_fp32(x, iy, wy, ix, wx, clamp=None, swap_strides=False):
    """resize_sep_kernel in fp32 in its own order (sequential taps, rows inside columns).  swap_strides: the plane read
    with Hin and Win exchanged (in[xi][yi] of a [Win, Hin] view), an x/y mix-up that stays in bounds."""
    P, Hin, Win = x.shape
    v = x.reshape(P, Win, Hin).transpose(1, 2) if swap_strides else x
    acc = torch.zeros(P, iy.shape[0], ix.shape[0])
    for j in range(ix.shape[1]):
        col = torch.zeros(P, iy.shape[0], ix.shape[0])
        cols = v[:, :, ix[:, j].long()]                                       # [P, Hin, Wout]
        for i in range(iy.shape[1]):
            col = col + wy[:, i][None, :, None] * cols[:, iy[:, i].long(), :]
        acc = acc + wx[:, j][None, None, :] * col
    return acc.clamp(*clamp) if clamp is not None else acc


@pytest.mark.parametrize("H,W,scale,pad,clamp", [(40, 72, 2.0, "reflect", None), (40, 72, 0.25, "reflect", (-1.0, 1.0)),
                                                 (64, 64, 4.0, "constant", (0.0, 1.0))])
def test_resize_bound(H, W, scale, pad, clamp):
    from minimagen_b200.helpers import resize_tables
    x = torch.randn(2, H, W, generator=_g(9)) * 0.8
    ho, iy, wy = resize_tables(H, scale, pad, "cpu")
    wo, ix, wx = resize_tables(W, scale, pad, "cpu")
    ref, bound = R.resize_ref(x, iy, wy, ix, wx, clamp)
    o = torch.empty(2, ho, wo)
    EMU.resize_separable(x, 2, H, W, o, ho, wo, iy, wy, ix, wx, clamp=clamp)
    check(o, ref, bound, f"resize {H}x{W} x{scale} emulation")
    check(resize_fp32(x, iy, wy, ix, wx, clamp), ref, bound, f"resize {H}x{W} x{scale} fp32 order")
    if H != W:
        _fails(resize_fp32(x, iy, wy, ix, wx, clamp, swap_strides=True), ref, bound, "resize: Hin/Win strides swapped")
    if pad == "reflect":
        # a border tap reflected off by one: -tap - 1 instead of -tap (the 'symmetric' boundary)
        _, iy1, wy1 = resize_tables(H, scale, "symmetric", "cpu")
        _fails(resize_fp32(x, iy1, wy1, ix, wx, clamp), ref, bound, "resize: border tap off by one")


@pytest.mark.parametrize("dim", [8, 128, 1024])
def test_posemb_bound(dim):
    t = torch.tensor([0, 1, 17, 500, 999])
    o = torch.empty(5, dim)
    EMU.posemb(t, 5, dim, o)
    ref, bound = R.posemb_ref(t, dim)
    check(o, ref, bound, f"posemb {dim}")
    half = dim // 2
    e = torch.exp(torch.arange(half) * -(torch.log(torch.tensor(10000.0)) / half))          # half instead of half - 1
    arg = t[:, None].float() * e[None, :]
    _fails(torch.cat((arg.sin(), arg.cos()), dim=-1), ref, bound, "posemb: half instead of half - 1")
    _fails(torch.cat((o[:, half:], o[:, :half]), dim=-1), ref, bound, "posemb: sin and cos swapped")


@pytest.mark.parametrize("L,D", [(11, 16), (300, 40)])
def test_text_pool_bound(L, D):
    B, max_len, m, off = 3, 256, 260, 4
    g = _g(10)
    proj, null = torch.randn(B, L, D, generator=g), torch.randn(max_len, D, generator=g)
    mask = (torch.rand(B, L, generator=g) > 0.3).to(torch.uint8)
    keep = torch.tensor([1, 0, 1], dtype=torch.uint8)
    c, p = torch.full((B, m, D), float("nan")), torch.empty(B, D)
    EMU.text_tokens(proj, B, L, D, mask, keep, null, max_len, c, m, off, p)
    rows = c[:, off:off + max_len]
    ref, bound = R.text_pool_ref(rows)
    check(p, ref, bound, "text pooled (emulation)")
    check(R.text_pool_fp32(rows), ref, bound, "text pooled (fp32 serial)")
    if L < max_len:
        _fails(rows.sum(dim=1) / L, ref, bound, "text pooled / Lc")
