"""GPU: the token-side kernels -- attention (mma.sync and wgmma), row LayerNorm forward / backward, the fp32 linear layers,
the fp32 GEMM, column sums and the row softmax of the training path -- against float64 references with elementwise error
bounds (tests/fp64_ref.py; tests/test_error_bounds.py shows on the CPU that the bounds catch subtly wrong kernels).

Every check prints the worst |err| / bound of its case.  The model-level tests compare whole U-Nets at the fp16
operand-rounding noise floor (~1e-3 rel-L2), so a defect below that in any one of these ops is only visible here."""
import pytest
import torch

import fp64_ref as R
from fp64_ref import HALF_MAX, check, check_rel_l2, half_out

pytestmark = pytest.mark.gpu
F16, F64 = torch.float16, torch.float64
# whole-tensor rel-L2 limits next to the elementwise bounds (check_rel_l2): fp32 outputs of the fp32 kernels, fp16 copies,
# attention (fp16 P and output)
REL_F32, REL_LN_F32, REL_F16, REL_ATTN = 2e-6, 3e-6, 1e-3, 2e-3


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed + sum(shape))
    return torch.randn(*shape, generator=g) * scale


def _cu(t):
    return None if t is None else t.cuda()


def _rejects(out, ref, bound, what):
    """A defect planted into the native output on the host must fail the check: the bound has teeth at this size."""
    with pytest.raises(AssertionError):
        check(out, ref, bound, "planted: " + what)


# ---------------------------------------------------------------------------------------------- attention
def _tc_eligible(n, m, ldo, o_bs):
    """the shapes mi_attention_fwd sends to the wgmma kernel (queries are packed: q_bs == n * ldq, ldq = inner)"""
    return n % 128 == 0 and m >= 128 and ldo % 8 == 0 and o_bs % 8 == 0


def _attention(native, q, kv, null_kv, mask, B, heads, n, m, shared, ldo=None, o_bs=None, planted=False):
    """Run mi_attention_fwd on both kernels where the wgmma one is eligible; check every output element (and the NaN
    sentinels between the output rows / images) against the float64 reference, and the whole output's rel-L2.  Returns
    the outputs per kernel."""
    inner = heads * 64
    ldo = ldo or inner
    o_bs = o_bs or n * ldo
    ldkv = 128 if shared else 2 * inner
    v_off, kv_hs = (64, 0) if shared else (inner, 64)
    qn, kvn = q.cuda(), kv.cuda()
    mk = _cu(mask)
    qv, kk, vv = R.attention_views(qn, n * inner, inner, kvn, kvn[:, v_off:], m * ldkv, ldkv, kv_hs, B, heads, n, m)
    ref, bound = R.attention_ref(qv, kk, vv, null_kv.to(F16).float(), mk)
    shape, strides = (B, heads, n, 64), (o_bs, 64, ldo, 1)
    ref_buf = torch.zeros(B * o_bs, dtype=F64, device="cuda")
    bound_buf = torch.ones(B * o_bs, dtype=F64, device="cuda")
    sentinel = torch.ones(B * o_bs, dtype=torch.bool, device="cuda")
    ref_buf.as_strided(shape, strides).copy_(ref)
    bound_buf.as_strided(shape, strides).copy_(bound)
    sentinel.as_strided(shape, strides).fill_(False)
    outs = {}
    for tc in ([False, True] if _tc_eligible(n, m, ldo, o_bs) else [False]):
        native.attention_tc = tc
        o = torch.full((B * o_bs,), float("nan"), dtype=F16, device="cuda")
        native.attention(qn, n * inner, inner, kvn, kvn[:, v_off:], m * ldkv, ldkv, kv_hs, null_kv.cuda(), mk, B, heads,
                         n, m, o, o_bs, ldo)
        torch.cuda.synchronize()
        what = f"attention[{'wgmma' if tc else 'mma.sync'}] B={B} h={heads} n={n} m={m} shared={shared}"
        check(o, ref_buf, bound_buf, what, sentinel=sentinel)
        check_rel_l2(o.as_strided(shape, strides), ref, REL_ATTN, what)
        if planted:       # another head's output in one query row
            d = o.clone()
            dv = d.as_strided(shape, strides)
            dv[B - 1, 0, n // 2] = dv[B - 1, 1, n // 2]
            _rejects(d, ref_buf, bound_buf, what + " other head's row")
        outs[tc] = o.as_strided(shape, strides)
    native.attention_tc = True
    return outs


ATTN_CASES = [(2, 8, 256, 260, False, False), (2, 8, 64, 258, False, True),
              (1, 8, 1024, 1024, True, False), (2, 8, 256, 256, True, True),
              (1, 2, 100, 37, False, True),
              (3, 8, 128, 59, False, False),      # one padded key block
              (2, 4, 384, 127, True, False),      # m + 1 == 128 exactly
              (1, 2, 4096, 4096, True, False),    # base U-Net 64x64 tokens
              (2, 8, 512, 300, False, True),      # key mask, two query tiles
              (2, 4, 384, 700, True, True),       # ... and inside the one-tile kernel (n % 256 != 0)
              (1, 8, 256, 2000, True, True)]      # ... over many key blocks


@pytest.mark.parametrize("B,heads,n,m,shared,use_mask", ATTN_CASES)
def test_attention(native, B, heads, n, m, shared, use_mask):
    inner = heads * 64
    q = (_rand(B * n, inner, seed=34) * 0.125).to(F16)
    ldkv = 128 if shared else 2 * inner
    kv = _rand(B * m, ldkv, seed=35).to(F16)
    null_kv = _rand(2, 64, seed=36)
    mask = None
    if use_mask:
        mask = (torch.rand(B, m, generator=torch.Generator().manual_seed(1)) > 0.3).to(torch.uint8)
    _attention(native, q, kv, null_kv, mask, B, heads, n, m, shared)


@pytest.mark.parametrize("B,heads,n,m,shared,ramp", [(1, 8, 1024, 1280, True, "up"), (2, 4, 256, 600, False, "up"),
                                                     (1, 8, 1024, 1280, True, "down"), (2, 4, 128, 1500, True, "rows")])
def test_attention_single_sweep_rescales(native, B, heads, n, m, shared, ramp):
    """Online softmax over long key sequences: key norms that grow along the sequence ("up") force a rescale of the
    running accumulator in almost every key block, shrinking ones ("down") none after the first, "rows" makes only some
    query rows of a CTA move."""
    inner = heads * 64
    g = torch.Generator().manual_seed(91)
    q = torch.randn(B * n, inner, generator=g) * 0.5
    if ramp == "rows":
        q[::7] *= 4.0
    ldkv = 128 if shared else 2 * inner
    kv = torch.randn(B * m, ldkv, generator=g)
    t = torch.linspace(0, 1, m).repeat(B)[:, None]
    scale = {"up": 1 + 5 * t, "down": 6 - 5 * t, "rows": 1 + 3 * t}[ramp]
    v_off = 64 if shared else inner
    kv[:, :v_off] *= scale
    _attention(native, q.to(F16), kv.to(F16), _rand(2, 64, seed=36), None, B, heads, n, m, shared)


@pytest.mark.parametrize("B,heads,n,m,shared,mask_kind", [
    (32, 8, 1024, 258, False, None),       # cfg-3 cross attention over the text + time tokens
    (32, 8, 1024, 1024, True, None),       # cfg-3 multi-query self attention, 32 x 32 tokens
    (2, 8, 256, 128, False, None), (2, 8, 256, 128, True, "random"),     # smallest key count of the wgmma kernel
    (2, 8, 256, 255, True, None), (2, 8, 256, 255, False, "random"),     # m + 1 == 256: no padding keys
    (2, 8, 384, 383, False, None), (2, 4, 256, 383, True, "random"),     # m + 1 == 384
    (2, 8, 64, 300, False, "random"),      # mma.sync partial query tile
    (3, 4, 192, 130, True, None),
    (2, 8, 256, 383, False, "blocks"),     # whole 128-key blocks masked (and 64-key blocks of the mma.sync kernel)
    (2, 8, 256, 300, True, "bytes"),       # mask bytes other than 0 / 1
    (3, 4, 256, 200, False, "all"),        # image 1: every real key masked -> null value
    (3, 4, 128, 150, True, "all"),
])
def test_attention_edges(native, B, heads, n, m, shared, mask_kind):
    """The masks arrive only through the drop-in CrossAttention.forward / Attention.forward API (the U-Net's own calls
    pass none), so the mask cases protect that API, not the benchmarked step."""
    inner = heads * 64
    q = (_rand(B * n, inner, seed=60) * 0.3).to(F16)
    ldkv = 128 if shared else 2 * inner
    kv = _rand(B * m, ldkv, seed=61)
    kv[:, 64 if shared else inner:] += 1.5      # values with a common offset: the bound is tight relative to |o|
    kv = kv.to(F16)
    null_kv = _rand(2, 64, seed=62)
    g = torch.Generator().manual_seed(63)
    mask = None
    if mask_kind == "random":
        mask = (torch.rand(B, m, generator=g) > 0.3).to(torch.uint8)
    elif mask_kind == "blocks":
        mask = (torch.rand(B, m, generator=g) > 0.3).to(torch.uint8)
        mask[:, 127:255] = 0                                   # padded keys 128..255
    elif mask_kind == "bytes":
        mask = torch.tensor([0, 1, 2, 7, 128, 255], dtype=torch.uint8)[torch.randint(0, 6, (B, m), generator=g)]
    elif mask_kind == "all":
        mask = (torch.rand(B, m, generator=g) > 0.3).to(torch.uint8)
        mask[1] = 0
    outs = _attention(native, q, kv, null_kv, mask, B, heads, n, m, shared, planted=B == 32)
    if mask_kind == "all":
        nv = null_kv[1].to(F16).cuda()
        for tc, o in outs.items():
            assert torch.equal(o[1], nv.expand_as(o[1])), f"all keys masked: rows != fp16(null_v) (wgmma={tc})"


@pytest.mark.parametrize("n,m", [(256, 260), (128, 59)])
def test_attention_strided_output(native, n, m):
    """Output rows with ldo > inner and images with o_bs > n * ldo: the NaN sentinels between heads' rows and between
    images must stay NaN."""
    B, heads = 2, 8
    inner = heads * 64
    q = (_rand(B * n, inner, seed=70) * 0.3).to(F16)
    kv = _rand(B * m, 2 * inner, seed=71)
    kv[:, inner:] += 1.5
    kv = kv.to(F16)
    ldo = inner + 72
    _attention(native, q, kv, _rand(2, 64, seed=72), None, B, heads, n, m, False, ldo=ldo, o_bs=n * ldo + 136)


# ---------------------------------------------------------------------------------------------- LayerNorm forward
def _ln_check(native, x, gamma, beta, res, pre_gelu, what, eps=1e-5, agg_rows=slice(None)):
    """Elementwise bounds of both outputs, and their rel-L2 over the rows `agg_rows` (the near-constant rows of
    _ln_inputs are left out of the aggregate: their elementwise bound is large by nature, rstd ~ eps^-1/2)."""
    Rr, C = x.shape
    o = torch.full((Rr, C), float("nan"), device="cuda")
    o16 = torch.full((Rr, C), float("nan"), dtype=F16, device="cuda")
    native.ln_rows(x, Rr, C, gamma, beta, eps, pre_gelu, res, o, o16)
    torch.cuda.synchronize()
    ref, bound = R.ln_ref(x, gamma, beta, eps, pre_gelu, res)
    what = f"{what} R={Rr} C={C} gelu={pre_gelu} beta={beta is not None} res={res is not None}"
    check(o, ref, bound, what + " fp32")
    check(o16, *half_out(ref, bound), what + " fp16")
    if ref[agg_rows].numel():
        check_rel_l2(o[agg_rows], ref[agg_rows], REL_LN_F32, what + " fp32")
        check_rel_l2(o16[agg_rows], ref[agg_rows].clamp(-HALF_MAX, HALF_MAX), REL_F16, what + " fp16")
    return o, ref, bound


def _ln_inputs(Rr, C, seed):
    x = (_rand(Rr, C, seed=seed) * 3 + 1).cuda()
    x[0] = 2.5 + 1e-4 * x[0]                 # near-constant rows (variance ~1e-8 << eps): first and last
    x[-1] = -1.5 + 1e-4 * x[-1]
    return x, _rand(C, seed=seed + 1).cuda(), _rand(C, seed=seed + 2).cuda(), _rand(Rr, C, seed=seed + 3).cuda()


@pytest.mark.parametrize("R,C,pre_gelu,res,beta", [(100, 16, 0, True, True), (513, 1024, 1, False, False),
                                                   (64, 2048, 0, True, False), (7, 8, 0, False, True),
                                                   (520, 128, 0, False, True)])
def test_ln_rows(native, R, C, pre_gelu, res, beta):
    x = _rand(R, C, seed=18) * 3 + 1
    gamma = _rand(C, seed=19)
    bt = _rand(C, seed=20) if beta else None
    r = _rand(R, C, seed=21) if res else None
    _ln_check(native, x.cuda(), gamma.cuda(), _cu(bt), _cu(r), pre_gelu, "ln_rows")


# C -> rows per warp of ln_rows_reg_kernel (csrc/elementwise.cu); other C run the generic kernel
LN_REG = {128: 4, 256: 2, 512: 1, 1024: 1}
LN_CASES = [(C, r) for C, k in LN_REG.items() for r in sorted({1, k * 37 + 1, k * 37 + k - 1, 65537})]
LN_CASES += [(C, r) for C in (36, 768, 1536, 2048) for r in (1, 37, 4099)]


@pytest.mark.parametrize("C,rows", LN_CASES)
def test_ln_rows_bounds(native, C, rows):
    """Every register kernel at R = 1, a row tail of one and of ROWS - 1 rows, and R >= 65536; the generic kernel; each
    with and without the GELU in front, beta and the residual; near-constant first / last rows."""
    x, gamma, beta, res = _ln_inputs(rows, C, seed=C + rows)
    for pre_gelu in (0, 1):
        for bt in (None, beta):
            for r in (None, res):
                o, ref, bound = _ln_check(native, x, gamma, bt, r, pre_gelu, "ln_rows", agg_rows=slice(1, -1))
    if rows == 65537 and C == 1024:             # (the last combination: GELU, beta, residual) gamma shifted in one row
        d = o.clone()
        d[-2:] = R.ln_ref(x[-2:], gamma.roll(1), beta, 1e-5, 1, res[-2:])[0].float()
        _rejects(d, ref, bound, "ln_rows gamma shifted by one channel in two rows")


@pytest.mark.parametrize("C", [128, 256, 512, 1024, 768])
def test_ln_rows_fp16_saturates(native, C):
    """Outputs beyond the fp16 range: exactly +-65504 in the fp16 copy (csrc/sat_half.cuh), the fp32 copy unaffected."""
    Rr = 77
    x, _, beta, res = _ln_inputs(Rr, C, seed=5 * C)
    gamma = _rand(C, seed=C).cuda() * 4e4
    o, ref, bound = _ln_check(native, x, gamma, beta, res, 0, "ln_rows saturating", agg_rows=slice(1, -1))
    o16 = torch.empty(Rr, C, dtype=F16, device="cuda")
    native.ln_rows(x, Rr, C, gamma, beta, 1e-5, 0, res, None, o16)
    big = ref.abs() >= 65520                 # would round to inf without saturation
    assert big.sum() > 100
    assert torch.equal(o16[big].float(), HALF_MAX * ref[big].sign().float())


# ---------------------------------------------------------------------------------------------- LayerNorm backward
@pytest.mark.parametrize("C", [48, 128, 512, 1024])
@pytest.mark.parametrize("pre_gelu", [0, 1])
def test_ln_rows_bwd(native, C, pre_gelu):
    """R = 32771 rows: every warp of the capped grid takes many rows; dgamma / dbeta accumulate onto non-zero values."""
    Rr = 32771
    x, gamma, _, dy = _ln_inputs(Rr, C, seed=C + pre_gelu)
    dg0, db0 = _rand(C, seed=1).cuda(), _rand(C, seed=2).cuda()
    dx = torch.full((Rr, C), float("nan"), device="cuda")
    dg, db = dg0.clone(), db0.clone()
    native.ln_rows_bwd(x, dy, Rr, C, gamma, 1e-5, pre_gelu, dx, dg, db)
    torch.cuda.synchronize()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    (rx, bx), (rg, bg), (rb, bb) = R.ln_bwd_ref(x, dy, gamma, 1e-5, pre_gelu, dg0, db0, R.ln_bwd_acc_len(Rr, sms))
    what = f"ln_rows_bwd R={Rr} C={C} gelu={pre_gelu}"
    check(dx, rx, bx, what + " dx")
    check(dg, rg, bg, what + " dgamma")
    check(db, rb, bb, what + " dbeta")


# ---------------------------------------------------------------------------------------------- fp32 linear
def _linear(native, M, K, N, in_act, out_act, add, scale, seed, what="linear_f32"):
    x, w, b = _rand(M, K, seed=seed).cuda(), _rand(N, K, seed=seed + 1, scale=K ** -0.5).cuda(), _rand(N, seed=seed + 2).cuda()
    a = _rand(M, N, seed=seed + 3).cuda() if add else None
    o = torch.full((M, N), float("nan"), device="cuda")
    o16 = torch.full((M, N), float("nan"), dtype=F16, device="cuda")
    native.linear_f32(x, M, K, w, b, N, in_act, out_act, a, o, o16, scale)
    torch.cuda.synchronize()
    ref, bound = R.linear_ref(x, w, b, in_act, out_act, a, scale)
    what = f"{what} M={M} K={K} N={N} in_act={in_act} out_act={out_act} add={add} scale={scale}"
    check(o, ref, bound, what + " fp32")
    check(o16, *half_out(ref, bound), what + " fp16")
    check_rel_l2(o, ref, REL_F32, what + " fp32")
    check_rel_l2(o16, ref.clamp(-HALF_MAX, HALF_MAX), REL_F16, what + " fp16")
    return o, o16, ref, bound, (x, w, b, a)


@pytest.mark.parametrize("M,K,N,in_act,out_act,add", [(2, 8, 32, 0, 1, False), (32, 1024, 2048, 1, 0, False),
                                                      (32, 512, 512, 0, 0, True), (516, 8, 1024, 0, 0, False),
                                                      (9, 768, 128, 0, 0, False)])
def test_linear_f32(native, M, K, N, in_act, out_act, add):
    _linear(native, M, K, N, in_act, out_act, add, 0.125, seed=22)


# linear_f32 (csrc/elementwise.cu) picks: M <= 8 -> one warp per column; 8 < M <= 64 with N K <= 4M -> the same over
# 8-row groups; otherwise the 32 x 128 tiled kernel (K chunks of 32, next chunk prefetched into registers)
@pytest.mark.parametrize("M,K,N,in_act,out_act,add,scale", [
    (5, 4, 131, 1, 0, True, 0.5), (5, 1028, 1001, 0, 1, False, 1.0), (7, 36, 131, 1, 1, True, -2.0),     # M <= 8
    (37, 36, 1001, 1, 1, True, -2.0), (9, 1028, 131, 0, 0, False, 0.125), (61, 4, 131, 0, 1, True, 1.0),  # 8-row groups
    (77, 36, 131, 1, 1, True, 1.5), (77, 1028, 1001, 0, 1, True, 1.0), (300, 4, 1001, 1, 0, True, 1.0),   # tiled
    (37, 1028, 4099, 1, 0, False, 0.25),     # tiled at M <= 64: N K > 4M
])
def test_linear_f32_kernels(native, M, K, N, in_act, out_act, add, scale):
    _linear(native, M, K, N, in_act, out_act, add, scale, seed=M + K + N)


@pytest.mark.parametrize("M", [5, 37, 77])
def test_linear_f32_fp16_saturates(native, M):
    o, o16, ref, bound, _ = _linear(native, M, 36, 131, 0, 0, True, 3e4, seed=M, what="linear_f32 saturating")
    big = ref.abs() >= 65520
    assert big.sum() > 100
    assert torch.equal(o16[big].float(), HALF_MAX * ref[big].sign().float())


def test_linear_f32_time_mlp(native):
    """The batched time-MLP GEMM of the cfg-3 SR U-Net (Unet(**Super.defaults, lowres_cond=True, text_embed_dim=768)) at
    batch 32: SiLU(t) [32, 1024] @ the 55 ResnetBlocks' concatenated time_mlp weights [66304, 1024]^T."""
    o, _, ref, bound, (x, w, b, a) = _linear(native, 32, 1024, 66304, 0, 0, False, 1.0, seed=80)
    d = o.clone()
    d[:, 40000] -= b[40000]
    _rejects(d, ref, bound, "time MLP bias dropped in one column")


# ---------------------------------------------------------------------------------------------- fp32 GEMM / colsum
@pytest.mark.parametrize("a_kfast,b_nfast", [(True, True), (True, False), (False, True), (False, False)])
@pytest.mark.parametrize("M,N,K", [(65, 130, 17), (130, 65, 1025)])
def test_gemm_f32(native, a_kfast, b_nfast, M, N, K):
    """All four operand layouts (a_sk == 1 or not, b_sn == 1 or not), ragged M / N / K; alpha != 1 accumulating onto a
    non-zero C over Z1 x Z2 = 2 x 3 batches with distinct strides; then alpha = 1, overwrite, with B's z2 stride 0 (one
    shared operand per z1, as AttentionFn's multi-query K / V)."""
    Z1, Z2 = 2, 3
    A = _rand(Z1 * Z2 * M * K + 5, seed=1).cuda()
    Bm = _rand(Z1 * Z2 * K * N + 3, seed=2).cuda()
    a_str = (K, 1) if a_kfast else (1, M)
    b_str = (N, 1) if b_nfast else (1, K)
    a_b, c_b = (Z2 * M * K + 5, M * K), (Z2 * M * N + 7, M * N)
    view = lambda t, sh, st, bb: t.as_strided((Z1, Z2) + sh, bb + st)
    C = torch.full((Z1 * c_b[0],), float("nan"), device="cuda")     # the 7-element gaps between z1 batches stay NaN
    view(C, (M, N), (N, 1), c_b).copy_(_rand(Z1, Z2, M, N, seed=3))
    sentinel = torch.ones(C.shape, dtype=torch.bool, device="cuda")
    view(sentinel, (M, N), (N, 1), c_b).fill_(False)
    for alpha, acc, b_b in ((0.37, True, (Z2 * K * N, K * N)), (1.0, False, (K * N + 3, 0))):
        Av, Bv = view(A, (M, K), a_str, a_b), view(Bm, (K, N), b_str, b_b)
        C0 = view(C, (M, N), (N, 1), c_b).clone()
        native.gemm_f32(A, Bm, C, M, N, K, a_str, b_str, (N, 1), Z1, Z2, a_b, b_b, c_b, alpha=alpha, accumulate=acc)
        torch.cuda.synchronize()
        ref, bound = R.gemm_ref(Av, Bv, C0, alpha, acc)
        ref_buf = torch.zeros(C.shape, dtype=F64, device="cuda")
        bound_buf = torch.ones(C.shape, dtype=F64, device="cuda")
        view(ref_buf, (M, N), (N, 1), c_b).copy_(ref)
        view(bound_buf, (M, N), (N, 1), c_b).copy_(bound)
        what = f"gemm_f32 M={M} N={N} K={K} a_kfast={a_kfast} b_nfast={b_nfast} alpha={alpha} acc={acc} b_b={b_b}"
        check(C, ref_buf, bound_buf, what, sentinel=sentinel)
        check_rel_l2(view(C, (M, N), (N, 1), c_b), ref, REL_F32, what)


@pytest.mark.parametrize("M,N,acc", [(3000, 300, False), (1024 * 512 + 777, 40, True), (1024 * 1100 + 5, 33, False)])
def test_colsum(native, M, N, acc):
    """More than 1024 * 512 rows: the split count is capped at 512, rows per split grow.  (Values with a common offset,
    so that the partial sum of one split stands out of the worst-case bound.)"""
    x = (_rand(M, N, seed=9) + 0.5).cuda()
    out0 = _rand(N, seed=10).cuda()
    out = out0.clone() if acc else torch.full((N,), float("nan"), device="cuda")
    native.colsum(x, M, N, out, accumulate=acc)
    torch.cuda.synchronize()
    ref, bound = R.colsum_ref(x, out0 if acc else None, R.colsum_acc_len(M))
    check(out, ref, bound, f"colsum M={M} N={N} acc={acc}")
    if M > 1024 * 1024:                    # one split's partial sum lost (its atomicAdd) in one column
        rpb = -(-M // 512)
        d = out.clone()
        d[3] -= x[rpb:2 * rpb, 3].sum()
        _rejects(d, ref, bound, "colsum one split dropped in one column")


# ---------------------------------------------------------------------------------------------- softmax rows
@pytest.mark.parametrize("L", [18, 259, 1025, 4097])
def test_softmax_rows(native, L):
    Rr = 1500
    s = (_rand(Rr, L, seed=L) * 4).cuda()
    s[::5] += 60.0                                     # rows far from 0 (exp would overflow without the max)
    s[1::7] *= 8
    p = s.clone()
    native.softmax_rows(p, Rr, L)
    torch.cuda.synchronize()
    check(p, *R.softmax_ref(s), f"softmax_rows L={L}")
    dP = (_rand(Rr, L, seed=L + 1) + 0.5).cuda()
    dS = dP.clone()
    native.softmax_rows_bwd(p, dS, Rr, L)
    torch.cuda.synchronize()
    check(dS, *R.softmax_bwd_ref(p, dP), f"softmax_rows_bwd L={L}")


@pytest.mark.parametrize("n,m,hk", [(1024, 258, 8), (1024, 1024, 1)])
def test_attention_fn(native, n, m, hk):
    """AttentionFn (fp32 batched GEMMs + row softmax, the training path's attention) forward and backward against float64
    autograd: cross attention over 258 tokens, multi-query self attention over 1024."""
    from minimagen_b200.autograd import AttentionFn
    B, heads = 2, 8
    q = (_rand(B, n, heads * 64, seed=1) * 0.125).cuda().requires_grad_(True)
    k = _rand(B, m, hk * 64, seed=2).cuda().requires_grad_(True)
    v = _rand(B, m, hk * 64, seed=3).cuda().requires_grad_(True)
    nk = _rand(2, 64, seed=4).cuda().requires_grad_(True)
    do = _rand(B, n, heads * 64, seed=5).cuda()
    o = AttentionFn.apply(q, k, v, nk, heads)
    got = dict(zip(("dq", "dk", "dv", "dnull"), torch.autograd.grad(o, (q, k, v, nk), do)), o=o)
    for name, (ref, bound) in R.attention_fn_ref(q, k, v, nk, heads, do).items():
        check(got[name], ref, bound, f"AttentionFn n={n} m={m} hk={hk} {name}")
