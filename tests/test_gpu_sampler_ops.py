"""The sampling loop's kernels outside the U-Net against float64 (tests/fp64_ref.py) and against torch's NaN semantics: the
step epilogue (fused cluster kernel and three-kernel form, plain and multistep, scalar and per-image guidance weights), its
exact select on tied and degenerate data, q_sample, the cascade resize, the timestep embedding and the text tokens.
Every bounded case prints its worst |err| / bound and its rel-L2."""
import pytest
import torch

import fp64_ref as R
from emu_ops import EmuOps
from fp64_ref import check, check_rel_l2
from test_error_bounds import _schedule

pytestmark = pytest.mark.gpu

EMU = EmuOps()
T = 1000
FUSED_MAX = 196608                          # the largest image the fused cluster kernel holds in registers
SIZES = [1, 3, 9, 768, 3 * 64 * 64, FUSED_MAX, FUSED_MAX + 1, 3 * 288 * 288]


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _cu(t):
    return None if t is None else t.cuda()


def _nan_equal(a, b, what):
    """Same NaN positions, and every other element bit-identical."""
    a, b = a.detach().cpu(), b.detach().cpu()
    na, nb = a.isnan(), b.isnan()
    assert torch.equal(na, nb), f"{what}: NaN at {int(na.sum())} elements, expected {int(nb.sum())}"
    assert torch.equal(a[~na], b[~nb]), f"{what}: non-NaN elements differ"


# ---------------------------------------------------------------------------------------------- select data
def _select_data(kind, B, n, seed):
    """[B, n] fp32 values whose |.| the select orders.  n is split into 8 CTA chunks of ceil(n / 8) by the fused kernel."""
    from minimagen_b200.Imagen import quantile_rank
    g = _g(seed)
    lo, hi, _ = quantile_rank(n, 0.9)
    x = torch.randn(B, n, generator=g) * 1.7
    if kind == "ties":                                   # quantised to k / 4: every value is tied
        return (x * 4).round() / 4
    if kind == "run":                                    # one value at 0.9 quantile, n / 5 copies spread over the boundaries
        v = x.abs().sort(dim=-1).values[:, lo:lo + 1]
        chunk = -(-n // 8)
        r = max(1, n // 70)
        for c in range(1, 8):
            a, b = max(0, c * chunk - r), min(n, c * chunk + r)
            if a < b:
                x[:, a:b] = v * torch.where(torch.rand(B, b - a, generator=g) < 0.5, -1.0, 1.0)
        if n < 16:
            x[:] = v
        return x
    if kind == "run_end":                                # sorted[lo] ends its run; sorted[lo + 1] is unique, in x[n - 1]
        out = torch.empty(B, n)
        for b in range(B):
            m = max(1, min(lo + 1, n // 10))
            below = torch.rand(lo + 1 - m, generator=g) * 0.9
            above = 1.25 + torch.rand(n - lo - 2, generator=g) if n - lo - 2 > 0 else torch.empty(0)
            body = torch.cat((below, torch.ones(m), above))
            body = body[torch.randperm(body.numel(), generator=g)]
            if lo + 1 < n:
                body = torch.cat((body, torch.tensor([1.125])))
            sign = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
            out[b] = body * sign
        return out
    if kind == "special":                                # constant, zeros of both signs, subnormals, a few +-inf
        x[0] = 0.6
        x[1] = torch.where(torch.rand(n, generator=g) < 0.5, -0.0, 0.0)
        sub = torch.randn(n, generator=g) * 1e-39        # subnormal (|v| < 2^-126), some of them exactly +-0
        x[2] = torch.where(torch.rand(n, generator=g) < 0.1, 0.0, sub)
        if B > 3 and n >= 100:
            idx = torch.randperm(n, generator=g)[:3]
            x[3, idx] = torch.tensor([float("inf"), -float("inf"), float("inf")])
        return x
    return x


SELECT_KINDS = ["gauss", "ties", "run", "run_end", "special"]


@pytest.mark.parametrize("kind", SELECT_KINDS)
@pytest.mark.parametrize("n", SIZES)
def test_step_select_is_exact(native, n, kind):
    """With the x0 tables a = 1, b = 0 the step's x0 is x_t itself, so s_out must be torch.quantile(|x_t|, 0.9) clamped to
    min_s, bit for bit: for the fused cluster kernel and the three-kernel form alike (n > 196 608 selects the latter), and
    for quantile_kernel (step_quantile) run on its own at every n.  The oracle is torch, not the other select."""
    from minimagen_b200.Imagen import quantile_rank
    B = 4
    x = _select_data(kind, B, n, seed=n + len(kind))
    lo, hi, wt = quantile_rank(n, 0.9)
    ones, zeros = torch.ones(T, device="cuda"), torch.zeros(T, device="cuda")
    t = torch.tensor([999, 0, 5, 500][:B]).cuda()
    xc, z = x.cuda(), torch.zeros(B, n, device="cuda")
    for min_s in (0.0, 1.0):
        expect = torch.quantile(x.abs(), 0.9, dim=-1).clamp(min=min_s)
        s = torch.full((B,), -1.0, device="cuda")
        out = torch.empty_like(xc)
        native.step_epilogue(xc, z, None, 1.0, t, ones, zeros, ones, zeros, zeros, z, B, n, lo, hi, wt, min_s, out, s_out=s)
        _nan_equal(s, expect, f"fused/auto select n={n} {kind} min_s={min_s}")
        s3 = torch.full((B,), -1.0, device="cuda")
        native.step_quantile(xc, B, n, lo, hi, wt, min_s, s3)
        _nan_equal(s3, expect, f"quantile_kernel n={n} {kind} min_s={min_s}")
        # c1 = 1, c2 = 0, sigma = 0: out = clamp(x, -s, s) / s (+ 0 * x_t, which is NaN where x_t is inf)
        sb = expect[:, None]
        fin = torch.isfinite(x)
        _nan_equal(out.cpu()[fin], (x.clamp(-sb, sb) / sb)[fin], f"clamp/divide n={n} {kind} min_s={min_s}")


# ---------------------------------------------------------------------------------------------- step epilogue vs fp64
def _tabs_cuda(kind):
    a, b, c1, c2, sigma, c3, grid = _schedule(kind)
    return [v.cuda() if v is not None else None for v in (a, b, c1, c2, sigma, c3)], grid


@pytest.mark.parametrize("guidance", ["none", "scalar", "per_image"])
@pytest.mark.parametrize("n", [768, 3 * 64 * 64, FUSED_MAX, FUSED_MAX + 1])
@pytest.mark.parametrize("kind", ["ddpm", "ddim", "dpmpp"])
def test_step_epilogue_bounds(native, kind, n, guidance):
    """out (and the multistep history) element by element against float64; s against the fp64 order statistics and, bit
    for bit, against torch.quantile of the native x0 (step_x0 is bit-exact); out separate from x_t and aliasing it."""
    from minimagen_b200.Imagen import quantile_rank
    tabs, grid = _tabs_cuda(kind)
    a, b, c1, c2, sigma, c3 = tabs
    B = 3
    g = _g(n + len(kind) + len(guidance))
    x = torch.randn(B, n, generator=g) * 1.3
    x[-1] *= 0.2
    eps, eps0, noise, hist = (torch.randn(B, n, generator=g) for _ in range(4))
    t = torch.tensor([grid[0], grid[len(grid) // 2], 0])
    eps0 = None if guidance == "none" else eps0
    w = torch.tensor([7.0, 3.0, 1.5]) if guidance == "per_image" else 3.0
    wn = w.cuda() if torch.is_tensor(w) else w
    multi = kind == "dpmpp"
    lo, hi, wt = quantile_rank(n, 0.9)
    x0r, bx0 = R.step_x0_ref(x, eps, eps0, w, t, a, b)
    sr, bs = R.step_threshold_ref(x0r, bx0, lo, hi, wt, 1.0)
    outr, bo, xsr, bxs = R.step_posterior_ref(x0r, bx0, sr, bs, x, noise, t, c1, c2, sigma, c3 if multi else None,
                                              hist if multi else None)
    xc, tc = x.cuda(), t.cuda()
    x0n = torch.empty_like(xc)
    if not torch.is_tensor(w):
        native.step_x0(xc, eps.cuda(), _cu(eps0), w, tc, a, b, B, n, x0n)
    results = []
    for alias in (False, True):
        xin = xc.clone()
        out = xin if alias else torch.empty_like(xc)
        s = torch.empty(B, device="cuda")
        h = hist.cuda()
        if multi:
            native.step_epilogue_multistep(xin, eps.cuda(), _cu(eps0), wn, tc, a, b, c1, c2, sigma, c3, noise.cuda(), h,
                                           B, n, lo, hi, wt, 1.0, out, s_out=s)
        else:
            native.step_epilogue(xin, eps.cuda(), _cu(eps0), wn, tc, a, b, c1, c2, sigma, noise.cuda(), B, n, lo, hi, wt,
                                 1.0, out, s_out=s)
        results.append((out.clone(), s.clone(), h.clone()))
    (out, s, h), (out2, s2, h2) = results
    assert torch.equal(out, out2) and torch.equal(s, s2) and torch.equal(h, h2), "aliasing out and x_t changed the result"
    what = f"{kind} n={n} {guidance}"
    check(s, sr, bs, f"{what} s")
    check(out, outr, bo, f"{what} out")
    check_rel_l2(out, outr, 1e-6, f"{what} out")
    if multi:
        check(h, xsr, bxs, f"{what} hist")
        check_rel_l2(h, xsr, 1e-6, f"{what} hist")
    if not torch.is_tensor(w):
        assert torch.equal(s.cpu(), torch.quantile(x0n.abs().cpu(), 0.9, dim=-1).clamp(min=1.0)), f"{what}: s not exact"


# ---------------------------------------------------------------------------------------------- NaN and inf parity
@pytest.mark.parametrize("n", [9, 3 * 64 * 64, FUSED_MAX + 1])
@pytest.mark.parametrize("multi", [False, True])
def test_step_nan_and_inf_parity(native, n, multi):
    """Image 0's x0 has one NaN, image 1 is +inf at 15 % of its elements, image 2 has two +-inf, image 3 is clean.  s_out,
    out and the history must have the NaN pattern of the torch restatement (torch.quantile is NaN for a row with a NaN, and
    lerp(inf, inf) is NaN, so the whole image is NaN); images 2 and 3 must be bit-identical to the restatement, and image 3
    to a run in which the other images are clean."""
    from minimagen_b200.Imagen import quantile_rank
    tabs, grid = _tabs_cuda("dpmpp" if multi else "ddpm")
    a, b, c1, c2, sigma, c3 = tabs
    B = 4
    g = _g(n + multi)
    x = torch.randn(B, n, generator=g)
    eps, eps0, noise, hist = (torch.randn(B, n, generator=g) for _ in range(4))
    t = torch.tensor([grid[1], grid[2], grid[3], 0])
    lo, hi, wt = quantile_rank(n, 0.9)
    xb, eb = x.clone(), eps.clone()
    eb[0, n // 2] = float("nan")
    xb[1, torch.randperm(n, generator=g)[:max(1, (15 * n + 99) // 100)]] = float("inf")
    if n >= 100:
        xb[2, :2] = torch.tensor([float("inf"), -float("inf")])

    def run_native(xx, ee):
        out, s, h = torch.empty(B, n, device="cuda"), torch.empty(B, device="cuda"), hist.cuda()
        if multi:
            native.step_epilogue_multistep(xx.cuda(), ee.cuda(), eps0.cuda(), 3.0, t.cuda(), a, b, c1, c2, sigma, c3,
                                           noise.cuda(), h, B, n, lo, hi, wt, 1.0, out, s_out=s)
        else:
            native.step_epilogue(xx.cuda(), ee.cuda(), eps0.cuda(), 3.0, t.cuda(), a, b, c1, c2, sigma, noise.cuda(), B,
                                 n, lo, hi, wt, 1.0, out, s_out=s)
        return out.cpu(), s.cpu(), h.cpu()

    def run_emu(xx, ee):
        out, s, h = torch.empty(B, n), torch.empty(B), hist.clone()
        ct = [v.cpu() for v in tabs if v is not None]
        if multi:
            EMU.step_epilogue_multistep(xx, ee, eps0, 3.0, t, *ct[:5], ct[5], noise, h, B, n, lo, hi, wt, 1.0, out,
                                            s_out=s)
        else:
            EMU.step_epilogue(xx, ee, eps0, 3.0, t, *ct[:5], noise, B, n, lo, hi, wt, 1.0, out, s_out=s)
        return out, s, h

    on, sn, hn = run_native(xb, eb)
    oe, se, he = run_emu(xb, eb)
    assert sn[:2].isnan().all() and not sn[2:].isnan().any(), sn
    assert on[:2].isnan().all(), "an image with a NaN x0 or >= 10 % inf must come out all NaN"
    _nan_equal(sn, se, f"n={n} s_out")
    _nan_equal(on, oe, f"n={n} out")
    if multi:
        assert hn[:2].isnan().all()
        _nan_equal(hn, he, f"n={n} hist")
    oc, sc, hc = run_native(x, eps)
    assert torch.equal(on[3], oc[3]) and torch.equal(sn[3], sc[3]) and torch.equal(hn[3], hc[3])


@pytest.mark.parametrize("unnormalize", [0, 1])
def test_finalize_keeps_nan(native, unnormalize):
    """step_finalize and inpaint_finalize clamp with torch.clamp's NaN semantics: a NaN pixel stays NaN."""
    g = _g(4 + unnormalize)
    B, C, hw = 2, 3, 40 * 40
    x = torch.randn(B, C, hw, generator=g) * 2
    x[0, 1, 7] = float("nan")
    x[1, 2, :5] = float("inf")
    x[1, 0, 3] = -float("nan")
    k = torch.randn(B, C, hw, generator=g)
    k[1, 1, 11] = float("nan")
    m = (torch.rand(B, hw, generator=g) > 0.5).float()
    m[1, 11] = 1.0
    fin = lambda v: (v.clamp(-1, 1) + 1) * 0.5 if unnormalize else v.clamp(-1, 1)
    out = torch.empty(B, C, hw, device="cuda")
    native.step_finalize(x.cuda(), x.numel(), unnormalize, out)
    _nan_equal(out, fin(x), "step_finalize")
    native.inpaint_finalize(x.cuda(), k.cuda(), m.cuda(), B, C, hw, unnormalize, out)
    _nan_equal(out, fin(torch.where(m[:, None] >= 0.5, k, x)), "inpaint_finalize")


# ---------------------------------------------------------------------------------------------- q_sample
@pytest.mark.parametrize("post", [(1.0, 0.0), (2.0, -1.0)])
def test_q_sample(native, post):
    from oracle import restatement as RS
    tabs = {k: v.cuda() for k, v in RS.ddpm_tables(T).items()}
    g = _g(12)
    B, n = 3, 3 * 64 * 64
    x0, z = torch.rand(B, n, generator=g), torch.randn(B, n, generator=g)
    t = torch.tensor([0, 417, 999])
    a, b = tabs["sqrt_alphas_cumprod"], tabs["sqrt_one_minus_alphas_cumprod"]
    out = torch.empty(B, n, device="cuda")
    native.q_sample(x0.cuda(), z.cuda(), t.cuda(), a, b, B, n, post[0], post[1], out)
    ref, bound = R.q_sample_ref(x0, z, t, a, b, *post)
    check(out, ref, bound, f"q_sample {post}")
    check_rel_l2(out, ref, 1e-6, f"q_sample {post}")


# ---------------------------------------------------------------------------------------------- cascade resize
@pytest.mark.parametrize("H,W,scale", [(40, 72, 2.0), (40, 72, 0.25), (64, 64, 4.0), (72, 40, 0.5)])
@pytest.mark.parametrize("pad", ["reflect", "constant"])
@pytest.mark.parametrize("clamp", [None, (-1.0, 1.0)])
def test_resize_separable(native, H, W, scale, pad, clamp):
    """Non-square planes with a table per axis (an x/y mix-up of tables or strides reads the wrong pixels), the 16-tap
    anti-aliased 4x downscale, both boundaries; with a clamp, NaN inputs stay NaN where their taps reach."""
    from minimagen_b200.helpers import resize_tables
    P = 6
    x = torch.randn(P, H, W, generator=_g(H * W + int(scale * 4))) * 0.8
    ho, iy, wy = resize_tables(H, scale, pad, "cpu")
    wo, ix, wx = resize_tables(W, scale, pad, "cpu")
    out = torch.full((P, ho, wo), float("nan"), device="cuda")
    native.resize_separable(x.cuda(), P, H, W, out, ho, wo, iy.cuda(), wy.cuda(), ix.cuda(), wx.cuda(), clamp=clamp)
    ref, bound = R.resize_ref(x, iy, wy, ix, wx, clamp)
    what = f"resize {H}x{W} x{scale} {pad} clamp={clamp}"
    check(out, ref, bound, what)
    check_rel_l2(out, ref, 1e-6, what)
    if clamp is not None:
        xn = x.clone()
        xn[1, H // 2, W // 3] = float("nan")
        native.resize_separable(xn.cuda(), P, H, W, out, ho, wo, iy.cuda(), wy.cuda(), ix.cuda(), wx.cuda(), clamp=clamp)
        o_e = torch.empty(P, ho, wo)
        EMU.resize_separable(xn, P, H, W, o_e, ho, wo, iy, wy, ix, wx, clamp=clamp)
        nan = out.isnan().cpu()
        assert nan.any() and torch.equal(nan, o_e.isnan()), f"{what}: NaN input not propagated through the clamp"


# ---------------------------------------------------------------------------------------------- conditioning
@pytest.mark.parametrize("dim", [8, 16, 128, 320, 1024])
def test_posemb(native, dim):
    t = torch.tensor([0, 1, 2, 17, 250, 500, 998, 999])
    out = torch.empty(t.numel(), dim, device="cuda")
    native.posemb(t.cuda(), t.numel(), dim, out)
    ref, bound = R.posemb_ref(t, dim)
    check(out, ref, bound, f"posemb dim={dim}")
    check_rel_l2(out, ref, 1e-4, f"posemb dim={dim}")


@pytest.mark.parametrize("mask_kind", ["none", "ragged", "zero_row"])
@pytest.mark.parametrize("L", [11, 256, 300])
@pytest.mark.parametrize("D", [16, 512, 1000])
def test_text_tokens(native, D, L, mask_kind):
    """Rows [row_off, row_off + 256) of c_out are exact selects (the rows around them keep their NaN sentinels); the
    pooled mean against float64 and, bit for bit, against the serial fp32 sum."""
    B, max_len, off = 4, 256, 4
    m = off + max_len + 3
    g = _g(D + L)
    proj, null = torch.randn(B, L, D, generator=g), torch.randn(max_len, D, generator=g)
    keep = torch.tensor([1, 0, 1, 1], dtype=torch.uint8)
    mask = None
    if mask_kind != "none":
        lens = torch.tensor([L, max(1, L // 3), 1, L - 1])
        mask = (torch.arange(L)[None, :] < lens[:, None]).to(torch.uint8)
        if mask_kind == "zero_row":
            mask[2] = 0
    c_e, p_e = torch.full((B, m, D), float("nan")), torch.empty(B, D)
    EMU.text_tokens(proj, B, L, D, mask, keep, null, max_len, c_e, m, off, p_e)
    c_n, p_n = torch.full((B, m, D), float("nan"), device="cuda"), torch.empty(B, D, device="cuda")
    native.text_tokens(proj.cuda(), B, L, D, _cu(mask), keep.cuda(), null.cuda(), max_len, c_n, m, off, p_n)
    _nan_equal(c_n, c_e, f"text rows D={D} L={L} {mask_kind}")
    assert c_n[:, :off].isnan().all() and c_n[:, off + max_len:].isnan().all()
    rows = c_e[:, off:off + max_len]
    ref, bound = R.text_pool_ref(rows)
    what = f"text pooled D={D} L={L} {mask_kind}"
    check(p_n, ref, bound, what)
    check_rel_l2(p_n, ref, 1e-6, what)
    assert torch.equal(p_n.cpu(), R.text_pool_fp32(rows)), f"{what}: not the serial fp32 sum"
