"""The per-call checkers of a training step (tests/checking_ops.py) are not vacuous: they run here, on a machine without a GPU,
over the torch emulation of the kernels' contract (tests/emu_ops.py: fp16 operands, fp32 accumulation) with the tensor-core
training routes switched on (autograd.ROUTE_TC_ON_CPU).

  * the emulation passes every call's float64 bound, and every method a step calls is checked;
  * one kernel-shaped defect per backward family, planted by wrapping that single emulated method, fails the check of that
    method.  Each defect prints the all-gradient rel-L2 against the clean step: the aggregate number a training step was
    judged by before (test_training.py: < 5e-3 against autograd, 1e-3 against train_tiny.pt).  Most of these defects sit
    far below both limits;
  * coverage: every training-side method of the ops interface has a checker and a GPU case that must reach it.

The bounds' accumulation lengths follow the kernels' plans for 132 SMs (an H100 SXM); the emulation's own summation order
is torch's, which the bounds cover as well as they cover the kernels'.
"""
import inspect
import re

import pytest
import torch

import fp64_ref as R
from checking_ops import ALLOWED, TRAINING_METHODS, CheckingOps, run_training_step, train_cases
from conftest import rel_l2
from emu_ops import EmuOps

SMS = 132
CASES = train_cases()


@pytest.fixture
def emu_tc(monkeypatch):
    """The emulated backend with the tensor-core training routes taken on the CPU; restored afterwards."""
    import minimagen_b200.autograd as ag
    import minimagen_b200.ops as ops_mod
    monkeypatch.setattr(ag, "ROUTE_TC_ON_CPU", True)
    prev = ops_mod._OPS
    e = EmuOps()
    yield e
    ops_mod.set_ops(prev)


def _step(ops, case):
    import minimagen_b200.ops as ops_mod
    ops_mod.set_ops(ops)
    return run_training_step(CASES[case][0], "cpu")


@pytest.mark.parametrize("case", ["base_d64_mid_attn", "cascade_unet1", "cascade_unet2"])
def test_emulated_training_step_passes_every_call_bound(emu_tc, case):
    proxy = CheckingOps(emu_tc, sms=SMS, fresh_accumulators=True)
    _step(proxy, case)
    print(f"\n{case} (emulated)")
    proxy.report()
    unchecked = proxy.called - proxy.checked - ALLOWED
    assert not unchecked, f"methods that ran without a float64 check: {sorted(unchecked)}"
    missing = CASES[case][1] - proxy.checked - proxy.features
    assert not missing, f"declared families not reached: {sorted(missing)}"


# ------------------------------------------------------------------------------------------------ planted kernel defects
def _wgrad_tc_split(emu):
    """conv_wgrad_tc: the last split's 8 x 8 pixel boxes (wgrad_tc_plan) missing from tap (0, 0)."""
    orig = emu.conv_wgrad_tc

    def f(dy16, x16, B, Ho, Wo, c_in, c_out, kh, kw, dw, stride=1):
        orig(dy16, x16, B, Ho, Wo, c_in, c_out, kh, kw, dw, stride)
        per, splits = R.wgrad_tc_plan(B, Ho, Wo, c_in, c_out, kh, SMS)
        box = torch.zeros(B * (Ho // 8) * (Wo // 8), dtype=torch.bool)
        box[(splits - 1) * per:] = True                                    # boxes in (image, box row, box column) order
        m = box.reshape(B, Ho // 8, 1, Wo // 8, 1, 1).expand(B, Ho // 8, 8, Wo // 8, 8, 1).reshape(B, Ho, Wo, 1)
        part = torch.empty_like(dw)
        orig((dy16.reshape(-1)[:B * Ho * Wo * c_out].reshape(B, Ho, Wo, c_out) * m).contiguous(), x16, B, Ho, Wo, c_in,
             c_out, kh, kw, part, stride)
        dw.reshape(c_out, c_in, kh, kw)[:, :, 0, 0] -= part.reshape(c_out, c_in, kh, kw)[:, :, 0, 0]
    return f


def _dgrad_border(emu):
    """conv_dgrad: the last dy column dropped at the right border."""
    orig = emu.conv_dgrad

    def f(dy, B, Ho, Wo, c_out, w, c_in, kh, kw, stride, pad, dx, Hi, Wi):
        d = dy.reshape(B, Ho, Wo, c_out).clone()
        d[:, :, -1] = 0
        orig(d, B, Ho, Wo, c_out, w, c_in, kh, kw, stride, pad, dx, Hi, Wi)
    return f


def _phase_taps(emu):
    """conv_igemm: sub-pixel phase mode 3 computed with mode 4's taps (a phase reads its neighbour's taps)."""
    orig = emu.conv_igemm

    def f(act, B, H, W, lda, c_off, c_in, wp, c_out, kh, kw, mode, *a, **k):
        return orig(act, B, H, W, lda, c_off, c_in, wp, c_out, kh, kw, 4 if mode == 3 else mode, *a, **k)
    return f


def _gn_bwd_split(emu):
    """gn_silu_bwd: the last pixel split (gn_bwd_splits) missing from the A1 sums, i.e. from dbeta and d shift."""
    orig = emu.gn_silu_bwd

    def f(x, dy, sums, B, hw, C, groups, gamma, beta, scale_shift, ss_ld, eps, dx, dgamma, dbeta, dss, dss_ld):
        orig(x, dy, sums, B, hw, C, groups, gamma, beta, scale_shift, ss_ld, eps, dx, dgamma, dbeta, dss, dss_ld)
        Z = R.gn_bwd_splits(B, hw, C, SMS)
        first = (Z - 1) * -(-hw // Z)
        d = torch.zeros_like(dy).reshape(B, hw, C)
        d[:, first:] = dy.reshape(B, hw, C)[:, first:]
        pdb = torch.zeros_like(dbeta)
        pss = None if dss is None else torch.zeros_like(dss)
        orig(x, d, sums, B, hw, C, groups, gamma, beta, scale_shift, ss_ld, eps, torch.empty_like(dx),
             torch.zeros_like(dgamma), pdb, pss, dss_ld)
        dbeta -= pdb
        if dss is not None:
            dss.as_strided((B, C), (dss_ld, 1), dss.storage_offset() + C).sub_(
                pss.as_strided((B, C), (dss_ld, 1), pss.storage_offset() + C))
    return f


def _ln_tanh_gelu(emu):
    """ln_rows_bwd: the tanh-approximate GELU' in place of the exact (erf) one, where a GELU precedes the LayerNorm."""
    orig = emu.ln_rows_bwd

    def f(inp, dy, rows, C, gamma, eps, pre_gelu, dx, dgamma, dbeta):
        if not pre_gelu:
            return orig(inp, dy, rows, C, gamma, eps, pre_gelu, dx, dgamma, dbeta)
        x = inp.reshape(rows, C)
        orig(torch.nn.functional.gelu(x).contiguous(), dy, rows, C, gamma, eps, False, dx, dgamma, dbeta)
        with torch.enable_grad():
            x_ = x.detach().clone().requires_grad_(True)
            gp = torch.autograd.grad(torch.nn.functional.gelu(x_, approximate="tanh"), x_, torch.ones_like(x_))[0]
        dx.reshape(rows, C).mul_(gp)
    return f


def _softmax_bwd_last_key(emu):
    """softmax_rows_bwd: the last key left out of the row dot product sum_j P_j dP_j."""
    def f(P, dP, rows, L):
        p, d = P.reshape(rows, L), dP.reshape(rows, L)
        d.copy_(p * (d - (p[:, :-1] * d[:, :-1]).sum(dim=-1, keepdim=True)))
    return f


def _gemm_ragged_k(emu):
    """gemm_f32: the last k of a K that is not a multiple of the 32-wide k tile dropped."""
    orig = emu.gemm_f32

    def f(A, B, C, M, N, K, *a, **k):
        return orig(A, B, C, M, N, K - 1 if K % 32 else K, *a, **k)
    return f


def _colsum_split(emu):
    """colsum: the last row split (colsum_acc_len's plan) lost."""
    orig = emu.colsum

    def f(x, M, Nc, out, accumulate=False):
        splits = min(-(-M // 1024), 512)
        xs = x.reshape(-1)[:M * Nc].reshape(M, Nc).clone()
        xs[(splits - 1) * -(-M // splits):] = 0
        orig(xs, M, Nc, out, accumulate)
    return f


def _upsample_order(emu):
    """upsample2x_bwd: the four taps summed column pair first, (a + c) + (b + d), instead of row pair first."""
    def f(dy, B, H, W, C, dx):
        q = dy.reshape(B, H, 2, W, 2, C)
        dx.reshape(B, H, W, C).copy_((q[:, :, 0, :, 0] + q[:, :, 1, :, 0]) + (q[:, :, 0, :, 1] + q[:, :, 1, :, 1]))
    return f


def _q_sample_next_t(emu):
    """q_sample: the schedule tables read at t + 1."""
    orig = emu.q_sample

    def f(x0, noise, t, tab_a, tab_b, B, n, post_scale, post_shift, out):
        orig(x0, noise, (t + 1).clamp(max=tab_a.numel() - 1), tab_a, tab_b, B, n, post_scale, post_shift, out)
    return f


DEFECTS = {
    "conv_wgrad_tc": ("base_d64_mid_attn", _wgrad_tc_split),
    "conv_dgrad": ("base_d64_mid_attn", _dgrad_border),
    "conv_igemm": ("base_d64_mid_attn", _phase_taps),
    "gn_silu_bwd": ("base_d64_mid_attn", _gn_bwd_split),
    "ln_rows_bwd": ("base_d64_mid_attn", _ln_tanh_gelu),
    "softmax_rows_bwd": ("base_d64_mid_attn", _softmax_bwd_last_key),
    "gemm_f32": ("base_d64_mid_attn", _gemm_ragged_k),
    "colsum": ("base_d64_mid_attn", _colsum_split),
    "upsample2x_bwd": ("base_d64_mid_attn", _upsample_order),
    "q_sample": ("cascade_unet2", _q_sample_next_t),
}
_CLEAN = {}


@pytest.mark.parametrize("method", list(DEFECTS))
def test_planted_kernel_defect_fails_its_call_check(emu_tc, method):
    """One step with the defect planted in `method`, checked for that method only (the float64 references of the other
    calls are what the clean test runs; each call's inputs are the step's own tensors, so a defect cannot fail another
    method's check).  The check must fail and name the method."""
    case, plant = DEFECTS[method]
    if case not in _CLEAN:
        _CLEAN[case] = _step(EmuOps(), case)
    clean = _CLEAN[case]
    setattr(emu_tc, method, plant(emu_tc))                                  # an instance attribute shadows the method
    proxy = CheckingOps(emu_tc, sms=SMS, fresh_accumulators=True, only={method}, strict=False)
    grads = _step(proxy, case)
    flat = lambda g: torch.cat([g[k].reshape(-1) for k in clean])
    rl = rel_l2(flat(grads), flat(clean))
    with pytest.raises(AssertionError) as e:
        proxy.raise_failures()
    print(f"\nplanted {plant.__name__.strip('_')}: caught in {method} ({len(proxy.failures)} failed calls); all-gradient "
          f"rel-L2 against the clean step {rl:.3e}\n  {str(e.value)[:300]}")
    assert proxy.failures and all(f.startswith(method + "(") for f in proxy.failures)


def test_planted_unscaled_gradient_cast_fails_its_conditioning_check(emu_tc, monkeypatch):
    """The backward's fp16 gradient casts unscaled (scale 1, as before autograd._grad_scales): every such cast is an exact
    fp16 rounding and passes its float64 check, but the copy no longer holds the gradient, and the conditioning check of
    cast_act must fail."""
    import minimagen_b200.autograd as ag
    monkeypatch.setattr(ag, "_grad_scales", lambda g: torch.ones(2, dtype=torch.float32, device=g.device))
    proxy = CheckingOps(emu_tc, sms=SMS, fresh_accumulators=True, only={"cast_act"}, strict=False)
    _step(proxy, "base_d64_mid_attn")
    with pytest.raises(AssertionError) as e:
        proxy.raise_failures()
    print(f"\nplanted unscaled gradient casts: {len(proxy.failures)} failed cast_act calls\n  {str(e.value)[-200:]}")
    assert proxy.failures and all(f.startswith("cast_act(") and "backward gradient" in f for f in proxy.failures)


# ------------------------------------------------------------------------------------------------ coverage
def test_every_training_method_has_a_checker_and_a_reaching_case():
    """The training-side section of NativeOps (everything after its "training side" banner), plus the two sampling-loop
    kernels a training step runs, must each have a `_check_` method and appear in some GPU case's declared families: a
    backward entry point added later cannot be missed."""
    from minimagen_b200.ops import NativeOps
    src = inspect.getsource(NativeOps)
    section = re.findall(r"^    def (\w+)\(", src[src.index("training side"):], flags=re.M)
    assert "gemm_f32" in section and "upsample2x_bwd" in section
    methods = (set(section) - ALLOWED) | TRAINING_METHODS
    no_checker = {m for m in methods if not hasattr(CheckingOps, "_check_" + m)}
    assert not no_checker, f"no per-call checker: {sorted(no_checker)}"
    declared = {f.split()[0] for _, fams in CASES.values() for f in fams}     # "conv_wgrad_tc k=3 s=1" reaches conv_wgrad_tc
    unreached = methods - declared
    assert not unreached, f"no training case declares: {sorted(unreached)}"
