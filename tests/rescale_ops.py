"""TEST INFRASTRUCTURE ONLY: the guidance-rescale entry points (mi_guidance_rescale_factor, mi_step_epilogue_rescaled) for
the test harness, next to the existing ones without changing them:

  * float64 references with error bounds, in the form of tests/fp64_ref.py (`rescale_factor_ref`, and
    `rescaled_eps_fp32`, the prediction the rescaled step uses, formed as the kernels form it);
  * `RescaleEmuOps`: the torch emulation of the ops interface (IntervalEmuOps: EmuOps with the multistep, RePaint and
    scheduled epilogues) plus the two entry points' contracts;
  * `RescaleCheckingOps`: CheckingOps plus a per-call float64 checker for each of the two, so that a run with guidance
    rescale has no unchecked kernel.
"""
import torch

import fp64_ref as R
from checking_ops import NAN, CheckingOps
from test_guidance_interval import IntervalEmuOps

F32, F64 = torch.float32, torch.float64


# ------------------------------------------------------------------------------------------------ float64 references
def scheduled_weights(w, w_sched, t, B):
    """image_scale (csrc/step.cu) as fp32 [B] on the CPU: w_b, or 1 + (w_b - 1) * w_sched[t_b] rounded op by op where the
    guidance table is not 1."""
    wt = w.detach().cpu().to(F32) if torch.is_tensor(w) else torch.full((B,), R._f32(w), dtype=F32)
    if w_sched is None:
        return wt
    s = w_sched.detach().cpu()[t.detach().cpu()]
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
    return f, 2 * R.U32 * f.abs() + R.ETA32


def rescaled_eps_fp32(eps_cond, eps_null, w, w_sched, t, f, B, n):
    """The prediction the rescaled step uses in place of g: fp32(g * f_b) [B, n] (g from guided_fp32), on the CPU."""
    return guided_fp32(eps_cond, eps_null, w, w_sched, t, B, n) * f.detach().cpu().reshape(-1)[:B, None]


# ------------------------------------------------------------------------------------------------ emulation
class RescaleEmuOps(IntervalEmuOps):
    """IntervalEmuOps plus the contracts of mi_guidance_rescale_factor and mi_step_epilogue_rescaled."""

    @staticmethod
    def _guided(eps_cond, eps_null, cond_scale, w_sched, t, B, n):
        """g = null + (cond - null) * w_b(t), fp32 op by op (image_scale of csrc/step.cu for the weights)."""
        w = cond_scale.to(F32) if torch.is_tensor(cond_scale) else torch.full((B,), float(cond_scale), dtype=F32)
        w = w.to(eps_cond.device)
        if w_sched is not None:
            sc = w_sched[t].to(w.device)
            w = torch.where(sc == 1, w, 1 + (w - 1) * sc)
        nl = eps_null.reshape(B, n)
        return nl + (eps_cond.reshape(B, n) - nl) * w[:, None]

    def guidance_rescale_factor(self, eps_cond, eps_null, cond_scale, w_sched, t, phi, B, n, f):
        """contract of mi_guidance_rescale_factor: fp64 sums of squares about the mean, f rounded once to fp32"""
        self._log("guidance_rescale_factor")
        c = eps_cond.reshape(B, n).double()
        g = self._guided(eps_cond, eps_null, cond_scale, w_sched, t, B, n).double()
        ssc = ((c - c.mean(dim=1, keepdim=True)) ** 2).sum(dim=1)
        ssg = ((g - g.mean(dim=1, keepdim=True)) ** 2).sum(dim=1)
        ph = phi.double()
        f.copy_(torch.where(ssg == 0, torch.ones_like(ssg), ph * (ssc / ssg).sqrt() + (1. - ph)).to(F32))

    def step_epilogue_rescaled(self, x_t, eps_cond, eps_null, cond_scale, w_sched, f, t, tab_a, tab_b, c1, c2, sigma, c3,
                               noise, hist, B, n, rank_lo, rank_hi, weight, min_s, out, s_out=None):
        """contract of mi_step_epilogue_rescaled == the step of fp32(g * f) without a guidance pass; with c3 and hist the
        multistep form (c3 term selected away where c3[t] == 0; hist <- the clamped x0)"""
        self._log("step_epilogue_rescaled")
        e = self._guided(eps_cond, eps_null, cond_scale, w_sched, t, B, n) * f[:, None]
        x0 = torch.empty_like(x_t)
        s = torch.empty(B, dtype=F32, device=x_t.device)
        self.step_x0(x_t, e, None, 1.0, t, tab_a, tab_b, B, n, x0)
        self.step_quantile(x0, B, n, rank_lo, rank_hi, weight, min_s, s)
        sb = s[:, None]
        xs = x0.reshape(B, n).clamp(-sb, sb) / sb
        mean = c1[t][:, None] * xs + c2[t][:, None] * x_t.reshape(B, n)
        if c3 is not None:
            c3t = c3[t][:, None]
            mean = torch.where(c3t != 0, mean + c3t * hist.reshape(B, n), mean)
            hist.reshape(B, n).copy_(xs)
        sig = torch.where(t == 0, torch.zeros_like(sigma[t]), sigma[t])[:, None]
        out.reshape(B, n).copy_(mean + sig * noise.reshape(B, n))
        if s_out is not None:
            s_out.copy_(s)


# ------------------------------------------------------------------------------------------------ per-call checks
class RescaleCheckingOps(CheckingOps):
    """CheckingOps plus the checkers of the two guidance-rescale entry points."""

    def _check_guidance_rescale_factor(self, eps_cond, eps_null, cond_scale, w_sched, t, phi, B, n, f):
        """f [B] within one fp32 ulp of the fp64 factor of the fp32 guided prediction (rescale_factor_ref)."""
        self._count("guidance_rescale_factor")
        w = cond_scale.detach().cpu().clone() if torch.is_tensor(cond_scale) else cond_scale
        ref, bound = rescale_factor_ref(eps_cond, eps_null, w, w_sched, t, phi, B, n)
        f.fill_(NAN)
        yield
        self._note("guidance_rescale_factor", R.check(f.reshape(-1)[:B], ref, bound, "guidance_rescale_factor f"))

    def _check_step_epilogue_rescaled(self, x_t, eps_cond, eps_null, cond_scale, w_sched, f, t, tab_a, tab_b, c1, c2,
                                      sigma, c3, noise, hist, B, n, rank_lo, rank_hi, weight, min_s, out, s_out=None):
        """The step of the fp32 rescaled prediction fp32(g * f_b) (rescaled_eps_fp32, formed as the kernel forms it) with
        no guidance pass: the checks of step_epilogue(_multistep) on that input."""
        w = cond_scale.detach().cpu().clone() if torch.is_tensor(cond_scale) else cond_scale
        eps = rescaled_eps_fp32(eps_cond, eps_null, w, w_sched, t, f, B, n)
        return self._step("step_epilogue_rescaled", x_t, eps, None, 1.0, t, tab_a, tab_b, c1, c2, sigma, c3, noise, hist,
                          B, n, rank_lo, rank_hi, weight, min_s, out, s_out)
