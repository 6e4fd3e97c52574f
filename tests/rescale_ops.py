"""TEST INFRASTRUCTURE ONLY: `RescaleEmuOps`, the torch emulation of the ops interface (IntervalEmuOps: EmuOps with the
multistep, RePaint and scheduled epilogues) plus the contracts of the guidance-rescale entry points
(mi_guidance_rescale_factor, mi_step_epilogue_rescaled).  Their float64 references (`rescale_factor_ref`, and
`rescaled_eps_fp32`, the prediction the rescaled step uses, formed as the kernels form it) are in tests/fp64_ref.py and
re-exported here; their per-call checkers are in tests/checking_ops.py.
"""
import torch

from fp64_ref import guided_fp32, rescale_factor_ref, rescaled_eps_fp32, scheduled_weights  # noqa: F401 (re-exported)
from test_guidance_interval import IntervalEmuOps

F32, F64 = torch.float32, torch.float64


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
