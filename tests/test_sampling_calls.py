"""The per-call checkers of the sampling loop's kernels (tests/checking_ops.py: step_epilogue, step_epilogue_multistep,
step_advance_t, step_advance_t_table, step_finalize) are not vacuous.  They run here, on a machine without a GPU, over the
torch emulation of the kernels' contract:

  * an eager DDIM and DPM-Solver++(2M) sampling loop over the tiny golden U-Net passes every step check;
  * the timestep walks pass their exact checks, over the grid and out of range;
  * the fp32 step in the kernels' order (test_error_bounds.step_fp32) passes, and each planted defect of it fails the
    check of the method it was planted in: a select rank off by one, the thresholds of the neighbouring image, the first
    image's guidance weight for every image, noise left on at t = 0, a history that is not clamped; likewise a walk that
    goes below t = 0 and a finalize that forgets the clamp.

The GPU runs the same checkers over the native kernels in test_gpu_flagship_calls.py, at the benchmark's batch.
"""
import pytest
import torch

from checking_ops import CheckingOps
from conftest import load_golden
from emu_ops import EmuOps
from test_error_bounds import _schedule, _step_data, step_fp32
from test_respaced import _tiny_imagen

SMS = 132
LOOP = {"step_epilogue", "step_epilogue_multistep", "step_advance_t", "step_advance_t_table", "step_finalize",
        "resize_separable", "q_sample"}


@pytest.mark.parametrize("sampler", ["ddim", "dpmpp_2m"])
def test_emulated_sampling_loop_passes_every_step_check(emu, sampler):
    import minimagen_b200.ops as ops_mod
    g = load_golden("sample_loop.pt")
    im = _tiny_imagen(g, 1000)
    im.use_cuda_graph = False
    proxy = CheckingOps(emu, sms=SMS, only=LOOP)
    ops_mod.set_ops(proxy)
    torch.manual_seed(4)
    im.sample(text_embeds=g["text_embeds"], text_masks=g["text_mask"], cond_scale=3., sampling_timesteps=4,
              sampler=sampler)
    step = "step_epilogue_multistep" if sampler == "dpmpp_2m" else "step_epilogue"
    assert proxy.family[step][0] == 4 and {step, "step_finalize"} <= proxy.checked
    print(f"\n{sampler} loop (emulated)")
    proxy.report()


def test_emulated_timestep_walks_pass_their_exact_checks():
    from minimagen_b200.diffusion_model import GaussianDiffusion
    proxy = CheckingOps(EmuOps(), sms=SMS)
    sch = GaussianDiffusion(timesteps=1000).sampling_schedule(6, 0.5, "cpu")
    t = torch.full((3,), 999, dtype=torch.long)
    for _ in range(len(sch.grid) + 1):
        proxy.step_advance_t_table(t, sch.next_t, 1000, 3)
        proxy.step_advance_t(t, 3)
    t = torch.tensor([-1, 1000, 1 << 40, 999, 0], dtype=torch.long)
    proxy.step_advance_t_table(t, sch.next_t, 1000, t.numel())
    assert t.tolist() == [0, 0, 0, int(sch.next_t[999]), 0]
    assert {"step_advance_t", "step_advance_t_table"} <= proxy.checked


# ------------------------------------------------------------------------------------------------ planted step defects
def _step_with(defect):
    """The step epilogue and its multistep form computed by step_fp32 (the fp32 step in the kernels' order) with one
    planted defect ("hist": the history takes the unclamped x0); (plain, multistep) in the ops interface's signatures."""
    def run(x_t, eps_cond, eps_null, w, t, tabs, noise, hist, B, n, lo, hi, wt, min_s, out, s_out):
        x0, s, o, xs = step_fp32(x_t.reshape(B, n), eps_cond.reshape(B, n), eps_null.reshape(B, n), w, t, tabs, lo, hi,
                                 wt, min_s, noise.reshape(B, n), None if hist is None else hist.reshape(B, n),
                                 defect=None if defect == "hist" else defect)
        out.reshape(B, n).copy_(o)
        if s_out is not None:
            s_out.copy_(s)
        if hist is not None:
            hist.reshape(B, n).copy_(x0 if defect == "hist" else xs)

    def plain(x_t, eps_cond, eps_null, w, t, a, b, c1, c2, sigma, noise, B, n, lo, hi, wt, min_s, out, s_out=None):
        run(x_t, eps_cond, eps_null, w, t, (a, b, c1, c2, sigma, None), noise, None, B, n, lo, hi, wt, min_s, out, s_out)

    def multi(x_t, eps_cond, eps_null, w, t, a, b, c1, c2, sigma, c3, noise, hist, B, n, lo, hi, wt, min_s, out,
              s_out=None):
        run(x_t, eps_cond, eps_null, w, t, (a, b, c1, c2, sigma, c3), noise, hist, B, n, lo, hi, wt, min_s, out, s_out)
    return plain, multi


def _run_step(ops, multi, alias):
    """One step call through `ops` on test_error_bounds' step data: three images at different t (one at t = 0, where the
    schedule's sigma is 0.25 so that noise left on shows), per-image weights 7 / 3 / 1.5, the last image's threshold below
    min_s = 1."""
    from minimagen_b200.Imagen import quantile_rank
    *tabs, grid = _schedule("dpmpp" if multi else "ddpm")
    a, b, c1, c2, sigma, c3 = tabs
    B, n = 3, 3 * 64 * 64
    x, eps, eps0, noise, hist, t, w = _step_data(B, n, 5, grid)
    lo, hi, wt = quantile_rank(n, 0.9)
    out, s = (x if alias else torch.empty_like(x)), torch.empty(B)
    if multi:
        ops.step_epilogue_multistep(x, eps, eps0, w, t, a, b, c1, c2, sigma, c3, noise, hist, B, n, lo, hi, wt, 1.0, out,
                                    s_out=s)
    else:
        ops.step_epilogue(x, eps, eps0, w, t, a, b, c1, c2, sigma, noise, B, n, lo, hi, wt, 1.0, out, s_out=s)


class _Planted:
    """An ops object holding only the planted methods (the proxy finds them by name)."""

    def __init__(self, **methods):
        self.__dict__.update(methods)


@pytest.mark.parametrize("multi", [False, True])
@pytest.mark.parametrize("alias", [False, True])
def test_fp32_step_passes_its_call_check(multi, alias):
    plain, ms = _step_with(None)
    proxy = CheckingOps(_Planted(step_epilogue=plain, step_epilogue_multistep=ms), sms=SMS)
    _run_step(proxy, multi, alias)
    proxy.report()
    assert proxy.checked == {"step_epilogue_multistep" if multi else "step_epilogue"}


STEP_DEFECTS = [("rank", False), ("neighbour", False), ("w0", False), ("sigma0", False), ("rank", True), ("hist", True)]


@pytest.mark.parametrize("defect,multi", STEP_DEFECTS, ids=[f"{d}-{'multistep' if m else 'plain'}" for d, m in STEP_DEFECTS])
def test_planted_step_defect_fails_its_call_check(defect, multi):
    method = "step_epilogue_multistep" if multi else "step_epilogue"
    plain, ms = _step_with(defect)
    proxy = CheckingOps(_Planted(step_epilogue=plain, step_epilogue_multistep=ms), sms=SMS, strict=False)
    _run_step(proxy, multi, alias=False)
    with pytest.raises(AssertionError) as e:
        proxy.raise_failures()
    print(f"\nplanted {defect}: {str(e.value)[:300]}")
    assert proxy.failures and all(f.startswith(method + "(") for f in proxy.failures)


def _walk_below_zero(t, B):
    t.sub_(1)


def _finalize_without_clamp(x, n, unnormalize, out):
    out.reshape(-1)[:n].copy_((x.reshape(-1)[:n] + 1.0) * 0.5 if unnormalize else x.reshape(-1)[:n])


def test_planted_walk_and_finalize_defects_fail_their_call_checks():
    proxy = CheckingOps(_Planted(step_advance_t=_walk_below_zero, step_finalize=_finalize_without_clamp), sms=SMS,
                        strict=False)
    proxy.step_advance_t(torch.tensor([3, 0, 999]), 3)
    x = torch.randn(2, 3, 8, 8, generator=torch.Generator().manual_seed(2)) * 2
    for unnormalize in (0, 1):
        proxy.step_finalize(x, x.numel(), unnormalize, torch.empty_like(x))
    assert [f.split("(")[0] for f in proxy.failures] == ["step_advance_t", "step_finalize", "step_finalize"]
