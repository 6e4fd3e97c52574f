"""Every kernel call of a real U-Net forward, and of a real training step, against float64, at the arguments the network
actually passes.

The kernel tests (test_gpu_image_fwd.py, test_gpu_image_bwd.py, test_gpu_token_ops.py, test_gpu_sampler_ops.py) chose their
shapes by hand; here the shapes, channel offsets, row pitches, strides, n_valid, statistics buffers, batch strides and
accumulators come from the lowering itself.  `CheckingOps` (tests/checking_ops.py) wraps the native backend: for each call it
NaN-fills the pure outputs, makes the call, synchronises, and checks the outputs against the float64 reference of
tests/fp64_ref.py built from THAT call's own arguments, with that reference's per-element bound.  The inputs of every call are
the native run's own tensors, so no error compounds from one call to the next: together with tests/test_lowering_exact.py
(the dataflow is exact) this replaces the whole-network rel-L2 (< 2e-3 forward, < 5e-3 over all gradients) as the sharp
check.

  * forward: epilogue / gn_stats statistics are checked as the INCREMENT of the accumulator over the call; every statistics
    accumulator is zero when first handed to a kernel and no two overlap (the ZeroArena carving);
  * training step (eager forward under grad mode, MSE loss, loss.backward(), train mode): every backward entry point, the
    training forward's own routes (cast_act + conv_igemm / conv_direct, gn_stats + gn_apply_silu with group sums, LinearFn
    on zero-padded 128-row tiles, attention as gemm_f32 + softmax_rows) and the sampling-loop kernels Imagen.forward runs
    (resize_separable, q_sample); every accumulator is zero at every hand-off.  Each case declares the families it must
    reach (checking_ops.train_cases) and fails if one was not reached;
  * completeness: the methods a run called minus the methods checked must be empty apart from `ALLOWED` (capability
    queries), so a kernel added later cannot slip through unchecked.

The float64 references are computed on the GPU (the operands' device).  The batch_streams = 2 case is a dataflow check of the
batch chunking (slices of the conditioning, of the scale/shift rows and of the output), not of concurrency: the proxy
synchronises after every call.  Nothing here is repeated or stressed: each case is one ordinary forward or training step.
"""
import time

import pytest
import torch

from checking_ops import ALLOWED, CheckingOps, run_training_step, train_cases

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ the cases
def _inputs(cfg, s, b, L=20, seed=3, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, 3, s, s, generator=g)
    tm = torch.ones(b, L, dtype=torch.bool)
    tm[-1, 5:] = False
    kw = dict(text_embeds=torch.randn(b, L, cfg.get("text_embed_dim", 512), generator=g), text_mask=tm)
    if cfg.get("lowres_cond"):
        kw.update(lowres_cond_img=torch.randn(b, 3, s, s, generator=g), lowres_noise_times=torch.full((b,), 200))
    t = torch.randint(0, 1000, (b,), generator=g)
    return x.to(device), t.to(device), {k: v.to(device) for k, v in kw.items()}


def _cases():
    from test_gpu_unet import CFGS
    from minimagen_b200.Unet import Super
    for name, cfg, s, _, b in CFGS[:3]:
        yield name, cfg, s, b, {}
    yield "cfg3_structure_64x64", dict(Super.defaults, lowres_cond=True, text_embed_dim=768), 64, 2, {}
    streams = dict(dim=64, dim_mults=(1, 2), num_resnet_blocks=1, layer_attns=(False, True), layer_cross_attns=(False, True),
                   lowres_cond=True, memory_efficient=True, text_embed_dim=768)
    yield "batch16_two_chunks", streams, 32, 16, dict(batch_streams=2)
    yield "cfg_batched", dict(dim=64, dim_mults=(1, 2), text_embed_dim=512), 32, 4, dict(cfg_batched=True)


CASES = list(_cases()) if torch.cuda.is_available() else []


def forward_case(name, device="cuda"):
    """(U-Net, x, t, conditioning, b, options) of the forward case `name` of _cases(), on `device`."""
    from minimagen_b200.Unet import Unet
    _, cfg, s, b, opt = next(c for c in _cases() if c[0] == name)
    torch.manual_seed(0)
    u = Unet(**cfg).eval().to(device)
    x, t, kw = _inputs(cfg, s, b, device=device)
    return u, x, t, kw, b, opt


def run_forward(ops, u, x, t, kw, b, opt):
    """One forward of a case with `ops` installed as the backend (left installed: the caller restores it)."""
    import minimagen_b200.ops as ops_mod
    ops_mod.set_ops(ops)
    with torch.no_grad():
        if opt.get("cfg_batched"):               # Imagen.cfg_batched: conditional and unconditional pass as one 2B batch
            two = lambda v: torch.cat((v, v))
            keep = torch.cat((torch.ones(b, dtype=torch.uint8), torch.zeros(b, dtype=torch.uint8))).to(x.device)
            return u._forward_impl(two(x), two(t), cond_keep=keep, **{k: two(v) for k, v in kw.items()})
        u.batch_streams = opt.get("batch_streams", 1)
        assert len(u._batch_chunks(b, x.is_cuda)) == u.batch_streams
        return u(x, t, **kw)


@pytest.mark.parametrize("name,cfg,s,b,opt", CASES, ids=[c[0] for c in CASES])
def test_every_call_of_a_forward(native, name, cfg, s, b, opt):
    u, x, t, kw, b, opt = forward_case(name)
    proxy = CheckingOps(native)
    t0 = time.time()
    out = run_forward(proxy, u, x, t, kw, b, opt)   # the `native` fixture restores the previous backend afterwards
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    n_acc = proxy.assert_accumulators_disjoint()
    props = torch.cuda.get_device_properties(0)
    print(f"\n{name} on {props.name}: {time.time() - t0:.1f} s, {n_acc} statistics accumulators (zero when handed out, disjoint)")
    for fam, (calls, worst) in sorted(proxy.family.items()):
        print(f"  {fam:28s} {calls:5d} calls   worst |err|/bound {worst:.3g}")
    unchecked = proxy.called - proxy.checked - ALLOWED
    assert not unchecked, f"kernels that ran without a float64 check: {sorted(unchecked)}"
    assert {"conv_igemm", "gn_apply_silu", "attention", "ln_rows", "linear_f32"} <= proxy.checked


TRAIN_CASES = train_cases() if torch.cuda.is_available() else {}


@pytest.mark.parametrize("name", list(TRAIN_CASES))
def test_every_call_of_a_training_step(native, name):
    """One eager training step per case (forward under grad mode in train mode, MSE loss, loss.backward()), every kernel call
    checked; the case must reach the families it declares (checking_ops.train_cases)."""
    import minimagen_b200.ops as ops_mod
    spec, declared = TRAIN_CASES[name]
    proxy = CheckingOps(native, fresh_accumulators=True)
    ops_mod.set_ops(proxy)                      # the `native` fixture restores the previous backend afterwards
    t0 = time.time()
    grads = run_training_step(spec, "cuda")
    torch.cuda.synchronize()
    dt = time.time() - t0
    assert all(torch.isfinite(g).all() for g in grads.values())
    props = torch.cuda.get_device_properties(0)
    print(f"\n{name} training step on {props.name} ({proxy.sms} SMs): {dt:.1f} s, {len(grads)} parameter gradients")
    proxy.report()
    unchecked = proxy.called - proxy.checked - ALLOWED
    assert not unchecked, f"kernels that ran without a float64 check: {sorted(unchecked)}"
    missing = declared - proxy.checked - proxy.features
    assert not missing, f"declared families not reached: {sorted(missing)}"
