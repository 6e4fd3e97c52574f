"""Every parameter gradient of a training step against float64, one tensor at a time, at the real loss scale.

The per-call checks (tests/checking_ops.py) compare each kernel with float64 on the operands it was given; on the tensor-core
backward routes those operands are fp16 copies of the gradient.  With an MSE-mean loss over b * 3 * H * W elements the
gradient at the output is ~2e-5 per element at 64 x 64, b = 8, and smaller deeper in the network: a plain fp16 cast would
make it subnormal and keep a bit or two of each element, and every call would still pass its check.  The backward therefore
casts each gradient scaled by a power of two chosen from its amax (minimagen_b200/autograd.py, `_grad_scales`).

Here one step of a 64-px U-Net (the network of tests/test_gpu_graphed_training.py's replay test, b = 8, 16 tokens of width
768) runs on the CPU over the emulation of the kernels' contract (tests/emu_ops.py: fp16 operands, fp32 accumulation) with
the tensor-core training routes taken (autograd.ROUTE_TC_ON_CPU).  Each parameter gradient is compared with torch autograd
through the reference restatement (oracle/restatement.py) in float64, with the same weights and inputs (its float64
lowering equals the restatement to 1e-12: tests/test_lowering_exact.py).  Every tensor's rel-L2 must stay within LIMIT;
the ten worst are printed.

  * MSE and L1 losses (Imagen(loss_type='l1') gives sign / N gradients of the same size);
  * the loss scaled by 2^32 and the gradients unscaled after: the scaled gradient cast must not saturate either;
  * planted control: with the scaling switched off the attention query projections (`to_q.weight`) fail.

tests/test_gpu_train_grad_accuracy.py runs the same comparison on the H100 at the benchmark's training size.
"""
import pytest
import torch
import torch.nn.functional as F

from checking_ops import perturbed_unet
from emu_ops import EmuOps

F64 = torch.float64
BASE_D64 = dict(dim=64, dim_mults=(1, 2), attend_at_middle=True, text_embed_dim=768, layer_cross_attns=(False, True))
# per parameter tensor, rel-L2 of the gradient against float64: > 3x the worst measured with the scaled casts (4.6e-3,
# init_conv.convs.2.weight under the L1 loss; 2.1e-3 under MSE); unscaled, the to_q weights reach 0.48 - 0.93
LIMIT = 1.5e-2


def rel_per_tensor(mine, ref):
    """{name: ||mine - ref|| / ||ref||} in float64 (0 where both are zero)."""
    out = {}
    for k, r in ref.items():
        a, b = mine[k].detach().to(F64).cpu(), r.detach().to(F64).cpu()
        d = float((a - b).norm())
        out[k] = d / float(b.norm()) if d else 0.0
    return out


def report(what, rels, n=10):
    worst = sorted(rels.items(), key=lambda kv: -kv[1])[:n]
    med = sorted(rels.values())[len(rels) // 2]
    print(f"\n{what}: {len(rels)} tensors, median rel-L2 {med:.2e}, the {n} worst (limit {LIMIT:.1e}):")
    for k, v in worst:
        print(f"  {v:.3e}  {k}")
    return worst[0]


def reference_grads(unet, cfg, x, t, kw, target, loss_fn, keep=None):
    """Every parameter gradient of loss_fn(U-Net(x), target) by torch autograd through the float64 restatement, on the device
    of the inputs.  keep (bool [b]): the conditioning-dropout draw; rows not kept take the null conditioning (the
    restatement runs each batch row independently, so the two cond_drop_prob settings are selected row by row)."""
    from oracle import restatement as R
    names = {k for k, p in unet.named_parameters()}
    sd = {k: v.detach().to(F64).requires_grad_(k in names) for k, v in unet.state_dict().items()}
    d = lambda v: v.to(F64) if torch.is_tensor(v) and v.is_floating_point() else v
    args = dict(text_embeds=d(kw["text_embeds"]), text_mask=kw.get("text_mask"), lowres_cond_img=d(kw.get("lowres_cond_img")),
                lowres_noise_times=kw.get("lowres_noise_times"))
    pred = R.unet_forward(sd, cfg, d(x), t, cond_drop_prob=0., **args)
    if keep is not None and not bool(keep.all()):
        null = R.unet_forward(sd, cfg, d(x), t, cond_drop_prob=1., **args)
        pred = torch.where(keep.bool().reshape(-1, 1, 1, 1), pred, null)
    loss_fn(pred, d(target)).backward()
    return {k: sd[k].grad for k in names}


# ------------------------------------------------------------------------------------------------ the CPU case
S, B, L = 64, 8, 16


@pytest.fixture(scope="module")
def case():
    """weights, inputs and the float64 reference gradients of both losses (computed once for the module)"""
    torch.manual_seed(0)
    unet = perturbed_unet(BASE_D64)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, 3, S, S, generator=g)
    tm = torch.ones(B, L, dtype=torch.bool)
    tm[-1, 9:] = False
    kw = dict(text_embeds=torch.randn(B, L, 768, generator=g), text_mask=tm)
    t = torch.randint(0, 1000, (B,), generator=g)
    target = torch.randn(x.shape, generator=g)
    ref = {name: reference_grads(unet, BASE_D64, x, t, kw, target, fn)
           for name, fn in (("mse", F.mse_loss), ("l1", F.l1_loss))}
    return unet, x, t, kw, target, ref


@pytest.fixture
def emu_tc(monkeypatch):
    """the emulated kernels with the tensor-core training routes taken on the CPU; restored afterwards"""
    import minimagen_b200.autograd as ag
    import minimagen_b200.ops as ops_mod
    monkeypatch.setattr(ag, "ROUTE_TC_ON_CPU", True)
    prev = ops_mod._OPS
    ops_mod.set_ops(EmuOps())
    yield ag
    ops_mod.set_ops(prev)


def _step(case, loss, scale=1.0):
    unet, x, t, kw, target, _ = case
    unet.zero_grad(set_to_none=True)
    fn = {"mse": F.mse_loss, "l1": F.l1_loss}[loss]
    (fn(unet(x, t, **kw), target) * scale).backward()
    return {k: p.grad / scale for k, p in unet.named_parameters()}


@pytest.mark.parametrize("loss,scale", [("mse", 1.0), ("l1", 1.0), ("mse", 2.0 ** 32)],
                         ids=["mse", "l1", "mse_loss_x2^32"])
def test_every_parameter_gradient_against_float64(case, emu_tc, loss, scale):
    rels = rel_per_tensor(_step(case, loss, scale), case[5][loss])
    worst = report(f"{loss} loss x {scale:g}, emulated fp16 backward vs float64", rels)
    assert worst[1] <= LIMIT, f"{worst[0]}: gradient rel-L2 {worst[1]:.3e} against float64 (limit {LIMIT:.1e})"


def test_planted_unscaled_gradient_casts_fail(case, emu_tc, monkeypatch):
    """Planted control: the gradients cast to fp16 as they are (scale 1) lose the attention query projections'."""
    monkeypatch.setattr(emu_tc, "_grad_scales", lambda g: torch.ones(2, dtype=torch.float32, device=g.device))
    rels = rel_per_tensor(_step(case, "mse"), case[5]["mse"])
    report("planted: unscaled fp16 gradient casts, mse loss", rels)
    bad = {k for k, v in rels.items() if v > LIMIT}
    assert any(k.endswith("to_q.weight") for k in bad), sorted(bad)
