"""Every parameter gradient of a training step on the H100 against float64, one tensor at a time, at the real loss scale
(tests/test_train_grad_accuracy.py is the CPU case and explains why: the backward's fp16 gradient operands).

One eager Imagen training step (forward, MSE loss, backward) on the native kernels, for the two cases of
tests/test_gpu_graphed_training.py: the benchmark's `train` row (base U-Net, dim 128, 64 x 64, b = 8, 16 tokens of width
768) and a super-resolution stage with v-prediction on a zero-terminal-SNR schedule.  The step's draws (timesteps, noise,
low-res augmentation noise, conditioning dropout) are recorded with that module's hooks, and the U-Net's inputs and the
loss target are taken as the step passed them.  The reference is torch autograd through the reference restatement
(oracle/restatement.py) in float64 on the device, with the same weights, inputs and dropout draw.  Every tensor's rel-L2
must stay within the CPU case's LIMIT; the ten worst are printed.
"""
import pytest
import torch

from test_gpu_graphed_training import CASES, DrawRecorder, _build
from test_train_grad_accuracy import LIMIT, reference_grads, rel_per_tensor, report

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", list(CASES))
def test_every_parameter_gradient_against_float64(native, monkeypatch, case):
    spec = CASES[case]
    n, b = spec["unet_number"], spec["b"]
    rec = DrawRecorder()
    rec.install(monkeypatch)
    im = _build(spec)
    u = im.unets[n - 1]
    s = spec["sizes"][-1]
    g = torch.Generator().manual_seed(3)
    imgs = torch.rand(b, 3, s, s, generator=g).cuda()
    te = torch.randn(b, 16, 768, generator=g).cuda()
    tm = torch.ones(b, 16, dtype=torch.bool)
    if n > 1:
        tm[-1, 9:] = False
    tm = tm.cuda()

    seen = {}
    forward, loss_fn = u.forward, im.loss_fn

    def record_forward(x, time, **kw):
        seen.update(x=x.detach().clone(), t=time.clone(),
                    kw={k: v.detach().clone() if torch.is_tensor(v) else v for k, v in kw.items()})
        return forward(x, time, **kw)

    def record_loss(pred, target):
        seen["target"] = target.detach().clone()
        return loss_fn(pred, target)

    monkeypatch.setattr(u, "forward", record_forward)
    monkeypatch.setattr(im, "loss_fn", record_loss)
    u.zero_grad(set_to_none=True)
    loss = im(imgs, text_embeds=te, text_masks=tm, unet_number=n)
    loss.backward()
    torch.cuda.synchronize()
    assert rec.names == spec["draws"], rec.names
    mine = {k: p.grad for k, p in u.named_parameters()}
    keep = rec.bufs[rec.names.index("keep")]
    ref = reference_grads(u, spec["unets"][n - 1], seen["x"], seen["t"], seen["kw"], seen["target"], loss_fn, keep)
    rels = rel_per_tensor(mine, ref)
    worst = report(f"{case}: loss {float(loss.detach()):.5f}, {int(keep.sum())}/{b} conditioned; native backward vs float64", rels)
    assert worst[1] <= LIMIT, f"{worst[0]}: gradient rel-L2 {worst[1]:.3e} against float64 (limit {LIMIT:.1e})"
