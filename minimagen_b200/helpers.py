"""Small host-side helpers with the names the reference's callers import from `minimagen.helpers`
(reference: minimagen/helpers.py).  Only `extract` / `prob_mask_like` / `right_pad_dims_to` / normalisation touch
tensors, and none of them is on the per-step path of this package (the step kernels do the schedule gathers)."""
from contextlib import contextmanager
from functools import wraps

import math

import torch


def exists(val):
    return val is not None


def default(val, d):
    if exists(val):
        return val
    return d() if callable(d) else d


def cast_tuple(val, length=None):
    """list -> tuple; scalar -> tuple repeated `length` (1 if None) times; checks the length (helpers.py:9-23)."""
    if isinstance(val, list):
        val = tuple(val)
    out = val if isinstance(val, tuple) else ((val,) * default(length, 1))
    if exists(length):
        assert len(out) == length
    return out


def identity(t, *args, **kwargs):
    return t


def maybe(fn):
    @wraps(fn)
    def inner(x):
        return fn(x) if exists(x) else x
    return inner


def eval_decorator(fn):
    """Run `fn` with the model in eval mode, restoring the previous mode afterwards (helpers.py:35-46)."""
    def inner(model, *args, **kwargs):
        was_training = model.training
        model.eval()
        try:
            return fn(model, *args, **kwargs)
        finally:
            model.train(was_training)
    return inner


def module_device(module):
    return next(module.parameters()).device


@contextmanager
def null_context(*args, **kwargs):
    yield


def extract(a, t, x_shape):
    """a[t] reshaped to (b, 1, 1, ...) to broadcast against x_shape (helpers.py:56-67)."""
    b = t.shape[0]
    return a.gather(-1, t).reshape(b, *((1,) * (len(x_shape) - 1)))


def log(t, eps=1e-12):
    return torch.log(t.clamp(min=eps))


def normalize_neg_one_to_one(img):
    return img * 2 - 1


def unnormalize_zero_to_one(normed_img):
    return (normed_img + 1) * 0.5


def prob_mask_like(shape, prob, device):
    """Boolean keep-mask with P(True) = prob; deterministic (no RNG draw) for prob in {0, 1} (helpers.py:121-135)."""
    if prob == 1:
        return torch.ones(shape, device=device, dtype=torch.bool)
    if prob == 0:
        return torch.zeros(shape, device=device, dtype=torch.bool)
    return torch.zeros(shape, device=device).float().uniform_(0, 1) < prob


def right_pad_dims_to(x, t):
    pad = x.ndim - t.ndim
    return t if pad <= 0 else t.view(*t.shape, *((1,) * pad))


_RESIZE_TABLES = {}


def resize_tables(n_in, scale, pad_mode, device):
    """Tap tables of one axis of resize_right.resize (the reference's resampler; source not vendored, this follows the
    published algorithm, SURVEY.md 8c): Keys cubic (a = -0.5), support 4, pixel-centre aligned grid, antialiasing by kernel
    stretching when down-scaling, weights renormalised to sum 1, boundary by `pad_mode`.  Returns (n_out, idx int32
    [n_out, taps], w fp32 [n_out, taps])."""
    key = (n_in, float(scale), pad_mode, str(device))
    hit = _RESIZE_TABLES.get(key)
    if hit is not None:
        return hit
    n_out = int(math.ceil(n_in * scale))
    aa = scale < 1.
    stretch = (1. / scale) if aa else 1.
    cur_support = 4. * stretch
    out_coords = torch.arange(n_out, dtype=torch.float32)
    proj = out_coords / scale + (n_in - 1) / 2 - (n_out - 1) / (2 * scale)
    left = torch.ceil(proj - cur_support / 2 - 1e-7).long()
    n_taps = int(math.ceil(cur_support - 1e-7))
    taps = left[:, None] + torch.arange(n_taps)[None, :]
    d = ((proj[:, None] - taps.to(torch.float32)) / stretch).abs()
    d2, d3 = d * d, d * d * d
    w = (1.5 * d3 - 2.5 * d2 + 1.) * (d <= 1.).float() + (-0.5 * d3 + 2.5 * d2 - 4. * d + 2.) * ((d > 1.) & (d <= 2.)).float()
    w = w / w.sum(dim=1, keepdim=True)
    if pad_mode == 'reflect':
        idx = torch.where(taps < 0, -taps, taps)
        idx = torch.where(idx >= n_in, 2 * (n_in - 1) - idx, idx)
    elif pad_mode == 'symmetric':
        idx = torch.where(taps < 0, -taps - 1, taps)
        idx = torch.where(idx >= n_in, 2 * n_in - 1 - idx, idx)
    elif pad_mode in ('edge', 'replicate'):
        idx = taps.clamp(0, n_in - 1)
    else:   # 'constant': zero outside
        w = w * ((taps >= 0) & (taps < n_in)).float()
        idx = taps.clamp(0, n_in - 1)
    res = (n_out, idx.clamp(0, n_in - 1).to(torch.int32).contiguous().to(device), w.float().contiguous().to(device))
    _RESIZE_TABLES[key] = res
    return res


def resize_image_to(image, target_image_size, clamp_range=None, pad_mode='reflect'):
    """Inter-stage resize of the cascade (helpers.py:138-164 -> resize_right.resize; called at Imagen.py:482): one
    separable-resampling kernel (mi_resize_separable) driven by the tap tables above.  `target_image_size` is an int, as
    in the reference (both axes scaled by target / width), or a pair (h, w): each axis gets its own scale, h / H and
    w / W."""
    if isinstance(target_image_size, (tuple, list)):
        th, tw = map(int, target_image_size)
        if tuple(image.shape[-2:]) == (th, tw):
            return image
        scale_h, scale_w = th / image.shape[-2], tw / image.shape[-1]
    else:
        orig = image.shape[-1]
        if orig == target_image_size:
            return image
        scale_h = scale_w = target_image_size / orig
    from .ops import get_ops
    x = image.to(torch.float32).contiguous()
    B, C, H, W = x.shape
    ho, iy, wy = resize_tables(H, scale_h, pad_mode, x.device)
    wo, ix, wx = resize_tables(W, scale_w, pad_mode, x.device)
    if isinstance(target_image_size, (tuple, list)):
        assert (ho, wo) == (th, tw), f'resizing {H} x {W} to {th} x {tw} gives {ho} x {wo}'
    out = torch.empty((B, C, ho, wo), dtype=torch.float32, device=x.device)
    get_ops().resize_separable(x, B * C, H, W, out, ho, wo, iy, wy, ix, wx, clamp=clamp_range)
    return out
