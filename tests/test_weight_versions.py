"""The eval and sampling path caches what it derives from the weights, keyed on each parameter's version counter:
  * the fp16 packed weights of the tensor-core convolutions and linear layers (layers._PackCache), the folded 3x3 + 1x1
    conv (Conv2d._pack_fold), the sub-pixel Upsample taps, the skip-scaled concat weights, the final conv's padded NCHW
    pack and the stem's 15 x 15 window (CrossEmbedLayer._stem_weights);
  * the attention q / kv / out packs (Attention / CrossAttention _pq, _pkv, _po);
  * the concatenated time-MLP weights (Unet._all_scale_shifts);
  * the static text projection (Unet.register_static_text);
  * the captured sampling step graphs (Imagen._graph_key sums the versions).
A CUDA graph replay of Imagen.graphed_train_step updates the parameters in place on the device without torch's
dispatcher, so the counters do not move, exactly as with an update through `.data`.  Here, on the torch emulation of
the kernels (tests/emu_ops.py), the parameters are updated through `.data`:
  * without `Imagen.bump_versions` every cache hits and serves the old weights, so the forward differs from that of a
    fresh U-Net with the same state_dict (if the caches are ever keyed on something else, this half fails and the test
    must be revisited);
  * with it every cache is rebuilt, the forward is bitwise that of the fresh U-Net, and the step-graph key changes.
"""
import pytest
import torch

from conftest import rel_l2

CFG = dict(dim=64, dim_mults=(1, 2), attend_at_middle=True, text_embed_dim=768, layer_cross_attns=(False, True))
CACHE_ATTRS = ("_fold_key", "_sub_key", "_cat_key", "_nchw_key", "_stem_key", "_tm_key")
PACK_ATTRS = ("_pack", "_pq", "_pkv", "_po")
KINDS = set(CACHE_ATTRS) | set(PACK_ATTRS)


def _imagen():
    from minimagen_b200.Imagen import Imagen
    from minimagen_b200.Unet import Unet
    torch.manual_seed(0)
    im = Imagen(unets=Unet(**CFG), text_encoder_name="t5_base", image_sizes=(32,), timesteps=100, cond_drop_prob=0.1)
    return im.eval()


def _inputs():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 3, 32, 32, generator=g)
    t = torch.tensor([10, 70])
    te = torch.randn(2, 8, 768, generator=g)
    tm = torch.ones(2, 8, dtype=torch.bool)
    tm[1, 5:] = False
    return x, t, te, tm


def _cache_keys(unet):
    """{(module name, cache): key} of every weight cache the forwards so far have filled."""
    from minimagen_b200.layers import _PackCache
    keys = {}
    for name, m in unet.named_modules():
        for a in CACHE_ATTRS:
            if getattr(m, a, None) is not None:
                keys[name, a] = getattr(m, a)
        for a in PACK_ATTRS:
            c = getattr(m, a, None)
            if isinstance(c, _PackCache) and c._key is not None:
                keys[name, a] = c._key
    return keys


def _forward(unet, x, t, te, tm):
    with torch.no_grad():
        return unet(x, t, text_embeds=te, text_mask=tm)


def _graph_key(im, te, tm):
    return im._graph_key(im.unets[0], (2, 3, 32, 32), im.noise_schedulers[0], te, tm, None, None, 3.0)


@pytest.mark.parametrize("bump", [False, True], ids=["without_bump", "with_bump"])
def test_in_place_update_reaches_every_weight_cache(emu, bump):
    from minimagen_b200.Imagen import bump_versions
    from minimagen_b200.Unet import Unet
    im = _imagen()
    u = im.unets[0]
    x, t, te, tm = _inputs()
    u.register_static_text(te)
    _forward(u, x, t, te, tm)                                    # fills every cache
    before = _cache_keys(u)
    assert {a for _, a in before} == KINDS, f"caches not reached: {sorted(KINDS - {a for _, a in before})}"
    assert u._static_text_proj(te) is not None
    key0 = _graph_key(im, te, tm)

    # what a graph replay of a training step does: new values in place, the version counters untouched
    params = list(u.parameters())
    versions = [p._version for p in params]
    g = torch.Generator().manual_seed(2)
    for p in params:
        p.data.add_(0.05 * torch.randn(p.shape, generator=g))
    assert [p._version for p in params] == versions
    fresh = Unet(**CFG).eval()
    fresh.load_state_dict(u.state_dict())
    want = _forward(fresh, x, t, te, tm)

    if bump:
        bump_versions(params)
        assert all(p._version == v + 1 for p, v in zip(params, versions))
    stale_text = u._static_text_proj(te) is not None
    got = _forward(u, x, t, te, tm)
    after = _cache_keys(u)
    err = rel_l2(got, want)
    print(f"\n{'with' if bump else 'without'} bump_versions: forward vs a fresh U-Net rel-L2 {err:.3e}; "
          f"{sum(after[k] != before[k] for k in before)} of {len(before)} weight caches rebuilt")
    if bump:
        assert not stale_text and _graph_key(im, te, tm) != key0
        rebuilt = [k for k in before if after[k] != before[k]]
        assert len(rebuilt) == len(before), f"caches kept: {sorted(set(before) - set(rebuilt))}"
        assert torch.equal(got, want)
    else:
        # every cache hits: the forward mixes the packed old weights with the fp32 layers' new ones
        assert stale_text and _graph_key(im, te, tm) == key0 and after == before
        assert err > 0.1
