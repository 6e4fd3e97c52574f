"""The U-Net lowering as a pure DATAFLOW: the product's own host code (minimagen_b200/{layers,Unet,autograd,train_path}.py)
run in float64 on an ops backend that never rounds, against a float64 run of the reference restatement.

Which tensor, channel offset, row pitch, statistics buffer, packed weight and folded scale every launch receives does not
depend on precision.  With every dtype widened to float64 (`exact` fixture: the host modules' dtype constants, `unet.double()`,
`EmuOps(lo=float64, hi=float64)`) the only differences left between the lowering and the restatement are float64
re-associations, so the two must agree per element to

    |out - ref| <= TOL * (1 + max|ref|),   TOL = 1e-12     (measured: 1e-15 .. 4e-15; each test prints its worst ratio)

-- six orders of magnitude below the fp16 operand-rounding floor (~1e-3 rel-L2) at which tests/test_host_logic.py and
tests/test_gpu_unet.py have to stop.  The arithmetic error of each kernel is bounded kernel by kernel elsewhere
(tests/test_gpu_*_ops.py, test_gpu_image_*.py; per call of a real forward in tests/test_gpu_lowering_calls.py).

Every buffer the host code allocates with torch.empty / empty_like is born full of NaN here (`_PoisonedTorch`), so an element
no launch wrote reaches the comparison as NaN instead of as whatever a warm allocator handed back.  (The poison sits at the
allocation, not inside the backend: several outputs are windows into a buffer other launches fill -- sub-pixel phases, the
stem's channel slices, token rows -- so a backend-side fill would be either vacuous or destructive.)

`test_planted_defect_*` plant one lowering defect each by wrapping one host helper or backend method; each must FAIL the exact
bound, and prints the rel-L2 it would have been judged by.  Measured on the random-init sr_d128 network: a GroupNorm
statistic taken from a copy that went through fp16 moves the output by 4.6e-7 rel-L2 (invisible at 3e-3, 2.7e5 x over the
exact bound), the doubled null-kv gradient leaves the all-gradient rel-L2 at 4.0e-4 (limit 5e-3); the other defects move this
network's output by 2e-2 .. 2e-1, so rel-L2 sees them here too -- they stay as proof that the bound does.
"""
import contextlib
import math
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2
from emu_ops import EmuOps
from oracle import restatement as R

F64 = torch.float64
TOL = 1e-12
REL_L2_LIMIT = 3e-3          # what test_host_logic.test_unet_forward_tensor_core_shaped_configs asserts


class _PoisonedTorch:
    """Stands for the `torch` module inside the host modules: buffers from empty / empty_like are NaN-filled."""

    def __getattr__(self, name):
        return getattr(torch, name)

    @staticmethod
    def _poison(t):
        return t.fill_(math.nan) if t.is_floating_point() else t

    def empty(self, *a, **k):
        return self._poison(torch.empty(*a, **k))

    def empty_like(self, *a, **k):
        return self._poison(torch.empty_like(*a, **k))


def _mods():
    import minimagen_b200.Unet, minimagen_b200.autograd, minimagen_b200.layers, minimagen_b200.train_path   # noqa: F401,E401
    m = sys.modules
    return (m["minimagen_b200.layers"], m["minimagen_b200.Unet"], m["minimagen_b200.autograd"],
            m["minimagen_b200.train_path"])


@pytest.fixture
def exact(monkeypatch):
    """float64 host code on the no-rounding backend; everything is restored afterwards."""
    import minimagen_b200.ops as ops_mod
    layers, unet_mod, autograd, train_path = _mods()
    for mod, names in ((layers, ("F16", "F32")), (unet_mod, ("F32",)), (autograd, ("F16", "F32")), (train_path, ("F32",))):
        for n in names:
            monkeypatch.setattr(mod, n, F64)
        monkeypatch.setattr(mod, "torch", _PoisonedTorch())
    e = EmuOps(lo=F64, hi=F64)
    prev = ops_mod._OPS
    ops_mod.set_ops(e)
    yield e
    ops_mod.set_ops(prev)


# ------------------------------------------------------------------------------------------------ networks and inputs
SR_D64 = dict(dim=64, dim_mults=(1, 2, 4), num_resnet_blocks=(1, 2, 2), layer_attns=(False, False, True),
              layer_cross_attns=(False, True, True), lowres_cond=True, memory_efficient=True)
BASE_D64 = dict(dim=64, dim_mults=(1, 2), attend_at_middle=True, text_embed_dim=768)
CFGS = {
    # the two of test_host_logic.test_unet_forward_tensor_core_shaped_configs, and test_gpu_unet's unet_default_d128 at 32x32
    "base_d64_mid_attn": (BASE_D64, 32, 2),
    "sr_d64": (SR_D64, 64, 2),                     # memory_efficient halves first: 32 / 16 / 8 pixel levels
    "unet_default_d128": (dict(text_embed_dim=768), 32, 2),
    # C_out = 128 / 256 / 512 blocks: two-source folded res_conv, stem, NCHW final conv, both Downsample placements
    "sr_d128": (dict(dim=128, dim_mults=(1, 2, 4), num_resnet_blocks=(1, 2, 1), layer_attns=(False, True, True),
                     layer_cross_attns=(False, True, True), lowres_cond=True, memory_efficient=True), 64, 2),
    "base_d128_lowres": (dict(dim=128, dim_mults=(1, 2, 4), layer_attns=(False, False, True),
                              layer_cross_attns=(True, False, True), lowres_cond=True, memory_efficient=False), 32, 2),
    # 40/20/10 pixels: no tensor-core conv geometry -> the direct-conv route
    "ragged_40x40_d64": (dict(dim=64, dim_mults=(1, 2, 4), layer_attns=(False, True, True),
                              layer_cross_attns=(False, True, True), text_embed_dim=768), 40, 3),
}


def _unet(cfg, seed=0):
    """A float64 U-Net whose norm gains / biases are not the 1 / 0 of a fresh init (a swapped or dropped one must show)."""
    from minimagen_b200.Unet import Unet
    torch.manual_seed(seed)
    u = Unet(**cfg).eval().double()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for p in u.parameters():
            if p.dim() == 1 or p.shape[0] == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=g, dtype=F64))
    return u, {k: v.detach().clone() for k, v in u.state_dict().items()}


def _inputs(cfg, s, b, seed=3, L=20, mask="ragged"):
    g = torch.Generator().manual_seed(seed)
    r = lambda *sh: torch.randn(*sh, generator=g, dtype=F64)
    x = r(b, 3, s, s)
    kw = dict(text_embeds=r(b, L, cfg.get("text_embed_dim", 512)))
    if mask == "ragged":
        tm = torch.ones(b, L, dtype=torch.bool)
        tm[-1, 5:] = False
        tm[0, L // 2] = False
        kw["text_mask"] = tm
    if cfg.get("lowres_cond"):
        kw.update(lowres_cond_img=r(b, 3, s, s), lowres_noise_times=torch.tensor([200, 3, 77][:b]))
    return x, torch.tensor([999, 0, 500][:b]), kw


def _ratio(out, ref):
    """max |out - ref| / (TOL * (1 + max|ref|)); an unwritten (NaN) element is infinitely wrong"""
    assert out.shape == ref.shape and out.dtype == F64 and ref.dtype == F64
    d = (out - ref).abs()
    if not torch.isfinite(d).all():
        return math.inf
    return float(d.max() / (TOL * (1 + ref.abs().max())))


def _exact(out, ref, what):
    r = _ratio(out, ref)
    print(f"{what}: worst |out - ref| / (1e-12 (1 + max|ref|)) = {r:.3e}")
    assert r <= 1, f"{what}: lowering differs from the float64 restatement ({r:.3e} x the bound)"


class CountingArena:
    """layers.ZeroArena that counts what it handed out and what it had to refuse."""

    def __new__(cls, device, n):
        layers = _mods()[0]

        class _A(layers.ZeroArena):
            hits = misses = 0

            def take(self, shape):
                t = super().take(shape)
                if t is None:
                    self.misses += 1
                else:
                    self.hits += 1
                    assert not t.any(), "the arena handed out an accumulator that is not zero"
                return t
        return _A(device, n)


@contextlib.contextmanager
def _arena(n_doubles, make=CountingArena):
    """Unet._forward_body installs the arena for CUDA inputs only: install it here the same way for the CPU run."""
    layers, unet_mod = _mods()[:2]
    made = []
    orig = unet_mod.Unet._forward_body_impl

    def impl(self, x, *a):
        layers._ARENA = make(x.device, n_doubles)
        made.append(layers._ARENA)
        return orig(self, x, *a)                      # _forward_body's `finally` removes the arena
    unet_mod.Unet._forward_body_impl = impl
    try:
        yield made
    finally:
        unet_mod.Unet._forward_body_impl = orig
        layers._ARENA = None


BIG = 1 << 18


def _modes(emu):
    return {e[0] for e in emu.conv_log}


# ------------------------------------------------------------------------------------------------ every config, default switches
@pytest.mark.parametrize("name", list(CFGS))
def test_configs_exact(exact, name):
    cfg, s, b = CFGS[name]
    u, sd = _unet(cfg)
    x, t, kw = _inputs(cfg, s, b)
    with torch.no_grad(), _arena(BIG) as arenas:
        out = u(x, t, **kw)
        null = u(x, t, cond_drop_prob=1., **kw)
        ref, ref_null = R.unet_forward(sd, cfg, x, t, **kw), R.unet_forward(sd, cfg, x, t, cond_drop_prob=1., **kw)
    assert all(a.hits > 0 and a.misses == 0 for a in arenas) and len(arenas) == 2
    calls, log = exact.calls, exact.conv_log
    dim = cfg.get("dim", 128)
    if name.startswith("ragged"):
        assert "conv_direct" in calls and "nchw_to_nhwc" in calls and not any(e[1:3] == (3, 3) for e in log)
    else:
        # no case may fall to the fp32 route unnoticed: stem, sub-pixel upsample, in-place Downsample, NCHW final conv
        assert "conv_direct" not in calls and "stem_unroll" in calls and (0, 15, 1, 128, dim) in log
        assert (0, 3, 3, dim, 16) in log and {2, 3, 4, 5} <= _modes(exact) and 1 not in _modes(exact)
        assert (6 in _modes(exact)) == (len(cfg.get("dim_mults", (1, 2, 4))) > 1)
        assert "attention" in calls and "gn_stats" in calls
    if dim == 128:
        fold = [e for e in log if e[0] == "res1x1"]
        assert {e[4] for e in fold} >= {128, 256} and all(e[1] for e in fold)          # only up blocks have a res_conv: always two sources
        assert {e[4] for e in log if e[1:3] == (3, 3)} >= {128, 256, 512}
    _exact(out, ref, f"{name} conditional")
    _exact(null, ref_null, f"{name} cond_drop_prob=1")


def test_arena_too_small_falls_back_part_way(exact):
    cfg, s, b = CFGS["sr_d64"]
    u, sd = _unet(cfg)
    x, t, kw = _inputs(cfg, s, b)
    with torch.no_grad():
        ref = R.unet_forward(sd, cfg, x, t, **kw)
        with _arena(600) as arenas:
            out = u(x, t, **kw)
        assert arenas[0].hits > 0 and arenas[0].misses > 0
        _exact(out, ref, "sr_d64, arena of 600 doubles")
        _exact(u(x, t, **kw), ref, "sr_d64, no arena")


# ------------------------------------------------------------------------------------------------ conditioning variants
def test_conditioning_variants_exact(exact):
    cfg, s, b = CFGS["sr_d64"]
    u, sd = _unet(cfg)
    with torch.no_grad(), _arena(BIG):
        x, t, kw = _inputs(cfg, s, b, mask=None)
        _exact(u(x, t, **kw), R.unet_forward(sd, cfg, x, t, **kw), "text_mask=None")
        x, t, kw = _inputs(cfg, s, b, L=300)                     # longer than max_text_len = 256: truncated
        assert kw["text_embeds"].shape[1] > u.max_text_len
        cut = dict(kw, text_mask=kw["text_mask"][:, :u.max_text_len])        # the restatement takes the mask already cut
        _exact(u(x, t, **kw), R.unet_forward(sd, cfg, x, t, **cut), "300 text tokens")
        x, t, kw = _inputs(cfg, s, b)
        nt = {k: v for k, v in kw.items() if not k.startswith("text_")}
        _exact(u(x, t, **nt), R.unet_forward(sd, cfg, x, t, **nt), "no text")
        cond, null = R.unet_forward(sd, cfg, x, t, **kw), R.unet_forward(sd, cfg, x, t, cond_drop_prob=1., **kw)
        _exact(u.forward_with_cond_scale(x, t, cond_scale=3., **kw), R.cfg_combine(cond, null, 3.), "forward_with_cond_scale(3.)")
        # Imagen.cfg_batched: the conditional and the unconditional pass as one 2B batch with a per-sample keep mask
        two = lambda v: torch.cat((v, v))
        keep = torch.cat((torch.ones(b, dtype=torch.uint8), torch.zeros(b, dtype=torch.uint8)))
        both = u._forward_impl(two(x), two(t), cond_keep=keep, **{k: two(v) for k, v in kw.items()})
        _exact(both, torch.cat((cond, null)), "cfg_batched (2B batch, cond_keep)")


def test_static_text_hit_and_miss_exact(exact):
    cfg, s, b = CFGS["base_d64_mid_attn"]
    u, sd = _unet(cfg)
    x, t, kw = _inputs(cfg, s, b)
    te = kw["text_embeds"]
    with torch.no_grad():
        u(x, t, **kw)
        n_lin = exact.calls.count("linear_f32")
        u.register_static_text(te)
        exact.calls.clear()
        _exact(u(x, t, **kw), R.unet_forward(sd, cfg, x, t, **kw), "static text: hit")
        assert exact.calls.count("linear_f32") == n_lin - 1
        te.mul_(0.5)                                              # changed without re-registering: must miss, not go stale
        exact.calls.clear()
        _exact(u(x, t, **kw), R.unet_forward(sd, cfg, x, t, **kw), "static text: miss")
        assert exact.calls.count("linear_f32") == n_lin


# ------------------------------------------------------------------------------------------------ the switch matrix
def _routes(emu):
    c = emu.calls
    return dict(conv_gn=c.count("conv_gn"), res1x1=c.count("conv_res1x1"), apply=c.count("gn_apply_silu"),
                cast=c.count("cast_act"), modes=_modes(emu) - {"res1x1"})


@pytest.fixture
def switch_net(exact):
    # 256 channels at 32x32 and 128 at 64x64: every FUSE_GN_CONV class has a layer the fused kernel's geometry accepts
    cfg, s, b = dict(dim=128, dim_mults=(2, 4), num_resnet_blocks=1, layer_attns=(False, True), layer_cross_attns=(False, True),
                     lowres_cond=True, memory_efficient=True), 64, 2
    u, sd = _unet(cfg)
    x, t, kw = _inputs(cfg, s, b)
    with torch.no_grad():
        ref = R.unet_forward(sd, cfg, x, t, **kw)

    def run(what, **switches):
        layers = _mods()[0]
        prev = {k: getattr(layers, k) for k in switches}
        for k, v in switches.items():
            setattr(layers, k, v)
        exact.calls.clear(), exact.conv_log.clear()
        try:
            with torch.no_grad(), _arena(BIG):
                out = u(x, t, **kw)
        finally:
            for k, v in prev.items():
                setattr(layers, k, v)
        _exact(out, ref, what)
        return _routes(exact)
    return run


def test_fold_and_fuse_switch_matrix_exact(switch_net):
    r = {}
    for fold in (True, False):
        for fuse in (False, True, 'pair', 'all'):
            for over in (True, False):
                r[fold, fuse, over] = switch_net(f"FOLD_RES_CONV={fold} FUSE_GN_CONV={fuse} FUSE_OVER_FOLD={over}",
                                                 FOLD_RES_CONV=fold, FUSE_GN_CONV=fuse, FUSE_OVER_FOLD=over)
    base = r[True, False, True]
    assert base["conv_gn"] == 0 and base["res1x1"] > 0
    for over in (True, False):
        assert r[False, False, over]["res1x1"] == 0 and r[False, False, over] == r[False, False, not over]
        assert r[True, False, over] == base                          # nothing to prefer over the fold while nothing is fused
        for fold in (True, False):
            n = [r[fold, f, over]["conv_gn"] for f in (False, 'pair', True, 'all')]
            assert n[0] == 0 < n[1] < n[2] <= n[3], n                # 'pair' < True (adds C_out = 128) <= 'all'
            assert r[fold, 'all', over]["apply"] < r[fold, False, over]["apply"]
        # a fused block2 displaces the fold only when FUSE_OVER_FOLD says so
        assert r[True, 'all', True]["res1x1"] < r[True, 'all', False]["res1x1"] == base["res1x1"]
        assert r[True, 'all', False]["conv_gn"] < r[True, 'all', True]["conv_gn"]
        assert r[False, 'all', over]["res1x1"] == 0


def test_remaining_switches_exact(switch_net):
    base = switch_net("defaults")
    assert {2, 3, 4, 5, 6} <= base["modes"] and 1 not in base["modes"]
    r = switch_net("SUBPIXEL_UPSAMPLE=False", SUBPIXEL_UPSAMPLE=False)
    assert not ({2, 3, 4, 5} & r["modes"]) and r["cast"] > base["cast"]          # nearest-x2 materialised by cast_act
    r = switch_net("INPLACE_DOWNSAMPLE=False", INPLACE_DOWNSAMPLE=False)
    assert 1 in r["modes"] and 6 not in r["modes"] and r["cast"] > base["cast"]  # four-phase split operand
    r = switch_net("GN_INPUT_F32=False", GN_INPUT_F32=False)
    assert r != base                                                             # fp16-only conv outputs: other casts
    r = switch_net("all three off, fused", SUBPIXEL_UPSAMPLE=False, INPLACE_DOWNSAMPLE=False, GN_INPUT_F32=False,
                   FUSE_GN_CONV='all')
    assert r["conv_gn"] > 0 and 1 in r["modes"]


# ------------------------------------------------------------------------------------------------ training path
@pytest.fixture
def exact_train(exact, monkeypatch):
    monkeypatch.setattr(_mods()[2], "ROUTE_TC_ON_CPU", True)
    return exact


def _train_case(name, plant=None):
    """MSE loss and every parameter gradient of unet_forward_train, and of torch autograd through the float64 restatement."""
    cfg, s, b = CFGS[name]
    u, _ = _unet(cfg)
    u.train()
    x, t, kw = _inputs(cfg, s, b, L=12)
    target = torch.randn(x.shape, generator=torch.Generator().manual_seed(9), dtype=F64)
    loss = F.mse_loss(u(x, t, **kw), target)
    loss.backward()
    mine = {k: p.grad.detach().clone() for k, p in u.named_parameters()}
    sd = {k: v.detach().clone().requires_grad_(k in mine) for k, v in u.state_dict().items()}
    ref_loss = F.mse_loss(R.unet_forward(sd, cfg, x, t, **kw), target)
    ref_loss.backward()
    assert all(sd[k].grad is not None for k in mine)
    return loss.detach(), ref_loss.detach(), mine, {k: sd[k].grad for k in mine}


@pytest.mark.parametrize("name", ["sr_d64", "base_d64_mid_attn"])
def test_training_loss_and_every_gradient_exact(exact_train, name):
    loss, ref_loss, mine, ref = _train_case(name)
    calls, log = exact_train.calls, exact_train.conv_log
    # the tensor-core routes were walked: weight gradient on wgmma, data gradient through the forward conv kernel (flipped
    # packed weight), Downsample data gradient as four sub-pixel phases of dy
    assert "conv_wgrad_tc" in calls and calls.count("conv_igemm") > 2 * calls.count("conv_dgrad")
    assert {m for m, kh, kw, _, _ in log if (kh, kw) == (2, 2)} == {2, 3, 4, 5} and 6 in _modes(exact_train)
    _exact(loss.reshape(1), ref_loss.reshape(1), f"{name} loss")
    worst = max((_ratio(mine[k], ref[k]), k) for k in mine)
    print(f"{name}: {len(mine)} parameter gradients, worst |g - ref| / (1e-12 (1 + max|ref|)) = {worst[0]:.3e} at {worst[1]}")
    assert worst[0] <= 1, worst


def _flat_rel_l2(mine, ref):
    return rel_l2(torch.cat([mine[k].reshape(-1) for k in mine]), torch.cat([ref[k].reshape(-1) for k in mine]))


def test_planted_defect_training(exact_train, monkeypatch):
    """(a) the null key/value gradient of the multi-query attention summed over the heads twice; (b) the bias gradient of one
    conv skipped (its buffer left at zero).  Judged as tests/test_training.py judges: one rel-L2 < 5e-3 over all gradients."""
    autograd = _mods()[2]
    orig = autograd.AttentionFn.backward

    def twice(ctx, do):
        dq, dk, dv, dnull, _ = orig(ctx, do)
        return dq, dk, dv, dnull * (ctx.cfg[0] if ctx.cfg[1] == 1 else 1), None
    with monkeypatch.context() as m:
        m.setattr(autograd.AttentionFn, "backward", staticmethod(twice))
        _, _, mine, ref = _train_case("base_d64_mid_attn")
    bad = {k for k in mine if _ratio(mine[k], ref[k]) > 1}
    print(f"planted: dnull summed over heads twice -> {sorted(bad)} fail the exact bound; all-gradient rel-L2 "
          f"{_flat_rel_l2(mine, ref):.3e} (limit 5e-3)")
    assert "mid_attn.fn.fn.null_kv" in bad and all(k.endswith("attn.fn.null_kv") or k == "mid_attn.fn.fn.null_kv" for k in bad)
    assert _flat_rel_l2(mine, ref) < 5e-3

    colsum, n = exact_train.colsum, [0]

    def skip(x, M, Nc, out, accumulate=False):
        n[0] += 1
        return out.zero_() if n[0] == 7 else colsum(x, M, Nc, out, accumulate)
    with monkeypatch.context() as m:
        m.setattr(exact_train, "colsum", skip)
        _, _, mine, ref = _train_case("base_d64_mid_attn")
    bad = {k for k in mine if _ratio(mine[k], ref[k]) > 1}
    print(f"planted: one bias gradient skipped -> {sorted(bad)} fail the exact bound; all-gradient rel-L2 "
          f"{_flat_rel_l2(mine, ref):.3e} (limit 5e-3)")
    assert len(bad) == 1 and bad.pop().endswith(".bias")


# ------------------------------------------------------------------------------------------------ planted lowering defects
def _plant_fold_scale(mp, emu, u):
    """skip scale missing from the folded res_conv weight columns only (Conv2d._pack_cat and the GroupNorm path keep it)"""
    layers = _mods()[0]
    orig = layers.Conv2d._pack_fold
    mp.setattr(layers.Conv2d, "_pack_fold", lambda self, rc, c0, scale: orig(self, rc, c0, 1.0))


def _plant_ss_pitch(mp, emu, u):
    """scale_shift row pitch of the last ResnetBlock one block short: image 1 reads its neighbour's columns"""
    unet_mod = _mods()[1]
    orig = unet_mod.Unet._all_scale_shifts

    def f(self, t):
        ss = orig(self, t)
        v = ss[self.final_res_block]
        ss[self.final_res_block] = v.as_strided(v.shape, (v.stride(0) - v.shape[1], 1), v.storage_offset())
        return ss
    mp.setattr(unet_mod.Unet, "_all_scale_shifts", f)


def _plant_v_offset(mp, emu, u):
    """the column offset of the V view ignored on one attention call (the host passes c_off = 0 to every conv, so the one
    operand offset it does compute is this one): V reads the K columns"""
    orig, n = emu.attention, [0]

    def f(q, q_bs, ldq, k, v, *a):
        n[0] += 1
        return orig(q, q_bs, ldq, k, k if n[0] == 2 else v, *a)
    mp.setattr(emu, "attention", f)


def _plant_phase_swap(mp, emu, u):
    """sub-pixel phases (0,1) and (1,0) of the first Upsample swapped: each writes its own pixels from the other's taps"""
    orig, n = emu.conv_igemm, [0]

    def f(act, B, H, W, lda, c_off, c_in, wp, c_out, kh, kw, mode, *a, **k):
        if mode in (3, 4) and n[0] < 2:
            n[0] += 1
            mode = 7 - mode
        return orig(act, B, H, W, lda, c_off, c_in, wp, c_out, kh, kw, mode, *a, **k)
    mp.setattr(emu, "conv_igemm", f)


def _plant_stale_stats(mp, emu, u):
    """Act.need_stats of one attention output computed from a copy that went through fp16 (a stale, rounded copy)"""
    layers = _mods()[0]
    orig, n = layers.Act.need_stats, [0]

    def f(self):
        if self.stats is None:
            n[0] += 1
            if n[0] == 2:
                B, H, W, C = self.shape
                self.stats = layers.stats_zeros((B, C // layers.STATS_BLOCK, 2), self.device)
                emu.gn_stats(self.any.half().double(), C, None, 0, 1.0, B, H * W, C // layers.STATS_BLOCK, self.stats)
        return orig(self)
    mp.setattr(layers.Act, "need_stats", f)


def _plant_nchw_channel(mp, emu, u):
    """the last real channel of the NCHW final conv never stored"""
    orig = emu.conv_igemm

    def f(*a, **k):
        if k.get("n_valid"):
            k["n_valid"] -= 1
        return orig(*a, **k)
    mp.setattr(emu, "conv_igemm", f)


class _ShortArena:
    """ZeroArena whose take advances by n - 2: consecutive accumulators share two entries"""

    def __new__(cls, device, n):
        layers = _mods()[0]

        class _A(layers.ZeroArena):
            def take(self, shape):
                t = super().take(shape)
                self.off -= 2
                return t
        return _A(device, n)


@pytest.mark.parametrize("plant", [_plant_fold_scale, _plant_ss_pitch, _ShortArena, _plant_v_offset, _plant_phase_swap,
                                   _plant_stale_stats, _plant_nchw_channel], ids=lambda p: p.__name__.strip("_"))
def test_planted_defect_fails_exact_bound(exact, monkeypatch, plant):
    """Each defect must fail the exact bound; the rel-L2 the 3e-3 tests would have judged it by is printed beside it (what
    the fp16-mode run adds to that figure is its own ~1e-3 of operand rounding)."""
    cfg, s, b = CFGS["sr_d128"]
    u, sd = _unet(cfg)
    x, t, kw = _inputs(cfg, s, b)
    with torch.no_grad():
        ref = R.unet_forward(sd, cfg, x, t, **kw)
        if plant is _ShortArena:
            with _arena(BIG, make=_ShortArena):
                out = u(x, t, **kw)
        else:
            plant(monkeypatch, exact, u)
            with _arena(BIG):
                out = u(x, t, **kw)
    ratio, rl = _ratio(out, ref), rel_l2(torch.nan_to_num(out), ref)
    verdict = "would PASS" if rl < REL_L2_LIMIT else "would also fail"
    print(f"planted {plant.__name__.strip('_')}: exact bound exceeded {ratio:.3e} x; rel-L2 {rl:.3e} {verdict} the "
          f"{REL_L2_LIMIT:g} limit" + (" (unwritten elements counted as 0)" if math.isinf(ratio) else ""))
    assert ratio > 1
