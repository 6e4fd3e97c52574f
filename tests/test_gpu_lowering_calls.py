"""Every kernel call of a real U-Net forward against float64, at the arguments the network actually passes.

The kernel tests (test_gpu_image_fwd.py, test_gpu_token_ops.py, test_gpu_sampler_ops.py) chose their shapes by hand; here the
shapes, channel offsets, row pitches, strides, n_valid and statistics buffers come from the lowering itself.  `CheckingOps`
wraps the native backend: for each call it NaN-fills the pure outputs, makes the call, synchronises, and checks the outputs
against the float64 reference of tests/fp64_ref.py built from THAT call's own arguments, with that reference's per-element
bound.  The inputs of every call are the native run's own tensors, so no error compounds from one call to the next: together
with tests/test_lowering_exact.py (the dataflow is exact) this replaces the whole-network rel-L2 < 2e-3 as the sharp check.

  * epilogue / gn_stats statistics are checked as the INCREMENT of the accumulator over the call;
  * completeness: the methods a forward called minus the methods checked must be empty apart from `ALLOWED` (capability
    queries), so a kernel added later cannot slip through unchecked;
  * every statistics accumulator is zero when first handed to a kernel and no two overlap (the ZeroArena carving).

The float64 references are computed on the GPU (the operands' device).  The batch_streams = 2 case is a dataflow check of the
batch chunking (slices of the conditioning, of the scale/shift rows and of the output), not of concurrency: the proxy
synchronises after every call.  Nothing here is repeated or stressed: each case is one ordinary forward.
"""
import contextlib
import io
import time

import pytest
import torch

import fp64_ref as R

pytestmark = pytest.mark.gpu

F16, F32, F64 = torch.float16, torch.float32, torch.float64
ALLOWED = {"igemm_supported", "conv_res1x1_supported", "conv_gn_supported"}      # capability queries: no kernel runs
NAN = float("nan")


def _strided(t, shape, strides):
    return t.as_strided(shape, strides, t.storage_offset())


def _describe(args, kwargs):
    d = lambda v: f"{str(v.dtype).replace('torch.', '')}{list(v.shape)}/{list(v.stride())}" if torch.is_tensor(v) else repr(v)
    return ", ".join([d(a) for a in args] + [f"{k}={d(v)}" for k, v in kwargs.items()])


class CheckingOps:
    def __init__(self, inner):
        self.inner = inner
        self.called, self.checked = set(), set()
        self.family = {}                       # method -> [calls, worst |err| / bound]
        self.accumulators = {}                 # data_ptr -> numel of every statistics accumulator seen

    def __getattr__(self, name):
        target = getattr(self.inner, name)
        if not callable(target):
            return target
        checker = getattr(self, "_check_" + name, None)

        def call(*args, **kwargs):
            self.called.add(name)
            if checker is None:
                return target(*args, **kwargs)
            try:
                with contextlib.redirect_stdout(io.StringIO()):          # R.check prints every comparison: keep the worst only
                    gen = checker(*args, **kwargs)
                    next(gen)                                            # prefill / snapshots
                    ret = target(*args, **kwargs)
                    self._sync()
                    try:
                        gen.send(ret)                                    # comparisons
                    except StopIteration:
                        pass
            except AssertionError as e:
                raise AssertionError(f"{name}({_describe(args, kwargs)}): {e}") from None
            self.checked.add(name)
            return ret
        return call

    def _sync(self):
        if torch.cuda.is_available():
            torch.cuda.synchronize()

    def _note(self, name, ratio):
        f = self.family.setdefault(name, [0, 0.0])
        f[1] = max(f[1], ratio)

    def _count(self, name):
        self.family.setdefault(name, [0, 0.0])[0] += 1

    def _accumulator(self, t):
        """A statistics accumulator about to be added into: zero the first time a kernel sees it."""
        if t.data_ptr() not in self.accumulators:
            self.accumulators[t.data_ptr()] = t.numel()
            assert not t.any(), "a statistics accumulator was handed to its first kernel non-zero"
        return t.clone()

    def assert_accumulators_disjoint(self):
        spans = sorted(self.accumulators.items())
        for (p0, n0), (p1, _) in zip(spans, spans[1:]):
            assert p0 + 8 * n0 <= p1, f"statistics accumulators overlap: {p0:#x}+{n0} doubles and {p1:#x}"
        return len(spans)

    def _stats_increment(self, name, acc, before, f, e, sb=16):
        """acc - before against the (sum, sum of squares) per (image, sb channels) of this call's output: `f` the fp32 values
        the kernel summed (its own fp32 output), or their reference with elementwise bound `e` when only fp16 was stored."""
        ref, bound = R.conv_stats_ref(f, sb)
        if e is not None:
            B, C = f.shape[0], f.shape[-1]
            blk = lambda t: t.reshape(B, -1, C // sb, sb).sum(dim=(1, 3))
            bound = bound + torch.stack((blk(e), blk(2 * f.abs() * e + e * e)), dim=-1)
        bound = bound + 4 * R.U64 * (before.abs() + acc.abs())             # the subtraction below
        self._count(name + " statistics")
        self._note(name + " statistics", R.check(acc - before, ref, bound, name + " statistics increment"))

    def _out(self, name, out32, out16, ref, bound):
        if out32 is not None:
            self._note(name, R.check(out32, ref, bound, name + " fp32 output"))
        if out16 is not None:
            self._note(name, R.check(out16, *R.half_out(ref, bound), name + " fp16 output"))

    # ---------------------------------------------------------------- convolutions
    def _check_conv_igemm(self, act, B, H, W, lda, c_off, c_in, wp, c_out, kh, kw, mode, bias, residual, out_f32, out_f16,
                          out_strides, block_n=0, out_sc=1, n_valid=0, act2=None, lda2=0, c_off2=0, c_in1=0, out_stats=None):
        self._count("conv_igemm")
        nv = n_valid if n_valid else c_out
        sb_, sh, sw = out_strides
        view = lambda t: None if t is None else _strided(t, (B, H, W, nv), (sb_, sh, sw, out_sc))
        o32, o16 = view(out_f32), view(out_f16)
        for o in (o32, o16):
            if o is not None:
                o.fill_(NAN)
        before = self._accumulator(out_stats) if out_stats is not None else None
        yield
        if mode == 6:
            a = act.reshape(B, 2 * H, 2 * W, lda)[..., c_off:c_off + c_in]
        else:
            P = 4 if mode == 1 else 1
            a = act.reshape(B, P, H, W, lda)[..., c_off:c_off + (c_in1 if act2 is not None else c_in)]
            if act2 is not None:
                a = torch.cat((a, act2.reshape(B, P, H, W, lda2)[..., c_off2:c_off2 + c_in - c_in1]), dim=-1)
            a = a if mode == 1 else a[:, 0]
        res = None if residual is None else _strided(residual, (B, H, W, c_out), (sb_, sh, sw, 1))
        ref, bound = R.conv_fwd_ref(a, wp, kh, kw, mode, bias, res)
        self._out("conv_igemm", o32, o16, ref[..., :nv], bound[..., :nv])
        if out_stats is not None:
            own = o32 is not None
            self._stats_increment("conv_igemm", out_stats, before, o32 if own else ref, None if own else bound)

    def _check_conv_res1x1(self, act, B, H, W, lda, c_in, act2, lda2, c_in1, x, ldx, x_cin, x2, ldx2, x_cin1, wp, c_out,
                           bias, residual, out_f32, out_f16, out_stats):
        self._count("conv_res1x1")
        for o in (out_f32, out_f16):
            if o is not None:
                o.fill_(NAN)
        before = self._accumulator(out_stats) if out_stats is not None else None
        yield
        cat2 = lambda t, ld, t2, ld2, c, c1: (
            t.reshape(B, H, W, ld)[..., :c] if t2 is None else
            torch.cat((t.reshape(B, H, W, ld)[..., :c1], t2.reshape(B, H, W, ld2)[..., :c - c1]), dim=-1))
        a, xs = cat2(act, lda, act2, lda2, c_in, c_in1), cat2(x, ldx, x2, ldx2, x_cin, x_cin1)
        res = None if residual is None else residual.reshape(B, H, W, c_out)
        ref, bound = R.conv_fwd_ref(a, wp, 3, 3, 0, bias, res, x=xs)
        rs = lambda t: None if t is None else t.reshape(B, H, W, c_out)
        self._out("conv_res1x1", rs(out_f32), rs(out_f16), ref, bound)
        if out_stats is not None:
            own = out_f32 is not None
            self._stats_increment("conv_res1x1", out_stats, before, rs(out_f32) if own else ref, None if own else bound)

    def _check_conv_gn(self, src0, c0, src1, c1, scale1, B, H, W, groups, stats0, stats1, gamma, beta, scale_shift, ss_ld,
                       eps, wp, c_out, bias, residual, out_f32, out_f16, out_stats):
        self._count("conv_gn")
        for o in (out_f32, out_f16):
            if o is not None:
                o.fill_(NAN)
        before = self._accumulator(out_stats) if out_stats is not None else None
        yield
        C = c0 + c1
        sums = R.group_sums(stats0, c0, groups, stats1, c1, scale1)
        ss = None if scale_shift is None else _strided(scale_shift, (B, 2 * C), (ss_ld, 1))
        rs = lambda t, c: None if t is None else t.reshape(B, H, W, c)
        ref, bound = R.conv_gn_ref(rs(src0, c0), groups, gamma, beta, ss, eps, sums, wp, bias, rs(residual, c_out),
                                   rs(src1, c1) if c1 else None, scale1)
        self._out("conv_gn", rs(out_f32, c_out), rs(out_f16, c_out), ref, bound)
        if out_stats is not None:
            own = out_f32 is not None
            self._stats_increment("conv_gn", out_stats, before, rs(out_f32, c_out) if own else ref, None if own else bound)

    def _check_conv_direct(self, inp, B, Hin, Win, c_in, ldi, w, c_out, kh, kw, stride, pad, bias, residual, out, Hout, Wout,
                           out_strides):
        self._count("conv_direct")
        o = _strided(out, (B, Hout, Wout, c_out), out_strides)
        o.fill_(NAN)
        yield
        assert (stride, pad) in ((1, kh // 2), (2, 1)), "geometry outside the reference's two"
        a = inp.reshape(B, Hin, Win, ldi)[..., :c_in]
        wp = w.reshape(c_out, c_in, kh, kw).permute(0, 2, 3, 1).reshape(c_out, -1)
        res = None if residual is None else _strided(residual, (B, Hout, Wout, c_out), out_strides)
        ref, bound = R.conv_fwd_ref(a, wp, kh, kw, 0 if stride == 1 else 6, bias, res)
        self._out("conv_direct", o, None, ref, bound)

    def _check_pack_conv_weight(self, w, scale=1.0):
        self._count("pack_conv_weight")
        out = yield
        w4 = w if w.dim() == 4 else w[:, :, None, None]
        ref = (R._d(w4) * R._f32(scale)).permute(0, 2, 3, 1).reshape(w4.shape[0], -1)
        self._note("pack_conv_weight", R.check(out, *R.half_out(ref, R.U32 * ref.abs()), "packed weight"))

    # ---------------------------------------------------------------- normalisation / casts
    def _check_gn_stats(self, src0, c0, src1, c1, scale1, B, hw, groups, sums):
        self._count("gn_stats")
        before = self._accumulator(sums)
        yield
        ref, bound = R.gn_stats_ref(src0.reshape(B, hw, c0), groups, src1.reshape(B, hw, c1) if c1 else None, scale1)
        bound = bound + 4 * R.U64 * (before.abs() + sums.abs())
        self._note("gn_stats", R.check(sums - before, ref, bound, "gn_stats increment"))

    def _check_gn_apply_silu(self, src0, c0, src1, c1, scale1, B, hw, groups, stats0, sb0, stats1, sb1, gamma, beta,
                             scale_shift, ss_ld, eps, out):
        self._count("gn_apply_silu")
        out.fill_(NAN)
        yield
        C = c0 + c1
        assert sb0 == 0 or (sb0 == 16 and (not c1 or sb1 == 16))
        sums = stats0 if sb0 == 0 else R.group_sums(stats0, c0, groups, stats1 if c1 else None, c1, scale1, sb0)
        ss = None if scale_shift is None else _strided(scale_shift, (B, 2 * C), (ss_ld, 1))
        ref, bound = R.gn_apply_silu_ref(src0.reshape(B, hw, c0), groups, gamma, beta, ss, eps, sums,
                                         src1=src1.reshape(B, hw, c1) if c1 else None, scale1=scale1, out16=out.dtype == F16)
        self._note("gn_apply_silu", R.check(out.reshape(B, hw, C), ref, bound, "gn_apply_silu"))

    def _check_cast_act(self, src0, c0, src1, c1, scale1, B, H, W, mode, out):
        self._count("cast_act")
        C = c0 + c1
        n_out = B * H * W * C * (4 if mode == 1 else 1)
        o = out.reshape(-1)[:n_out]                                        # mode 0 writes the first B*H*W rows of `out`
        o.fill_(NAN)
        yield
        x = R.gn_concat(src0.reshape(B, H, W, c0), src1.reshape(B, H, W, c1) if c1 else None, scale1)
        if mode == 1:
            x = x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
        elif mode == 2:
            x = torch.stack([x[:, (p >> 1)::2, (p & 1)::2] for p in range(4)], dim=1)
        bound = R.U32 * x.abs() if c1 else torch.zeros_like(x)             # the fp32 product with the skip scale
        ref, bound = R.half_out(x, bound) if out.dtype == F16 else (x, bound)
        self._note("cast_act", R.check(o.reshape(x.shape), ref, bound, f"cast_act mode {mode}"))

    def _check_ln_rows(self, inp, rows, C, gamma, beta, eps, pre_gelu, residual, out_f32, out_f16):
        self._count("ln_rows")
        for o in (out_f32, out_f16):
            if o is not None:
                o.fill_(NAN)
        yield
        ref, bound = R.ln_ref(inp.reshape(rows, C), gamma.reshape(C), None if beta is None else beta.reshape(C), eps,
                              bool(pre_gelu), None if residual is None else residual.reshape(rows, C))
        rs = lambda t: None if t is None else t.reshape(rows, C)
        self._out("ln_rows", rs(out_f32), rs(out_f16), ref, bound)

    # ---------------------------------------------------------------- conditioning
    def _check_linear_f32(self, inp, M, K, W, bias, Nout, in_act, out_act, addend, out_f32, out_f16, out_scale=1.0):
        self._count("linear_f32")
        for o in (out_f32, out_f16):
            if o is not None:
                o.fill_(NAN)
        yield
        ref, bound = R.linear_ref(inp.reshape(M, K), W.reshape(Nout, K), bias, in_act, out_act,
                                  None if addend is None else addend.reshape(M, Nout), out_scale)
        rs = lambda t: None if t is None else t.reshape(M, Nout)
        self._out("linear_f32", rs(out_f32), rs(out_f16), ref, bound)

    def _check_silu(self, inp, out):
        self._count("silu")
        out.fill_(NAN)
        yield
        y = R._silu(R._d(inp))
        self._note("silu", R.check(out, y, 16 * R.U32 * y.abs() + R.ETA_SILU, "silu"))

    def _check_posemb(self, t, B, dim, out):
        self._count("posemb")
        out.fill_(NAN)
        yield
        self._note("posemb", R.check(out, *R.posemb_ref(t, dim), "posemb"))

    def _check_text_tokens(self, proj, B, L, D, mask, keep, null_embed, max_len, c_out, m, row_off, pooled):
        self._count("text_tokens")
        rows = c_out.reshape(B, m, D)[:, row_off:row_off + max_len]
        rows.fill_(NAN)
        pooled.fill_(NAN)
        yield
        Lc = min(L, max_len)
        tok = torch.zeros((B, max_len, D), dtype=F32, device=proj.device)
        tok[:, :Lc] = proj.reshape(B, L, D)[:, :Lc]
        cond = keep.bool()[:, None].expand(B, max_len).clone()
        if mask is not None:
            cond[:, :Lc] &= mask.bool()[:, :Lc]
            cond[:, Lc:] = False
        want = torch.where(cond[:, :, None], tok, null_embed.reshape(1, max_len, D))
        assert torch.equal(rows, want), "text_tokens: conditioning rows are a selection, they must be exact"
        self._note("text_tokens", R.check(pooled, *R.text_pool_ref(rows), "text_tokens pooled mean"))

    def _check_place_rows(self, src, B, r, D, dst, m, row_off):
        self._count("place_rows")
        rows = dst.reshape(B, m, D)[:, row_off:row_off + r]
        rows.fill_(NAN)
        yield
        assert torch.equal(rows, src.reshape(B, r, D)), "place_rows is a copy"
        self._note("place_rows", 0.0)

    def _check_select_rows(self, a, null_row, keep, addend, B, Nn, out):
        self._count("select_rows")
        out.fill_(NAN)
        yield
        y = torch.where(keep.bool()[:, None], a.reshape(B, Nn), null_row.reshape(1, Nn))
        if addend is not None:
            y = y + addend.reshape(B, Nn)                                   # one fp32 add: the same bits
        assert torch.equal(out.reshape(B, Nn), y), "select_rows: a selection and one fp32 add"
        self._note("select_rows", 0.0)

    def _check_nchw_to_nhwc(self, a, ca, b, cb, B, hw, c_pad, out):
        self._count("nchw_to_nhwc")
        out.fill_(NAN)
        yield
        want = torch.zeros((B, hw, c_pad), dtype=F32, device=a.device)
        want[:, :, :ca] = a.reshape(B, ca, hw).permute(0, 2, 1)
        if b is not None and cb:
            want[:, :, ca:ca + cb] = b.reshape(B, cb, hw).permute(0, 2, 1)
        assert torch.equal(out.reshape(B, hw, c_pad), want), "nchw_to_nhwc is a transposing copy with zero padding"
        self._note("nchw_to_nhwc", 0.0)

    def _check_stem_unroll(self, a, ca, b, cb, B, H, W, out):
        self._count("stem_unroll")
        out.fill_(NAN)
        yield
        x = a if b is None or cb == 0 else torch.cat((a, b), dim=1)
        xp = torch.nn.functional.pad(x, (7, 8))
        want = torch.zeros((B, H, W, 16, 8), dtype=F64, device=a.device)
        for j in range(15):
            want[:, :, :, j, :x.shape[1]] = xp[:, :, :, j:j + W].permute(0, 2, 3, 1)
        ref, bound = R.half_out(want.reshape(B, H, W, 128), torch.zeros((), dtype=F64, device=a.device))
        self._note("stem_unroll", R.check(out.reshape(B, H, W, 128), ref, bound, "stem_unroll"))

    # ---------------------------------------------------------------- attention
    def _check_attention(self, q, q_bs, ldq, k, v, kv_bs, ldkv, kv_hs, null_kv, mask, B, heads, n, m, out, o_bs, ldo):
        self._count("attention")
        o = _strided(out, (B, heads, n, 64), (o_bs, 64, ldo, 1))
        o.fill_(NAN)
        yield
        qv, kv, vv = R.attention_views(q, q_bs, ldq, k, v, kv_bs, ldkv, kv_hs, B, heads, n, m)
        ref, bound = R.attention_ref(qv, kv, vv, null_kv.detach().to(F16), mask)
        self._note("attention", R.check(o, ref, bound, "attention"))


# ------------------------------------------------------------------------------------------------ the cases
def _inputs(cfg, s, b, L=20, seed=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, 3, s, s, generator=g)
    tm = torch.ones(b, L, dtype=torch.bool)
    tm[-1, 5:] = False
    kw = dict(text_embeds=torch.randn(b, L, cfg.get("text_embed_dim", 512), generator=g), text_mask=tm)
    if cfg.get("lowres_cond"):
        kw.update(lowres_cond_img=torch.randn(b, 3, s, s, generator=g), lowres_noise_times=torch.full((b,), 200))
    t = torch.randint(0, 1000, (b,), generator=g)
    return x.cuda(), t.cuda(), {k: v.cuda() for k, v in kw.items()}


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


@pytest.mark.parametrize("name,cfg,s,b,opt", CASES, ids=[c[0] for c in CASES])
def test_every_call_of_a_forward(native, name, cfg, s, b, opt):
    import minimagen_b200.ops as ops_mod
    from minimagen_b200.Unet import Unet
    torch.manual_seed(0)
    u = Unet(**cfg).eval().cuda()
    x, t, kw = _inputs(cfg, s, b)
    proxy = CheckingOps(native)
    ops_mod.set_ops(proxy)                      # the `native` fixture restores the previous backend afterwards
    t0 = time.time()
    with torch.no_grad():
        if opt.get("cfg_batched"):               # Imagen.cfg_batched: conditional and unconditional pass as one 2B batch
            two = lambda v: torch.cat((v, v))
            keep = torch.cat((torch.ones(b, dtype=torch.uint8), torch.zeros(b, dtype=torch.uint8))).cuda()
            out = u._forward_impl(two(x), two(t), cond_keep=keep, **{k: two(v) for k, v in kw.items()})
        else:
            u.batch_streams = opt.get("batch_streams", 1)
            assert len(u._batch_chunks(b, True)) == u.batch_streams
            out = u(x, t, **kw)
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
