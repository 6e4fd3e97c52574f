"""TEST INFRASTRUCTURE ONLY: `FootprintOps`, a proxy around an ops backend that checks every kernel call writes nothing
but its outputs.

include/minimagen_b200.h: "the caller owns every buffer (inputs, outputs, workspaces); nothing is allocated or retained by
the library".  So the bytes an entry point may write follow from its arguments: its output views (`_writes_<method>`, one
per kernel-launching method of NativeOps, from the ops.py docstrings and the header) and the workspaces NativeOps allocates
for it.  For each call the proxy

  1. relocates the arguments: the tensor arguments are grouped by untyped storage, each distinct storage is copied into a
     fresh buffer between two guard bands, and every argument is rebuilt there as a view with its own shape, strides and
     offset (so aliasing -- `out` is `x_t`, k and v are views of one projection, the sub-pixel phases are offset views of
     one output -- and alignment, the guards being multiples of 512 bytes, are kept).  A guard is the larger of 64 KiB
     and one image's extent of the largest view the call writes in that storage, so a store for image B, the channels
     past n_valid or a row past H lands in it rather than in someone else's memory;
  2. routes the allocations the call makes through `minimagen_b200.ops.torch` (the workspaces, an s_out the caller did
     not pass, the packed weights pack_conv_weight* return) into guarded buffers too, for the duration of the call: a
     workspace is fully writable, its guards are not;
  3. makes the call, synchronises, and checks (a) every guard byte still holds GUARD_BYTE and (b) every byte of every
     relocated storage outside the call's write footprint is bitwise what it was (the original, untouched by the call, is
     the snapshot).  That covers the read-only inputs, the other channels of a concat buffer, the neighbouring accumulators
     of a ZeroArena and the rows outside [row_off, row_off + max_len);
  4. copies the storages back into the originals (the run continues on the kernel's own results) and frees the relocations.

A failure names the method, the argument and the region (the guard before, the guard after, or inside the storage outside
the footprint), the first offending byte as an index of the argument, and the number of stray bytes.  It composes inside
CheckingOps -- CheckingOps(FootprintOps(native)) -- which keeps CheckingOps' bookkeeping on the run's own pointers, and
works alone where float64 references would be too slow.  Eager runs only: relocation cannot be captured in a graph.
"""
import contextlib
import inspect
import time

import torch

from checking_ops import ALLOWED

GUARD_BYTE = 0xFF               # NaN as fp16, fp32 and fp64 alike: no kernel stores it by computing a value
GUARD_MIN = 64 << 10
ALIGN = 512


def _round(n, a=ALIGN):
    return -(-n // a) * a


def _view(t, shape, strides, off=0):
    """The strided view of `t` (relative to its own offset) a call may write; None for an absent tensor."""
    return None if t is None else t.as_strided(tuple(shape), tuple(strides), t.storage_offset() + off)


def _first(t, *shape):
    """The first prod(shape) elements of `t` from its data pointer, shaped `shape` (the leading dim the image's)."""
    if t is None:
        return None
    st, s = [], 1
    for d in reversed(shape):
        st.append(s)
        s *= d
    return _view(t, shape, st[::-1])


def _key(t):
    return (t.device, t.untyped_storage().data_ptr())


def _bytes(storage, device):
    return torch.empty(0, dtype=torch.uint8, device=device).set_(storage, 0, (storage.nbytes(),), (1,))


_INT = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def _index(t, byte):
    """The index of `t` at byte offset `byte` of its storage: greedy
    over the strides, largest first, leaving the outermost index unclamped (image B past the last, -1 before the first).
    Returns (index, exact) -- exact False when the byte falls between the argument's elements (a gap of its strides)."""
    es = t.element_size()
    e = byte // es - t.storage_offset()
    if t.dim() == 0:
        return [], e == 0
    dims = sorted(range(t.dim()), key=lambda d: -abs(t.stride(d)) if t.stride(d) else 0)
    idx, rem = [0] * t.dim(), e
    for j, d in enumerate(dims):
        s = t.stride(d)
        if s == 0:
            continue
        i = rem // s
        if j:
            i = max(0, min(t.shape[d] - 1, i))
        idx[d], rem = i, rem - i * s
    return idx, rem == 0


class _Buffer:
    """A guarded copy of one storage (or a guarded allocation): [guard | storage bytes, padded to 8 | guard]."""

    def __init__(self, nbytes, guard, device, src=None):
        self.nbytes, self.pad, self.g0 = nbytes, _round(nbytes, 8), guard
        self.buf = torch.empty(guard + self.pad + guard, dtype=torch.uint8, device=device)
        self.buf.fill_(GUARD_BYTE)
        self.mid = self.buf[guard:guard + nbytes]
        self.src = src
        if src is not None:
            self.mid.copy_(src)

    def rebuild(self, t):
        es = t.element_size()
        return self.buf.view(t.dtype).as_strided(t.shape, t.stride(), self.g0 // es + t.storage_offset())

    def guards(self):
        """[(region, first offending byte relative to the storage's start, count)] of the two guards."""
        out = []
        for region, g, lo in (("guard before", self.buf[:self.g0], -self.g0),
                              ("guard after", self.buf[self.g0 + self.nbytes:], self.nbytes)):
            bad = g.ne(GUARD_BYTE)
            n = int(bad.sum())
            if n:
                # the guard before: the byte nearest the storage; after: the first past its end
                i = int(bad.nonzero()[-1 if region == "guard before" else 0])
                out.append((region, lo + i, n))
        return out


class _GuardedTorch:
    """`torch` as minimagen_b200.ops sees it during one call: empty / full allocate guarded buffers."""

    def __init__(self, owner):
        self._owner = owner

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *size, dtype=None, device=None, **_):
        size = tuple(size[0]) if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)) else size
        dtype = dtype or torch.get_default_dtype()
        n = 1
        for d in size:
            n *= int(d)
        es = torch.empty((), dtype=dtype).element_size()
        b = _Buffer(n * es, GUARD_MIN, torch.device(device) if device is not None else torch.device("cpu"))
        self._owner._allocs.append(b)
        return b.buf.view(dtype)[b.g0 // es:b.g0 // es + n].view(size)

    def full(self, size, value, dtype=None, device=None, **_):
        t = self.empty(size, dtype=dtype, device=device)
        t.fill_(value)
        return t


class FootprintOps:
    def __init__(self, inner, strict=True):
        """strict=False: a failed check is recorded in `failures` and the run goes on; `raise_failures` raises the first."""
        self.inner = inner
        self.strict = strict
        self.failures = []
        self.called, self.checked = set(), set()
        self.family = {}                     # method -> calls
        self.relocated = 0                   # bytes copied into guarded buffers, over all calls
        self.calls = 0
        self.seconds = 0.0
        self._allocs = None

    def __getattr__(self, name):
        target = getattr(self.inner, name)
        if not callable(target):
            return target
        fp = getattr(self, "_writes_" + name, None)

        def call(*args, **kwargs):
            self.called.add(name)
            if fp is None:
                return target(*args, **kwargs)
            t0 = time.perf_counter()
            ret, msgs = self._call(name, target, fp, args, kwargs)
            self.seconds += time.perf_counter() - t0
            self.checked.add(name)
            self.calls += 1
            self.family[name] = self.family.get(name, 0) + 1
            for m in msgs:
                if self.strict:
                    raise AssertionError(m)
                self.failures.append(m)
            return ret
        return call

    def raise_failures(self):
        if self.failures:
            raise AssertionError(f"{len(self.failures)} stray writes, the first: {self.failures[0]}")

    def report(self):
        print(f"  footprint: {self.calls} calls of {len(self.checked)} methods, {self.relocated / 2 ** 30:.2f} GiB "
              f"relocated, {self.seconds:.1f} s in the checks")

    @staticmethod
    def _sync():
        if torch.cuda.is_available():
            torch.cuda.synchronize()

    def _call(self, name, target, fp, args, kwargs):
        import minimagen_b200.ops as ops_mod
        bound = inspect.signature(fp).bind(*args, **kwargs)
        bound.apply_defaults()
        named = [(n, v) for n, v in bound.arguments.items() if torch.is_tensor(v)]
        writes = [w for w in fp(*args, **kwargs) if w is not None]
        self._sync()                             # an input may come from another stream (batch_streams)
        # group by storage; a guard covers one image of the largest view written in it
        groups = {}
        for n, t in named:
            groups.setdefault(_key(t), [t.untyped_storage(), t.device, []])[2].append((n, t))
        guard = {k: GUARD_MIN for k in groups}
        masks = {}
        for v in writes:
            k = _key(v)
            es = v.element_size()
            ext = (1 + sum((d - 1) * abs(s) for d, s in zip(v.shape[1:], v.stride()[1:]))) if v.dim() > 1 else 1
            one = max(ext, abs(v.stride(0)) if v.dim() else 1) * es
            guard[k] = max(guard[k], _round(one))
            st, dev, _ = groups[k]
            if k not in masks:
                masks[k] = torch.zeros(_round(st.nbytes(), 8), dtype=torch.uint8, device=dev)
            masks[k].view(_INT[es]).as_strided(v.shape, v.stride(), v.storage_offset()).fill_(-1)
        bufs = {}
        with torch.no_grad():
            for k, (st, dev, _) in groups.items():
                bufs[k] = _Buffer(st.nbytes(), guard[k], dev, _bytes(st, dev))
                self.relocated += st.nbytes()
            new = {n: bufs[_key(t)].rebuild(t) for n, t in named}
            a = bound.arguments
            a.update(new)
            self._allocs = []
            saved = ops_mod.torch
            ops_mod.torch = _GuardedTorch(self)
            try:
                ret = target(*bound.args, **bound.kwargs)
                self._sync()
            finally:
                ops_mod.torch = saved
                allocs, self._allocs = self._allocs, None
            msgs = []
            for k, b in bufs.items():
                args_here = groups[k][2]
                for region, off, cnt in b.guards():
                    msgs.append(self._msg(name, args_here, region, off, cnt))
                bad = b.mid.ne(b.src)
                if k in masks:
                    bad &= masks[k][:b.nbytes].eq(0)
                cnt = int(bad.sum())
                if cnt:
                    off = int(bad.to(torch.uint8).argmax())
                    msgs.append(self._msg(name, args_here, "storage outside the footprint", off, cnt))
                b.src.copy_(b.mid)                   # the run goes on with the call's own results
            for b in allocs:
                for region, off, cnt in b.guards():
                    msgs.append(f"{name}: {cnt} stray bytes in the {region} of the {b.nbytes}-byte workspace it "
                                f"allocated, the first at byte {off:+d}")
            if torch.is_tensor(ret) and any(ret.untyped_storage().data_ptr() == b.buf.untyped_storage().data_ptr()
                                            for b in allocs):
                ret = ret.clone()
        del bufs, masks, allocs
        return ret, msgs

    @staticmethod
    def _msg(name, args_here, region, off, cnt):
        """The argument the stray byte at `off` (bytes from the storage's start) belongs to, with its index there."""
        best = None
        for n, t in args_here:
            idx, exact = _index(t, off)
            if best is None or (exact and not best[2]):
                best = (n, idx, exact)
        n, idx, exact = best
        names = ", ".join(a for a, _ in args_here)
        where = f"element {list(idx)} of `{n}`" + ("" if exact else " (between its elements)")
        return f"{name}: {cnt} stray bytes in the {region} (the storage of `{names}`), the first at byte {off:+d}: {where}"

    # ------------------------------------------------------------------------------------------------ write footprints
    # One per kernel-launching method of the ops interface, with its parameters: the views the call may write.
    def _writes_pack_conv_weight(self, w, scale=1.0):
        return []                                # the packed weight is allocated in the call: fully writable

    def _writes_pack_conv_weight_dgrad(self, w):
        return []

    def _writes_conv_igemm(self, act, B, H, W, lda, c_off, c_in, wp, c_out, kh, kw, mode, bias, residual, out_f32, out_f16,
                           out_strides, block_n=0, out_sc=1, n_valid=0, act2=None, lda2=0, c_off2=0, c_in1=0,
                           out_stats=None):
        nv = n_valid if n_valid else c_out
        sb, sh, sw = out_strides
        return [_view(o, (B, H, W, nv), (sb, sh, sw, out_sc)) for o in (out_f32, out_f16)] + \
            [_first(out_stats, B, c_out // 16, 2)]

    def _writes_conv_res1x1(self, act, B, H, W, lda, c_in, act2, lda2, c_in1, x, ldx, x_cin, x2, ldx2, x_cin1, wp, c_out,
                            bias, residual, out_f32, out_f16, out_stats):
        return [_first(out_f32, B, H * W * c_out), _first(out_f16, B, H * W * c_out), _first(out_stats, B, c_out // 16, 2)]

    def _writes_conv_gn(self, src0, c0, src1, c1, scale1, B, H, W, groups, stats0, stats1, gamma, beta, scale_shift, ss_ld,
                        eps, wp, c_out, bias, residual, out_f32, out_f16, out_stats):
        return [_first(out_f32, B, H * W * c_out), _first(out_f16, B, H * W * c_out), _first(out_stats, B, c_out // 16, 2)]

    def _writes_conv_direct(self, inp, B, Hin, Win, c_in, ldi, w, c_out, kh, kw, stride, pad, bias, residual, out, Hout,
                            Wout, out_strides):
        return [_view(out, (B, Hout, Wout, c_out), out_strides)]

    def _writes_gn_stats(self, src0, c0, src1, c1, scale1, B, hw, groups, sums):
        return [_first(sums, B, groups, 2)]

    def _writes_gn_apply_silu(self, src0, c0, src1, c1, scale1, B, hw, groups, stats0, sb0, stats1, sb1, gamma, beta,
                              scale_shift, ss_ld, eps, out):
        return [_first(out, B, hw * (c0 + c1))]

    def _writes_cast_act(self, src0, c0, src1, c1, scale1, B, H, W, mode, out):
        return [_first(out, B, H * W * (c0 + c1) * (4 if mode == 1 else 1))]

    def _writes_ln_rows(self, inp, rows, C, gamma, beta, eps, pre_gelu, residual, out_f32, out_f16):
        return [_first(out_f32, rows, C), _first(out_f16, rows, C)]

    def _writes_linear_f32(self, inp, M, K, W, bias, Nout, in_act, out_act, addend, out_f32, out_f16, out_scale=1.0):
        return [_first(out_f32, M, Nout), _first(out_f16, M, Nout)]

    def _writes_posemb(self, t, B, dim, out):
        return [_first(out, B, dim)]

    def _writes_text_tokens(self, proj, B, L, D, mask, keep, null_embed, max_len, c_out, m, row_off, pooled):
        return [_view(c_out, (B, max_len, D), (m * D, D, 1), row_off * D), _first(pooled, B, D)]

    def _writes_place_rows(self, src, B, r, D, dst, m, row_off):
        return [_view(dst, (B, r, D), (m * D, D, 1), row_off * D)]

    def _writes_select_rows(self, a, null_row, keep, addend, B, Nn, out):
        return [_first(out, B, Nn)]

    def _writes_nchw_to_nhwc(self, a, ca, b, cb, B, hw, c_pad, out):
        return [_first(out, B, hw * c_pad)]

    def _writes_stem_unroll(self, a, ca, b, cb, B, H, W, out):
        return [_first(out, B, H * W * 128)]

    def _writes_resize_separable(self, inp, planes, hin, win, out, hout, wout, iy, wy, ix, wx, clamp=None):
        return [_first(out, planes, hout * wout)]

    def _writes_silu(self, inp, out):
        return [_first(out, inp.numel())]

    def _writes_attention(self, q, q_bs, ldq, k, v, kv_bs, ldkv, kv_hs, null_kv, mask, B, heads, n, m, out, o_bs, ldo):
        return [_view(out, (B, heads, n, 64), (o_bs, 64, ldo, 1))]           # and its workspace, allocated in the call

    def _writes_step_x0(self, x_t, eps_cond, eps_null, cond_scale, t, tab_a, tab_b, B, n, x0):
        return [_first(x0, B, n)]

    def _writes_step_quantile(self, x0, B, n, rank_lo, rank_hi, weight, min_s, s):
        return [_first(s, B)]

    def _writes_step_posterior(self, x0, x_t, noise, s, t, c1, c2, sigma, B, n, out):
        return [_first(out, B, n)]

    @staticmethod
    def _step(B, n, out, s_out, hist=None):
        return [_first(out, B, n), _first(s_out, B), _first(hist, B, n)]   # and the x0 workspace, allocated in the call

    def _writes_step_epilogue(self, x_t, eps_cond, eps_null, cond_scale, t, tab_a, tab_b, c1, c2, sigma, noise, B, n,
                              rank_lo, rank_hi, weight, min_s, out, s_out=None):
        return self._step(B, n, out, s_out)

    def _writes_step_epilogue_multistep(self, x_t, eps_cond, eps_null, cond_scale, t, tab_a, tab_b, c1, c2, sigma, c3,
                                        noise, hist, B, n, rank_lo, rank_hi, weight, min_s, out, s_out=None):
        return self._step(B, n, out, s_out, hist)

    def _writes_step_epilogue_scheduled(self, x_t, eps_cond, eps_null, cond_scale, w_sched, t, tab_a, tab_b, c1, c2, sigma,
                                        noise, B, n, rank_lo, rank_hi, weight, min_s, out, s_out=None):
        return self._step(B, n, out, s_out)

    def _writes_step_epilogue_multistep_scheduled(self, x_t, eps_cond, eps_null, cond_scale, w_sched, t, tab_a, tab_b, c1,
                                                  c2, sigma, c3, noise, hist, B, n, rank_lo, rank_hi, weight, min_s, out,
                                                  s_out=None):
        return self._step(B, n, out, s_out, hist)

    def _writes_guidance_rescale_factor(self, eps_cond, eps_null, cond_scale, w_sched, t, phi, B, n, f):
        return [_first(f, B)]                                               # and its workspace

    def _writes_step_epilogue_rescaled(self, x_t, eps_cond, eps_null, cond_scale, w_sched, f, t, tab_a, tab_b, c1, c2,
                                       sigma, c3, noise, hist, B, n, rank_lo, rank_hi, weight, min_s, out, s_out=None):
        return self._step(B, n, out, s_out, hist)

    def _writes_step_advance_t(self, t, B):
        return [_first(t, B)]

    def _writes_step_advance_t_table(self, t, next_t, T, B):
        return [_first(t, B)]

    def _writes_step_finalize(self, x, n, unnormalize, out):
        return [_first(out, n)]

    def _writes_inpaint_prologue(self, x, t, r, ra, rb, sqrt_acp, sqrt_1m_acp, k, m, z_renoise, z_known, T, B, C, hw):
        return [_first(x, B, C * hw)]

    def _writes_inpaint_advance(self, t, r, next_t, R, T, B):
        return [_first(t, B), _first(r, B)]

    def _writes_inpaint_finalize(self, x, k, m, B, C, hw, unnormalize, out):
        return [_first(out, B, C * hw)]

    def _writes_q_sample(self, x0, noise, t, tab_a, tab_b, B, n, post_scale, post_shift, out):
        return [_first(out, B, n)]

    def _writes_randn_keyed(self, out, seeds, B, n, kind, stage, t=None, r=None, R=None, label=0):
        return [_first(out, B, n)]

    def _writes_gemm_f32(self, A, B, C, M, N, K, a_str, b_str, c_str, Z1=1, Z2=1, a_b=(0, 0), b_b=(0, 0), c_b=(0, 0),
                         alpha=1.0, accumulate=False):
        return [_view(C, (Z1, Z2, M, N), (c_b[0], c_b[1], c_str[0], c_str[1]))]

    def _writes_colsum(self, x, M, Nc, out, accumulate=False):
        return [_first(out, Nc)]

    def _writes_conv_dgrad(self, dy, B, Ho, Wo, c_out, w, c_in, kh, kw, stride, pad, dx, Hi, Wi):
        return [_first(dx, B, Hi * Wi * c_in)]

    def _writes_conv_wgrad(self, dy, x, B, Hi, Wi, c_in, Ho, Wo, c_out, kh, kw, stride, pad, dw):
        return [_first(dw, c_out, c_in * kh * kw)]

    def _writes_conv_wgrad_tc(self, dy16, x16, B, Ho, Wo, c_in, c_out, kh, kw, dw, stride=1):
        return [_first(dw, c_out, c_in * kh * kw)]                          # and its workspace

    def _writes_gn_silu_bwd(self, x, dy, sums, B, hw, C, groups, gamma, beta, scale_shift, ss_ld, eps, dx, dgamma, dbeta,
                            dss, dss_ld):
        return [_first(dx, B, hw * C), _first(dgamma, C), _first(dbeta, C), _view(dss, (B, 2 * C), (dss_ld, 1))]

    def _writes_ln_rows_bwd(self, inp, dy, R, C, gamma, eps, pre_gelu, dx, dgamma, dbeta):
        return [_first(dx, R, C), _first(dgamma, C), _first(dbeta, C)]

    def _writes_softmax_rows(self, s, R, L):
        return [_first(s, R, L)]

    def _writes_softmax_rows_bwd(self, P, dP, R, L):
        return [_first(dP, R, L)]

    def _writes_upsample2x_bwd(self, dy, B, H, W, C, dx):
        return [_first(dx, B, H * W * C)]


def unchecked(proxy):
    """The methods a run called without a footprint check (the capability queries and the launch-mode setting aside)."""
    return proxy.called - proxy.checked - ALLOWED


@contextlib.contextmanager
def installed(ops):
    """Install `ops` as the process-wide backend for the block, restoring the previous one afterwards."""
    import minimagen_b200.ops as ops_mod
    prev = ops_mod._OPS
    ops_mod.set_ops(ops)
    try:
        yield ops
    finally:
        ops_mod.set_ops(prev)
