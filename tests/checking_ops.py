"""TEST INFRASTRUCTURE ONLY: `CheckingOps`, a proxy around an ops backend that checks every kernel call against float64.

For each call the proxy NaN-fills the pure outputs (and snapshots in-place inputs and accumulators), makes the call,
synchronises, and checks the outputs against the float64 reference of tests/fp64_ref.py built from THAT call's own
arguments, with that reference's per-element bound.  The inputs of every call are the run's own tensors, so no error
compounds from one call to the next.  Used by tests/test_gpu_lowering_calls.py around the native backend (a real forward,
and a real training step) and by tests/test_training_calls.py around the torch emulation on the CPU (to show that the
checkers are not vacuous).

  * epilogue / gn_stats statistics are checked as the INCREMENT of the accumulator over the call;
  * completeness: the methods a run called minus the methods checked must be empty apart from `ALLOWED` (capability
    queries), so a kernel added later cannot slip through unchecked;
  * accumulators: in a forward, every statistics accumulator is zero when first handed to a kernel and no two overlap (the
    ZeroArena carving); in a training step (`fresh_accumulators`), where every GroupNorm statistics / dgamma / dbeta
    accumulator is a fresh torch.zeros that the caching allocator recycles, every accumulator is zero at every hand-off;
  * conditioning: a cast_act that writes the fp16 copy of a gradient inside an autograd backward must hold it to a tensor
    rel-L2 of 2^-10, as normal-range fp16 does: an exact rounding of a mostly subnormal copy passes the float64 check and
    still loses the gradient.

Every kernel-launching method of the ops interface has a checker here, the sampling features' included (the RePaint
prologue / advance / finalize, the keyed draws, the scheduled and the rescaled step epilogues, the three-kernel step);
tests/test_sampling_feature_calls.py holds that against NativeOps itself, so one proxy checks a sample that combines them.

`sms` is the SM count the per-kernel summation plans (and so the bounds' accumulation lengths) depend on: the device's
multi_processor_count, or 132 (an H100 SXM) for the CPU emulation.

The image-sized checkers (convolutions, GroupNorm, casts, the stem, the NCHW -> NHWC copy) build their float64 references
and compare a few images at a time, and when one image's reference exceeds SLICE_ELEMENTS (a 1024 x 1024 conv: 8 - 16x
over), one band of rows at a time (`_bands`).  A conv band reads the rows its taps reach beyond it (the halo of its mode:
k // 2 rows for a k x k or the 15 x 1 stem conv, one phase row for the phase-split stride-2 conv and the sub-pixel Upsample
phases, two input rows for the stride-2 conv read in place) and keeps only its own output rows.  Every elementwise bound is
per element, so banding changes no verdict; the statistics (the conv epilogue's increment, gn_stats) are reduced per band
in float64 and the bands' sums, and bounds, added before the one comparison per image.  So a forward at 256 x 256 (b = 32,
2 GiB per activation in float64) or at 1024 x 1024 keeps its reference memory to a few GiB.  `images` restricts the
comparisons to some images (a test of a large batch that checks the images next to an index boundary).
"""
import contextlib
import io

import torch

import fp64_ref
import fp64_ref as R

F16, F32, F64 = torch.float16, torch.float32, torch.float64
ALLOWED = {"igemm_supported", "conv_res1x1_supported", "conv_gn_supported",
           "conv_wgrad_tc_supported",                                       # capability queries: no kernel runs
           "set_launch_mode"}                                               # a library setting: no kernel runs
NAN = float("nan")

# The training-side methods of the ops interface (NativeOps' "training side" section) and the two sampling-loop kernels a
# training step also runs (Imagen.forward / _p_losses): the coverage test requires a checker and a reaching case for each.
TRAINING_METHODS = {"gemm_f32", "colsum", "conv_dgrad", "conv_wgrad", "conv_wgrad_tc", "gn_silu_bwd", "ln_rows_bwd",
                    "softmax_rows", "softmax_rows_bwd", "upsample2x_bwd", "pack_conv_weight_dgrad", "q_sample",
                    "resize_separable"}


def _strided(t, shape, strides):
    return t.as_strided(shape, strides, t.storage_offset())


def _describe(args, kwargs):
    d = lambda v: f"{str(v.dtype).replace('torch.', '')}{list(v.shape)}/{list(v.stride())}" if torch.is_tensor(v) else repr(v)
    return ", ".join([d(a) for a in args] + [f"{k}={d(v)}" for k, v in kwargs.items()])


def default_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


SLICE_ELEMENTS = 1 << 26        # float64 elements per reference tensor of one piece of a check (512 MiB)


def _bands(B, H, per_row, halo=0, step=1, images=None):
    """The pieces a check computes its reference in: [(image slice, [(h0, h1), ...] its bands of rows)].  Whole images, a
    few at a time, while one image's largest reference tensor (H rows of per_row elements) fits SLICE_ELEMENTS; else one
    image at a time in bands of rows whose reference, with the `halo` rows read beyond the band on either side, fits.
    Band edges are multiples of `step`.  images: only these images, one slice each."""
    if H * per_row > SLICE_ELEMENTS:
        rows = max(step, (SLICE_ELEMENTS // per_row - 2 * halo) // step * step)
        bands = [(h, min(H, h + rows)) for h in range(0, H, rows)]
        return [(slice(b, b + 1), bands) for b in (range(B) if images is None else images)]
    if images is not None:
        return [(slice(b, b + 1), [(0, H)]) for b in images]
    n = max(1, SLICE_ELEMENTS // max(1, H * per_row))
    return [(slice(b, min(B, b + n)), [(0, H)]) for b in range(0, B, n)]


def _at(t, i):
    return None if t is None else t[i]


def _rows(t, i, h0, h1):
    return None if t is None else t[i, h0:h1]


def _add(acc, part):
    """Elementwise sum of (reference, bound) pairs; acc None to start."""
    return part if acc is None else (acc[0] + part[0], acc[1] + part[1])


class CheckingOps:
    def __init__(self, inner, sms=None, fresh_accumulators=False, only=None, strict=True, images=None):
        """only: check just these methods (the others run unchecked): lets a run with one planted defect skip the float64
        references of every other call.  strict=False: a failed check is recorded in `failures` and the run goes on (the
        outputs are the backend's own either way), so that one run gives both the verdict and the gradients;
        `raise_failures` raises the first one afterwards.  images: the image-sized checkers compare only these images."""
        self.inner = inner
        self.sms = default_sms() if sms is None else sms
        self.fresh = fresh_accumulators
        self.only = only
        self.strict = strict
        self.images = images
        self.image, self.per_image = None, {}   # the one image being compared; (method, image) -> worst |err| / bound
        self.failures = []
        self.called, self.checked = set(), set()
        self.family = {}                       # method -> [calls, worst |err| / bound]
        self.last = 0.0                        # worst |err| / bound of the latest checked call
        self.features = set()                  # call shapes that matter, reached and checked (conv modes, multi-query, ...)
        self.keyed = []                        # (kind, stage, per-image labels) of every randn_keyed call, in order
        self.accumulators = {}                 # data_ptr -> numel of every statistics accumulator seen

    def __getattr__(self, name):
        target = getattr(self.inner, name)
        if not callable(target):
            return target
        checker = getattr(self, "_check_" + name, None)
        if self.only is not None and name not in self.only:
            checker = None

        def call(*args, **kwargs):
            self.called.add(name)
            if checker is None:
                return target(*args, **kwargs)
            ran, ret = False, None
            self.last = 0.0
            try:
                with contextlib.redirect_stdout(io.StringIO()):          # R.check prints every comparison: keep the worst only
                    gen = checker(*args, **kwargs)
                    next(gen)                                            # prefill / snapshots
                    ran, ret = True, target(*args, **kwargs)
                    self._sync()
                    try:
                        gen.send(ret)                                    # comparisons
                    except StopIteration:
                        pass
            except AssertionError as e:
                msg = f"{name}({_describe(args, kwargs)}): {e}"
                if self.strict:
                    raise AssertionError(msg) from None
                self.failures.append(msg)
                return ret if ran else target(*args, **kwargs)
            self.checked.add(name)
            return ret
        return call

    def raise_failures(self):
        if self.failures:
            raise AssertionError(f"{len(self.failures)} failed calls, the first: {self.failures[0]}")

    def _sync(self):
        if torch.cuda.is_available():
            torch.cuda.synchronize()

    def _note(self, name, ratio):
        f = self.family.setdefault(name, [0, 0.0])
        f[1] = max(f[1], ratio)
        self.last = max(self.last, ratio)
        if self.image is not None:
            key = (name, self.image)
            self.per_image[key] = max(self.per_image.get(key, 0.0), ratio)

    def _count(self, name):
        self.family.setdefault(name, [0, 0.0])[0] += 1

    def _accumulator(self, t):
        """An accumulator about to be added into: zero the first time a kernel sees it (every time in a training step).
        Returns its value before the call."""
        if self.fresh:
            assert not t.any(), "an accumulator was handed to a kernel non-zero"
        elif t.data_ptr() not in self.accumulators:
            self.accumulators[t.data_ptr()] = t.numel()
            assert not t.any(), "a statistics accumulator was handed to its first kernel non-zero"
        return t.clone()

    def assert_accumulators_disjoint(self):
        spans = sorted(self.accumulators.items())
        for (p0, n0), (p1, _) in zip(spans, spans[1:]):
            assert p0 + 8 * n0 <= p1, f"statistics accumulators overlap: {p0:#x}+{n0} doubles and {p1:#x}"
        return len(spans)

    def report(self):
        for fam, (calls, worst) in sorted(self.family.items()):
            print(f"  {fam:28s} {calls:5d} calls   worst |err|/bound {worst:.3g}")

    def _bands(self, B, H, per_row, halo=0, step=1):
        """_bands with this proxy's `images`; while a piece of one image is compared, its ratios also go to per_image."""
        for i, rows in _bands(B, H, per_row, halo, step, self.images):
            self.image = i.start if i.stop - i.start == 1 else None
            yield i, rows
        self.image = None

    @staticmethod
    def _stats_band(f, e, P, sb=16):
        """The float64 (sum, sum of squares) per (image, sb channels) of one band of this call's output, and its bound (the
        image has P pixels): `f` the fp32 values the kernel summed (its own fp32 output), or their reference with
        elementwise bound `e` when only fp16 was stored.  Both add up over the bands of an image."""
        ref, bound = R.conv_stats_ref(f, sb, P)
        if e is not None:
            B, C = f.shape[0], f.shape[-1]
            blk = lambda t: t.reshape(B, -1, C // sb, sb).sum(dim=(1, 3))
            bound = bound + torch.stack((blk(e), blk(2 * f.abs() * e + e * e)), dim=-1)
        return ref, bound

    def _stats_increment(self, name, acc, before, ref, bound):
        """acc - before against the statistics `ref` (bound `bound`) of this call's output, summed over its bands.  Per
        image: acc, before and ref may be the same slice of images of a call (the caller counts the call)."""
        bound = bound + 4 * R.U64 * (before.abs() + acc.abs())             # the subtraction below
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
        self.features |= {f"conv_igemm mode {mode}", f"conv_igemm c_out={c_out}", f"conv_igemm K={kh * kw * c_in}",
                          f"conv_igemm W={W}"}
        if H * W < 128:
            self.features.add("conv_igemm multi-image tiles")               # a 128-pixel tile spans 128 / (H W) images
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
        if out_stats is not None:
            self._count("conv_igemm statistics")
            acc, before = out_stats.reshape(B, -1, 2), before.reshape(B, -1, 2)
        # a band of output rows [h0, h1) reads input rows [s h0 - halo, s h1 + halo) (s = 2: the stride-2 conv read in
        # place, whose input has 2H rows; mode 1's input rows are phase rows)
        s, halo = (2, 2) if mode == 6 else (1, kh // 2 if mode == 0 else 1)
        for i, rows in self._bands(B, H, W * max(4 * c_in, c_out), halo):
            st = None
            for h0, h1 in rows:
                lo, hi = max(0, s * h0 - halo), min(s * H, s * h1 + halo)
                ref, bound = R.conv_fwd_ref(a[i][..., lo:hi, :, :], wp, kh, kw, mode, bias,
                                            None if res is None else res[i, lo // s:hi // s])
                band = slice(h0 - lo // s, h1 - lo // s)                     # the band's rows of the slab's output
                ref, bound = ref[:, band], bound[:, band]
                self._out("conv_igemm", _rows(o32, i, h0, h1), _rows(o16, i, h0, h1), ref[..., :nv], bound[..., :nv])
                if out_stats is not None:
                    st = _add(st, self._stats_band(o32[i, h0:h1], None, H * W) if o32 is not None else
                             self._stats_band(ref, bound, H * W))
            if out_stats is not None:
                self._stats_increment("conv_igemm", acc[i], before[i], *st)

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
        rs = lambda t: None if t is None else t.reshape(B, H, W, c_out)
        res, o32, o16 = rs(residual), rs(out_f32), rs(out_f16)
        if out_stats is not None:
            self._count("conv_res1x1 statistics")
            acc, before = out_stats.reshape(B, -1, 2), before.reshape(B, -1, 2)
        for i, rows in self._bands(B, H, W * max(c_in + x_cin, c_out), 1):
            st = None
            for h0, h1 in rows:
                lo, hi = max(0, h0 - 1), min(H, h1 + 1)
                ref, bound = R.conv_fwd_ref(a[i, lo:hi], wp, 3, 3, 0, bias, None if res is None else res[i, lo:hi],
                                            x=xs[i, lo:hi])
                ref, bound = ref[:, h0 - lo:h1 - lo], bound[:, h0 - lo:h1 - lo]
                self._out("conv_res1x1", _rows(o32, i, h0, h1), _rows(o16, i, h0, h1), ref, bound)
                if out_stats is not None:
                    st = _add(st, self._stats_band(o32[i, h0:h1], None, H * W) if o32 is not None else
                             self._stats_band(ref, bound, H * W))
            if out_stats is not None:
                self._stats_increment("conv_res1x1", acc[i], before[i], *st)

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
            self._count("conv_gn statistics")
            st = (self._stats_band(rs(out_f32, c_out), None, H * W) if out_f32 is not None else
                  self._stats_band(ref, bound, H * W))
            self._stats_increment("conv_gn", out_stats, before, *st)

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

    def _check_pack_conv_weight_dgrad(self, w):
        """(I, KH KW O): the taps flipped, in / out channels swapped, tap-major / channel-minor -- one fp16 rounding of each
        fp32 weight, nothing else, so it must be exact."""
        self._count("pack_conv_weight_dgrad")
        out = yield
        w4 = w if w.dim() == 4 else w[:, :, None, None]
        ref = R._d(w4).flip(2, 3).transpose(0, 1).permute(0, 2, 3, 1).reshape(w4.shape[1], -1)
        want, _ = R.half_out(ref, torch.zeros((), dtype=F64, device=ref.device))
        self._note("pack_conv_weight_dgrad", R.check(out, want, 0.0, "data-gradient packed weight"))

    # ---------------------------------------------------------------- normalisation / casts
    def _check_gn_stats(self, src0, c0, src1, c1, scale1, B, hw, groups, sums):
        self._count("gn_stats")
        before = self._accumulator(sums).reshape(B, -1, 2)
        yield
        acc, s0, s1 = sums.reshape(B, -1, 2), src0.reshape(B, hw, c0), src1.reshape(B, hw, c1) if c1 else None
        for i, bands in self._bands(B, hw, c0 + c1):
            st = None
            for p0, p1 in bands:
                st = _add(st, R.gn_stats_ref(s0[i, p0:p1], groups, None if s1 is None else s1[i, p0:p1], scale1, HW=hw))
            ref, bound = st
            bound = bound + 4 * R.U64 * (before[i].abs() + acc[i].abs())
            self._note("gn_stats", R.check(acc[i] - before[i], ref, bound, "gn_stats increment"))

    def _check_gn_apply_silu(self, src0, c0, src1, c1, scale1, B, hw, groups, stats0, sb0, stats1, sb1, gamma, beta,
                             scale_shift, ss_ld, eps, out):
        self._count("gn_apply_silu")
        out.fill_(NAN)
        yield
        C = c0 + c1
        assert sb0 == 0 or (sb0 == 16 and (not c1 or sb1 == 16))
        sums = stats0 if sb0 == 0 else R.group_sums(stats0, c0, groups, stats1 if c1 else None, c1, scale1, sb0)
        sums = sums.reshape(B, groups, 2)
        ss = None if scale_shift is None else _strided(scale_shift, (B, 2 * C), (ss_ld, 1))
        s0, s1, o = src0.reshape(B, hw, c0), src1.reshape(B, hw, c1) if c1 else None, out.reshape(B, hw, C)
        for i, bands in self._bands(B, hw, C):
            for p0, p1 in bands:
                ref, bound = R.gn_apply_silu_ref(s0[i, p0:p1], groups, gamma, beta, _at(ss, i), eps, sums[i],
                                                 src1=None if s1 is None else s1[i, p0:p1], scale1=scale1,
                                                 out16=out.dtype == F16, HW=hw)
                self._note("gn_apply_silu", R.check(o[i, p0:p1], ref, bound, "gn_apply_silu"))

    def _check_cast_act(self, src0, c0, src1, c1, scale1, B, H, W, mode, out):
        self._count("cast_act")
        C = c0 + c1
        n_out = B * H * W * C * (4 if mode == 1 else 1)
        o = out.reshape(-1)[:n_out]                                        # mode 0 writes the first B*H*W rows of `out`
        o.fill_(NAN)
        backward = torch._C._current_graph_task_id() >= 0                  # called from an autograd backward
        err = nrm = 0.0
        yield
        s0, s1 = src0.reshape(B, H, W, c0), src1.reshape(B, H, W, c1) if c1 else None
        # the output rows of input rows [h0, h1): the same rows, rows [2 h0, 2 h1) of the nearest x2 upsample, or phase
        # rows [h0 / 2, h1 / 2) of each of the four phases (bands of even rows)
        ob = o.reshape((B, H, W, C) if mode == 0 else (B, 2 * H, 2 * W, C) if mode == 1 else (B, 4, H // 2, W // 2, C))
        for i, rows in self._bands(B, H, 4 * W * C, step=2 if mode == 2 else 1):
            for h0, h1 in rows:
                x = R.gn_concat(s0[i, h0:h1], None if s1 is None else s1[i, h0:h1], scale1)
                if mode == 0:
                    got = ob[i, h0:h1]
                elif mode == 1:
                    x, got = x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2), ob[i, 2 * h0:2 * h1]
                else:
                    x = torch.stack([x[:, (p >> 1)::2, (p & 1)::2] for p in range(4)], dim=1)
                    got = ob[i, :, h0 // 2:h1 // 2]
                bound = R.U32 * x.abs() if c1 else torch.zeros_like(x)     # the fp32 product with the skip scale
                ref, bound = R.half_out(x, bound) if out.dtype == F16 else (x, bound)
                self._note("cast_act", R.check(got, ref, bound, f"cast_act mode {mode}"))
                if out.dtype == F16 and backward:
                    err, nrm = err + float((got.to(F64) - x).norm()) ** 2, nrm + float(x.norm()) ** 2
        if out.dtype == F16 and backward:
            # conditioning: an fp16 copy of a gradient must still hold it.  A gradient cast unscaled (~1e-5 per element
            # under an MSE-mean loss) is mostly subnormal in fp16; rounded exactly, it passes the check above and loses
            # most of its bits.  Normal-range fp16 keeps the tensor's rel-L2 within 2^-11; the limit is 2^-10.
            rel = (err / nrm) ** 0.5 if nrm else 0.0
            assert rel <= 2.0 ** -10, (f"cast_act: the fp16 copy of a backward gradient is off by rel-L2 {rel:.3e} "
                                       f"(> 2^-10): cast it scaled into fp16's normal range")

    def _check_ln_rows(self, inp, rows, C, gamma, beta, eps, pre_gelu, residual, out_f32, out_f16):
        self._count("ln_rows")
        self.features.add(f"ln_rows C={C}")
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
        if not keep.bool().all():
            self.features.add(f"text_tokens null rows B={B}")
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
        for i, bands in self._bands(B, hw, 2 * c_pad):
            for p0, p1 in bands:
                want = torch.zeros((i.stop - i.start, p1 - p0, c_pad), dtype=F32, device=a.device)
                want[:, :, :ca] = a.reshape(B, ca, hw)[i, :, p0:p1].permute(0, 2, 1)
                if b is not None and cb:
                    want[:, :, ca:ca + cb] = b.reshape(B, cb, hw)[i, :, p0:p1].permute(0, 2, 1)
                assert torch.equal(out.reshape(B, hw, c_pad)[i, p0:p1], want), \
                    "nchw_to_nhwc is a transposing copy with zero padding"
        self._note("nchw_to_nhwc", 0.0)

    def _check_stem_unroll(self, a, ca, b, cb, B, H, W, out):
        self._count("stem_unroll")
        out.fill_(NAN)
        yield
        x = a if b is None or cb == 0 else torch.cat((a, b), dim=1)
        o = out.reshape(B, H, W, 128)
        for i, rows in self._bands(B, H, W * 128):
            for h0, h1 in rows:
                xp = torch.nn.functional.pad(x[i, :, h0:h1], (7, 8))       # the window is horizontal: no halo rows
                want = torch.zeros((xp.shape[0], h1 - h0, W, 16, 8), dtype=F64, device=a.device)
                for j in range(15):
                    want[:, :, :, j, :x.shape[1]] = xp[:, :, :, j:j + W].permute(0, 2, 3, 1)
                ref, bound = R.half_out(want.reshape(-1, h1 - h0, W, 128), torch.zeros((), dtype=F64, device=a.device))
                self._note("stem_unroll", R.check(o[i, h0:h1], ref, bound, "stem_unroll"))

    # ---------------------------------------------------------------- attention
    def _check_attention(self, q, q_bs, ldq, k, v, kv_bs, ldkv, kv_hs, null_kv, mask, B, heads, n, m, out, o_bs, ldo):
        self._count("attention")
        self.features.add(f"attention B={B} n={n}")
        o = _strided(out, (B, heads, n, 64), (o_bs, 64, ldo, 1))
        o.fill_(NAN)
        yield
        qv, kv, vv = R.attention_views(q, q_bs, ldq, k, v, kv_bs, ldkv, kv_hs, B, heads, n, m)
        ref, bound = R.attention_ref(qv, kv, vv, null_kv.detach().to(F16), mask)
        self._note("attention", R.check(o, ref, bound, "attention"))

    # ---------------------------------------------------------------- sampling-loop kernels a training step runs
    def _check_q_sample(self, x0, noise, t, tab_a, tab_b, B, n, post_scale, post_shift, out):
        self._count("q_sample")
        out.fill_(NAN)
        yield
        ref, bound = R.q_sample_ref(x0.reshape(B, n), noise.reshape(B, n), t, tab_a, tab_b, post_scale, post_shift)
        self._note("q_sample", R.check(out.reshape(B, n), ref, bound, "q_sample"))

    def _check_resize_separable(self, inp, planes, hin, win, out, hout, wout, iy, wy, ix, wx, clamp=None):
        self._count("resize_separable")
        out.fill_(NAN)
        yield
        ref, bound = R.resize_ref(inp.reshape(planes, hin, win), iy, wy, ix, wx, clamp)
        self._note("resize_separable", R.check(out.reshape(planes, hout, wout), ref, bound, "resize_separable"))

    # ---------------------------------------------------------------- the sampling step
    def _step(self, name, x_t, eps_cond, eps_null, cond_scale, t, tab_a, tab_b, c1, c2, sigma, c3, noise, hist, B, n,
              rank_lo, rank_hi, weight, min_s, out, s_out):
        """step_epilogue(_multistep) against step_x0_ref -> step_threshold_ref -> step_posterior_ref of tests/fp64_ref.py.
        x_t (which `out` may alias) and the history (overwritten with the clamped x0) are snapshotted before the call; s_out,
        when the caller passes one, is checked against the threshold's bound, and the new history against the clamped x0's.
        The bounds hold for finite data, which is what a sampling loop produces."""
        self._count(name)
        snap = lambda v: None if v is None else v.detach().reshape(B, n).cpu().clone()
        x0, h0 = snap(x_t), snap(hist)
        w = cond_scale.detach().cpu().clone() if torch.is_tensor(cond_scale) else cond_scale
        tt = t.detach().cpu().clone()
        if out.data_ptr() != x_t.data_ptr():
            out.fill_(NAN)
        if s_out is not None:
            s_out.fill_(NAN)
        yield
        xr, bx = R.step_x0_ref(x0, eps_cond.reshape(B, n), None if eps_null is None else eps_null.reshape(B, n), w, tt,
                               tab_a, tab_b)
        sr, bs = R.step_threshold_ref(xr, bx, rank_lo, rank_hi, weight, min_s)
        outr, bo, xsr, bxs = R.step_posterior_ref(xr, bx, sr, bs, x0, noise.reshape(B, n), tt, c1, c2, sigma, c3, h0)
        worst = R.check(out.reshape(B, n), outr, bo, f"{name} out")
        if s_out is not None:
            worst = max(worst, R.check(s_out.reshape(-1)[:B], sr, bs, f"{name} threshold s"))
        if hist is not None:
            worst = max(worst, R.check(hist.reshape(B, n), xsr, bxs, f"{name} history (clamped x0)"))
        self._note(name, worst)

    def _check_step_epilogue(self, x_t, eps_cond, eps_null, cond_scale, t, tab_a, tab_b, c1, c2, sigma, noise, B, n, rank_lo,
                             rank_hi, weight, min_s, out, s_out=None):
        return self._step("step_epilogue", x_t, eps_cond, eps_null, cond_scale, t, tab_a, tab_b, c1, c2, sigma, None, noise,
                          None, B, n, rank_lo, rank_hi, weight, min_s, out, s_out)

    def _check_step_epilogue_multistep(self, x_t, eps_cond, eps_null, cond_scale, t, tab_a, tab_b, c1, c2, sigma, c3, noise,
                                       hist, B, n, rank_lo, rank_hi, weight, min_s, out, s_out=None):
        return self._step("step_epilogue_multistep", x_t, eps_cond, eps_null, cond_scale, t, tab_a, tab_b, c1, c2, sigma, c3,
                          noise, hist, B, n, rank_lo, rank_hi, weight, min_s, out, s_out)

    def _check_step_epilogue_scheduled(self, x_t, eps_cond, eps_null, cond_scale, w_sched, t, tab_a, tab_b, c1, c2, sigma,
                                       noise, B, n, rank_lo, rank_hi, weight, min_s, out, s_out=None):
        """The step epilogue at the scheduled weights w_b(t[b]) (fp64_ref.scheduled_weights, each image at its own t)."""
        self.features.add("step_epilogue_scheduled per-image w")
        return self._step("step_epilogue_scheduled", x_t, eps_cond, eps_null, R.scheduled_weights(cond_scale, w_sched, t, B),
                          t, tab_a, tab_b, c1, c2, sigma, None, noise, None, B, n, rank_lo, rank_hi, weight, min_s, out,
                          s_out)

    def _check_step_epilogue_multistep_scheduled(self, x_t, eps_cond, eps_null, cond_scale, w_sched, t, tab_a, tab_b, c1,
                                                 c2, sigma, c3, noise, hist, B, n, rank_lo, rank_hi, weight, min_s, out,
                                                 s_out=None):
        return self._step("step_epilogue_multistep_scheduled", x_t, eps_cond, eps_null,
                          R.scheduled_weights(cond_scale, w_sched, t, B), t, tab_a, tab_b, c1, c2, sigma, c3, noise, hist, B,
                          n, rank_lo, rank_hi, weight, min_s, out, s_out)

    def _check_guidance_rescale_factor(self, eps_cond, eps_null, cond_scale, w_sched, t, phi, B, n, f):
        """f [B] within one fp32 ulp of the fp64 factor of the fp32 guided prediction (fp64_ref.rescale_factor_ref)."""
        self._count("guidance_rescale_factor")
        w = cond_scale.detach().cpu().clone() if torch.is_tensor(cond_scale) else cond_scale
        ref, bound = R.rescale_factor_ref(eps_cond, eps_null, w, w_sched, t, phi, B, n)
        f.fill_(NAN)
        yield
        self._note("guidance_rescale_factor", R.check(f.reshape(-1)[:B], ref, bound, "guidance_rescale_factor f"))

    def _check_step_epilogue_rescaled(self, x_t, eps_cond, eps_null, cond_scale, w_sched, f, t, tab_a, tab_b, c1, c2,
                                      sigma, c3, noise, hist, B, n, rank_lo, rank_hi, weight, min_s, out, s_out=None):
        """The step of the fp32 rescaled prediction fp32(g * f_b) (fp64_ref.rescaled_eps_fp32, formed as the kernel forms
        it) with no guidance pass: the checks of step_epilogue(_multistep) on that input."""
        self.features.add("step_epilogue_rescaled " + ("multistep" if hist is not None else "plain") +
                          (" scheduled" if w_sched is not None else ""))
        w = cond_scale.detach().cpu().clone() if torch.is_tensor(cond_scale) else cond_scale
        eps = R.rescaled_eps_fp32(eps_cond, eps_null, w, w_sched, t, f, B, n)
        return self._step("step_epilogue_rescaled", x_t, eps, None, 1.0, t, tab_a, tab_b, c1, c2, sigma, c3, noise, hist,
                          B, n, rank_lo, rank_hi, weight, min_s, out, s_out)

    # the three-kernel form of the step (the step epilogue's pieces), against the same references
    def _check_step_x0(self, x_t, eps_cond, eps_null, cond_scale, t, tab_a, tab_b, B, n, x0):
        self._count("step_x0")
        x0.fill_(NAN)
        yield
        ref, bound = R.step_x0_ref(x_t.reshape(B, n), eps_cond.reshape(B, n),
                                   None if eps_null is None else eps_null.reshape(B, n), cond_scale, t, tab_a, tab_b)
        self._note("step_x0", R.check(x0.reshape(B, n), ref, bound, "step_x0"))

    def _check_step_quantile(self, x0, B, n, rank_lo, rank_hi, weight, min_s, s):
        """The threshold of the fp32 x0 the call reads: exact operands (zero input bound)."""
        self._count("step_quantile")
        s.fill_(NAN)
        yield
        x = R._d(x0.reshape(B, n)).cpu()
        ref, bound = R.step_threshold_ref(x, torch.zeros_like(x), rank_lo, rank_hi, weight, min_s)
        self._note("step_quantile", R.check(s.reshape(-1)[:B], ref, bound, "step_quantile s"))

    def _check_step_posterior(self, x0, x_t, noise, s, t, c1, c2, sigma, B, n, out):
        self._count("step_posterior")
        xt0 = x_t.detach().reshape(B, n).clone()
        if out.data_ptr() != x_t.data_ptr():
            out.fill_(NAN)
        yield
        x = R._d(x0.reshape(B, n)).cpu()
        sv = R._d(s.reshape(-1)[:B]).cpu()
        ref, bound, _, _ = R.step_posterior_ref(x, torch.zeros_like(x), sv, torch.zeros_like(sv), xt0, noise.reshape(B, n),
                                                t, c1, c2, sigma)
        self._note("step_posterior", R.check(out.reshape(B, n), ref, bound, "step_posterior"))

    # ---------------------------------------------------------------- RePaint and keyed draws
    def _check_inpaint_prologue(self, x, t, r, ra, rb, sqrt_acp, sqrt_1m_acp, k, m, z_renoise, z_known, T, B, C, hw):
        """In place on x: against fp64_ref.inpaint_prologue_ref within its per-element bound, and the pixels neither branch
        takes bitwise unchanged.  z_renoise must not be read where r == 0: those images of it are NaN during the call (and
        restored after it), unless it is z_known itself (the eager loop passes the 'inpaint' draw in its place at r = 0)."""
        self._count("inpaint_prologue")
        xv, mv = x.reshape(B, C, hw), m.reshape(B, 1, hw)
        x0, tt, rr = xv.detach().clone(), t[:B].clone(), r[:B].clone()
        valid = (tt >= 0) & (tt < T)
        if bool((valid & (rr > 0)).any()):
            self.features.add("inpaint_prologue re-noise")
        if bool((valid & (rr == 0)).any()):
            self.features.add("inpaint_prologue r = 0")
        if bool((mv == 0.5).any()):
            self.features.add("inpaint_prologue m = 0.5")
        zr = z_renoise.reshape(B, C, hw)
        idle = rr <= 0
        shared = z_renoise.untyped_storage().data_ptr() == z_known.untyped_storage().data_ptr()
        saved = None
        if bool(idle.any()) and not shared:
            saved = zr[idle].clone()
            zr[idle] = NAN
        yield
        if saved is not None:
            zr[idle] = saved
        ref, bound, touched = R.inpaint_prologue_ref(x0, tt, rr, ra, rb, sqrt_acp, sqrt_1m_acp, k.reshape(B, C, hw), mv,
                                                     zr, z_known.reshape(B, C, hw), T)
        bits = lambda v: v.detach().view(torch.int32)[~touched]
        assert torch.equal(bits(xv), bits(x0)), "inpaint_prologue: a pixel neither branch takes must be left bitwise as it was"
        self._note("inpaint_prologue", R.check(xv, ref, bound, "inpaint_prologue"))

    def _check_inpaint_advance(self, t, r, next_t, R, T, B):
        """r <- r + 1 while r + 1 < R[0] at 0 < t < T, else r <- 0 and t <- next_t[t] (0 outside [0, T)): exact."""
        self._count("inpaint_advance")
        t0, r0 = t[:B].clone(), r[:B].clone()
        yield
        valid = (t0 >= 0) & (t0 < T)
        rep = valid & (t0 > 0) & (r0 + 1 < R.reshape(-1)[0])
        want_t = torch.where(rep, t0, torch.where(valid, next_t[t0.clamp(0, T - 1)], torch.zeros_like(t0)))
        want_r = torch.where(rep, r0 + 1, torch.zeros_like(r0))
        if bool(rep.any()):
            self.features.add("inpaint_advance repeat")
        if bool((~rep).any()):
            self.features.add("inpaint_advance next point")
        assert torch.equal(t[:B], want_t) and torch.equal(r[:B], want_r), \
            "inpaint_advance: (t, r) <- the next RePaint iteration is exact"
        self._note("inpaint_advance", 0.0)

    def _check_inpaint_finalize(self, x, k, m, B, C, hw, unnormalize, out):
        """clamp(where(m >= 0.5, k, x), -1, 1) with torch's NaN semantics, then (v + 1) * 0.5 when unnormalising: a select
        and two fp32 roundings in this order, so the result must be bit for bit torch's (NaN in x survives where m < 0.5)."""
        self._count("inpaint_finalize")
        xv = x.reshape(B, C, hw)
        x0 = xv.detach().clone()
        o = out.reshape(B, C, hw)
        if o.data_ptr() != x.data_ptr():
            o.fill_(NAN)
        yield
        v = torch.where(m.reshape(B, 1, hw) >= 0.5, k.reshape(B, C, hw), x0).clamp(-1.0, 1.0)
        want = (v + 1.0) * 0.5 if unnormalize else v
        same = torch.equal(o.isnan(), want.isnan()) and torch.equal(o[~o.isnan()], want[~want.isnan()])
        assert same, "inpaint_finalize: a select, a clamp and one fp32 add and product, it must be bitwise torch's"
        self._note("inpaint_finalize", 0.0)

    def _check_randn_keyed(self, out, seeds, B, n, kind, stage, t=None, r=None, R=None, label=0):
        """Image b's normals against tests/keyed_noise_restatement.py in float64 from the same Philox bits, within its
        relative bound (keyed_noise_restatement.ulp_bound, from CUDA's documented ulp errors).  The labels are read as the
        kernel reads them: t[b] * R[0] + r[b] from the device tensors when t is given (r, R optional), else `label`.  Each
        call's (kind, stage, labels) goes to `keyed` and to `features`."""
        import keyed_noise_restatement as K
        self._count("randn_keyed")
        if t is None:
            labels = [int(label)] * B
        else:
            lab = t[:B].cpu() * (int(R.reshape(-1)[0]) if R is not None else 1) + (r[:B].cpu() if r is not None else 0)
            labels = [int(v) for v in lab]
        name = {v: k for k, v in K.KINDS.items()}[int(kind)]
        self.keyed.append((name, int(stage), tuple(labels)))
        self.features.add(f"randn_keyed {name} stage {int(stage)}")
        if t is not None:
            self.features.add(f"randn_keyed {name} stage {int(stage)} device labels")
        self.features |= {f"randn_keyed {name} stage {int(stage)} label {v}" for v in labels}
        ov = out.reshape(B, n)
        ov.fill_(NAN)
        yield
        z64 = torch.from_numpy(K.randn_keyed([int(s) for s in seeds[:B].cpu()], n, int(kind), int(stage), labels))
        z64 = z64.to(ov.device)
        self._note("randn_keyed", fp64_ref.check(ov, z64, K.ulp_bound() * z64.abs() + 2.0 ** -126, f"randn_keyed {name}"))

    def _check_step_advance_t(self, t, B):
        """t <- max(t - 1, 0): exact."""
        self._count("step_advance_t")
        t0 = t[:B].clone()
        yield
        assert torch.equal(t[:B], (t0 - 1).clamp(min=0)), "step_advance_t: t <- max(t - 1, 0) is exact"
        self._note("step_advance_t", 0.0)

    def _check_step_advance_t_table(self, t, next_t, T, B):
        """t <- next_t[t], and 0 for a t outside [0, T): exact."""
        self._count("step_advance_t_table")
        t0 = t[:B].clone()
        yield
        inside = (t0 >= 0) & (t0 < T)
        want = torch.where(inside, next_t[t0.clamp(0, T - 1)], torch.zeros_like(t0))
        assert torch.equal(t[:B], want), "step_advance_t_table: t <- next_t[t] is exact"
        self._note("step_advance_t_table", 0.0)

    def _check_step_finalize(self, x, n, unnormalize, out):
        """clamp(x, -1, 1) with torch's NaN semantics, then (v + 1) * 0.5 when unnormalising: two fp32 roundings in this
        order, so the result must be bit for bit torch's."""
        self._count("step_finalize")
        x0 = x.reshape(-1)[:n].clone()
        o = out.reshape(-1)[:n]
        if o.data_ptr() != x.data_ptr():
            o.fill_(NAN)
        yield
        v = x0.clamp(-1.0, 1.0)
        want = (v + 1.0) * 0.5 if unnormalize else v
        same = torch.equal(o.isnan(), want.isnan()) and torch.equal(o[~o.isnan()], want[~want.isnan()])
        assert same, "step_finalize: a clamp and one fp32 add and product, it must be bitwise torch's"
        self._note("step_finalize", 0.0)

    # ---------------------------------------------------------------- training side (backward kernels)
    def _check_gemm_f32(self, A, B, C, M, N, K, a_str, b_str, c_str, Z1=1, Z2=1, a_b=(0, 0), b_b=(0, 0), c_b=(0, 0),
                        alpha=1.0, accumulate=False):
        self._count("gemm_f32")
        if Z2 > 1 and b_b[1] == 0:
            self.features.add("gemm_f32 multi-query")                       # one K / V head broadcast over the query heads
        elif Z2 > 1:
            self.features.add("gemm_f32 per-head")
        if K % 32:
            self.features.add("gemm_f32 ragged K")
        Av = _strided(A, (Z1, Z2, M, K), (a_b[0], a_b[1], a_str[0], a_str[1]))
        Bv = _strided(B, (Z1, Z2, K, N), (b_b[0], b_b[1], b_str[0], b_str[1]))
        Cv = _strided(C, (Z1, Z2, M, N), (c_b[0], c_b[1], c_str[0], c_str[1]))
        # the C views of different z (and the elements of one view) must not share an element: every offset hit once
        ar = lambda n, s: torch.arange(n, device=C.device, dtype=torch.int64) * s
        offs = (ar(Z1, c_b[0])[:, None, None, None] + ar(Z2, c_b[1])[None, :, None, None]
                + ar(M, c_str[0])[None, None, :, None] + ar(N, c_str[1])[None, None, None, :]).reshape(-1)
        assert int(offs.min()) >= 0 and int(torch.bincount(offs).max()) == 1, "gemm_f32: the C views overlap"
        del offs
        C0 = Cv.clone() if accumulate else None
        if not accumulate:
            Cv.fill_(NAN)
        yield
        ref, bound = R.gemm_ref(Av, Bv, C0, alpha, accumulate)
        self._note("gemm_f32", R.check(Cv, ref, bound, f"gemm_f32 K={K}" + (" (multi-query B)" if Z2 > 1 and b_b[1] == 0 else "")))

    def _check_colsum(self, x, M, Nc, out, accumulate=False):
        self._count("colsum")
        out0 = out.clone() if accumulate else None
        if not accumulate:
            out.fill_(NAN)
        yield
        ref, bound = R.colsum_ref(x.reshape(-1)[:M * Nc].reshape(M, Nc), out0, R.colsum_acc_len(M))
        self._note("colsum", R.check(out.reshape(Nc), ref, bound, "colsum"))

    def _check_softmax_rows(self, s, rows, L):
        self._count("softmax_rows")
        if L % 32:
            self.features.add("softmax_rows ragged L")
        s0 = s.reshape(-1)[:rows * L].reshape(rows, L).clone()             # in place: the reference reads the scores before
        yield
        self._note("softmax_rows", R.check(s.reshape(-1)[:rows * L].reshape(rows, L), *R.softmax_ref(s0), "softmax_rows"))

    def _check_softmax_rows_bwd(self, P, dP, rows, L):
        self._count("softmax_rows_bwd")
        view = lambda t: t.reshape(-1)[:rows * L].reshape(rows, L)
        d0 = view(dP).clone()                                              # in place on dP
        yield
        self._note("softmax_rows_bwd", R.check(view(dP), *R.softmax_bwd_ref(view(P), d0), "softmax_rows_bwd"))

    def _check_gn_silu_bwd(self, x, dy, sums, B, hw, C, groups, gamma, beta, scale_shift, ss_ld, eps, dx, dgamma, dbeta,
                           dss, dss_ld):
        self._count("gn_silu_bwd")
        dx.fill_(NAN)
        dssv = None if dss is None else _strided(dss, (B, 2 * C), (dss_ld, 1))
        if dssv is not None:
            dssv.fill_(NAN)
        dg0, db0 = self._accumulator(dgamma), self._accumulator(dbeta)      # accumulated onto
        yield
        ss = None if scale_shift is None else _strided(scale_shift, (B, 2 * C), (ss_ld, 1))
        (rx, bx), (rg, bg), (rb, bb), (rsc, bsc), (rsh, bsh) = R.gn_silu_bwd_ref(
            x.reshape(B, hw, C), dy.reshape(B, hw, C), gamma, beta, ss, groups, eps, dg0, db0,
            R.gn_bwd_acc_len(B, hw, C, self.sms))
        w = max(R.check(dx.reshape(B, hw, C), rx, bx, "gn_silu_bwd dx"),
                R.check(dgamma, rg, bg, "gn_silu_bwd dgamma"),
                R.check(dbeta, rb, bb, "gn_silu_bwd dbeta"))
        if dssv is not None:
            w = max(w, R.check(dssv[:, :C], rsc, bsc, "gn_silu_bwd dscale"), R.check(dssv[:, C:], rsh, bsh, "gn_silu_bwd dshift"))
        self._note("gn_silu_bwd", w)

    def _check_ln_rows_bwd(self, inp, dy, rows, C, gamma, eps, pre_gelu, dx, dgamma, dbeta):
        """dbeta is None for ChanLayerNorm (no beta): the reference gets zeros and that output is skipped."""
        self._count("ln_rows_bwd")
        if pre_gelu:
            self.features.add("ln_rows_bwd pre_gelu")
        dx.fill_(NAN)
        dev = inp.device
        dg0 = self._accumulator(dgamma) if dgamma is not None else torch.zeros(C, dtype=F32, device=dev)
        db0 = self._accumulator(dbeta) if dbeta is not None else torch.zeros(C, dtype=F32, device=dev)
        yield
        (rx, bx), (rg, bg), (rb, bb) = R.ln_bwd_ref(inp.reshape(rows, C), dy.reshape(rows, C), gamma.reshape(C), eps,
                                                    bool(pre_gelu), dg0.reshape(C), db0.reshape(C),
                                                    R.ln_bwd_acc_len(rows, self.sms))
        w = R.check(dx.reshape(rows, C), rx, bx, f"ln_rows_bwd dx (pre_gelu {int(bool(pre_gelu))})")
        if dgamma is not None:
            w = max(w, R.check(dgamma.reshape(C), rg, bg, "ln_rows_bwd dgamma"))
        if dbeta is not None:
            w = max(w, R.check(dbeta.reshape(C), rb, bb, "ln_rows_bwd dbeta"))
        self._note("ln_rows_bwd", w)

    def _check_conv_wgrad_tc(self, dy16, x16, B, Ho, Wo, c_in, c_out, kh, kw, dw, stride=1):
        """x16 is [B, s Ho, s Wo, c_in]; padding k // 2 (stride 1) or 1 (the stride-2 Downsample).  LinearFn passes its
        zero-padded fp16 rows as (Mp / 64) images of 8 x 8 pixels: the same contraction over rows."""
        self._count("conv_wgrad_tc")
        self.features.add("conv_wgrad_tc rows" if (Ho, Wo, kh) == (8, 8, 1) else f"conv_wgrad_tc k={kh} s={stride}")
        if c_in % 128 == 0:
            self.features.add("conv_wgrad_tc two N blocks")
        dw.fill_(NAN)                                                      # overwritten
        yield
        pad = 1 if stride == 2 else kh // 2
        dyv = dy16.reshape(-1)[:B * Ho * Wo * c_out].reshape(B, Ho, Wo, c_out)
        xv = x16.reshape(-1)[:B * stride * Ho * stride * Wo * c_in].reshape(B, stride * Ho, stride * Wo, c_in)
        ref, bound = R.conv_wgrad_ref(dyv, xv, stride, pad, kh, kw, R.wgrad_tc_acc_len(B, Ho, Wo, c_in, c_out, kh, self.sms))
        self._note("conv_wgrad_tc", R.check(dw.reshape(c_out, c_in, kh, kw), ref, bound, f"conv_wgrad_tc k={kh} s={stride}"))

    def _check_conv_wgrad(self, dy, x, B, Hi, Wi, c_in, Ho, Wo, c_out, kh, kw, stride, pad, dw):
        """The call's own semantics: Conv2dFn's final conv passes (x, dy) swapped, and the same reference applies to them."""
        self._count("conv_wgrad")
        self.features.add("conv_wgrad flat" if c_in < 32 and kh * kw > 1 else "conv_wgrad tiled")
        dw.fill_(NAN)
        yield
        ref, bound = R.conv_wgrad_ref(dy.reshape(B, Ho, Wo, c_out), x.reshape(B, Hi, Wi, c_in), stride, pad, kh, kw,
                                      R.wgrad_f32_acc_len(B, Ho, Wo, c_in, c_out, kh, kw, self.sms))
        self._note("conv_wgrad", R.check(dw.reshape(c_out, c_in, kh, kw), ref, bound, f"conv_wgrad k={kh} s={stride}"))

    def _check_conv_dgrad(self, dy, B, Ho, Wo, c_out, w, c_in, kh, kw, stride, pad, dx, Hi, Wi):
        self._count("conv_dgrad")
        dx.fill_(NAN)
        yield
        ref, bound = R.conv_dgrad_ref(dy.reshape(B, Ho, Wo, c_out), w.reshape(c_out, c_in, kh, kw), stride, pad, Hi, Wi)
        self._note("conv_dgrad", R.check(dx.reshape(B, Hi, Wi, c_in), ref, bound, f"conv_dgrad k={kh} s={stride}"))

    def _check_upsample2x_bwd(self, dy, B, H, W, C, dx):
        self._count("upsample2x_bwd")
        dx.fill_(NAN)
        yield
        want = R.upsample2x_bwd_ref(dy.reshape(B, 2 * H, 2 * W, C))
        assert torch.equal(dx.reshape(B, H, W, C), want), "upsample2x_bwd: a fixed-order fp32 sum, it must be bitwise equal"
        self._note("upsample2x_bwd", 0.0)


# ------------------------------------------------------------------------------------------------ training-step cases
SR_D64 = dict(dim=64, dim_mults=(1, 2, 4), num_resnet_blocks=(1, 2, 2), layer_attns=(False, False, True),
              layer_cross_attns=(False, True, True), lowres_cond=True, memory_efficient=True)
BASE_D64 = dict(dim=64, dim_mults=(1, 2), attend_at_middle=True, text_embed_dim=768)
SR_D128 = dict(dim=128, dim_mults=(1, 2, 4), num_resnet_blocks=(1, 2, 1), layer_attns=(False, True, True),
               layer_cross_attns=(False, True, True), lowres_cond=True, memory_efficient=True)
RAGGED = dict(dim=64, dim_mults=(1, 2, 4), layer_attns=(False, True, True), layer_cross_attns=(False, True, True),
              text_embed_dim=768)


def train_cases():
    """name -> (run spec, the families the case must reach).  A family is a method name or a call shape that matters
    (CheckingOps.features).  A unet spec is ("unet", cfg, image size, batch); a cascade spec ("cascade", unet_number) is one
    Imagen.forward of the tests/golden/train_tiny.pt cascade."""
    from minimagen_b200.Unet import Super
    conv_bwd = {"conv_igemm", "pack_conv_weight_dgrad", "gn_silu_bwd", "colsum", "conv_dgrad"}
    return {
        # tensor-core routes: weight gradient on wgmma at k = 3 and at the stride-2 Downsample, data gradient through the
        # forward conv (flipped packed weight) and the Downsample's four sub-pixel phases; cross-attention; the stem's flat
        # fp32 weight gradient (C_in = 6) and the final conv's swapped one
        "sr_d64": (("unet", SR_D64, 64, 2), conv_bwd | {
            "conv_wgrad_tc k=3 s=1", "conv_wgrad_tc k=4 s=2", "conv_igemm mode 2", "conv_igemm mode 3", "conv_igemm mode 4",
            "conv_igemm mode 5", "conv_wgrad flat", "gemm_f32 per-head", "softmax_rows", "softmax_rows_bwd",
            "ln_rows_bwd", "upsample2x_bwd"}),
        # multi-query attention (one K / V head), LinearFn over 2 x 258 context rows zero-padded to 640 (weight gradient over
        # 8 x 8 "images" of rows), GELU in front of the feed-forward LayerNorm, softmax over 1 + 1024 keys
        "base_d64_mid_attn": (("unet", BASE_D64, 32, 2), conv_bwd | {
            "gemm_f32 multi-query", "gemm_f32 ragged K", "conv_wgrad_tc rows", "ln_rows_bwd pre_gelu",
            "softmax_rows ragged L", "softmax_rows_bwd", "conv_wgrad_tc k=3 s=1", "conv_igemm mode 6"}),
        # C_out 128 / 256 / 512: 256-wide tiles in the data gradient, wgrad_tc with C_in % 128 == 0 (two N blocks)
        "sr_d128": (("unet", SR_D128, 64, 2), conv_bwd | {"conv_wgrad_tc two N blocks", "conv_wgrad_tc k=3 s=1"}),
        # 40 / 20 / 10 pixels: the fp32 route (direct conv forward, conv_dgrad, tiled conv_wgrad), fp32 GEMM linear
        # fallback, softmax over key counts that are not multiples of 32
        "ragged_40x40_d64": (("unet", RAGGED, 40, 3), {
            "conv_direct", "conv_dgrad", "conv_wgrad tiled", "gemm_f32", "colsum", "softmax_rows ragged L",
            "softmax_rows_bwd", "gn_silu_bwd", "ln_rows_bwd"}),
        # Imagen.forward: the cascade resize and both q_sample calls of _p_losses, the small-channel path
        "cascade_unet1": (("cascade", 1), {"resize_separable", "q_sample", "conv_wgrad", "conv_dgrad", "gn_silu_bwd"}),
        "cascade_unet2": (("cascade", 2), {"resize_separable", "q_sample", "conv_wgrad", "conv_dgrad", "gn_silu_bwd",
                                           "upsample2x_bwd"}),
        # the flagship network's backward at real channel counts
        "cfg3_structure_64x64": (("unet", dict(Super.defaults, lowres_cond=True, text_embed_dim=768), 64, 2), conv_bwd | {
            "conv_wgrad_tc k=3 s=1", "conv_wgrad_tc two N blocks", "softmax_rows_bwd", "ln_rows_bwd", "upsample2x_bwd"}),
    }


def perturbed_unet(cfg, seed=0):
    """A U-Net in train mode whose norm gains / biases are not the 1 / 0 of a fresh init (a swapped or dropped one must
    show), as in tests/test_lowering_exact.py."""
    from minimagen_b200.Unet import Unet
    torch.manual_seed(seed)
    u = Unet(**cfg).train()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for p in u.parameters():
            if p.dim() == 1 or p.shape[0] == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
    return u


def run_training_step(spec, device):
    """One eager training step (forward under grad mode, MSE loss, loss.backward()) through whatever ops backend is
    installed.  Returns {parameter name: gradient}."""
    import torch.nn.functional as F
    if spec[0] == "cascade":
        from conftest import load_golden
        from minimagen_b200.Imagen import Imagen
        from minimagen_b200.Unet import Unet
        g = load_golden("train_tiny.pt")
        im = Imagen(unets=[Unet(**c["cfg"]) for c in g["cases"]], text_encoder_name="t5_small",
                    image_sizes=g["image_sizes"], timesteps=g["timesteps"], cond_drop_prob=g["cond_drop_prob"])
        for u, c in zip(im.unets, g["cases"]):
            u.load_state_dict(c["state_dict"])
        im = im.to(device).train()
        gen = torch.Generator().manual_seed(3)
        images = torch.rand(3, 3, 40, 40, generator=gen).to(device)        # larger than both stages: resized inside
        torch.manual_seed(5)                                                # timesteps, noise, conditioning dropout
        loss = im(images, text_embeds=g["text_embeds"].to(device), text_masks=g["text_mask"].to(device),
                  unet_number=spec[1])
        loss.backward()
        unet = im.unets[spec[1] - 1]
    else:
        _, cfg, s, b = spec
        unet = perturbed_unet(cfg).to(device)
        g = torch.Generator().manual_seed(3)
        x = torch.randn(b, 3, s, s, generator=g)
        tm = torch.ones(b, 20, dtype=torch.bool)
        tm[-1, 5:] = False
        kw = dict(text_embeds=torch.randn(b, 20, cfg.get("text_embed_dim", 512), generator=g), text_mask=tm)
        if cfg.get("lowres_cond"):
            kw.update(lowres_cond_img=torch.randn(b, 3, s, s, generator=g), lowres_noise_times=torch.full((b,), 200))
        t = torch.randint(0, 1000, (b,), generator=g)
        target = torch.randn(x.shape, generator=g)
        mv = lambda v: v.to(device)
        loss = F.mse_loss(unet(mv(x), mv(t), **{k: mv(v) for k, v in kw.items()}), mv(target))
        loss.backward()
    assert torch.isfinite(loss.detach())
    return {k: p.grad.detach().clone() for k, p in unet.named_parameters() if p.grad is not None}
