// HBM-bound elementwise / reduction kernels of the U-Net hot path (NHWC activations, fp32 residual stream).
// Each kernel cites the reference op it replaces.  All are plain CUDA-core kernels: coalesced 16-byte accesses,
// fp32 math, double accumulation where a global reduction is involved.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "clamp_nan.cuh"
#include "kernels.cuh"
#include "launch.cuh"
#include "sat_half.cuh"

namespace mi {

namespace {

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// Load 4 consecutive channels [c, c+4) of pixel `pix` from the virtual concatenation
//   cat(src0[.., C0], src1[.., C1] * scale1)     (reference: torch.cat((x, skip * 2**-0.5), dim=1), Unet.py:445)
__device__ __forceinline__ float4 load_cat4(const float* __restrict__ src0, int C0, const float* __restrict__ src1,
                                             int C1, float scale1, long long pix, int c) {
    if (c < C0) return *reinterpret_cast<const float4*>(src0 + pix * C0 + c);
    float4 v = *reinterpret_cast<const float4*>(src1 + pix * C1 + (c - C0));
    v.x *= scale1; v.y *= scale1; v.z *= scale1; v.w *= scale1;
    return v;
}

// 8 consecutive channels [c, c+8) of the virtual concat, from fp32 or fp16 sources (C0 % 8 == 0 for fp16)
template <typename T>
__device__ __forceinline__ void load_cat8(const T* __restrict__ src0, int C0, const T* __restrict__ src1, int C1,
                                          float scale1, long long pix, int c, float (&v)[8]) {
    if constexpr (sizeof(T) == 4) {
        const float4 a = load_cat4(src0, C0, src1, C1, scale1, pix, c);
        const float4 d = load_cat4(src0, C0, src1, C1, scale1, pix, c + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = d.x; v[5] = d.y; v[6] = d.z; v[7] = d.w;
    } else {
        const bool first = c < C0;
        const uint4 raw = first ? *reinterpret_cast<const uint4*>(src0 + pix * C0 + c)
                                : *reinterpret_cast<const uint4*>(src1 + pix * C1 + (c - C0));
        const __half2* h = reinterpret_cast<const __half2*>(&raw);
        const float sc = first ? 1.0f : scale1;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 f = __half22float2(h[i]);
            v[2 * i] = f.x * sc;
            v[2 * i + 1] = f.y * sc;
        }
    }
}

__device__ __forceinline__ uint2 pack_half4(float a, float b, float c, float d) {
    __half2 lo = sat_half2(a, b), hi = sat_half2(c, d);
    uint2 r;
    r.x = *reinterpret_cast<uint32_t*>(&lo);
    r.y = *reinterpret_cast<uint32_t*>(&hi);
    return r;
}

// ------------------------------------------------------------------------------------------------ GroupNorm stats
// nn.GroupNorm(groups, C) statistics (layers.py:127): per (sample, group) sum and sum of squares over (C/groups)*H*W.
// grid = (ceil(HW / chunk), B) with chunk ~ 32K elements / C pixels, so small images still fill the GPU;
// sums[b][g][0..1] accumulated with double atomics (buffer pre-zeroed by the caller).

template <typename InT>
__global__ void __launch_bounds__(256)
gn_stats_kernel(const InT* __restrict__ src0, int C0, const InT* __restrict__ src1, int C1, float scale1, int HW,
                int groups, double* __restrict__ sums, int chunk) {
    pdl_wait();
    pdl_trigger();
    extern __shared__ double s_acc[];   // [groups][2]
    const int C = C0 + C1;
    const int V = C >> 3;               // 8-channel vectors
    const int Cg = C / groups;
    const int b = blockIdx.y;
    const int p0 = blockIdx.x * chunk;
    const int npix = min(chunk, HW - p0);
    for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) s_acc[i] = 0.0;
    __syncthreads();

    int cv0, plane, nplanes, cv_step;
    if (V <= (int)blockDim.x) {
        nplanes = blockDim.x / V; cv0 = threadIdx.x % V; plane = threadIdx.x / V; cv_step = V;
        if (plane >= nplanes) cv0 = V;   // inactive
    } else {
        nplanes = 1; cv0 = threadIdx.x; plane = 0; cv_step = blockDim.x;
    }
    const long long pix_base = (long long)b * HW + p0;
    for (int cv = cv0; cv < V; cv += cv_step) {
        const int c = cv << 3;
        float s[8], q[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) { s[e] = 0.f; q[e] = 0.f; }
        int p = plane;
        for (; p + nplanes < npix; p += 2 * nplanes) {         // two independent vector loads in flight
            float v0[8], v1[8];
            load_cat8<InT>(src0, C0, src1, C1, scale1, pix_base + p, c, v0);
            load_cat8<InT>(src0, C0, src1, C1, scale1, pix_base + p + nplanes, c, v1);
#pragma unroll
            for (int e = 0; e < 8; ++e) { s[e] += v0[e] + v1[e]; q[e] += v0[e] * v0[e] + v1[e] * v1[e]; }
        }
        for (; p < npix; p += nplanes) {
            float v0[8];
            load_cat8<InT>(src0, C0, src1, C1, scale1, pix_base + p, c, v0);
#pragma unroll
            for (int e = 0; e < 8; ++e) { s[e] += v0[e]; q[e] += v0[e] * v0[e]; }
        }
        const int g0 = c / Cg, g7 = (c + 7) / Cg;
        if (g0 == g7) {
            double ds = 0.0, dq = 0.0;
#pragma unroll
            for (int e = 0; e < 8; ++e) { ds += (double)s[e]; dq += (double)q[e]; }
            atomicAdd(&s_acc[2 * g0], ds);
            atomicAdd(&s_acc[2 * g0 + 1], dq);
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const int g = (c + e) / Cg;
                atomicAdd(&s_acc[2 * g], (double)s[e]);
                atomicAdd(&s_acc[2 * g + 1], (double)q[e]);
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) atomicAdd(&sums[(long long)b * groups * 2 + i], s_acc[i]);
}

// ------------------------------------------------------------------------------------------------ GroupNorm apply
// Block.forward (layers.py:138-144): y = SiLU( GN(x) * (scale + 1) + shift ), written as the conv's fp16 operand
// (tensor-core path) or fp32 (small-channel path).
// HBM-bound (4 B read + 2 B written per element).  Each CTA first folds GroupNorm, its affine and the FiLM
// (scale, shift) into ONE per-channel multiply-add   y = x * A[c] + Bc[c]   kept in shared memory (cost C, amortised
// over kGnApplyPix * C elements), so the streaming loop is 2 x LDG.128 + 4 x LDS.128 + 8 FMA + 8 SiLU + 1 x STG.128.
// grid = (ceil(HW / pix_per_cta), B)
constexpr int kGnSlab = 256;      // channels per CTA of gn_apply_silu_kernel (a multiple of 8)

template <typename InT, typename OutT, bool kFast>
__global__ void __launch_bounds__(256)
gn_apply_silu_kernel(const InT* __restrict__ src0, int C0, const InT* __restrict__ src1, int C1, float scale1,
                     int HW, int groups, const double* __restrict__ stats0, int sb0, const double* __restrict__ stats1,
                     int sb1, const float* __restrict__ gamma, const float* __restrict__ beta,
                     const float* __restrict__ scale_shift, int ss_ld, float eps, OutT* __restrict__ out,
                     int pix_per_cta) {
    pdl_wait();
    pdl_trigger();
    extern __shared__ float s_ab[];   // A[C], Bc[C]
    __shared__ float s_mean[32], s_rstd[32];
    const int C = C0 + C1;
    const int Cg = C / groups;
    const int b = blockIdx.y;
    if (threadIdx.x < groups) {
        const int g = threadIdx.x;
        double su = 0.0, sq = 0.0;
        if (sb0 == 0) {
            // statistics were reduced per (image, group) over the whole virtual concat (mi_gn_stats)
            su = stats0[((long long)b * groups + g) * 2];
            sq = stats0[((long long)b * groups + g) * 2 + 1];
        } else {
            // per-source block statistics written by the producing conv epilogues: gather the blocks of this group
            const int lo = g * Cg, hi = lo + Cg;
            const int lo0 = min(lo, C0), hi0 = min(hi, C0);
            for (int e = lo0 / sb0; e < hi0 / sb0; ++e) {
                su += stats0[((long long)b * (C0 / sb0) + e) * 2];
                sq += stats0[((long long)b * (C0 / sb0) + e) * 2 + 1];
            }
            const int lo1 = max(lo, C0) - C0, hi1 = max(hi, C0) - C0;
            for (int e = lo1 / max(sb1, 1); e < hi1 / max(sb1, 1); ++e) {
                su += (double)scale1 * stats1[((long long)b * (C1 / sb1) + e) * 2];
                sq += (double)scale1 * (double)scale1 * stats1[((long long)b * (C1 / sb1) + e) * 2 + 1];
            }
        }
        const double n = (double)Cg * HW;
        const double mean = su / n;
        double var = sq / n - mean * mean;
        if (var < 0) var = 0;
        s_mean[g] = (float)mean;
        s_rstd[g] = (float)(1.0 / sqrt(var + (double)eps));
    }
    __syncthreads();
    // this CTA's channel slab [c_lo, c_lo + slab): only its coefficients are built (at C = 1024..4096 a CTA that covered all
    // channels of a few pixels spent as long on the table as on the data)
    const int slab = min(C, kGnSlab);
    const int c_lo = blockIdx.z * slab;
    const int c_n = min(slab, C - c_lo);
    float* sA = s_ab;
    float* sB = s_ab + slab;
    for (int cl = threadIdx.x; cl < c_n; cl += blockDim.x) {
        const int ch = c_lo + cl;
        const int g = ch / Cg;
        float a = s_rstd[g] * gamma[ch];
        float bb = beta[ch] - s_mean[g] * a;
        if (scale_shift) {
            const float sc = scale_shift[(long long)b * ss_ld + ch] + 1.0f;
            const float sh = scale_shift[(long long)b * ss_ld + C + ch];
            a *= sc;
            bb = bb * sc + sh;
        }
        sA[cl] = a;
        sB[cl] = bb;
    }
    __syncthreads();
    const int V8 = c_n >> 3;
    const int p0 = blockIdx.x * pix_per_cta;
    const int npix = min(pix_per_cta, HW - p0);
    const int total = npix * V8;
    const long long pix_base = (long long)b * HW + p0;
    auto one = [&](int idx, const float (&v_in)[8]) {
        const int cl = (idx % V8) << 3;
        const long long pix = pix_base + idx / V8;
        float v[8];
        const float4 a0 = *reinterpret_cast<const float4*>(sA + cl), a1 = *reinterpret_cast<const float4*>(sA + cl + 4);
        const float4 b0 = *reinterpret_cast<const float4*>(sB + cl), b1 = *reinterpret_cast<const float4*>(sB + cl + 4);
        v[0] = fmaf(v_in[0], a0.x, b0.x); v[1] = fmaf(v_in[1], a0.y, b0.y); v[2] = fmaf(v_in[2], a0.z, b0.z); v[3] = fmaf(v_in[3], a0.w, b0.w);
        v[4] = fmaf(v_in[4], a1.x, b1.x); v[5] = fmaf(v_in[5], a1.y, b1.y); v[6] = fmaf(v_in[6], a1.z, b1.z); v[7] = fmaf(v_in[7], a1.w, b1.w);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            if constexpr (kFast) v[e] = __fdividef(v[e], 1.0f + __expf(-v[e]));
            else v[e] = silu_f(v[e]);
        }
        const int c = c_lo + cl;
        if constexpr (sizeof(OutT) == 2) {
            const uint2 lo = pack_half4(v[0], v[1], v[2], v[3]), hi = pack_half4(v[4], v[5], v[6], v[7]);
            *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(out) + pix * C + c) = make_uint4(lo.x, lo.y, hi.x, hi.y);
        } else {
            float* o = reinterpret_cast<float*>(out) + pix * C + c;
            *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
            *reinterpret_cast<float4*>(o + 4) = make_float4(v[4], v[5], v[6], v[7]);
        }
    };
    // two independent items per iteration: both loads are in flight before either is consumed
    int idx = threadIdx.x;
    for (; idx + (int)blockDim.x < total; idx += 2 * blockDim.x) {
        const int i1 = idx + blockDim.x;
        float x0[8], x1[8];
        load_cat8<InT>(src0, C0, src1, C1, scale1, pix_base + idx / V8, c_lo + ((idx % V8) << 3), x0);
        load_cat8<InT>(src0, C0, src1, C1, scale1, pix_base + i1 / V8, c_lo + ((i1 % V8) << 3), x1);
        one(idx, x0);
        one(i1, x1);
    }
    if (idx < total) {
        float x0[8];
        load_cat8<InT>(src0, C0, src1, C1, scale1, pix_base + idx / V8, c_lo + ((idx % V8) << 3), x0);
        one(idx, x0);
    }
}

// ------------------------------------------------------------------------------------------------ cast / resample
// Raw (un-normalised) conv operands: res_conv input (layers.py:439), Downsample input (layers.py:319, stride 2 ->
// phase split), Upsample input (layers.py:513 nn.Upsample(nearest, x2)), with the skip concat folded in.
//   mode 0: out[b][h][w][c]                     = in[b][h][w][c]
//   mode 1: out[b][2h+i][2w+j][c]               = in[b][h][w][c]                  (nearest x2)
//   mode 2: out[b][(h&1)*2+(w&1)][h/2][w/2][c]  = in[b][h][w][c]                  (phase split for 4x4 s2 convs)
template <typename InT, typename OutT>
__global__ void __launch_bounds__(256)
cast_kernel(const InT* __restrict__ src0, int C0, const InT* __restrict__ src1, int C1, float scale1, int B, int H,
            int W, int mode, OutT* __restrict__ out) {
    pdl_wait();
    pdl_trigger();
    const int C = C0 + C1;
    const int V8 = C >> 3;
    const long long total = (long long)B * H * W * V8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int c = (int)(idx % V8) << 3;
    const long long pix = idx / V8;
    float v8[8];
    load_cat8<InT>(src0, C0, src1, C1, scale1, pix, c, v8);
    const float4 a = make_float4(v8[0], v8[1], v8[2], v8[3]);
    const float4 d = make_float4(v8[4], v8[5], v8[6], v8[7]);
    const int w = (int)(pix % W);
    const int h = (int)((pix / W) % H);
    const long long b = pix / ((long long)W * H);
    long long opix[4];
    int nout = 1;
    if (mode == 0) {
        opix[0] = pix;
    } else if (mode == 1) {
        nout = 4;
        const long long base = (b * 2 * H + 2 * h) * (2LL * W) + 2 * w;
        opix[0] = base; opix[1] = base + 1; opix[2] = base + 2LL * W; opix[3] = base + 2LL * W + 1;
    } else {
        const int p = (h & 1) * 2 + (w & 1);
        opix[0] = ((b * 4 + p) * (H >> 1) + (h >> 1)) * (long long)(W >> 1) + (w >> 1);
    }
    for (int i = 0; i < nout; ++i) {
        if constexpr (sizeof(OutT) == 2) {
            const uint2 lo = pack_half4(a.x, a.y, a.z, a.w), hi = pack_half4(d.x, d.y, d.z, d.w);
            *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(out) + opix[i] * C + c) = make_uint4(lo.x, lo.y, hi.x, hi.y);
        } else {
            float* o = reinterpret_cast<float*>(out) + opix[i] * C + c;
            *reinterpret_cast<float4*>(o) = a;
            *reinterpret_cast<float4*>(o + 4) = d;
        }
    }
}

// ------------------------------------------------------------------------------------------------ row LayerNorm
// F.layer_norm over the last dim (layers.py:342 LayerNorm; layers.py:174-177 ChanLayerNorm == per-pixel LN in NHWC;
// Unet.py:142 nn.LayerNorm).  Optional exact-erf GELU applied to the input first (ChanFeedForward, layers.py:158-159),
// optional residual added after (x = attn(x) + x, layers.py:435/:497).  One warp per row, two-pass variance.
__global__ void __launch_bounds__(256)
ln_rows_kernel(const float* __restrict__ in, long long R, int C, const float* __restrict__ gamma,
               const float* __restrict__ beta, float eps, int pre_gelu, const float* __restrict__ residual,
               float* __restrict__ out_f32, __half* __restrict__ out_f16) {
    pdl_wait();
    pdl_trigger();
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= R) return;
    const int lane = threadIdx.x & 31;
    const float* x = in + row * C;
    float s = 0.f;
    for (int c = lane * 4; c < C; c += 128) {
        float4 v = *reinterpret_cast<const float4*>(x + c);
        if (pre_gelu) { v.x = gelu_erf_f(v.x); v.y = gelu_erf_f(v.y); v.z = gelu_erf_f(v.z); v.w = gelu_erf_f(v.w); }
        s += (v.x + v.y) + (v.z + v.w);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)C;
    float q = 0.f;
    for (int c = lane * 4; c < C; c += 128) {
        float4 v = *reinterpret_cast<const float4*>(x + c);
        if (pre_gelu) { v.x = gelu_erf_f(v.x); v.y = gelu_erf_f(v.y); v.z = gelu_erf_f(v.z); v.w = gelu_erf_f(v.w); }
        const float a = v.x - mean, b2 = v.y - mean, c2 = v.z - mean, d = v.w - mean;
        q += (a * a + b2 * b2) + (c2 * c2 + d * d);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q / (float)C + eps);
    for (int c = lane * 4; c < C; c += 128) {
        float4 v = *reinterpret_cast<const float4*>(x + c);
        if (pre_gelu) { v.x = gelu_erf_f(v.x); v.y = gelu_erf_f(v.y); v.z = gelu_erf_f(v.z); v.w = gelu_erf_f(v.w); }
        const float4 g = *reinterpret_cast<const float4*>(gamma + c);
        float4 y;
        y.x = (v.x - mean) * rstd * g.x; y.y = (v.y - mean) * rstd * g.y;
        y.z = (v.z - mean) * rstd * g.z; y.w = (v.w - mean) * rstd * g.w;
        if (beta) {
            const float4 bt = *reinterpret_cast<const float4*>(beta + c);
            y.x += bt.x; y.y += bt.y; y.z += bt.z; y.w += bt.w;
        }
        if (residual) {
            const float4 r = *reinterpret_cast<const float4*>(residual + row * C + c);
            y.x += r.x; y.y += r.y; y.z += r.z; y.w += r.w;
        }
        if (out_f32) *reinterpret_cast<float4*>(out_f32 + row * C + c) = y;
        if (out_f16) *reinterpret_cast<uint2*>(out_f16 + row * C + c) = pack_half4(y.x, y.y, y.z, y.w);
    }
}

// The same for C = 128 * NV (NV = 1, 2, 4, 8: every LayerNorm of the U-Nets): the row lives in registers -- ONE global read
// instead of three -- and a warp works on ROWS rows at a time so that several rows' loads are in flight (the three-pass kernel
// above ran at ~2 TB/s: one 512-byte row per warp, three dependent load -> shuffle-reduce phases).  Same summation order, so
// the results are bit-identical to ln_rows_kernel.
template <int NV, int ROWS>
__global__ void __launch_bounds__(256)
ln_rows_reg_kernel(const float* __restrict__ in, long long R, const float* __restrict__ gamma, const float* __restrict__ beta,
                   float eps, int pre_gelu, const float* __restrict__ residual, float* __restrict__ out_f32,
                   __half* __restrict__ out_f16) {
    pdl_wait();
    pdl_trigger();
    constexpr int C = 128 * NV;
    const int lane = threadIdx.x & 31;
    const long long row0 = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * ROWS;
    if (row0 >= R) return;
    float4 v[ROWS][NV];
#pragma unroll
    for (int r = 0; r < ROWS; ++r)
#pragma unroll
        for (int k = 0; k < NV; ++k)
            v[r][k] = row0 + r < R ? *reinterpret_cast<const float4*>(in + (row0 + r) * C + lane * 4 + 128 * k)
                                   : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 g[NV], bt[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        g[k] = *reinterpret_cast<const float4*>(gamma + lane * 4 + 128 * k);
        bt[k] = beta ? *reinterpret_cast<const float4*>(beta + lane * 4 + 128 * k) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float mean[ROWS], rstd[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            float4& x = v[r][k];
            if (pre_gelu) { x.x = gelu_erf_f(x.x); x.y = gelu_erf_f(x.y); x.z = gelu_erf_f(x.z); x.w = gelu_erf_f(x.w); }
            s += (x.x + x.y) + (x.z + x.w);
        }
        mean[r] = s;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int r = 0; r < ROWS; ++r) mean[r] += __shfl_xor_sync(0xffffffffu, mean[r], o);
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        mean[r] /= (float)C;
        float q = 0.f;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const float a = v[r][k].x - mean[r], b2 = v[r][k].y - mean[r], c2 = v[r][k].z - mean[r], d = v[r][k].w - mean[r];
            q += (a * a + b2 * b2) + (c2 * c2 + d * d);
        }
        rstd[r] = q;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int r = 0; r < ROWS; ++r) rstd[r] += __shfl_xor_sync(0xffffffffu, rstd[r], o);
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        if (row0 + r >= R) break;
        const float rs = rsqrtf(rstd[r] / (float)C + eps);
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const long long off = (row0 + r) * C + lane * 4 + 128 * k;
            float4 y;
            y.x = (v[r][k].x - mean[r]) * rs * g[k].x; y.y = (v[r][k].y - mean[r]) * rs * g[k].y;
            y.z = (v[r][k].z - mean[r]) * rs * g[k].z; y.w = (v[r][k].w - mean[r]) * rs * g[k].w;
            if (beta) { y.x += bt[k].x; y.y += bt[k].y; y.z += bt[k].z; y.w += bt[k].w; }
            if (residual) {
                const float4 rr = *reinterpret_cast<const float4*>(residual + off);
                y.x += rr.x; y.y += rr.y; y.z += rr.z; y.w += rr.w;
            }
            if (out_f32) *reinterpret_cast<float4*>(out_f32 + off) = y;
            if (out_f16) *reinterpret_cast<uint2*>(out_f16 + off) = pack_half4(y.x, y.y, y.z, y.w);
        }
    }
}

// ------------------------------------------------------------------------------------------------ small fp32 linear
// out[M][N] = act_out( act_in(in)[M][K] @ W[N][K]^T + bias + addend ).  For the conditioning MLPs (M = batch rows;
// Unet.py:101-161, layers.py:396-399) and for projections whose K/N are not tensor-core shaped (tiny config).
// One warp per (8-row tile, output column); lanes split K.
template <int kLinRows>
__global__ void __launch_bounds__(256)
linear_f32_kernel(const float* __restrict__ in, int M, int K, const float* __restrict__ W, const float* __restrict__ bias,
                  int N, int in_act, int out_act, const float* __restrict__ addend, float* __restrict__ out_f32,
                  __half* __restrict__ out_f16, float out_scale) {
    pdl_wait();
    pdl_trigger();
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int m0 = blockIdx.y * kLinRows;
    if (n >= N) return;
    const int lane = threadIdx.x & 31;
    const int rows = min(kLinRows, M - m0);
    float acc[kLinRows];
#pragma unroll
    for (int r = 0; r < kLinRows; ++r) acc[r] = 0.f;
    const float* w = W + (long long)n * K;
    for (int k = lane * 4; k < K; k += 128) {
        const float4 wv = *reinterpret_cast<const float4*>(w + k);
#pragma unroll
        for (int r = 0; r < kLinRows; ++r) {
            if (r < rows) {
                float4 xv = *reinterpret_cast<const float4*>(in + (long long)(m0 + r) * K + k);
                if (in_act == 1) { xv.x = silu_f(xv.x); xv.y = silu_f(xv.y); xv.z = silu_f(xv.z); xv.w = silu_f(xv.w); }
                acc[r] += xv.x * wv.x + xv.y * wv.y + xv.z * wv.z + xv.w * wv.w;
            }
        }
    }
#pragma unroll
    for (int r = 0; r < kLinRows; ++r) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
    }
    if (lane == 0) {
        const float bv = bias ? bias[n] : 0.f;
        for (int r = 0; r < rows; ++r) {
            float y = acc[r] + bv;
            const long long oi = (long long)(m0 + r) * N + n;
            if (addend) y += addend[oi];
            if (out_act == 1) y = silu_f(y);
            y *= out_scale;
            if (out_f32) out_f32[oi] = y;
            if (out_f16) out_f16[oi] = sat_half(y);
        }
    }
}

// Shared-memory tiled variant for M > 8 (the batched time-MLP GEMM: 32 rows x ~66K columns x K = 1024, i.e. a 270 MB
// weight stream that must be read exactly once).  CTA tile = 32 rows x 128 columns, K chunks of 32; thread (ty, tx)
// owns rows 4*ty..4*ty+3 and columns tx, tx+32, tx+64, tx+96.
constexpr int kTM = 32, kTN = 128, kTK = 32;

__global__ void __launch_bounds__(256)
linear_tiled_kernel(const float* __restrict__ in, int M, int K, const float* __restrict__ W, const float* __restrict__ bias,
                    int N, int in_act, int out_act, const float* __restrict__ addend, float* __restrict__ out_f32,
                    __half* __restrict__ out_f16, float out_scale) {
    pdl_wait();
    pdl_trigger();
    __shared__ __align__(16) float xs[kTK][kTM + 4];      // [k][row]
    __shared__ float ws[kTK][kTN + 1];                    // [k][col], +1: conflict-free transposed stores
    const int n0 = blockIdx.x * kTN, m0 = blockIdx.y * kTM;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    // software pipeline: the next chunk's global loads are issued before the current chunk's FMAs
    const int xrow = threadIdx.x >> 3, kq = (threadIdx.x & 7) * 4;
    float4 xr, wr[4];
    auto fetch = [&](int k0) {
        xr = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m0 + xrow < M && k0 + kq < K) xr = *reinterpret_cast<const float4*>(in + (long long)(m0 + xrow) * K + k0 + kq);
#pragma unroll
        for (int pass = 0; pass < 4; ++pass) {   // w chunk: 128 cols x 32 k, 8 threads (128 B) per column
            const int col = pass * 32 + (threadIdx.x >> 3);
            wr[pass] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (n0 + col < N && k0 + kq < K)
                wr[pass] = __ldg(reinterpret_cast<const float4*>(W + (long long)(n0 + col) * K + k0 + kq));
        }
    };
    fetch(0);
    for (int k0 = 0; k0 < K; k0 += kTK) {
        {
            float4 v = xr;
            if (in_act == 1) { v.x = silu_f(v.x); v.y = silu_f(v.y); v.z = silu_f(v.z); v.w = silu_f(v.w); }
            xs[kq][xrow] = v.x; xs[kq + 1][xrow] = v.y; xs[kq + 2][xrow] = v.z; xs[kq + 3][xrow] = v.w;
        }
#pragma unroll
        for (int pass = 0; pass < 4; ++pass) {
            const int col = pass * 32 + (threadIdx.x >> 3);
            ws[kq][col] = wr[pass].x; ws[kq + 1][col] = wr[pass].y; ws[kq + 2][col] = wr[pass].z; ws[kq + 3][col] = wr[pass].w;
        }
        __syncthreads();
        if (k0 + kTK < K) fetch(k0 + kTK);
#pragma unroll
        for (int k = 0; k < kTK; ++k) {
            const float4 a = *reinterpret_cast<const float4*>(&xs[k][ty * 4]);
            const float b0 = ws[k][tx], b1 = ws[k][tx + 32], b2 = ws[k][tx + 64], b3 = ws[k][tx + 96];
            acc[0][0] += a.x * b0; acc[0][1] += a.x * b1; acc[0][2] += a.x * b2; acc[0][3] += a.x * b3;
            acc[1][0] += a.y * b0; acc[1][1] += a.y * b1; acc[1][2] += a.y * b2; acc[1][3] += a.y * b3;
            acc[2][0] += a.z * b0; acc[2][1] += a.z * b1; acc[2][2] += a.z * b2; acc[2][3] += a.z * b3;
            acc[3][0] += a.w * b0; acc[3][1] += a.w * b1; acc[3][2] += a.w * b2; acc[3][3] += a.w * b3;
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx + 32 * j;
            if (n >= N) continue;
            const long long oi = (long long)m * N + n;
            float y = acc[i][j] + (bias ? bias[n] : 0.f);
            if (addend) y += addend[oi];
            if (out_act == 1) y = silu_f(y);
            y *= out_scale;
            if (out_f32) out_f32[oi] = y;
            if (out_f16) out_f16[oi] = sat_half(y);
        }
    }
}

// ------------------------------------------------------------------------------------------------ conditioning bits
// SinusoidalPosEmb.forward (layers.py:461-465): emb_j = exp(j * -(ln(1e4)/(half-1))) in fp32, arg = float(t) * emb_j,
// out = cat(sin(arg), cos(arg)).
__global__ void posemb_kernel(const long long* __restrict__ t, int B, int dim, float neg_log_step,
                              float* __restrict__ out) {
    pdl_wait();
    pdl_trigger();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int half = dim >> 1;
    if (i >= B * half) return;
    const int b = i / half, j = i % half;
    const float f = expf((float)j * neg_log_step);
    const float arg = (float)t[b] * f;
    out[(long long)b * dim + j] = sinf(arg);
    out[(long long)b * dim + half + j] = cosf(arg);
}

// Unet._text_condition (Unet.py:578-610): pad/truncate projected text tokens to 256 rows, substitute the learned null
// embedding where (text_mask & keep) is false, write them below the time tokens of the conditioning sequence, and
// mean-pool the 256 rows.   grid = B, block = min(D, 256)
__global__ void text_tokens_kernel(const float* __restrict__ proj /*[B][L][D]*/, int L, int D,
                                   const uint8_t* __restrict__ mask /*[B][L] or null*/,
                                   const uint8_t* __restrict__ keep /*[B]*/, const float* __restrict__ null_embed,
                                   int max_len, float* __restrict__ c_out /*[B][m][D]*/, int m, int row_off,
                                   float* __restrict__ pooled /*[B][D]*/) {
    pdl_wait();
    pdl_trigger();
    const int b = blockIdx.x;
    const bool kp = keep[b] != 0;
    const int Lc = min(L, max_len);
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
        float s = 0.f;
        for (int l = 0; l < max_len; ++l) {
            const float v = (l < Lc) ? proj[((long long)b * L + l) * D + d] : 0.f;
            bool cond = kp;
            if (mask) cond = cond && (l < Lc) && (mask[(long long)b * L + l] != 0);
            const float o = cond ? v : null_embed[(long long)l * D + d];
            c_out[((long long)b * m + row_off + l) * D + d] = o;
            s += o;
        }
        pooled[(long long)b * D + d] = s / (float)max_len;
    }
}

// copy rows [B][r][D] into the conditioning sequence [B][m][D] at row offset (time tokens, Unet.py:534/:629)
__global__ void place_rows_kernel(const float* __restrict__ src, int B, int r, int D, float* __restrict__ dst, int m,
                                  int row_off) {
    pdl_wait();
    pdl_trigger();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * r * D) return;
    const int d = (int)(i % D);
    const int rr = (int)((i / D) % r);
    const long long b = i / ((long long)D * r);
    dst[(b * m + row_off + rr) * D + d] = src[i];
}

// where(keep[b], a[b][:], null[:]) (+ addend) -- Unet.py:619-626
__global__ void select_rows_kernel(const float* __restrict__ a, const float* __restrict__ nullv,
                                   const uint8_t* __restrict__ keep, const float* __restrict__ addend, int B, int N,
                                   float* __restrict__ out) {
    pdl_wait();
    pdl_trigger();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * N) return;
    const int n = (int)(i % N);
    const long long b = i / N;
    float v = keep[b] ? a[i] : nullv[n];
    if (addend) v += addend[i];
    out[i] = v;
}

// NCHW fp32 (two sources, e.g. x and lowres_cond_img: torch.cat(dim=1), Unet.py:397) -> NHWC fp32 with C padded to Cp
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ a, int Ca, const float* __restrict__ b2, int Cb, int B,
                                    int HW, int Cp, float* __restrict__ out) {
    pdl_wait();
    pdl_trigger();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * HW * Cp) return;
    const int c = (int)(i % Cp);
    const long long pix = i / Cp;
    const long long b = pix / HW, p = pix % HW;
    float v = 0.f;
    if (c < Ca) v = a[(b * Ca + c) * HW + p];
    else if (c < Ca + Cb) v = b2[(b * Cb + (c - Ca)) * HW + p];
    out[i] = v;
}

// weight packing: OIHW fp32 -> [O][(r*KW+s)*I + c] fp16 (* scale)  (one-time, on load_state_dict)
__global__ void pack_conv_weight_kernel(const float* __restrict__ w, int O, int I, int KH, int KW, float scale,
                                        __half* __restrict__ out) {
    pdl_wait();
    pdl_trigger();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)O * I * KH * KW;
    if (i >= total) return;
    const int c = (int)(i % I);
    const int t = (int)((i / I) % (KH * KW));
    const long long o = i / ((long long)I * KH * KW);
    out[i] = __float2half_rn(w[((o * I + c) * KH + t / KW) * KW + t % KW] * scale);
}

// The same weight packed for the DATA gradient of a stride-1 'same' conv / a linear layer: the conv of dy with the taps flipped
// and in / out channels swapped, out[i][((KH-1-r)*KW + (KW-1-s))*O + o] = w[o][i][r][s]  (one kernel instead of flip + transpose +
// copy + pack in the training step).
__global__ void pack_conv_weight_dgrad_kernel(const float* __restrict__ w, int O, int I, int KH, int KW, __half* __restrict__ out) {
    pdl_wait();
    pdl_trigger();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int taps = KH * KW;
    const long long total = (long long)O * I * taps;
    if (idx >= total) return;
    const int o = (int)(idx % O);
    const int t = (int)((idx / O) % taps);
    const long long i = idx / ((long long)O * taps);
    const int r = KH - 1 - t / KW, s = KW - 1 - t % KW;
    out[idx] = __float2half_rn(w[(((long long)o * I + i) * KH + r) * KW + s]);
}

// Stem operand for the tensor-core path of CrossEmbedLayer (layers.py:294-305, kernels 3/7/15, stride 1):
// horizontally unrolled window  out[b][h][w][j*8 + c] = in_c[b][h][w + j - 7]  (j < 15, c < Ca+Cb <= 8, else 0), fp16.
// With it the k x k convs (all zero-embedded in one 15 x 15 window) become a 15-tap (vertical) implicit GEMM over
// 128 "channels": K = 15 * 128, N = dim.  Inputs are the NCHW fp32 images x and lowres_cond_img (torch.cat, Unet.py:397).
// One CTA = kStemRows image rows x 64 columns: the 6 (<= 8) input channels of the (64 + 14)-pixel source window are read
// once (coalesced per channel), packed to one 16-byte fp16 pixel each in shared memory, and the 16 x replicated
// operand rows go out as consecutive 16-byte stores (LDS.128 + STG.128 per thread, 100 % write-coalesced).
constexpr int kStemRows = 4, kStemCols = 64, kStemWin = kStemCols + 14;
__global__ void __launch_bounds__(256)
stem_unroll_kernel(const float* __restrict__ a, int Ca, const float* __restrict__ b2, int Cb, int B, int H, int W,
                   __half* __restrict__ out) {
    pdl_wait();
    pdl_trigger();
    __shared__ uint4 s_px[kStemRows][kStemWin + 2];
    const int w0 = blockIdx.x * kStemCols;
    const int h0 = blockIdx.y * kStemRows;
    const long long b = blockIdx.z;
    for (int i = threadIdx.x; i < kStemRows * kStemWin; i += blockDim.x) {
        const int r = i / kStemWin, t = i - r * kStemWin;
        const int h = h0 + r, ws = w0 + t - 7;
        __half v[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            float f = 0.f;
            if (h < H && ws >= 0 && ws < W) {
                if (c < Ca) f = a[((b * Ca + c) * H + h) * W + ws];
                else if (c < Ca + Cb) f = b2[((b * Cb + (c - Ca)) * H + h) * W + ws];
            }
            v[c] = sat_half(f);
        }
        s_px[r][t] = *reinterpret_cast<const uint4*>(v);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kStemRows * kStemCols * 16; i += blockDim.x) {
        const int j = i & 15;
        const int p = (i >> 4) & (kStemCols - 1);
        const int r = i >> 10;                         // / (16 * kStemCols)
        const int h = h0 + r, w = w0 + p;
        if (h >= H || w >= W) continue;
        const uint4 v = j < 15 ? s_px[r][p + j] : make_uint4(0u, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(out + (((b * H + h) * W + w) * 16 + j) * 8) = v;
    }
}

// Inter-stage resize of the cascade (helpers.py:138-164 -> resize_right.resize, SURVEY.md 8f-1): separable resampling
// with per-output-coordinate tap tables (indices already reflected / clamped, weights already normalised -- built by the
// host, minimagen_b200/helpers.py).  Rows first, then columns, like the two-pass reference:
//   out[b][c][y][x] = clamp( sum_j wx[x][j] * ( sum_i wy[y][i] * in[b][c][iy[y][i]][ix[x][j]] ) )
__global__ void __launch_bounds__(256)
resize_sep_kernel(const float* __restrict__ in, int Hin, int Win, float* __restrict__ out, int Hout, int Wout,
                  const int* __restrict__ iy, const float* __restrict__ wy, int ty, const int* __restrict__ ix,
                  const float* __restrict__ wx, int tx, int has_clamp, float lo, float hi, long long total) {
    pdl_wait();
    pdl_trigger();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int x = (int)(idx % Wout);
    const int y = (int)((idx / Wout) % Hout);
    const long long plane = idx / ((long long)Wout * Hout);
    const float* src = in + plane * (long long)Hin * Win;
    float acc = 0.f;
    for (int j = 0; j < tx; ++j) {
        const int xi = ix[x * tx + j];
        float col = 0.f;
        for (int i = 0; i < ty; ++i) col = __fadd_rn(col, __fmul_rn(wy[y * ty + i], src[(long long)iy[y * ty + i] * Win + xi]));
        acc = __fadd_rn(acc, __fmul_rn(wx[x * tx + j], col));
    }
    if (has_clamp) acc = clamp_nan(acc, lo, hi);      // a NaN stays NaN, as torch.clamp
    out[idx] = acc;
}

__global__ void silu_kernel(const float* __restrict__ in, long long n, float* __restrict__ out) {
    pdl_wait();
    pdl_trigger();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = silu_f(in[i]);
}

inline unsigned grid1d(long long total, int block) { return (unsigned)((total + block - 1) / block); }

}  // namespace

// ================================================================================================ launchers
int gn_stats(const void* src0, int C0, const void* src1, int C1, float scale1, int in_is_f16, int B, int HW, int groups,
             double* sums, cudaStream_t st) {
    const int C = C0 + C1;
    if (C % 8 || C0 % 4 || groups < 1 || groups > 256 || C % groups) return -1;
    if (in_is_f16 && (C0 % 8)) return -1;
    int chunk = 32768 / C;
    if (chunk < 4) chunk = 4;
    if (chunk > HW) chunk = HW;
    dim3 grid((HW + chunk - 1) / chunk, B);
    const size_t smem = 2 * groups * sizeof(double);
    if (in_is_f16)
        launch_k(gn_stats_kernel<__half>, grid, 256, smem, st, (const __half*)src0, C0, (const __half*)src1, C1, scale1, HW,
                                                         groups, sums, chunk);
    else
        launch_k(gn_stats_kernel<float>, grid, 256, smem, st, (const float*)src0, C0, (const float*)src1, C1, scale1, HW,
                                                        groups, sums, chunk);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int gn_apply_silu(const void* src0, int C0, const void* src1, int C1, float scale1, int in_is_f16, int B, int HW,
                  int groups, const double* stats0, int sb0, const double* stats1, int sb1, const float* gamma,
                  const float* beta, const float* scale_shift, int ss_ld, float eps, void* out, int out_is_f16,
                  cudaStream_t st) {
    const int C = C0 + C1;
    if (C % 8 || C0 % 4 || groups > 32 || C % groups) return -1;
    if (in_is_f16 && (C0 % 8)) return -1;
    if (scale_shift && ss_ld < 2 * C) return -1;
    const int Cg = C / groups;
    if (sb0 > 0) {   // block statistics: every group boundary must fall on block boundaries of the source it lies in
        if (C0 % sb0 || Cg % sb0 || (C1 && (sb1 <= 0 || C1 % sb1 || Cg % sb1 || !stats1))) return -1;
        if (C1 && (C0 % sb1)) return -1;
    }
    const int slab = C < kGnSlab ? C : kGnSlab;              // channels per CTA (grid.z walks the slabs)
    int pix = 16384 / slab;            // ~16K elements per CTA (8K / 32K / 64K measured slower, tools/bench_ops.py gn)
    if (pix < 1) pix = 1;
    if (pix > HW) pix = HW;
    const size_t smem = 2 * (size_t)slab * sizeof(float);
    dim3 grid((HW + pix - 1) / pix, B, (C + slab - 1) / slab);
#define MI_GN_LAUNCH(IN, OUT, FAST)                                                                                 \
    launch_k(gn_apply_silu_kernel<IN, OUT, FAST>, grid, 256, smem, st, (const IN*)src0, C0, (const IN*)src1, C1, scale1, HW, \
                                                                 groups, stats0, sb0, stats1, sb1, gamma, beta,      \
                                                                 scale_shift, ss_ld, eps, (OUT*)out, pix)
    if (in_is_f16) {
        if (out_is_f16) MI_GN_LAUNCH(__half, __half, true); else MI_GN_LAUNCH(__half, float, false);
    } else {
        if (out_is_f16) MI_GN_LAUNCH(float, __half, true); else MI_GN_LAUNCH(float, float, false);
    }
#undef MI_GN_LAUNCH
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int cast_act(const void* src0, int C0, const void* src1, int C1, float scale1, int in_is_f16, int B, int H, int W,
             int mode, void* out, int out_is_f16, cudaStream_t st) {
    const int C = C0 + C1;
    if (C % 8 || C0 % 4 || mode < 0 || mode > 2) return -1;
    if (in_is_f16 && (C0 % 8)) return -1;
    if (mode == 2 && ((H | W) & 1)) return -1;
    const unsigned grid = grid1d((long long)B * H * W * (C / 8), 256);
    if (in_is_f16) {
        if (out_is_f16) launch_k(cast_kernel<__half, __half>, grid, 256, 0, st, (const __half*)src0, C0, (const __half*)src1, C1, scale1, B, H, W, mode, (__half*)out);
        else launch_k(cast_kernel<__half, float>, grid, 256, 0, st, (const __half*)src0, C0, (const __half*)src1, C1, scale1, B, H, W, mode, (float*)out);
    } else {
        if (out_is_f16) launch_k(cast_kernel<float, __half>, grid, 256, 0, st, (const float*)src0, C0, (const float*)src1, C1, scale1, B, H, W, mode, (__half*)out);
        else launch_k(cast_kernel<float, float>, grid, 256, 0, st, (const float*)src0, C0, (const float*)src1, C1, scale1, B, H, W, mode, (float*)out);
    }
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int ln_rows(const float* in, long long R, int C, const float* gamma, const float* beta, float eps, int pre_gelu,
            const float* residual, float* out_f32, __half* out_f16, cudaStream_t st) {
    if (C % 4) return -1;
    if (C == 128) launch_k(ln_rows_reg_kernel<1, 4>, grid1d(R, 32), 256, 0, st, in, R, gamma, beta, eps, pre_gelu, residual, out_f32, out_f16);
    else if (C == 256) launch_k(ln_rows_reg_kernel<2, 2>, grid1d(R, 16), 256, 0, st, in, R, gamma, beta, eps, pre_gelu, residual, out_f32, out_f16);
    else if (C == 512) launch_k(ln_rows_reg_kernel<4, 1>, grid1d(R, 8), 256, 0, st, in, R, gamma, beta, eps, pre_gelu, residual, out_f32, out_f16);
    else if (C == 1024) launch_k(ln_rows_reg_kernel<8, 1>, grid1d(R, 8), 256, 0, st, in, R, gamma, beta, eps, pre_gelu, residual, out_f32, out_f16);
    else launch_k(ln_rows_kernel, grid1d(R, 8), 256, 0, st, in, R, C, gamma, beta, eps, pre_gelu, residual, out_f32, out_f16);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int linear_f32(const float* in, int M, int K, const float* W, const float* bias, int N, int in_act, int out_act,
               const float* addend, float* out_f32, __half* out_f16, float out_scale, cudaStream_t st) {
    if (K % 4) return -1;
    if (M > 8 && M <= 64 && (long long)N * K <= (4LL << 20)) {
        // small weight matrices (text / time conditioning MLPs at batch 32): latency-bound, so spread them over many
        // warps -- one warp per (8-row group, output column) with the whole weight row in flight at once
        dim3 grid((N + 7) / 8, (M + 7) / 8);
        launch_k(linear_f32_kernel<8>, grid, 256, 0, st, in, M, K, W, bias, N, in_act, out_act, addend, out_f32, out_f16,
                                                   out_scale);
    } else if (M > 8) {     // 32 x 128 shared-memory tiles: every weight row is streamed once per 32 input rows
        dim3 grid((N + kTN - 1) / kTN, (M + kTM - 1) / kTM);
        launch_k(linear_tiled_kernel, grid, 256, 0, st, in, M, K, W, bias, N, in_act, out_act, addend, out_f32, out_f16,
                                                  out_scale);
    } else {
        dim3 grid((N + 7) / 8, 1);
        launch_k(linear_f32_kernel<8>, grid, 256, 0, st, in, M, K, W, bias, N, in_act, out_act, addend, out_f32, out_f16,
                                                   out_scale);
    }
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int stem_unroll(const float* a, int Ca, const float* b, int Cb, int B, int H, int W, __half* out, cudaStream_t st) {
    if (Ca + Cb > 8 || Ca < 1) return -1;
    dim3 grid((W + kStemCols - 1) / kStemCols, (H + kStemRows - 1) / kStemRows, B);
    launch_k(stem_unroll_kernel, grid, 256, 0, st, a, Ca, b, Cb, B, H, W, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int resize_sep(const float* in, long long planes, int Hin, int Win, float* out, int Hout, int Wout, const int* iy,
               const float* wy, int ty, const int* ix, const float* wx, int tx, int has_clamp, float lo, float hi,
               cudaStream_t st) {
    if (ty < 1 || tx < 1 || planes < 1) return -1;
    const long long total = planes * Hout * Wout;
    launch_k(resize_sep_kernel, grid1d(total, 256), 256, 0, st, in, Hin, Win, out, Hout, Wout, iy, wy, ty, ix, wx, tx,
             has_clamp, lo, hi, total);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int silu_f32(const float* in, long long n, float* out, cudaStream_t st) {
    launch_k(silu_kernel, grid1d(n, 256), 256, 0, st, in, n, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int posemb(const long long* t, int B, int dim, float* out, cudaStream_t st) {
    const int half = dim / 2;
    // reference: emb = math.log(10000) / (half_dim - 1) in double, multiplied into an fp32 tensor
    const float neg_log_step = (float)(-(log(10000.0) / (double)(half - 1)));
    launch_k(posemb_kernel, grid1d((long long)B * half, 128), 128, 0, st, t, B, dim, neg_log_step, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int text_tokens(const float* proj, int B, int L, int D, const uint8_t* mask, const uint8_t* keep,
                const float* null_embed, int max_len, float* c_out, int m, int row_off, float* pooled,
                cudaStream_t st) {
    launch_k(text_tokens_kernel, B, D < 256 ? D : 256, 0, st, proj, L, D, mask, keep, null_embed, max_len, c_out, m, row_off,
                                                        pooled);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int place_rows(const float* src, int B, int r, int D, float* dst, int m, int row_off, cudaStream_t st) {
    launch_k(place_rows_kernel, grid1d((long long)B * r * D, 256), 256, 0, st, src, B, r, D, dst, m, row_off);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int select_rows(const float* a, const float* nullv, const uint8_t* keep, const float* addend, int B, int N, float* out,
                cudaStream_t st) {
    launch_k(select_rows_kernel, grid1d((long long)B * N, 256), 256, 0, st, a, nullv, keep, addend, B, N, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int nchw_to_nhwc(const float* a, int Ca, const float* b, int Cb, int B, int HW, int Cp, float* out, cudaStream_t st) {
    launch_k(nchw_to_nhwc_kernel, grid1d((long long)B * HW * Cp, 256), 256, 0, st, a, Ca, b, Cb, B, HW, Cp, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int pack_conv_weight_dgrad(const float* w, int O, int I, int KH, int KW, __half* out, cudaStream_t st) {
    launch_k(pack_conv_weight_dgrad_kernel, grid1d((long long)O * I * KH * KW, 256), 256, 0, st, w, O, I, KH, KW, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int pack_conv_weight(const float* w, int O, int I, int KH, int KW, float scale, __half* out, cudaStream_t st) {
    launch_k(pack_conv_weight_kernel, grid1d((long long)O * I * KH * KW, 256), 256, 0, st, w, O, I, KH, KW, scale, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace mi
