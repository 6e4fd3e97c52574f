// Backward kernels of the TRAINING side of the path (SURVEY.md 8f-2: Imagen.forward / _p_losses, reference
// minimagen/Imagen.py:512-650, and autograd through Unet.forward).  fp32 on CUDA cores, NHWC like the forward kernels.
// (Data gradients of tensor-core-shaped convolutions do not come through here: they run on the forward wgmma implicit-GEMM
// kernels with flipped / transposed packed weights, see minimagen_b200/autograd.py.)
//
//   gemm_f32            C[z] (+)= alpha * op(A[z]) op(B[z]), arbitrary element strides, two-level batch index
//                       -> nn.Linear backward (layers.py / Unet.py MLPs), attention forward/backward in fp32
//                          (S = q k^T, dP = dO v^T, dq = dS k, dk = dS^T q, dv = P^T dO)
//   colsum_f32          bias gradients
//   conv2d_dgrad_f32    dL/dx of nn.Conv2d (any k / stride / pad) for the non-tensor-core shapes (tiny config, stem)
//   conv2d_wgrad_f32    dL/dW of nn.Conv2d: tiled pixel contraction with fp32 atomics
//   gn_silu_bwd         Block.forward's GroupNorm -> (scale + 1, shift) -> SiLU (layers.py:136-144): dx, dgamma, dbeta,
//                       d(scale | shift)
//   ln_rows_bwd         LayerNorm / ChanLayerNorm rows (+ the exact-erf GELU in front of ChanFeedForward's second norm)
//   softmax_rows(_bwd)  attention softmax over the key axis
//   upsample2x_bwd      nn.Upsample(scale_factor=2, 'nearest') (layers.py:513)
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "kernels.cuh"
#include "launch.cuh"

namespace mi {

// SM count of the current device (grid sizing of the split reductions)
static int num_sms() {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n > 0 ? n : 132;
}

namespace {

// ------------------------------------------------------------------------------------------------ GEMM
struct GemmArgs {
    const float* A; const float* B; float* C;
    int M, N, K;
    long long a_sm, a_sk, b_sk, b_sn, c_sm, c_sn;
    long long a_b1, a_b2, b_b1, b_b2, c_b1, c_b2;
    int Z2;
    float alpha;
    int accumulate;
};

constexpr int kGT = 64, kGK = 16;

__global__ void __launch_bounds__(256)
gemm_f32_kernel(const GemmArgs g) {
    pdl_wait();
    pdl_trigger();
    __shared__ float As[kGK][kGT + 1];
    __shared__ float Bs[kGK][kGT + 1];
    const int z = blockIdx.z, z1 = z / g.Z2, z2 = z - z1 * g.Z2;
    const float* A = g.A + z1 * g.a_b1 + z2 * g.a_b2;
    const float* B = g.B + z1 * g.b_b1 + z2 * g.b_b2;
    float* C = g.C + z1 * g.c_b1 + z2 * g.c_b2;
    const int m0 = blockIdx.y * kGT, n0 = blockIdx.x * kGT;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    const bool a_kfast = g.a_sk == 1, b_nfast = g.b_sn == 1;
    for (int k0 = 0; k0 < g.K; k0 += kGK) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int idx = tid + i * 256;
            int mm, kk;
            if (a_kfast) { kk = idx & 15; mm = idx >> 4; } else { mm = idx & 63; kk = idx >> 6; }
            const int m = m0 + mm, k = k0 + kk;
            As[kk][mm] = (m < g.M && k < g.K) ? A[m * g.a_sm + k * g.a_sk] : 0.f;
            int nn, kb;
            if (b_nfast) { nn = idx & 63; kb = idx >> 6; } else { kb = idx & 15; nn = idx >> 4; }
            const int n = n0 + nn, k2 = k0 + kb;
            Bs[kb][nn] = (n < g.N && k2 < g.K) ? B[k2 * g.b_sk + n * g.b_sn] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kGK; ++kk) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= g.M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= g.N) continue;
            float* c = C + m * g.c_sm + n * g.c_sn;
            const float v = g.alpha * acc[i][j];
            *c = g.accumulate ? (*c + v) : v;
        }
    }
}

// ------------------------------------------------------------------------------------------------ column sums
__global__ void __launch_bounds__(256)
colsum_kernel(const float* __restrict__ x, long long M, int N, long long rows_per_block, float* __restrict__ out) {
    pdl_wait();
    pdl_trigger();
    __shared__ float red[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int n = blockIdx.x * 32 + tx;
    const long long r0 = (long long)blockIdx.y * rows_per_block;
    const long long r1 = min(M, r0 + rows_per_block);
    float s = 0.f;
    if (n < N)
        for (long long r = r0 + ty; r < r1; r += 8) s += x[r * N + n];
    red[ty][tx] = s;
    __syncthreads();
    if (ty == 0 && n < N) {
#pragma unroll
        for (int i = 1; i < 8; ++i) s += red[i][tx];
        atomicAdd(out + n, s);
    }
}

// ------------------------------------------------------------------------------------------------ conv data gradient
__global__ void __launch_bounds__(256)
conv_dgrad_kernel(const float* __restrict__ dy, int B, int Ho, int Wo, int Cout, const float* __restrict__ w, int Cin,
                  int KH, int KW, int stride, int pad, float* __restrict__ dx, int Hi, int Wi) {
    pdl_wait();
    pdl_trigger();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)B * Hi * Wi * Cin;
    if (idx >= total) return;
    const int ci = (int)(idx % Cin);
    const long long pix = idx / Cin;
    const int wi = (int)(pix % Wi);
    const int hi = (int)((pix / Wi) % Hi);
    const int b = (int)(pix / ((long long)Wi * Hi));
    const int taps = KH * KW;
    const long long wco = (long long)Cin * taps;          // stride between output channels in OIHW
    float acc = 0.f;
    for (int r = 0; r < KH; ++r) {
        const int th = hi + pad - r;
        if (th < 0 || th % stride) continue;
        const int ho = th / stride;
        if (ho >= Ho) continue;
        for (int s = 0; s < KW; ++s) {
            const int tw = wi + pad - s;
            if (tw < 0 || tw % stride) continue;
            const int wo = tw / stride;
            if (wo >= Wo) continue;
            const float* dyp = dy + (((long long)b * Ho + ho) * Wo + wo) * Cout;
            const float* wp = w + ((long long)ci * KH + r) * KW + s;
            for (int co = 0; co < Cout; ++co) acc = fmaf(dyp[co], wp[co * wco], acc);
        }
    }
    dx[idx] = acc;
}

// Few output channels, stride 1 (the 128 -> 3 final conv): the whole weight fits in shared memory, re-laid [tap][co][ci] so that the
// lanes of a warp (consecutive ci) read consecutive words; one block covers kDgPix pixels x C_in.
constexpr int kDgPix = 32;
__global__ void __launch_bounds__(256)
conv_dgrad_smallco_kernel(const float* __restrict__ dy, int B, int Ho, int Wo, int Cout, const float* __restrict__ w, int Cin,
                          int KH, int KW, int pad, float* __restrict__ dx, int Hi, int Wi) {
    pdl_wait();
    pdl_trigger();
    extern __shared__ float ws[];                             // [taps][Cout][Cin]
    const int taps = KH * KW;
    for (int i = threadIdx.x; i < Cout * Cin * taps; i += blockDim.x) {
        const int t = i % taps, ci = (i / taps) % Cin, co = i / (taps * Cin);          // OIHW order of the source
        ws[(t * Cout + co) * Cin + ci] = w[i];
    }
    __syncthreads();
    const long long npix = (long long)B * Hi * Wi;
    const long long p0 = (long long)blockIdx.x * kDgPix;
    for (int e = threadIdx.x; e < kDgPix * Cin; e += blockDim.x) {
        const long long pix = p0 + e / Cin;
        if (pix >= npix) break;
        const int ci = e % Cin;
        const int wi = (int)(pix % Wi), hi = (int)((pix / Wi) % Hi), b = (int)(pix / ((long long)Wi * Hi));
        float acc = 0.f;
        for (int r = 0; r < KH; ++r) {
            const int ho = hi + pad - r;
            if (ho < 0 || ho >= Ho) continue;
            for (int s2 = 0; s2 < KW; ++s2) {
                const int wo = wi + pad - s2;
                if (wo < 0 || wo >= Wo) continue;
                const float* dyp = dy + (((long long)b * Ho + ho) * Wo + wo) * Cout;
                const float* wp = ws + ((r * KW + s2) * Cout) * Cin + ci;
                for (int co = 0; co < Cout; ++co) acc = fmaf(dyp[co], wp[co * Cin], acc);
            }
        }
        dx[pix * Cin + ci] = acc;
    }
}

// ------------------------------------------------------------------------------------------------ conv weight gradient
// dW[co][ci][r][s] = sum over output pixels of dy[pix][co] * x[pix shifted by tap (r, s)][ci].
// grid = (co tiles x ci tiles, taps, pixel splits); a block accumulates a 32 x 32 (co, ci) tile over its pixel range
// (32 pixels per shared-memory stage, 2 x 2 outputs per thread) and adds it to dW with fp32 atomics (dW zeroed by the launcher).
// kFlat (few input channels: the 3-channel stem with 3 / 7 / 15-wide kernels): the second tile axis runs over the flattened
// (ci, r, s) index n = ci * taps + tap of dW[co][n] instead of over ci at a fixed tap -- a 32-wide ci tile holding 3 channels
// wasted 29/32 of the work (9.8 of 39 ms of a b = 32 training step).
constexpr int kWgT = 32, kWgP = 32;

template <bool kFlat>
__global__ void __launch_bounds__(256)
conv_wgrad_kernel(const float* __restrict__ dy, const float* __restrict__ x, int B, int Hi, int Wi, int Cin, int Ho, int Wo,
                  int Cout, int KH, int KW, int stride, int pad, long long pix_per_block, float* __restrict__ dw) {
    pdl_wait();
    pdl_trigger();
    __shared__ float dys[kWgP][kWgT + 1];
    __shared__ float xs[kWgP][kWgT + 1];
    const int taps = KH * KW;
    const int ci_tiles = ((kFlat ? Cin * taps : Cin) + kWgT - 1) / kWgT;
    const int co0 = (blockIdx.x / ci_tiles) * kWgT, ci0 = (blockIdx.x % ci_tiles) * kWgT;
    // this thread's column of the x tile: channel and tap are fixed over the pixel loop
    const int cn = ci0 + (threadIdx.x & 31);
    const bool col_ok = cn < (kFlat ? Cin * taps : Cin);
    const int tap = kFlat ? cn % taps : (int)blockIdx.y;
    const int cch = kFlat ? cn / taps : cn;
    const int r = tap / KW, s = tap % KW;
    const long long total = (long long)B * Ho * Wo;
    const long long p0 = (long long)blockIdx.z * pix_per_block;
    const long long p1 = min(total, p0 + pix_per_block);
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
    for (long long pb = p0; pb < p1; pb += kWgP) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int idx = tid + i * 256;
            const int c = idx & 31, pp = idx >> 5;
            const long long p = pb + pp;
            float dv = 0.f, xv = 0.f;
            if (p < p1) {
                const int wo = (int)(p % Wo);
                const int ho = (int)((p / Wo) % Ho);
                const int b = (int)(p / ((long long)Wo * Ho));
                if (co0 + c < Cout) dv = dy[p * Cout + co0 + c];
                const int hi = ho * stride + r - pad, wi = wo * stride + s - pad;
                if (col_ok && hi >= 0 && hi < Hi && wi >= 0 && wi < Wi)
                    xv = x[(((long long)b * Hi + hi) * Wi + wi) * Cin + cch];
            }
            dys[pp][c] = dv;
            xs[pp][c] = xv;
        }
        __syncthreads();
#pragma unroll 8
        for (int pp = 0; pp < kWgP; ++pp) {
            const float a0 = dys[pp][2 * ty], a1 = dys[pp][2 * ty + 1];
            const float b0 = xs[pp][2 * tx], b1 = xs[pp][2 * tx + 1];
            acc[0][0] = fmaf(a0, b0, acc[0][0]); acc[0][1] = fmaf(a0, b1, acc[0][1]);
            acc[1][0] = fmaf(a1, b0, acc[1][0]); acc[1][1] = fmaf(a1, b1, acc[1][1]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int co = co0 + 2 * ty + i, ci = ci0 + 2 * tx + j;
            if (kFlat) {
                if (co < Cout && ci < Cin * taps) atomicAdd(dw + (long long)co * Cin * taps + ci, acc[i][j]);
            } else {
                if (co < Cout && ci < Cin) atomicAdd(dw + ((long long)co * Cin + ci) * taps + blockIdx.y, acc[i][j]);
            }
        }
}

// ------------------------------------------------------------------------------------------------ GroupNorm/FiLM/SiLU bwd
__device__ __forceinline__ void gn_group_stats(const double* __restrict__ sums, int b, int g, int groups, double n, float eps,
                                               float& mean, float& rstd) {
    const double su = sums[((long long)b * groups + g) * 2], sq = sums[((long long)b * groups + g) * 2 + 1];
    const double m = su / n;
    double var = sq / n - m * m;
    if (var < 0) var = 0;
    mean = (float)m;
    rstd = (float)(1.0 / sqrt(var + (double)eps));
}

__device__ __forceinline__ float silu_grad(float v) {
    const float sg = 1.0f / (1.0f + expf(-v));
    return sg * (1.0f + v * (1.0f - sg));
}

// pass 1: A1[b][c] = sum_p dv, A2[b][c] = sum_p dv * xn   (dv = dy * silu'(v), v = the pre-activation)
__global__ void __launch_bounds__(256)
gn_bwd_sums_kernel(const float* __restrict__ x, const float* __restrict__ dy, const double* __restrict__ sums, int HW, int C,
                   int groups, const float* __restrict__ gamma, const float* __restrict__ beta,
                   const float* __restrict__ ss, int ss_ld, float eps, float* __restrict__ A) {
    pdl_wait();
    pdl_trigger();
    __shared__ float r1[8][33], r2[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int b = blockIdx.y, c = blockIdx.x * 32 + tx;
    float a1 = 0.f, a2 = 0.f;
    if (c < C) {
        const int Cg = C / groups;
        float mean, rstd;
        gn_group_stats(sums, b, c / Cg, groups, (double)Cg * HW, eps, mean, rstd);
        const float sc = ss ? ss[(long long)b * ss_ld + c] + 1.0f : 1.0f;
        const float sh = ss ? ss[(long long)b * ss_ld + C + c] : 0.f;
        const float ga = gamma[c], be = beta[c];
        const float* xp = x + (long long)b * HW * C + c;
        const float* dp = dy + (long long)b * HW * C + c;
        // pixel range of this block: gridDim.z splits HW so that small-batch / few-channel layers still fill the GPU
        const int chunk = (HW + gridDim.z - 1) / gridDim.z;
        const int p_lo = blockIdx.z * chunk, p_hi = min(HW, p_lo + chunk);
        for (int p = p_lo + ty; p < p_hi; p += 8) {
            const float xn = (xp[(long long)p * C] - mean) * rstd;
            const float v = (xn * ga + be) * sc + sh;
            const float dv = dp[(long long)p * C] * silu_grad(v);
            a1 += dv;
            a2 = fmaf(dv, xn, a2);
        }
    }
    r1[ty][tx] = a1; r2[ty][tx] = a2;
    __syncthreads();
    if (ty == 0 && c < C) {
#pragma unroll
        for (int i = 1; i < 8; ++i) { a1 += r1[i][tx]; a2 += r2[i][tx]; }
        if (gridDim.z == 1) {
            A[((long long)b * C + c) * 2] = a1;
            A[((long long)b * C + c) * 2 + 1] = a2;
        } else {                                            // A zeroed by the launcher
            atomicAdd(&A[((long long)b * C + c) * 2], a1);
            atomicAdd(&A[((long long)b * C + c) * 2 + 1], a2);
        }
    }
}

// pass 2 (one block per image): parameter gradients and the two group means the data gradient needs
__global__ void __launch_bounds__(256)
gn_bwd_reduce_kernel(const float* __restrict__ A, int HW, int C, int groups, const float* __restrict__ gamma,
                     const float* __restrict__ beta, const float* __restrict__ ss, int ss_ld, float* __restrict__ dgamma,
                     float* __restrict__ dbeta, float* __restrict__ dss, int dss_ld, float* __restrict__ gm,
                     const double* __restrict__ sums, float eps) {
    pdl_wait();
    pdl_trigger();
    __shared__ float s1[32], s2[32];
    const int b = blockIdx.x;
    if (threadIdx.x < 32) { s1[threadIdx.x] = 0.f; s2[threadIdx.x] = 0.f; }
    __syncthreads();
    const int Cg = C / groups;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const float a1 = A[((long long)b * C + c) * 2], a2 = A[((long long)b * C + c) * 2 + 1];
        const float sc = ss ? ss[(long long)b * ss_ld + c] + 1.0f : 1.0f;
        const float ga = gamma[c], be = beta[c];
        if (dss) {
            dss[(long long)b * dss_ld + c] = ga * a2 + be * a1;          // d scale: sum dv * (xn*gamma + beta)
            dss[(long long)b * dss_ld + C + c] = a1;                     // d shift
        }
        atomicAdd(dgamma + c, sc * a2);
        atomicAdd(dbeta + c, sc * a1);
        const float gp = ga * sc;
        atomicAdd(&s1[c / Cg], gp * a1);
        atomicAdd(&s2[c / Cg], gp * a2);
    }
    __syncthreads();
    if (threadIdx.x < groups) {
        const float inv = 1.0f / ((float)Cg * (float)HW);
        float mean, rstd;
        gn_group_stats(sums, b, threadIdx.x, groups, (double)Cg * HW, eps, mean, rstd);
        float* o = gm + ((long long)b * groups + threadIdx.x) * 4;
        o[0] = s1[threadIdx.x] * inv;
        o[1] = s2[threadIdx.x] * inv;
        o[2] = mean;                        // the fp64 -> fp32 statistics once per (image, group), not once per element
        o[3] = rstd;
    }
}

// pass 3: dx = rstd * (gamma' * dv - m1 - xn * m2); four consecutive channels per thread (C % 4 == 0: same group when Cg % 4 == 0,
// handled per element otherwise)
__global__ void __launch_bounds__(256)
gn_bwd_dx_kernel(const float* __restrict__ x, const float* __restrict__ dy, int HW, int C, int groups,
                 const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ ss, int ss_ld,
                 const float* __restrict__ gm, float* __restrict__ dx, long long total4) {
    pdl_wait();
    pdl_trigger();
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= total4) return;
    const long long idx = q * 4;
    const int c0 = (int)(idx % C);
    const int b = (int)(idx / ((long long)HW * C));
    const int Cg = C / groups;
    const float4 xv = *reinterpret_cast<const float4*>(x + idx);
    const float4 dv4 = *reinterpret_cast<const float4*>(dy + idx);
    const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, ds[4] = {dv4.x, dv4.y, dv4.z, dv4.w};
    float o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int c = c0 + i;
        const float* st = gm + ((long long)b * groups + c / Cg) * 4;
        const float m1 = st[0], m2 = st[1], mean = st[2], rstd = st[3];
        const float sc = ss ? ss[(long long)b * ss_ld + c] + 1.0f : 1.0f;
        const float sh = ss ? ss[(long long)b * ss_ld + C + c] : 0.f;
        const float ga = gamma[c];
        const float xn = (xs[i] - mean) * rstd;
        const float v = (xn * ga + beta[c]) * sc + sh;
        const float dv = ds[i] * silu_grad(v);
        o[i] = rstd * (ga * sc * dv - m1 - xn * m2);
    }
    *reinterpret_cast<float4*>(dx + idx) = make_float4(o[0], o[1], o[2], o[3]);
}

// ------------------------------------------------------------------------------------------------ LayerNorm rows bwd
__device__ __forceinline__ float gelu_erf_fw(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_erf_grad(float x) {
    return 0.5f * (1.0f + erff(x * 0.70710678118654752f)) + x * 0.3989422804014327f * expf(-0.5f * x * x);
}

__global__ void __launch_bounds__(256)
ln_bwd_kernel(const float* __restrict__ in, const float* __restrict__ dy, long long R, int C, const float* __restrict__ gamma,
              float eps, int pre_gelu, float* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta) {
    pdl_wait();
    pdl_trigger();
    extern __shared__ float sacc[];          // [2][C] block-local dgamma / dbeta
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) sacc[i] = 0.f;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int warps = blockDim.x >> 5;
    for (long long row = (long long)blockIdx.x * warps + (threadIdx.x >> 5); row < R; row += (long long)gridDim.x * warps) {
        const float* x = in + row * C;
        const float* d = dy + row * C;
        float s = 0.f;
        for (int c = lane; c < C; c += 32) { const float v = x[c]; s += pre_gelu ? gelu_erf_fw(v) : v; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        const float mean = s / (float)C;
        float q = 0.f;
        for (int c = lane; c < C; c += 32) { float v = x[c]; v = (pre_gelu ? gelu_erf_fw(v) : v) - mean; q = fmaf(v, v, q); }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
        const float rstd = rsqrtf(q / (float)C + eps);
        float s1 = 0.f, s2 = 0.f;
        for (int c = lane; c < C; c += 32) {
            float v = x[c]; v = pre_gelu ? gelu_erf_fw(v) : v;
            const float xn = (v - mean) * rstd, gd = gamma[c] * d[c];
            s1 += gd; s2 = fmaf(gd, xn, s2);
            atomicAdd(&sacc[c], d[c] * xn);
            atomicAdd(&sacc[C + c], d[c]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
        s1 /= (float)C; s2 /= (float)C;
        for (int c = lane; c < C; c += 32) {
            const float raw = x[c];
            const float v = pre_gelu ? gelu_erf_fw(raw) : raw;
            const float xn = (v - mean) * rstd;
            float g = rstd * (gamma[c] * d[c] - s1 - xn * s2);
            if (pre_gelu) g *= gelu_erf_grad(raw);
            dx[row * C + c] = g;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
        if (dgamma) atomicAdd(dgamma + i, sacc[i]);
        if (dbeta) atomicAdd(dbeta + i, sacc[C + i]);
    }
}

// ------------------------------------------------------------------------------------------------ softmax rows
__global__ void __launch_bounds__(256)
softmax_rows_kernel(float* __restrict__ s, long long R, int L) {
    pdl_wait();
    pdl_trigger();
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= R) return;
    const int lane = threadIdx.x & 31;
    float* p = s + row * L;
    float mx = -INFINITY;
    for (int j = lane; j < L; j += 32) mx = fmaxf(mx, p[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int j = lane; j < L; j += 32) { const float e = expf(p[j] - mx); p[j] = e; sum += e; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.0f / sum;
    for (int j = lane; j < L; j += 32) p[j] *= inv;
}

// dS = P * (dP - sum_j P dP), written over dP
__global__ void __launch_bounds__(256)
softmax_rows_bwd_kernel(const float* __restrict__ P, float* __restrict__ dP, long long R, int L) {
    pdl_wait();
    pdl_trigger();
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= R) return;
    const int lane = threadIdx.x & 31;
    const float* p = P + row * L;
    float* d = dP + row * L;
    float dot = 0.f;
    for (int j = lane; j < L; j += 32) dot = fmaf(p[j], d[j], dot);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    for (int j = lane; j < L; j += 32) d[j] = p[j] * (d[j] - dot);
}

// ------------------------------------------------------------------------------------------------ nearest x2 upsample bwd
__global__ void __launch_bounds__(256)
upsample2x_bwd_kernel(const float* __restrict__ dy, int B, int H, int W, int C, float* __restrict__ dx) {
    pdl_wait();
    pdl_trigger();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)B * H * W * C;
    if (idx >= total) return;
    const int c = (int)(idx % C);
    const long long pix = idx / C;
    const int w = (int)(pix % W);
    const int h = (int)((pix / W) % H);
    const long long b = pix / ((long long)W * H);
    const long long o = ((b * 2 * H + 2 * h) * (2LL * W) + 2 * w) * C + c;
    const long long rs = 2LL * W * C;
    dx[idx] = (dy[o] + dy[o + C]) + (dy[o + rs] + dy[o + rs + C]);
}

inline unsigned g1d(long long n, int per) { return (unsigned)((n + per - 1) / per); }

}  // namespace

int gemm_f32(const float* A, const float* B, float* C, int M, int N, int K, long long a_sm, long long a_sk, long long b_sk,
             long long b_sn, long long c_sm, long long c_sn, int Z1, int Z2, long long a_b1, long long a_b2, long long b_b1,
             long long b_b2, long long c_b1, long long c_b2, float alpha, int accumulate, cudaStream_t st) {
    if (M <= 0 || N <= 0 || K <= 0 || Z1 <= 0 || Z2 <= 0 || (long long)Z1 * Z2 > 65535) return -1;
    GemmArgs g{A, B, C, M, N, K, a_sm, a_sk, b_sk, b_sn, c_sm, c_sn, a_b1, a_b2, b_b1, b_b2, c_b1, c_b2, Z2, alpha, accumulate};
    dim3 grid((N + kGT - 1) / kGT, (M + kGT - 1) / kGT, Z1 * Z2);
    launch_k(gemm_f32_kernel, grid, 256, 0, st, g);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int colsum_f32(const float* x, long long M, int N, float* out, int accumulate, cudaStream_t st) {
    if (M <= 0 || N <= 0) return -1;
    if (!accumulate && cudaMemsetAsync(out, 0, (size_t)N * sizeof(float), st) != cudaSuccess) return -2;
    long long splits = (M + 1023) / 1024;
    if (splits > 512) splits = 512;
    const long long rpb = (M + splits - 1) / splits;
    dim3 grid((N + 31) / 32, (unsigned)((M + rpb - 1) / rpb));
    launch_k(colsum_kernel, grid, 256, 0, st, x, M, N, rpb, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int conv2d_dgrad_f32(const float* dy, int B, int Ho, int Wo, int Cout, const float* w, int Cin, int KH, int KW, int stride,
                     int pad, float* dx, int Hi, int Wi, cudaStream_t st) {
    if (stride < 1 || KH < 1 || KW < 1) return -1;
    const long long total = (long long)B * Hi * Wi * Cin;
    const size_t wbytes = (size_t)Cout * Cin * KH * KW * sizeof(float);
    if (stride == 1 && Cout <= 8 && wbytes <= 40 * 1024) {
        const long long npix = (long long)B * Hi * Wi;
        launch_k(conv_dgrad_smallco_kernel, dim3((unsigned)((npix + kDgPix - 1) / kDgPix)), 256, wbytes, st, dy, B, Ho, Wo, Cout, w,
                 Cin, KH, KW, pad, dx, Hi, Wi);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
    }
    launch_k(conv_dgrad_kernel, g1d(total, 256), 256, 0, st, dy, B, Ho, Wo, Cout, w, Cin, KH, KW, stride, pad, dx, Hi, Wi);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int conv2d_wgrad_f32(const float* dy, const float* x, int B, int Hi, int Wi, int Cin, int Ho, int Wo, int Cout, int KH,
                     int KW, int stride, int pad, float* dw, cudaStream_t st) {
    if (stride < 1 || KH < 1 || KW < 1) return -1;
    if (cudaMemsetAsync(dw, 0, (size_t)Cout * Cin * KH * KW * sizeof(float), st) != cudaSuccess) return -2;
    const long long total = (long long)B * Ho * Wo;
    const bool flat = Cin < kWgT && KH * KW > 1;
    if (flat) {
        const int tiles = ((Cout + kWgT - 1) / kWgT) * ((Cin * KH * KW + kWgT - 1) / kWgT);
        long long splits = (16LL * num_sms() + tiles - 1) / tiles;
        const long long max_splits = (total + 4 * kWgP - 1) / (4 * kWgP);
        if (splits > max_splits) splits = max_splits;
        if (splits < 1) splits = 1;
        if (splits > 65535) splits = 65535;
        long long ppb = (total + splits - 1) / splits;
        ppb = (ppb + kWgP - 1) / kWgP * kWgP;
        dim3 grid(tiles, 1, (unsigned)((total + ppb - 1) / ppb));
        launch_k(conv_wgrad_kernel<true>, grid, 256, 0, st, dy, x, B, Hi, Wi, Cin, Ho, Wo, Cout, KH, KW, stride, pad, ppb, dw);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
    }
    const int tiles = ((Cout + kWgT - 1) / kWgT) * ((Cin + kWgT - 1) / kWgT);
    // 256-thread blocks with 8 KB of shared memory: ~8 resident per SM -> aim at two full waves of those (the ragged layers that
    // land here -- 3-channel stem / 3-channel output, 15 x 15 taps -- have few (tile, tap) pairs and long pixel loops)
    long long splits = (16LL * num_sms() + tiles * KH * KW - 1) / (tiles * KH * KW);
    const long long max_splits = (total + 4 * kWgP - 1) / (4 * kWgP);
    if (splits > max_splits) splits = max_splits;
    if (splits < 1) splits = 1;
    if (splits > 65535) splits = 65535;
    long long ppb = (total + splits - 1) / splits;
    ppb = (ppb + kWgP - 1) / kWgP * kWgP;
    dim3 grid(tiles, KH * KW, (unsigned)((total + ppb - 1) / ppb));
    launch_k(conv_wgrad_kernel<false>, grid, 256, 0, st, dy, x, B, Hi, Wi, Cin, Ho, Wo, Cout, KH, KW, stride, pad, ppb, dw);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int gn_silu_bwd(const float* x, const float* dy, const double* sums, int B, int HW, int C, int groups, const float* gamma,
                const float* beta, const float* ss, int ss_ld, float eps, float* dx, float* dgamma, float* dbeta,
                float* dss, int dss_ld, float* workspace, cudaStream_t st) {
    if (groups < 1 || groups > 32 || C % groups) return -1;
    if (C % 4) return -1;
    float* A = workspace;                                   // [B][C][2]
    float* gm = workspace + (long long)B * C * 2;           // [B][groups][4]: m1, m2, mean, rstd
    const int blocks_xy = ((C + 31) / 32) * B;
    int Z = (8 * num_sms() + blocks_xy - 1) / blocks_xy;          // ~8 blocks per SM over the whole grid
    if (Z > HW / 64) Z = HW / 64;
    if (Z < 1) Z = 1;
    if (Z > 1 && cudaMemsetAsync(A, 0, (size_t)B * C * 2 * sizeof(float), st) != cudaSuccess) return -2;
    dim3 g1((C + 31) / 32, B, Z);
    launch_k(gn_bwd_sums_kernel, g1, 256, 0, st, x, dy, sums, HW, C, groups, gamma, beta, ss, ss_ld, eps, A);
    launch_k(gn_bwd_reduce_kernel, B, 256, 0, st, (const float*)A, HW, C, groups, gamma, beta, ss, ss_ld, dgamma, dbeta, dss,
             dss_ld, gm, sums, eps);
    const long long total4 = (long long)B * HW * C / 4;
    launch_k(gn_bwd_dx_kernel, g1d(total4, 256), 256, 0, st, x, dy, HW, C, groups, gamma, beta, ss, ss_ld, (const float*)gm, dx,
             total4);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int ln_rows_bwd(const float* in, const float* dy, long long R, int C, const float* gamma, float eps, int pre_gelu, float* dx,
                float* dgamma, float* dbeta, cudaStream_t st) {
    if (C < 1 || (size_t)2 * C * sizeof(float) > 48 * 1024) return -1;
    long long blocks = (R + 7) / 8;
    if (blocks > 2 * num_sms()) blocks = 2 * num_sms();
    launch_k(ln_bwd_kernel, (unsigned)blocks, 256, (size_t)2 * C * sizeof(float), st, in, dy, R, C, gamma, eps, pre_gelu, dx,
             dgamma, dbeta);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int softmax_rows(float* s, long long R, int L, cudaStream_t st) {
    launch_k(softmax_rows_kernel, g1d(R, 8), 256, 0, st, s, R, L);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int softmax_rows_bwd(const float* P, float* dP, long long R, int L, cudaStream_t st) {
    launch_k(softmax_rows_bwd_kernel, g1d(R, 8), 256, 0, st, P, dP, R, L);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int upsample2x_bwd(const float* dy, int B, int H, int W, int C, float* dx, cudaStream_t st) {
    launch_k(upsample2x_bwd_kernel, g1d((long long)B * H * W * C, 256), 256, 0, st, dy, B, H, W, C, dx);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace mi
