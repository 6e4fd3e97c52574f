// DDPM reverse-step epilogue (everything in Imagen._p_sample after the U-Net call), NCHW fp32 like the reference:
//   1. classifier-free-guidance combine            null + (cond - null) * w                 (Unet.py:506)
//      + predict_start_from_noise                  x0 = a[t] * x_t - b[t] * eps             (diffusion_model.py:159-162)
//   2. dynamic threshold                           s = max(quantile(|x0|, p), 1) per image  (Imagen.py:313-320)
//      exact: radix select on the uint32 bit patterns of |x0| (order statistics lo / hi chosen on the host with
//      torch's own fp32 rank arithmetic), linear interpolation like at::lerp
//   3. clamp(x0, -s, s) / s, posterior mean c1[t] * x0 + c2[t] * x_t, + sigma[t] * noise (zero at t == 0)
//                                                                  (Imagen.py:323, diffusion_model.py:118-125, Imagen.py:361-370)
// The per-image schedule gathers (helpers.extract) happen inside the kernels from the fp32 tables.
// Products and sums are kept un-fused (__fmul_rn/__fadd_rn) so that the arithmetic matches torch's op-by-op rounding.
// The guidance weight w is cond_scale for every image, or w[b] per image when the optional array w [B] is given (the _w
// entry points): one captured step then serves every scale and every per-image scale vector.  The _ws entry points also
// take a guidance table w_sched [T] (Imagen.sample(guidance_interval=, guidance_schedule=)): image b then combines with
// w_b(t[b]) = w[b] where w_sched[t[b]] == 1, else 1 + (w[b] - 1) * w_sched[t[b]], rounded op by op.
// Guidance rescale (mi_guidance_rescale_factor, mi_step_epilogue_rescaled; Imagen.sample(guidance_rescale=), Lin et al.
// 2024): with g the guided prediction as above (fp32, op by op) and c = eps_cond, per image b
//   SS_c = sum (c - mean c)^2, SS_g = sum (g - mean g)^2   in fp64 (fixed-order chunked two-pass sums, no atomics),
//   f_b  = fp32(phi_b * sqrt(SS_c / SS_g) + (1 - phi_b))  the whole expression in fp64, rounded once; 1 where SS_g == 0,
//          NaN where the image has a NaN,
// and the rescaled step uses eps = fp32(g * f_b) (the kRescale instances of guided_x0); x0, threshold and posterior are
// unchanged, so it is bit for bit the plain step fed fp32(g * f) with no guidance pass.
// Steps 1 and 3 are written once (guided_x0, posterior_elem) and shared by the three-kernel form and the fused kernel.
// The select of step 2 exists twice, and each is the other's test reference: quantile_kernel (one CTA per image, keys
// streamed from global memory, any n) and the one inside step_epilogue_kernel (an 8-CTA cluster per image, keys held in
// registers, n <= 196 608).  Both end in step_threshold.
//
// Keyed sampling noise (mi_randn_keyed, Imagen.sample(seed=)): a stateless counter-based generator, so that every draw is
// a pure function of (image seed, stage, draw kind, label, element index) -- independent of the batch layout, the rank
// count, graph or eager execution and skipped steps, and computable inside a captured graph that reads everything from
// device buffers.
//   key      the image's 64-bit seed s as (lo32, hi32)
//   counter  (q, label mod 2^32, kind, stage): element j of the image's flattened C*H*W NCHW data is lane j % 4 of quad
//            q = j / 4; kind is 0 'init', 1 'step', 2 'lowres', 3 'renoise', 4 'inpaint'; stage is the U-Net number
//   bits     Philox4x32-10 with the Random123 / cuRAND constants M = 0xD2511F53, 0xCD9E8D57, W = 0x9E3779B9, 0xBB67AE85
//   normals  Box-Muller on each pair (x_a, x_b) = (x0, x1), (x2, x3) of the quad:
//              u = ((x_a >> 9) + 0.5) 2^-23 in (0, 1) and v = (x_b >> 8) 2^-24 in [0, 1), both exact in fp32
//              (u keeps 23 bits: (m + 0.5) with a 24-bit m would need 25 significant bits);
//              rho = sqrtf(-2 logf(u)); the pair's normals are rho cospif(2v) and rho sinpif(2v).
//            Precise functions, products rounded on their own (__fmul_rn).  |z| <= sqrt(-2 ln 2^-24) = 5.77 by
//            construction, since u >= 2^-24.
#include <cuda_runtime.h>
#include <curand_philox4x32_x.h>
#include <float.h>
#include <stdint.h>

#include <cooperative_groups.h>

#include "clamp_nan.cuh"
#include "kernels.cuh"
#include "launch.cuh"

namespace mi {

namespace {

// The guidance weight of image b at its timestep tb, scheduled by w_sched[tb] when the table is given.
__device__ __forceinline__ float image_scale(const float* w, const float* w_sched, float cond_scale, int b, long long tb) {
    const float wb = w ? w[b] : cond_scale;
    if (!w_sched) return wb;
    const float s = w_sched[tb];
    return s == 1.f ? wb : __fadd_rn(1.f, __fmul_rn(__fsub_rn(wb, 1.f), s));
}

// The guidance combine g = null + (cond - null) * w, rounded op by op.
__device__ __forceinline__ float guide(float c, float nl, float w) { return __fadd_rn(nl, __fmul_rn(__fsub_rn(c, nl), w)); }

// Step 1 at element idx: eps = null + (cond - null) * w when eps_null is given, then x0 = a[t] * x_t - b[t] * eps.
// kRescale (guidance rescale): eps <- eps * f, f the image's factor from rescale_factor_kernel.
template <bool kRescale = false>
__device__ __forceinline__ float guided_x0(const float* x_t, const float* eps_cond, const float* eps_null,
                                           float cond_scale, float a, float b, long long idx, float f = 1.f) {
    float e = eps_cond[idx];
    if (eps_null) e = guide(e, eps_null[idx], cond_scale);
    if constexpr (kRescale) e = __fmul_rn(e, f);
    return __fsub_rn(__fmul_rn(a, x_t[idx]), __fmul_rn(b, e));
}

// The threshold from the two selected order statistics (bit patterns of |x0|): at::lerp in its vectorised CPU form,
// base + coeff * (end - start) with weight < 0.5 ? (start, w) : (end, w - 1), then s.clamp_(min=min_s).
// NaN follows torch: has_nan (some |x0| key above +inf's 0x7F800000) gives s = NaN, as torch.quantile of a row containing
// NaN; lerp(inf, inf) is NaN (at least n - rank_lo values are +-inf); and the min_s clamp keeps a NaN.  The posterior
// then makes the whole image NaN (clamp(x0, -s, s) / s), as the reference does.
__device__ __forceinline__ float step_threshold(uint32_t v_lo, uint32_t v_hi, float weight, float min_s, bool has_nan) {
    if (has_nan) return __uint_as_float(0x7FFFFFFFu);
    const float lo = __uint_as_float(v_lo), hi = __uint_as_float(v_hi);
    const float diff = __fsub_rn(hi, lo);
    const float s = (weight < 0.5f) ? fmaf(weight, diff, lo) : fmaf(__fsub_rn(weight, 1.0f), diff, hi);
    return fmax_nan(s, min_s);
}

// Step 3 at element idx: xs = clamp(x0, -s, s) / s, mean = c1 * xs + c2 * x_t, and out = mean + sig * noise.
// kHist (the multistep form): mean += c3 * x0_hist, skipped where c3 == 0, and xs replaces x0_hist.
// `out` may alias `x_t`: x_t[idx] is read before out[idx] is written.
template <bool kHist>
__device__ __forceinline__ void posterior_elem(float x0, float s, float c1, float c2, float c3, float sig,
                                               const float* x_t, const float* __restrict__ noise,
                                               float* __restrict__ x0_hist, float* out, long long idx) {
    float xs = fminf(fmaxf(x0, -s), s);
    xs = __fdiv_rn(xs, s);
    float mean = __fadd_rn(__fmul_rn(c1, xs), __fmul_rn(c2, x_t[idx]));
    if constexpr (kHist) {
        if (c3 != 0.f) mean = __fadd_rn(mean, __fmul_rn(c3, x0_hist[idx]));
        x0_hist[idx] = xs;
    }
    out[idx] = __fadd_rn(mean, __fmul_rn(sig, noise[idx]));
}

// kRescale: the guided eps times rescale[b] (guided_x0); the extra argument comes last.
template <bool kRescale>
__global__ void __launch_bounds__(256)
x0_kernel(const float* __restrict__ x_t, const float* __restrict__ eps_cond, const float* __restrict__ eps_null,
          float cond_scale, const long long* __restrict__ t, const float* __restrict__ tab_recip,
          const float* __restrict__ tab_recipm1, int n_per_img, float* __restrict__ x0, const float* __restrict__ w,
          const float* __restrict__ w_sched, const float* __restrict__ rescale) {
    pdl_wait();
    pdl_trigger();
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_per_img) return;
    const long long idx = (long long)b * n_per_img + i;
    const long long tb = t[b];
    x0[idx] = guided_x0<kRescale>(x_t, eps_cond, eps_null, image_scale(w, w_sched, cond_scale, b, tb), tab_recip[tb],
                                  tab_recipm1[tb], idx, kRescale ? rescale[b] : 1.f);
}

// One CTA per image.  Exact k-th order statistics of |x| by 4 x 8-bit radix passes over the float bit patterns.
constexpr int kSelThreads = 1024;

__device__ __forceinline__ uint32_t absbits(float v) { return __float_as_uint(v) & 0x7FFFFFFFu; }
// |v| bit patterns above +inf's are NaN
constexpr uint32_t kInfBits = 0x7F800000u;

__global__ void __launch_bounds__(kSelThreads)
quantile_kernel(const float* __restrict__ x0, int n, int rank_lo, int rank_hi, float weight, float min_s,
                float* __restrict__ s_out) {
    pdl_wait();
    pdl_trigger();
    __shared__ unsigned hist[257];
    __shared__ uint32_t sh_prefix, sh_k, sh_eq;
    __shared__ uint32_t sh_min[32];
    const float* x = x0 + (long long)blockIdx.x * n;
    const int tid = threadIdx.x, lane = tid & 31;
    uint32_t prefix = 0, maskbits = 0, k = (uint32_t)rank_lo;
    const int n_round = (n + 31) & ~31;
    bool nan_key = false;                       // this thread has seen a NaN (pass 0 reads every key)
    int has_nan = 0;

    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        for (int i = tid; i < 257; i += kSelThreads) hist[i] = 0;
        __syncthreads();
        for (int i = tid; i < n_round; i += kSelThreads) {
            unsigned bin = 256;
            if (i < n) {
                const uint32_t key = absbits(x[i]);
                nan_key |= key > kInfBits;
                if ((key & maskbits) == prefix) bin = (key >> shift) & 0xFF;
            }
            const unsigned peers = __match_any_sync(0xffffffffu, bin);
            if (lane == (__ffs(peers) - 1)) atomicAdd(&hist[bin], __popc(peers));
        }
        if (pass == 0) has_nan = __syncthreads_or(nan_key);
        else __syncthreads();
        if (tid == 0) {
            uint32_t cum = 0;
            int d = 0;
            for (; d < 256; ++d) {
                if (k < cum + hist[d]) break;
                cum += hist[d];
            }
            sh_prefix = prefix | ((uint32_t)d << shift);
            sh_k = k - cum;
            sh_eq = hist[d];
        }
        __syncthreads();
        prefix = sh_prefix;
        k = sh_k;
        maskbits |= 0xFFu << shift;
        __syncthreads();
    }
    // prefix == bit pattern of sorted[rank_lo]; k == index inside its run of equal values; sh_eq == run length
    const uint32_t v_lo = prefix;
    uint32_t v_hi = v_lo;
    if (rank_hi > rank_lo && k + 1 >= sh_eq) {
        // next order statistic = smallest key strictly greater than v_lo
        uint32_t mn = 0xFFFFFFFFu;
        for (int i = tid; i < n; i += kSelThreads) {
            const uint32_t key = absbits(x[i]);
            if (key > v_lo && key < mn) mn = key;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        if (lane == 0) sh_min[tid >> 5] = mn;
        __syncthreads();
        if (tid < 32) {
            mn = sh_min[tid];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            if (tid == 0) sh_min[0] = mn;
        }
        __syncthreads();
        v_hi = sh_min[0];
        if (v_hi == 0xFFFFFFFFu) v_hi = v_lo;   // cannot happen for rank_hi < n
    }
    if (tid == 0) s_out[blockIdx.x] = step_threshold(v_lo, v_hi, weight, min_s, has_nan);
}

// kHist: the multistep form (mi_step_epilogue_multistep) of posterior_elem.  The extra arguments come last so that the
// kHist = false instance is the plain kernel.
template <bool kHist>
__global__ void __launch_bounds__(256)
posterior_kernel(const float* __restrict__ x0, const float* x_t, const float* __restrict__ noise,
                 const float* __restrict__ s, const long long* __restrict__ t, const float* __restrict__ tab_c1,
                 const float* __restrict__ tab_c2, const float* __restrict__ tab_sigma, int n_per_img,
                 float* out,     // out may alias x_t (same index read before written by the same thread)
                 const float* __restrict__ tab_c3, float* __restrict__ x0_hist) {
    pdl_wait();
    pdl_trigger();
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_per_img) return;
    const long long idx = (long long)b * n_per_img + i;
    const long long tb = t[b];
    const float sb = s[b];
    const float c1 = tab_c1[tb], c2 = tab_c2[tb];
    const float sig = (tb == 0) ? 0.f : tab_sigma[tb];   // nonzero_mask * exp(0.5 * log_var)
    const float c3 = kHist ? tab_c3[tb] : 0.f;
    posterior_elem<kHist>(x0[idx], sb, c1, c2, c3, sig, x_t, noise, x0_hist, out, idx);
}


// ------------------------------------------------------------------------------------------------ fused step epilogue
// The whole of Imagen._p_sample after the U-Net as ONE kernel (SURVEY 8b `mi_step_epilogue`): an 8-CTA cluster per image
//   1. computes guided_x0 for its n/8 elements and KEEPS them in registers (kSelPerThread per thread),
//   2. runs the exact radix select on their |.| bit patterns: the passes of quantile_kernel, with each CTA's 256-bin
//      histogram summed over the cluster through distributed shared memory; every CTA derives the same (v_lo, v_hi)
//      and therefore the same threshold s,
//   3. applies posterior_elem to the register-resident x0, re-reading x_t (L2-hot) and the noise.
// The image is read from memory once instead of once per radix pass, the x0 tensor never exists in memory (one write +
// two reads of the image less than the three-kernel form) and two launches disappear from the step.  `out` may alias
// `x_t` (in-place update of the sampling state): every element is read and written by the same thread.
// kHist: the multistep form, as posterior_kernel<true>; the history is only touched in the final register loop.
// kRescale: guidance rescale, the guided eps times rescale[img] (guided_x0).
constexpr int kSelCluster = 8, kSelPerThread = 24;

template <bool kHist, bool kRescale>
__global__ void __cluster_dims__(kSelCluster, 1, 1) __launch_bounds__(kSelThreads)
step_epilogue_kernel(const float* x_t, const float* __restrict__ eps_cond, const float* __restrict__ eps_null,
                     float cond_scale, const long long* __restrict__ t, const float* __restrict__ tab_recip,
                     const float* __restrict__ tab_recipm1, const float* __restrict__ tab_c1,
                     const float* __restrict__ tab_c2, const float* __restrict__ tab_sigma,
                     const float* __restrict__ noise, int n, int rank_lo, int rank_hi, float weight, float min_s,
                     float* out, float* __restrict__ s_out, const float* __restrict__ tab_c3,
                     float* __restrict__ x0_hist, const float* __restrict__ w, const float* __restrict__ w_sched,
                     const float* __restrict__ rescale) {
    pdl_wait();
    pdl_trigger();
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    // this CTA's histogram of the current pass (read remotely by the peers) and the cluster-wide one; entry 256 is not a
    // bin: it holds whether this CTA's x0 has a NaN, so that ghist[256] != 0 when the image has one
    __shared__ unsigned hist[257];
    __shared__ unsigned ghist[257];
    __shared__ uint32_t sh_prefix, sh_k, sh_eq, sh_cta_min, sh_maskbits;
    __shared__ uint32_t sh_min[32];
    const int img = blockIdx.x / kSelCluster;
    const unsigned rank = cluster.block_rank();
    const int tid = threadIdx.x, lane = tid & 31;
    const int chunk = (n + kSelCluster - 1) / kSelCluster;
    const int beg = rank * chunk;
    const int cnt = max(0, min(chunk, n - beg));
    const long long base = (long long)img * n + beg;
    const long long tb = t[img];
    const float ca = tab_recip[tb], cb = tab_recipm1[tb];
    const float scale = image_scale(w, w_sched, cond_scale, img, tb);
    const float fac = kRescale ? rescale[img] : 1.f;

    float x0v[kSelPerThread];
    bool nan_key = false;
#pragma unroll
    for (int j = 0; j < kSelPerThread; ++j) {
        const int i = tid + j * kSelThreads;
        x0v[j] = i < cnt ? guided_x0<kRescale>(x_t, eps_cond, eps_null, scale, ca, cb, base + i, fac) : 0.f;
        nan_key |= isnan(x0v[j]);       // (not absbits(.) > kInfBits: ptxas would keep those keys for pass 0, and spill)
    }
    // Each pass reads its mask from shared memory.  With the mask a compile-time constant of the unrolled passes, ptxas
    // precomputes the next pass's masked keys next to x0v, and at 64 registers that spills.  Thread 0 updates it after
    // the barrier that ends the pass's reads.
    uint32_t prefix = 0, k = (uint32_t)rank_lo;
    const int cta_nan = __syncthreads_or(nan_key);
    if (tid == 0) {
        sh_maskbits = 0;
        hist[256] = cta_nan;                                       // never re-zeroed: summed again by every pass
    }
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        if (tid < 256) hist[tid] = 0;
        __syncthreads();
        const uint32_t maskbits = sh_maskbits;
#pragma unroll
        for (int j = 0; j < kSelPerThread; ++j) {
            const uint32_t key = absbits(x0v[j]);
            const bool live = (tid + j * kSelThreads < cnt) && ((key & maskbits) == prefix);
            const unsigned bin = live ? ((key >> shift) & 0xFF) : 256u;
            const unsigned peers = __match_any_sync(0xffffffffu, bin);
            if (live && lane == (__ffs(peers) - 1)) atomicAdd(&hist[bin], __popc(peers));
        }
        cluster.sync();                                            // every CTA's histogram is complete
        if (tid < 257) {
            unsigned tt = 0;
#pragma unroll
            for (int r = 0; r < kSelCluster; ++r) tt += *cluster.map_shared_rank(&hist[tid], r);
            ghist[tid] = tt;
        }
        __syncthreads();
        if (tid < 32) {
            // digit select: lane owns bins [8*lane, 8*lane+8); warp scan of the lane totals, then a scan inside one lane
            unsigned loc[8], tot = 0;
#pragma unroll
            for (int e = 0; e < 8; ++e) { loc[e] = ghist[8 * lane + e]; tot += loc[e]; }
            unsigned incl = tot;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            const unsigned excl = incl - tot;
            if (k >= excl && k < incl) {                           // exactly one lane (k < total count)
                unsigned cum = excl;
                int d = 0;
                for (; d < 8; ++d) {
                    if (k < cum + loc[d]) break;
                    cum += loc[d];
                }
                sh_prefix = prefix | ((uint32_t)(8 * lane + d) << shift);
                sh_k = k - cum;
                sh_eq = loc[d];
            }
        }
        __syncthreads();
        prefix = sh_prefix;
        k = sh_k;
        if (tid == 0) sh_maskbits = maskbits | (0xFFu << shift);
        cluster.sync();                                            // peers are done reading hist before it is re-zeroed
    }
    const uint32_t v_lo = prefix;
    uint32_t v_hi = v_lo;
    if (rank_hi > rank_lo && k + 1 >= sh_eq) {                      // uniform over the cluster (same k, same sh_eq)
        uint32_t mn = 0xFFFFFFFFu;
#pragma unroll
        for (int j = 0; j < kSelPerThread; ++j) {
            const uint32_t key = absbits(x0v[j]);
            if ((tid + j * kSelThreads < cnt) && key > v_lo && key < mn) mn = key;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        if (lane == 0) sh_min[tid >> 5] = mn;
        __syncthreads();
        if (tid < 32) {
            mn = sh_min[tid];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            if (tid == 0) sh_cta_min = mn;
        }
        cluster.sync();
        if (tid == 0) {                                            // every CTA reduces the eight CTA minima itself
            uint32_t m = 0xFFFFFFFFu;
            for (int r = 0; r < kSelCluster; ++r) m = min(m, *cluster.map_shared_rank(&sh_cta_min, r));
            sh_min[0] = m;
        }
        cluster.sync();                                            // peers keep their smem alive until everyone has read it
        v_hi = sh_min[0];
        if (v_hi == 0xFFFFFFFFu) v_hi = v_lo;
    }
    const float sb = step_threshold(v_lo, v_hi, weight, min_s, ghist[256] != 0);
    if (s_out && rank == 0 && tid == 0) s_out[img] = sb;

    const float c1 = tab_c1[tb], c2 = tab_c2[tb];
    const float sig = (tb == 0) ? 0.f : tab_sigma[tb];
    const float c3 = kHist ? tab_c3[tb] : 0.f;
#pragma unroll
    for (int j = 0; j < kSelPerThread; ++j) {
        const int i = tid + j * kSelThreads;
        if (i < cnt) posterior_elem<kHist>(x0v[j], sb, c1, c2, c3, sig, x_t, noise, x0_hist, out, base + i);
    }
}

// t <- max(t - 1, 0): the sampling loop's next timestep (diffusion_model.py:81-87 walks T-1 .. 0), advanced on the device
// at the end of the captured step so that a loop iteration is nothing but a graph replay.
__global__ void advance_t_kernel(long long* t, int B) {
    pdl_wait();
    pdl_trigger();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B) t[i] = t[i] > 0 ? t[i] - 1 : 0;
}

// t <- next_t[t]: the same walk over a respaced grid tau_S > ... > tau_1 = 0 (next_t[tau_i] = tau_{i-1}, next_t[0] = 0), so a
// captured step replays any number of sampling steps.  A t outside [0, T) goes to 0 instead of indexing past the table.
__global__ void advance_t_table_kernel(long long* t, const long long* __restrict__ next_t, int T, int B) {
    pdl_wait();
    pdl_trigger();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B) {
        const long long tb = t[i];
        t[i] = (tb >= 0 && tb < T) ? next_t[tb] : 0;
    }
}

// img.clamp_(-1, 1); (img + 1) * 0.5      (Imagen.py:418-419, helpers.py:183)
__global__ void finalize_kernel(const float* __restrict__ x, long long n, int unnormalize, float* __restrict__ out) {
    pdl_wait();
    pdl_trigger();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float v = clamp_nan(x[i], -1.f, 1.f);
    if (unnormalize) v = __fmul_rn(__fadd_rn(v, 1.f), 0.5f);
    out[i] = v;
}

// q_sample: a[t] * x0 + b[t] * noise   (diffusion_model.py:142-145); optional pre-normalisation x*2-1 is NOT applied
// here (the reference noises the [0,1] image first, Imagen.py:483, and normalises afterwards, Imagen.py:393).
__global__ void q_sample_kernel(const float* __restrict__ x0, const float* __restrict__ noise,
                                const long long* __restrict__ t, const float* __restrict__ tab_a,
                                const float* __restrict__ tab_b, int n_per_img, float post_scale, float post_shift,
                                float* __restrict__ out) {
    pdl_wait();
    pdl_trigger();
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_per_img) return;
    const long long idx = (long long)b * n_per_img + i;
    const long long tb = t[b];
    float v = __fadd_rn(__fmul_rn(tab_a[tb], x0[idx]), __fmul_rn(tab_b[tb], noise[idx]));
    v = __fadd_rn(__fmul_rn(v, post_scale), post_shift);   // post_scale=2, post_shift=-1: normalize_neg_one_to_one
    out[idx] = v;
}

// RePaint inpainting, one iteration's prologue, in place on x [B, C, hw] (m, k broadcast over C; m: [B, hw]):
//   r[b] > 0:  x <- ra[t] x + rb[t] z_renoise                          (re-noise from the next grid point back to t)
//   m >= 0.5:  x <- sqrt_acp[t] k + sqrt_1m_acp[t] z_known             (paste the known region, noised to t)
// Same op order as a torch restatement (explicit _rn, no contraction).  The paste is a select, so where m < 0.5 and
// r[b] = 0 x is left bitwise unchanged.  z_renoise is only read where r[b] > 0; a t outside [0, T) leaves the image alone.
__global__ void inpaint_prologue_kernel(float* __restrict__ x, const long long* __restrict__ t,
                                        const long long* __restrict__ r, const float* __restrict__ ra,
                                        const float* __restrict__ rb, const float* __restrict__ sqrt_acp,
                                        const float* __restrict__ sqrt_1m_acp, const float* __restrict__ k,
                                        const float* __restrict__ m, const float* __restrict__ z_renoise,
                                        const float* __restrict__ z_known, int T, int C, int hw) {
    pdl_wait();
    pdl_trigger();
    const int b = blockIdx.y;
    const long long n_per_img = (long long)C * hw;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_per_img) return;
    const long long tb = t[b];
    if (tb < 0 || tb >= T) return;
    const long long idx = (long long)b * n_per_img + i;
    float v = x[idx];
    if (r[b] > 0) v = __fadd_rn(__fmul_rn(ra[tb], v), __fmul_rn(rb[tb], z_renoise[idx]));
    if (m[(long long)b * hw + i % hw] >= 0.5f)
        v = __fadd_rn(__fmul_rn(sqrt_acp[tb], k[idx]), __fmul_rn(sqrt_1m_acp[tb], z_known[idx]));
    x[idx] = v;
}

// The RePaint loop counter: r <- r + 1 while r + 1 < R at a grid point 0 < t < T; otherwise r <- 0 and t moves to the next
// grid point (next_t[t]; a t outside [0, T) goes to 0).  R is read from the device so a captured graph serves every R.
__global__ void inpaint_advance_kernel(long long* t, long long* r, const long long* __restrict__ next_t,
                                       const long long* __restrict__ R, int T, int B) {
    pdl_wait();
    pdl_trigger();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const long long tb = t[i], rr = r[i];
    if (tb > 0 && tb < T && rr + 1 < R[0]) {
        r[i] = rr + 1;
    } else {
        r[i] = 0;
        t[i] = (tb >= 0 && tb < T) ? next_t[tb] : 0;
    }
}

// finalize(where(m >= 0.5, k, x)): the last paste of the known region fused with clamp_(-1, 1) and (v + 1) * 0.5
__global__ void inpaint_finalize_kernel(const float* __restrict__ x, const float* __restrict__ k,
                                        const float* __restrict__ m, int C, int hw, int unnormalize,
                                        float* __restrict__ out) {
    pdl_wait();
    pdl_trigger();
    const int b = blockIdx.y;
    const long long n_per_img = (long long)C * hw;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_per_img) return;
    const long long idx = (long long)b * n_per_img + i;
    float v = m[(long long)b * hw + i % hw] >= 0.5f ? k[idx] : x[idx];
    v = clamp_nan(v, -1.f, 1.f);
    if (unnormalize) v = __fmul_rn(__fadd_rn(v, 1.f), 0.5f);
    out[idx] = v;
}

// Box-Muller on one pair of Philox words (header comment): u, v and 2v are exact; logf and sincospif (cospif and sinpif
// with one argument reduction) are the precise library functions (1 ulp), sqrtf is correctly rounded.
__device__ __forceinline__ float2 box_muller(uint32_t xa, uint32_t xb) {
    const float u = __fmul_rn(__fadd_rn((float)(xa >> 9), 0.5f), 0x1p-23f);
    const float v2 = __fmul_rn((float)(xb >> 8), 0x1p-23f);                 // 2v
    const float rho = sqrtf(__fmul_rn(-2.f, logf(u)));
    float s, c;
    sincospif(v2, &s, &c);
    return make_float2(__fmul_rn(rho, c), __fmul_rn(rho, s));
}

// out [B, n]: image b's keyed normals, one Philox call (four values) per thread.  The label is the host's `label`, or
// t[b] * (R ? R[0] : 1) + (r ? r[b] : 0) read on the device when t is given (a captured step draws at the current t).
// vec4: n % 4 == 0 and out 16-byte aligned, one float4 store per thread; otherwise scalar stores up to the row's end.
__global__ void __launch_bounds__(256)
randn_keyed_kernel(float* __restrict__ out, const long long* __restrict__ seeds, long long n, int kind, int stage,
                   const long long* __restrict__ t, const long long* __restrict__ r, const long long* __restrict__ R,
                   long long label, int vec4) {
    pdl_wait();
    pdl_trigger();
    const int b = blockIdx.y;
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= (n + 3) / 4) return;
    const long long lab = t ? t[b] * (R ? R[0] : 1LL) + (r ? r[b] : 0LL) : label;
    const unsigned long long s = (unsigned long long)seeds[b];
    const uint4 x = curand_Philox4x32_10(make_uint4((uint32_t)q, (uint32_t)lab, (uint32_t)kind, (uint32_t)stage),
                                         make_uint2((uint32_t)s, (uint32_t)(s >> 32)));
    const float2 z01 = box_muller(x.x, x.y), z23 = box_muller(x.z, x.w);
    float* row = out + (long long)b * n;
    const long long j = 4 * q;
    if (vec4) {
        *reinterpret_cast<float4*>(row + j) = make_float4(z01.x, z01.y, z23.x, z23.y);
        return;
    }
    const float z[4] = {z01.x, z01.y, z23.x, z23.y};
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (j + k < n) row[j + k] = z[k];
}


// ------------------------------------------------------------------------------------------------ guidance rescale factor
// Per image b: SS_c = sum (c - mean c)^2 and SS_g = sum (g - mean g)^2 in fp64 over its n values, g = guide(c, null, w_b(t)),
// then f[b] = fp32(phi_b sqrt(SS_c / SS_g) + (1 - phi_b)) (1 where SS_g == 0).  Deterministic, no atomics:
//   rescale_partial_kernel  one CTA per (kRsChunk-value chunk, image): the chunk's sums and, in a second pass over the
//                           (L2-hot) chunk, its sums of squares about the chunk mean; both reduced in a fixed order;
//   rescale_factor_kernel   one CTA per image: the chunks merged in a fixed order (Chan et al.: M2 = sum M2_k +
//                           n_k (m_k - m)^2, which an offset mean cannot cancel), then f.
constexpr int kRsThreads = 256, kRsChunk = 8192;

// (a, b) summed over the CTA in a fixed order (shuffle tree per warp, then the warps in order); every thread gets it.
__device__ __forceinline__ double2 block_sum2(double a, double b, double2* sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) sh[warp] = make_double2(a, b);
    __syncthreads();
    if (threadIdx.x == 0) {
        double2 tot = sh[0];
        for (int i = 1; i < kRsThreads / 32; ++i) { tot.x += sh[i].x; tot.y += sh[i].y; }
        sh[kRsThreads / 32] = tot;
    }
    __syncthreads();
    const double2 r = sh[kRsThreads / 32];
    __syncthreads();                                  // sh is reused by the caller's next reduction
    return r;
}

__global__ void __launch_bounds__(kRsThreads)
rescale_partial_kernel(const float* __restrict__ eps_cond, const float* __restrict__ eps_null,
                       const float* __restrict__ w, const float* __restrict__ w_sched, const long long* __restrict__ t,
                       int n, int nchunks, double4* __restrict__ part) {
    pdl_wait();
    pdl_trigger();
    __shared__ double2 sh[kRsThreads / 32 + 1];
    const int b = blockIdx.y, k = blockIdx.x;
    const int beg = k * kRsChunk, cnt = min(kRsChunk, n - beg);
    const long long base = (long long)b * n + beg;
    const float wb = image_scale(w, w_sched, 1.f, b, t[b]);
    double sc = 0., sg = 0.;
    for (int i = threadIdx.x; i < cnt; i += kRsThreads) {
        const float c = eps_cond[base + i];
        sc += c;
        sg += guide(c, eps_null[base + i], wb);
    }
    const double2 s = block_sum2(sc, sg, sh);
    const double mc = s.x / cnt, mg = s.y / cnt;
    double qc = 0., qg = 0.;
    for (int i = threadIdx.x; i < cnt; i += kRsThreads) {
        const float c = eps_cond[base + i];
        const double dc = (double)c - mc, dg = (double)guide(c, eps_null[base + i], wb) - mg;
        qc += dc * dc;
        qg += dg * dg;
    }
    const double2 q = block_sum2(qc, qg, sh);
    if (threadIdx.x == 0) part[(long long)b * nchunks + k] = make_double4(s.x, q.x, s.y, q.y);
}

__global__ void __launch_bounds__(kRsThreads)
rescale_factor_kernel(const double4* __restrict__ part, const float* __restrict__ phi, int n, int nchunks,
                      float* __restrict__ f) {
    pdl_wait();
    pdl_trigger();
    __shared__ double2 sh[kRsThreads / 32 + 1];
    const int b = blockIdx.x;
    const double4* p = part + (long long)b * nchunks;
    double sc = 0., sg = 0.;
    for (int k = threadIdx.x; k < nchunks; k += kRsThreads) { sc += p[k].x; sg += p[k].z; }
    const double2 s = block_sum2(sc, sg, sh);
    const double mc = s.x / n, mg = s.y / n;
    double qc = 0., qg = 0.;
    for (int k = threadIdx.x; k < nchunks; k += kRsThreads) {
        const double4 v = p[k];
        const double cnt = (double)min(kRsChunk, n - k * kRsChunk);
        const double dc = v.x / cnt - mc, dg = v.z / cnt - mg;
        qc += v.y + cnt * dc * dc;
        qg += v.w + cnt * dg * dg;
    }
    const double2 q = block_sum2(qc, qg, sh);
    if (threadIdx.x == 0) {
        const double ph = phi[b];
        f[b] = q.y == 0. ? 1.f : (float)(ph * sqrt(q.x / q.y) + (1. - ph));
    }
}

}  // namespace

int randn_keyed(float* out, const long long* seeds, int B, long long n, int kind, int stage, const long long* t,
                const long long* r, const long long* R, long long label, cudaStream_t st) {
    if (B < 0 || n < 0 || kind < 0 || kind > 4 || stage < 0) return -1;
    if (B == 0 || n == 0) return 0;
    if (!out || !seeds) return -1;
    const long long nq = (n + 3) / 4;
    if (nq > (1LL << 32) || B > 65535) return -1;           // the quad index is a 32-bit counter word
    const int vec4 = n % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    dim3 grid((unsigned)((nq + 255) / 256), B);
    launch_k(randn_keyed_kernel, grid, 256, 0, st, out, seeds, n, kind, stage, t, r, R, label, vec4);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int inpaint_prologue(float* x, const long long* t, const long long* r, const float* ra, const float* rb,
                     const float* sqrt_acp, const float* sqrt_1m_acp, const float* k, const float* m,
                     const float* z_renoise, const float* z_known, int T, int B, int C, int hw, cudaStream_t st) {
    if (T <= 0 || B < 0 || C <= 0 || hw <= 0) return -1;
    if (B == 0) return 0;
    const long long n = (long long)C * hw;
    if ((n + 255) / 256 > 0x7fffffffLL || B > 65535) return -1;
    dim3 grid((unsigned)((n + 255) / 256), B);
    launch_k(inpaint_prologue_kernel, grid, 256, 0, st, x, t, r, ra, rb, sqrt_acp, sqrt_1m_acp, k, m, z_renoise, z_known,
             T, C, hw);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int inpaint_advance(long long* t, long long* r, const long long* next_t, const long long* R, int T, int B,
                    cudaStream_t st) {
    if (T <= 0 || B < 0) return -1;
    if (B == 0) return 0;
    launch_k(inpaint_advance_kernel, (B + 127) / 128, 128, 0, st, t, r, next_t, R, T, B);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int inpaint_finalize(const float* x, const float* k, const float* m, int B, int C, int hw, int unnormalize, float* out,
                     cudaStream_t st) {
    if (B < 0 || C <= 0 || hw <= 0) return -1;
    if (B == 0) return 0;
    const long long n = (long long)C * hw;
    if ((n + 255) / 256 > 0x7fffffffLL || B > 65535) return -1;
    dim3 grid((unsigned)((n + 255) / 256), B);
    launch_k(inpaint_finalize_kernel, grid, 256, 0, st, x, k, m, C, hw, unnormalize, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

template <bool kRescale>
static int step_x0_impl(const float* x_t, const float* eps_cond, const float* eps_null, float cond_scale, const float* w,
                        const float* w_sched, const long long* t, const float* tab_recip, const float* tab_recipm1, int B,
                        int n_per_img, float* x0, const float* rescale, cudaStream_t st) {
    dim3 grid((n_per_img + 255) / 256, B);
    launch_k(x0_kernel<kRescale>, grid, 256, 0, st, x_t, eps_cond, eps_null, cond_scale, t, tab_recip, tab_recipm1,
             n_per_img, x0, w, w_sched, rescale);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int step_x0(const float* x_t, const float* eps_cond, const float* eps_null, float cond_scale, const float* w,
            const float* w_sched, const long long* t, const float* tab_recip, const float* tab_recipm1, int B,
            int n_per_img, float* x0, cudaStream_t st) {
    return step_x0_impl<false>(x_t, eps_cond, eps_null, cond_scale, w, w_sched, t, tab_recip, tab_recipm1, B, n_per_img,
                               x0, nullptr, st);
}

int step_quantile(const float* x0, int B, int n_per_img, int rank_lo, int rank_hi, float weight, float min_s,
                  float* s_out, cudaStream_t st) {
    if (rank_lo < 0 || rank_hi < rank_lo || rank_hi >= n_per_img) return -1;
    launch_k(quantile_kernel, B, kSelThreads, 0, st, x0, n_per_img, rank_lo, rank_hi, weight, min_s, s_out);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

template <bool kHist>
static int step_posterior_impl(const float* x0, const float* x_t, const float* noise, const float* s,
                               const long long* t, const float* tab_c1, const float* tab_c2, const float* tab_sigma,
                               const float* tab_c3, int B, int n_per_img, float* out, float* x0_hist, cudaStream_t st) {
    dim3 grid((n_per_img + 255) / 256, B);
    launch_k(posterior_kernel<kHist>, grid, 256, 0, st, x0, x_t, noise, s, t, tab_c1, tab_c2, tab_sigma, n_per_img, out,
             tab_c3, x0_hist);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int step_posterior(const float* x0, const float* x_t, const float* noise, const float* s, const long long* t,
                   const float* tab_c1, const float* tab_c2, const float* tab_sigma, int B, int n_per_img, float* out,
                   cudaStream_t st) {
    return step_posterior_impl<false>(x0, x_t, noise, s, t, tab_c1, tab_c2, tab_sigma, nullptr, B, n_per_img, out,
                                      nullptr, st);
}

bool step_epilogue_fused_ok(int n_per_img) {
    return (n_per_img + kSelCluster - 1) / kSelCluster <= kSelThreads * kSelPerThread;
}

template <bool kHist, bool kRescale = false>
static int step_epilogue_impl(const float* x_t, const float* eps_cond, const float* eps_null, float cond_scale,
                              const float* w, const float* w_sched, const long long* t, const float* tab_recip,
                              const float* tab_recipm1, const float* tab_c1, const float* tab_c2, const float* tab_sigma, const float* tab_c3, const float* noise,
                              float* x0_hist, int B, int n_per_img, int rank_lo, int rank_hi, float weight,
                              float min_s, float* out, float* s_out, float* x0_ws, cudaStream_t st,
                              const float* rescale = nullptr) {
    if (rank_lo < 0 || rank_hi < rank_lo || rank_hi >= n_per_img) return -1;
    if (step_epilogue_fused_ok(n_per_img)) {
        launch_k(step_epilogue_kernel<kHist, kRescale>, B * kSelCluster, kSelThreads, 0, st, x_t, eps_cond, eps_null,
                 cond_scale, t, tab_recip, tab_recipm1, tab_c1, tab_c2, tab_sigma, noise, n_per_img, rank_lo, rank_hi,
                 weight, min_s, out, s_out, tab_c3, x0_hist, w, w_sched, rescale);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
    }
    // images beyond the register-resident select (> 196 608 values, e.g. 3 x 1024 x 1024): x0 through the caller's scratch
    if (!x0_ws || !s_out) return -1;
    int rc = step_x0_impl<kRescale>(x_t, eps_cond, eps_null, cond_scale, w, w_sched, t, tab_recip, tab_recipm1, B,
                                    n_per_img, x0_ws, rescale, st);
    if (rc) return rc;
    rc = step_quantile(x0_ws, B, n_per_img, rank_lo, rank_hi, weight, min_s, s_out, st);
    if (rc) return rc;
    return step_posterior_impl<kHist>(x0_ws, x_t, noise, s_out, t, tab_c1, tab_c2, tab_sigma, tab_c3, B, n_per_img, out,
                                      x0_hist, st);
}

int step_epilogue(const float* x_t, const float* eps_cond, const float* eps_null, float cond_scale, const float* w,
                  const float* w_sched, const long long* t,
                  const float* tab_recip, const float* tab_recipm1, const float* tab_c1, const float* tab_c2,
                  const float* tab_sigma, const float* noise, int B, int n_per_img, int rank_lo, int rank_hi,
                  float weight, float min_s, float* out, float* s_out, float* x0_ws, cudaStream_t st) {
    return step_epilogue_impl<false>(x_t, eps_cond, eps_null, cond_scale, w, w_sched, t, tab_recip, tab_recipm1, tab_c1, tab_c2,
                                     tab_sigma, nullptr, noise, nullptr, B, n_per_img, rank_lo, rank_hi, weight, min_s,
                                     out, s_out, x0_ws, st);
}

int step_epilogue_multistep(const float* x_t, const float* eps_cond, const float* eps_null, float cond_scale,
                            const float* w, const float* w_sched, const long long* t, const float* tab_recip,
                            const float* tab_recipm1, const float* tab_c1,
                            const float* tab_c2, const float* tab_sigma, const float* tab_c3, const float* noise,
                            float* x0_hist, int B, int n_per_img, int rank_lo, int rank_hi, float weight, float min_s,
                            float* out, float* s_out, float* x0_ws, cudaStream_t st) {
    if (!tab_c3 || !x0_hist) return -1;
    return step_epilogue_impl<true>(x_t, eps_cond, eps_null, cond_scale, w, w_sched, t, tab_recip, tab_recipm1, tab_c1, tab_c2,
                                    tab_sigma, tab_c3, noise, x0_hist, B, n_per_img, rank_lo, rank_hi, weight, min_s,
                                    out, s_out, x0_ws, st);
}

int step_epilogue_rescaled(const float* x_t, const float* eps_cond, const float* eps_null, const float* w,
                           const float* w_sched, const float* f, const long long* t, const float* tab_recip,
                           const float* tab_recipm1, const float* tab_c1, const float* tab_c2, const float* tab_sigma,
                           const float* tab_c3, const float* noise, float* x0_hist, int B, int n_per_img, int rank_lo,
                           int rank_hi, float weight, float min_s, float* out, float* s_out, float* x0_ws,
                           cudaStream_t st) {
    if (!eps_null || !w || !f || (tab_c3 == nullptr) != (x0_hist == nullptr)) return -1;
    if (tab_c3)
        return step_epilogue_impl<true, true>(x_t, eps_cond, eps_null, 1.f, w, w_sched, t, tab_recip, tab_recipm1, tab_c1,
                                              tab_c2, tab_sigma, tab_c3, noise, x0_hist, B, n_per_img, rank_lo, rank_hi,
                                              weight, min_s, out, s_out, x0_ws, st, f);
    return step_epilogue_impl<false, true>(x_t, eps_cond, eps_null, 1.f, w, w_sched, t, tab_recip, tab_recipm1, tab_c1,
                                           tab_c2, tab_sigma, nullptr, noise, nullptr, B, n_per_img, rank_lo, rank_hi,
                                           weight, min_s, out, s_out, x0_ws, st, f);
}

long long guidance_rescale_workspace_doubles(int B, int n_per_img) {
    if (B <= 0 || n_per_img <= 0) return 0;
    return 4LL * B * ((n_per_img + kRsChunk - 1) / kRsChunk);
}

int guidance_rescale_factor(const float* eps_cond, const float* eps_null, const float* w, const float* w_sched,
                            const long long* t, const float* phi, int B, int n_per_img, float* f, double* ws,
                            cudaStream_t st) {
    if (B < 0 || n_per_img <= 0 || B > 65535) return -1;
    if (B == 0) return 0;
    if (!eps_cond || !eps_null || !w || !t || !phi || !f || !ws) return -1;
    const int nchunks = (n_per_img + kRsChunk - 1) / kRsChunk;
    double4* part = reinterpret_cast<double4*>(ws);
    launch_k(rescale_partial_kernel, dim3(nchunks, B), kRsThreads, 0, st, eps_cond, eps_null, w, w_sched, t, n_per_img,
             nchunks, part);
    if (cudaGetLastError() != cudaSuccess) return -2;
    launch_k(rescale_factor_kernel, B, kRsThreads, 0, st, (const double4*)part, phi, n_per_img, nchunks, f);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int step_advance_t(long long* t, int B, cudaStream_t st) {
    launch_k(advance_t_kernel, (B + 127) / 128, 128, 0, st, t, B);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int step_advance_t_table(long long* t, const long long* next_t, int T, int B, cudaStream_t st) {
    if (T <= 0 || B < 0) return -1;
    if (B == 0) return 0;
    launch_k(advance_t_table_kernel, (B + 127) / 128, 128, 0, st, t, next_t, T, B);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int step_finalize(const float* x, long long n, int unnormalize, float* out, cudaStream_t st) {
    launch_k(finalize_kernel, (unsigned)((n + 255) / 256), 256, 0, st, x, n, unnormalize, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int q_sample(const float* x0, const float* noise, const long long* t, const float* tab_a, const float* tab_b, int B,
             int n_per_img, float post_scale, float post_shift, float* out, cudaStream_t st) {
    dim3 grid((n_per_img + 255) / 256, B);
    launch_k(q_sample_kernel, grid, 256, 0, st, x0, noise, t, tab_a, tab_b, n_per_img, post_scale, post_shift, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace mi
