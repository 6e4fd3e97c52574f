// Fused attention for the U-Net's two attention flavours (dim_head = 64 is hard-wired by the reference):
//   * CrossAttention.forward  (minimagen/layers.py:220-251): 8 heads, keys = [learned null kv] + m context tokens
//   * Attention.forward       (minimagen/layers.py:52-104):  multi-query (ONE shared k/v head), keys = [null kv] + n
// One kernel: S = Q K^T (Q pre-scaled by dim_head^-0.5 via the packed to_q weight), optional key mask
// (masked_fill(~mask, -FLT_MAX), null key never masked), softmax in fp32 (online / flash style, the b x h x n x j score
// tensor the reference materialises is never written), O = P V.  Tensor-core math via mma.sync.m16n8k16 (fp16 in,
// fp32 accumulate); the GEMM-heavy projections around it run on the wgmma path (conv_tc.cu).
//
// CTA = 4 warps = 64 query rows of one (batch, head); key blocks of 64 staged in shared memory (V transposed).
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>

#include "kernels.cuh"
#include "launch.cuh"

namespace mi {

namespace {

constexpr int kD = 64;          // dim_head
constexpr int kBQ = 64;         // queries per CTA
constexpr int kBK = 64;         // keys per block
constexpr int kPad = 8;         // smem row padding (halfs) -> conflict-free fragment reads

__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t pack2(float x, float y) {
    __half2 h = __floats2half2_rn(x, y);
    return *reinterpret_cast<uint32_t*>(&h);
}

__global__ void __launch_bounds__(128)
attn_fwd_kernel(const __half* __restrict__ q, long long q_bs, int ldq, const __half* __restrict__ k,
                const __half* __restrict__ v, long long kv_bs, int ldkv, int kv_hs, const float* __restrict__ null_kv,
                const uint8_t* __restrict__ mask, int n, int m, __half* __restrict__ out, long long o_bs, int ldo) {
    pdl_wait();
    pdl_trigger();
    __shared__ __align__(16) __half Ks[kBK][kD + kPad];    // [key][dim]
    __shared__ __align__(16) __half Vt[kD][kBK + kPad];    // [dim][key]
    __shared__ float s_maskadd[kBK];                       // 0, -FLT_MAX (masked) or -inf (beyond the last key)

    const int b = blockIdx.z, h = blockIdx.y;
    const int q0 = blockIdx.x * kBQ;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gid = lane >> 2, tig = lane & 3;
    const int J = m + 1;   // keys including the null key at index 0

    // ---- Q fragments (16 rows x 64 dims per warp), straight from global
    uint32_t qa[4][4];
    {
        const int r0 = q0 + warp * 16 + gid, r1 = r0 + 8;
        const __half* qb = q + (long long)b * q_bs + h * kD;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            const int c = ks * 16 + tig * 2;
            qa[ks][0] = (r0 < n) ? *reinterpret_cast<const uint32_t*>(qb + (long long)r0 * ldq + c) : 0u;
            qa[ks][1] = (r1 < n) ? *reinterpret_cast<const uint32_t*>(qb + (long long)r1 * ldq + c) : 0u;
            qa[ks][2] = (r0 < n) ? *reinterpret_cast<const uint32_t*>(qb + (long long)r0 * ldq + c + 8) : 0u;
            qa[ks][3] = (r1 < n) ? *reinterpret_cast<const uint32_t*>(qb + (long long)r1 * ldq + c + 8) : 0u;
        }
    }

    float o_acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f; }
    float row_max[2] = {-INFINITY, -INFINITY};
    float row_sum[2] = {0.f, 0.f};

    const __half* kb = k + (long long)b * kv_bs + (long long)h * kv_hs;
    const __half* vb = v + (long long)b * kv_bs + (long long)h * kv_hs;

    for (int j0 = 0; j0 < J; j0 += kBK) {
        __syncthreads();   // previous block fully consumed
        // ---- stage K block and V^T block: 64 keys x 64 dims, 8 halfs (16 B) per thread-step
        for (int i = threadIdx.x; i < kBK * (kD / 8); i += blockDim.x) {
            const int key = i >> 3, dv = (i & 7) * 8;
            const int j = j0 + key;
            uint4 kv4 = make_uint4(0, 0, 0, 0), vv4 = make_uint4(0, 0, 0, 0);
            if (j == 0) {
                __half tk[8], tv[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    tk[e] = __float2half_rn(null_kv[dv + e]);
                    tv[e] = __float2half_rn(null_kv[kD + dv + e]);
                }
                kv4 = *reinterpret_cast<uint4*>(tk);
                vv4 = *reinterpret_cast<uint4*>(tv);
            } else if (j < J) {
                kv4 = *reinterpret_cast<const uint4*>(kb + (long long)(j - 1) * ldkv + dv);
                vv4 = *reinterpret_cast<const uint4*>(vb + (long long)(j - 1) * ldkv + dv);
            }
            *reinterpret_cast<uint4*>(&Ks[key][dv]) = kv4;
            const __half* vh = reinterpret_cast<const __half*>(&vv4);
#pragma unroll
            for (int e = 0; e < 8; ++e) Vt[dv + e][key] = vh[e];
        }
        if (threadIdx.x < kBK) {
            const int j = j0 + threadIdx.x;
            float add = 0.f;
            if (j >= J) add = -INFINITY;
            else if (j > 0 && mask && mask[(long long)b * m + (j - 1)] == 0) add = -FLT_MAX;
            s_maskadd[threadIdx.x] = add;
        }
        __syncthreads();

        // ---- S = Q K^T : 16 x 64 per warp
        float s[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&Ks[nt * 8 + gid][ks * 16 + tig * 2]);
                const uint32_t b1 = *reinterpret_cast<const uint32_t*>(&Ks[nt * 8 + gid][ks * 16 + tig * 2 + 8]);
                mma_16816(s[nt], qa[ks], b0, b1);
            }
        }
        // ---- mask + online softmax (rows gid and gid+8; the 4 lanes of a quad share a row)
        float bm[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const float a0 = s_maskadd[nt * 8 + tig * 2], a1 = s_maskadd[nt * 8 + tig * 2 + 1];
            // masked_fill semantics: a masked score is REPLACED by -FLT_MAX (not added to)
            s[nt][0] = (a0 == 0.f) ? s[nt][0] : a0;
            s[nt][1] = (a1 == 0.f) ? s[nt][1] : a1;
            s[nt][2] = (a0 == 0.f) ? s[nt][2] : a0;
            s[nt][3] = (a1 == 0.f) ? s[nt][3] : a1;
            bm[0] = fmaxf(bm[0], fmaxf(s[nt][0], s[nt][1]));
            bm[1] = fmaxf(bm[1], fmaxf(s[nt][2], s[nt][3]));
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            bm[r] = fmaxf(bm[r], __shfl_xor_sync(0xffffffffu, bm[r], 1));
            bm[r] = fmaxf(bm[r], __shfl_xor_sync(0xffffffffu, bm[r], 2));
        }
        float corr[2], nm[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            nm[r] = fmaxf(row_max[r], bm[r]);          // finite: key 0 (null) is never masked / out of range
            corr[r] = expf(row_max[r] - nm[r]);        // exp(-inf) = 0 on the first block
            row_max[r] = nm[r];
            row_sum[r] *= corr[r];
        }
        uint32_t pa[4][4];   // P as A fragments: 4 k-steps of 16 keys
        float bs[2] = {0.f, 0.f};
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const float p0 = expf(s[nt][0] - nm[0]), p1 = expf(s[nt][1] - nm[0]);
            const float p2 = expf(s[nt][2] - nm[1]), p3 = expf(s[nt][3] - nm[1]);
            bs[0] += p0 + p1;
            bs[1] += p2 + p3;
            const int ks = nt >> 1;
            if ((nt & 1) == 0) { pa[ks][0] = pack2(p0, p1); pa[ks][1] = pack2(p2, p3); }
            else               { pa[ks][2] = pack2(p0, p1); pa[ks][3] = pack2(p2, p3); }
        }
        row_sum[0] += bs[0];
        row_sum[1] += bs[1];
#pragma unroll
        for (int dt = 0; dt < 8; ++dt) {
            o_acc[dt][0] *= corr[0]; o_acc[dt][1] *= corr[0];
            o_acc[dt][2] *= corr[1]; o_acc[dt][3] *= corr[1];
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&Vt[dt * 8 + gid][ks * 16 + tig * 2]);
                const uint32_t b1 = *reinterpret_cast<const uint32_t*>(&Vt[dt * 8 + gid][ks * 16 + tig * 2 + 8]);
                mma_16816(o_acc[dt], pa[ks], b0, b1);
            }
        }
    }

    // ---- finalize: divide by the row sums (reduced over the quad) and store fp16
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        row_sum[r] += __shfl_xor_sync(0xffffffffu, row_sum[r], 1);
        row_sum[r] += __shfl_xor_sync(0xffffffffu, row_sum[r], 2);
    }
    const float inv0 = 1.f / row_sum[0], inv1 = 1.f / row_sum[1];
    const int r0 = q0 + warp * 16 + gid, r1 = r0 + 8;
    __half* ob = out + (long long)b * o_bs + h * kD;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
        const int c = dt * 8 + tig * 2;
        if (r0 < n) *reinterpret_cast<uint32_t*>(ob + (long long)r0 * ldo + c) = pack2(o_acc[dt][0] * inv0, o_acc[dt][1] * inv0);
        if (r1 < n) *reinterpret_cast<uint32_t*>(ob + (long long)r1 * ldo + c) = pack2(o_acc[dt][2] * inv1, o_acc[dt][3] * inv1);
    }
}

}  // namespace

int attention_fwd(const __half* q, long long q_bs, int ldq, const __half* k, const __half* v, long long kv_bs, int ldkv,
                  int kv_hs, const float* null_kv, const uint8_t* mask, int B, int heads, int n, int m, __half* out,
                  long long o_bs, int ldo, cudaStream_t st) {
    if ((ldq % 8) || (ldkv % 8) || (ldo % 2) || (kv_hs % 8)) return -1;
    if ((reinterpret_cast<uintptr_t>(k) & 15) || (reinterpret_cast<uintptr_t>(v) & 15) || (kv_bs % 8)) return -1;
    dim3 grid((n + kBQ - 1) / kBQ, heads, B);
    launch_k(attn_fwd_kernel, grid, 128, 0, st, q, q_bs, ldq, k, v, kv_bs, ldkv, kv_hs, null_kv, mask, n, m, out, o_bs, ldo);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace mi
