// Attention core on the Hopper tensor cores (wgmma + TMA + mbarrier), head dim 64.
//
// Replaces the softmax(q k^T) v core of Attention.forward (layers.py:56-104; one shared k/v head = multi-query) and
// CrossAttention.forward (layers.py:226-251; per-head k/v over the text tokens), both with the learned null key/value
// prepended (layers.py:67-70, :240-242).  q arrives pre-scaled (dim_head**-0.5 folded into to_q).
//
// One CTA = 128 queries of one (batch, head); warpgroup 0 is the TMA producer (Q once, then K and V^T blocks of 128 keys
// through a two-stage mbarrier ring), warpgroups 1 and 2 each own 64 of the queries:
//   S = Q K_j^T       wgmma m64n128k16, Q and K from shared memory, S in registers (fp32)
//   P = exp(S - m)    online softmax in registers: running row maximum m, O and the row sums rescaled when m rises
//   O += P V_j        wgmma m64n64k16 with P as the register A operand (the S accumulator layout IS the A fragment
//                     layout, so P never leaves the registers), V^T from shared memory
// K comes from a padded copy with the null key prepended, V from a TRANSPOSED padded copy (keys contiguous = the K-major B
// operand of the second GEMM); both, and the key-validity bits (null key, key_mask, padding), are written by
// attn_prep_kernel into a caller-provided workspace.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.cuh"
#include "launch.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace mi {

namespace {

constexpr int kD = 64, kBQ = 128, kBK = 128;
constexpr int kThreads = 384;
constexpr int kStages = 2;
constexpr uint32_t kQBytes = kBQ * kD * 2;            // 16 KB
constexpr uint32_t kKBytes = kBK * kD * 2;            // 16 KB: [128 keys][64 dims]
constexpr uint32_t kVBytes = kD * kBK * 2;            // 16 KB: two [64 dims][64 keys] chunks
constexpr uint32_t kStageBytes = kKBytes + kVBytes;
constexpr uint32_t kSmemBytes = kQBytes + kStages * kStageBytes + 1024 + 256;

// ------------------------------------------------------------------------------------------------ operand preparation
// Kp[bh][key][64]: key 0 = null key, keys 1..m = k, keys > m = 0.   Vt[bh][dim][key]: the same, transposed.
// valid[b][key / 32]: bit (key % 32) = this padded key takes part in the softmax -- the null key always, key 1..m unless the
// caller's key mask (b, m; layers.py:86-93 / :242-245) clears it, the padding never.
__global__ void __launch_bounds__(256)
attn_prep_kernel(const __half* __restrict__ k, const __half* __restrict__ v, long long kv_bs, int ldkv, int kv_hs,
                 const float* __restrict__ null_kv, int hkv, int m, int Mp, __half* __restrict__ Kp,
                 __half* __restrict__ Vt, const uint8_t* __restrict__ mask, uint32_t* __restrict__ valid) {
    pdl_wait();
    pdl_trigger();
    if ((blockIdx.y % hkv) == 0 && threadIdx.x < 64) {         // one kv head per image writes the two words of these 64 keys
        const int bb = blockIdx.y / hkv;
        const int key = blockIdx.x * 64 + threadIdx.x;
        const bool ok = key == 0 || (key <= m && (mask == nullptr || mask[(long long)bb * m + key - 1] != 0));
        const uint32_t w = __ballot_sync(0xffffffffu, ok);
        if ((threadIdx.x & 31) == 0) valid[(long long)bb * (Mp / 32) + key / 32] = w;
    }
    __shared__ __half tile[64][kD + 2];               // 64 keys x 64 dims of V (padded: conflict-free transpose)
    const int bh = blockIdx.y, b = bh / hkv, h = bh % hkv;
    const int key0 = blockIdx.x * 64;
    const __half* kb = k + (long long)b * kv_bs + (long long)h * kv_hs;
    const __half* vb = v + (long long)b * kv_bs + (long long)h * kv_hs;
    for (int i = threadIdx.x; i < 64 * kD; i += blockDim.x) {
        const int r = i / kD, d = i % kD;
        const int key = key0 + r;                      // padded index: 0 = null, 1..m = real
        __half kk = __float2half_rn(0.f), vv = kk;
        if (key == 0) { kk = __float2half_rn(null_kv[d]); vv = __float2half_rn(null_kv[kD + d]); }
        else if (key <= m) { kk = kb[(long long)(key - 1) * ldkv + d]; vv = vb[(long long)(key - 1) * ldkv + d]; }
        Kp[((long long)bh * Mp + key) * kD + d] = kk;
        tile[r][d] = vv;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 64 * kD; i += blockDim.x) {
        const int d = i / 64, r = i % 64;
        Vt[((long long)bh * kD + d) * Mp + key0 + r] = tile[r][d];
    }
}

struct AttnArgs {
    int n, heads, hkv, Mp, nblk;
    __half* out; long long o_bs; int ldo;
    const uint32_t* valid;                     // [B][Mp / 32] key validity bits (attn_prep_kernel)
    int* err;
};

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

__global__ void __launch_bounds__(kThreads, 1)
attn_wg_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
               const __grid_constant__ CUtensorMap tmV, const __grid_constant__ AttnArgs a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* sKV = sQ + kQBytes;                // [kStages] x (K block, V^T block)
    uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + kStages * kStageBytes);
    uint64_t* q_full = bars;
    uint64_t* full_bar = bars + 1;              // [kStages]
    uint64_t* empty_bar = bars + 1 + kStages;   // [kStages]: one arrival per consumer warpgroup

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
    const int q0 = blockIdx.x * kBQ, h = blockIdx.y, b = blockIdx.z;
    const int hk = a.hkv == 1 ? 0 : h;
    const int kv_row0 = (b * a.hkv + hk) * a.Mp;     // first padded key of this (batch, kv head) in Kp
    const int vt_row0 = (b * a.hkv + hk) * kD;       // first dim row of this (batch, kv head) in Vt
    int* err = a.err;

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&tmQ);
        ptx::prefetch_tensormap(&tmK);
        ptx::prefetch_tensormap(&tmV);
        ptx::mbar_init(q_full, 1);
        for (int i = 0; i < kStages; ++i) { ptx::mbar_init(&full_bar[i], 1); ptx::mbar_init(&empty_bar[i], 2); }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();

    if (wg == 0) {
        // ===================== TMA producer =====================
        if (warp == 0) {
            if (ptx::elect_one()) {
                ptx::mbar_arrive_expect_tx(q_full, kQBytes);
                ptx::tma_load_2d(&tmQ, q_full, sQ, h * kD, b * a.n + q0);
            }
            int stage = 0;
            uint32_t phase = 0;
            for (int j = 0; j < a.nblk; ++j) {
                ptx::mbar_wait(&empty_bar[stage], phase ^ 1, err, 8100 + stage);
                if (ptx::elect_one()) {
                    uint8_t* sK = sKV + stage * kStageBytes;
                    uint8_t* sV = sK + kKBytes;
                    ptx::mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
                    ptx::tma_load_2d(&tmK, &full_bar[stage], sK, 0, kv_row0 + j * kBK);
                    ptx::tma_load_2d(&tmV, &full_bar[stage], sV, j * kBK, vt_row0);
                    ptx::tma_load_2d(&tmV, &full_bar[stage], sV + kVBytes / 2, j * kBK + 64, vt_row0);
                }
                if (++stage == kStages) { stage = 0; phase ^= 1; }
            }
            pdl_trigger();
        }
        return;
    }

    // ===================== consumers: queries [64 cw, 64 cw + 64) of the tile =====================
    // fragment element 4j + 2r + e of S (resp. O) = row 16 wq + lane/4 + 8r, key (resp. dim) 8j + 2(lane%4) + e
    const int cw = wg - 1, wq = warp & 3;
    constexpr float kLog2e = 1.4426950408889634f;
    float o[kD / 2];
#pragma unroll
    for (int i = 0; i < kD / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const uint32_t* vrow = a.valid + (long long)b * (a.Mp / 32);
    const uint64_t dq = ptx::make_sw128_desc(ptx::smem_u32(sQ + cw * (64 * 128)));
    ptx::mbar_wait(q_full, 0, err, 8200);
    int stage = 0;
    uint32_t phase = 0;
    for (int j = 0; j < a.nblk; ++j) {
        ptx::mbar_wait(&full_bar[stage], phase, err, 8300 + stage);
        const uint32_t sK = ptx::smem_u32(sKV + stage * kStageBytes);
        const uint32_t sV = sK + kKBytes;
        float s[kBK / 2];
        const uint64_t dk = ptx::make_sw128_desc(sK);
        ptx::wg_fence();
#pragma unroll
        for (int k = 0; k < kD / 16; ++k) ptx::Wgmma<kBK, 0>::run(s, dq + 2 * k, dk + 2 * k, k != 0);
        ptx::wg_commit();
        ptx::wg_wait<0>();
        ptx::wg_fence_regs(s);

        // key validity of this block (null key, mask, padding): all-ones words take the fast path
        uint32_t vb[kBK / 32];
        bool tail = false;
#pragma unroll
        for (int w = 0; w < kBK / 32; ++w) { vb[w] = __ldg(vrow + j * (kBK / 32) + w); tail = tail || vb[w] != 0xffffffffu; }
        if (tail) {
#pragma unroll
            for (int i = 0; i < kBK / 2; ++i) {
                const int key = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
                if (!((vb[key >> 5] >> (key & 31)) & 1u)) s[i] = -INFINITY;
            }
        }
        float scale[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            float mx = -INFINITY;
#pragma unroll
            for (int jj = 0; jj < kBK / 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * r], s[4 * jj + 2 * r + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m_run[r], mx);
            // a row whose keys so far are all masked keeps m = -inf: no contribution, nothing to rescale
            scale[r] = m_new == -INFINITY ? 1.f : ptx::ex2_approx((m_run[r] - m_new) * kLog2e);
            m_run[r] = m_new;
        }
        uint32_t p[kBK / 16][4];
        float lsum[2] = {0.f, 0.f};
#pragma unroll
        for (int jj = 0; jj < kBK / 8; ++jj) {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const float mneg = m_run[r] == -INFINITY ? 0.f : -m_run[r] * kLog2e;
                const float p0 = ptx::ex2_approx(fmaf(s[4 * jj + 2 * r], kLog2e, mneg));
                const float p1 = ptx::ex2_approx(fmaf(s[4 * jj + 2 * r + 1], kLog2e, mneg));
                lsum[r] += p0 + p1;
                // A fragment of k-step jj/2: regs {row r0 keys 0-7, row r1 keys 0-7, row r0 keys 8-15, row r1 keys 8-15}
                p[jj >> 1][(jj & 1) * 2 + r] = pack_h2(p0, p1);
            }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * scale[r] + lsum[r];
#pragma unroll
        for (int i = 0; i < kD / 2; ++i) o[i] *= scale[(i >> 1) & 1];

        ptx::wg_fence();
#pragma unroll
        for (int kk = 0; kk < kBK / 16; ++kk) {
            // 16 keys: chunk kk / 4 of V^T ([64 dims][64 keys]), 32-byte step kk % 4 inside the 128-byte rows
            const uint64_t dv = ptx::make_sw128_desc(sV + (kk >> 2) * (kVBytes / 2)) + 2 * (kk & 3);
            ptx::WgmmaRS<kD>::run(o, p[kk], dv, 1);
        }
        ptx::wg_commit();
        ptx::wg_wait<0>();
        ptx::wg_fence_regs(o);
        if ((threadIdx.x & 127) == 0) ptx::mbar_arrive(&empty_bar[stage]);
        if (++stage == kStages) { stage = 0; phase ^= 1; }
    }

    // ---- epilogue: O / l, fp16, head h's 64 columns of the output rows
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        float l = l_run[r];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv = 1.f / l;
        const int row = q0 + cw * 64 + wq * 16 + (lane >> 2) + 8 * r;
        __half* orow = a.out + (long long)b * a.o_bs + (long long)row * a.ldo + h * kD + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < kD / 8; ++jj)
            *reinterpret_cast<uint32_t*>(orow + 8 * jj) = pack_h2(o[4 * jj + 2 * r] * inv, o[4 * jj + 2 * r + 1] * inv);
    }
}

}  // namespace

long long attention_tc_workspace_bytes(int B, int heads, int kv_hs, int m) {
    const int hkv = kv_hs == 0 ? 1 : heads;
    const long long Mp = ((long long)(m + 1) + kBK - 1) / kBK * kBK;
    return 2 * (long long)B * hkv * Mp * kD * (long long)sizeof(__half) + (long long)B * (Mp / 32) * (long long)sizeof(uint32_t);
}

bool attention_tc_supported(int n, int ldq, int ldo, long long q_bs) {
    return n > 0 && (n % kBQ) == 0 && (ldq % 8) == 0 && (ldo % 8) == 0 && q_bs == (long long)n * ldq;
}

int attention_tc_fwd(const __half* q, long long q_bs, int ldq, const __half* k, const __half* v, long long kv_bs, int ldkv,
                     int kv_hs, const float* null_kv, const uint8_t* key_mask, int B, int heads, int n, int m, __half* out,
                     long long o_bs, int ldo, void* workspace, long long workspace_bytes, int* err_flag, cudaStream_t st) {
    if (!attention_tc_supported(n, ldq, ldo, q_bs) || (o_bs % 8) || (reinterpret_cast<uintptr_t>(q) & 15) ||
        (reinterpret_cast<uintptr_t>(out) & 15) || (reinterpret_cast<uintptr_t>(workspace) & 127))
        return -1;
    if (workspace_bytes < attention_tc_workspace_bytes(B, heads, kv_hs, m)) return -1;
    PFN_tmaEncodeTiled enc = get_tma_encode();
    if (!enc) return -1;
    const int hkv = kv_hs == 0 ? 1 : heads;
    const int Mp = (m + 1 + kBK - 1) / kBK * kBK;
    __half* Kp = reinterpret_cast<__half*>(workspace);
    __half* Vt = Kp + (long long)B * hkv * Mp * kD;
    uint32_t* valid = reinterpret_cast<uint32_t*>(Vt + (long long)B * hkv * Mp * kD);      // [B][Mp / 32]
    launch_k(attn_prep_kernel, dim3(Mp / 64, B * hkv), 256, 0, st, k, v, kv_bs, ldkv, kv_hs, null_kv, hkv, m, Mp, Kp, Vt,
             key_mask, valid);
    if (cudaGetLastError() != cudaSuccess) return -2;

    CUtensorMap tmQ, tmK, tmV;
    cuuint32_t estr[2] = {1, 1};
    {
        cuuint64_t dim[2] = {(cuuint64_t)ldq, (cuuint64_t)B * n};
        cuuint64_t str[1] = {(cuuint64_t)ldq * 2};
        cuuint32_t box[2] = {kD, kBQ};
        if (enc(&tmQ, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(q), dim, str, box, estr,
                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
            return -1;
    }
    {
        cuuint64_t dim[2] = {kD, (cuuint64_t)B * hkv * Mp};
        cuuint64_t str[1] = {kD * 2};
        cuuint32_t box[2] = {kD, kBK};
        if (enc(&tmK, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, Kp, dim, str, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) !=
            CUDA_SUCCESS)
            return -1;
    }
    {
        cuuint64_t dim[2] = {(cuuint64_t)Mp, (cuuint64_t)B * hkv * kD};
        cuuint64_t str[1] = {(cuuint64_t)Mp * 2};
        cuuint32_t box[2] = {64, kD};
        if (enc(&tmV, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, Vt, dim, str, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) !=
            CUDA_SUCCESS)
            return -1;
    }
    AttnArgs a{};
    a.n = n; a.heads = heads; a.hkv = hkv; a.Mp = Mp; a.nblk = Mp / kBK;
    a.out = out; a.o_bs = o_bs; a.ldo = ldo; a.valid = valid; a.err = err_flag;
    static bool attr_set = false;
    if (!attr_set) {
        if (cudaFuncSetAttribute(attn_wg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess)
            return -2;
        attr_set = true;
    }
    launch_k(attn_wg_kernel, dim3(n / kBQ, heads, B), kThreads, kSmemBytes, st, tmQ, tmK, tmV, a);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace mi
