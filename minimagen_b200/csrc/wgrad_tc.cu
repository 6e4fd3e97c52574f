// Weight gradient of a convolution (stride 1 'same' k = 1 / 3, or the 4 x 4 stride-2 pad-1 Downsample) on the tensor cores
// (training side, SURVEY.md 8f-2):
//
//     dW[co][ci][r][s] = sum over output pixels p = (b, h, w) of  dY[p][co] * X[b][stride*h + r - pad][stride*w + s - pad][ci]
//
// = for every tap one GEMM  dW_t[C_out][C_in] = dY^T[C_out][P] x X_t[P][C_in]  whose CONTRACTION runs over the pixels.  dY and X
// are NHWC fp16 (channels contiguous), i.e. both operands are "MN-major" for wgmma: the kernel loads (8 x 8 pixels) x 64
// channel boxes with TMA (128B swizzle: one pixel = one 128-byte row, 8 rows = one 1024-byte atom), the tap's shift is applied to
// X's box coordinates (TMA zero-fills outside the image = the conv's zero padding; for stride 2 the box spans 16 x 16 input pixels
// and TMA element strides keep every second one), and the wgmma transpose flags mark A and B as MN-major; the matrix
// descriptors step through K in 8-row atoms (SBO = 1024 B) and through the 64-channel blocks of N with LBO = one box (8 KB).
// fp32 accumulation in registers over this CTA's pixel range; the pixel axis is split over gridDim.y CTAs per (co tile, ci tile,
// tap); every CTA stores its partial tile to the workspace [split][tap][C_out][C_in] and wgrad_reduce_kernel sums the splits
// into the OIHW result.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one elected lane), warpgroups 1 and 2 = consumers, each owning 64 of
// the 128 output channels of the tile.
#include <cuda_runtime.h>

#include "conv_tc.cuh"
#include "kernels.cuh"
#include "launch.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace mi {

namespace {

constexpr int kWgThreads = 384;
constexpr int kPx = 64;                                   // pixels per pipeline stage: one 8 x 8 box
constexpr uint32_t kBoxBytes = kPx * 128;                 // 64 pixels x 64 channels fp16 = 8 KiB
constexpr int kMaxStages = 6;

struct WgradArgs {
    int B, H, W, Cin, Cout, kh, kw, pad, stride;     // H x W = the OUTPUT (dY) grid
    int tiles_co, tiles_ci, n_blocks;                     // n_blocks = 64-channel blocks of the N (C_in) tile: 1 or 2
    int tiles_w, tiles_h;                                 // 8 x 8 pixel boxes per image
    long long total_px_tiles, px_tiles_per_cta;
    int stages;
    float* ws;                                            // partial tiles [split][tap][C_out][C_in]
    int* err;
};

template <int NB>
__global__ void __launch_bounds__(kWgThreads, 1)
conv_wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmX,
                     const __grid_constant__ WgradArgs a) {
    constexpr int N = NB * 64;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    constexpr uint32_t stage_bytes = (2 + NB) * kBoxBytes;       // dY: two 64-channel blocks (M = 128); X: NB blocks
    const int STAGES = a.stages;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * stage_bytes);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + kMaxStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
    int* err = a.err;
    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&tmY);
        ptx::prefetch_tensormap(&tmX);
        for (int i = 0; i < STAGES; ++i) { ptx::mbar_init(&full_bar[i], 1); ptx::mbar_init(&empty_bar[i], 2); }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();

    // this CTA's problem: (co tile, ci tile, tap) and a range of 8 x 8 pixel boxes
    int id = blockIdx.x;
    const int tap = id % (a.kh * a.kw); id /= a.kh * a.kw;
    const int ci_t = id % a.tiles_ci;
    const int co_t = id / a.tiles_ci;
    const int dh = tap / a.kw - a.pad, dw_ = tap % a.kw - a.pad;
    const long long p0 = (long long)blockIdx.y * a.px_tiles_per_cta;
    long long p1 = p0 + a.px_tiles_per_cta;
    if (p1 > a.total_px_tiles) p1 = a.total_px_tiles;
    const int n_steps = (int)(p1 > p0 ? p1 - p0 : 0);

    if (wg == 0) {
        if (warp == 0) {
            // ===================== TMA producer =====================
            int stage = 0;
            uint32_t phase = 0;
            for (int i = 0; i < n_steps; ++i) {
                const long long pt = p0 + i;
                const int tw = (int)(pt % a.tiles_w);
                const int th = (int)((pt / a.tiles_w) % a.tiles_h);
                const int b = (int)(pt / ((long long)a.tiles_w * a.tiles_h));
                ptx::mbar_wait(&empty_bar[stage], phase ^ 1, err, 7100 + stage);
                if (ptx::elect_one()) {
                    uint8_t* s = smem + stage * stage_bytes;
                    ptx::mbar_arrive_expect_tx(&full_bar[stage], stage_bytes);
                    ptx::tma_load_5d(&tmY, &full_bar[stage], s, co_t * 128, tw * 8, th * 8, 0, b);
                    ptx::tma_load_5d(&tmY, &full_bar[stage], s + kBoxBytes, co_t * 128 + 64, tw * 8, th * 8, 0, b);
                    for (int nb = 0; nb < NB; ++nb)
                        ptx::tma_load_5d(&tmX, &full_bar[stage], s + (2 + nb) * kBoxBytes, ci_t * N + nb * 64,
                                         tw * 8 * a.stride + dw_, th * 8 * a.stride + dh, 0, b);
                }
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            pdl_trigger();
        }
    } else if (n_steps > 0) {
        // ===================== consumers: D[64 co][N ci] += dY^T (MN-major A) x X (MN-major B), K = 64 pixels per stage ==========
        const int cw = wg - 1;
        float acc[N / 2];
        int stage = 0, prev = -1;
        uint32_t phase = 0;
        for (int i = 0; i < n_steps; ++i) {
            ptx::mbar_wait(&full_bar[stage], phase, err, 7200 + stage);
            const uint32_t sa = ptx::smem_u32(smem + stage * stage_bytes);
            const uint64_t da = ptx::make_sw128_desc(sa + cw * kBoxBytes, kBoxBytes);
            const uint64_t db = ptx::make_sw128_desc(sa + 2 * kBoxBytes, kBoxBytes);
            ptx::wg_fence();
#pragma unroll
            for (int k = 0; k < kPx / 16; ++k)      // 16 pixels = two 8-row atoms = 2048 B further along K
                ptx::Wgmma<N, 1>::run(acc, da + (uint64_t)(k * 128), db + (uint64_t)(k * 128), (i | k) != 0);
            ptx::wg_commit();
            ptx::wg_wait<1>();
            if (prev >= 0 && (threadIdx.x & 127) == 0) ptx::mbar_arrive(&empty_bar[prev]);
            prev = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        ptx::wg_wait<0>();
        ptx::wg_fence_regs(acc);
        // ---- this split's partial tile: fragment element 4j + 2r + e = co row 16 wq + lane/4 + 8r, ci column 8j + 2(lane%4) + e
        const int wq = warp & 3;
        const int taps = a.kh * a.kw;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int co = co_t * 128 + cw * 64 + wq * 16 + (lane >> 2) + 8 * r;
            float* dst = a.ws + (((long long)blockIdx.y * taps + tap) * a.Cout + co) * a.Cin + ci_t * N + 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < N / 8; ++j)
                *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[4 * j + 2 * r], acc[4 * j + 2 * r + 1]);
        }
    }
}

// dW[co][ci][tap] = sum over splits of ws[split][tap][co][ci]
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ ws, int splits, int taps, long long cc, float* __restrict__ dw) {
    pdl_wait();
    pdl_trigger();
    const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= cc * taps) return;
    const int t = (int)(o % taps);
    const long long cci = o / taps;
    float acc = 0.f;
    for (int s = 0; s < splits; ++s) acc += ws[((long long)s * taps + t) * cc + cci];
    dw[o] = acc;
}

struct WgradPlan { int n_blocks, tiles_co, tiles_ci, groups; long long total_px_tiles, px_tiles_per_cta, splits; };

WgradPlan wgrad_plan(int B, int H, int W, int Cin, int Cout, int kh, int kw) {
    WgradPlan p{};
    p.n_blocks = (Cin % 128 == 0) ? 2 : 1;
    p.tiles_co = Cout / 128; p.tiles_ci = Cin / (p.n_blocks * 64);
    p.total_px_tiles = (long long)B * (W / 8) * (H / 8);
    p.groups = p.tiles_co * p.tiles_ci * kh * kw;
    int dev = 0, num_sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
    long long splits = (2LL * num_sms + p.groups - 1) / p.groups;            // about two CTAs per SM over the whole grid
    if (splits > p.total_px_tiles) splits = p.total_px_tiles;
    if (splits < 1) splits = 1;
    if (splits > 65535) splits = 65535;
    p.px_tiles_per_cta = (p.total_px_tiles + splits - 1) / splits;
    p.splits = (p.total_px_tiles + p.px_tiles_per_cta - 1) / p.px_tiles_per_cta;
    return p;
}

}  // namespace

long long conv_wgrad_tc_workspace_bytes(int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride) {
    if (!conv_wgrad_tc_supported(H, W, Cin, Cout, kh, kw, stride) || B < 1) return 0;
    const WgradPlan p = wgrad_plan(B, H, W, Cin, Cout, kh, kw);
    return p.splits * kh * kw * (long long)Cout * Cin * (long long)sizeof(float);
}

// H x W = the output (dY) grid; stride 1: 'same' k = 1 / 3 (pad = k / 2); stride 2: k = 4, pad = 1 (input 2H x 2W)
bool conv_wgrad_tc_supported(int H, int W, int Cin, int Cout, int kh, int kw, int stride) {
    const bool geom = (stride == 1 && kh == kw && (kh & 1) && kh <= 3) || (stride == 2 && kh == 4 && kw == 4);
    return H > 0 && W > 0 && H % 8 == 0 && W % 8 == 0 && Cin > 0 && Cin % 64 == 0 && Cout > 0 && Cout % 128 == 0 && geom;
}

int conv_wgrad_tc(const __half* dy, const __half* x, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride,
                  float* dw, float* workspace, long long workspace_bytes, cudaStream_t stream) {
    if (!conv_wgrad_tc_supported(H, W, Cin, Cout, kh, kw, stride) || B < 1) return -1;
    if ((reinterpret_cast<uintptr_t>(dy) & 15) || (reinterpret_cast<uintptr_t>(x) & 15) || !workspace ||
        (reinterpret_cast<uintptr_t>(workspace) & 15))
        return -1;
    if (workspace_bytes < conv_wgrad_tc_workspace_bytes(B, H, W, Cin, Cout, kh, kw, stride)) return -1;
    PFN_tmaEncodeTiled enc = get_tma_encode();
    if (!enc) return -1;
    const WgradPlan plan = wgrad_plan(B, H, W, Cin, Cout, kh, kw);

    WgradArgs a{};
    a.B = B; a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.kh = kh; a.kw = kw; a.pad = stride == 2 ? 1 : kh / 2; a.stride = stride;
    a.n_blocks = plan.n_blocks;
    a.tiles_co = plan.tiles_co; a.tiles_ci = plan.tiles_ci;
    a.tiles_w = W / 8; a.tiles_h = H / 8;
    a.total_px_tiles = plan.total_px_tiles;
    a.ws = workspace; a.err = nullptr;
    const int groups = plan.groups;
    const long long splits = plan.splits;
    a.px_tiles_per_cta = plan.px_tiles_per_cta;
    const uint32_t stage_bytes = (2 + a.n_blocks) * kBoxBytes;
    a.stages = kMaxStages;
    const uint32_t smem = a.stages * stage_bytes + 1024 + 256;

    CUtensorMap tmY, tmX;
    for (int which = 0; which < 2; ++which) {
        const cuuint64_t C = which ? Cin : Cout;
        const cuuint64_t S = which ? stride : 1;                 // X lives on the (stride*H) x (stride*W) input grid
        cuuint32_t box[5] = {64, (cuuint32_t)(8 * S), (cuuint32_t)(8 * S), 1, 1};
        cuuint32_t estr[5] = {1, (cuuint32_t)S, (cuuint32_t)S, 1, 1};
        cuuint64_t gdim[5] = {C, (cuuint64_t)W * S, (cuuint64_t)H * S, 1, (cuuint64_t)B};
        cuuint64_t gstr[4] = {C * 2, (cuuint64_t)W * S * C * 2, (cuuint64_t)H * S * W * S * C * 2, (cuuint64_t)H * S * W * S * C * 2};
        if (enc(which ? &tmX : &tmY, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<__half*>(which ? x : dy), gdim, gstr, box, estr,
                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
            return -1;
    }
    static bool attr_set = false;
    if (!attr_set) {
        if (cudaFuncSetAttribute(conv_wgrad_tc_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess ||
            cudaFuncSetAttribute(conv_wgrad_tc_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess)
            return -2;
        attr_set = true;
    }
    dim3 grid(groups, (unsigned)splits);
    if (a.n_blocks == 2) launch_k(conv_wgrad_tc_kernel<2>, grid, kWgThreads, smem, stream, tmY, tmX, a);
    else launch_k(conv_wgrad_tc_kernel<1>, grid, kWgThreads, smem, stream, tmY, tmX, a);
    const long long cc = (long long)Cout * Cin, total = cc * kh * kw;
    launch_k(wgrad_reduce_kernel, dim3((unsigned)((total + 255) / 256)), 256, 0, stream, (const float*)workspace, (int)splits, kh * kw, cc, dw);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace mi
