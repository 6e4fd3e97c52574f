// Implicit-GEMM convolution on the Hopper tensor cores (wgmma + TMA), im2col-free.
//
// Replaces every dense `nn.Conv2d` / `nn.Linear` on the U-Net hot path whose channel counts are multiples of 64
// (reference call sites: minimagen/layers.py:129 (Block.project 3x3), :415 (res_conv 1x1), :319 (Downsample 4x4 s2),
// :514 (Upsample conv), :157/:160 (ChanFeedForward 1x1), :41-42/:48/:213-214/:217 (attention projections);
// minimagen/Unet.py:234).
//
// GEMM view:  D[M = B*H*W pixels, N = C_out] = sum over taps t, channels c of  A_t[pixel shifted by tap t, c] * Wp[n, t*C_in + c]
//   * activations live in HBM as NHWC fp16 (optionally with a leading "phase" axis, see below);
//   * one A tile (128 pixels x 64 channels) for tap (dh, dw) is ONE TMA box load from the 5-D tensor
//     (C, W, H, P, B) at coordinates (c0, w0 + dw, h0 + dh, p, b0): TMA zero-fills out-of-bounds coordinates, which
//     IS the convolution's zero padding -- no im2col buffer, no halo handling in the kernel;
//   * stride-2 convs read a phase-split copy of the input (P = 4 phases), or the un-split input with TMA element strides 2,
//     so that every tap is again one box;
//   * weights are pre-packed [C_out][taps*C_in] fp16 (K-major), one 2-D TMA box (64 x BLOCK_N) per k-block;
//   * both operands land in shared memory in the 128-byte-swizzled K-major layout wgmma reads directly;
//   * a folded 1x1 conv (ResnetBlock.res_conv) appends k-blocks of a second operand x, read at the centre tap;
//   * persistent CTAs (one per SM) walk the tile list round-robin; the producer runs ahead through the operand ring while
//     the consumers store the previous tile.
//
// Warp roles (384 threads): warpgroup 0 = producer (one elected lane issues the TMA loads), warpgroups 1 and 2 = consumers:
// wgmma m64nBLOCK_Nk16 with fp32 accumulators in registers, then +bias +residual -> global fp32 and/or fp16 (+ GroupNorm
// block statistics) straight from the accumulator fragments.  The consumers share the tiles in one of two schedules:
//   * cooperative (BLOCK_N = 256, and the fused GroupNorm kernel): both consumers work on every tile, each owning 64 of
//     the 128 pixel rows.  Their epilogue leaves the tensor cores idle, which long-K tiles amortise;
//   * ping-pong (TMA kernel, BLOCK_N <= 128): consumer c owns the CTA's tiles c, c + 2, c + 4, ... whole (two wgmma per
//     k16 step, rows 0-63 and 64-127), so one consumer's epilogue runs under the other's mainloop.
// In the TMA kernel the producer warpgroup gives its registers to the consumers (setmaxnreg 40 / 232): that is what lets
// a consumer hold 128 accumulators, of a 256-wide cooperative tile or of a 128-wide ping-pong one.
//
// Transposed schedule (C_out = 128, TR): D^T[128 channels, pixels] = Wp . A^T runs on the cooperative 256-wide kernel
// unchanged but for the producer and the epilogue.  The weight box (64 K x 128 channels) fills the 16 KiB stage slot and
// is the wgmma A operand; a 256-pixel activation box (BW x BH = 256 of one image, tile_box) fills the 32 KiB
// slot and is B.  Consumer cw owns output channels [64 cw, 64 cw + 64) of 256 pixels, so a C_out = 128 conv moves the
// operand bytes per FLOP of a 128x256 tile instead of a 128x128 one.  Its epilogue stores channel-strided from the
// fragments (8 channels x 4 pixels per warp store) and, every value of a warp being in one 16-channel block of one image,
// sums its statistics with one shuffle reduction and one atomic pair per warp and tile.
//
// Fused GroupNorm variant (Block.forward, minimagen/layers.py:131-145: GroupNorm -> (scale + 1, shift) -> SiLU -> 3x3 conv):
// the whole producer warpgroup builds the A tile instead of TMA -- it reads the fp32 NHWC source(s) (optionally the virtual
// concat cat(x, skip * s), Unet.py:445), applies y = SiLU(x * A[b,c] + Bc[b,c]) with per-(image, channel) coefficients folded
// from the producers' GroupNorm block statistics, affine, FiLM and skip scale, and writes fp16 in the swizzled layout; the
// normalised tensor never exists in HBM.
#include "conv_tc.cuh"

#include <cuda_runtime.h>
#include <mutex>
#include <stdio.h>

#include "kernels.cuh"
#include "launch.cuh"
#include "ptx.cuh"
#include "sat_half.cuh"
#include "wgmma.cuh"

namespace mi {

namespace {

constexpr int kNumThreads = 384;                               // warpgroup 0: producer, 1-2: consumers
constexpr uint32_t kABytes = kConvBlockM * kConvBlockK * 2;    // 16 KiB per stage
constexpr uint32_t kRingBudget = 192 * 1024;                   // operand ring (+ barriers + GN coefficients <= 227 KB)
constexpr uint32_t kAuxBytes = 512;                            // barriers [0, 256), GroupNorm mean / rstd [256, 512)
constexpr uint32_t kSmemMax = 227 * 1024;
// register split of the TMA kernel: 128 * 40 + 256 * 232 <= 64K registers per SM
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
static_assert(128 * kProducerRegs + 256 * kConsumerRegs <= 65536, "register file overcommitted");
// ping-pong turn-taking: named barrier kTurnBar + c releases consumer c into its next mainloop (id 1 is the GroupNorm
// producer's)
constexpr int kTurnBar = 2;
// statistics reduction of the ping-pong tiles: named barrier kStatBar + c syncs consumer c's four warps around the scratch
// that follows the aux block, [2 consumers][4 warps][BLOCK_N / 16 blocks][sum, sum of squares] doubles
constexpr int kStatBar = 4;
constexpr uint32_t stat_scratch_bytes(int block_n) { return 2 * 4 * (block_n / 16 > 0 ? block_n / 16 : 1) * 2 * 8; }

template <int BLOCK_N>
struct Cfg {
    static constexpr uint32_t kBBytes = BLOCK_N * kConvBlockK * 2;
    static constexpr uint32_t kStageBytes = kABytes + kBBytes;
    static constexpr int kStages = (kRingBudget / kStageBytes) > 8 ? 8 : (kRingBudget / kStageBytes);
    static constexpr uint32_t kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + kAuxBytes;   // + 8 * C_in (GN)
};

__device__ __forceinline__ float silu(float v) { return __fdividef(v, 1.0f + __expf(-v)); }

template <int BLOCK_N, bool GN, bool TR = false>
__global__ void __launch_bounds__(kNumThreads, 1)
conv_wg_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
               const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmX,
               const __grid_constant__ CUtensorMap tmX2, const __grid_constant__ ConvTcArgs args,
               const __grid_constant__ GnPrologueArgs gn) {
    using C = Cfg<BLOCK_N>;
    constexpr int STAGES = C::kStages;
    static_assert(2 * STAGES * 8 <= 256, "barrier block overlaps the GroupNorm scratch");
    static_assert(!TR || (BLOCK_N == 256 && !GN), "the transposed tile is the cooperative 256-wide one");
    constexpr bool PP = !GN && !TR && BLOCK_N <= 128;    // ping-pong schedule (else cooperative)
    constexpr int HALVES = PP ? 2 : 1;            // 64-row halves of a tile one consumer computes
    constexpr int TILE_PIX = TR ? BLOCK_N : kConvBlockM;   // pixels per tile

    extern __shared__ uint8_t smem_raw[];
    // SWIZZLE_128B operands need 1024-byte aligned stage bases
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * C::kStageBytes);
    uint64_t* full_bar = bars;                    // [STAGES]  producer -> consumers
    uint64_t* empty_bar = bars + STAGES;          // [STAGES]  consumers -> producer (one arrival per consuming warpgroup)

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int wg = threadIdx.x >> 7;
    int* err = args.err_flag;

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&tmB);
        if (!GN) {
            ptx::prefetch_tensormap(&tmA);
            ptx::prefetch_tensormap(&tmA2);
        }
        for (int i = 0; i < STAGES; ++i) {
            // GN: the four producer warps' arrivals + the weight load's expect_tx arrival
            ptx::mbar_init(&full_bar[i], GN ? 5 : 1);
            ptx::mbar_init(&empty_bar[i], PP ? 1 : 2);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();      // everything above is independent of the previous kernel's output

    const int num_tap_kb = args.num_taps * args.chunks_per_tap;
    const int num_kb = num_tap_kb + args.x_chunks;
    const int tiles_m = args.tiles_w * args.tiles_h * args.tiles_b;
    const int total_tiles = tiles_m * args.tiles_n;
    const int BW = 1 << args.bw_log2, BH = 1 << args.bh_log2;
    const int BB = TILE_PIX >> (args.bw_log2 + args.bh_log2);

    if (wg == 0) {
        if constexpr (!GN) {
            // ===================== TMA producer (warp 0 stays converged, one elected lane issues) =====================
            ptx::setmaxnreg_dec<kProducerRegs>();
            if (warp == 0) {
                int stage = 0;
                uint32_t phase = 0;
                for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                    const int nt = tile % args.tiles_n;
                    const int mt = tile / args.tiles_n;
                    const int w0 = (mt % args.tiles_w) * BW;
                    const int h0 = ((mt / args.tiles_w) % args.tiles_h) * BH;
                    const int b0 = (mt / (args.tiles_w * args.tiles_h)) * BB;
                    const int n0 = nt * BLOCK_N;
                    for (int kb = 0; kb < num_kb; ++kb) {
                        ptx::mbar_wait(&empty_bar[stage], phase ^ 1, err, 100 + stage);
                        if (ptx::elect_one()) {
                            // transposed: the 128-channel weight tile is the wgmma A operand (16 KiB slot), the
                            // 256-pixel activation tile the B operand
                            uint8_t* sa = smem + stage * C::kStageBytes + (TR ? kABytes : 0);
                            uint8_t* sb = smem + stage * C::kStageBytes + (TR ? 0 : kABytes);
                            ptx::mbar_arrive_expect_tx(&full_bar[stage], C::kStageBytes);
                            if (kb < num_tap_kb) {
                                const int t = kb / args.chunks_per_tap, j = kb - t * args.chunks_per_tap;
                                const int cw = w0 * args.in_stride + args.dw[t], ch = h0 * args.in_stride + args.dh[t];
                                if (j < args.a_split)
                                    ptx::tma_load_5d(&tmA, &full_bar[stage], sa, args.a_chan_off + j * kConvBlockK, cw, ch,
                                                     args.ph[t], b0);
                                else   // second half of a virtual channel concat (skip connection)
                                    ptx::tma_load_5d(&tmA2, &full_bar[stage], sa,
                                                     args.a_chan_off2 + (j - args.a_split) * kConvBlockK, cw, ch, args.ph[t], b0);
                            } else {   // folded 1x1 conv: k-chunk jx of x at the centre tap
                                const int jx = kb - num_tap_kb;
                                if (jx < args.x_split)
                                    ptx::tma_load_5d(&tmX, &full_bar[stage], sa, args.x_chan_off + jx * kConvBlockK, w0, h0, 0, b0);
                                else
                                    ptx::tma_load_5d(&tmX2, &full_bar[stage], sa,
                                                     args.x_chan_off2 + (jx - args.x_split) * kConvBlockK, w0, h0, 0, b0);
                            }
                            ptx::tma_load_2d(&tmB, &full_bar[stage], sb, kb * kConvBlockK, n0);
                        }
                        if (++stage == STAGES) { stage = 0; phase ^= 1; }
                    }
                }
                pdl_trigger();      // last loads issued: the next kernel may be scheduled behind this one's final tile(s)
            }
        } else {
            // ===================== GroupNorm / FiLM / SiLU producer: fp32 global -> fp16 swizzled A tile =====================
            // A tile row m (pixel) occupies bytes [128 m, 128 m + 128); its 16-byte chunk q (channels 8q .. 8q+7) sits at
            // position q ^ (m & 7) -- the layout TMA's SWIZZLE_128B writes, so the consumers are the same for both producers.
            float* s_mean = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);   // [32]
            float* s_rstd = s_mean + 32;                                                        // [32]
            float* sA = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + kAuxBytes); // A[C] then Bc[C]
            const int tt = threadIdx.x;                 // 0..127
            const int lq = tt & 7;                      // channels [8 lq, 8 lq + 8) of the k-chunk
            const int prow = tt >> 3;                   // rows prow + 16 i, i = 0..7
            const int C0 = gn.C0, C1 = gn.C1, Ctot = C0 + C1, Cg = Ctot / gn.groups;
            const int H = args.H, W = args.W;
            float* sB = sA + Ctot;
            int stage = 0;
            uint32_t phase = 0;
            int cur_b = -1;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int nt = tile % args.tiles_n;
                const int mt = tile / args.tiles_n;
                const int w0 = (mt % args.tiles_w) * BW;
                const int h0 = ((mt / args.tiles_w) % args.tiles_h) * BH;
                const int b = mt / (args.tiles_w * args.tiles_h);      // one image per tile (H * W >= 128)
                const int n0 = nt * BLOCK_N;
                if (b != cur_b) {
                    // coefficient table of image b for all input channels: y = SiLU(x * A[c] + Bc[c]) (the arithmetic of
                    // gn_apply_silu_kernel); rebuilt only when the image changes
                    ptx::bar_sync(1, 128);                 // every producer thread has finished reading the previous table
                    if (tt < gn.groups) {
                        const int g = tt;
                        double su = 0.0, sq = 0.0;
                        const int lo = g * Cg, hi = lo + Cg;
                        const int lo0 = min(lo, C0), hi0 = min(hi, C0);
                        for (int e = lo0 / 16; e < hi0 / 16; ++e) {
                            su += gn.stats0[((long long)b * (C0 / 16) + e) * 2];
                            sq += gn.stats0[((long long)b * (C0 / 16) + e) * 2 + 1];
                        }
                        const int lo1 = max(lo, C0) - C0, hi1 = max(hi, C0) - C0;
                        for (int e = lo1 / 16; e < hi1 / 16; ++e) {
                            su += (double)gn.scale1 * gn.stats1[((long long)b * (C1 / 16) + e) * 2];
                            sq += (double)gn.scale1 * (double)gn.scale1 * gn.stats1[((long long)b * (C1 / 16) + e) * 2 + 1];
                        }
                        const double n = (double)Cg * H * W;
                        const double mean = su / n;
                        double var = sq / n - mean * mean;
                        if (var < 0) var = 0;
                        s_mean[g] = (float)mean;
                        s_rstd[g] = (float)(1.0 / sqrt(var + (double)gn.eps));
                    }
                    ptx::bar_sync(1, 128);
                    for (int cc = tt; cc < Ctot; cc += 128) {
                        const int g = cc / Cg;
                        float a = s_rstd[g] * gn.gamma[cc];
                        float bb = gn.beta[cc] - s_mean[g] * a;
                        if (gn.scale_shift) {
                            const float sc = gn.scale_shift[(long long)b * gn.ss_ld + cc] + 1.0f;
                            const float shv = gn.scale_shift[(long long)b * gn.ss_ld + Ctot + cc];
                            a *= sc;
                            bb = bb * sc + shv;
                        }
                        if (cc >= C0) a *= gn.scale1;                     // skip * 2^-1/2 folded into the multiplier
                        sA[cc] = a;
                        sB[cc] = bb;
                    }
                    cur_b = b;
                    ptx::bar_sync(1, 128);
                }
                const long long img = (long long)b * H * W;
                for (int kb = 0; kb < num_kb; ++kb) {
                    const int t = kb / args.chunks_per_tap, j = kb - t * args.chunks_per_tap;
                    const int dh = args.dh[t], dw = args.dw[t];
                    const float* cA = sA + j * kConvBlockK + lq * 8;
                    const float* cB = sB + j * kConvBlockK + lq * 8;
                    const float4 a0 = *reinterpret_cast<const float4*>(cA), a1 = *reinterpret_cast<const float4*>(cA + 4);
                    const float4 b0 = *reinterpret_cast<const float4*>(cB), b1 = *reinterpret_cast<const float4*>(cB + 4);
                    const bool first = j < args.a_split;
                    const int Cs = first ? C0 : C1;
                    const float* src = (first ? gn.src0 + (long long)j * kConvBlockK
                                              : gn.src1 + (long long)(j - args.a_split) * kConvBlockK) + img * Cs + lq * 8;

                    ptx::mbar_wait(&empty_bar[stage], phase ^ 1, err, 600 + stage);
                    uint8_t* sa = smem + stage * C::kStageBytes;
                    if (warp == 0 && ptx::elect_one()) {
                        ptx::mbar_arrive_expect_tx(&full_bar[stage], C::kBBytes);
                        ptx::tma_load_2d(&tmB, &full_bar[stage], sa + kABytes, kb * kConvBlockK, n0);
                    }
                    float4 x0[8], x1[8];
                    bool ok[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int m = i * 16 + prow;
                        const int gw = w0 + (m & (BW - 1)) + dw;
                        const int gh = h0 + ((m >> args.bw_log2) & (BH - 1)) + dh;
                        ok[i] = gh >= 0 && gh < H && gw >= 0 && gw < W;
                        if (ok[i]) {
                            const float4* s4 = reinterpret_cast<const float4*>(src + ((long long)gh * W + gw) * Cs);
                            x0[i] = __ldg(s4);
                            x1[i] = __ldg(s4 + 1);
                        }
                    }
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int m = i * 16 + prow;
                        uint4 o = make_uint4(0u, 0u, 0u, 0u);
                        if (ok[i]) {
                            const __half2 h0_ = sat_half2(silu(fmaf(x0[i].x, a0.x, b0.x)), silu(fmaf(x0[i].y, a0.y, b0.y)));
                            const __half2 h1_ = sat_half2(silu(fmaf(x0[i].z, a0.z, b0.z)), silu(fmaf(x0[i].w, a0.w, b0.w)));
                            const __half2 h2_ = sat_half2(silu(fmaf(x1[i].x, a1.x, b1.x)), silu(fmaf(x1[i].y, a1.y, b1.y)));
                            const __half2 h3_ = sat_half2(silu(fmaf(x1[i].z, a1.z, b1.z)), silu(fmaf(x1[i].w, a1.w, b1.w)));
                            o.x = *reinterpret_cast<const uint32_t*>(&h0_); o.y = *reinterpret_cast<const uint32_t*>(&h1_);
                            o.z = *reinterpret_cast<const uint32_t*>(&h2_); o.w = *reinterpret_cast<const uint32_t*>(&h3_);
                        }
                        *reinterpret_cast<uint4*>(sa + m * 128 + ((lq ^ (m & 7)) << 4)) = o;
                    }
                    ptx::fence_proxy_async_smem();        // generic-proxy stores -> visible to wgmma (async proxy)
                    __syncwarp();
                    if (lane == 0) ptx::mbar_arrive(&full_bar[stage]);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
            pdl_trigger();
        }
    } else {
        // ===================== consumers: rows [64 cw, 64 cw + 64) of every tile (cooperative), or every row of the
        // ===================== CTA's tiles cw, cw + 2, ... (ping-pong)
        if constexpr (!GN) ptx::setmaxnreg_inc<kConsumerRegs>();
        const int cw = wg - 1;
        const int wq = warp & 3;                        // warp inside the warpgroup: rows 16 wq .. 16 wq + 15 of a half
        const int cq = 2 * (lane & 3);                  // first of this thread's two columns in every 8-column group
        float acc[HALVES][BLOCK_N / 2];
        int stage = 0;
        uint32_t phase = 0;
        // moves the ring position n k-blocks on: in ping-pong, past the other consumer's tile
        auto skip = [&](int n) {
            stage += n % STAGES;
            phase ^= (uint32_t)(n / STAGES) & 1u;
            if (stage >= STAGES) { stage -= STAGES; phase ^= 1; }
        };
        if (PP) skip(cw * num_kb);
        // epilogue geometry of this thread's rows (m, m + 8) in each of its 64-row halves: row 2 h + r
        int bw_r[2 * HALVES], bh_r[2 * HALVES], bb_r[2 * HALVES], bb_warp[HALVES];
#pragma unroll
        for (int h = 0; h < HALVES; ++h) {
            const int m_warp = (PP ? h : cw) * 64 + wq * 16;   // the warp's 16 rows belong to one image (stats need
            bb_warp[h] = m_warp >> (args.bw_log2 + args.bh_log2);   // H*W % 32 == 0); the two halves may not
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int m = m_warp + (lane >> 2) + 8 * r;
                bw_r[2 * h + r] = m & (BW - 1);
                bh_r[2 * h + r] = (m >> args.bw_log2) & (BH - 1);
                bb_r[2 * h + r] = m >> (args.bw_log2 + args.bh_log2);
            }
        }
        // ping-pong, one image per tile: the statistics of a tile's rows are summed over the warpgroup in shared memory.
        // Cooperative tiles keep per-warp atomics: the two extra warpgroup barriers per tile cost cfg 3 0.3-0.6 ms per
        // step there (64.1-64.3 vs 63.6-63.8 ms on an H100 SXM at 700 W)
        constexpr int NQ = BLOCK_N / 16 > 0 ? BLOCK_N / 16 : 1;
        const bool tile_stats = PP && args.stats != nullptr && BB == 1;
        double* st_red = reinterpret_cast<double*>(reinterpret_cast<uint8_t*>(bars) + kAuxBytes);   // [2][4][NQ][2]
        const bool vec = args.out_sc == 1 && ((reinterpret_cast<uintptr_t>(args.out_f32) & 7) == 0) &&
                         ((reinterpret_cast<uintptr_t>(args.residual) & 7) == 0) &&
                         ((reinterpret_cast<uintptr_t>(args.out_f16) & 3) == 0);

        for (int tile = blockIdx.x + (PP ? cw : 0) * gridDim.x; tile < total_tiles; tile += (PP ? 2 : 1) * gridDim.x) {
            const int nt = tile % args.tiles_n;
            const int mt = tile / args.tiles_n;
            const int n0 = nt * BLOCK_N;
            // Ping-pong turn: start this tile's mainloop only once the other consumer has waited on every k-block of the
            // CTA's previous tile.  Every k-block before this tile then has been loaded, so each full_bar this mainloop
            // waits on is at most one phase behind the one it waits for, and the parity wait cannot succeed on a phase
            // two fills old (the previous tile's operands): skip() jumps a whole tile of ring slots, so without the turn
            // a slot's previous fill could still be pending, in the other consumer's tile.  The turns also keep the two
            // mainloops from sharing the tensor cores; the epilogues overlap the other mainloop.
            if (PP && tile != (int)blockIdx.x) ptx::bar_sync(kTurnBar + cw, 256);
            int prev = -1;
            for (int kb = 0; kb < num_kb; ++kb) {
                ptx::mbar_wait(&full_bar[stage], phase, err, 300 + stage);
                const uint32_t sa = ptx::smem_u32(smem + stage * C::kStageBytes);
                const uint64_t db = ptx::make_sw128_desc(sa + kABytes);
                ptx::wg_fence();
#pragma unroll
                for (int k = 0; k < kConvBlockK / 16; ++k)
#pragma unroll
                    for (int h = 0; h < HALVES; ++h) {
                        const uint64_t da = ptx::make_sw128_desc(sa + (PP ? h : cw) * (64 * 128));
                        // advance 16 fp16 = 32 B along K inside the swizzle atom: +2 in the (addr >> 4) field
                        ptx::Wgmma<BLOCK_N, 0>::run(acc[h], da + 2 * k, db + 2 * k, (kb | k) != 0);
                    }
                ptx::wg_commit();
                ptx::wg_wait<1>();                      // the previous k-block's MMAs have retired: free its stage
                if (prev >= 0 && (threadIdx.x & 127) == 0) ptx::mbar_arrive(&empty_bar[prev]);
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            // the other consumer's turn, if the CTA has a next tile (so every arrival meets a bar_sync)
            if (PP && tile + (int)gridDim.x < total_tiles) ptx::bar_arrive(kTurnBar + (cw ^ 1), 256);
            if (PP) skip(num_kb);
            ptx::wg_wait<0>();
#pragma unroll
            for (int h = 0; h < HALVES; ++h) ptx::wg_fence_regs(acc[h]);
            if (prev >= 0 && (threadIdx.x & 127) == 0) ptx::mbar_arrive(&empty_bar[prev]);

            // ---- epilogue: fragment element 4j + 2r + e of half h = row (h, r), column n0 + 8j + cq + e
            const int tw0 = (mt % args.tiles_w) * BW;
            const int th0 = ((mt / args.tiles_w) % args.tiles_h) * BH;
            const int tb0 = (mt / (args.tiles_w * args.tiles_h)) * BB;
            if constexpr (TR) {
                // ---- transposed epilogue: fragment element 4j + 2r + e = output channel c0 + 8r, tile pixel 8j + cq + e.
                // The tile is whole and in image tb0, and the warp's values are all in 16-channel block c0 / 16: one
                // statistics pair per warp.  Like the row-major epilogue, a thread sums 8 values in fp32 (then fp64).
                const int c0 = 64 * cw + 16 * wq + (lane >> 2);
                const float bv[2] = {args.bias ? __ldg(args.bias + c0) : 0.f, args.bias ? __ldg(args.bias + c0 + 8) : 0.f};
                const long long base = (long long)tb0 * args.out_sb + (long long)th0 * args.out_sh +
                                       (long long)(tw0 + cq) * args.out_sw + c0;
                float* const o32 = args.out_f32 ? args.out_f32 + base : nullptr;
                __half* const o16 = args.out_f16 ? args.out_f16 + base : nullptr;
                const float* const res = args.residual ? args.residual + base : nullptr;
                // offsets inside a tile fit in 31 bits (host); pixels 8j .. 8j + 7 lie in one tile row (BW >= 8), so
                // the offset of pixel 8j steps by 8 columns, or to the next row where 8j wraps BW
                const int sw = (int)args.out_sw, step = 8 * sw, wrap = (int)args.out_sh - (BW - 8) * sw;
                float* a = acc[0];
                // pass 1: bias and residual into the accumulators.  The residual may be the output buffer itself, so a
                // load cannot move above an earlier store: with no store between them the loads are in flight together
                // instead of each waiting behind the previous element's store
                int oj = 0;
#pragma unroll
                for (int j = 0; j < BLOCK_N / 8; ++j) {
                    if (j > 0) oj += ((8 * j) & (BW - 1)) ? step : wrap;
#pragma unroll
                    for (int r = 0; r < 2; ++r)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            float& f = a[4 * j + 2 * r + e];
                            f += bv[r];
                            if (res) f += res[oj + e * sw + 8 * r];
                        }
                }
                // pass 2: stores and statistics
                const bool stats = args.stats != nullptr;
                double su = 0.0, sq = 0.0;
                oj = 0;
#pragma unroll
                for (int jj = 0; jj < BLOCK_N / 16; ++jj) {
                    float s8 = 0.f, q8 = 0.f;
#pragma unroll
                    for (int j = 2 * jj; j < 2 * jj + 2; ++j) {
                        if (j > 0) oj += ((8 * j) & (BW - 1)) ? step : wrap;
#pragma unroll
                        for (int r = 0; r < 2; ++r) {
                            const float* f = a + 4 * j + 2 * r;
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int o = oj + e * sw + 8 * r;
                                if (o32) o32[o] = f[e];
                                if (o16) o16[o] = sat_half(f[e]);
                            }
                            if (stats) {
                                s8 += f[0] + f[1];
                                q8 += f[0] * f[0] + f[1] * f[1];
                            }
                        }
                    }
                    if (stats) {
                        su += (double)s8;
                        sq += (double)q8;
                    }
                }
                if (stats) {
#pragma unroll
                    for (int o = 1; o <= 16; o <<= 1) {
                        su += __shfl_xor_sync(0xffffffffu, su, o);
                        sq += __shfl_xor_sync(0xffffffffu, sq, o);
                    }
                    if (lane == 0) {
                        double* dst = args.stats + ((long long)tb0 * args.stats_blocks + (c0 >> 4)) * 2;
                        atomicAdd(dst, su);
                        atomicAdd(dst + 1, sq);
                    }
                }
                continue;
            }
            const bool fast = vec && n0 + BLOCK_N <= args.n_valid;
#pragma unroll
            for (int hf = 0; hf < HALVES; ++hf) {
                bool valid[2];
                long long pix[2];
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int w = tw0 + bw_r[2 * hf + r], h = th0 + bh_r[2 * hf + r], b = tb0 + bb_r[2 * hf + r];
                    valid[r] = (b < args.B) && (h < args.H) && (w < args.W);
                    pix[r] = (long long)b * args.out_sb + (long long)h * args.out_sh + (long long)w * args.out_sw;
                }
                const float* a = acc[hf];
                float st_s[BLOCK_N / 16 > 0 ? BLOCK_N / 16 : 1], st_q[BLOCK_N / 16 > 0 ? BLOCK_N / 16 : 1];
#pragma unroll
                for (int q = 0; q < BLOCK_N / 16; ++q) { st_s[q] = 0.f; st_q[q] = 0.f; }
#pragma unroll
                for (int j = 0; j < BLOCK_N / 8; ++j) {
                    const int n = n0 + 8 * j + cq;
                    if (fast) {
                        float2 bv = make_float2(0.f, 0.f);
                        if (args.bias) bv = __ldg(reinterpret_cast<const float2*>(args.bias + n));
#pragma unroll
                        for (int r = 0; r < 2; ++r) {
                            if (!valid[r]) continue;
                            const long long o = pix[r] + n;
                            float2 f = make_float2(a[4 * j + 2 * r] + bv.x, a[4 * j + 2 * r + 1] + bv.y);
                            if (args.residual) {
                                const float2 rv = *reinterpret_cast<const float2*>(args.residual + o);
                                f.x += rv.x; f.y += rv.y;
                            }
                            st_s[j >> 1] += f.x + f.y;
                            st_q[j >> 1] += f.x * f.x + f.y * f.y;
                            if (args.out_f32) *reinterpret_cast<float2*>(args.out_f32 + o) = f;
                            if (args.out_f16) *reinterpret_cast<__half2*>(args.out_f16 + o) = sat_half2(f.x, f.y);
                        }
                    } else {
#pragma unroll
                        for (int r = 0; r < 2; ++r) {
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                if (!valid[r] || n + e >= args.n_valid) continue;
                                float f = a[4 * j + 2 * r + e] + (args.bias ? __ldg(args.bias + n + e) : 0.f);
                                const long long o = pix[r] + (long long)(n + e) * args.out_sc;
                                if (args.residual && args.out_sc == 1) f += args.residual[o];
                                st_s[j >> 1] += f;
                                st_q[j >> 1] += f * f;
                                if (args.out_f32) args.out_f32[o] = f;
                                if (args.out_f16) args.out_f16[o] = sat_half(f);
                            }
                        }
                    }
                }
                if (args.stats) {
                    // GroupNorm statistics of the tensor being written, per (image, 16-channel block): the warp's 16 rows
                    // x 16 columns of each block reduce over all 32 lanes
                    const int b_img = tb0 + bb_warp[hf];
                    const bool any = __any_sync(0xffffffffu, valid[0] || valid[1]);
#pragma unroll
                    for (int q = 0; q < BLOCK_N / 16; ++q) {
#pragma unroll
                        for (int o = 1; o <= 16; o <<= 1) {
                            st_s[q] += __shfl_xor_sync(0xffffffffu, st_s[q], o);
                            st_q[q] += __shfl_xor_sync(0xffffffffu, st_q[q], o);
                        }
                        if (lane == 0 && tile_stats) {
                            double* r = st_red + ((cw * 4 + wq) * NQ + q) * 2;
                            r[0] = (hf == 0 ? 0.0 : r[0]) + (double)st_s[q];
                            r[1] = (hf == 0 ? 0.0 : r[1]) + (double)st_q[q];
                        } else if (lane == 0 && any) {
                            double* dst = args.stats + ((long long)b_img * args.stats_blocks + (n0 >> 4) + q) * 2;
                            atomicAdd(dst, (double)st_s[q]);
                            atomicAdd(dst + 1, (double)st_q[q]);
                        }
                    }
                }
            }
            if (tile_stats) {
                // one atomic pair per (consumer warpgroup, tile, 16-channel block) instead of one per warp and half: every
                // CTA works on the same image at once, and the per-warp atomics queued on its few addresses
                ptx::bar_sync(kStatBar + cw, 128);
                if (wq == 0 && lane < NQ) {
                    const double* r = st_red + (cw * 4 * NQ + lane) * 2;
                    double s = r[0], sq = r[1];
#pragma unroll
                    for (int w = 1; w < 4; ++w) { s += r[w * NQ * 2]; sq += r[w * NQ * 2 + 1]; }
                    double* dst = args.stats + ((long long)tb0 * args.stats_blocks + (n0 >> 4) + lane) * 2;
                    atomicAdd(dst, s);
                    atomicAdd(dst + 1, sq);
                }
                ptx::bar_sync(kStatBar + cw, 128);     // the scratch is read before the next tile writes it
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ host side

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    });
    return fn;
}

int ilog2_exact(int v) {
    int l = 0;
    while ((1 << l) < v) ++l;
    return ((1 << l) == v) ? l : -1;
}

int num_sms_of_current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    static int cache[64] = {0};
    if (dev < 64 && cache[dev] != 0) return cache[dev];
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (dev < 64) cache[dev] = n;
    return n;
}

// Tile box of tile_pix (128, or 256 for the transposed schedule) pixels: BW x BH pixels x BB images, BW and BH powers of
// two.  W a power of two or a multiple of tile_pix: BW = min(W, tile_pix), BH = tile_pix / BW (at most H; a short image
// spans BB images).  Any other W that is a multiple of 8 and whose largest power-of-two divisor BW (< tile_pix) gives
// BH = tile_pix / BW rows dividing H: exact one-image tiles of that box (W = 96: 32 x 4; 48: 16 x 8; 24: 8 x 16 at 128
// pixels).  Otherwise BW = tile_pix, BH = 1 and the last tile of every row is masked (W > tile_pix only).
void tile_box(int H, int W, int tile_pix, int& BW, int& BH) {
    const int low = W & -W;                                  // largest power of two dividing W
    if (low != W && W % tile_pix != 0 && low >= 8 && H % (tile_pix / low) == 0) {
        BW = low;
        BH = tile_pix / low;
        return;
    }
    BW = W >= tile_pix ? tile_pix : W;
    BH = tile_pix / BW;
    if (BH > H) BH = H;
}

void tile_geometry(int H, int W, int B, int tile_pix, ConvTcArgs& a) {
    int BW, BH;
    tile_box(H, W, tile_pix, BW, BH);
    const int BB = tile_pix / (BW * BH);
    a.bw_log2 = ilog2_exact(BW);
    a.bh_log2 = ilog2_exact(BH);
    a.tiles_w = (W + BW - 1) / BW;
    a.tiles_h = H / BH;
    a.tiles_b = (B + BB - 1) / BB;
    a.B = B; a.H = H; a.W = W;
}

// Largest BLOCK_N of {256,128,64,32,16} dividing C_out that still gives every SM a tile; never shrink below 64 for that.
// A 256-wide tile moves 25 % fewer operand bytes per FLOP than a 128-wide one; its 128 accumulators per consumer thread
// fit because of the setmaxnreg split (only the TMA kernel has it: the fused GroupNorm kernel stays 128 wide).
// The width also picks the schedule: 256 is cooperative, <= 128 ping-pong.  Taking the 128-wide ping-pong tile for
// C_out % 256 == 0 at <= 36 k-blocks per tile won 0-7 % per launch at 3x3 -> 256 on 64x64 (tools/bench_ops.py conv, b = 32,
// H100 SXM at a 400 W power limit) but lost 0.2-0.3 ms per cfg-3 step (85.7-85.9 vs 85.4-85.7 ms), so it is not used.
int pick_block_n(int Cout, int tiles_m, int hint, int num_sms) {
    const int cands[5] = {256, 128, 64, 32, 16};
    if (hint < 0) hint = -hint;
    if (hint > 0 && Cout % hint == 0)
        for (int i = 0; i < 5; ++i)
            if (cands[i] == hint) return hint;
    int block_n = 16;
    for (int i = 0; i < 5; ++i) {
        if (Cout % cands[i] != 0) continue;
        block_n = cands[i];
        if (tiles_m * (Cout / cands[i]) >= num_sms || cands[i] <= 64) break;
    }
    return block_n;
}

CUresult encode_act(PFN_encodeTiled enc, CUtensorMap* m, const void* ptr, cuuint64_t channels, cuuint64_t ld, int W, int H,
                    int phases, int B, int in_stride, int tile_pix, const ConvTcArgs& a) {
    // (C, W, H, P, B), fp16, box (64, BW, BH, 1, BB), 128B swizzle, OOB -> zeros.  in_stride == 2 (Downsample read in place):
    // the tensor is the (2H x 2W) input, the box spans 2*BW x 2*BH pixels and the element strides make TMA keep every second
    // pixel -> the same tile_pix-pixel tile lands in shared memory
    const cuuint64_t IS = in_stride;
    const int BW = 1 << a.bw_log2, BH = 1 << a.bh_log2, BB = tile_pix >> (a.bw_log2 + a.bh_log2);
    cuuint64_t gdim[5] = {channels, (cuuint64_t)W * IS, (cuuint64_t)H * IS, (cuuint64_t)phases, (cuuint64_t)B};
    cuuint64_t gstr[4] = {ld * 2, (cuuint64_t)W * IS * ld * 2, (cuuint64_t)H * IS * W * IS * ld * 2,
                          (cuuint64_t)phases * H * IS * W * IS * ld * 2};
    cuuint32_t box[5] = {kConvBlockK, (cuuint32_t)(BW * IS), (cuuint32_t)(BH * IS), 1, (cuuint32_t)BB};
    cuuint32_t estr[5] = {1, (cuuint32_t)IS, (cuuint32_t)IS, 1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(ptr), gdim, gstr, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

CUresult encode_weights(PFN_encodeTiled enc, CUtensorMap* m, const void* ptr, cuuint64_t K, int Cout, int block_n) {
    cuuint64_t gdim[2] = {K, (cuuint64_t)Cout};
    cuuint64_t gstr[1] = {K * 2};
    cuuint32_t box[2] = {kConvBlockK, (cuuint32_t)block_n};
    cuuint32_t estr[2] = {1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), gdim, gstr, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

// The transposed schedule computes D^T[C_out = 128, pixels] = W . A^T on the cooperative 256-wide kernel: the weight tile
// is the wgmma A operand (M = the 128 output channels, 64 per consumer) and a 256-pixel activation tile the B operand
// (N = 256), so a C_out = 128 conv gets the 128x256 tile's operand bytes per FLOP.  It needs whole 256-pixel tiles inside
// one image (the statistics of a warp then fall in one image), TMA boxes of <= 256 pixels per dimension (the in-place
// stride-2 read doubles them), and every channel stored channel-contiguous (its stores go 8 channels x 4 pixels a warp).
bool transposed_ok(const ConvTcProblem& p, const ConvTcArgs& a) {
    if (p.Cout != 128 || a.n_valid != p.Cout || a.out_sc != 1) return false;
    int BW, BH;
    tile_box(p.H, p.W, 256, BW, BH);
    if (p.W % BW || ilog2_exact(BW) < 3 || BW * a.in_stride > 256 || BW * BH != 256) return false;
    // the epilogue addresses a tile's outputs with 32-bit offsets from its first pixel
    if (BH * a.out_sh + BW * a.out_sw + p.Cout > INT32_MAX) return false;
    return p.H % BH == 0 && BH * a.in_stride <= 256;
}

template <int BLOCK_N, bool GN, bool TR = false>
int launch(const CUtensorMap& tmA, const CUtensorMap& tmA2, const CUtensorMap& tmB, const CUtensorMap& tmX,
           const CUtensorMap& tmX2, const ConvTcArgs& args, const GnPrologueArgs& gn, uint32_t extra_smem,
           cudaStream_t stream) {
    using C = Cfg<BLOCK_N>;
    static bool attr_set = false;   // per-template-instance; benign race (idempotent call)
    if (!attr_set) {
        if (cudaFuncSetAttribute(conv_wg_kernel<BLOCK_N, GN, TR>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax) !=
            cudaSuccess)
            return -10;
        attr_set = true;
    }
    const int total_tiles = args.tiles_w * args.tiles_h * args.tiles_b * args.tiles_n;
    const int num_sms = num_sms_of_current_device();
    const int grid = total_tiles < num_sms ? total_tiles : num_sms;
    const uint32_t smem = C::kSmemBytes + (!GN && !TR && BLOCK_N <= 128 ? stat_scratch_bytes(BLOCK_N) : 0u) + extra_smem;
    launch_k(conv_wg_kernel<BLOCK_N, GN, TR>, grid, kNumThreads, smem, stream, tmA, tmA2, tmB, tmX, tmX2, args, gn);
    return cudaGetLastError() == cudaSuccess ? 0 : -11;
}

}  // namespace

PFN_tmaEncodeTiled get_tma_encode() { return get_encode(); }

const char* conv_tc_strerror(int code) {
    switch (code) {
        case 0: return "ok";
        case -1: return "conv_tc: C_in (per tap) must be a positive multiple of 64";
        case -2: return "conv_tc: C_out must be a multiple of 16";
        case -3: return "conv_tc: W must be >= 128, a power of two >= 8, or a multiple of 8 whose largest power-of-two divisor BW gives " \
                       "128 / BW rows dividing H";
        case -4: return "conv_tc: too many taps (max 16)";
        case -5: return "conv_tc: cuTensorMapEncodeTiled unavailable";
        case -6: return "conv_tc: tensor map encode failed (activations)";
        case -7: return "conv_tc: tensor map encode failed (weights)";
        case -8: return "conv_tc: pointer/stride alignment (16 B) violated";
        case -9: return "conv_tc: the folded 1x1 operand needs a stride-1 conv over one phase";
        case -10: return "conv_tc: cudaFuncSetAttribute(max dynamic smem) failed";
        case -11: return "conv_tc: kernel launch failed";
        default: return "conv_tc: unknown error";
    }
}

bool conv_tc_supported(int H, int W, int Cin, int Cout) {
    if (Cin <= 0 || Cin % kConvBlockK != 0 || Cout <= 0 || Cout % 16 != 0) return false;
    if (W >= 128) return true;                            // BW = 128, BH = 1, or an exact box (tile_box); else ragged
    if (ilog2_exact(W) < 0) {                             // W % 8 == 0: BW = W & -W, BH = 128 / BW rows of one image
        const int low = W & -W;
        return W > 0 && low >= 8 && H % (128 / low) == 0;
    }
    if (W < 8) return false;                              // W in {8,16,32,64}
    const int bh = 128 / W;
    if (H >= bh) return H % bh == 0;                      // BH = 128 / W rows of one image
    return ilog2_exact(H) >= 0;                           // BH = H, the tile spans 128 / (W*H) images
}

int conv_tc_launch(const ConvTcProblem& p, cudaStream_t stream) {
    if (p.Cin <= 0 || p.Cin % kConvBlockK != 0) return -1;
    if (p.Cout % 16 != 0) return -2;
    if (p.num_taps < 1 || p.num_taps > kConvMaxTaps) return -4;
    if (!conv_tc_supported(p.H, p.W, p.Cin, p.Cout)) return -3;
    if ((reinterpret_cast<uintptr_t>(p.act) & 15) || (reinterpret_cast<uintptr_t>(p.wpacked) & 15) ||
        (p.lda % 8) != 0)
        return -8;
    PFN_encodeTiled enc = get_encode();
    if (!enc) return -5;

    ConvTcArgs a{};
    a.num_taps = p.num_taps;
    a.chunks_per_tap = p.Cin / kConvBlockK;
    a.a_chan_off = p.a_chan_off;
    a.in_stride = p.in_stride == 2 ? 2 : 1;
    a.out_sb = p.out_sb; a.out_sh = p.out_sh; a.out_sw = p.out_sw;
    a.out_sc = p.out_sc > 0 ? p.out_sc : 1;
    a.n_valid = p.n_valid > 0 ? p.n_valid : p.Cout;
    a.out_f32 = p.out_f32; a.out_f16 = p.out_f16; a.bias = p.bias; a.residual = p.residual;
    a.err_flag = p.err_flag;
    a.stats = p.stats; a.stats_blocks = p.Cout / 16;
    for (int t = 0; t < p.num_taps; ++t) { a.dh[t] = p.dh[t]; a.dw[t] = p.dw[t]; a.ph[t] = p.ph[t]; }

    // schedule: the block_n hint 256 asks for the transposed one at C_out = 128, any other width the row-major tiles.
    // Without a hint the transposed schedule runs where it applies and gives every SM a tile: on an H100 SXM at 700 W
    // every cfg-3 C_out = 128 class measured faster on it, the sub-pixel phases and the residual (block2) epilogue
    // included (tools/bench_ops.py conv 256 128)
    const int num_sms = num_sms_of_current_device();
    const int hint = p.block_n_hint < 0 ? -p.block_n_hint : p.block_n_hint;
    const bool tr_ok = transposed_ok(p, a);
    const bool tr = hint == 256 ? tr_ok
                                : (hint == 0 || p.Cout % hint != 0) && tr_ok && (long long)p.B * p.H * p.W / 256 >= num_sms;
    const int tile_pix = tr ? 256 : kConvBlockM;
    tile_geometry(p.H, p.W, p.B, tile_pix, a);
    const int tiles_m = a.tiles_w * a.tiles_h * a.tiles_b;
    const int block_n = tr ? 128 : pick_block_n(p.Cout, tiles_m, p.block_n_hint, num_sms);
    a.tiles_n = p.Cout / block_n;

    CUtensorMap tmA, tmA2, tmB, tmX, tmX2;
    a.a_split = (p.act2 ? p.Cin1 : p.Cin) / kConvBlockK;
    a.a_chan_off2 = p.a_chan_off2;
    if (encode_act(enc, &tmA, p.act, p.a_channels, p.lda, p.W, p.H, p.phases, p.B, a.in_stride, tile_pix, a) != CUDA_SUCCESS)
        return -6;
    tmA2 = tmA;
    if (p.act2) {
        if (p.Cin1 <= 0 || p.Cin1 % kConvBlockK || p.Cin1 >= p.Cin || (p.lda2 % 8) || (reinterpret_cast<uintptr_t>(p.act2) & 15) ||
            a.in_stride != 1)
            return -8;
        if (encode_act(enc, &tmA2, p.act2, p.lda2, p.lda2, p.W, p.H, p.phases, p.B, 1, tile_pix, a) != CUDA_SUCCESS) return -6;
    }
    // folded 1x1 conv over a second operand x (res_conv): its own tensor map(s), read at the centre tap
    tmX = tmA; tmX2 = tmA;
    if (p.x_act) {
        if (p.phases != 1 || a.in_stride != 1) return -9;
        if (p.Cx <= 0 || p.Cx % kConvBlockK || (p.x_lda % 8) || (reinterpret_cast<uintptr_t>(p.x_act) & 15)) return -8;
        if (p.x_act2 && (p.Cx1 <= 0 || p.Cx1 % kConvBlockK || p.Cx1 >= p.Cx || (p.x_lda2 % 8) ||
                         (reinterpret_cast<uintptr_t>(p.x_act2) & 15)))
            return -8;
        a.x_chunks = p.Cx / kConvBlockK;
        a.x_split = (p.x_act2 ? p.Cx1 : p.Cx) / kConvBlockK;
        a.x_chan_off = p.x_chan_off; a.x_chan_off2 = p.x_chan_off2;
        if (encode_act(enc, &tmX, p.x_act, p.x_lda, p.x_lda, p.W, p.H, 1, p.B, 1, tile_pix, a) != CUDA_SUCCESS) return -6;
        tmX2 = tmX;
        if (p.x_act2 &&
            encode_act(enc, &tmX2, p.x_act2, p.x_lda2, p.x_lda2, p.W, p.H, 1, p.B, 1, tile_pix, a) != CUDA_SUCCESS)
            return -6;
    }
    const cuuint64_t K = (cuuint64_t)p.num_taps * p.Cin + (p.x_act ? (cuuint64_t)p.Cx : 0);
    if (encode_weights(enc, &tmB, p.wpacked, K, p.Cout, block_n) != CUDA_SUCCESS) return -7;

    const GnPrologueArgs gn{};
    if (tr) return launch<256, false, true>(tmA, tmA2, tmB, tmX, tmX2, a, gn, 0, stream);
    switch (block_n) {
        case 256: return launch<256, false>(tmA, tmA2, tmB, tmX, tmX2, a, gn, 0, stream);
        case 128: return launch<128, false>(tmA, tmA2, tmB, tmX, tmX2, a, gn, 0, stream);
        case 64: return launch<64, false>(tmA, tmA2, tmB, tmX, tmX2, a, gn, 0, stream);
        case 32: return launch<32, false>(tmA, tmA2, tmB, tmX, tmX2, a, gn, 0, stream);
        default: return launch<16, false>(tmA, tmA2, tmB, tmX, tmX2, a, gn, 0, stream);
    }
}

// ------------------------------------------------------------------------------------------------ fused GroupNorm conv

bool conv_gn_supported(int H, int W, int C0, int C1, int Cout, int groups) {
    const int C = C0 + C1;
    if (H <= 0 || W <= 0 || H % 32 || W % 8 || C0 <= 0 || C0 % 64 || C1 < 0 || C1 % 64 || Cout <= 0 || Cout % 128) return false;
    if (!conv_tc_supported(H, W, C, Cout) || H * W < kConvBlockM) return false;   // one image per 128-pixel tile
    if (groups < 1 || groups > 32 || C % groups) return false;
    if (Cfg<128>::kSmemBytes + 8u * (uint32_t)C > kSmemMax) return false;        // coefficient table A[C], Bc[C]
    return (C / groups) % 16 == 0;
}

int conv_gn_launch(const ConvGnProblem& p, cudaStream_t stream) {
    if (!conv_gn_supported(p.H, p.W, p.C0, p.C1, p.Cout, p.groups)) return -3;
    if (p.C1 && (!p.src1 || !p.stats1)) return -8;
    if (!p.src0 || !p.stats0 || !p.gamma || !p.beta) return -8;
    if ((reinterpret_cast<uintptr_t>(p.src0) & 15) || (reinterpret_cast<uintptr_t>(p.src1) & 15) ||
        (reinterpret_cast<uintptr_t>(p.wpacked) & 15))
        return -8;
    PFN_encodeTiled enc = get_encode();
    if (!enc) return -5;
    const int C = p.C0 + p.C1;

    ConvTcArgs a{};
    a.num_taps = 9;
    for (int t = 0; t < 9; ++t) { a.dh[t] = (int8_t)(t / 3 - 1); a.dw[t] = (int8_t)(t % 3 - 1); a.ph[t] = 0; }
    a.chunks_per_tap = C / kConvBlockK;
    a.a_split = p.C0 / kConvBlockK;
    a.in_stride = 1;
    tile_geometry(p.H, p.W, p.B, kConvBlockM, a);
    a.out_sb = (long long)p.H * p.W * p.Cout; a.out_sh = (long long)p.W * p.Cout; a.out_sw = p.Cout; a.out_sc = 1;
    a.n_valid = p.Cout;
    a.out_f32 = p.out_f32; a.out_f16 = p.out_f16; a.bias = p.bias; a.residual = p.residual; a.err_flag = p.err_flag;
    a.stats = p.out_stats; a.stats_blocks = p.Cout / 16;
    a.tiles_n = p.Cout / 128;

    GnPrologueArgs g{};
    g.src0 = p.src0; g.src1 = p.src1;
    g.C0 = p.C0; g.C1 = p.C1; g.groups = p.groups; g.scale1 = p.scale1; g.eps = p.eps;
    g.stats0 = p.stats0; g.stats1 = p.stats1; g.gamma = p.gamma; g.beta = p.beta;
    g.scale_shift = p.scale_shift; g.ss_ld = p.ss_ld;

    CUtensorMap tmB;
    if (encode_weights(enc, &tmB, p.wpacked, (cuuint64_t)9 * C, p.Cout, 128) != CUDA_SUCCESS) return -7;
    return launch<128, true>(tmB, tmB, tmB, tmB, tmB, a, g, 8u * (uint32_t)C, stream);
}

}  // namespace mi
