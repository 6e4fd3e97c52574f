// Host/device interface of the wgmma implicit-GEMM convolution (see conv_tc.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mi {

constexpr int kConvBlockM = 128;   // pixels per tile (two 64-row wgmma warpgroups)
constexpr int kConvBlockK = 64;    // fp16 channels per k-block (= one 128-byte swizzle row)
constexpr int kConvMaxTaps = 16;   // 4x4 kernel

// Kernel-side arguments (passed as one __grid_constant__ struct).
struct ConvTcArgs {
    int num_taps, chunks_per_tap;
    int bw_log2, bh_log2;                 // tile box: BW x BH pixels x BB images, BW*BH*BB == 128
    int tiles_w, tiles_h, tiles_b, tiles_n;
    int B, H, W;                          // output pixel grid (== TMA pixel grid of every phase)
    int a_chan_off;                       // first input channel inside the activation buffer
    int in_stride;                        // 1, or 2: taps address the (2H x 2W) input directly (TMA element stride 2)
    int a_split, a_chan_off2;             // k-chunks >= a_split come from the second activation tensor (virtual concat)
    int x_chunks, x_split;                // folded 1x1 conv (ResnetBlock.res_conv): extra k-chunks of a second operand x,
    int x_chan_off, x_chan_off2;          //   read at the centre tap; chunks >= x_split come from its second tensor (concat)
    long long out_sb, out_sh, out_sw;     // output (and residual) strides in elements
    long long out_sc;                     // channel stride (1 = NHWC-style contiguous channels; H*W for NCHW output)
    int n_valid;                          // channels >= n_valid are computed (zero-padded weights) but not stored
    float* out_f32;                       // optional
    __half* out_f16;                      // optional
    const float* bias;                    // optional, [C_out]
    const float* residual;                // optional, fp32, same strides as the output
    int* err_flag;                        // optional: pipeline-timeout code is written here before trapping
    double* stats;                        // optional [B][C_out/16][2]: (sum, sum of squares) of the output per 16-channel block
    int stats_blocks;                     // C_out / 16
    int8_t dh[kConvMaxTaps], dw[kConvMaxTaps], ph[kConvMaxTaps];
};

// Host-side problem description.
struct ConvTcProblem {
    const void* act;        // fp16 activations, layout [B][phases][H][W][lda]
    int B, H, W;            // pixel grid of each phase == output pixel grid
    int phases;             // 1, or 4 for the phase-split input of a stride-2 conv
    int in_stride;          // 0/1, or 2: act is the un-split [B][2H][2W][lda] input of a stride-2 conv; dh/dw are full-res offsets
    int lda;                // elements per pixel in the activation buffer (>= a_chan_off + Cin)
    int a_channels;         // channel extent visible to TMA (usually lda)
    int a_chan_off;         // first channel used
    int Cin;                // channels per tap
    const void* act2;       // optional second activation tensor: channels [Cin1, Cin) of every tap come from it
    int lda2, a_chan_off2, Cin1;
    const void* wpacked;    // fp16 [Cout][num_taps*Cin (+ Cx)]
    int Cout;
    // optional folded 1x1 conv over a second operand x (stride-1 convs): out += W1x1 x, with the 1x1 weights
    // appended to every row of wpacked as Cx extra K columns; x may itself be a virtual concat (x_act2 holds channels >= Cx1)
    const void* x_act; int x_lda, x_chan_off, Cx;
    const void* x_act2; int x_lda2, x_chan_off2, Cx1;
    int num_taps;
    int8_t dh[kConvMaxTaps], dw[kConvMaxTaps], ph[kConvMaxTaps];
    float* out_f32; __half* out_f16; const float* bias; const float* residual;
    long long out_sb, out_sh, out_sw;
    long long out_sc;       // 0 or 1 = contiguous channels
    int n_valid;            // 0 = all C_out channels are stored
    int block_n_hint;       // 0 = auto; otherwise the preferred tile width (sign ignored): 256 runs the cooperative
                            // schedule (at C_out = 128 the transposed one, where its geometry allows), <= 128 the
                            // ping-pong one (see conv_tc.cu)
    double* stats;          // optional GroupNorm block statistics of the output (pre-zeroed), see ConvTcArgs
    int* err_flag;
};

// GroupNorm / FiLM / SiLU prologue of the fused Block kernel (conv_tc.cu)
struct GnPrologueArgs {
    const float* src0;            // fp32 NHWC [B][H][W][C0]
    const float* src1;            // fp32 NHWC [B][H][W][C1] or null
    int C0, C1, groups;           // channels of source 0 / source 1 (virtual concat), GroupNorm groups
    float scale1, eps;            // source-1 scale (skip connection 2^-1/2), GroupNorm eps
    const double* stats0;         // [B][C0/16][2] block statistics of source 0
    const double* stats1;         // [B][C1/16][2] block statistics of source 1 (unscaled) or null
    const float* gamma;           // [C0+C1]
    const float* beta;            // [C0+C1]
    const float* scale_shift;     // optional: row b at scale_shift + b*ss_ld = [scale(C) | shift(C)]
    int ss_ld;
};

struct ConvGnProblem {
    const float* src0; int C0;    // fp32 NHWC [B][H][W][C0]
    const float* src1; int C1;    // optional second source [B][H][W][C1]
    float scale1;
    int B, H, W, groups;
    const double* stats0; const double* stats1;
    const float* gamma; const float* beta; const float* scale_shift; int ss_ld; float eps;
    const void* wpacked; int Cout;          // fp16 [Cout][9*(C0+C1)]
    const float* bias; const float* residual;
    float* out_f32; __half* out_f16; double* out_stats;
    int* err_flag;
};

bool conv_gn_supported(int H, int W, int C0, int C1, int Cout, int groups);
int conv_gn_launch(const ConvGnProblem& p, cudaStream_t stream);

bool conv_tc_supported(int H, int W, int Cin, int Cout);
int conv_tc_launch(const ConvTcProblem& p, cudaStream_t stream);
const char* conv_tc_strerror(int code);

}  // namespace mi
