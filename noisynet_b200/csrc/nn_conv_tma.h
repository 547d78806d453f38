// Persistent TMA-im2col implicit-GEMM conv kernel (nn_conv_tma.cu): plan + launch interface used by the
// entry points in nn_conv_umma.cu (forward: fused noisy conv; dgrad: forward over grad_output with flipped weights).
#pragma once
#include "nn_common.cuh"

// K order of this kernel: per filter tap, the channels in chunks of 64 (SWIZZLE_128B rows) and one tail chunk of
// 16 / 32 / 64 channels (SWIZZLE_32B / 64B / 128B); a pipeline stage ("group") holds up to two chunks of one tap.
struct TmaPlan {
    int Cp, taps, n_c64, tail_w, wt, nc, gpt, n_groups;   // wt = padded channels per tap, nc = chunks per tap, gpt = groups per tap
    int n_t, n_tiles, n_mma, n_half, main_col, sig_col;   // n-tiling as in the tiled kernels; n_half = rows of one weight-copy box
    int stages, a_stage, b_stage, n_prod, threads;
    int tap_bytes;                                         // bytes of one tap of one n-tile in the weight image (both halves)
    size_t smem_bytes, wp_bytes;
};

// Cin_k: channels of the tensor that is convolved (layer input for forward, grad_output for dgrad); pad: effective padding.
bool nn_tma_make_plan(int Cin_k, int KH, int KW, int stride, int pad, int n_out, bool has_sigma, int OH, int OW, TmaPlan* out);

struct TmaConvCall {
    TmaPlan pl;
    int B, H, W;                 // convolved tensor [B, H, W, Cp] bf16 NHWC
    int OH, OW, KH, KW, stride, pad;
    int Cout;                    // real output channels
    const void* xp;
    const void* wp;              // NN_PACK_TMA image
    float y_scale, s_scale;
    float* y;                    // plain output (noise_mode == 0) [B, Cout, OH, OW] fp32
    float* y_noisy;              // noisy output (noise_mode != 0)
    int noise_mode;
    float current;
    const float* scale_dev;
    const float* z_inject;       // optional N(0,1) draws replacing the Philox stream (parity tests)
    nn_rng rng;
    int* err_flag;
    void *ev0, *ev1;             // optional cudaEvent_t pair recorded immediately around the kernel launch (nn_debug_main_kernel_ms)
};
int nn_tma_conv_launch(const TmaConvCall& c, int device, cudaStream_t st);

// ---- weight gradient with TMA-staged operands (k_wgrad_tma): the (tap, 64-channel chunk) columns of the gradient
struct TmaWgradPlan {
    int Cp, Coutp, taps, n_c64, tail_w;        // tail_w: 0 or 8 channels per tap (the remainder launch)
    int n_atoms, tiles_k, cols_pad, m_tiles_n, num_kb, kb_per_split, splits, stages;
    size_t smem_bytes, main_bytes, partial_bytes;      // partial = [main | remainder accumulators]
};
bool nn_tma_wgrad_plan(int Cin, int KH, int KW, int stride, int pad, int Cout, int64_t Mpix, int device, TmaWgradPlan* out);
struct TmaWgradCall {
    TmaWgradPlan pl;
    int B, H, W, OH, OW, KH, KW, stride, pad, Cout;
    const void* xp;               // layer input  [B, H, W, Cp] bf16
    const void* gyp;              // grad_output  [B * OH * OW, Coutp] bf16
    float* partial;               // [splits][Cout][cols_pad]
    int* err_flag;
};
int nn_tma_wgrad_launch(const TmaWgradCall& c, int device, cudaStream_t st);

// 128-byte tensor map (CUtensorMap) of a row-major bf16 matrix for the linear layers of the gathered kernel (k_conv_umma)
int nn_tma_encode_rows(void* map_out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t pitch_bytes);
