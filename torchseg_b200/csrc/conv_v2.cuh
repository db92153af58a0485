// Host-side descriptor of one implicit-GEMM launch for the persistent kernel (conv_v2.cu).
#pragma once
#include <cuda_runtime.h>

#include "conv_common.cuh"

namespace convv2 {

struct Desc {
    // activation (A operand) tensor: NHWC bf16 [aN, aH, aW, aC] with channel stride acs
    const void* act;
    int aN, aH, aW, aC, acs;
    int act_stride;   // 1: plain view; 2: four parity views (stride-2 fprop)
    int stem;         // 1: overlapped-window view of the s2d image (aH = H/2, aW = W/2)
    int flat;         // 1: 1x1 stride-1 conv flattened to a GEMM over all pixels
    // taps (map coordinates relative to the output-tile origin) and K chunks per tap
    convhost::Tap taps[convhost::kMaxTaps];
    int ntaps, kchunks;
    // weights (B operand): bf16 [w_rows][w_k]
    const void* w;
    int w_rows;
    long long w_k;
    int ncols;        // output columns of this launch (tiled by BN)
    // launch output grid and addressing (elements)
    int Nl, Pl, Ql;
    long long out_n_stride, out_p_stride, out_q_stride, out_base;
    int k_real, k_store, out_f32, accumulate;
    const float* bias;
    float* sum;
    float* sumsq;
    void* out;
    int relu;          // inference epilogue (folded BN): ReLU after bias (+ res)
    const void* res;   // bf16 residual addressed exactly like `out`
    float* ws;         // caller's workspace for the per-CTA statistics (needed when sum != nullptr)
    long long ws_floats;
    // flat 1x1 only: the A operand is bf16(relu(act·in_scale[c] + in_shift[c])), normalised in shared memory
    const float* in_scale;
    const float* in_shift;
};

struct WgradDesc {
    const void* x;   // NHWC bf16 [N,H,W,C] (channel stride xcs)
    const void* dy;  // NHWC bf16 [N,P,Q,K] (channel stride dycs)
    int N, H, W, C, xcs, P, Q, K, dycs, stride;
    convhost::Tap taps[convhost::kMaxTaps];  // in (r, s) order; bk unused
    int ntaps;
    long long dw_row_stride;
    float* dw;
    float* ws;         // caller's workspace: one dW-shaped slice per pixel split (one split, adding in place, when it is too small)
    long long ws_floats;
};

// With statistics and `stat_slots`, the per-CTA statistics are left in d.ws ([slot][2][k_real], one slot per CTA) and
// their count is returned in *stat_slots for the caller to reduce; otherwise they are added into d.sum / d.sumsq here.
int launch(const Desc& d, cudaStream_t st, int* stat_slots = nullptr);
int launch_wgrad_rows(const WgradDesc& d, cudaStream_t st);
int launch_wgrad_taps(const WgradDesc& d, int R, int pad, int dil, cudaStream_t st);   // conv_wgrad_taps.cu

}  // namespace convv2
