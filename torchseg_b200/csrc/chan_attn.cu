// DANet's channel-attention soft-max (CAM) and the learnable-gamma residual y = x + gamma·o shared by its position and
// channel attention modules (Fu et al., "Dual Attention Network for Scene Segmentation", CVPR 2019).
//
// The CAM products E = X Xᵀ, A·X and their gradients run on the wgmma convolution kernels; what is here is the
// element-wise part between them. No atomics: every output has one writer, and dgamma's per-CTA partials go through
// tsb_det_reduce in slot order.
#include "tsb_common.cuh"

namespace {

constexpr int kThreads = 256;

// A = softmax_row(rowmax(E) − E): one warp per row. t_j = fl(rowmax − E_j) as torch forms it; its maximum is
// fl(rowmax − rowmin) because rounding is monotonic. Each lane sums its strided columns in order, then a fixed butterfly.
__global__ void __launch_bounds__(kThreads) cam_softmax_fwd_kernel(const float* __restrict__ E,
                                                                   __nv_bfloat16* __restrict__ A, long long rows, int C) {
    const int lane = threadIdx.x & 31;
    const long long step = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += step) {
        const float* e = E + r * C;
        float mx = -INFINITY, mn = INFINITY;
        for (int j = lane; j < C; j += 32) {
            const float v = e[j];
            mx = fmaxf(mx, v);
            mn = fminf(mn, v);
        }
        mx = warp_max(mx);
        mn = -warp_max(-mn);
        const float m = __fsub_rn(mx, mn);
        float s = 0.f;
        for (int j = lane; j < C; j += 32) s += expf(__fsub_rn(__fsub_rn(mx, e[j]), m));
        const float inv = 1.f / warp_sum(s);
        __nv_bfloat16* a = A + r * C;
        for (int j = lane; j < C; j += 32) a[j] = __float2bfloat16_rn(expf(__fsub_rn(__fsub_rn(mx, e[j]), m)) * inv);
    }
}

// r_i = Σ_j A_ij · dA_ij: one warp per row
__global__ void __launch_bounds__(kThreads) cam_rowdot_kernel(const __nv_bfloat16* __restrict__ A,
                                                              const float* __restrict__ dA, float* __restrict__ r,
                                                              long long rows, int C) {
    const int lane = threadIdx.x & 31;
    const long long step = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < rows; i += step) {
        float s = 0.f;
        for (int j = lane; j < C; j += 32) s = fmaf(__bfloat162float(A[i * C + j]), dA[i * C + j], s);
        s = warp_sum(s);
        if (lane == 0) r[i] = s;
    }
}

// dẼ_ij = A_ij (dA_ij − r_i), the same instructions wherever it is evaluated, so that G below is exactly symmetric
__device__ __forceinline__ float cam_dsoft(const __nv_bfloat16* A, const float* dA, const float* r, long long base, int i,
                                          int j, int C) {
    const long long o = base + (long long)i * C + j;
    return __fmul_rn(__bfloat162float(A[o]), __fsub_rn(dA[o], r[i]));
}

// G = −(dẼ + dẼᵀ) on 32 x 32 tiles; the transposed tile goes through shared memory. block (32, 8), grid (C/32, C/32, B)
__global__ void __launch_bounds__(kThreads) cam_softmax_bwd_kernel(const __nv_bfloat16* __restrict__ A,
                                                                   const float* __restrict__ dA,
                                                                   const float* __restrict__ r,
                                                                   __nv_bfloat16* __restrict__ G, int C) {
    __shared__ float t[32][33];
    const int b = blockIdx.z, i0 = blockIdx.y * 32, j0 = blockIdx.x * 32, tx = threadIdx.x, ty = threadIdx.y;
    const long long base = (long long)b * C * C;
    const float* rb = r + (long long)b * C;
    for (int k = ty; k < 32; k += 8) {   // t[k][tx] = dẼ[j0 + k][i0 + tx]
        const int row = j0 + k, col = i0 + tx;
        t[k][tx] = (row < C && col < C) ? cam_dsoft(A, dA, rb, base, row, col, C) : 0.f;
    }
    __syncthreads();
    for (int k = ty; k < 32; k += 8) {
        const int i = i0 + k, j = j0 + tx;
        if (i < C && j < C)
            G[base + (long long)i * C + j] = __float2bfloat16_rn(-__fadd_rn(cam_dsoft(A, dA, rb, base, i, j, C), t[tx][k]));
    }
}

// y = bf16(fmaf(gamma, o, x)), 8 channels per item
__global__ void __launch_bounds__(kThreads) gamma_residual_fwd_kernel(const __nv_bfloat16* __restrict__ x, int xcs,
                                                                      const __nv_bfloat16* __restrict__ o, int ocs,
                                                                      const float* __restrict__ gamma,
                                                                      __nv_bfloat16* __restrict__ y, int ycs,
                                                                      long long npix, int C8) {
    const float g = __ldg(gamma);
    const long long n = npix * C8, step = (long long)gridDim.x * blockDim.x;
    for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < n; it += step) {
        const long long p = it / C8;
        const int c = (int)(it - p * C8) * 8;
        float a[8], v[8];
        unpack8(*reinterpret_cast<const uint4*>(x + p * xcs + c), a);
        unpack8(*reinterpret_cast<const uint4*>(o + p * ocs + c), v);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = fmaf(g, v[e], a[e]);
        *reinterpret_cast<uint4*>(y + p * ycs + c) = pack8(v);
    }
}

// do = bf16(gamma · dy); this CTA's Σ dy·o into workspace slot blockIdx.x
__global__ void __launch_bounds__(kThreads) gamma_residual_bwd_kernel(const __nv_bfloat16* __restrict__ dy, int dycs,
                                                                      const __nv_bfloat16* __restrict__ o, int ocs,
                                                                      const float* __restrict__ gamma,
                                                                      __nv_bfloat16* __restrict__ dout, int docs,
                                                                      long long npix, int C8, float* __restrict__ ws) {
    __shared__ float red[33];
    const float g = __ldg(gamma);
    const long long n = npix * C8, step = (long long)gridDim.x * blockDim.x;
    float s = 0.f;
    for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < n; it += step) {
        const long long p = it / C8;
        const int c = (int)(it - p * C8) * 8;
        float d[8], v[8];
        unpack8(*reinterpret_cast<const uint4*>(dy + p * dycs + c), d);
        unpack8(*reinterpret_cast<const uint4*>(o + p * ocs + c), v);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            s = fmaf(d[e], v[e], s);
            d[e] *= g;
        }
        *reinterpret_cast<uint4*>(dout + p * docs + c) = pack8(d);
    }
    s = block_sum<kThreads>(s, red);
    if (threadIdx.x == 0) ws[blockIdx.x] = s;
}

bool vec_ok(const void* p, int cs, int C) { return p != nullptr && tsb_aligned16(p) && cs % 8 == 0 && cs >= C; }

}  // namespace

extern "C" int tsb_chan_attn_softmax_fwd(const float* E, void* A, int B, int C, tsb_stream_t stream) {
    TSB_REQUIRE(E != nullptr && A != nullptr, "tsb_chan_attn_softmax_fwd: null E or A");
    TSB_REQUIRE(B >= 1 && C >= 1 && B <= 65535 && (long long)C * C <= (1LL << 30),
                "tsb_chan_attn_softmax_fwd: bad shape B=%d C=%d", B, C);
    const long long rows = (long long)B * C;
    cam_softmax_fwd_kernel<<<tsb_grid_for(rows, kThreads / 32, 8), kThreads, 0, (cudaStream_t)stream>>>(
        E, (__nv_bfloat16*)A, rows, C);
    TSB_CUDA_CHECK_LAUNCH("chan_attn_softmax_fwd");
    return TSB_OK;
}

extern "C" int tsb_chan_attn_softmax_bwd(const void* A, const float* dA, float* rowdot_ws, void* G, int B, int C,
                                         tsb_stream_t stream) {
    TSB_REQUIRE(A != nullptr && dA != nullptr && rowdot_ws != nullptr && G != nullptr,
                "tsb_chan_attn_softmax_bwd: null A, dA, rowdot_ws or G");
    TSB_REQUIRE(B >= 1 && C >= 1 && B <= 65535 && (long long)C * C <= (1LL << 30),
                "tsb_chan_attn_softmax_bwd: bad shape B=%d C=%d", B, C);
    cudaStream_t st = (cudaStream_t)stream;
    const long long rows = (long long)B * C;
    cam_rowdot_kernel<<<tsb_grid_for(rows, kThreads / 32, 8), kThreads, 0, st>>>((const __nv_bfloat16*)A, dA, rowdot_ws,
                                                                               rows, C);
    TSB_CUDA_CHECK_LAUNCH("chan_attn_rowdot");
    const dim3 grid((C + 31) / 32, (C + 31) / 32, B);
    cam_softmax_bwd_kernel<<<grid, dim3(32, 8), 0, st>>>((const __nv_bfloat16*)A, dA, rowdot_ws, (__nv_bfloat16*)G, C);
    TSB_CUDA_CHECK_LAUNCH("chan_attn_softmax_bwd");
    return TSB_OK;
}

extern "C" int tsb_gamma_residual_fwd(const void* x, int xcs, const void* o, int ocs, const float* gamma, void* y, int ycs,
                                      long long npix, int C, tsb_stream_t stream) {
    TSB_REQUIRE(gamma != nullptr && npix > 0 && C > 0 && C % 8 == 0, "tsb_gamma_residual_fwd: bad args (C must be a "
                "positive multiple of 8, gamma non-null)");
    TSB_REQUIRE(vec_ok(x, xcs, C) && vec_ok(o, ocs, C) && vec_ok(y, ycs, C),
                "tsb_gamma_residual_fwd: x, o, y must be 16-byte aligned with channel strides that are multiples of 8 "
                "and >= C");
    const int C8 = C / 8;
    gamma_residual_fwd_kernel<<<tsb_grid_for(npix * C8, kThreads, 8), kThreads, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x, xcs, (const __nv_bfloat16*)o, ocs, gamma, (__nv_bfloat16*)y, ycs, npix, C8);
    TSB_CUDA_CHECK_LAUNCH("gamma_residual_fwd");
    return TSB_OK;
}

extern "C" int tsb_gamma_residual_bwd(const void* dy, int dycs, const void* o, int ocs, const float* gamma, void* dout,
                                      int docs, float* dgamma, long long npix, int C, float* ws, long long ws_floats,
                                      tsb_stream_t stream) {
    TSB_REQUIRE(gamma != nullptr && dgamma != nullptr && npix > 0 && C > 0 && C % 8 == 0,
                "tsb_gamma_residual_bwd: bad args (C must be a positive multiple of 8, gamma and dgamma non-null)");
    TSB_REQUIRE(vec_ok(dy, dycs, C) && vec_ok(o, ocs, C) && vec_ok(dout, docs, C),
                "tsb_gamma_residual_bwd: dy, o, dout must be 16-byte aligned with channel strides that are multiples of "
                "8 and >= C");
    const int C8 = C / 8;
    const int grid = tsb_grid_for(npix * C8, kThreads, 4);
    TSB_REQUIRE(ws != nullptr && grid <= ws_floats, "tsb_gamma_residual_bwd: workspace needs %d floats", grid);
    cudaStream_t st = (cudaStream_t)stream;
    gamma_residual_bwd_kernel<<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)dy, dycs, (const __nv_bfloat16*)o, ocs,
                                                         gamma, (__nv_bfloat16*)dout, docs, npix, C8, ws);
    TSB_CUDA_CHECK_LAUNCH("gamma_residual_bwd");
    return tsb_det_reduce(dgamma, ws, grid, 1, 1, st);
}
