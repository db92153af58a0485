// Depthwise 3x3 convolution (groups = C, padding 1, dilation 1, stride 1 or 2) on NHWC bf16 activations, sm_90a.
// Replaces the `groups=in_channels` nn.Conv2d of SeparableConvBnRelu (TorchSeg furnace/base_model/xception.py:14-16)
// and its cuDNN dgrad / wgrad. A depthwise conv does 9 multiply-adds per element it reads, so these are HBM-bound
// CUDA-core kernels: one thread owns one 8-channel (16-byte) vector of one output pixel, the nine taps are gathered
// from L1/L2, and the weights (the fp32 [C][3][3] master, rounded to bf16 on load like every conv operand) are staged
// in shared memory transposed to [9][C]. All sums are fp32 in a fixed (r, s) tap order; nothing uses atomics.
#include "nhwc_vec.cuh"

namespace {
constexpr int kMaxC = 4096;   // [9][C] fp32 weights in shared memory: 144 KB at the limit

__device__ __forceinline__ void stage_weights(const float* __restrict__ w, int C, float* s_w) {
    for (int i = threadIdx.x; i < C * 9; i += blockDim.x) {
        const int c = i / 9, t = i - c * 9;
        s_w[t * C + c] = bf16_round(w[i]);
    }
    __syncthreads();
}

// y[n,p,q,c] = Σ_{r,s} x[n, p·st−1+r, q·st−1+s, c] · w[c,r,s]; taps in the zero halo add nothing
template <int ST>
__global__ void __launch_bounds__(kThreads)
dw_fprop_kernel(const __nv_bfloat16* __restrict__ x, int xcs, const float* __restrict__ w, __nv_bfloat16* __restrict__ y,
                int ycs, int H, int W, int P, int Q, int C8, long long total) {
    extern __shared__ float s_w[];
    const int C = C8 * 8;
    stage_weights(w, C, s_w);
    for_each_vec(total, C8, [&](long long p64, int c8) {
        const int pix = (int)p64;
        const int q = pix % Q, np = pix / Q;
        const int p = np % P, n = np / P;
        const int h0 = p * ST - 1, w0 = q * ST - 1;
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const int h = h0 + r;
            if (h < 0 || h >= H) continue;
#pragma unroll
            for (int s = 0; s < 3; ++s) {
                const int ww = w0 + s;
                if (ww < 0 || ww >= W) continue;
                float xv[8], wv[8];
                Vec8<__nv_bfloat16>::load(x + ((long long)(n * H + h) * W + ww) * xcs + c8 * 8, xv);
                Vec8<float>::load(s_w + (r * 3 + s) * C + c8 * 8, wv);
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[k] = fmaf(xv[k], wv[k], acc[k]);
            }
        }
        Vec8<__nv_bfloat16>::store(y + (long long)pix * ycs + c8 * 8, acc);
    });
}

// dx[n,h,w,c] (+)= Σ_{r,s} dy[n,p,q,c] · w[c,r,s] over the (p, q) with p·st−1+r = h, q·st−1+s = w: the exact gather form
// of the transposed conv (for stride 2 only the taps of the matching output parity contribute), one writer per element
template <int ST, bool kAcc>
__global__ void __launch_bounds__(kThreads, 1)   // (…, 1): without it ptxas spills 4-16 bytes at 32-40 registers
dw_dgrad_kernel(const __nv_bfloat16* __restrict__ dy, int dycs, const float* __restrict__ w, __nv_bfloat16* dx, int dxcs,
                int H, int W, int P, int Q, int C8, long long total) {
    extern __shared__ float s_w[];
    const int C = C8 * 8;
    stage_weights(w, C, s_w);
    const long long stride = (long long)gridDim.x * kThreads;
    const long long start = (long long)blockIdx.x * kThreads + threadIdx.x;
    VecWalk wk(C8, start, stride);
    for (long long i = start; i < total; i += stride, wk.next()) {
        const int pix = (int)wk.p, c8 = wk.c8;
        const int wq = pix % W, nh = pix / W;
        const int h = nh % H, n = nh / H;
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const int ph = h + 1 - r;   // output row p = ph / ST when ph >= 0 and ST divides ph
            if (ph < 0 || (ph >> (ST - 1)) >= P || (ph & (ST - 1))) continue;
            const int p = ph >> (ST - 1);
#pragma unroll
            for (int s = 0; s < 3; ++s) {
                const int qw = wq + 1 - s;
                if (qw < 0 || (qw >> (ST - 1)) >= Q || (qw & (ST - 1))) continue;
                const int q = qw >> (ST - 1);
                float gv[8], wv[8];
                Vec8<__nv_bfloat16>::load(dy + ((long long)(n * P + p) * Q + q) * dycs + c8 * 8, gv);
                Vec8<float>::load(s_w + (r * 3 + s) * C + c8 * 8, wv);
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[k] = fmaf(gv[k], wv[k], acc[k]);
            }
        }
        __nv_bfloat16* o = dx + (long long)pix * dxcs + c8 * 8;
        if (kAcc) {
            float old[8];
            Vec8<__nv_bfloat16>::load(o, old);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] = old[k] + acc[k];
        }
        Vec8<__nv_bfloat16>::store(o, acc);
    }
}

// dw[c,r,s] = Σ_{n,p,q} dy[n,p,q,c] · x[n, p·st−1+r, q·st−1+s, c]. CTA b sums the output pixels of its chunk (thread
// (lane, g) owns channel group g and every lanes-th pixel, all nine taps in registers), reduces over lanes through
// shared memory in lane order and stores its [C][9] partial into workspace slot b; tsb_det_reduce adds the slots.
template <int ST>
__global__ void __launch_bounds__(kThreads)
dw_wgrad_kernel(const __nv_bfloat16* __restrict__ x, int xcs, const __nv_bfloat16* __restrict__ dy, int dycs, int H, int W,
                int P, int Q, int C8, int npix, float* __restrict__ parts) {
    extern __shared__ float s_buf[];  // [lanes][groups][8]
    const int groups = min(C8, kThreads);
    const int lanes = kThreads / groups;
    const int g = threadIdx.x % groups, lane = threadIdx.x / groups;
    const int chunk = (npix + gridDim.x - 1) / gridDim.x;
    const int p0 = blockIdx.x * chunk, p1 = min(npix, p0 + chunk);
    float* slot = parts + (long long)blockIdx.x * C8 * 72;
    for (int g0 = 0; g0 < C8; g0 += groups) {
        const int cg = g0 + g;
        float acc[9][8];
#pragma unroll
        for (int t = 0; t < 9; ++t)
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[t][k] = 0.f;
        if (cg < C8 && lane < lanes) {
            for (int pix = p0 + lane; pix < p1; pix += lanes) {
                const int q = pix % Q, np = pix / Q;
                const int p = np % P, n = np / P;
                float gv[8];
                Vec8<__nv_bfloat16>::load(dy + (long long)pix * dycs + cg * 8, gv);
                const int h0 = p * ST - 1, w0 = q * ST - 1;
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const int h = h0 + r;
                    if (h < 0 || h >= H) continue;
#pragma unroll
                    for (int s = 0; s < 3; ++s) {
                        const int ww = w0 + s;
                        if (ww < 0 || ww >= W) continue;
                        float xv[8];
                        Vec8<__nv_bfloat16>::load(x + ((long long)(n * H + h) * W + ww) * xcs + cg * 8, xv);
#pragma unroll
                        for (int k = 0; k < 8; ++k) acc[r * 3 + s][k] = fmaf(gv[k], xv[k], acc[r * 3 + s][k]);
                    }
                }
            }
        }
#pragma unroll
        for (int t = 0; t < 9; ++t) {
            if (lane < lanes) {
#pragma unroll
                for (int k = 0; k < 8; ++k) s_buf[(lane * groups + g) * 8 + k] = acc[t][k];
            }
            __syncthreads();
            if (cg < C8 && lane < lanes) {
                for (int k = lane; k < 8; k += lanes) {
                    float s = 0.f;
                    for (int l = 0; l < lanes; ++l) s += s_buf[(l * groups + g) * 8 + k];
                    slot[(cg * 8 + k) * 9 + t] = s;
                }
            }
            __syncthreads();
        }
    }
}

int dw_grid(long long work) { return tsb_grid_for(work, kThreads, 8); }

// shared argument checks; P, Q are the output size (p·st−1+r with padding 1: (H − 1) / st + 1)
int check(const char* fn, const void* a, int acs, const void* b, int bcs, const float* w, int N, int H, int W, int C,
          int stride) {
    TSB_REQUIRE(a && b && w, "%s: null pointer", fn);
    TSB_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0, "%s: bad shape N=%d H=%d W=%d C=%d", fn, N, H, W, C);
    TSB_REQUIRE(C % 8 == 0 && C <= kMaxC, "%s: C=%d must be a multiple of 8 and at most %d", fn, C, kMaxC);
    TSB_REQUIRE(stride == 1 || stride == 2, "%s: stride %d is not supported (3x3, padding 1, stride 1 or 2)", fn, stride);
    TSB_REQUIRE(TSB_VEC_OK(C, acs, a) && TSB_VEC_OK(C, bcs, b),
                "%s: channel strides (%d, %d) must be multiples of 8 and at least C=%d, activations 16-byte aligned", fn,
                acs, bcs, C);
    TSB_REQUIRE((long long)N * H * W < (1LL << 31), "%s: N*H*W must be below 2^31", fn);
    return TSB_OK;
}

size_t weight_smem(int C) { return sizeof(float) * 9 * (size_t)C; }
}  // namespace

extern "C" int tsb_dwconv_fprop(const void* x, int xcs, const float* w, void* y, int ycs, int N, int H, int W, int C,
                                int stride, tsb_stream_t stream) {
    int rc = check("tsb_dwconv_fprop", x, xcs, y, ycs, w, N, H, W, C, stride);
    if (rc) return rc;
    const int P = (H - 1) / stride + 1, Q = (W - 1) / stride + 1, C8 = C / 8;
    const long long total = (long long)N * P * Q * C8;
    const size_t smem = weight_smem(C);
    cudaStream_t st = (cudaStream_t)stream;
    const void* fn = stride == 1 ? (const void*)dw_fprop_kernel<1> : (const void*)dw_fprop_kernel<2>;
    if (smem > 48 * 1024 && (rc = tsb_ensure_dyn_smem(fn, smem))) return rc;
    if (stride == 1)
        dw_fprop_kernel<1><<<dw_grid(total), kThreads, smem, st>>>((const __nv_bfloat16*)x, xcs, w, (__nv_bfloat16*)y, ycs, H, W, P, Q, C8, total);
    else
        dw_fprop_kernel<2><<<dw_grid(total), kThreads, smem, st>>>((const __nv_bfloat16*)x, xcs, w, (__nv_bfloat16*)y, ycs, H, W, P, Q, C8, total);
    TSB_CUDA_CHECK_LAUNCH("dwconv_fprop");
    return TSB_OK;
}

extern "C" int tsb_dwconv_dgrad(const void* dy, int dycs, const float* w, void* dx, int dxcs, int N, int H, int W, int C,
                                int stride, int accumulate, tsb_stream_t stream) {
    int rc = check("tsb_dwconv_dgrad", dy, dycs, dx, dxcs, w, N, H, W, C, stride);
    if (rc) return rc;
    const int P = (H - 1) / stride + 1, Q = (W - 1) / stride + 1, C8 = C / 8;
    const long long total = (long long)N * H * W * C8;
    const size_t smem = weight_smem(C);
    cudaStream_t st = (cudaStream_t)stream;
    const void* fn = stride == 1 ? (accumulate ? (const void*)dw_dgrad_kernel<1, true> : (const void*)dw_dgrad_kernel<1, false>)
                                 : (accumulate ? (const void*)dw_dgrad_kernel<2, true> : (const void*)dw_dgrad_kernel<2, false>);
    if (smem > 48 * 1024 && (rc = tsb_ensure_dyn_smem(fn, smem))) return rc;
#define L(S, A) dw_dgrad_kernel<S, A><<<dw_grid(total), kThreads, smem, st>>>((const __nv_bfloat16*)dy, dycs, w, (__nv_bfloat16*)dx, dxcs, H, W, P, Q, C8, total)
    if (stride == 1) { if (accumulate) L(1, true); else L(1, false); }
    else { if (accumulate) L(2, true); else L(2, false); }
#undef L
    TSB_CUDA_CHECK_LAUNCH("dwconv_dgrad");
    return TSB_OK;
}

extern "C" int tsb_dwconv_wgrad(const void* x, int xcs, const void* dy, int dycs, float* dw, int N, int H, int W, int C,
                                int stride, float* ws, long long ws_floats, tsb_stream_t stream) {
    int rc = check("tsb_dwconv_wgrad", x, xcs, dy, dycs, dw, N, H, W, C, stride);
    if (rc) return rc;
    const int P = (H - 1) / stride + 1, Q = (W - 1) / stride + 1, C8 = C / 8;
    const int npix = N * P * Q;
    const int grid = colred_grid(npix, C8, 8, tsb_num_sms() * 8LL);
    TSB_REQUIRE(ws && (long long)grid * C * 9 <= ws_floats, "tsb_dwconv_wgrad: workspace needs %lld floats",
                (long long)grid * C * 9);
    const size_t smem = colred_smem(C8, 1);
    cudaStream_t st = (cudaStream_t)stream;
    if (stride == 1)
        dw_wgrad_kernel<1><<<grid, kThreads, smem, st>>>((const __nv_bfloat16*)x, xcs, (const __nv_bfloat16*)dy, dycs, H, W, P, Q, C8, npix, ws);
    else
        dw_wgrad_kernel<2><<<grid, kThreads, smem, st>>>((const __nv_bfloat16*)x, xcs, (const __nv_bfloat16*)dy, dycs, H, W, P, Q, C8, npix, ws);
    TSB_CUDA_CHECK_LAUNCH("dwconv_wgrad");
    return tsb_det_reduce(dw, ws, grid, (long long)C * 9, (long long)C * 9, st);
}
