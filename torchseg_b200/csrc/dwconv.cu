// Depthwise 3x3 convolution (groups = C, padding = dilation d >= 1 at stride 1, or padding 1 at stride 2) on NHWC bf16
// activations, sm_90a. Replaces the `groups=in_channels` nn.Conv2d of the two SeparableConvBnRelu blocks (TorchSeg
// furnace/base_model/xception.py:14-16, furnace/seg_opr/seg_oprs.py:76-94) and its cuDNN dgrad / wgrad; the tap
// offsets are (r − 1)·d, (s − 1)·d, so at stride 1 the output keeps the input's size whatever the dilation. A depthwise
// conv does 9 multiply-adds per element it reads, so these are HBM-bound CUDA-core kernels: one thread owns one
// 8-channel (16-byte) vector of one output pixel, the nine taps are gathered from L1/L2, and the weights (the fp32
// [C][3][3] master, rounded to bf16 on load like every conv operand) are staged in shared memory transposed to [9][C]. All sums are fp32 in a fixed (r, s) tap order; nothing uses atomics.
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

// DIL: the dilation when it is a compile-time constant (1: the X39 layers and every stride-2 layer, whose code stays
// that of the dilation-free kernels, no extra registers or spills), 0: the runtime `dil` (the dilated ASPP / decoder)

// y[n,p,q,c] = Σ_{r,s} x[n, p·st+(r−1)·d, q·st+(s−1)·d, c] · w[c,r,s]; taps in the zero halo (for d >= H or W, all
// but the centre) add nothing
template <int ST, int DIL>
__global__ void __launch_bounds__(kThreads)
dw_fprop_kernel(const __nv_bfloat16* __restrict__ x, int xcs, const float* __restrict__ w, __nv_bfloat16* __restrict__ y,
                int ycs, int H, int W, int P, int Q, int C8, int dil_rt, long long total) {
    const int dil = DIL ? DIL : dil_rt;
    extern __shared__ float s_w[];
    const int C = C8 * 8;
    stage_weights(w, C, s_w);
    for_each_vec(total, C8, [&](long long p64, int c8) {
        const int pix = (int)p64;
        const int q = pix % Q, np = pix / Q;
        const int p = np % P, n = np / P;
        const int h0 = p * ST - dil, w0 = q * ST - dil;
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const int h = h0 + r * dil;
            if (h < 0 || h >= H) continue;
#pragma unroll
            for (int s = 0; s < 3; ++s) {
                const int ww = w0 + s * dil;
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

// dx[n,h,w,c] (+)= Σ_{r,s} dy[n,p,q,c] · w[c,r,s] over the (p, q) with p·st+(r−1)·d = h, q·st+(s−1)·d = w: the exact
// gather form of the transposed conv (for stride 2 only the taps of the matching output parity contribute), one writer
// per element
template <int ST, int DIL, bool kAcc>
__global__ void __launch_bounds__(kThreads, 1)   // (…, 1): without it ptxas spills 4-16 bytes at 32-40 registers
dw_dgrad_kernel(const __nv_bfloat16* __restrict__ dy, int dycs, const float* __restrict__ w, __nv_bfloat16* dx, int dxcs,
                int H, int W, int P, int Q, int C8, int dil_rt, long long total) {
    const int dil = DIL ? DIL : dil_rt;
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
            const int ph = h + (1 - r) * dil;   // output row p = ph / ST when ph >= 0 and ST divides ph
            if (ph < 0 || (ph >> (ST - 1)) >= P || (ph & (ST - 1))) continue;
            const int p = ph >> (ST - 1);
#pragma unroll
            for (int s = 0; s < 3; ++s) {
                const int qw = wq + (1 - s) * dil;
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

// dw[c,r,s] = Σ_{n,p,q} dy[n,p,q,c] · x[n, p·st+(r−1)·d, q·st+(s−1)·d, c]. CTA b sums the output pixels of its chunk
// (thread (lane, g) owns channel group g and every lanes-th pixel, all nine taps in registers), reduces over lanes through
// shared memory in lane order and stores its [C][9] partial into workspace slot b; tsb_det_reduce adds the slots.
template <int ST, int DIL>
__global__ void __launch_bounds__(kThreads)
dw_wgrad_kernel(const __nv_bfloat16* __restrict__ x, int xcs, const __nv_bfloat16* __restrict__ dy, int dycs, int H, int W,
                int P, int Q, int C8, int dil_rt, int npix, float* __restrict__ parts) {
    const int dil = DIL ? DIL : dil_rt;
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
                const int h0 = p * ST - dil, w0 = q * ST - dil;
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const int h = h0 + r * dil;
                    if (h < 0 || h >= H) continue;
#pragma unroll
                    for (int s = 0; s < 3; ++s) {
                        const int ww = w0 + s * dil;
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

// shared argument checks; P, Q are the output size ((H − 1) / st + 1: padding = dilation at stride 1, 1 at stride 2)
int check(const char* fn, const void* a, int acs, const void* b, int bcs, const float* w, int N, int H, int W, int C,
          int stride, int dil) {
    TSB_REQUIRE(a && b && w, "%s: null pointer", fn);
    TSB_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0, "%s: bad shape N=%d H=%d W=%d C=%d", fn, N, H, W, C);
    TSB_REQUIRE(C % 8 == 0 && C <= kMaxC, "%s: C=%d must be a multiple of 8 and at most %d", fn, C, kMaxC);
    TSB_REQUIRE(stride == 1 || stride == 2, "%s: stride %d is not supported (3x3, stride 1 or 2)", fn, stride);
    TSB_REQUIRE(dil >= 1, "%s: dilation %d must be at least 1", fn, dil);
    TSB_REQUIRE(stride == 1 || dil == 1, "%s: stride 2 needs dilation 1 (got dilation %d)", fn, dil);
    TSB_REQUIRE(TSB_VEC_OK(C, acs, a) && TSB_VEC_OK(C, bcs, b),
                "%s: channel strides (%d, %d) must be multiples of 8 and at least C=%d, activations 16-byte aligned", fn,
                acs, bcs, C);
    TSB_REQUIRE((long long)N * H * W < (1LL << 31), "%s: N*H*W must be below 2^31", fn);
    return TSB_OK;
}

size_t weight_smem(int C) { return sizeof(float) * 9 * (size_t)C; }
}  // namespace

// the kernel instances: <stride, 1> at dilation 1, <1, 0> (runtime dilation) otherwise
#define DW_DISPATCH(LAUNCH)     \
    do {                        \
        if (stride == 2) {      \
            LAUNCH(2, 1);       \
        } else if (dil == 1) {  \
            LAUNCH(1, 1);       \
        } else {                \
            LAUNCH(1, 0);       \
        }                       \
    } while (0)

extern "C" int tsb_dwconv2d_fprop(const void* x, int xcs, const float* w, void* y, int ycs, int N, int H, int W, int C,
                                  int stride, int dil, tsb_stream_t stream) {
    int rc = check("tsb_dwconv2d_fprop", x, xcs, y, ycs, w, N, H, W, C, stride, dil);
    if (rc) return rc;
    const int P = (H - 1) / stride + 1, Q = (W - 1) / stride + 1, C8 = C / 8;
    const long long total = (long long)N * P * Q * C8;
    const size_t smem = weight_smem(C);
    cudaStream_t st = (cudaStream_t)stream;
#define L(S, D)                                                                                                           \
    if (smem > 48 * 1024 && (rc = tsb_ensure_dyn_smem((const void*)dw_fprop_kernel<S, D>, smem))) return rc;             \
    dw_fprop_kernel<S, D><<<dw_grid(total), kThreads, smem, st>>>((const __nv_bfloat16*)x, xcs, w, (__nv_bfloat16*)y, ycs, \
                                                                  H, W, P, Q, C8, dil, total)
    DW_DISPATCH(L);
#undef L
    TSB_CUDA_CHECK_LAUNCH("dwconv_fprop");
    return TSB_OK;
}

extern "C" int tsb_dwconv2d_dgrad(const void* dy, int dycs, const float* w, void* dx, int dxcs, int N, int H, int W, int C,
                                  int stride, int dil, int accumulate, tsb_stream_t stream) {
    int rc = check("tsb_dwconv2d_dgrad", dy, dycs, dx, dxcs, w, N, H, W, C, stride, dil);
    if (rc) return rc;
    const int P = (H - 1) / stride + 1, Q = (W - 1) / stride + 1, C8 = C / 8;
    const long long total = (long long)N * H * W * C8;
    const size_t smem = weight_smem(C);
    cudaStream_t st = (cudaStream_t)stream;
#define LA(S, D, A)                                                                                                       \
    if (smem > 48 * 1024 && (rc = tsb_ensure_dyn_smem((const void*)dw_dgrad_kernel<S, D, A>, smem))) return rc;          \
    dw_dgrad_kernel<S, D, A><<<dw_grid(total), kThreads, smem, st>>>((const __nv_bfloat16*)dy, dycs, w,                   \
                                                                     (__nv_bfloat16*)dx, dxcs, H, W, P, Q, C8, dil, total)
#define L(S, D)            \
    if (accumulate) {      \
        LA(S, D, true);    \
    } else {               \
        LA(S, D, false);   \
    }                      \
    (void)0
    DW_DISPATCH(L);
#undef L
#undef LA
    TSB_CUDA_CHECK_LAUNCH("dwconv_dgrad");
    return TSB_OK;
}

extern "C" int tsb_dwconv2d_wgrad(const void* x, int xcs, const void* dy, int dycs, float* dw, int N, int H, int W, int C,
                                  int stride, int dil, float* ws, long long ws_floats, tsb_stream_t stream) {
    int rc = check("tsb_dwconv2d_wgrad", x, xcs, dy, dycs, dw, N, H, W, C, stride, dil);
    if (rc) return rc;
    const int P = (H - 1) / stride + 1, Q = (W - 1) / stride + 1, C8 = C / 8;
    const int npix = N * P * Q;
    const int grid = colred_grid(npix, C8, 8, tsb_num_sms() * 8LL);
    TSB_REQUIRE(ws && (long long)grid * C * 9 <= ws_floats, "tsb_dwconv2d_wgrad: workspace needs %lld floats",
                (long long)grid * C * 9);
    const size_t smem = colred_smem(C8, 1);
    cudaStream_t st = (cudaStream_t)stream;
#define L(S, D)                                                                                                        \
    dw_wgrad_kernel<S, D><<<grid, kThreads, smem, st>>>((const __nv_bfloat16*)x, xcs, (const __nv_bfloat16*)dy, dycs, H, \
                                                        W, P, Q, C8, dil, npix, ws)
    DW_DISPATCH(L);
#undef L
    TSB_CUDA_CHECK_LAUNCH("dwconv_wgrad");
    return tsb_det_reduce(dw, ws, grid, (long long)C * 9, (long long)C * 9, st);
}
#undef DW_DISPATCH

extern "C" int tsb_dwconv_fprop(const void* x, int xcs, const float* w, void* y, int ycs, int N, int H, int W, int C,
                                int stride, tsb_stream_t stream) {
    return tsb_dwconv2d_fprop(x, xcs, w, y, ycs, N, H, W, C, stride, 1, stream);
}

extern "C" int tsb_dwconv_dgrad(const void* dy, int dycs, const float* w, void* dx, int dxcs, int N, int H, int W, int C,
                                int stride, int accumulate, tsb_stream_t stream) {
    return tsb_dwconv2d_dgrad(dy, dycs, w, dx, dxcs, N, H, W, C, stride, 1, accumulate, stream);
}

extern "C" int tsb_dwconv_wgrad(const void* x, int xcs, const void* dy, int dycs, float* dw, int N, int H, int W, int C,
                                int stride, float* ws, long long ws_floats, tsb_stream_t stream) {
    return tsb_dwconv2d_wgrad(x, xcs, dy, dycs, dw, N, H, W, C, stride, 1, ws, ws_floats, stream);
}
