// EncNet's Context Encoding layer (Zhang et al., CVPR 2018), the mean over its codewords, and the SE-loss with the
// class-presence vector built on the device (include/tsb.h).
//
// Encoding: for the N pixels x_i (bf16, D channels) of image b, codewords c_k (fp32 [K][D]) and smoothing factors s_k,
//   d²_ik = ‖x_i − c_k‖² (direct differences), a_ik = softmax_k(s_k d²_ik), E_bk = Σ_i a_ik x_i − (Σ_i a_ik) c_k.
// One CTA per (image, slot) strides over the image's pixels in tiles of kTP pixels:
//   phase 1 — one warp per pixel: the pixel's D values live in the lanes' registers (lane l holds the channel pairs
//             64j + 2l, 64j + 2l + 1), each d²_ik is one warp reduction, and lane k owns codeword k for the soft-max;
//   phase 2 — the CTA adds the tile's Σ_i a_ik x_id (resp. the backward's Σ_i g_ik x_id) into a [D][K] shared-memory
//             accumulator; every (d, k) has one owner thread, which adds the tile's pixels in order.
// Each CTA stores its partial sums into its own workspace slot, and a second small launch adds the slots in a fixed
// order, so the results are identical from run to run. The number of slots per image is fixed (kSlots), so the workspace
// does not grow with the map size. Each pixel is read once from global memory.
#include "tsb_common.cuh"

#include <math.h>

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kTP = 32;       // pixels per tile
constexpr int kSlots = 16;    // workspace slots (CTAs) per image
constexpr int kMaxNJ = 16;    // D <= 64 * kMaxNJ
constexpr int kMaxKD = 16384; // codewords in shared memory: K * D * 4 B <= 64 KB

__device__ __forceinline__ void load_pixel(const __nv_bfloat16* __restrict__ px, int nj, int lane, float* xv,
                                           __nv_bfloat16* xt_row) {
#pragma unroll
    for (int j = 0; j < kMaxNJ; ++j) {
        if (j < nj) {
            const int d = 64 * j + 2 * lane;
            const uint32_t u = *reinterpret_cast<const uint32_t*>(px + d);
            xv[2 * j] = bf16lo(u);
            xv[2 * j + 1] = bf16hi(u);
            *reinterpret_cast<uint32_t*>(xt_row + d) = u;
        }
    }
}

__device__ __forceinline__ void zero_pixel(int nj, int lane, float* xv, __nv_bfloat16* xt_row) {
#pragma unroll
    for (int j = 0; j < kMaxNJ; ++j) {
        if (j < nj) {
            xv[2 * j] = xv[2 * j + 1] = 0.f;
            *reinterpret_cast<uint32_t*>(xt_row + 64 * j + 2 * lane) = 0u;
        }
    }
}

// lane k (< K) receives d²_k = Σ_d (x_d − c_kd)²
template <int K>
__device__ __forceinline__ float sq_dist(const float* xv, const float* __restrict__ cw, int D, int nj, int lane) {
    float d2 = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const float* c = cw + k * D;
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < kMaxNJ; ++j) {
            if (j < nj) {
                const float2 cc = *reinterpret_cast<const float2*>(c + 64 * j + 2 * lane);
                const float e0 = xv[2 * j] - cc.x, e1 = xv[2 * j + 1] - cc.y;
                s = fmaf(e0, e0, s);
                s = fmaf(e1, e1, s);
            }
        }
        s = warp_sum(s);
        if (lane == k) d2 = s;
    }
    return d2;
}

// acc[d * K + k] += Σ_{p < kTP} wt[p * K + k] * x[p][d], one owner thread per (d, k), pixels in order
template <int K>
__device__ __forceinline__ void tile_accumulate(float* acc, const float* wt, const __nv_bfloat16* xt, int D) {
    for (int o = threadIdx.x; o < K * D; o += kThreads) {
        const int d = o / K, k = o - d * K;
        float s = 0.f;
#pragma unroll 8
        for (int p = 0; p < kTP; ++p) s = fmaf(wt[p * K + k], __bfloat162float(xt[p * D + d]), s);
        acc[o] += s;
    }
}

template <int K>
__global__ void __launch_bounds__(kThreads, 1) enc_fwd_kernel(const __nv_bfloat16* __restrict__ x, int xcs, int N, int D,
                                                           const float* __restrict__ codewords,
                                                           const float* __restrict__ scale, float* __restrict__ a_out,
                                                           float* __restrict__ d2_out, float* __restrict__ ws) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int KD = K * D;
    float* cw = reinterpret_cast<float*>(smem);               // [K][D]
    float* acc = cw + KD;                                     // [D][K]
    float* at = acc + KD;                                     // [kTP][K]
    __nv_bfloat16* xt = reinterpret_cast<__nv_bfloat16*>(at + kTP * K);   // [kTP][D]
    const int slot = blockIdx.x, b = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nj = D / 64;
    for (int i = threadIdx.x; i < KD; i += kThreads) {
        cw[i] = codewords[i];
        acc[i] = 0.f;
    }
    const float sk = lane < K ? scale[lane] : 0.f;
    float suma = 0.f;   // thread k < K: Σ_i a_ik over this CTA's pixels
    __syncthreads();
    const int ntiles = (N + kTP - 1) / kTP;
    for (int tile = slot; tile < ntiles; tile += kSlots) {
        for (int p = warp; p < kTP; p += kWarps) {
            const int i = tile * kTP + p;
            float xv[2 * kMaxNJ];
            float a = 0.f;
            if (i < N) {
                const long long row = (long long)b * N + i;
                load_pixel(x + row * xcs, nj, lane, xv, xt + p * D);
                const float d2 = sq_dist<K>(xv, cw, D, nj, lane);
                const float l = lane < K ? sk * d2 : -INFINITY;
                const float m = warp_max(l);
                const float e = lane < K ? expf(l - m) : 0.f;
                a = e / warp_sum(e);
                if (lane < K && a_out) {
                    a_out[row * K + lane] = a;
                    d2_out[row * K + lane] = d2;
                }
            } else {
                zero_pixel(nj, lane, xv, xt + p * D);
            }
            if (lane < K) at[p * K + lane] = a;
        }
        __syncthreads();
        tile_accumulate<K>(acc, at, xt, D);
        if (threadIdx.x < K)
            for (int p = 0; p < kTP; ++p) suma += at[p * K + threadIdx.x];
        __syncthreads();
    }
    float* out = ws + ((long long)b * kSlots + slot) * (KD + K);
    for (int i = threadIdx.x; i < KD; i += kThreads) out[i] = acc[i];
    if (threadIdx.x < K) out[KD + threadIdx.x] = suma;
}

// E[(b*D + d)*K + k] = bf16(Σ_slots Σ a x − (Σ_slots Σ a) c_kd); sum_a[b*K + k] = Σ_slots Σ a
__global__ void enc_fwd_finalize_kernel(const float* __restrict__ ws, int B, int D, int K,
                                        const float* __restrict__ codewords, float* __restrict__ sum_a,
                                        __nv_bfloat16* __restrict__ E) {
    const int KD = K * D;
    const long long total = (long long)B * KD;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(t / KD), o = (int)(t - (long long)b * KD);
        const int d = o / K, k = o - d * K;
        const float* w = ws + (long long)b * kSlots * (KD + K);
        float sax = 0.f, sa = 0.f;
#pragma unroll
        for (int s = 0; s < kSlots; ++s) {
            sax += w[(long long)s * (KD + K) + o];
            sa += w[(long long)s * (KD + K) + KD + k];
        }
        E[t] = __float2bfloat16_rn(sax - sa * codewords[k * D + d]);
        if (d == 0) sum_a[b * K + k] = sa;
    }
}

template <int K>
__global__ void __launch_bounds__(kThreads, 1) enc_bwd_kernel(const __nv_bfloat16* __restrict__ dE,
                                                           const __nv_bfloat16* __restrict__ x, int xcs, int N, int D,
                                                           const float* __restrict__ codewords,
                                                           const float* __restrict__ scale, const float* __restrict__ a_in,
                                                           const float* __restrict__ d2_in, __nv_bfloat16* __restrict__ dx,
                                                           int dxcs, float* __restrict__ ws) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int KD = K * D;
    float* cw = reinterpret_cast<float*>(smem);               // [K][D]
    float* acc = cw + KD;                                     // [D][K]  Σ g x
    float* gt = acc + KD;                                     // [kTP][K] g
    float* gdt = gt + kTP * K;                                // [kTP][K] g d²
    __nv_bfloat16* dEs = reinterpret_cast<__nv_bfloat16*>(gdt + kTP * K);   // [K][D]
    __nv_bfloat16* xt = dEs + KD;                                            // [kTP][D]
    const int slot = blockIdx.x, b = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nj = D / 64;
    for (int o = threadIdx.x; o < KD; o += kThreads) {
        cw[o] = codewords[o];
        acc[o] = 0.f;
        const int d = o / K, k = o - d * K;
        dEs[k * D + d] = dE[(long long)b * KD + o];
    }
    const float sk = lane < K ? scale[lane] : 0.f;
    float sg = 0.f, sgd = 0.f;   // thread k < K: Σ_i g_ik, Σ_i g_ik d²_ik
    __syncthreads();
    const int ntiles = (N + kTP - 1) / kTP;
    for (int tile = slot; tile < ntiles; tile += kSlots) {
        for (int p = warp; p < kTP; p += kWarps) {
            const int i = tile * kTP + p;
            float xv[2 * kMaxNJ];
            float g = 0.f, d2 = 0.f;
            if (i < N) {
                const long long row = (long long)b * N + i;
                load_pixel(x + row * xcs, nj, lane, xv, xt + p * D);
                const float a = lane < K ? a_in[row * K + lane] : 0.f;
                d2 = lane < K ? d2_in[row * K + lane] : 0.f;
                // t_k = Σ_d dE_kd (x_d − c_kd)
                float t = 0.f;
#pragma unroll
                for (int k = 0; k < K; ++k) {
                    const float* c = cw + k * D;
                    const __nv_bfloat16* e = dEs + k * D;
                    float s = 0.f;
#pragma unroll
                    for (int j = 0; j < kMaxNJ; ++j) {
                        if (j < nj) {
                            const int d = 64 * j + 2 * lane;
                            const float2 cc = *reinterpret_cast<const float2*>(c + d);
                            const uint32_t u = *reinterpret_cast<const uint32_t*>(e + d);
                            s = fmaf(bf16lo(u), xv[2 * j] - cc.x, s);
                            s = fmaf(bf16hi(u), xv[2 * j + 1] - cc.y, s);
                        }
                    }
                    s = warp_sum(s);
                    if (lane == k) t = s;
                }
                g = a * (t - warp_sum(a * t));
                // dx_d = Σ_k a_k dE_kd + 2 g_k s_k (x_d − c_kd)
                const float g2s = 2.f * g * sk;
                float dxv[2 * kMaxNJ];
#pragma unroll
                for (int j = 0; j < 2 * kMaxNJ; ++j) dxv[j] = 0.f;
#pragma unroll
                for (int k = 0; k < K; ++k) {
                    const float ak = __shfl_sync(0xffffffffu, a, k);
                    const float gk = __shfl_sync(0xffffffffu, g2s, k);
                    const float* c = cw + k * D;
                    const __nv_bfloat16* e = dEs + k * D;
#pragma unroll
                    for (int j = 0; j < kMaxNJ; ++j) {
                        if (j < nj) {
                            const int d = 64 * j + 2 * lane;
                            const float2 cc = *reinterpret_cast<const float2*>(c + d);
                            const uint32_t u = *reinterpret_cast<const uint32_t*>(e + d);
                            dxv[2 * j] += fmaf(ak, bf16lo(u), gk * (xv[2 * j] - cc.x));
                            dxv[2 * j + 1] += fmaf(ak, bf16hi(u), gk * (xv[2 * j + 1] - cc.y));
                        }
                    }
                }
                __nv_bfloat16* dp = dx + row * dxcs;
#pragma unroll
                for (int j = 0; j < kMaxNJ; ++j)
                    if (j < nj) *reinterpret_cast<uint32_t*>(dp + 64 * j + 2 * lane) = pack_bf16(dxv[2 * j], dxv[2 * j + 1]);
            } else {
                zero_pixel(nj, lane, xv, xt + p * D);
            }
            if (lane < K) {
                gt[p * K + lane] = g;
                gdt[p * K + lane] = g * d2;
            }
        }
        __syncthreads();
        tile_accumulate<K>(acc, gt, xt, D);
        if (threadIdx.x < K)
            for (int p = 0; p < kTP; ++p) {
                sg += gt[p * K + threadIdx.x];
                sgd += gdt[p * K + threadIdx.x];
            }
        __syncthreads();
    }
    float* out = ws + ((long long)b * kSlots + slot) * (KD + 2 * K);
    for (int i = threadIdx.x; i < KD; i += kThreads) out[i] = acc[i];
    if (threadIdx.x < K) {
        out[KD + threadIdx.x] = sg;
        out[KD + K + threadIdx.x] = sgd;
    }
}

// dc[k*D + d] += −Σ_b Σa_bk dE_bkd − 2 s_k (Σ g x − (Σ g) c_kd);  ds[k] += Σ g d²   (all slots of all images, in order)
__global__ void enc_bwd_finalize_kernel(const float* __restrict__ ws, const __nv_bfloat16* __restrict__ dE,
                                        const float* __restrict__ sum_a, int B, int D, int K,
                                        const float* __restrict__ codewords, const float* __restrict__ scale,
                                        float* __restrict__ dc, float* __restrict__ ds) {
    const int KD = K * D, stride = KD + 2 * K, nslots = B * kSlots;
    for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < KD; o += gridDim.x * blockDim.x) {
        const int d = o / K, k = o - d * K;
        float sgx = 0.f, sg = 0.f, sgd = 0.f, sad = 0.f;
#pragma unroll 8
        for (int s = 0; s < nslots; ++s) {
            const float* w = ws + (long long)s * stride;
            sgx += w[o];
            sg += w[KD + k];
            sgd += w[KD + K + k];
        }
        for (int b = 0; b < B; ++b) sad = fmaf(sum_a[b * K + k], __bfloat162float(dE[(long long)b * KD + o]), sad);
        const float c = codewords[k * D + d];
        dc[k * D + d] += -sad - 2.f * scale[k] * (sgx - sg * c);
        if (d == 0) ds[k] += sgd;
    }
}

int check_encoding(const char* fn, const void* x, int xcs, int B, int N, int D, const float* codewords, const float* scale,
                   int K) {
    TSB_REQUIRE(x && codewords && scale, "%s: null pointer", fn);
    TSB_REQUIRE(B > 0 && N > 0, "%s: bad shape B=%d N=%d", fn, B, N);
    if (K % 8 != 0 || K < 8 || K > 32)
        TSB_FAIL(TSB_ERR_UNSUPPORTED, "%s: K=%d must be a multiple of 8 and at most 32", fn, K);
    if (D % 64 != 0 || D < 64 || D > 64 * kMaxNJ || K * D > kMaxKD)
        TSB_FAIL(TSB_ERR_UNSUPPORTED, "%s: D=%d must be a multiple of 64, at most %d, with K*D <= %d", fn, D, 64 * kMaxNJ,
                 kMaxKD);
    TSB_REQUIRE(xcs >= D && xcs % 8 == 0 && tsb_aligned16(x),
                "%s: channel stride %d must be a multiple of 8 and at least D=%d, x 16-byte aligned", fn, xcs, D);
    TSB_REQUIRE((long long)B * N < (1LL << 31), "%s: B*N must be below 2^31", fn);
    return TSB_OK;
}

size_t fwd_smem(int K, int D) { return 2 * sizeof(float) * K * D + sizeof(float) * kTP * K + 2 * (size_t)kTP * D; }
size_t bwd_smem(int K, int D) {
    return 2 * sizeof(float) * K * D + 2 * sizeof(float) * kTP * K + 2 * (size_t)K * D + 2 * (size_t)kTP * D;
}

#define ENC_DISPATCH(L)      \
    switch (K) {             \
        case 8: L(8); break;   \
        case 16: L(16); break; \
        case 24: L(24); break; \
        default: L(32); break; \
    }

}  // namespace

extern "C" int tsb_encoding_fwd(const void* x, int xcs, int B, int N, int D, const float* codewords, const float* scale,
                                int K, float* a, float* d2, float* sum_a, void* E, float* ws, long long ws_floats,
                                tsb_stream_t stream) {
    int rc = check_encoding("tsb_encoding_fwd", x, xcs, B, N, D, codewords, scale, K);
    if (rc) return rc;
    TSB_REQUIRE(sum_a && E, "tsb_encoding_fwd: null pointer (sum_a, E)");
    TSB_REQUIRE((a == nullptr) == (d2 == nullptr), "tsb_encoding_fwd: a and d2 are both saved or both null");
    const long long need = (long long)B * kSlots * (K * D + K);
    TSB_REQUIRE(ws && need <= ws_floats, "tsb_encoding_fwd: workspace needs %lld floats", need);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = fwd_smem(K, D);
    const dim3 grid(kSlots, B);
#define L(KK)                                                                                                          \
    if ((rc = tsb_ensure_dyn_smem((const void*)enc_fwd_kernel<KK>, smem))) return rc;                                  \
    enc_fwd_kernel<KK><<<grid, kThreads, smem, st>>>((const __nv_bfloat16*)x, xcs, N, D, codewords, scale, a, d2, ws)
    ENC_DISPATCH(L);
#undef L
    TSB_CUDA_CHECK_LAUNCH("encoding_fwd");
    enc_fwd_finalize_kernel<<<tsb_grid_for((long long)B * K * D, kThreads, 4), kThreads, 0, st>>>(
        ws, B, D, K, codewords, sum_a, (__nv_bfloat16*)E);
    TSB_CUDA_CHECK_LAUNCH("encoding_fwd_finalize");
    return TSB_OK;
}

extern "C" int tsb_encoding_bwd(const void* dE, const void* x, int xcs, int B, int N, int D, const float* codewords,
                                const float* scale, int K, const float* a, const float* d2, const float* sum_a, void* dx,
                                int dxcs, float* dcodewords, float* dscale, float* ws, long long ws_floats,
                                tsb_stream_t stream) {
    int rc = check_encoding("tsb_encoding_bwd", x, xcs, B, N, D, codewords, scale, K);
    if (rc) return rc;
    TSB_REQUIRE(dE && a && d2 && sum_a && dx && dcodewords && dscale, "tsb_encoding_bwd: null pointer");
    TSB_REQUIRE(dxcs >= D && dxcs % 8 == 0 && tsb_aligned16(dx),
                "tsb_encoding_bwd: dx channel stride %d must be a multiple of 8 and at least D=%d, dx 16-byte aligned",
                dxcs, D);
    const long long need = (long long)B * kSlots * (K * D + 2 * K);
    TSB_REQUIRE(ws && need <= ws_floats, "tsb_encoding_bwd: workspace needs %lld floats", need);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = bwd_smem(K, D);
    const dim3 grid(kSlots, B);
#define L(KK)                                                                                                          \
    if ((rc = tsb_ensure_dyn_smem((const void*)enc_bwd_kernel<KK>, smem))) return rc;                                  \
    enc_bwd_kernel<KK><<<grid, kThreads, smem, st>>>((const __nv_bfloat16*)dE, (const __nv_bfloat16*)x, xcs, N, D,     \
                                                     codewords, scale, a, d2, (__nv_bfloat16*)dx, dxcs, ws)
    ENC_DISPATCH(L);
#undef L
    TSB_CUDA_CHECK_LAUNCH("encoding_bwd");
    enc_bwd_finalize_kernel<<<tsb_grid_for((long long)K * D, kThreads, 4), kThreads, 0, st>>>(
        ws, (const __nv_bfloat16*)dE, sum_a, B, D, K, codewords, scale, dcodewords, dscale);
    TSB_CUDA_CHECK_LAUNCH("encoding_bwd_finalize");
    return TSB_OK;
}
#undef ENC_DISPATCH

// ---- mean over the channels of each pixel ------------------------------------------------------------------------
namespace {
__global__ void chan_mean_fwd_kernel(const __nv_bfloat16* __restrict__ x, int xcs, long long npix, int C,
                                     __nv_bfloat16* __restrict__ y) {
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < npix; p += (long long)gridDim.x * blockDim.x) {
        const __nv_bfloat16* r = x + p * xcs;
        float s = 0.f;
        for (int c = 0; c < C; ++c) s += __bfloat162float(r[c]);
        y[p] = __float2bfloat16_rn(s / (float)C);
    }
}

__global__ void chan_mean_bwd_kernel(const __nv_bfloat16* __restrict__ dy, long long npix, int C,
                                     __nv_bfloat16* __restrict__ dx, int dxcs) {
    const long long total = npix * C;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long p = t / C;
        dx[p * dxcs + (t - p * C)] = __float2bfloat16_rn(__bfloat162float(dy[p]) / (float)C);
    }
}
}  // namespace

extern "C" int tsb_chan_mean_fwd(const void* x, int xcs, long long npix, int C, void* y, tsb_stream_t stream) {
    TSB_REQUIRE(x && y, "tsb_chan_mean_fwd: null pointer");
    TSB_REQUIRE(npix > 0 && C > 0 && xcs >= C, "tsb_chan_mean_fwd: bad shape npix=%lld C=%d xcs=%d", npix, C, xcs);
    chan_mean_fwd_kernel<<<tsb_grid_for(npix, kThreads, 4), kThreads, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x, xcs, npix, C, (__nv_bfloat16*)y);
    TSB_CUDA_CHECK_LAUNCH("chan_mean_fwd");
    return TSB_OK;
}

extern "C" int tsb_chan_mean_bwd(const void* dy, long long npix, int C, void* dx, int dxcs, tsb_stream_t stream) {
    TSB_REQUIRE(dy && dx, "tsb_chan_mean_bwd: null pointer");
    TSB_REQUIRE(npix > 0 && C > 0 && dxcs >= C, "tsb_chan_mean_bwd: bad shape npix=%lld C=%d dxcs=%d", npix, C, dxcs);
    chan_mean_bwd_kernel<<<tsb_grid_for(npix * C, kThreads, 4), kThreads, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)dy, npix, C, (__nv_bfloat16*)dx, dxcs);
    TSB_CUDA_CHECK_LAUNCH("chan_mean_bwd");
    return TSB_OK;
}

// ---- SE-loss: BCELoss(sigmoid(z), presence(label)) ------------------------------------------------------------------
namespace {
constexpr int kMaxSEClasses = 4096;

__global__ void se_presence_kernel(const int64_t* __restrict__ labels, long long HW, int C,
                                   uint32_t* __restrict__ presence) {
    __shared__ uint32_t bits[kMaxSEClasses / 32];
    const int nw = (C + 31) / 32, b = blockIdx.y;
    for (int w = threadIdx.x; w < nw; w += blockDim.x) bits[w] = 0u;
    __syncthreads();
    const int64_t* lab = labels + (long long)b * HW;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x) {
        const int64_t l = lab[i];
        if (l >= 0 && l < C) {
            const uint32_t m = 1u << (l & 31);
            if (!(bits[l >> 5] & m)) atomicOr(&bits[l >> 5], m);
        }
    }
    __syncthreads();
    for (int w = threadIdx.x; w < nw; w += blockDim.x)
        if (bits[w]) atomicOr(&presence[b * nw + w], bits[w]);   // OR does not depend on the order
}

// torch's BCELoss on sigmoid(z): ℓ = −(t max(log p, −100) + (1 − t) max(log(1 − p), −100)), mean over B·C, and its
// gradient through the sigmoid, (p − t) · p(1−p) / max(p(1−p), 1e-12) / n. Evaluated in fp64, as torch does on a float64
// sigmoid (B·C values: the precision costs nothing here), so where 1 − p rounds to 0 the −100 clamp decides as it does
// there; the loss is summed in a fixed tree order.
__global__ void __launch_bounds__(kThreads) se_loss_kernel(const float* __restrict__ z, int zs, int B, int C,
                                                           const uint32_t* __restrict__ presence, float* __restrict__ loss,
                                                           float* __restrict__ dz, int dzs) {
    __shared__ double red[kThreads];
    const int nw = (C + 31) / 32, n = B * C;
    double acc = 0.0;
    for (int t = threadIdx.x; t < n; t += kThreads) {
        const int b = t / C, c = t - b * C;
        const double v = z[(long long)b * zs + c];
        const bool on = (presence[b * nw + (c >> 5)] >> (c & 31)) & 1u;
        const double p = 1.0 / (1.0 + exp(-v)), q = 1.0 - p, pq = p * q;
        acc -= fmax(log(on ? p : q), -100.0);
        dz[(long long)b * dzs + c] = (float)((p - (on ? 1.0 : 0.0)) / fmax(pq, 1e-12) * pq / n);
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int s = kThreads / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) *loss = (float)(red[0] / n);
}
}  // namespace

extern "C" int tsb_se_loss_fwd_bwd(const int64_t* labels, int B, long long HW, const float* z, int zs, int C,
                                   uint32_t* presence, float* loss, float* dz_unit, int dzs, tsb_stream_t stream) {
    TSB_REQUIRE(labels && z && presence && loss && dz_unit, "tsb_se_loss_fwd_bwd: null pointer");
    TSB_REQUIRE(B > 0 && HW > 0 && C > 0 && zs >= C && dzs >= C, "tsb_se_loss_fwd_bwd: bad shape B=%d HW=%lld C=%d zs=%d dzs=%d",
                B, HW, C, zs, dzs);
    if (C > kMaxSEClasses) TSB_FAIL(TSB_ERR_UNSUPPORTED, "tsb_se_loss_fwd_bwd: C=%d exceeds %d classes", C, kMaxSEClasses);
    TSB_REQUIRE((long long)B * C < (1LL << 31), "tsb_se_loss_fwd_bwd: B*C must be below 2^31");
    cudaStream_t st = (cudaStream_t)stream;
    const int nw = (C + 31) / 32;
    TSB_CUDA_CALL(cudaMemsetAsync(presence, 0, sizeof(uint32_t) * B * nw, st));
    long long per = (HW + kThreads * 8 - 1) / (kThreads * 8);
    const dim3 grid((unsigned)(per < 64 ? per : 64), B);
    se_presence_kernel<<<grid, kThreads, 0, st>>>(labels, HW, C, presence);
    TSB_CUDA_CHECK_LAUNCH("se_presence");
    se_loss_kernel<<<1, kThreads, 0, st>>>(z, zs, B, C, presence, loss, dz_unit, dzs);
    TSB_CUDA_CHECK_LAUNCH("se_loss");
    return TSB_OK;
}
