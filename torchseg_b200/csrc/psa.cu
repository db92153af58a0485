// Point-wise spatial attention helpers (PSANet, TorchSeg model/psanet/ade.psanet.R101_v1c/network.py:119-138):
//   softmax over the 3600 attention channels of every pixel (torch.softmax(att.view(b,c,-1), dim=1) — in NHWC the
//   reduction dimension is the contiguous one), its backward, and the 2-D transposes that turn the per-image
//   `torch.bmm(reduce_x, softmax)` into the 1x1 implicit-GEMM convolution kernels (weights = the image's own
//   feature map, one launch per image).
// All three are HBM-bound: one read + one write of the [pixels, channels] matrix.
#include "tsb_common.cuh"
#include "nhwc_vec.cuh"

namespace {

constexpr int kSmThreads = 256;
constexpr int kMaxVecPerThread = 4;   // C <= 256 * 4 * 8 = 8192 channels per row

__device__ __forceinline__ float block_max256(float v, float* smem) {
    v = warp_max(v);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) smem[wid] = v;
    __syncthreads();
    if (wid == 0) {
        float t = (lane < kSmThreads / 32) ? smem[lane] : -INFINITY;
        t = warp_max(t);
        if (lane == 0) smem[32] = t;
    }
    __syncthreads();
    float r = smem[32];
    __syncthreads();
    return r;
}

// one CTA per row; the row lives in registers between the three passes (max, sum, normalise)
template <typename TI>
__global__ void __launch_bounds__(kSmThreads)
softmax_rows_kernel(const TI* __restrict__ in, int ics, __nv_bfloat16* __restrict__ out, int ocs, int C8,
                    int Cp8) {
    __shared__ float red[33];
    const long long row = blockIdx.x;
    const TI* src = in + row * ics;
    __nv_bfloat16* dst = out + row * ocs;
    float v[kMaxVecPerThread][8];
    float m = -INFINITY;
#pragma unroll
    for (int j = 0; j < kMaxVecPerThread; ++j) {
        int c8 = threadIdx.x + j * kSmThreads;
        if (c8 < C8) {
            Vec8<TI>::load(src + c8 * 8, v[j]);
#pragma unroll
            for (int k = 0; k < 8; ++k) m = fmaxf(m, v[j][k]);
        }
    }
    m = block_max256(m, red);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxVecPerThread; ++j) {
        int c8 = threadIdx.x + j * kSmThreads;
        if (c8 < C8) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                v[j][k] = expf(v[j][k] - m);
                s += v[j][k];
            }
        }
    }
    s = block_sum<kSmThreads>(s, red);
    const float inv = 1.f / s;
#pragma unroll
    for (int j = 0; j < kMaxVecPerThread; ++j) {
        int c8 = threadIdx.x + j * kSmThreads;
        if (c8 < C8) {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[j][k] *= inv;
            Vec8<__nv_bfloat16>::store(dst + c8 * 8, v[j]);
        } else if (c8 < Cp8) {
            *reinterpret_cast<uint4*>(dst + c8 * 8) = make_uint4(0u, 0u, 0u, 0u);   // zero the GEMM-K padding
        }
    }
}

// dA = S * (dS - Σ_c S·dS)
__global__ void __launch_bounds__(kSmThreads)
softmax_rows_bwd_kernel(const __nv_bfloat16* __restrict__ S, int scs, const __nv_bfloat16* __restrict__ dS, int dscs,
                        __nv_bfloat16* __restrict__ dA, int dacs, int C8, int Cp8) {
    __shared__ float red[33];
    const long long row = blockIdx.x;
    const __nv_bfloat16* s = S + row * scs;
    const __nv_bfloat16* g = dS + row * dscs;
    __nv_bfloat16* dst = dA + row * dacs;
    float p[kMaxVecPerThread][8], d[kMaxVecPerThread][8];
    float dot = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxVecPerThread; ++j) {
        int c8 = threadIdx.x + j * kSmThreads;
        if (c8 < C8) {
            Vec8<__nv_bfloat16>::load(s + c8 * 8, p[j]);
            Vec8<__nv_bfloat16>::load(g + c8 * 8, d[j]);
#pragma unroll
            for (int k = 0; k < 8; ++k) dot = fmaf(p[j][k], d[j][k], dot);
        }
    }
    dot = block_sum<kSmThreads>(dot, red);
#pragma unroll
    for (int j = 0; j < kMaxVecPerThread; ++j) {
        int c8 = threadIdx.x + j * kSmThreads;
        if (c8 < C8) {
#pragma unroll
            for (int k = 0; k < 8; ++k) d[j][k] = p[j][k] * (d[j][k] - dot);
            Vec8<__nv_bfloat16>::store(dst + c8 * 8, d[j]);
        } else if (c8 < Cp8) {
            *reinterpret_cast<uint4*>(dst + c8 * 8) = make_uint4(0u, 0u, 0u, 0u);
        }
    }
}

// out[c, r] = in[r, c] for r < R, c < Cc; out[c, r] = 0 for R <= r < Rp. 32x32 tiles through padded smem.
template <typename TI>
__global__ void __launch_bounds__(256)
transpose_pad_kernel(const TI* __restrict__ in, int ics, __nv_bfloat16* __restrict__ out, int ocs, int R, int Cc, int Rp) {
    __shared__ float tile[32][33];
    const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        int r = r0 + ty + k * 8, c = c0 + tx;
        float v = 0.f;
        if (r < R && c < Cc) v = (float)in[(long long)r * ics + c];
        tile[ty + k * 8][tx] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        int c = c0 + ty + k * 8, r = r0 + tx;
        if (c < Cc && r < Rp) out[(long long)c * ocs + r] = __float2bfloat16_rn(tile[tx][ty + k * 8]);
    }
}

}  // namespace

extern "C" int tsb_softmax_rows_fwd(const void* in, int idtype, int ics, void* out, int ocs, long long rows, int C, int Cp,
                                    tsb_stream_t stream) {
    TSB_REQUIRE(in && out && rows > 0 && C > 0, "tsb_softmax_rows_fwd: bad args");
    TSB_REQUIRE(idtype == TSB_BF16 || idtype == TSB_F32, "tsb_softmax_rows_fwd: bad dtype");
    TSB_REQUIRE(Cp >= C && TSB_VEC_OK(C, ics, in) && TSB_VEC_OK(Cp, ocs, out),
                "tsb_softmax_rows_fwd: C, Cp, strides must be multiples of 8, Cp >= C, strides >= C / Cp, pointers 16B aligned");
    TSB_REQUIRE(Cp <= kSmThreads * kMaxVecPerThread * 8, "tsb_softmax_rows_fwd: at most %d channels", kSmThreads * kMaxVecPerThread * 8);
    TSB_REQUIRE(rows < (1ll << 31), "tsb_softmax_rows_fwd: too many rows");
    if (idtype == TSB_BF16)
        softmax_rows_kernel<__nv_bfloat16><<<(unsigned)rows, kSmThreads, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)in, ics, (__nv_bfloat16*)out, ocs, C / 8, Cp / 8);
    else
        softmax_rows_kernel<float><<<(unsigned)rows, kSmThreads, 0, (cudaStream_t)stream>>>((const float*)in, ics, (__nv_bfloat16*)out, ocs, C / 8, Cp / 8);
    TSB_CUDA_CHECK_LAUNCH("softmax_rows");
    return TSB_OK;
}

extern "C" int tsb_softmax_rows_bwd(const void* S, int scs, const void* dS, int dscs, void* dA, int dacs, long long rows,
                                    int C, int Cp, tsb_stream_t stream) {
    TSB_REQUIRE(S && dS && dA && rows > 0 && C > 0, "tsb_softmax_rows_bwd: bad args");
    TSB_REQUIRE(Cp >= C && TSB_VEC_OK(C, scs, S) && TSB_VEC_OK(C, dscs, dS) && TSB_VEC_OK(Cp, dacs, dA),
                "tsb_softmax_rows_bwd: C, Cp, strides must be multiples of 8, Cp >= C, strides >= C / Cp, pointers 16B aligned");
    TSB_REQUIRE(Cp <= kSmThreads * kMaxVecPerThread * 8, "tsb_softmax_rows_bwd: at most %d channels", kSmThreads * kMaxVecPerThread * 8);
    TSB_REQUIRE(rows < (1ll << 31), "tsb_softmax_rows_bwd: too many rows");
    softmax_rows_bwd_kernel<<<(unsigned)rows, kSmThreads, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)S, scs, (const __nv_bfloat16*)dS, dscs, (__nv_bfloat16*)dA, dacs, C / 8, Cp / 8);
    TSB_CUDA_CHECK_LAUNCH("softmax_rows_bwd");
    return TSB_OK;
}

extern "C" int tsb_transpose_pad(const void* in, int idtype, int ics, void* out_bf16, int ocs, int R, int Cc, int Rp,
                                 tsb_stream_t stream) {
    TSB_REQUIRE(in && out_bf16 && R > 0 && Cc > 0 && Rp >= R && ocs >= Rp && ics >= Cc, "tsb_transpose_pad: bad args");
    TSB_REQUIRE(idtype == TSB_BF16 || idtype == TSB_F32, "tsb_transpose_pad: bad dtype");
    dim3 grid((Rp + 31) / 32, (Cc + 31) / 32);
    if (idtype == TSB_BF16)
        transpose_pad_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)in, ics, (__nv_bfloat16*)out_bf16, ocs, R, Cc, Rp);
    else
        transpose_pad_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)in, ics, (__nv_bfloat16*)out_bf16, ocs, R, Cc, Rp);
    TSB_CUDA_CHECK_LAUNCH("transpose_pad");
    return TSB_OK;
}
