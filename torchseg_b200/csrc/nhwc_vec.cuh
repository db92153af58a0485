// 8-channel (16-byte for bf16) vector access helpers for NHWC tensors with a channel stride, and the grid-stride walk
// of the streaming NHWC kernels built on them.
#pragma once
#include "tsb_common.cuh"

// Threads per CTA of every NHWC streaming kernel; the walk's stride and the column-reduction geometry depend on it.
constexpr int kThreads = 256;

// an NHWC operand read or written with 16-byte vectors: C > 0, C and its channel stride multiples of 8, cs >= C, aligned
#define TSB_VEC_OK(C, cs, ptr) ((C) > 0 && (C) % 8 == 0 && (cs) % 8 == 0 && (cs) >= (C) && tsb_aligned16(ptr))

// Host-side geometry of the per-channel column reductions (one kThreads CTA = `groups` 8-channel groups per pass x
// `lanes` pixel lanes): shared memory for nacc accumulators per channel and lane, and the number of CTAs (workspace
// slots) that gives every lane at least pix_per_lane of npix pixels, at most `cap`.
static inline int colred_groups(int C8) { return C8 < kThreads ? C8 : kThreads; }
static inline size_t colred_smem(int C8, int nacc) {
    const int groups = colred_groups(C8);
    return sizeof(float) * (size_t)(kThreads / groups) * groups * nacc * 8;
}
static inline int colred_grid(long long npix, int C8, int pix_per_lane, long long cap) {
    const long long per_cta = (long long)(kThreads / colred_groups(C8)) * pix_per_lane;
    long long need = (npix + per_cta - 1) / per_cta;
    if (need > cap) need = cap;
    return (int)(need < 1 ? 1 : need);
}

// Calls f(DType<TI>{}, DType<TO>{}) for the fp32 / bf16 pair named by two TSB_* dtype codes; false for any other code.
template <typename T> struct DType { using type = T; };
template <typename F> bool dispatch_dtype_pair(int a, int b, F&& f) {
    if (a == TSB_BF16 && b == TSB_BF16) f(DType<__nv_bfloat16>{}, DType<__nv_bfloat16>{});
    else if (a == TSB_BF16 && b == TSB_F32) f(DType<__nv_bfloat16>{}, DType<float>{});
    else if (a == TSB_F32 && b == TSB_BF16) f(DType<float>{}, DType<__nv_bfloat16>{});
    else if (a == TSB_F32 && b == TSB_F32) f(DType<float>{}, DType<float>{});
    else return false;
    return true;
}

#ifdef __CUDACC__
template <typename T> struct Vec8;

template <> struct Vec8<__nv_bfloat16> {
    static __device__ __forceinline__ void load(const __nv_bfloat16* p, float f[8]) {
        uint4 u = *reinterpret_cast<const uint4*>(p);
        unpack8(u, f);
    }
    static __device__ __forceinline__ void store(__nv_bfloat16* p, const float f[8]) {
        *reinterpret_cast<uint4*>(p) = pack8(f);
    }
};
template <> struct Vec8<float> {
    static __device__ __forceinline__ void load(const float* p, float f[8]) {
        float4 a = *reinterpret_cast<const float4*>(p);
        float4 b = *reinterpret_cast<const float4*>(p + 4);
        f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
        f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
    }
    static __device__ __forceinline__ void store(float* p, const float f[8]) {
        *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
        *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
    }
};

// Grid-stride walk over (pixel, 8-channel group) pairs: i = pixel * C8 + c8 advances by `stride` per trip. The naive
// `i % C8`, `i / C8` costs a 64-bit integer division per 16-byte vector (~100 issue slots — half the issue bandwidth of
// a streaming kernel, ncu: 50 % issue-active on bn_apply); the walker divides once per thread.
struct VecWalk {
    long long p, dp;
    int c8, dc, C8;
    __device__ __forceinline__ VecWalk(int C8_, long long start, long long stride) : C8(C8_) {
        p = start / C8_;
        c8 = (int)(start - p * C8_);
        dp = stride / C8_;
        dc = (int)(stride - dp * C8_);
    }
    __device__ __forceinline__ void next() {
        p += dp;
        c8 += dc;
        if (c8 >= C8) { c8 -= C8; ++p; }
    }
};

// The grid-stride walk over the `total` = pixels x C8 (pixel, 8-channel group) pairs of a kThreads-thread launch:
// body(p, c8) for each pair of this thread.
template <typename F>
__device__ __forceinline__ void for_each_vec(long long total, int C8, F&& body) {
    const long long stride = (long long)gridDim.x * kThreads;
    const long long start = (long long)blockIdx.x * kThreads + threadIdx.x;
    VecWalk wk(C8, start, stride);
    for (long long i = start; i < total; i += stride, wk.next()) body(wk.p, wk.c8);
}
#endif

