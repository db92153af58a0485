// Common device/host helpers for libtsb (H100 / sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/tsb.h"

// ----------------------------------------------------------------------------------------------
// Error plumbing: every entry point returns 0 or a negative code and records a thread-local string.
// ----------------------------------------------------------------------------------------------
void tsb_set_error(const char* fmt, ...);
void tsb_count_launch(int n);
int tsb_ensure_dyn_smem(const void* func, size_t bytes);   // per-(device, function), thread-safe

// Deterministic cross-CTA sums. A kernel that would add per-CTA partials into one output with float atomics (whose
// order, hence rounding, changes from run to run) instead stores partial b into slot b of the caller's workspace
// (`ws`, `ws_floats` of the entry point); tsb_det_reduce then adds sum_b slot[b][i] (b in increasing order) to out[i].
// Slot b of the partials starts at parts + b * stride.
int tsb_det_reduce(float* out, const float* parts, int nparts, long long n, long long stride, cudaStream_t st);

#define TSB_FAIL(code, ...)            \
    do {                               \
        tsb_set_error(__VA_ARGS__);    \
        return (code);                 \
    } while (0)

#define TSB_REQUIRE(cond, ...)                         \
    do {                                               \
        if (!(cond)) TSB_FAIL(TSB_ERR_ARG, __VA_ARGS__); \
    } while (0)

#define TSB_CUDA_CHECK_LAUNCH(name)                                                     \
    do {                                                                                \
        cudaError_t e__ = cudaGetLastError();                                           \
        if (e__ != cudaSuccess)                                                         \
            TSB_FAIL(TSB_ERR_CUDA, "%s: launch failed: %s", name, cudaGetErrorString(e__)); \
        tsb_count_launch(1);                                                            \
    } while (0)

#define TSB_CUDA_CALL(expr)                                                             \
    do {                                                                                \
        cudaError_t e__ = (expr);                                                       \
        if (e__ != cudaSuccess)                                                         \
            TSB_FAIL(TSB_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(e__));    \
    } while (0)

static inline int tsb_num_sms() {
    static int sms[64] = {0};   // per device; a racing first call writes the same value twice
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (sms[dev] == 0) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
        sms[dev] = v;
    }
    return sms[dev];
}

static inline bool tsb_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// grid sized as a multiple of the SM count (grid-stride kernels)
static inline int tsb_grid_for(long long work_items, int per_block, int blocks_per_sm) {
    long long need = (work_items + per_block - 1) / per_block;
    long long cap = (long long)tsb_num_sms() * blocks_per_sm;
    if (need < 1) need = 1;
    return (int)(need < cap ? need : cap);
}

// ----------------------------------------------------------------------------------------------
// Device helpers
// ----------------------------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Block-wide sum, result valid in thread 0 (and broadcast to all through smem).
template <int kThreads>
__device__ __forceinline__ float block_sum(float v, float* smem /* >= 33 floats */) {
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) smem[wid] = v;
    __syncthreads();
    if (wid == 0) {
        float t = (lane < kThreads / 32) ? smem[lane] : 0.f;
        t = warp_sum(t);
        if (lane == 0) smem[32] = t;
    }
    __syncthreads();
    float r = smem[32];
    __syncthreads();
    return r;
}

// 128-bit streaming global accesses
__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ void stg_v4(void* p, const uint4& v) {
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// weight-gradient epilogues: store into this split's workspace slice, or add in place when the CTA is the only writer
__device__ __forceinline__ void put_f2(float* p, float a, float b, bool add) {
    float2 v = make_float2(a, b);
    if (add) { const float2 o = *reinterpret_cast<const float2*>(p); v.x += o.x; v.y += o.y; }
    *reinterpret_cast<float2*>(p) = v;
}
__device__ __forceinline__ void put_f1(float* p, float a, bool add) { *p = add ? *p + a : a; }

__device__ __forceinline__ float bf16lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// 8 consecutive bf16 <-> 8 floats
__device__ __forceinline__ void unpack8(const uint4& u, float f[8]) {
    f[0] = bf16lo(u.x); f[1] = bf16hi(u.x);
    f[2] = bf16lo(u.y); f[3] = bf16hi(u.y);
    f[4] = bf16lo(u.z); f[5] = bf16hi(u.z);
    f[6] = bf16lo(u.w); f[7] = bf16hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float f[8]) {
    uint4 u;
    u.x = pack_bf16(f[0], f[1]);
    u.y = pack_bf16(f[2], f[3]);
    u.z = pack_bf16(f[4], f[5]);
    u.w = pack_bf16(f[6], f[7]);
    return u;
}

// Generic element load/store as float for the two boundary dtypes.
template <typename T> __device__ __forceinline__ float ld_as_float(const T* p);
template <> __device__ __forceinline__ float ld_as_float<float>(const float* p) { return __ldg(p); }
template <> __device__ __forceinline__ float ld_as_float<__nv_bfloat16>(const __nv_bfloat16* p) {
    return __bfloat162float(*p);
}
template <typename T> __device__ __forceinline__ void st_from_float(T* p, float v);
template <> __device__ __forceinline__ void st_from_float<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void st_from_float<__nv_bfloat16>(__nv_bfloat16* p, float v) {
    *p = __float2bfloat16_rn(v);
}

// ----------------------------------------------------------------------------------------------
// Deterministic expf shared bit-for-bit with oracle/tsb_oracle.c (tsb_exp_det there):
// every operation is an explicit IEEE fp32 op (fmaf / mul / add), no fast-math, no contraction
// ambiguity, so the CPU oracle and the GPU produce identical p_target bits (OHEM index parity).
// Valid for x <= 0 (softmax arguments after max subtraction); returns 0 below -86.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ float tsb_exp_det(float x) {
    // branch-free: inputs below -86 (< 4.5e-38: cannot change a sum containing exp(0) = 1; keeps all results normal) are
    // evaluated at -86 and replaced by 0 with one select — a branch per class cost ~6 issue slots in the OHEM kernels
    const bool tiny = x < -86.0f;
    x = tiny ? -86.0f : x;
    const float LOG2E = 1.4426950408889634f;
    const float LN2_HI = 0.693145751953125f;          // 0x3f317200
    const float LN2_LO = 1.428606765330187e-06f;      // ln2 - LN2_HI
    float t = __fmul_rn(x, LOG2E);
    // n = rintf(t) (round-to-nearest-even) via the 1.5*2^23 trick: exact for |t| < 2^22 (here t in [-124.1, 0]) and it
    // leaves the integer in the low mantissa bits, so neither FRND nor F2I (quarter-rate conversion pipe) is issued
    const float MAGIC = 12582912.0f;   // 0x4B400000
    float z = __fadd_rn(t, MAGIC);
    float n = __fsub_rn(z, MAGIC);
    float r = fmaf(n, -LN2_HI, x);
    r = fmaf(n, -LN2_LO, r);
    // degree-6 polynomial for e^r on [-ln2/2, ln2/2]
    float p = 1.0f / 720.0f;
    p = fmaf(p, r, 1.0f / 120.0f);
    p = fmaf(p, r, 1.0f / 24.0f);
    p = fmaf(p, r, 1.0f / 6.0f);
    p = fmaf(p, r, 0.5f);
    p = fmaf(p, r, 1.0f);
    p = fmaf(p, r, 1.0f);
    // p * 2^n on the exponent field (exact: the result is normal). (bits(z) << 23) == (n << 23) mod 2^32 because the
    // magic constant's own bits are shifted out.
    const float e = __int_as_float(__float_as_int(p) + (int)((unsigned)__float_as_int(z) << 23));
    return tiny ? 0.0f : e;
}

#endif  // __CUDACC__
