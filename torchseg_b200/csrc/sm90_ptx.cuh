// Thin inline-PTX wrappers for the Hopper (sm_90a) async machinery used by the implicit-GEMM convolution kernels:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA from shared-memory descriptors), fences.
#pragma once
#include <stdint.h>

namespace sm90 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Warp index broadcast from lane 0. ptxas cannot prove threadIdx.x / 32 warp-uniform; a warp-role branch on it makes
// every wgmma behind it a "divergent path", and ptxas then waits for each wgmma before issuing the next (C7520).
__device__ __forceinline__ int warp_uniform_idx() { return __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0); }

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug traps (→ launch error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    for (uint32_t spin = 0; !mbar_try_wait(bar, parity); ++spin) {
        if (spin > (1u << 26)) __trap();
    }
}

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const void* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
        "[%2];" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// ------------------------------------------------------------------ wgmma (warpgroup MMA)
// Registers written by ordinary instructions must be fenced before a wgmma reads them as accumulators.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Pins accumulator registers at this point of the program, so the compiler cannot move their reads or writes across
// the asynchronous wgmma (before wgmma_fence, after wgmma_wait).
template <int N>
__device__ __forceinline__ void fence_operands(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 in, fp32 accumulators in registers, issued by a whole warpgroup.
// TA / TB = 0: K-major operand, 1: MN-major (transposed) operand. scale_d = 0 overwrites D.
// Fragment of thread t (warp w = t / 32 of the warpgroup, lane l): d[4j + 2h + e] = D[16w + l/4 + 8h][8j + 2(l%4) + e].
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}

// ------------------------------------------------------------------ stage ring
// The shared-memory stage ring between one TMA producer thread and the consumer warps of a wgmma kernel. full[s]
// completes when the TMA bytes of stage s have landed, empty[s] when every consumer warp has retired the MMAs that read
// it. Both sides walk the stages in the same order and flip the parity on every wrap.
//
// A consumer releases a stage one stage late: after issuing stage s it commits and waits until at most one group is
// pending, which retires the MMAs of stage s-1, so the tensor pipe never drains between stages. wait_group covers only
// the calling warp's MMAs, so every consumer warp releases the stage (lane 0 arrives). The ring touches no
// accumulator: the kernel pins its accumulators (fence_operands) where ordinary instructions read or write them.
struct StageRing {
    uint64_t* full;
    uint64_t* empty;
    int stages;
    int slot = 0;
    uint32_t phase = 0;
    int prev = -1;   // consumer: the stage whose MMAs may still be in flight

    __device__ __forceinline__ StageRing(uint64_t* full_bar, uint64_t* empty_bar, int n)
        : full(full_bar), empty(empty_bar), stages(n) {}
    // one thread, before fence_barrier_init()
    __device__ __forceinline__ void init(uint32_t consumer_warps) {
        for (int s = 0; s < stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], consumer_warps); }
    }
    __device__ __forceinline__ void advance() {
        if (++slot == stages) { slot = 0; phase ^= 1u; }
    }
    // producer: wait until the consumers have released the current stage; fill it through full_bar(), then advance()
    __device__ __forceinline__ void acquire() { mbar_wait(&empty[slot], phase ^ 1u); }
    __device__ __forceinline__ uint64_t* full_bar() { return &full[slot]; }
    // consumer: wait for the current stage's data; the MMAs of the stage follow
    __device__ __forceinline__ void wait_full() {
        mbar_wait(&full[slot], phase);
        wgmma_fence();
    }
    // consumer, after issuing the current stage: commit it, release the previous one, advance
    __device__ __forceinline__ void commit_release_prev() {
        wgmma_commit();
        if (prev >= 0) {
            wgmma_wait<1>();
            if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[prev]);
        }
        prev = slot;
        advance();
    }
    // consumer, after the last stage: retire every MMA and release the last stage
    __device__ __forceinline__ void drain() {
        wgmma_wait<0>();
        if (prev >= 0 && (threadIdx.x & 31) == 0) mbar_arrive(&empty[prev]);
        prev = -1;
    }
};

// ------------------------------------------------------------------ descriptors
// Shared-memory matrix descriptor (sm_90 GMMA layout): start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46),
// base_offset [49,52), layout_type [62,64) (1 = SWIZZLE_128B). The start address is OR-ed into bits [0,14) by the caller.
__host__ __device__ constexpr uint64_t desc_hi_sw128(uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) |
           ((uint64_t)1 << 62);
}
// Descriptor of an operand starting at shared address `lo` (in 16-byte units), base_offset 0. This holds also for a
// start shifted by whole 128-byte rows inside the 1024-byte swizzle pattern (the taps of a row tile): H100 takes the
// swizzle phase from the absolute shared address, and putting the row phase (lo >> 3) & 7 into base_offset was measured
// to give wrong results.
__device__ __forceinline__ uint64_t desc_at(uint64_t hi, uint32_t lo) { return hi | (uint64_t)(lo & 0x3FFFu); }


}  // namespace sm90
