// Fused dense self-attention over the pixels of each image (OCNet's object context, Base-OC) on Hopper wgmma (sm_90a):
//
//   o[b,i,:] = Σ_j softmax_j(scale · q[b,i,:]·k[b,j,:]) · v[b,j,:]        i < Nq, j < Nk, d_k = d_v = 256
//
// and its gradient. S = QKᵀ and P = softmax(S) live in registers and shared memory only; nothing of size Nq·Nk reaches
// HBM. Self-attention has Nq = Nk = N; OCRNet's pixel-region relation has the Nq pixels of an image as queries and its
// Nk = K class regions as keys and values (the tsb_cross_attention_* entry points).
// DANet's position attention, d_k = 64 and d_v = 512, has its own kernels further down (the "(64, 512)" section); what
// follows up to there describes the (256, 256) plan.
//
// Tiling: every operand tile is 64 rows x 256 channels bf16 (32 KB), loaded by TMA through a 3-D map (channels, N, B)
// as four 64-channel boxes with the 128-byte swizzle; rows past Nq (q, dO) or Nk (k, v) are zero-filled by the map and
// never leave the image.
// Score products (QKᵀ, KQᵀ, dO·Vᵀ, V·dOᵀ) are m64n64k16 wgmmas with both operands K-major; the products with a
// probability tile (P·V, Pᵀ·dO, dS·K, dSᵀ·Q) take P / dS from shared memory (written by the threads, K-major, swizzled
// like a TMA tile) and the value-side tile as an MN-major B operand, as two m64n128k16 halves.
//
// Masking: zero-filled keys would score 0, so keys j >= Nk are set to −∞ (forward) or given P = 0 (backward); query rows
// i >= Nq are computed on zeros, never stored, and their lse / δ never read.
//
// Determinism: no atomics. The forward and the dQ pass are query-stationary, the dK/dV pass is key-stationary, so every
// output element has exactly one writer and a fixed summation order.
#include "conv_common.cuh"
#include "sm90_ptx.cuh"

using namespace sm90;

namespace {

constexpr int kDim = 256;                         // head dimension (d_k = d_v)
constexpr int kChunk = 64 * 128;                  // 64 rows x 64 channels bf16: one swizzled TMA box
constexpr int kTile = 4 * kChunk;                 // 64 rows x 256 channels
constexpr int kThreads = 256;                     // two warpgroups
constexpr uint32_t kChunkU = kChunk >> 4;         // in descriptor units (16 B)
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

struct alignas(64) AttnParams {
    CUtensorMap a, b, c, d;     // forward: q, k, v; backward: q, k, v, dout
    __nv_bfloat16* out0;        // forward: o; backward: dk (key pass) / dq (query pass)
    __nv_bfloat16* out1;        // backward key pass: dv
    int cs0, cs1;
    float* lse;                 // forward output (may be null) / backward input
    const float* delta;
    int Nq, Nk;                 // queries and keys (= values) per image; the (64, 512) kernels have Nq = Nk
    float c2;                   // scale · log2(e): the softmax runs in base 2
    float scale;
    int accumulate;             // query pass: dq += result
};

__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
    return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~uintptr_t(1023));
}

// rows [row0, row0 + 64) of image b, all 256 channels, as four swizzled 64-channel boxes
__device__ __forceinline__ void load_tile(uint8_t* dst, const CUtensorMap* map, uint64_t* bar, int row0, int b) {
#pragma unroll
    for (int c = 0; c < 4; ++c) tma_load_3d(dst + c * kChunk, map, bar, 64 * c, row0, b);
}

// s[64 x 64] = A[64 x 256] · B[64 x 256]ᵀ, both operands K-major tiles
__device__ __forceinline__ void score_mma(float (&s)[32], uint32_t a_lo, uint32_t b_lo) {
    const uint64_t hk = desc_hi_sw128(16, 1024);
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int k = 0; k < 4; ++k)
            wgmma_m64n64<0, 0>(s, desc_at(hk, a_lo + c * kChunkU + 2 * k), desc_at(hk, b_lo + c * kChunkU + 2 * k),
                               (c | k) ? 1u : 0u);
}

// acc[64 x 128] += P[64 x 64] · X[64 rows x 128 channels]: P K-major (one swizzled 8 KB block), X the two 64-channel
// chunks starting at x_lo of a tile (MN-major)
__device__ __forceinline__ void prob_mma(float (&acc)[64], uint32_t p_lo, uint32_t x_lo) {
    const uint64_t hk = desc_hi_sw128(16, 1024), hmn = desc_hi_sw128(kChunk, 1024);
#pragma unroll
    for (int k = 0; k < 4; ++k)   // 16 rows of X = 2048 B = 128 descriptor units
        wgmma_m64n128<0, 1>(acc, desc_at(hk, p_lo + 2 * k), desc_at(hmn, x_lo + 128 * k), 1u);
}

__device__ __forceinline__ void mma_retire() {
    wgmma_commit();
    wgmma_wait<0>();
}

// Fragment of an m64n64 accumulator (sm90_ptx.cuh): element 4j + 2h + e is row 16w + lane/4 + 8h, column 8j + 2(lane%4) + e.
// Stores it as bf16 into a 64 x 64 K-major operand block with the 128-byte swizzle (16-byte chunk j of row r at j ^ (r & 7)).
__device__ __forceinline__ void store_operand(uint8_t* blk, const float (&f)[32], int wq, int lane) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = 16 * wq + (lane >> 2) + 8 * h;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            *reinterpret_cast<uint32_t*>(blk + r * 128 + ((j ^ (r & 7)) << 4) + 4 * (lane & 3)) =
                pack_bf16(f[4 * j + 2 * h], f[4 * j + 2 * h + 1]);
    }
}

__device__ __forceinline__ void bar_named(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// ---------------------------------------------------------------------------------------------------------------------
// forward: 128 queries per CTA, 64 per warpgroup; K/V tiles double-buffered; online softmax in base 2
// smem: Q [2 tiles] | stage 0: K, V | stage 1: K, V | P [2 x 8 KB] | barriers
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kFwdSmem = 1024 + 6 * kTile + 2 * kChunk + 64;

__global__ void __launch_bounds__(kThreads, 1) attn_fwd_kernel(const __grid_constant__ AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align1024(smem_raw);
    uint8_t* s_q = smem;
    uint8_t* s_kv = smem + 2 * kTile;
    uint8_t* s_p = smem + 6 * kTile;
    uint64_t* bar = reinterpret_cast<uint64_t*>(s_p + 2 * kChunk);   // [0] Q, [1 + s] stage s
    const int b = blockIdx.y, q0 = blockIdx.x * 128, Nq = p.Nq, Nk = p.Nk;
    const int ntiles = (Nk + 63) / 64;
    const int warp = warp_uniform_idx(), lane = threadIdx.x & 31, wg = warp >> 2, wq = warp & 3;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.a); tma_prefetch_desc(&p.b); tma_prefetch_desc(&p.c);
        for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(&bar[0], 2 * kTile);
        load_tile(s_q, &p.a, &bar[0], q0, b);
        load_tile(s_q + kTile, &p.a, &bar[0], q0 + 64, b);
        for (int s = 0; s < 2 && s < ntiles; ++s) {
            mbar_arrive_expect_tx(&bar[1 + s], 2 * kTile);
            load_tile(s_kv + s * 2 * kTile, &p.b, &bar[1 + s], 64 * s, b);
            load_tile(s_kv + s * 2 * kTile + kTile, &p.c, &bar[1 + s], 64 * s, b);
        }
    }

    float o[2][64];
#pragma unroll
    for (int i = 0; i < 64; ++i) { o[0][i] = 0.f; o[1][i] = 0.f; }
    float m2[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // running max (base 2) and this thread's partial sums
    const uint32_t q_lo = smem_u32(s_q + wg * kTile) >> 4;
    uint8_t* my_p = s_p + wg * kChunk;
    const uint32_t p_lo = smem_u32(my_p) >> 4;
    mbar_wait(&bar[0], 0);
    for (int t = 0; t < ntiles; ++t) {
        const int s = t & 1;
        mbar_wait(&bar[1 + s], (t >> 1) & 1);
        const uint32_t k_lo = smem_u32(s_kv + s * 2 * kTile) >> 4, v_lo = k_lo + (kTile >> 4);
        float sc[32];
        wgmma_fence();
        score_mma(sc, q_lo, k_lo);
        mma_retire();
        fence_operands(sc);
        float mx[2] = {m2[0], m2[1]};
        const int key0 = 64 * t + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float& x = sc[4 * j + 2 * h + e];
                    x = (key0 + 8 * j + e < Nk) ? x * p.c2 : -INFINITY;
                    mx[h] = fmaxf(mx[h], x);
                }
        float corr[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
            corr[h] = exp2f(m2[h] - mx[h]);   // 0 on the first tile (m2 = −∞; key 0 is always valid, so mx is finite)
            m2[h] = mx[h];
            l[h] *= corr[h];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float& x = sc[4 * j + 2 * h + e];
                    x = exp2f(x - mx[h]);
                    l[h] += x;
                }
        store_operand(my_p, sc, wq, lane);
#pragma unroll
        for (int i = 0; i < 64; ++i) {   // accumulator element i is row 16w + lane/4 + 8 ((i >> 1) & 1)
            o[0][i] *= corr[(i >> 1) & 1];
            o[1][i] *= corr[(i >> 1) & 1];
        }
        fence_proxy_async();
        bar_named(1 + wg, 128);
        fence_operands(o[0]);
        fence_operands(o[1]);
        wgmma_fence();
        prob_mma(o[0], p_lo, v_lo);
        prob_mma(o[1], p_lo, v_lo + 2 * kChunkU);
        mma_retire();
        fence_operands(o[0]);
        fence_operands(o[1]);
        __syncthreads();   // both warpgroups are done with stage s
        if (threadIdx.x == 0 && t + 2 < ntiles) {
            mbar_arrive_expect_tx(&bar[1 + s], 2 * kTile);
            load_tile(s_kv + s * 2 * kTile, &p.b, &bar[1 + s], 64 * (t + 2), b);
            load_tile(s_kv + s * 2 * kTile + kTile, &p.c, &bar[1 + s], 64 * (t + 2), b);
        }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
        const int row = q0 + 64 * wg + 16 * wq + (lane >> 2) + 8 * h;
        if (row >= Nq) continue;
        const float inv = 1.f / l[h];
        __nv_bfloat16* dst = p.out0 + ((long long)b * Nq + row) * p.cs0 + 2 * (lane & 3);
#pragma unroll
        for (int half = 0; half < 2; ++half)
#pragma unroll
            for (int j = 0; j < 16; ++j)
                *reinterpret_cast<uint32_t*>(dst + 128 * half + 8 * j) =
                    pack_bf16(o[half][4 * j + 2 * h] * inv, o[half][4 * j + 2 * h + 1] * inv);
        if (p.lse != nullptr && (lane & 3) == 0) p.lse[(long long)b * Nq + row] = (m2[h] + log2f(l[h])) * kLn2;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// backward, delta_i = Σ_c dO_ic · O_ic: one warp per row, 8 channels per lane
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) attn_delta_kernel(const __nv_bfloat16* __restrict__ o, int ocs,
                                                         const __nv_bfloat16* __restrict__ dout, int docs,
                                                         float* __restrict__ delta, int rows) {
    const int lane = threadIdx.x & 31;
    for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += (gridDim.x * blockDim.x) >> 5) {
        float a[8], g[8];
        unpack8(*reinterpret_cast<const uint4*>(o + (long long)r * ocs + 8 * lane), a);
        unpack8(*reinterpret_cast<const uint4*>(dout + (long long)r * docs + 8 * lane), g);
        float s = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) s = fmaf(a[e], g[e], s);
        s = warp_sum(s);
        if (lane == 0) delta[r] = s;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// backward, key-stationary: 64 keys per CTA, the image's query tiles double-buffered. Warpgroup 0 recomputes Sᵀ = K·Qᵀ, forms Pᵀ and
// accumulates dV = Pᵀ·dO; warpgroup 1 computes dPᵀ = V·dOᵀ, takes Pᵀ (fp32) from warpgroup 0 through shared memory, forms
// dSᵀ = Pᵀ ⊙ (dPᵀ − δ) and accumulates dK = scale · dSᵀ·Q. Each warpgroup holds one [64 x 256] fp32 accumulator.
// smem: K | V | stage 0: Q, dO | stage 1: Q, dO | Pᵀ bf16 | dSᵀ bf16 | Pᵀ fp32 (fragment order) | barriers
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kKvSmem = 1024 + 6 * kTile + 2 * kChunk + 32 * kThreads / 2 * 4 + 64;

__global__ void __launch_bounds__(kThreads, 1) attn_bwd_kv_kernel(const __grid_constant__ AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align1024(smem_raw);
    uint8_t* s_k = smem;
    uint8_t* s_v = smem + kTile;
    uint8_t* s_st = smem + 2 * kTile;
    uint8_t* s_p = smem + 6 * kTile;
    uint8_t* s_ds = s_p + kChunk;
    float* s_pf = reinterpret_cast<float*>(s_ds + kChunk);
    uint64_t* bar = reinterpret_cast<uint64_t*>(s_pf + 32 * 128);   // [0] K/V, [1 + s] stage s
    const int b = blockIdx.y, k0 = blockIdx.x * 64, Nq = p.Nq, Nk = p.Nk;
    const int ntiles = (Nq + 63) / 64;
    const int warp = warp_uniform_idx(), lane = threadIdx.x & 31, wg = warp >> 2, wq = warp & 3;
    const int tid = threadIdx.x & 127;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.a); tma_prefetch_desc(&p.b); tma_prefetch_desc(&p.c); tma_prefetch_desc(&p.d);
        for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(&bar[0], 2 * kTile);
        load_tile(s_k, &p.b, &bar[0], k0, b);
        load_tile(s_v, &p.c, &bar[0], k0, b);
        for (int s = 0; s < 2 && s < ntiles; ++s) {
            mbar_arrive_expect_tx(&bar[1 + s], 2 * kTile);
            load_tile(s_st + s * 2 * kTile, &p.a, &bar[1 + s], 64 * s, b);
            load_tile(s_st + s * 2 * kTile + kTile, &p.d, &bar[1 + s], 64 * s, b);
        }
    }

    float acc[2][64];   // warpgroup 0: dV, warpgroup 1: dK (unscaled)
#pragma unroll
    for (int i = 0; i < 64; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    const uint32_t k_lo = smem_u32(s_k) >> 4, v_lo = smem_u32(s_v) >> 4;
    const uint32_t p_lo = smem_u32(s_p) >> 4, ds_lo = smem_u32(s_ds) >> 4;
    const float* lse = p.lse + (long long)b * Nq;
    const float* delta = p.delta + (long long)b * Nq;
    mbar_wait(&bar[0], 0);
    for (int t = 0; t < ntiles; ++t) {
        const int s = t & 1;
        mbar_wait(&bar[1 + s], (t >> 1) & 1);
        const uint32_t q_lo = smem_u32(s_st + s * 2 * kTile) >> 4, do_lo = q_lo + (kTile >> 4);
        const int qc = 64 * t + 2 * (lane & 3);   // query (column) of fragment element 4j + 2h + e: qc + 8j + e
        float f[32];
        wgmma_fence();
        score_mma(f, wg == 0 ? k_lo : v_lo, wg == 0 ? q_lo : do_lo);
        mma_retire();
        fence_operands(f);
        if (wg == 0) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int qi = qc + 8 * j + e;
                    const float l2 = qi < Nq ? __ldg(lse + qi) * kLog2e : 0.f;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float& x = f[4 * j + 2 * h + e];
                        x = qi < Nq ? exp2f(x * p.c2 - l2) : 0.f;
                    }
                }
#pragma unroll
            for (int i = 0; i < 32; ++i) s_pf[i * 128 + tid] = f[i];
            store_operand(s_p, f, wq, lane);
            fence_proxy_async();
            bar_named(1, kThreads);   // Pᵀ is in shared memory
            fence_operands(acc[0]);
            fence_operands(acc[1]);
            wgmma_fence();
            prob_mma(acc[0], p_lo, do_lo);
            prob_mma(acc[1], p_lo, do_lo + 2 * kChunkU);
        } else {
            bar_named(1, kThreads);
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int qi = qc + 8 * j + e;
                    const float dl = qi < Nq ? __ldg(delta + qi) : 0.f;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int i = 4 * j + 2 * h + e;
                        f[i] = s_pf[i * 128 + tid] * (f[i] - dl);
                    }
                }
            store_operand(s_ds, f, wq, lane);
            fence_proxy_async();
            bar_named(2, 128);
            fence_operands(acc[0]);
            fence_operands(acc[1]);
            wgmma_fence();
            prob_mma(acc[0], ds_lo, q_lo);
            prob_mma(acc[1], ds_lo, q_lo + 2 * kChunkU);
        }
        mma_retire();
        fence_operands(acc[0]);
        fence_operands(acc[1]);
        __syncthreads();   // stage s and the P / dS blocks are free
        if (threadIdx.x == 0 && t + 2 < ntiles) {
            mbar_arrive_expect_tx(&bar[1 + s], 2 * kTile);
            load_tile(s_st + s * 2 * kTile, &p.a, &bar[1 + s], 64 * (t + 2), b);
            load_tile(s_st + s * 2 * kTile + kTile, &p.d, &bar[1 + s], 64 * (t + 2), b);
        }
    }
    const float mul = wg == 0 ? 1.f : p.scale;
    __nv_bfloat16* out = wg == 0 ? p.out1 : p.out0;
    const int cs = wg == 0 ? p.cs1 : p.cs0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = k0 + 16 * wq + (lane >> 2) + 8 * h;
        if (row >= Nk) continue;
        __nv_bfloat16* dst = out + ((long long)b * Nk + row) * cs + 2 * (lane & 3);
#pragma unroll
        for (int half = 0; half < 2; ++half)
#pragma unroll
            for (int j = 0; j < 16; ++j)
                *reinterpret_cast<uint32_t*>(dst + 128 * half + 8 * j) =
                    pack_bf16(acc[half][4 * j + 2 * h] * mul, acc[half][4 * j + 2 * h + 1] * mul);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// backward, query-stationary: 64 queries per CTA, the image's key tiles double-buffered. Warpgroup 0 recomputes S = Q·Kᵀ and P,
// warpgroup 1 computes dP = dO·Vᵀ and dS = P ⊙ (dP − δ); then warpgroup w accumulates channels [128w, 128w + 128) of
// dQ = scale · dS·K.
// smem: Q | dO | stage 0: K, V | stage 1: K, V | dS bf16 | P fp32 (fragment order) | barriers
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kQSmem = 1024 + 6 * kTile + kChunk + 32 * kThreads / 2 * 4 + 64;

__global__ void __launch_bounds__(kThreads, 1) attn_bwd_q_kernel(const __grid_constant__ AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align1024(smem_raw);
    uint8_t* s_q = smem;
    uint8_t* s_do = smem + kTile;
    uint8_t* s_st = smem + 2 * kTile;
    uint8_t* s_ds = smem + 6 * kTile;
    float* s_pf = reinterpret_cast<float*>(s_ds + kChunk);
    uint64_t* bar = reinterpret_cast<uint64_t*>(s_pf + 32 * 128);
    const int b = blockIdx.y, q0 = blockIdx.x * 64, Nq = p.Nq, Nk = p.Nk;
    const int ntiles = (Nk + 63) / 64;
    const int warp = warp_uniform_idx(), lane = threadIdx.x & 31, wg = warp >> 2, wq = warp & 3;
    const int tid = threadIdx.x & 127;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.a); tma_prefetch_desc(&p.b); tma_prefetch_desc(&p.c); tma_prefetch_desc(&p.d);
        for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(&bar[0], 2 * kTile);
        load_tile(s_q, &p.a, &bar[0], q0, b);
        load_tile(s_do, &p.d, &bar[0], q0, b);
        for (int s = 0; s < 2 && s < ntiles; ++s) {
            mbar_arrive_expect_tx(&bar[1 + s], 2 * kTile);
            load_tile(s_st + s * 2 * kTile, &p.b, &bar[1 + s], 64 * s, b);
            load_tile(s_st + s * 2 * kTile + kTile, &p.c, &bar[1 + s], 64 * s, b);
        }
    }

    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    // the two rows of this thread's fragment: base-2 lse (warpgroup 0) or δ (warpgroup 1)
    float rv[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = q0 + 16 * wq + (lane >> 2) + 8 * h;
        rv[h] = row < Nq ? (wg == 0 ? p.lse[(long long)b * Nq + row] * kLog2e : p.delta[(long long)b * Nq + row]) : 0.f;
    }
    const uint32_t q_lo = smem_u32(s_q) >> 4, do_lo = smem_u32(s_do) >> 4, ds_lo = smem_u32(s_ds) >> 4;
    mbar_wait(&bar[0], 0);
    for (int t = 0; t < ntiles; ++t) {
        const int s = t & 1;
        mbar_wait(&bar[1 + s], (t >> 1) & 1);
        const uint32_t k_lo = smem_u32(s_st + s * 2 * kTile) >> 4, v_lo = k_lo + (kTile >> 4);
        float f[32];
        wgmma_fence();
        score_mma(f, wg == 0 ? q_lo : do_lo, wg == 0 ? k_lo : v_lo);
        mma_retire();
        fence_operands(f);
        const int kc = 64 * t + 2 * (lane & 3);
        if (wg == 0) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float& x = f[4 * j + 2 * h + e];
                        x = kc + 8 * j + e < Nk ? exp2f(x * p.c2 - rv[h]) : 0.f;
                    }
#pragma unroll
            for (int i = 0; i < 32; ++i) s_pf[i * 128 + tid] = f[i];
            bar_named(1, kThreads);   // P is in shared memory
        } else {
            bar_named(1, kThreads);
#pragma unroll
            for (int i = 0; i < 32; ++i) f[i] = s_pf[i * 128 + tid] * (f[i] - rv[(i >> 1) & 1]);
            store_operand(s_ds, f, wq, lane);
            fence_proxy_async();
        }
        bar_named(1, kThreads);   // dS is in shared memory
        fence_operands(acc);
        wgmma_fence();
        prob_mma(acc, ds_lo, k_lo + 2 * wg * kChunkU);
        mma_retire();
        fence_operands(acc);
        __syncthreads();
        if (threadIdx.x == 0 && t + 2 < ntiles) {
            mbar_arrive_expect_tx(&bar[1 + s], 2 * kTile);
            load_tile(s_st + s * 2 * kTile, &p.b, &bar[1 + s], 64 * (t + 2), b);
            load_tile(s_st + s * 2 * kTile + kTile, &p.c, &bar[1 + s], 64 * (t + 2), b);
        }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = q0 + 16 * wq + (lane >> 2) + 8 * h;
        if (row >= Nq) continue;
        __nv_bfloat16* dst = p.out0 + ((long long)b * Nq + row) * p.cs0 + 128 * wg + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            uint32_t* d = reinterpret_cast<uint32_t*>(dst + 8 * j);
            float v0 = acc[4 * j + 2 * h] * p.scale, v1 = acc[4 * j + 2 * h + 1] * p.scale;
            if (p.accumulate) {
                const uint32_t u = *d;
                v0 += bf16lo(u);
                v1 += bf16hi(u);
            }
            *d = pack_bf16(v0, v1);
        }
    }
}

// =====================================================================================================================
// (d_k, d_v) = (64, 512): DANet's position attention. q / k tiles are one 64-channel box (8 KB). v, o and dv are split
// into 256-channel slices along blockIdx.z, so an O or dV accumulator is the same [64 x 256] fp32 per warpgroup (128
// registers per thread) as at (256, 256); each slice's CTA recomputes S = QKᵀ, 1/8 of the cost of its P·V. The 512-deep
// dP = dO·Vᵀ needs the whole value width, so the backward runs a dV pass per slice (which needs no dP) and separate
// key- and query-stationary passes for dK and dQ.
// =====================================================================================================================
constexpr int kNarrow = 64;                // d_k
constexpr int kWide = 512;                 // d_v
constexpr int kSlice = 256;                // value channels per CTA of the forward and the dV pass
constexpr int kWideTile = 8 * kChunk;      // 64 rows x 512 channels
constexpr int kWideStage = kChunk + kTile; // a q or k box and a 256-channel value slice

// kBoxes 64-channel boxes of rows [row0, row0 + 64) of image b, starting at channel c0
template <int kBoxes>
__device__ __forceinline__ void load_boxes(uint8_t* dst, const CUtensorMap* map, uint64_t* bar, int c0, int row0, int b) {
#pragma unroll
    for (int c = 0; c < kBoxes; ++c) tma_load_3d(dst + c * kChunk, map, bar, c0 + 64 * c, row0, b);
}

// s[64 x 64] = A[64 x 64·kBoxes] · B[64 x 64·kBoxes]ᵀ, both operands K-major
template <int kBoxes>
__device__ __forceinline__ void score_mma_boxes(float (&s)[32], uint32_t a_lo, uint32_t b_lo) {
    const uint64_t hk = desc_hi_sw128(16, 1024);
#pragma unroll
    for (int c = 0; c < kBoxes; ++c)
#pragma unroll
        for (int k = 0; k < 4; ++k)
            wgmma_m64n64<0, 0>(s, desc_at(hk, a_lo + c * kChunkU + 2 * k), desc_at(hk, b_lo + c * kChunkU + 2 * k),
                               (c | k) ? 1u : 0u);
}

// acc[64 x 64] += P[64 x 64] · X[64 rows x 64 channels]: P K-major, X one box (MN-major)
__device__ __forceinline__ void prob_mma_box(float (&acc)[32], uint32_t p_lo, uint32_t x_lo) {
    const uint64_t hk = desc_hi_sw128(16, 1024), hmn = desc_hi_sw128(kChunk, 1024);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64<0, 1>(acc, desc_at(hk, p_lo + 2 * k), desc_at(hmn, x_lo + 128 * k), 1u);
}

// ---------------------------------------------------------------------------------------------------------------------
// forward at (64, 512): 128 queries and one 256-channel value slice per CTA, K / V tiles double-buffered. Both slices
// compute the same scores and soft-max statistics; slice 0 writes lse.
// smem: Q [2 boxes] | stage 0: K box, V slice | stage 1: K box, V slice | P [2 x 8 KB] | barriers
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kFwdWideSmem = 1024 + 2 * kChunk + 2 * kWideStage + 2 * kChunk + 64;

__global__ void __launch_bounds__(kThreads, 1) attn_fwd_wide_kernel(const __grid_constant__ AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align1024(smem_raw);
    uint8_t* s_q = smem;
    uint8_t* s_kv = smem + 2 * kChunk;
    uint8_t* s_p = s_kv + 2 * kWideStage;
    uint64_t* bar = reinterpret_cast<uint64_t*>(s_p + 2 * kChunk);   // [0] Q, [1 + s] stage s
    const int b = blockIdx.y, q0 = blockIdx.x * 128, vc = blockIdx.z * kSlice, N = p.Nq;
    const int ntiles = (N + 63) / 64;
    const int warp = warp_uniform_idx(), lane = threadIdx.x & 31, wg = warp >> 2, wq = warp & 3;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.a); tma_prefetch_desc(&p.b); tma_prefetch_desc(&p.c);
        for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(&bar[0], 2 * kChunk);
        load_boxes<1>(s_q, &p.a, &bar[0], 0, q0, b);
        load_boxes<1>(s_q + kChunk, &p.a, &bar[0], 0, q0 + 64, b);
        for (int s = 0; s < 2 && s < ntiles; ++s) {
            mbar_arrive_expect_tx(&bar[1 + s], kWideStage);
            load_boxes<1>(s_kv + s * kWideStage, &p.b, &bar[1 + s], 0, 64 * s, b);
            load_boxes<4>(s_kv + s * kWideStage + kChunk, &p.c, &bar[1 + s], vc, 64 * s, b);
        }
    }

    float o[2][64];
#pragma unroll
    for (int i = 0; i < 64; ++i) { o[0][i] = 0.f; o[1][i] = 0.f; }
    float m2[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    const uint32_t q_lo = smem_u32(s_q + wg * kChunk) >> 4;
    uint8_t* my_p = s_p + wg * kChunk;
    const uint32_t p_lo = smem_u32(my_p) >> 4;
    mbar_wait(&bar[0], 0);
    for (int t = 0; t < ntiles; ++t) {
        const int s = t & 1;
        mbar_wait(&bar[1 + s], (t >> 1) & 1);
        const uint32_t k_lo = smem_u32(s_kv + s * kWideStage) >> 4, v_lo = k_lo + kChunkU;
        float sc[32];
        wgmma_fence();
        score_mma_boxes<1>(sc, q_lo, k_lo);
        mma_retire();
        fence_operands(sc);
        float mx[2] = {m2[0], m2[1]};
        const int key0 = 64 * t + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float& x = sc[4 * j + 2 * h + e];
                    x = (key0 + 8 * j + e < N) ? x * p.c2 : -INFINITY;
                    mx[h] = fmaxf(mx[h], x);
                }
        float corr[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
            corr[h] = exp2f(m2[h] - mx[h]);
            m2[h] = mx[h];
            l[h] *= corr[h];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float& x = sc[4 * j + 2 * h + e];
                    x = exp2f(x - mx[h]);
                    l[h] += x;
                }
        store_operand(my_p, sc, wq, lane);
#pragma unroll
        for (int i = 0; i < 64; ++i) {
            o[0][i] *= corr[(i >> 1) & 1];
            o[1][i] *= corr[(i >> 1) & 1];
        }
        fence_proxy_async();
        bar_named(1 + wg, 128);
        fence_operands(o[0]);
        fence_operands(o[1]);
        wgmma_fence();
        prob_mma(o[0], p_lo, v_lo);
        prob_mma(o[1], p_lo, v_lo + 2 * kChunkU);
        mma_retire();
        fence_operands(o[0]);
        fence_operands(o[1]);
        __syncthreads();   // both warpgroups are done with stage s
        if (threadIdx.x == 0 && t + 2 < ntiles) {
            mbar_arrive_expect_tx(&bar[1 + s], kWideStage);
            load_boxes<1>(s_kv + s * kWideStage, &p.b, &bar[1 + s], 0, 64 * (t + 2), b);
            load_boxes<4>(s_kv + s * kWideStage + kChunk, &p.c, &bar[1 + s], vc, 64 * (t + 2), b);
        }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
        const int row = q0 + 64 * wg + 16 * wq + (lane >> 2) + 8 * h;
        if (row >= N) continue;
        const float inv = 1.f / l[h];
        __nv_bfloat16* dst = p.out0 + ((long long)b * N + row) * p.cs0 + vc + 2 * (lane & 3);
#pragma unroll
        for (int half = 0; half < 2; ++half)
#pragma unroll
            for (int j = 0; j < 16; ++j)
                *reinterpret_cast<uint32_t*>(dst + 128 * half + 8 * j) =
                    pack_bf16(o[half][4 * j + 2 * h] * inv, o[half][4 * j + 2 * h + 1] * inv);
        if (p.lse != nullptr && blockIdx.z == 0 && (lane & 3) == 0)
            p.lse[(long long)b * N + row] = (m2[h] + log2f(l[h])) * kLn2;
    }
}

// backward at (64, 512), δ_i = Σ_c dO_ic · O_ic over 512 channels: one warp per row, 8 channels per lane per 256
__global__ void __launch_bounds__(256) attn_delta_wide_kernel(const __nv_bfloat16* __restrict__ o, int ocs,
                                                              const __nv_bfloat16* __restrict__ dout, int docs,
                                                              float* __restrict__ delta, int rows) {
    const int lane = threadIdx.x & 31;
    for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += (gridDim.x * blockDim.x) >> 5) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < kWide; c += 256) {
            float a[8], g[8];
            unpack8(*reinterpret_cast<const uint4*>(o + (long long)r * ocs + c + 8 * lane), a);
            unpack8(*reinterpret_cast<const uint4*>(dout + (long long)r * docs + c + 8 * lane), g);
#pragma unroll
            for (int e = 0; e < 8; ++e) s = fmaf(a[e], g[e], s);
        }
        s = warp_sum(s);
        if (lane == 0) delta[r] = s;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// backward at (64, 512), dV: key-stationary, 128 keys and one 256-channel slice per CTA, query tiles double-buffered.
// Each warpgroup recomputes Pᵀ = exp(scale · K·Qᵀ − lse) for its 64 keys and accumulates its [64 x 256] slice of
// dV = Pᵀ·dO. No dP is needed.
// smem: K [2 boxes] | stage 0: Q box, dO slice | stage 1: Q box, dO slice | Pᵀ [2 x 8 KB] | barriers
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kDvWideSmem = kFwdWideSmem;

__global__ void __launch_bounds__(kThreads, 1) attn_bwd_dv_wide_kernel(const __grid_constant__ AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align1024(smem_raw);
    uint8_t* s_k = smem;
    uint8_t* s_st = smem + 2 * kChunk;
    uint8_t* s_p = s_st + 2 * kWideStage;
    uint64_t* bar = reinterpret_cast<uint64_t*>(s_p + 2 * kChunk);   // [0] K, [1 + s] stage s
    const int b = blockIdx.y, k0 = blockIdx.x * 128, vc = blockIdx.z * kSlice, N = p.Nq;
    const int ntiles = (N + 63) / 64;
    const int warp = warp_uniform_idx(), lane = threadIdx.x & 31, wg = warp >> 2, wq = warp & 3;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.a); tma_prefetch_desc(&p.b); tma_prefetch_desc(&p.d);
        for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(&bar[0], 2 * kChunk);
        load_boxes<1>(s_k, &p.b, &bar[0], 0, k0, b);
        load_boxes<1>(s_k + kChunk, &p.b, &bar[0], 0, k0 + 64, b);
        for (int s = 0; s < 2 && s < ntiles; ++s) {
            mbar_arrive_expect_tx(&bar[1 + s], kWideStage);
            load_boxes<1>(s_st + s * kWideStage, &p.a, &bar[1 + s], 0, 64 * s, b);
            load_boxes<4>(s_st + s * kWideStage + kChunk, &p.d, &bar[1 + s], vc, 64 * s, b);
        }
    }

    float acc[2][64];
#pragma unroll
    for (int i = 0; i < 64; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    const uint32_t k_lo = smem_u32(s_k + wg * kChunk) >> 4;
    uint8_t* my_p = s_p + wg * kChunk;
    const uint32_t p_lo = smem_u32(my_p) >> 4;
    const float* lse = p.lse + (long long)b * N;
    mbar_wait(&bar[0], 0);
    for (int t = 0; t < ntiles; ++t) {
        const int s = t & 1;
        mbar_wait(&bar[1 + s], (t >> 1) & 1);
        const uint32_t q_lo = smem_u32(s_st + s * kWideStage) >> 4, do_lo = q_lo + kChunkU;
        float f[32];
        wgmma_fence();
        score_mma_boxes<1>(f, k_lo, q_lo);
        mma_retire();
        fence_operands(f);
        const int qc = 64 * t + 2 * (lane & 3);   // query (column) of fragment element 4j + 2h + e: qc + 8j + e
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int qi = qc + 8 * j + e;
                const float l2 = qi < N ? __ldg(lse + qi) * kLog2e : 0.f;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float& x = f[4 * j + 2 * h + e];
                    x = qi < N ? exp2f(x * p.c2 - l2) : 0.f;
                }
            }
        store_operand(my_p, f, wq, lane);
        fence_proxy_async();
        bar_named(1 + wg, 128);
        fence_operands(acc[0]);
        fence_operands(acc[1]);
        wgmma_fence();
        prob_mma(acc[0], p_lo, do_lo);
        prob_mma(acc[1], p_lo, do_lo + 2 * kChunkU);
        mma_retire();
        fence_operands(acc[0]);
        fence_operands(acc[1]);
        __syncthreads();   // both warpgroups are done with stage s
        if (threadIdx.x == 0 && t + 2 < ntiles) {
            mbar_arrive_expect_tx(&bar[1 + s], kWideStage);
            load_boxes<1>(s_st + s * kWideStage, &p.a, &bar[1 + s], 0, 64 * (t + 2), b);
            load_boxes<4>(s_st + s * kWideStage + kChunk, &p.d, &bar[1 + s], vc, 64 * (t + 2), b);
        }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = k0 + 64 * wg + 16 * wq + (lane >> 2) + 8 * h;
        if (row >= N) continue;
        __nv_bfloat16* dst = p.out1 + ((long long)b * N + row) * p.cs1 + vc + 2 * (lane & 3);
#pragma unroll
        for (int half = 0; half < 2; ++half)
#pragma unroll
            for (int j = 0; j < 16; ++j)
                *reinterpret_cast<uint32_t*>(dst + 128 * half + 8 * j) =
                    pack_bf16(acc[half][4 * j + 2 * h], acc[half][4 * j + 2 * h + 1]);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// backward at (64, 512), dK (kKeyPass, key-stationary) and dQ (query-stationary): 64 rows per CTA. Warpgroup 0
// recomputes the scores from the 64-channel operands and P; warpgroup 1 computes the 512-deep dP from the value-side
// operands, forms dS = P ⊙ (dP − δ) and accumulates scale · dS·X' into the [64 x 64] result.
//   key pass:   X = K, X' = Q (streamed), Y = V,  Y' = dO: dKᵀ rows, lse and δ indexed by the tile's column (query)
//   query pass: X = Q, X' = K (streamed), Y = dO, Y' = V:  dQ rows,  lse and δ indexed by the row (query)
// X' is double-buffered, the 64 KB Y' single-buffered: the next tile's loads go out as soon as warpgroup 1 has retired
// dP (the barrier that hands P over), so they overlap dS and the dS·X' product.
// smem: X box | Y [8 boxes] | X' [2 boxes] | Y' [8 boxes] | P fp32 [2 x 16 KB] (fragment order) | dS bf16 | barriers
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kDsWideSmem = 1024 + kChunk + kWideTile + 2 * kChunk + kWideTile + 2 * 32 * 128 * 4 + kChunk + 64;

template <bool kKeyPass>
__global__ void __launch_bounds__(kThreads, 1) attn_bwd_ds_wide_kernel(const __grid_constant__ AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align1024(smem_raw);
    uint8_t* s_x = smem;
    uint8_t* s_y = s_x + kChunk;
    uint8_t* s_xs = s_y + kWideTile;
    uint8_t* s_ys = s_xs + 2 * kChunk;
    float* s_pf = reinterpret_cast<float*>(s_ys + kWideTile);
    uint8_t* s_ds = reinterpret_cast<uint8_t*>(s_pf + 2 * 32 * 128);
    uint64_t* bar = reinterpret_cast<uint64_t*>(s_ds + kChunk);   // [0] X / Y, [1 + s] tiles t with t % 2 == s
    const CUtensorMap* mx = kKeyPass ? &p.b : &p.a;
    const CUtensorMap* mxs = kKeyPass ? &p.a : &p.b;
    const CUtensorMap* my = kKeyPass ? &p.c : &p.d;
    const CUtensorMap* mys = kKeyPass ? &p.d : &p.c;
    const int b = blockIdx.y, r0 = blockIdx.x * 64, N = p.Nq;
    const int ntiles = (N + 63) / 64;
    const int warp = warp_uniform_idx(), lane = threadIdx.x & 31, wg = warp >> 2, wq = warp & 3;
    const int tid = threadIdx.x & 127;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.a); tma_prefetch_desc(&p.b); tma_prefetch_desc(&p.c); tma_prefetch_desc(&p.d);
        for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(&bar[0], kChunk + kWideTile);
        load_boxes<1>(s_x, mx, &bar[0], 0, r0, b);
        load_boxes<8>(s_y, my, &bar[0], 0, r0, b);
        mbar_arrive_expect_tx(&bar[1], kChunk + kWideTile);
        load_boxes<1>(s_xs, mxs, &bar[1], 0, 0, b);
        load_boxes<8>(s_ys, mys, &bar[1], 0, 0, b);
    }

    float acc[32];   // warpgroup 1
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    const float* lse = p.lse + (long long)b * N;
    const float* delta = p.delta + (long long)b * N;
    float rv[2] = {0.f, 0.f};   // query pass: the base-2 lse (warpgroup 0) or δ (warpgroup 1) of this thread's two rows
    if (!kKeyPass) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + 16 * wq + (lane >> 2) + 8 * h;
            rv[h] = row < N ? (wg == 0 ? lse[row] * kLog2e : delta[row]) : 0.f;
        }
    }
    const uint32_t x_lo = smem_u32(s_x) >> 4, y_lo = smem_u32(s_y) >> 4, ys_lo = smem_u32(s_ys) >> 4;
    const uint32_t ds_lo = smem_u32(s_ds) >> 4;
    mbar_wait(&bar[0], 0);
    for (int t = 0; t < ntiles; ++t) {
        const int s = t & 1;
        mbar_wait(&bar[1 + s], (t >> 1) & 1);
        const uint32_t xs_lo = smem_u32(s_xs + s * kChunk) >> 4;
        float* pf = s_pf + s * 32 * 128;
        const int cc = 64 * t + 2 * (lane & 3);   // streamed row (column) of fragment element 4j + 2h + e: cc + 8j + e
        float f[32];
        wgmma_fence();
        if (wg == 0)
            score_mma_boxes<1>(f, x_lo, xs_lo);
        else
            score_mma_boxes<8>(f, y_lo, ys_lo);
        mma_retire();
        fence_operands(f);
        if (wg == 0) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int ci = cc + 8 * j + e;
                    const float l2 = kKeyPass && ci < N ? __ldg(lse + ci) * kLog2e : 0.f;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float& x = f[4 * j + 2 * h + e];
                        x = ci < N ? exp2f(x * p.c2 - (kKeyPass ? l2 : rv[h])) : 0.f;
                    }
                }
#pragma unroll
            for (int i = 0; i < 32; ++i) pf[i * 128 + tid] = f[i];
            bar_named(1, kThreads);   // P is in shared memory, and warpgroup 1 has retired dP: Y' is free
            if (threadIdx.x == 0 && t + 1 < ntiles) {
                // X' of stage s ^ 1 was last read by tile t − 1, which warpgroup 1 finished before the barrier
                mbar_arrive_expect_tx(&bar[2 - s], kChunk + kWideTile);
                load_boxes<1>(s_xs + (s ^ 1) * kChunk, mxs, &bar[2 - s], 0, 64 * (t + 1), b);
                load_boxes<8>(s_ys, mys, &bar[2 - s], 0, 64 * (t + 1), b);
            }
        } else {
            bar_named(1, kThreads);
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int ci = cc + 8 * j + e;
                    const float dl = kKeyPass && ci < N ? __ldg(delta + ci) : 0.f;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int i = 4 * j + 2 * h + e;
                        f[i] = pf[i * 128 + tid] * (f[i] - (kKeyPass ? dl : rv[h]));
                    }
                }
            store_operand(s_ds, f, wq, lane);
            fence_proxy_async();
            bar_named(2, 128);
            fence_operands(acc);
            wgmma_fence();
            prob_mma_box(acc, ds_lo, xs_lo);
            mma_retire();
            fence_operands(acc);
        }
    }
    if (wg == 0) return;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = r0 + 16 * wq + (lane >> 2) + 8 * h;
        if (row >= N) continue;
        __nv_bfloat16* dst = p.out0 + ((long long)b * N + row) * p.cs0 + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            uint32_t* d = reinterpret_cast<uint32_t*>(dst + 8 * j);
            float v0 = acc[4 * j + 2 * h] * p.scale, v1 = acc[4 * j + 2 * h + 1] * p.scale;
            if (p.accumulate) {
                const uint32_t u = *d;
                v0 += bf16lo(u);
                v1 += bf16hi(u);
            }
            *d = pack_bf16(v0, v1);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
int check_operand(const char* who, const char* name, const void* ptr, int cs, int dim) {
    TSB_REQUIRE(ptr != nullptr, "%s: null %s", who, name);
    TSB_REQUIRE(tsb_aligned16(ptr) && cs >= dim && cs % 8 == 0,
                "%s: %s must be 16-byte aligned with a channel stride that is a multiple of 8 and >= %d (got %d)", who,
                name, dim, cs);
    return TSB_OK;
}

// the implemented (d_k, d_v) pairs: (256, 256) (OCNet) and (64, 512) (DANet's position attention)
int check_shape(const char* who, int B, int N, int dim_k, int dim_v, float scale) {
    TSB_REQUIRE(B >= 1 && N >= 1, "%s: bad shape B=%d N=%d", who, B, N);
    TSB_REQUIRE((long long)B * N < (1LL << 31) && B <= 65535, "%s: B*N must be below 2^31 and B at most 65535", who);
    TSB_REQUIRE(scale > 0.f && scale < INFINITY, "%s: scale must be positive and finite", who);
    if (!(dim_k == kDim && dim_v == kDim) && !(dim_k == kNarrow && dim_v == kWide))
        TSB_FAIL(TSB_ERR_UNSUPPORTED, "%s: d_k=%d d_v=%d, only (d_k, d_v) = (%d, %d) or (%d, %d) is supported", who, dim_k,
                 dim_v, kDim, kDim, kNarrow, kWide);
    return TSB_OK;
}

// cross attention (Nq queries, Nk keys / values per image): (d_k, d_v) = (256, 256) only
int check_cross_shape(const char* who, int B, int Nq, int Nk, int dim_k, int dim_v, float scale) {
    TSB_REQUIRE(B >= 1 && Nq >= 1 && Nk >= 1, "%s: bad shape B=%d Nq=%d Nk=%d", who, B, Nq, Nk);
    TSB_REQUIRE((long long)B * Nq < (1LL << 31) && (long long)B * Nk < (1LL << 31) && B <= 65535,
                "%s: B*Nq and B*Nk must be below 2^31 and B at most 65535", who);
    TSB_REQUIRE(scale > 0.f && scale < INFINITY, "%s: scale must be positive and finite", who);
    if (!(dim_k == kDim && dim_v == kDim))
        TSB_FAIL(TSB_ERR_UNSUPPORTED, "%s: d_k=%d d_v=%d, only (d_k, d_v) = (%d, %d) is supported", who, dim_k, dim_v,
                 kDim, kDim);
    return TSB_OK;
}

int encode_rows(CUtensorMap* m, const void* x, int cs, int B, int N, int dim) {
    return convhost::encode_3d(m, x, dim, (uint64_t)N, (uint64_t)B, (uint64_t)cs * 2, (uint64_t)N * cs * 2, 64, 64, 1);
}

#define ATTN_CHECK(expr) do { int rc_ = (expr); if (rc_) return rc_; } while (0)

// the forward after the shape check: q and o have Nq rows per image, k and v Nk (Nq == Nk at (64, 512))
int attention_fwd(const char* who, const void* q, int qcs, const void* k, int kcs, const void* v, int vcs, void* o,
                  int ocs, float* lse, int B, int Nq, int Nk, int dim_k, int dim_v, float scale, cudaStream_t st) {
    ATTN_CHECK(check_operand(who, "q", q, qcs, dim_k));
    ATTN_CHECK(check_operand(who, "k", k, kcs, dim_k));
    ATTN_CHECK(check_operand(who, "v", v, vcs, dim_v));
    ATTN_CHECK(check_operand(who, "o", o, ocs, dim_v));
    TSB_REQUIRE(lse == nullptr || tsb_aligned16(lse), "%s: lse must be 16-byte aligned", who);
    AttnParams prm;
    memset(&prm, 0, sizeof(prm));
    ATTN_CHECK(encode_rows(&prm.a, q, qcs, B, Nq, dim_k));
    ATTN_CHECK(encode_rows(&prm.b, k, kcs, B, Nk, dim_k));
    ATTN_CHECK(encode_rows(&prm.c, v, vcs, B, Nk, dim_v));
    prm.out0 = (__nv_bfloat16*)o; prm.cs0 = ocs;
    prm.lse = lse; prm.Nq = Nq; prm.Nk = Nk; prm.c2 = scale * kLog2e; prm.scale = scale;
    if (dim_k == kNarrow) {
        ATTN_CHECK(tsb_ensure_dyn_smem(reinterpret_cast<const void*>(attn_fwd_wide_kernel), kFwdWideSmem));
        attn_fwd_wide_kernel<<<dim3((Nq + 127) / 128, B, kWide / kSlice), kThreads, kFwdWideSmem, st>>>(prm);
        TSB_CUDA_CHECK_LAUNCH("attention_fwd_wide");
        return TSB_OK;
    }
    ATTN_CHECK(tsb_ensure_dyn_smem(reinterpret_cast<const void*>(attn_fwd_kernel), kFwdSmem));
    attn_fwd_kernel<<<dim3((Nq + 127) / 128, B), kThreads, kFwdSmem, st>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("attention_fwd");
    return TSB_OK;
}

// the (64, 512) backward: δ, then dV per value slice, dK, and dQ (after dK, so that dq == dk with dq_accumulate adds
// onto the finished dK)
int attention_bwd_wide(AttnParams& prm, const void* o, int ocs, const void* dout, int docs, float* delta_ws, void* dq,
                       int dqcs, void* dk, int dkcs, void* dv, int dvcs, int dq_accumulate, int B, int N,
                       cudaStream_t st) {
    const int rows = B * N;
    attn_delta_wide_kernel<<<tsb_grid_for(rows, 8, 8), 256, 0, st>>>((const __nv_bfloat16*)o, ocs,
                                                                     (const __nv_bfloat16*)dout, docs, delta_ws, rows);
    TSB_CUDA_CHECK_LAUNCH("attention_delta_wide");
    prm.out1 = (__nv_bfloat16*)dv; prm.cs1 = dvcs;
    ATTN_CHECK(tsb_ensure_dyn_smem(reinterpret_cast<const void*>(attn_bwd_dv_wide_kernel), kDvWideSmem));
    attn_bwd_dv_wide_kernel<<<dim3((N + 127) / 128, B, kWide / kSlice), kThreads, kDvWideSmem, st>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("attention_bwd_dv_wide");
    prm.out1 = nullptr; prm.cs1 = 0;
    const dim3 grid((N + 63) / 64, B);
    prm.out0 = (__nv_bfloat16*)dk; prm.cs0 = dkcs;
    ATTN_CHECK(tsb_ensure_dyn_smem(reinterpret_cast<const void*>(attn_bwd_ds_wide_kernel<true>), kDsWideSmem));
    attn_bwd_ds_wide_kernel<true><<<grid, kThreads, kDsWideSmem, st>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("attention_bwd_dk_wide");
    prm.out0 = (__nv_bfloat16*)dq; prm.cs0 = dqcs;
    prm.accumulate = dq_accumulate ? 1 : 0;
    ATTN_CHECK(tsb_ensure_dyn_smem(reinterpret_cast<const void*>(attn_bwd_ds_wide_kernel<false>), kDsWideSmem));
    attn_bwd_ds_wide_kernel<false><<<grid, kThreads, kDsWideSmem, st>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("attention_bwd_dq_wide");
    return TSB_OK;
}

// the backward after the shape check: q, o, dout, dq, lse and δ have Nq rows per image, k, v, dk and dv Nk
int attention_bwd(const char* who, const void* q, int qcs, const void* k, int kcs, const void* v, int vcs,
                  const void* o, int ocs, const void* dout, int docs, const float* lse, float* delta_ws, void* dq,
                  int dqcs, void* dk, int dkcs, void* dv, int dvcs, int dq_accumulate, int B, int Nq, int Nk, int dim_k,
                  int dim_v, float scale, cudaStream_t st) {
    ATTN_CHECK(check_operand(who, "q", q, qcs, dim_k));
    ATTN_CHECK(check_operand(who, "k", k, kcs, dim_k));
    ATTN_CHECK(check_operand(who, "v", v, vcs, dim_v));
    ATTN_CHECK(check_operand(who, "o", o, ocs, dim_v));
    ATTN_CHECK(check_operand(who, "dout", dout, docs, dim_v));
    ATTN_CHECK(check_operand(who, "dq", dq, dqcs, dim_k));
    ATTN_CHECK(check_operand(who, "dk", dk, dkcs, dim_k));
    ATTN_CHECK(check_operand(who, "dv", dv, dvcs, dim_v));
    TSB_REQUIRE(lse != nullptr && delta_ws != nullptr, "%s: null lse or delta_ws", who);
    AttnParams prm;
    memset(&prm, 0, sizeof(prm));
    ATTN_CHECK(encode_rows(&prm.a, q, qcs, B, Nq, dim_k));
    ATTN_CHECK(encode_rows(&prm.b, k, kcs, B, Nk, dim_k));
    ATTN_CHECK(encode_rows(&prm.c, v, vcs, B, Nk, dim_v));
    ATTN_CHECK(encode_rows(&prm.d, dout, docs, B, Nq, dim_v));
    prm.lse = const_cast<float*>(lse); prm.delta = delta_ws;
    prm.Nq = Nq; prm.Nk = Nk; prm.c2 = scale * kLog2e; prm.scale = scale;
    if (dim_k == kNarrow)
        return attention_bwd_wide(prm, o, ocs, dout, docs, delta_ws, dq, dqcs, dk, dkcs, dv, dvcs, dq_accumulate, B, Nq,
                                  st);
    const int rows = B * Nq;
    attn_delta_kernel<<<tsb_grid_for(rows, 8, 8), 256, 0, st>>>((const __nv_bfloat16*)o, ocs, (const __nv_bfloat16*)dout,
                                                                docs, delta_ws, rows);
    TSB_CUDA_CHECK_LAUNCH("attention_delta");
    // key pass first: with dq == dk and dq_accumulate the query pass then adds dQ onto the finished dK
    prm.out0 = (__nv_bfloat16*)dk; prm.cs0 = dkcs;
    prm.out1 = (__nv_bfloat16*)dv; prm.cs1 = dvcs;
    ATTN_CHECK(tsb_ensure_dyn_smem(reinterpret_cast<const void*>(attn_bwd_kv_kernel), kKvSmem));
    attn_bwd_kv_kernel<<<dim3((Nk + 63) / 64, B), kThreads, kKvSmem, st>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("attention_bwd_kv");
    prm.out0 = (__nv_bfloat16*)dq; prm.cs0 = dqcs;
    prm.out1 = nullptr; prm.cs1 = 0;
    prm.accumulate = dq_accumulate ? 1 : 0;
    ATTN_CHECK(tsb_ensure_dyn_smem(reinterpret_cast<const void*>(attn_bwd_q_kernel), kQSmem));
    attn_bwd_q_kernel<<<dim3((Nq + 63) / 64, B), kThreads, kQSmem, st>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("attention_bwd_q");
    return TSB_OK;
}

}  // namespace

extern "C" int tsb_attention_fwd(const void* q, int qcs, const void* k, int kcs, const void* v, int vcs, void* o, int ocs,
                                 float* lse, int B, int N, int dim_k, int dim_v, float scale, tsb_stream_t stream) {
    const char* who = "tsb_attention_fwd";
    ATTN_CHECK(check_shape(who, B, N, dim_k, dim_v, scale));
    return attention_fwd(who, q, qcs, k, kcs, v, vcs, o, ocs, lse, B, N, N, dim_k, dim_v, scale, (cudaStream_t)stream);
}

extern "C" int tsb_attention_bwd(const void* q, int qcs, const void* k, int kcs, const void* v, int vcs, const void* o,
                                 int ocs, const void* dout, int docs, const float* lse, float* delta_ws, void* dq, int dqcs,
                                 void* dk, int dkcs, void* dv, int dvcs, int dq_accumulate, int B, int N, int dim_k,
                                 int dim_v, float scale, tsb_stream_t stream) {
    const char* who = "tsb_attention_bwd";
    ATTN_CHECK(check_shape(who, B, N, dim_k, dim_v, scale));
    return attention_bwd(who, q, qcs, k, kcs, v, vcs, o, ocs, dout, docs, lse, delta_ws, dq, dqcs, dk, dkcs, dv, dvcs,
                         dq_accumulate, B, N, N, dim_k, dim_v, scale, (cudaStream_t)stream);
}

extern "C" int tsb_cross_attention_fwd(const void* q, int qcs, const void* k, int kcs, const void* v, int vcs, void* o,
                                       int ocs, float* lse, int B, int Nq, int Nk, int dim_k, int dim_v, float scale,
                                       tsb_stream_t stream) {
    const char* who = "tsb_cross_attention_fwd";
    ATTN_CHECK(check_cross_shape(who, B, Nq, Nk, dim_k, dim_v, scale));
    return attention_fwd(who, q, qcs, k, kcs, v, vcs, o, ocs, lse, B, Nq, Nk, dim_k, dim_v, scale, (cudaStream_t)stream);
}

extern "C" int tsb_cross_attention_bwd(const void* q, int qcs, const void* k, int kcs, const void* v, int vcs,
                                       const void* o, int ocs, const void* dout, int docs, const float* lse,
                                       float* delta_ws, void* dq, int dqcs, void* dk, int dkcs, void* dv, int dvcs, int B,
                                       int Nq, int Nk, int dim_k, int dim_v, float scale, tsb_stream_t stream) {
    const char* who = "tsb_cross_attention_bwd";
    ATTN_CHECK(check_cross_shape(who, B, Nq, Nk, dim_k, dim_v, scale));
    return attention_bwd(who, q, qcs, k, kcs, v, vcs, o, ocs, dout, docs, lse, delta_ws, dq, dqcs, dk, dkcs, dv, dvcs, 0,
                         B, Nq, Nk, dim_k, dim_v, scale, (cudaStream_t)stream);
}
