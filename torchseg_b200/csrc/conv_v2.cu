// Persistent implicit-GEMM convolution (fprop / dgrad / stem) on Hopper wgmma (sm_90a).
//
//   * persistent CTAs (one per SM) striding over output tiles of one N-tile → prologue (barriers, descriptor prefetch)
//     paid once, BN statistics accumulated in registers across all tiles of the CTA;
//   * the B operand (packed weights of this N-tile) stays RESIDENT in shared memory when it fits (C=64 layers,
//     1x1 convs, stems) instead of being re-fetched from L2 for every tile;
//   * ROW tiles (TH = 1, TW = 128): the horizontal taps of one filter row share ONE TMA box of TW+span pixels; the
//     taps are addressed by shifting the wgmma descriptor start by whole 128-byte rows, cutting the L2→SM activation
//     traffic of a 3x3 layer 3x.
//   * outputs of <= 64 columns (BN = 64) put the pixels on the wgmma N side: D^T[64 co, px] = W · X^T, one
//     m64n128k16 per warpgroup per k16 step on its own 128-pixel m-tile, both warpgroups reading one weight tile. Per
//     128 clk of MMA a CTA reads 2 x (2 KB + 4 KB) of shared-memory operands, as the BN = 128 tile does, instead of the
//     2 x (2 KB + 2 KB) per 64 clk that saturate the shared-memory port with a 128-pixel x 64-channel tile.
// Warp roles: warps 0-7 = two consumer warpgroups (wgmma into register accumulators; BN = 128: rows 0-63 / 64-127 of
// one 128-pixel tile, epilogue straight from the fragments; BN = 64: one 128-pixel tile each, epilogue transposed to
// pixel-major rows through shared memory), warp 8 = TMA producer.
#include "conv_common.cuh"
#include "conv_v2.cuh"
#include "sm90_ptx.cuh"

using namespace sm90;
using namespace convhost;

namespace {

constexpr int kConsumers = 2;                          // warpgroups
constexpr int kThreads = kConsumers * 128 + 32;        // + one producer warp
constexpr int kMaxStages = 8;
constexpr int kAStageBytes = 17 * 1024;  // (128 + 8) pixel rows x 128 B, rounded up to a 1024-byte multiple

struct TapGroup {
    int dh, dw0, map, ntaps;
    int row_off[3];  // pixel-row offset of each tap inside the group's box
    int bk[3];       // K offset of each tap in B (streamed mode)
    int tap_idx[3];  // global tap index (resident mode)
};

struct alignas(64) V2Params {
    CUtensorMap mapA[4];
    CUtensorMap mapB;
    TapGroup groups[kMaxTaps];
    int a_bytes[4];  // TMA bytes of one A box per map
    int ngroups, ntaps_total, kchunks;
    int tiles_w, tiles_h, m_tiles;
    int tw_shift, TW, TH;
    int P, Q;
    long long out_n_stride, out_p_stride, out_q_stride, out_base;
    int k_real, k_store, out_f32, accumulate;
    int relu;      // inference epilogue: y = max(acc + bias (+ res), 0)
    const void* res;   // optional bf16 residual with the OUTPUT's addressing (same strides / base), added before the ReLU
    const float* bias;
    float* sum;
    float* sumsq;
    float* part;   // [gridDim.x][2][k_real] per-CTA statistics, summed in CTA order by tsb_det_reduce
    void* out;
    // shared-memory plan
    int nstages, stage_bytes, res_bytes;
};

// BN = 64 epilogue: each consumer warp turns its 16 channels x 16 pixels of the transposed fragment into pixel-major
// rows through a [16 px][kStgStride] fp32 buffer of its own. Stride 20 keeps the fragment writes (8 channels x 4 pixel
// pairs per instruction) and the float4 reads (16 pixels x 2 channel halves) free of bank conflicts.
constexpr int kStgStride = 20;
constexpr int kStgWarpBytes = 16 * kStgStride * 4;

template <int BN, bool RES>
__global__ void __launch_bounds__(kThreads, 1) igemm_v2_kernel(const __grid_constant__ V2Params p) {
    // BN = 64: D^T[64 out-ch, px] = W[64, k] · X[px, k]^T. The weight tile is the wgmma A operand, shared by both
    // warpgroups, and each warpgroup takes its own 128-pixel m-tile as B (m64n128k16): a CTA work unit is a pair of
    // m-tiles. BN = 128: D[px, 128 out-ch] = X · W^T, one m-tile per unit, rows 0-63 / 64-127 per warpgroup.
    // CTA b takes the m-tiles b, b + G, b + 2G, ... (G = gridDim.x) in that order, kTiles per unit, at either BN.
    constexpr bool kPixN = (BN == 64);
    constexpr int kTiles = kPixN ? 2 : 1;            // m-tiles per work unit = activation boxes per stage
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* res_b = smem;                       // resident weights (RES)
    uint8_t* stages = smem + p.res_bytes;        // ring of A (+B) stages
    uint8_t* tail = stages + p.nstages * p.stage_bytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);
    uint64_t* b_ready = full_bar + 2 * kMaxStages;
    float* s_stage = reinterpret_cast<float*>(tail + 256);  // BN = 64: [consumer warp][16 px][kStgStride]
    // BN = 64 with statistics: the rounded outputs of a unit, [tile][128 px][64 ch] bf16, 16-byte chunks of a pixel row
    // swizzled by px & 7. The per-warp statistics slots [consumer warp][2*BN] share the space: they are written after
    // the last unit.
    uint8_t* s_out = tail + 256 + (kPixN ? kConsumers * 4 * kStgWarpBytes : 0);
    float* s_stats = reinterpret_cast<float*>(s_out);
    StageRing ring(full_bar, full_bar + kMaxStages, p.nstages);

    const int warp = warp_uniform_idx(), lane = threadIdx.x & 31;
    const int n0 = blockIdx.y * BN;
    const int my_tiles = (p.m_tiles > (int)blockIdx.x) ? (p.m_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const int my_units = (my_tiles + kTiles - 1) / kTiles;
    constexpr int kBTile = BN * 128;
    constexpr int kWOff = kTiles * kAStageBytes;     // streamed weights follow the activation boxes of a stage
    constexpr int kProducer = kConsumers * 4;

    if (warp == kProducer && lane == 0) {
        tma_prefetch_desc(&p.mapB);
        tma_prefetch_desc(&p.mapA[0]);
        ring.init(kConsumers * 4);
        mbar_init(b_ready, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == kProducer) {
        if (lane == 0 && my_units > 0) {
            if (RES) {  // weights of this N-tile: loaded once per CTA
                mbar_arrive_expect_tx(b_ready, (uint32_t)(p.ntaps_total * p.kchunks * kBTile));
                for (int g = 0; g < p.ngroups; ++g)
                    for (int t = 0; t < p.groups[g].ntaps; ++t)
                        for (int kc = 0; kc < p.kchunks; ++kc)
                            tma_load_2d(res_b + (p.groups[g].tap_idx[t] * p.kchunks + kc) * kBTile, &p.mapB, b_ready,
                                        p.groups[g].bk[t] + kc * 64, n0);
            }
            for (int i = 0; i < my_units; ++i) {
                // the last unit of an odd tile count has one box: the second warpgroup's slot is left as it was and its
                // results are not stored
                const int nbox = min(kTiles, my_tiles - i * kTiles);
                int q0[kTiles], p0[kTiles], n_img[kTiles];
#pragma unroll
                for (int b = 0; b < kTiles; ++b) {
                    const int tile = blockIdx.x + (i * kTiles + b) * gridDim.x;
                    q0[b] = (tile % p.tiles_w) * p.TW;
                    p0[b] = ((tile / p.tiles_w) % p.tiles_h) * p.TH;
                    n_img[b] = tile / (p.tiles_w * p.tiles_h);
                }
                for (int g = 0; g < p.ngroups; ++g) {
                    const int gmap = p.groups[g].map, ntaps = p.groups[g].ntaps;
                    const uint32_t bytes = (uint32_t)(nbox * p.a_bytes[gmap]) + (RES ? 0u : (uint32_t)(ntaps * kBTile));
                    for (int kc = 0; kc < p.kchunks; ++kc) {
                        ring.acquire();
                        uint8_t* a_s = stages + ring.slot * p.stage_bytes;
                        mbar_arrive_expect_tx(ring.full_bar(), bytes);
#pragma unroll
                        for (int b = 0; b < kTiles; ++b)
                            if (b < nbox)
                                tma_load_4d(a_s + b * kAStageBytes, &p.mapA[gmap], ring.full_bar(), kc * 64,
                                            q0[b] + p.groups[g].dw0, p0[b] + p.groups[g].dh, n_img[b]);
                        if (!RES) {
                            for (int t = 0; t < ntaps; ++t)
                                tma_load_2d(a_s + kWOff + t * kBTile, &p.mapB, ring.full_bar(), p.groups[g].bk[t] + kc * 64, n0);
                        }
                        ring.advance();
                    }
                }
            }
        }
    } else {
        const int c = warp >> 2, wq = warp & 3;
        const bool do_stats = (p.sum != nullptr);
        const uint64_t desc_hi = desc_hi_sw128(16, 1024);   // K-major, 8-row groups 1024 B apart (both operands)
        const uint32_t stages_lo = smem_u32(stages) >> 4;
        const uint32_t res_lo = smem_u32(res_b) >> 4;
        // this warpgroup's activation rows in a stage: its own box (BN = 64) or its 64-pixel half of the box (BN = 128)
        const uint32_t x_off = (uint32_t)c * (kPixN ? (uint32_t)(kAStageBytes >> 4) : 512u);
        // running column sums over all tiles of the CTA (columns 8j + cq + e) of thread fragment rows m0 and m0 + 8 of
        // every tile, in tile order; at BN = 64 read back from the unit's rounded outputs in shared memory, so that both
        // tile widths sum every channel in the same order
        const int m0 = c * 64 + wq * 16 + (lane >> 2);
        const int cq = 2 * (lane & 3);                 // first of the thread's two columns in every 8-column group
        float run1[BN / 4], run2[BN / 4];
#pragma unroll
        for (int q = 0; q < BN / 4; ++q) { run1[q] = 0.f; run2[q] = 0.f; }
        if (RES && my_units > 0) mbar_wait(b_ready, 0);
        for (int i = 0; i < my_units; ++i) {   // the ring's slot and phase run on across units; each unit drains
            float acc[64];
#pragma unroll
            for (int q = 0; q < 64; ++q) acc[q] = 0.f;
            fence_operands(acc);
            for (int g = 0; g < p.ngroups; ++g) {
                const int ntaps = p.groups[g].ntaps;
                for (int kc = 0; kc < p.kchunks; ++kc) {
                    ring.wait_full();
                    const uint32_t st_lo = stages_lo + (uint32_t)(ring.slot * p.stage_bytes >> 4);
                    // a group has at most 3 taps: unrolled by 2, the issue code holds 12 HGMMA (by default ptxas unrolls
                    // the streamed-weights variant by 4)
#pragma unroll 2
                    for (int t = 0; t < ntaps; ++t) {
                        const uint32_t x_lo = st_lo + x_off + (uint32_t)p.groups[g].row_off[t] * 8u;
                        const uint32_t w_lo = RES ? res_lo + (uint32_t)((p.groups[g].tap_idx[t] * p.kchunks + kc) * kBTile >> 4)
                                                  : st_lo + (uint32_t)((kWOff + t * kBTile) >> 4);
#pragma unroll
                        for (int k = 0; k < 4; ++k) {  // 16 bf16 = 32 B = 2 descriptor units inside the swizzle atom
                            const uint64_t dx = desc_at(desc_hi, x_lo + 2 * k), dw = desc_at(desc_hi, w_lo + 2 * k);
                            if constexpr (kPixN) wgmma_m64n128<0, 0>(acc, dw, dx, 1u);
                            else wgmma_m64n128<0, 0>(acc, dx, dw, 1u);
                        }
                    }
                    ring.commit_release_prev();
                }
            }
            ring.drain();
            fence_operands(acc);
            if constexpr (kPixN) {
                const int tile = blockIdx.x + (2 * i + c) * gridDim.x;
                const bool tile_ok = 2 * i + c < my_tiles;   // false for the empty half of the last unit
                const int tw_i = tile % p.tiles_w;
                const int th_i = (tile / p.tiles_w) % p.tiles_h;
                const int n_img = tile / (p.tiles_w * p.tiles_h);
                // fragment: acc[4j + 2h + e] = D^T[channel 16 wq + lane/4 + 8h][pixel 8j + 2 (lane % 4) + e]
                const int ch = n0 + 16 * wq + (lane >> 2);
                const bool bias0 = p.bias != nullptr && ch < p.k_real, bias1 = p.bias != nullptr && ch + 8 < p.k_real;
                const float b0 = bias0 ? __ldg(p.bias + ch) : 0.f, b1 = bias1 ? __ldg(p.bias + ch + 8) : 0.f;
                float* stg = s_stage + (threadIdx.x >> 5) * (16 * kStgStride);
                // after the transpose a lane holds one pixel and 8 consecutive channels
                const int px = lane & 15;
                const int col = n0 + 16 * wq + 8 * (lane >> 4);   // multiple of 8, as is k_store: all 8 stored or none
                const float* rd = stg + px * kStgStride + 8 * (lane >> 4);
#pragma unroll
                for (int k = 0; k < 8; ++k) {   // 16 pixels (fragment columns j = 2k, 2k + 1) per step
#pragma unroll
                    for (int jj = 0; jj < 2; ++jj)
#pragma unroll
                        for (int h = 0; h < 2; ++h)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                float a = acc[4 * (2 * k + jj) + 2 * h + e];
                                if (h ? bias1 : bias0) a += h ? b1 : b0;
                                stg[(8 * jj + 2 * (lane & 3) + e) * kStgStride + (lane >> 2) + 8 * h] = a;
                            }
                    __syncwarp();
                    const float4 lo = *reinterpret_cast<const float4*>(rd), hi = *reinterpret_cast<const float4*>(rd + 4);
                    __syncwarp();
                    float v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
                    const int m = 16 * k + px;
                    const int pp = th_i * p.TH + (m >> p.tw_shift), qq = tw_i * p.TW + (m & (p.TW - 1));
                    const bool valid = tile_ok && (pp < p.P) && (qq < p.Q);
                    const bool st = valid && col < p.k_store;
                    const long long off = p.out_base + (long long)n_img * p.out_n_stride + (long long)pp * p.out_p_stride +
                                          (long long)qq * p.out_q_stride + col;
                    if (p.res != nullptr && st) {     // folded-BN inference tail of a residual block: + shortcut
                        float r[8];
                        unpack8(*reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.res) + off), r);
#pragma unroll
                        for (int e = 0; e < 8; ++e) v[e] += r[e];
                    }
                    if (p.relu) {
#pragma unroll
                        for (int e = 0; e < 8; ++e) v[e] = fmaxf(v[e], 0.f);
                    }
                    if (p.out_f32) {
                        if (st) {
                            float4* o = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + off);
                            o[0] = make_float4(v[0], v[1], v[2], v[3]);
                            o[1] = make_float4(v[4], v[5], v[6], v[7]);
                        }
                    } else {
                        uint4* o = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + off);
                        if (p.accumulate && st) {
                            float r[8];
                            unpack8(*o, r);
#pragma unroll
                            for (int e = 0; e < 8; ++e) v[e] += r[e];
                        }
                        // round once to bf16; statistics are taken of the rounded values the next layer will see
                        const uint4 u = pack8(v);
                        if (st) *o = u;
                        if (do_stats)
                            *reinterpret_cast<uint4*>(s_out + (c * 128 + m) * 128 + (((2 * wq + (lane >> 4)) ^ (px & 7)) << 4)) = u;
                    }
                }
                if (do_stats) {
                    // every value the statistics see, in the order of the fragment rows of one 128-pixel tile; (pp, qq)
                    // are launch-grid coordinates (a stride-2 parity class's own sub-grid for the transposed forward), so
                    // only the stores above use the output strides
                    asm volatile("bar.sync 1, %0;" ::"n"(kConsumers * 128) : "memory");
#pragma unroll
                    for (int s = 0; s < 2; ++s) {
                        if (2 * i + s < my_tiles) {
                            const int t2 = blockIdx.x + (2 * i + s) * gridDim.x;
                            const int tw2 = t2 % p.tiles_w, th2 = (t2 / p.tiles_w) % p.tiles_h;
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                const int m = m0 + 8 * h;
                                const int pp = th2 * p.TH + (m >> p.tw_shift), qq = tw2 * p.TW + (m & (p.TW - 1));
                                if (pp < p.P && qq < p.Q) {
                                    const uint8_t* row = s_out + (s * 128 + m) * 128 + 2 * cq;
#pragma unroll
                                    for (int j = 0; j < 8; ++j) {
                                        const uint32_t u = *reinterpret_cast<const uint32_t*>(row + ((j ^ (m & 7)) << 4));
                                        const float v0 = bf16lo(u), v1 = bf16hi(u);
                                        run1[2 * j] += v0; run2[2 * j] = fmaf(v0, v0, run2[2 * j]);
                                        run1[2 * j + 1] += v1; run2[2 * j + 1] = fmaf(v1, v1, run2[2 * j + 1]);
                                    }
                                }
                            }
                        }
                    }
                    asm volatile("bar.sync 1, %0;" ::"n"(kConsumers * 128) : "memory");   // s_out is free again
                }
            } else {
                // warpgroup c owns pixel rows [64c, 64c + 64) of the tile; thread fragment rows m0 and m0 + 8
                const int tile = blockIdx.x + i * gridDim.x;
                const int tw_i = tile % p.tiles_w;
                const int th_i = (tile / p.tiles_w) % p.tiles_h;
                const int n_img = tile / (p.tiles_w * p.tiles_h);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = m0 + 8 * h;
                    const int pp = th_i * p.TH + (m >> p.tw_shift), qq = tw_i * p.TW + (m & (p.TW - 1));
                    const bool valid = (pp < p.P) && (qq < p.Q);
                    const long long pix_off = p.out_base + (long long)n_img * p.out_n_stride + (long long)pp * p.out_p_stride +
                                              (long long)qq * p.out_q_stride;
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j) {
                        const int col = n0 + 8 * j + cq;     // even; k_store is a multiple of 8, so col + 1 is in range too
                        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                        if (p.bias != nullptr) {
                            if (col < p.k_real) v0 += __ldg(p.bias + col);
                            if (col + 1 < p.k_real) v1 += __ldg(p.bias + col + 1);
                        }
                        const bool st = valid && col < p.k_store;
                        if (p.res != nullptr && st) {     // folded-BN inference tail of a residual block: + shortcut
                            const uint32_t u = *reinterpret_cast<const uint32_t*>(reinterpret_cast<const __nv_bfloat16*>(p.res) + pix_off + col);
                            v0 += bf16lo(u);
                            v1 += bf16hi(u);
                        }
                        if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                        if (p.out_f32) {
                            if (st) *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + pix_off + col) = make_float2(v0, v1);
                        } else {
                            uint32_t* o = reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.out) + pix_off + col);
                            if (p.accumulate && st) {
                                const uint32_t u = *o;
                                v0 += bf16lo(u);
                                v1 += bf16hi(u);
                            }
                            // round once to bf16; statistics are taken of the rounded values the next layer will see
                            const uint32_t u = pack_bf16(v0, v1);
                            v0 = bf16lo(u);
                            v1 = bf16hi(u);
                            if (st) *o = u;
                        }
                        if (do_stats && valid) {
                            run1[2 * j] += v0; run2[2 * j] = fmaf(v0, v0, run2[2 * j]);
                            run1[2 * j + 1] += v1; run2[2 * j + 1] = fmaf(v1, v1, run2[2 * j + 1]);
                        }
                    }
                }
            }
        }
        if (do_stats) {
            // lanes with the same lane % 4 hold the same columns: reduce over lane / 4, then across warps in smem
#pragma unroll
            for (int q = 0; q < BN / 4; ++q) {
#pragma unroll
                for (int off = 4; off < 32; off <<= 1) {
                    run1[q] += __shfl_xor_sync(0xffffffffu, run1[q], off);
                    run2[q] += __shfl_xor_sync(0xffffffffu, run2[q], off);
                }
            }
            if (lane < 4) {
                float* sw = s_stats + (threadIdx.x >> 5) * 2 * BN;   // re-derived: keeping `warp` live spills at BN = 128
#pragma unroll
                for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        sw[8 * j + cq + e] = run1[2 * j + e];
                        sw[BN + 8 * j + cq + e] = run2[2 * j + e];
                    }
            }
            asm volatile("bar.sync 1, %0;" ::"n"(kConsumers * 128) : "memory");  // the consumer warpgroups only
            // fixed summation order everywhere (no float atomics): per-warp slots, summed in warp order; the CTA's
            // totals go to its workspace slot and tsb_det_reduce adds the slots in CTA order
            float* part = p.part + (long long)blockIdx.x * 2 * p.k_real;
            for (int i = threadIdx.x; i < BN; i += kConsumers * 128) {
                if (n0 + i < p.k_real) {
                    float t1 = 0.f, t2 = 0.f;
                    for (int w = 0; w < kConsumers * 4; ++w) { t1 += s_stats[w * 2 * BN + i]; t2 += s_stats[w * 2 * BN + BN + i]; }
                    part[n0 + i] = t1;
                    part[p.k_real + n0 + i] = t2;
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// wgrad, row-tile variant: the horizontal taps of one filter row share ONE activation box.
//   dW[co, (s, ci)] += Σ_px dY[px, co] · X[px + s·step, ci]      for the ntaps (<= 3) taps of the group
// A = dYᵀ (MN-major, 2 boxes of 64 out-channels, one per consumer warpgroup), B = ONE box of 64+span pixels x 64
// in-channels (MN-major); tap t reads the same smem rows shifted by t·step pixels, so the activations are loaded once
// for all taps of the row. K = 64 pixels per stage.
// ------------------------------------------------------------------------------------------------
constexpr int kWrStages = 8;
constexpr int kWrABytes = 2 * 64 * 128;   // two 64-channel dY boxes of 64 pixels
constexpr int kWrBBytes = 10 * 1024;      // (64 + 8) pixel rows x 128 B, rounded up
constexpr int kWrStageBytes = kWrABytes + kWrBBytes;
constexpr int kWrSmem = kWrStages * kWrStageBytes + 256 + 1024;

struct WrGroup { int dh, dw0, map, ntaps, step; int tap_idx[3]; };
struct alignas(64) WrParams {
    CUtensorMap mapA;
    CUtensorMap mapB[4];
    WrGroup groups[kMaxTaps];
    int b_bytes[4];
    int ngroups, cchunks;
    int tiles_w, tiles_h, total_tiles, tiles_per_split;
    int TW;
    int K, C;
    long long dw_row_stride;
    float* dw;                // dW-shaped slice per split (workspace), part_stride apart; or dW itself when `add`
    long long part_stride;
    int add;                  // one split: add in place
};

__global__ void __launch_bounds__(kThreads, 1) wgrad_rows_kernel(const __grid_constant__ WrParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kWrStages * kWrStageBytes);
    StageRing ring(full_bar, full_bar + kWrStages, kWrStages);
    const int warp = warp_uniform_idx(), lane = threadIdx.x & 31;
    const int co0 = blockIdx.y * 128;
    const int g = blockIdx.z / p.cchunks, cc = blockIdx.z - g * p.cchunks;
    const WrGroup G = p.groups[g];
    const int t_begin = blockIdx.x * p.tiles_per_split;
    const int t_end = min(p.total_tiles, t_begin + p.tiles_per_split);
    const int total_iters = t_end - t_begin;
    constexpr int kProducer = kConsumers * 4;

    if (warp == kProducer && lane == 0) {
        tma_prefetch_desc(&p.mapA);
        tma_prefetch_desc(&p.mapB[G.map]);
        ring.init(kConsumers * 4);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == kProducer) {
        if (lane == 0) {
            for (int it = 0; it < total_iters; ++it) {
                ring.acquire();
                const int t = t_begin + it;
                const int tw_i = t % p.tiles_w;
                const int row = (t / p.tiles_w) % p.tiles_h;
                const int n_img = t / (p.tiles_w * p.tiles_h);
                const int q0 = tw_i * p.TW;
                uint8_t* a_s = smem + ring.slot * kWrStageBytes;
                mbar_arrive_expect_tx(ring.full_bar(), (uint32_t)(kWrABytes + p.b_bytes[G.map]));
                tma_load_4d(a_s, &p.mapA, ring.full_bar(), co0, q0, row, n_img);
                tma_load_4d(a_s + 64 * 128, &p.mapA, ring.full_bar(), co0 + 64, q0, row, n_img);  // OOB → zeros
                tma_load_4d(a_s + kWrABytes, &p.mapB[G.map], ring.full_bar(), cc * 64, q0 + G.dw0, row + G.dh, n_img);
                ring.advance();
            }
        }
    } else {   // every split stores its (possibly all-zero) tile: the slices are summed in split order afterwards
        const int c = warp >> 2, wq = warp & 3;
        const uint64_t desc_hi = desc_hi_sw128(64 * 128, 1024);   // MN-major: 8-pixel groups 1024 B apart
        const uint32_t base_lo = smem_u32(smem) >> 4;
        float acc[3][32];
#pragma unroll
        for (int t = 0; t < 3; ++t)
#pragma unroll
            for (int q = 0; q < 32; ++q) acc[t][q] = 0.f;
#pragma unroll
        for (int t = 0; t < 3; ++t) fence_operands(acc[t]);
        for (int it = 0; it < total_iters; ++it) {
            ring.wait_full();
            const uint32_t a_lo = base_lo + (uint32_t)(ring.slot * (kWrStageBytes >> 4)) + (uint32_t)c * 512u;
            const uint32_t b_lo = base_lo + (uint32_t)(ring.slot * (kWrStageBytes >> 4)) + (kWrABytes >> 4);
#pragma unroll
            for (int t = 0; t < 3; ++t) {
                if (t < G.ntaps) {
#pragma unroll
                    for (int k = 0; k < 4; ++k)   // one MMA consumes 16 pixels = 2048 B = 128 descriptor units
                        wgmma_m64n64<1, 1>(acc[t], desc_at(desc_hi, a_lo + 128 * k),
                                           desc_at(desc_hi, b_lo + (uint32_t)(t * G.step * 8) + 128 * k), 1u);
                }
            }
            ring.commit_release_prev();
        }
        ring.drain();
#pragma unroll
        for (int t = 0; t < 3; ++t) fence_operands(acc[t]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int co = co0 + c * 64 + wq * 16 + (lane >> 2) + 8 * h;
            if (co >= p.K) continue;
#pragma unroll
            for (int t = 0; t < 3; ++t) {
                if (t >= G.ntaps) continue;
                float* dst = p.dw + blockIdx.x * p.part_stride + (long long)co * p.dw_row_stride + (long long)G.tap_idx[t] * p.C + cc * 64 +
                             2 * (lane & 3);
#pragma unroll
                for (int j = 0; j < 8; ++j) put_f2(dst + 8 * j, acc[t][4 * j + 2 * h], acc[t][4 * j + 2 * h + 1], p.add);
            }
        }
    }
}

template <int BN, bool RES>
int launch_v2(const V2Params& prm, int grid_x, int n_tiles, size_t smem, cudaStream_t st) {
    { int rc_ = tsb_ensure_dyn_smem(reinterpret_cast<const void*>(igemm_v2_kernel<BN, RES>), smem); if (rc_) return rc_; }
    igemm_v2_kernel<BN, RES><<<dim3(grid_x, n_tiles), kThreads, smem, st>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("igemm_v2");
    return TSB_OK;
}

}  // namespace

namespace convv2 {

int launch(const Desc& d, cudaStream_t st, int* stat_slots) {
    V2Params prm;
    memset(&prm, 0, sizeof(prm));
    const int BN = (d.ncols <= 64) ? 64 : 128;
    const int n_tiles = (d.ncols + BN - 1) / BN;
    // ---- spatial tiling: row tiles when the output rows are long enough
    int TW, TH;
    const bool rows = !d.flat && d.Ql >= 96;
    if (d.flat || rows) { TW = 128; TH = 1; }
    else pick_tile(d.Ql, 128, &TW, &TH);
    // ---- group the taps: same (map, dh) → one box, taps addressed by a row offset (row tiles only)
    int span_map[4] = {0, 0, 0, 0};
    int ng = 0;
    for (int t = 0; t < d.ntaps; ++t) {
        const Tap& T = d.taps[t];
        int g = -1;
        if (rows) {
            for (int k = 0; k < ng; ++k)
                if (prm.groups[k].map == T.map && prm.groups[k].dh == T.dh && prm.groups[k].ntaps < 3 &&
                    abs(T.dw - prm.groups[k].dw0) <= 8) { g = k; break; }
        }
        if (g < 0) {
            g = ng++;
            prm.groups[g].map = T.map; prm.groups[g].dh = T.dh; prm.groups[g].dw0 = T.dw; prm.groups[g].ntaps = 0;
        }
        TapGroup& G = prm.groups[g];
        if (T.dw < G.dw0) {  // keep dw0 = min dw of the group
            int shift = G.dw0 - T.dw;
            for (int k = 0; k < G.ntaps; ++k) G.row_off[k] += shift;
            G.dw0 = T.dw;
        }
        G.row_off[G.ntaps] = T.dw - G.dw0;
        G.bk[G.ntaps] = T.bk;
        G.tap_idx[G.ntaps] = t;
        G.ntaps++;
    }
    for (int g = 0; g < ng; ++g)
        for (int k = 0; k < prm.groups[g].ntaps; ++k)
            if (prm.groups[g].row_off[k] > span_map[prm.groups[g].map]) span_map[prm.groups[g].map] = prm.groups[g].row_off[k];
    int box_w[4];   // A box width of each map: TW + span of the map
    for (int m = 0; m < 4; ++m) {
        TSB_REQUIRE(span_map[m] <= 8, "conv_v2: tap span too large");
        box_w[m] = TW + span_map[m];
        prm.a_bytes[m] = box_w[m] * TH * 128;
    }
    prm.ngroups = ng;
    prm.ntaps_total = d.ntaps;
    prm.kchunks = d.kchunks;
    int rc = d.stem ? encode_stem_map(&prm.mapA[0], d.act, d.aN, d.aH, d.aW, box_w[0], TH)
                    : encode_act_maps(prm.mapA, d.act, d.aN, d.aH, d.aW, d.aC, d.acs, d.act_stride, box_w, TH);
    if (rc) return rc;
    rc = encode_2d(&prm.mapB, d.w, (uint64_t)d.w_k, (uint64_t)d.w_rows, (uint64_t)d.w_k * 2, 64, BN);
    if (rc) return rc;
    // ---- geometry / epilogue
    prm.tiles_w = (d.Ql + TW - 1) / TW;
    prm.tiles_h = (d.Pl + TH - 1) / TH;
    prm.m_tiles = prm.tiles_w * prm.tiles_h * d.Nl;
    prm.TW = TW; prm.TH = TH; prm.tw_shift = ilog2(TW);
    prm.P = d.Pl; prm.Q = d.Ql;
    prm.out_n_stride = d.out_n_stride; prm.out_p_stride = d.out_p_stride; prm.out_q_stride = d.out_q_stride;
    prm.out_base = d.out_base;
    prm.k_real = d.k_real; prm.k_store = d.k_store; prm.out_f32 = d.out_f32; prm.accumulate = d.accumulate;
    prm.bias = d.bias; prm.sum = d.sum; prm.sumsq = d.sumsq; prm.out = d.out;
    prm.relu = d.relu; prm.res = d.res;
    // ---- shared-memory plan: resident weights, then the stage ring (one activation box per m-tile of a work unit,
    // + the streamed weight tiles), then barriers and the epilogue space: BN = 128, the statistics slots; BN = 64, the
    // transpose buffers and, with statistics, the unit's rounded outputs (which the statistics slots reuse)
    const int kBTile = BN * 128;
    const int unit_tiles = (BN == 64) ? 2 : 1;
    const long long res_need = (long long)d.ntaps * d.kchunks * kBTile;
    const bool resident = res_need <= 112 * 1024 && prm.m_tiles > 0;
    const int tail = 256 + (BN == 64 ? kConsumers * 4 * kStgWarpBytes + (d.sum ? 2 * 128 * 64 * 2 : 0)
                                     : kConsumers * 4 * 2 * BN * 4);
    const int budget = 227 * 1024 - 1024 /*align*/ - tail;
    int max_group_taps = 1;
    for (int g = 0; g < ng; ++g) if (prm.groups[g].ntaps > max_group_taps) max_group_taps = prm.groups[g].ntaps;
    prm.res_bytes = resident ? (int)res_need : 0;
    prm.stage_bytes = unit_tiles * kAStageBytes + (resident ? 0 : max_group_taps * kBTile);
    int ns = (budget - prm.res_bytes) / prm.stage_bytes;
    if (ns > kMaxStages) ns = kMaxStages;
    TSB_REQUIRE(ns >= 2, "conv_v2: shared-memory plan needs at least 2 stages");
    prm.nstages = ns;
    const size_t smem = 1024 + (size_t)prm.res_bytes + (size_t)ns * prm.stage_bytes + tail;
#ifdef TSB_DEBUG_CONV_PLAN
    fprintf(stderr, "conv_v2 plan: BN %d %s, %d taps x %d K-chunks, resident %d B, %d stages x %d B, tail %d B, smem %zu B\n",
            BN, resident ? "resident" : "streamed", d.ntaps, d.kchunks, prm.res_bytes, ns, prm.stage_bytes, tail, smem);
#endif
    if (BN == 64) {   // the pixel-major epilogue stores 8 channels as one 16-byte (bf16) or two 16-byte (fp32) vectors
        const int vec = d.out_f32 ? 4 : 8;
        TSB_REQUIRE(tsb_aligned16(d.out) && (d.res == nullptr || tsb_aligned16(d.res)) && d.out_base % vec == 0 &&
                    d.out_n_stride % vec == 0 && d.out_p_stride % vec == 0 && d.out_q_stride % vec == 0,
                    "conv_v2: the output must be 16-byte aligned at every pixel");
    }
    int grid_x = tsb_num_sms() / n_tiles;
    if (grid_x < 1) grid_x = 1;
    if (grid_x > prm.m_tiles) grid_x = prm.m_tiles;
    if (grid_x < 1) grid_x = 1;
    if (d.sum != nullptr) {
        TSB_REQUIRE(d.ws && (long long)grid_x * 2 * d.k_real <= d.ws_floats, "conv: statistics workspace needs %lld floats",
                    (long long)grid_x * 2 * d.k_real);
        prm.part = d.ws;
    }
    int rc2 = (BN == 64) ? (resident ? launch_v2<64, true>(prm, grid_x, n_tiles, smem, st) : launch_v2<64, false>(prm, grid_x, n_tiles, smem, st))
                         : (resident ? launch_v2<128, true>(prm, grid_x, n_tiles, smem, st) : launch_v2<128, false>(prm, grid_x, n_tiles, smem, st));
    if (rc2 || d.sum == nullptr) return rc2;
    if (stat_slots != nullptr) { *stat_slots = grid_x; return TSB_OK; }
    rc2 = tsb_det_reduce(d.sum, prm.part, grid_x, d.k_real, 2LL * d.k_real, st);
    if (rc2) return rc2;
    // the sumsq slots follow the sum slots of the same CTA: a stride of 2·k_real between CTAs
    return tsb_det_reduce(d.sumsq, prm.part + d.k_real, grid_x, d.k_real, 2LL * d.k_real, st);
}


// row-tile wgrad: returns TSB_ERR_UNSUPPORTED when the shape is not eligible (caller falls back to the patch kernel)
int launch_wgrad_rows(const WgradDesc& d, cudaStream_t st) {
    if (d.Q < 64) return TSB_ERR_UNSUPPORTED;
    WrParams prm;
    memset(&prm, 0, sizeof(prm));
    const int TW = 64;
    int span_map[4] = {0, 0, 0, 0};
    int ng = 0;
    for (int t = 0; t < d.ntaps; ++t) {
        const Tap& T = d.taps[t];
        int g = -1;
        for (int k = 0; k < ng; ++k) {
            WrGroup& G = prm.groups[k];
            if (G.map != T.map || G.dh != T.dh || G.ntaps >= 3) continue;
            // taps arrive in increasing dw; keep a uniform step inside the group
            int last = G.dw0 + (G.ntaps - 1) * G.step;
            int step = T.dw - last;
            if (step <= 0 || step > 4) continue;
            if (G.ntaps == 1 || step == G.step) { g = k; if (G.ntaps == 1) G.step = step; break; }
        }
        if (g < 0) {
            g = ng++;
            prm.groups[g].map = T.map; prm.groups[g].dh = T.dh; prm.groups[g].dw0 = T.dw; prm.groups[g].ntaps = 0;
            prm.groups[g].step = 1;
        }
        WrGroup& G = prm.groups[g];
        G.tap_idx[G.ntaps++] = t;
    }
    for (int g = 0; g < ng; ++g) {
        int span = (prm.groups[g].ntaps - 1) * prm.groups[g].step;
        if (span > 8) return TSB_ERR_UNSUPPORTED;
        if (span > span_map[prm.groups[g].map]) span_map[prm.groups[g].map] = span;
    }
    prm.ngroups = ng;
    prm.cchunks = d.C / 64;
    int box_w[4];
    for (int m = 0; m < 4; ++m) {
        box_w[m] = TW + span_map[m];
        prm.b_bytes[m] = box_w[m] * 128;
    }
    int rc = encode_4d(&prm.mapA, d.dy, d.K, d.Q, d.P, d.N, (uint64_t)d.dycs * 2, (uint64_t)d.Q * d.dycs * 2,
                       (uint64_t)d.P * d.Q * d.dycs * 2, 64, TW, 1, 1);
    if (rc) return rc;
    rc = encode_act_maps(prm.mapB, d.x, d.N, d.H, d.W, d.C, d.xcs, d.stride, box_w, 1);
    if (rc) return rc;
    prm.TW = TW;
    prm.tiles_w = (d.Q + TW - 1) / TW;
    prm.tiles_h = d.P;
    prm.total_tiles = prm.tiles_w * prm.tiles_h * d.N;
    prm.K = d.K; prm.C = d.C; prm.dw_row_stride = d.dw_row_stride;
    const int co_tiles = (d.K + 127) / 128;
    const int zdim = ng * prm.cchunks;
    // about two waves of CTAs, at least 16 tiles per split
    const SplitPlan sp = plan_splits(wave_splits(zdim * co_tiles, prm.total_tiles, 16), prm.total_tiles,
                                     (long long)d.K * d.dw_row_stride, d.dw, d.ws, d.ws_floats);
    prm.tiles_per_split = sp.tiles_per_split;
    prm.add = sp.add; prm.dw = sp.dst; prm.part_stride = sp.part_stride;
    { int rc_ = tsb_ensure_dyn_smem(reinterpret_cast<const void*>(wgrad_rows_kernel), kWrSmem); if (rc_) return rc_; }
    wgrad_rows_kernel<<<dim3(sp.splits, co_tiles, zdim), kThreads, kWrSmem, st>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("wgrad_rows");
    return finish_splits(sp, d.dw, st);
}

}  // namespace convv2
