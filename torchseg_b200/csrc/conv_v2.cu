// Persistent implicit-GEMM convolution (fprop / dgrad / stem) on Hopper wgmma (sm_90a).
//
//   * persistent CTAs (one per SM) striding over output tiles of one N-tile → prologue (barriers, descriptor prefetch)
//     paid once, BN statistics accumulated in registers across all tiles of the CTA;
//   * the B operand (packed weights of this N-tile) stays RESIDENT in shared memory when it fits (C=64 layers,
//     1x1 convs, stems) instead of being re-fetched from L2 for every tile;
//   * ROW tiles (TH = 1, TW = 128): the horizontal taps of one filter row share ONE TMA box of TW+span pixels; the
//     taps are addressed by shifting the wgmma descriptor start by whole 128-byte rows, cutting the L2→SM activation
//     traffic of a 3x3 layer 3x.
// Warp roles: warps 0-7 = two consumer warpgroups (rows 0-63 / 64-127 of the 128-pixel tile: wgmma into register
// accumulators, then the epilogue straight from the fragments), warp 8 = TMA producer.
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
    int nstages, stage_bytes, res_bytes, use_base_offset;
};

template <int BN>
__device__ __forceinline__ void wgmma_kmajor(float (&d)[BN / 2], uint64_t da, uint64_t db) {
    if constexpr (BN == 64) wgmma_m64n64<0, 0>(d, da, db, 1u);
    else wgmma_m64n128<0, 0>(d, da, db, 1u);
}

template <int BN, bool RES>
__global__ void __launch_bounds__(kThreads, 1) igemm_v2_kernel(const __grid_constant__ V2Params p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* res_b = smem;                       // resident weights (RES)
    uint8_t* stages = smem + p.res_bytes;        // ring of A (+B) stages
    uint8_t* tail = stages + p.nstages * p.stage_bytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);
    uint64_t* empty_bar = full_bar + kMaxStages;
    uint64_t* b_ready = empty_bar + kMaxStages;
    float* s_stats = reinterpret_cast<float*>(tail + 256);  // [consumer warp][2*BN]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n0 = blockIdx.y * BN;
    const int my_tiles = (p.m_tiles > (int)blockIdx.x) ? (p.m_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    constexpr int kBTile = BN * 128;
    constexpr int kProducer = kConsumers * 4;

    if (warp == kProducer && lane == 0) {
        tma_prefetch_desc(&p.mapB);
        tma_prefetch_desc(&p.mapA[0]);
        for (int s = 0; s < p.nstages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumers * 4); }
        mbar_init(b_ready, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == kProducer) {
        if (lane == 0 && my_tiles > 0) {
            if (RES) {  // weights of this N-tile: loaded once per CTA
                mbar_arrive_expect_tx(b_ready, (uint32_t)(p.ntaps_total * p.kchunks * kBTile));
                for (int g = 0; g < p.ngroups; ++g)
                    for (int t = 0; t < p.groups[g].ntaps; ++t)
                        for (int kc = 0; kc < p.kchunks; ++kc)
                            tma_load_2d(res_b + (p.groups[g].tap_idx[t] * p.kchunks + kc) * kBTile, &p.mapB, b_ready,
                                        p.groups[g].bk[t] + kc * 64, n0);
            }
            int sl = 0;
            uint32_t ph = 0;
            for (int i = 0; i < my_tiles; ++i) {
                const int tile = blockIdx.x + i * gridDim.x;
                const int tw_i = tile % p.tiles_w;
                const int th_i = (tile / p.tiles_w) % p.tiles_h;
                const int n_img = tile / (p.tiles_w * p.tiles_h);
                const int q0 = tw_i * p.TW, p0 = th_i * p.TH;
                for (int g = 0; g < p.ngroups; ++g) {
                    const int gmap = p.groups[g].map, ntaps = p.groups[g].ntaps;
                    const int cw = q0 + p.groups[g].dw0, chh = p0 + p.groups[g].dh;
                    const uint32_t bytes = (uint32_t)p.a_bytes[gmap] + (RES ? 0u : (uint32_t)(ntaps * kBTile));
                    for (int kc = 0; kc < p.kchunks; ++kc) {
                        mbar_wait(&empty_bar[sl], ph ^ 1u);
                        uint8_t* a_s = stages + sl * p.stage_bytes;
                        mbar_arrive_expect_tx(&full_bar[sl], bytes);
                        tma_load_4d(a_s, &p.mapA[gmap], &full_bar[sl], kc * 64, cw, chh, n_img);
                        if (!RES) {
                            for (int t = 0; t < ntaps; ++t)
                                tma_load_2d(a_s + kAStageBytes + t * kBTile, &p.mapB, &full_bar[sl], p.groups[g].bk[t] + kc * 64, n0);
                        }
                        if (++sl == p.nstages) { sl = 0; ph ^= 1u; }
                    }
                }
            }
        }
    } else {
        // consumer warpgroup c owns pixel rows [64c, 64c + 64) of every tile; thread fragment rows m0 and m0 + 8
        const int c = warp >> 2, wq = warp & 3;
        const int m0 = c * 64 + wq * 16 + (lane >> 2);
        const int cq = 2 * (lane & 3);                 // first of the thread's two columns in every 8-column group
        const bool do_stats = (p.sum != nullptr);
        const uint64_t desc_hi = desc_hi_sw128(16, 1024);   // K-major, 8-row groups 1024 B apart
        const uint32_t stages_lo = smem_u32(stages) >> 4;
        const uint32_t res_lo = smem_u32(res_b) >> 4;
        float run1[BN / 4], run2[BN / 4];   // running column sums over all tiles of the CTA (columns 8j + cq + e)
#pragma unroll
        for (int q = 0; q < BN / 4; ++q) { run1[q] = 0.f; run2[q] = 0.f; }
        if (RES && my_tiles > 0) mbar_wait(b_ready, 0);
        int sl = 0;
        uint32_t ph = 0;
        for (int i = 0; i < my_tiles; ++i) {
            float acc[BN / 2];
#pragma unroll
            for (int q = 0; q < BN / 2; ++q) acc[q] = 0.f;
            for (int g = 0; g < p.ngroups; ++g) {
                const int ntaps = p.groups[g].ntaps;
                for (int kc = 0; kc < p.kchunks; ++kc) {
                    mbar_wait(&full_bar[sl], ph);
                    fence_operands(acc);
                    wgmma_fence();
                    const uint32_t st_lo = stages_lo + (uint32_t)(sl * p.stage_bytes >> 4);
#pragma unroll
                    for (int t = 0; t < 3; ++t) {
                        if (t < ntaps) {
                            const uint32_t a_lo = st_lo + (uint32_t)c * 512u + (uint32_t)p.groups[g].row_off[t] * 8u;
                            const uint32_t b_lo = RES ? res_lo + (uint32_t)((p.groups[g].tap_idx[t] * p.kchunks + kc) * kBTile >> 4)
                                                      : st_lo + (uint32_t)((kAStageBytes + t * kBTile) >> 4);
#pragma unroll
                            for (int k = 0; k < 4; ++k)   // 16 bf16 = 32 B = 2 descriptor units inside the swizzle atom
                                wgmma_kmajor<BN>(acc, desc_at(desc_hi, a_lo + 2 * k, p.use_base_offset),
                                                 desc_at(desc_hi, b_lo + 2 * k, 0));
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    fence_operands(acc);
                    // wait_group covers only this warp's MMAs: every consumer warp releases the stage
                    if (lane == 0) mbar_arrive(&empty_bar[sl]);
                    if (++sl == p.nstages) { sl = 0; ph ^= 1u; }
                }
            }
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
            // fixed summation order everywhere (no float atomics): per-warp slots, summed in warp order; the CTA's
            // totals go to its workspace slot and tsb_det_reduce adds the slots in CTA order
            if (lane < 4) {
                float* sw = s_stats + warp * 2 * BN;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        sw[8 * j + cq + e] = run1[2 * j + e];
                        sw[BN + 8 * j + cq + e] = run2[2 * j + e];
                    }
            }
            asm volatile("bar.sync 1, %0;" ::"n"(kConsumers * 128) : "memory");  // the consumer warpgroups only
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
    int use_base_offset;
};

__global__ void __launch_bounds__(kThreads, 1) wgrad_rows_kernel(const __grid_constant__ WrParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kWrStages * kWrStageBytes);
    uint64_t* empty_bar = full_bar + kWrStages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
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
        for (int s = 0; s < kWrStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumers * 4); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == kProducer) {
        if (lane == 0) {
            for (int it = 0; it < total_iters; ++it) {
                const int s = it % kWrStages;
                const uint32_t ph = (uint32_t)(it / kWrStages) & 1u;
                mbar_wait(&empty_bar[s], ph ^ 1u);
                const int t = t_begin + it;
                const int tw_i = t % p.tiles_w;
                const int row = (t / p.tiles_w) % p.tiles_h;
                const int n_img = t / (p.tiles_w * p.tiles_h);
                const int q0 = tw_i * p.TW;
                uint8_t* a_s = smem + s * kWrStageBytes;
                mbar_arrive_expect_tx(&full_bar[s], (uint32_t)(kWrABytes + p.b_bytes[G.map]));
                tma_load_4d(a_s, &p.mapA, &full_bar[s], co0, q0, row, n_img);
                tma_load_4d(a_s + 64 * 128, &p.mapA, &full_bar[s], co0 + 64, q0, row, n_img);  // OOB → zeros
                tma_load_4d(a_s + kWrABytes, &p.mapB[G.map], &full_bar[s], cc * 64, q0 + G.dw0, row + G.dh, n_img);
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
        int s = 0;
        uint32_t ph = 0;
        for (int it = 0; it < total_iters; ++it) {
            mbar_wait(&full_bar[s], ph);
#pragma unroll
            for (int t = 0; t < 3; ++t) fence_operands(acc[t]);
            wgmma_fence();
            const uint32_t a_lo = base_lo + (uint32_t)(s * (kWrStageBytes >> 4)) + (uint32_t)c * 512u;
            const uint32_t b_lo = base_lo + (uint32_t)(s * (kWrStageBytes >> 4)) + (kWrABytes >> 4);
#pragma unroll
            for (int t = 0; t < 3; ++t) {
                if (t < G.ntaps) {
#pragma unroll
                    for (int k = 0; k < 4; ++k)   // one MMA consumes 16 pixels = 2048 B = 128 descriptor units
                        wgmma_m64n64<1, 1>(acc[t], desc_at(desc_hi, a_lo + 128 * k, 0),
                                           desc_at(desc_hi, b_lo + (uint32_t)(t * G.step * 8) + 128 * k, p.use_base_offset), 1u);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int t = 0; t < 3; ++t) fence_operands(acc[t]);
            // wait_group covers only this warp's MMAs: every consumer warp releases the stage
            if (lane == 0) mbar_arrive(&empty_bar[s]);
            if (++s == kWrStages) { s = 0; ph ^= 1u; }
        }
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

int g_allow_rows = 1;
int g_allow_resident = 1;

template <int BN, bool RES>
int launch_v2(const V2Params& prm, int grid_x, int n_tiles, size_t smem, cudaStream_t st) {
    { int rc_ = tsb_ensure_dyn_smem(reinterpret_cast<const void*>(igemm_v2_kernel<BN, RES>), smem); if (rc_) return rc_; }
    igemm_v2_kernel<BN, RES><<<dim3(grid_x, n_tiles), kThreads, smem, st>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("igemm_v2");
    return TSB_OK;
}

}  // namespace

extern int g_tsb_ohem_hoist;
extern int g_tsb_ohem_exact;
extern "C" int tsb_debug_set(int key, int value) {
    if (key == 1) convv2::g_use_base_offset = value;
    else if (key == 2) g_allow_rows = value;
    else if (key == 3) g_allow_resident = value;
    else if (key == 5) convv2::g_wgrad_waves = value;
    else if (key == 6) g_tsb_ohem_hoist = value;
    else if (key == 8) convv2::g_allow_taps = value;
    else if (key == 10) g_tsb_ohem_exact = value;
    else return TSB_ERR_ARG;
    return TSB_OK;
}

namespace convv2 {

int g_wgrad_waves = 2;
int g_use_base_offset = 0;  // H100 takes the 128B-swizzle phase from the absolute shared address: row-shifted starts need no base_offset

int launch(const Desc& d, cudaStream_t st) {
    V2Params prm;
    memset(&prm, 0, sizeof(prm));
    const int BN = (d.ncols <= 64) ? 64 : 128;
    const int n_tiles = (d.ncols + BN - 1) / BN;
    // ---- spatial tiling: row tiles when the output rows are long enough
    int TW, TH;
    const bool rows = g_allow_rows && !d.flat && d.Ql >= 96;
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
    for (int m = 0; m < 4; ++m) {
        TSB_REQUIRE(span_map[m] <= 8, "conv_v2: tap span too large");
        prm.a_bytes[m] = (TW + span_map[m]) * TH * 128;
    }
    prm.ngroups = ng;
    prm.ntaps_total = d.ntaps;
    prm.kchunks = d.kchunks;
    // ---- A tensor maps (box width = TW + span of the map)
    const __nv_bfloat16* base = reinterpret_cast<const __nv_bfloat16*>(d.act);
    int rc;
    if (d.stem) {
        const uint64_t row = (uint64_t)(d.aW + 4) * 16 * 2;
        rc = encode_4d(&prm.mapA[0], base, 64, (uint64_t)d.aW, (uint64_t)d.aH, (uint64_t)d.aN, 32, row, row * d.aH, 64, TW + span_map[0], TH, 1);
        if (rc) return rc;
    } else if (d.act_stride == 1) {
        rc = encode_4d(&prm.mapA[0], base, d.aC, d.aW, d.aH, d.aN, (uint64_t)d.acs * 2, (uint64_t)d.aW * d.acs * 2,
                       (uint64_t)d.aH * d.aW * d.acs * 2, 64, TW + span_map[0], TH, 1);
        if (rc) return rc;
    } else {
        for (int ph = 0; ph < 2; ++ph)
            for (int pw = 0; pw < 2; ++pw) {
                int Hh = (d.aH - ph + 1) / 2, Ww = (d.aW - pw + 1) / 2;
                if (Hh <= 0) Hh = 1;
                if (Ww <= 0) Ww = 1;
                rc = encode_4d(&prm.mapA[ph * 2 + pw], base + ((long long)ph * d.aW + pw) * d.acs, d.aC, Ww, Hh, d.aN,
                               (uint64_t)2 * d.acs * 2, (uint64_t)2 * d.aW * d.acs * 2, (uint64_t)d.aH * d.aW * d.acs * 2, 64,
                               TW + span_map[ph * 2 + pw], TH, 1);
                if (rc) return rc;
            }
    }
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
    prm.use_base_offset = g_use_base_offset;
    // ---- shared-memory plan
    const int kBTile = BN * 128;
    const long long res_need = (long long)d.ntaps * d.kchunks * kBTile;
    const bool resident = g_allow_resident && res_need <= 112 * 1024 && prm.m_tiles > 0;
    const int tail = 256 + kConsumers * 4 * 2 * BN * 4;
    const int budget = 227 * 1024 - 1024 /*align*/ - tail;
    int max_group_taps = 1;
    for (int g = 0; g < ng; ++g) if (prm.groups[g].ntaps > max_group_taps) max_group_taps = prm.groups[g].ntaps;
    prm.res_bytes = resident ? (int)res_need : 0;
    prm.stage_bytes = kAStageBytes + (resident ? 0 : max_group_taps * kBTile);
    int ns = (budget - prm.res_bytes) / prm.stage_bytes;
    if (ns > kMaxStages) ns = kMaxStages;
    TSB_REQUIRE(ns >= 2, "conv_v2: shared-memory plan needs at least 2 stages");
    prm.nstages = ns;
    const size_t smem = 1024 + (size_t)prm.res_bytes + (size_t)ns * prm.stage_bytes + tail;
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
    rc2 = tsb_det_reduce(d.sum, prm.part, grid_x, d.k_real, 2LL * d.k_real, st);
    if (rc2) return rc2;
    // the sumsq slots follow the sum slots of the same CTA: a stride of 2·k_real between CTAs
    return tsb_det_reduce(d.sumsq, prm.part + d.k_real, grid_x, d.k_real, 2LL * d.k_real, st);
}


// row-tile wgrad: returns TSB_ERR_UNSUPPORTED when the shape is not eligible (caller falls back to the patch kernel)
int launch_wgrad_rows(const WgradDesc& d, cudaStream_t st) {
    if (!g_allow_rows || d.Q < 64) return TSB_ERR_UNSUPPORTED;
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
    for (int m = 0; m < 4; ++m) prm.b_bytes[m] = (TW + span_map[m]) * 128;
    int rc = encode_4d(&prm.mapA, d.dy, d.K, d.Q, d.P, d.N, (uint64_t)d.dycs * 2, (uint64_t)d.Q * d.dycs * 2,
                       (uint64_t)d.P * d.Q * d.dycs * 2, 64, TW, 1, 1);
    if (rc) return rc;
    const __nv_bfloat16* xb = reinterpret_cast<const __nv_bfloat16*>(d.x);
    if (d.stride == 1) {
        rc = encode_4d(&prm.mapB[0], xb, d.C, d.W, d.H, d.N, (uint64_t)d.xcs * 2, (uint64_t)d.W * d.xcs * 2,
                       (uint64_t)d.H * d.W * d.xcs * 2, 64, TW + span_map[0], 1, 1);
        if (rc) return rc;
    } else {
        for (int ph = 0; ph < 2; ++ph)
            for (int pw = 0; pw < 2; ++pw) {
                int Hh = (d.H - ph + 1) / 2, Ww = (d.W - pw + 1) / 2;
                if (Hh <= 0) Hh = 1;
                if (Ww <= 0) Ww = 1;
                rc = encode_4d(&prm.mapB[ph * 2 + pw], xb + ((long long)ph * d.W + pw) * d.xcs, d.C, Ww, Hh, d.N,
                               (uint64_t)2 * d.xcs * 2, (uint64_t)2 * d.W * d.xcs * 2, (uint64_t)d.H * d.W * d.xcs * 2, 64,
                               TW + span_map[ph * 2 + pw], 1, 1);
                if (rc) return rc;
            }
    }
    prm.TW = TW;
    prm.tiles_w = (d.Q + TW - 1) / TW;
    prm.tiles_h = d.P;
    prm.total_tiles = prm.tiles_w * prm.tiles_h * d.N;
    prm.K = d.K; prm.C = d.C; prm.dw_row_stride = d.dw_row_stride; prm.dw = d.dw;
    prm.use_base_offset = g_use_base_offset;
    const int co_tiles = (d.K + 127) / 128;
    const int zdim = ng * prm.cchunks;
    int base = zdim * co_tiles;
    int want = (g_wgrad_waves * tsb_num_sms() + base - 1) / base;
    int max_splits = (prm.total_tiles + 15) / 16;
    if (want > max_splits) want = max_splits;
    const long long n_dw = (long long)d.K * d.dw_row_stride;
    if (want > (d.ws ? d.ws_floats / n_dw : 0)) want = (int)(d.ws ? d.ws_floats / n_dw : 0);
    if (want < 1) want = 1;
    prm.tiles_per_split = (prm.total_tiles + want - 1) / want;
    int splits = (prm.total_tiles + prm.tiles_per_split - 1) / prm.tiles_per_split;
    prm.add = splits == 1;
    prm.dw = prm.add ? d.dw : d.ws;
    prm.part_stride = prm.add ? 0 : n_dw;
    { int rc_ = tsb_ensure_dyn_smem(reinterpret_cast<const void*>(wgrad_rows_kernel), kWrSmem); if (rc_) return rc_; }
    wgrad_rows_kernel<<<dim3(splits, co_tiles, zdim), kThreads, kWrSmem, st>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("wgrad_rows");
    return prm.add ? TSB_OK : tsb_det_reduce(d.dw, prm.dw, splits, n_dw, n_dw, st);
}

}  // namespace convv2
