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
    // input prologue (flat 1x1 only): A = bf16(relu(x·in_scale[c] + in_shift[c])), applied to each landed stage
    const float* in_scale;
    const float* in_shift;
};

// BN = 64 epilogue: each consumer warp turns its 16 channels x 16 pixels of the transposed fragment into pixel-major
// rows through a [16 px][kStgStride] fp32 buffer of its own. Stride 20 keeps the fragment writes (8 channels x 4 pixel
// pairs per instruction) and the float4 reads (16 pixels x 2 channel halves) free of bank conflicts.
constexpr int kStgStride = 20;
constexpr int kStgWarpBytes = 16 * kStgStride * 4;

#define IGEMM_V2_NAME igemm_v2_kernel
#define IGEMM_V2_PRO false
#include "igemm_v2_kernel.inc"
#define IGEMM_V2_NAME igemm_v2_bnrelu_kernel
#define IGEMM_V2_PRO true
#include "igemm_v2_kernel.inc"

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
    const void* k = prm.in_scale ? reinterpret_cast<const void*>(igemm_v2_bnrelu_kernel<BN, RES>)
                                 : reinterpret_cast<const void*>(igemm_v2_kernel<BN, RES>);
    { int rc_ = tsb_ensure_dyn_smem(k, smem); if (rc_) return rc_; }
    if (prm.in_scale) igemm_v2_bnrelu_kernel<BN, RES><<<dim3(grid_x, n_tiles), kThreads, smem, st>>>(prm);
    else igemm_v2_kernel<BN, RES><<<dim3(grid_x, n_tiles), kThreads, smem, st>>>(prm);
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
        if (rows) {   // join a group when its box stays within 8 extra pixels (taps may arrive in either dw order)
            for (int k = 0; k < ng; ++k) {
                const TapGroup& G = prm.groups[k];
                if (G.map != T.map || G.dh != T.dh || G.ntaps >= 3) continue;
                int hi = G.dw0;
                for (int j = 0; j < G.ntaps; ++j) hi = max(hi, G.dw0 + G.row_off[j]);
                if (max(hi, T.dw) - min(G.dw0, T.dw) <= 8) { g = k; break; }
            }
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
    TSB_REQUIRE(d.in_scale == nullptr || (d.flat && !d.stem && d.ntaps == 1), "conv_v2: the input prologue needs a flat 1x1 launch");
    prm.in_scale = d.in_scale; prm.in_shift = d.in_shift;
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
    // the sumsq slots follow the sum slots of the same CTA: a stride of 2·k_real between CTAs
    return tsb_det_reduce_pair(d.sum, d.sumsq, prm.part, grid_x, d.k_real, st);
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
