// wgrad of 3x3 stride-1 convolutions with ALL NINE TAPS IN ONE CTA ("taps" kernel).
//
//   dW[co, (r,s), ci] = Σ_px dY[px, co] · X[px + ((r-1)·dil, (s-1)·dil), ci]
//
// GEMM roles (swapped with respect to wgrad_rows_kernel): the M side carries ci, the N side carries co, one accumulator
// per tap. Consumer warpgroup r owns filter row r:
//   A = X   : MN-major straight out of NHWC shared-memory rows (64 input channels = 128 B per pixel); tap (r, s) reads
//             row-slot r shifted by s·dil pixel rows, so each filter row's activations are staged once for its 3 taps;
//   B = dY  : MN-major, N = 64 output channels, K = 64 pixels per stage, staged once for all nine taps;
//   D_(r,s)[64 ci, 64 co] in registers, 3 x 32 fp32 per thread.
//
// Why: the row kernel maps co to M and runs one CTA per filter row, reading dY (and X) three times; here dY is staged
// once for all nine taps and X once per filter row.
//
// Per stage (64 pixels = TH rows of TW): dY box {64 co, TW, TH} (8 KB) + three X boxes {64 ci, TW + 2·dil, TH} (one per
// filter row, at rows p0 + (r-1)·dil; the zero-filled out-of-bounds halo IS the padding).
#include "conv_common.cuh"
#include "conv_v2.cuh"
#include "sm90_ptx.cuh"

using namespace sm90;
using namespace convhost;

namespace {

constexpr int kTpConsumers = 3;                       // warpgroups, one per filter row
constexpr int kTpThreads = kTpConsumers * 128 + 32;   // + one TMA producer warp
constexpr int kTpMaxStages = 6;
constexpr int kTpDyBytes = 64 * 128;

struct alignas(64) TpParams {
    CUtensorMap mapDy;   // {K, Q, P, N}, box {64, TW, TH, 1}
    CUtensorMap mapX;    // {C, W, H, N}, box {64, TW + 2·dil, TH, 1}
    int TW, TH, dil;
    int tiles_w, tiles_h, total_tiles, tiles_per_split;
    int slot_bytes;      // one X row-slot: (TW + 2·dil)·TH·128
    int stage_bytes, nstages;
    int koff[4];         // byte offset of K-step k inside an X slot: pixel (k·16) of the tile in the (TW+2·dil)-wide rows
    int kdy[4];          // ... and inside the dY tile (always k·2048)
    int K, C;
    long long dw_row_stride;   // R·S·C
    float* dw;                 // dW-shaped slice per split (workspace), part_stride apart; or dW itself when `add`
    long long part_stride;
    int add;                   // one split: add in place
};

__global__ void __launch_bounds__(kTpThreads, 1) wgrad_taps_kernel(const __grid_constant__ TpParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* tail = smem + p.nstages * p.stage_bytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);
    StageRing ring(full_bar, full_bar + kTpMaxStages, p.nstages);
    const int warp = warp_uniform_idx(), lane = threadIdx.x & 31;
    const int co0 = blockIdx.y * 64, ci0 = blockIdx.z * 64;
    const int t_begin = blockIdx.x * p.tiles_per_split;
    const int t_end = min(p.total_tiles, t_begin + p.tiles_per_split);
    const int iters = t_end - t_begin;
    constexpr int kProducer = kTpConsumers * 4;

    if (warp == kProducer && lane == 0) {
        tma_prefetch_desc(&p.mapDy);
        tma_prefetch_desc(&p.mapX);
        ring.init(kTpConsumers * 4);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == kProducer) {
        if (lane == 0) {
            const uint32_t bytes = (uint32_t)(kTpDyBytes + 3 * p.slot_bytes);
            for (int it = 0; it < iters; ++it) {
                ring.acquire();
                const int t = t_begin + it;
                const int q0 = (t % p.tiles_w) * p.TW;
                const int p0 = ((t / p.tiles_w) % p.tiles_h) * p.TH;
                const int n_img = t / (p.tiles_w * p.tiles_h);
                uint8_t* st = smem + ring.slot * p.stage_bytes;
                mbar_arrive_expect_tx(ring.full_bar(), bytes);
                tma_load_4d(st, &p.mapDy, ring.full_bar(), co0, q0, p0, n_img);
#pragma unroll
                for (int r = 0; r < 3; ++r)
                    tma_load_4d(st + kTpDyBytes + r * p.slot_bytes, &p.mapX, ring.full_bar(), ci0, q0 - p.dil,
                                p0 + (r - 1) * p.dil, n_img);
                ring.advance();
            }
        }
    } else {   // every split stores its (possibly all-zero) tile: the slices are summed in split order afterwards
        const int r = warp >> 2, wq = warp & 3;
        const uint64_t desc_hi = desc_hi_sw128(64 * 128, 1024);   // MN-major, one 64-element atom; 8-pixel groups 1 KB apart
        const uint32_t base_lo = smem_u32(smem) >> 4;
        const uint32_t tap16 = (uint32_t)p.dil * 8u;             // 16-byte units between horizontally adjacent taps
        uint32_t ka[4], kb[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) { ka[k] = (uint32_t)p.koff[k] >> 4; kb[k] = (uint32_t)p.kdy[k] >> 4; }
        float acc[3][32];
#pragma unroll
        for (int t = 0; t < 3; ++t)
#pragma unroll
            for (int q = 0; q < 32; ++q) acc[t][q] = 0.f;
#pragma unroll
        for (int t = 0; t < 3; ++t) fence_operands(acc[t]);
        for (int it = 0; it < iters; ++it) {
            ring.wait_full();
            const uint32_t st_lo = base_lo + (uint32_t)(ring.slot * (p.stage_bytes >> 4));
            const uint32_t x_lo = st_lo + (kTpDyBytes >> 4) + (uint32_t)r * ((uint32_t)p.slot_bytes >> 4);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint64_t db = desc_at(desc_hi, st_lo + kb[k]);
#pragma unroll
                for (int t = 0; t < 3; ++t)
                    wgmma_m64n64<1, 1>(acc[t], desc_at(desc_hi, x_lo + t * tap16 + ka[k]), db, 1u);
            }
            ring.commit_release_prev();
        }
        ring.drain();
#pragma unroll
        for (int t = 0; t < 3; ++t) fence_operands(acc[t]);
        // fragment: rows = input channels ci0 + 16·wq + lane/4 (+8), columns = output channels co0 + 8j + 2(lane%4) (+1)
        // dW is [K][3][3][C] fp32
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int ci = ci0 + wq * 16 + (lane >> 2) + 8 * h;
            if (ci >= p.C) continue;
#pragma unroll
            for (int t = 0; t < 3; ++t) {
                float* dst = p.dw + blockIdx.x * p.part_stride + (long long)(r * 3 + t) * p.C + ci;
#pragma unroll
                for (int j = 0; j < 8; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int co = co0 + 8 * j + 2 * (lane & 3) + e;
                        if (co < p.K) put_f1(dst + (long long)co * p.dw_row_stride, acc[t][4 * j + 2 * h + e], p.add);
                    }
            }
        }
    }
}

}  // namespace

namespace convv2 {

// returns TSB_ERR_UNSUPPORTED when the shape is not eligible (caller falls back to the row / patch kernels)
int launch_wgrad_taps(const WgradDesc& d, int R, int pad, int dil, cudaStream_t st) {
    if (R != 3 || d.stride != 1 || pad != dil || dil < 1 || dil > 8) return TSB_ERR_UNSUPPORTED;
    if (d.C % 64 != 0 || d.K % 8 != 0 || d.P != d.H || d.Q != d.W) return TSB_ERR_UNSUPPORTED;
    TpParams prm;
    memset(&prm, 0, sizeof(prm));
    int TW = 64;
    while (TW > 8 && TW / 2 >= d.Q) TW /= 2;      // widest power of two that is not more than ~2x the row
    const int TH = 64 / TW;
    prm.TW = TW; prm.TH = TH; prm.dil = dil;
    const int XW = TW + 2 * dil;
    prm.slot_bytes = XW * TH * 128;
    for (int k = 0; k < 4; ++k) {
        const int px = k * 16;
        prm.koff[k] = ((px / TW) * XW + (px % TW)) * 128;
        prm.kdy[k] = px * 128;
    }
    if (TW < 16) return TSB_ERR_UNSUPPORTED;       // a 16-pixel K-step must stay inside one tile row
    prm.stage_bytes = (kTpDyBytes + 3 * prm.slot_bytes + 1023) / 1024 * 1024;
    int ns = (227 * 1024 - 1024 /*align*/ - 256 /*barriers*/) / prm.stage_bytes;
    if (ns > kTpMaxStages) ns = kTpMaxStages;
    if (ns < 2) return TSB_ERR_UNSUPPORTED;
    prm.nstages = ns;
    int rc = encode_4d(&prm.mapDy, d.dy, d.K, d.Q, d.P, d.N, (uint64_t)d.dycs * 2, (uint64_t)d.Q * d.dycs * 2,
                       (uint64_t)d.P * d.Q * d.dycs * 2, 64, TW, TH, 1);
    if (rc) return rc;
    rc = encode_4d(&prm.mapX, d.x, d.C, d.W, d.H, d.N, (uint64_t)d.xcs * 2, (uint64_t)d.W * d.xcs * 2,
                   (uint64_t)d.H * d.W * d.xcs * 2, 64, XW, TH, 1);
    if (rc) return rc;
    prm.tiles_w = (d.Q + TW - 1) / TW;
    prm.tiles_h = (d.P + TH - 1) / TH;
    prm.total_tiles = prm.tiles_w * prm.tiles_h * d.N;
    prm.K = d.K; prm.C = d.C; prm.dw_row_stride = d.dw_row_stride;
    const int co_tiles = (d.K + 63) / 64, ci_tiles = d.C / 64;
    const int base = co_tiles * ci_tiles;
    // one CTA per SM (persistent over a contiguous pixel range); at least 8 tiles per CTA so the drain of the nine
    // accumulators (96 fp32 reductions per thread) stays small next to the main loop, and the split count that
    // minimises waves x tiles-per-CTA (wave quantisation)
    const int sms = tsb_num_sms();
    int max_splits = (prm.total_tiles + 7) / 8;
    if (max_splits < 1) max_splits = 1;
    if (max_splits > 2 * sms) max_splits = 2 * sms;
    int want = 1;
    long long best = -1;
    for (int sp = 1; sp <= max_splits; ++sp) {
        const long long per = (prm.total_tiles + sp - 1) / sp;
        const long long waves = ((long long)base * sp + sms - 1) / sms;
        const long long cost = waves * (per + 6);     // + ~6 stage-times of prologue / accumulator drain per CTA
        if (best < 0 || cost < best) { best = cost; want = sp; }
    }
    const SplitPlan sp = plan_splits(want, prm.total_tiles, (long long)d.K * d.dw_row_stride, d.dw, d.ws, d.ws_floats);
    prm.tiles_per_split = sp.tiles_per_split;
    prm.add = sp.add; prm.dw = sp.dst; prm.part_stride = sp.part_stride;
    const size_t smem = 1024 + (size_t)ns * prm.stage_bytes + 256;
    rc = tsb_ensure_dyn_smem(reinterpret_cast<const void*>(wgrad_taps_kernel), smem);
    if (rc) return rc;
    wgrad_taps_kernel<<<dim3(sp.splits, co_tiles, ci_tiles), kTpThreads, smem, st>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("wgrad_taps");
    return finish_splits(sp, d.dw, st);
}

}  // namespace convv2
