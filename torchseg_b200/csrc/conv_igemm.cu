// im2col-free implicit-GEMM convolution on Hopper wgmma tensor cores (sm_90a): the C ABI entry points.
//
//   fprop / dgrad / stem : the persistent kernel of conv_v2.cu;
//   wgrad                : the nine-tap kernel (3x3 stride 1, conv_wgrad_taps.cu), the row-tile kernel (long rows,
//                          conv_v2.cu), else the generic kernel below:
//                          D[128 out-ch, 64*nb in-ch] += dY^T[128, 64 px] * X_shift[64 px, 64*nb]; both operands are
//                          MN-major (channels contiguous) straight out of NHWC memory, K = pixels.
//
// Replaces the cuDNN lowering of nn.Conv2d in the reference's seg_oprs.py ConvBnRelu, base_model/resnet.py and the
// BiSeNet heads (SURVEY.md §8 a1,a2).
#include "conv_common.cuh"
#include "conv_v2.cuh"
#include "sm90_ptx.cuh"

using namespace sm90;
using namespace convhost;

namespace {

struct alignas(64) WgParams {
    CUtensorMap mapA;     // dY
    CUtensorMap mapB[4];  // X views
    Tap taps[kMaxTaps];   // bk unused
    int ntaps, cchunks, nb, nboxes;
    int tiles_w, tiles_h, total_tiles, tiles_per_split;
    int tw_shift, TW, TH;
    int K;                    // real out channels
    int C;                    // in channels per tap in dw (row segment length)
    long long dw_row_stride;  // elements between consecutive out channels in dw
    float* dw;                // dW-shaped slice per split (workspace), part_stride apart; or dW itself when `add`
    long long part_stride;
    int add;                  // one split: add in place
};

// ------------------------------------------------------------------------------------------------
// MN-major GEMM for weight gradients: dW[co, (tap, ci)] += Σ_pixels dY[pix, co] * X[pix + tap, ci]
// Warps 0-7: two consumer warpgroups (out channels [64c, 64c + 64) of the 128-channel tile), warp 8: TMA producer.
// ------------------------------------------------------------------------------------------------
constexpr int kWgConsumers = 2;
constexpr int kWgThreads = kWgConsumers * 128 + 32;
constexpr int kWgStages = 4;
constexpr int kWgBoxBytes = 64 * 128;                            // 64 pixels x 64 channels bf16
constexpr int kWgStageBytes = 2 * kWgBoxBytes + 4 * kWgBoxBytes;  // A (2 boxes) + up to 4 B boxes
constexpr int kWgBarOff = kWgStages * kWgStageBytes;
constexpr int kWgSmemTotal = kWgBarOff + 256 + 1024;

__global__ void __launch_bounds__(kWgThreads, 1) wgrad_mnmajor_kernel(const __grid_constant__ WgParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kWgBarOff);
    uint64_t* empty_bar = full_bar + kWgStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int split = blockIdx.x;
    const int co0 = blockIdx.y * 128;
    const int box0 = blockIdx.z * p.nb;
    const int nb = min(p.nb, p.nboxes - box0);
    const int t_begin = split * p.tiles_per_split;
    const int t_end = min(p.total_tiles, t_begin + p.tiles_per_split);
    const int total_iters = t_end - t_begin;
    constexpr int kProducer = kWgConsumers * 4;

    if (warp == kProducer && lane == 0) {
        tma_prefetch_desc(&p.mapA);
        tma_prefetch_desc(&p.mapB[0]);
        for (int s = 0; s < kWgStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kWgConsumers * 4); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == kProducer) {
        if (lane == 0) {
            for (int it = 0; it < total_iters; ++it) {
                const int s = it % kWgStages;
                const uint32_t ph = (uint32_t)(it / kWgStages) & 1u;
                mbar_wait(&empty_bar[s], ph ^ 1u);
                const int t = t_begin + it;
                const int tw_i = t % p.tiles_w;
                const int th_i = (t / p.tiles_w) % p.tiles_h;
                const int n_img = t / (p.tiles_w * p.tiles_h);
                const int q0 = tw_i * p.TW, p0 = th_i * p.TH;
                uint8_t* a_s = smem + s * kWgStageBytes;
                uint8_t* b_s = a_s + 2 * kWgBoxBytes;
                mbar_arrive_expect_tx(&full_bar[s], (uint32_t)((2 + nb) * kWgBoxBytes));
                tma_load_4d(a_s, &p.mapA, &full_bar[s], co0, q0, p0, n_img);
                tma_load_4d(a_s + kWgBoxBytes, &p.mapA, &full_bar[s], co0 + 64, q0, p0, n_img);  // OOB → zeros
                for (int j = 0; j < nb; ++j) {
                    const int b = box0 + j;
                    const int tap = b / p.cchunks, cc = b - tap * p.cchunks;
                    const Tap T = p.taps[tap];
                    tma_load_4d(b_s + j * kWgBoxBytes, &p.mapB[T.map], &full_bar[s], cc * 64, q0 + T.dw, p0 + T.dh, n_img);
                }
            }
        }
    } else {   // every split stores its (possibly all-zero) tile: the slices are summed in split order afterwards
        const int c = warp >> 2, wq = warp & 3;
        // MN-major, SWIZZLE_128B: one 64-channel atom per operand box, 8-pixel groups SBO = 1024 B apart; one MMA
        // consumes 16 pixels = 2048 B = 128 descriptor units
        const uint64_t desc_hi = desc_hi_sw128(kWgBoxBytes, 1024);
        const uint32_t base_lo = smem_u32(smem) >> 4;
        float acc[4][32];
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int q = 0; q < 32; ++q) acc[j][q] = 0.f;
        int s = 0;
        uint32_t ph = 0;
        for (int it = 0; it < total_iters; ++it) {
            mbar_wait(&full_bar[s], ph);
#pragma unroll
            for (int j = 0; j < 4; ++j) fence_operands(acc[j]);
            wgmma_fence();
            const uint32_t a_lo = base_lo + (uint32_t)(s * (kWgStageBytes >> 4)) + (uint32_t)c * (kWgBoxBytes >> 4);
            const uint32_t b_lo = base_lo + (uint32_t)(s * (kWgStageBytes >> 4)) + ((2 * kWgBoxBytes) >> 4);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (j < nb) {
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        wgmma_m64n64<1, 1>(acc[j], desc_at(desc_hi, a_lo + 128 * k, 0),
                                           desc_at(desc_hi, b_lo + (uint32_t)j * (kWgBoxBytes >> 4) + 128 * k, 0), 1u);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int j = 0; j < 4; ++j) fence_operands(acc[j]);
            // wait_group covers only this warp's MMAs: every consumer warp releases the stage
            if (lane == 0) mbar_arrive(&empty_bar[s]);
            if (++s == kWgStages) { s = 0; ph ^= 1u; }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int co = co0 + c * 64 + wq * 16 + (lane >> 2) + 8 * h;
            if (co >= p.K) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (j >= nb) continue;
                const int b = box0 + j;
                const int tap = b / p.cchunks, cc = b - tap * p.cchunks;
                float* dst = p.dw + split * p.part_stride + (long long)co * p.dw_row_stride + (long long)tap * p.C + cc * 64 + 2 * (lane & 3);
#pragma unroll
                for (int q = 0; q < 8; ++q) put_f2(dst + 8 * q, acc[j][4 * q + 2 * h], acc[j][4 * q + 2 * h + 1], p.add);
            }
        }
    }
}

int launch_wg(const WgParams& prm, int splits, int co_tiles, int groups, cudaStream_t st) {
    { int rc_ = tsb_ensure_dyn_smem(reinterpret_cast<const void*>(wgrad_mnmajor_kernel), kWgSmemTotal); if (rc_) return rc_; }
    wgrad_mnmajor_kernel<<<dim3(splits, co_tiles, groups), kWgThreads, kWgSmemTotal, st>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("wgrad_mnmajor");
    return TSB_OK;
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
static int fprop_impl(const tsb_conv_shape* s, const void* x, int xcs, const void* w, const float* bias, void* y, int ydtype,
                      int ycs, float* sum, float* sumsq, float* ws, long long ws_floats, const void* res, int relu,
                      tsb_stream_t stream) {
    int rc = check_conv_shape(s, "tsb_conv2d_fprop");
    if (rc) return rc;
    TSB_REQUIRE(x && w && y, "tsb_conv2d_fprop: null pointer");
    TSB_REQUIRE(s->C % 64 == 0, "tsb_conv2d_fprop: C must be a multiple of 64 (got %d)", s->C);
    TSB_REQUIRE(xcs % 8 == 0 && xcs >= s->C && tsb_aligned16(x) && tsb_aligned16(w), "tsb_conv2d_fprop: x alignment");
    TSB_REQUIRE(ydtype == TSB_BF16 || ydtype == TSB_F32, "tsb_conv2d_fprop: bad ydtype");
    TSB_REQUIRE(ycs % 8 == 0 && tsb_aligned16(y), "tsb_conv2d_fprop: y channel stride must be a multiple of 8");
    TSB_REQUIRE((sum == nullptr) == (sumsq == nullptr), "tsb_conv2d_fprop: sum and sumsq go together");
    TSB_REQUIRE(!(sum && ydtype != TSB_BF16), "tsb_conv2d_fprop: statistics need bf16 output");
    cudaStream_t st = (cudaStream_t)stream;

    int N = s->N, H = s->H, W = s->W, P = s->P, Q = s->Q;
    const bool flat = (s->R == 1 && s->stride == 1 && s->pad == 0);
    if (flat) {  // 1x1: pure GEMM over all pixels
        long long npix = (long long)N * H * W;
        TSB_REQUIRE(npix < (1ll << 31), "tsb_conv2d_fprop: too many pixels");
        W = (int)npix; H = 1; N = 1; P = 1; Q = W;
    }
    convv2::Desc d;
    memset(&d, 0, sizeof(d));
    int nt = 0;
    for (int r = 0; r < s->R; ++r)
        for (int ss = 0; ss < s->S; ++ss) {
            Tap& T = d.taps[nt++];
            int th = r * s->dil - s->pad, tw = ss * s->dil - s->pad;
            if (s->stride == 1) { T.dh = th; T.dw = tw; T.map = 0; }
            else {
                int ph = posmod(th, 2), pw = posmod(tw, 2);
                T.dh = (th - ph) / 2; T.dw = (tw - pw) / 2; T.map = ph * 2 + pw;
            }
            T.bk = (r * s->S + ss) * s->C;
        }
    int kst = (s->K + 7) / 8 * 8;
    if (kst > ycs) kst = ycs;
    d.act = x; d.aN = N; d.aH = H; d.aW = W; d.aC = s->C; d.acs = xcs; d.act_stride = s->stride; d.flat = flat;
    d.ntaps = nt; d.kchunks = s->C / 64;
    d.w = w; d.w_rows = s->K; d.w_k = (long long)s->R * s->S * s->C; d.ncols = kst;
    d.Nl = N; d.Pl = P; d.Ql = Q;
    d.out_n_stride = (long long)P * Q * ycs; d.out_p_stride = (long long)Q * ycs; d.out_q_stride = ycs; d.out_base = 0;
    d.k_real = s->K; d.k_store = kst; d.out_f32 = (ydtype == TSB_F32); d.accumulate = 0;
    d.bias = bias; d.sum = sum; d.sumsq = sumsq; d.out = y;
    d.relu = relu; d.res = res;
    d.ws = ws; d.ws_floats = ws_floats;
    return convv2::launch(d, st);
}

extern "C" int tsb_conv2d_fprop(const tsb_conv_shape* s, const void* x, int xcs, const void* w, const float* bias,
                                void* y, int ydtype, int ycs, float* sum, float* sumsq, float* ws, long long ws_floats,
                                tsb_stream_t stream) {
    return fprop_impl(s, x, xcs, w, bias, y, ydtype, ycs, sum, sumsq, ws, ws_floats, nullptr, 0, stream);
}

extern "C" int tsb_conv2d_fprop_fused(const tsb_conv_shape* s, const void* x, int xcs, const void* w, const float* bias,
                                      const void* res, int rescs, int relu, void* y, int ydtype, int ycs,
                                      tsb_stream_t stream) {
    TSB_REQUIRE(res == nullptr || (rescs == ycs && ydtype == TSB_BF16 && tsb_aligned16(res)),
                "tsb_conv2d_fprop_fused: the residual must be a bf16 tensor laid out exactly like the output (rescs == ycs)");
    return fprop_impl(s, x, xcs, w, bias, y, ydtype, ycs, nullptr, nullptr, nullptr, 0, res, relu != 0, stream);
}

extern "C" int tsb_conv2d_dgrad(const tsb_conv_shape* s, const void* dy, int dycs, const void* wt, void* dx, int dxcs,
                                int accumulate, tsb_stream_t stream) {
    int rc = check_conv_shape(s, "tsb_conv2d_dgrad");
    if (rc) return rc;
    TSB_REQUIRE(dy && wt && dx, "tsb_conv2d_dgrad: null pointer");
    TSB_REQUIRE(s->K % 64 == 0, "tsb_conv2d_dgrad: K must be a multiple of 64 (pad the classifier to 64), got %d", s->K);
    TSB_REQUIRE(s->C % 8 == 0 && dycs % 8 == 0 && dycs >= s->K && dxcs % 8 == 0 && dxcs >= s->C && tsb_aligned16(dy) && tsb_aligned16(dx) && tsb_aligned16(wt),
                "tsb_conv2d_dgrad: alignment");
    cudaStream_t st = (cudaStream_t)stream;
    const int classes = (s->stride == 1) ? 1 : 4;
    for (int cls = 0; cls < classes; ++cls) {
        const int ph = cls >> 1, pw = cls & 1;
        convv2::Desc d;
        memset(&d, 0, sizeof(d));
        int N = s->N, P = s->P, Q = s->Q;          // dY geometry (the A operand)
        int Hl, Wl;                                 // launch output grid
        const bool flat = (s->R == 1 && s->stride == 1 && s->pad == 0);
        if (s->stride == 1) { Hl = s->H; Wl = s->W; }
        else { Hl = (s->H - ph + 1) / 2; Wl = (s->W - pw + 1) / 2; }
        if (Hl <= 0 || Wl <= 0) continue;
        if (flat) {
            long long npix = (long long)N * P * Q;
            TSB_REQUIRE(npix < (1ll << 31), "tsb_conv2d_dgrad: too many pixels");
            Q = (int)npix; P = 1; N = 1; Hl = 1; Wl = Q;
        }
        int nt = 0;
        for (int r = 0; r < s->R; ++r) {
            int th = (s->stride == 1 ? 0 : ph) + s->pad - r * s->dil;
            if (s->stride == 2 && posmod(th, 2) != 0) continue;
            for (int ss = 0; ss < s->S; ++ss) {
                int tw = (s->stride == 1 ? 0 : pw) + s->pad - ss * s->dil;
                if (s->stride == 2 && posmod(tw, 2) != 0) continue;
                Tap& T = d.taps[nt++];
                T.dh = (s->stride == 1) ? th : th / 2;   // th even here, exact
                T.dw = (s->stride == 1) ? tw : tw / 2;
                T.map = 0;
                // wt is [C][R][S][K] with flipped taps: index (R-1-r, S-1-ss)
                T.bk = ((s->R - 1 - r) * s->S + (s->S - 1 - ss)) * s->K;
            }
        }
        if (flat) {
            d.out_n_stride = 0; d.out_p_stride = 0; d.out_q_stride = dxcs; d.out_base = 0;
        } else if (s->stride == 1) {
            d.out_n_stride = (long long)s->H * s->W * dxcs;
            d.out_p_stride = (long long)s->W * dxcs;
            d.out_q_stride = dxcs;
            d.out_base = 0;
        } else {
            d.out_n_stride = (long long)s->H * s->W * dxcs;
            d.out_p_stride = (long long)2 * s->W * dxcs;
            d.out_q_stride = (long long)2 * dxcs;
            d.out_base = ((long long)ph * s->W + pw) * dxcs;
        }
        d.act = dy; d.aN = N; d.aH = P; d.aW = Q; d.aC = s->K; d.acs = dycs; d.act_stride = 1; d.flat = flat;
        d.ntaps = nt; d.kchunks = s->K / 64;
        d.w = wt; d.w_rows = s->C; d.w_k = (long long)s->R * s->S * s->K; d.ncols = s->C;
        d.Nl = N; d.Pl = Hl; d.Ql = Wl;
        d.k_real = s->C; d.k_store = s->C; d.out_f32 = 0; d.accumulate = accumulate;
        d.out = dx;
        rc = convv2::launch(d, st);
        if (rc) return rc;
    }
    return TSB_OK;
}

namespace {
int pick_nb(int nboxes) {
    if (nboxes % 4 == 0) return 4;
    if (nboxes % 3 == 0) return 3;
    if (nboxes % 2 == 0) return 2;
    return 1;
}
int wgrad_common(WgParams& prm, int N, int P, int Q, int K, float* ws, long long ws_floats, cudaStream_t st) {
    prm.tiles_w = (Q + prm.TW - 1) / prm.TW;
    prm.tiles_h = (P + prm.TH - 1) / prm.TH;
    prm.total_tiles = prm.tiles_w * prm.tiles_h * N;
    prm.nboxes = prm.ntaps * prm.cchunks;
    prm.nb = pick_nb(prm.nboxes);
    const int groups = prm.nboxes / prm.nb;
    const int co_tiles = (K + 127) / 128;
    // split the pixel range so the grid covers ~2 waves of SMs, at least 8 tiles per CTA
    int base = groups * co_tiles;
    int want = (convv2::g_wgrad_waves * tsb_num_sms() + base - 1) / base;
    int max_splits = (prm.total_tiles + 7) / 8;
    if (want > max_splits) want = max_splits;
    const long long n_dw = (long long)K * prm.dw_row_stride;
    if (want > (ws ? ws_floats / n_dw : 0)) want = (int)(ws ? ws_floats / n_dw : 0);
    if (want < 1) want = 1;
    prm.tiles_per_split = (prm.total_tiles + want - 1) / want;
    int splits = (prm.total_tiles + prm.tiles_per_split - 1) / prm.tiles_per_split;
    float* dw = prm.dw;
    prm.add = splits == 1;
    if (!prm.add) { prm.dw = ws; prm.part_stride = n_dw; }
    int rc = launch_wg(prm, splits, co_tiles, groups, st);
    return (rc || prm.add) ? rc : tsb_det_reduce(dw, prm.dw, splits, n_dw, n_dw, st);
}
}  // namespace

extern "C" int tsb_conv2d_wgrad(const tsb_conv_shape* s, const void* x, int xcs, const void* dy, int dycs, float* dw,
                                float* ws, long long ws_floats, tsb_stream_t stream) {
    int rc = check_conv_shape(s, "tsb_conv2d_wgrad");
    if (rc) return rc;
    TSB_REQUIRE(x && dy && dw, "tsb_conv2d_wgrad: null pointer");
    TSB_REQUIRE(s->C % 64 == 0, "tsb_conv2d_wgrad: C must be a multiple of 64 (got %d)", s->C);
    TSB_REQUIRE(xcs % 8 == 0 && dycs % 8 == 0 && dycs >= s->K && tsb_aligned16(x) && tsb_aligned16(dy) && tsb_aligned16(dw),
                "tsb_conv2d_wgrad: alignment");
    cudaStream_t st = (cudaStream_t)stream;
    WgParams prm;
    memset(&prm, 0, sizeof(prm));
    int N = s->N, H = s->H, W = s->W, P = s->P, Q = s->Q;
    const bool flat = (s->R == 1 && s->stride == 1 && s->pad == 0);
    if (flat) {
        long long npix = (long long)N * H * W;
        TSB_REQUIRE(npix < (1ll << 31), "tsb_conv2d_wgrad: too many pixels");
        W = (int)npix; H = 1; N = 1; P = 1; Q = W;
    }
    int TW, TH;
    if (flat) { TW = 64; TH = 1; } else pick_tile(Q, 64, &TW, &TH);
    prm.TW = TW; prm.TH = TH; prm.tw_shift = ilog2(TW);
    rc = encode_4d(&prm.mapA, dy, s->K, Q, P, N, (uint64_t)dycs * 2, (uint64_t)Q * dycs * 2, (uint64_t)P * Q * dycs * 2, 64, TW, TH, 1);
    if (rc) return rc;
    rc = encode_act_maps(prm.mapB, x, N, H, W, s->C, xcs, s->stride, TW, TH);
    if (rc) return rc;
    int nt = 0;
    for (int r = 0; r < s->R; ++r)
        for (int ss = 0; ss < s->S; ++ss) {
            Tap& T = prm.taps[nt++];
            int th = r * s->dil - s->pad, tw = ss * s->dil - s->pad;
            if (s->stride == 1) { T.dh = th; T.dw = tw; T.map = 0; }
            else {
                int ph = posmod(th, 2), pw = posmod(tw, 2);
                T.dh = (th - ph) / 2; T.dw = (tw - pw) / 2; T.map = ph * 2 + pw;
            }
            T.bk = 0;
        }
    prm.ntaps = nt;
    prm.cchunks = s->C / 64;
    prm.K = s->K;
    prm.C = s->C;
    prm.dw_row_stride = (long long)s->R * s->S * s->C;
    prm.dw = dw;
    if (!flat && s->R > 1) {
        convv2::WgradDesc d;
        memset(&d, 0, sizeof(d));
        d.x = x; d.dy = dy; d.N = N; d.H = H; d.W = W; d.C = s->C; d.xcs = xcs; d.P = P; d.Q = Q; d.K = s->K; d.dycs = dycs;
        d.stride = s->stride;
        for (int t = 0; t < nt; ++t) d.taps[t] = prm.taps[t];
        d.ntaps = nt; d.dw_row_stride = prm.dw_row_stride; d.dw = dw;
        d.ws = ws; d.ws_floats = ws_floats;
        rc = convv2::launch_wgrad_taps(d, s->R, s->pad, s->dil, st);   // 3x3 stride 1: all nine taps in one CTA
        if (rc != TSB_ERR_UNSUPPORTED) return rc;
        rc = convv2::launch_wgrad_rows(d, st);
        if (rc != TSB_ERR_UNSUPPORTED) return rc;
    }
    return wgrad_common(prm, N, P, Q, s->K, ws, ws_floats, st);
}

// ---------------------------------------------------------------------------------- 7x7/2 stem
namespace {
// overlapped-window view of the s2d image: coordinate (e, ow, oh, n) → xs2d[n][oh][ow .. ow+3][0..15]
int encode_stem_map(CUtensorMap* m, const void* xs2d, int N, int H2, int W2, int TW, int TH) {
    const uint64_t row = (uint64_t)(W2 + 4) * 16 * 2;
    return encode_4d(m, xs2d, 64, (uint64_t)W2, (uint64_t)H2, (uint64_t)N, 32, row, row * H2, 64, TW, TH, 1);
}
}  // namespace

static int stem_fprop_impl(const void* xs2d, int N, int H, int W, const void* wp, int K, void* y, int ycs, float* sum,
                           float* sumsq, float* ws, long long ws_floats, const float* bias, int relu, tsb_stream_t stream) {
    TSB_REQUIRE(xs2d && wp && y && N > 0 && H > 0 && W > 0 && K > 0, "tsb_conv_stem_fprop: bad args");
    TSB_REQUIRE(H % 2 == 0 && W % 2 == 0 && ycs % 8 == 0 && K % 8 == 0, "tsb_conv_stem_fprop: H,W even; K, ycs multiples of 8");
    TSB_REQUIRE((sum == nullptr) == (sumsq == nullptr), "tsb_conv_stem_fprop: sum and sumsq go together");
    const int H2 = H / 2, W2 = W / 2;
    convv2::Desc d;
    memset(&d, 0, sizeof(d));
    for (int a = 0; a < 4; ++a) { d.taps[a].dh = a - 2; d.taps[a].dw = 0; d.taps[a].map = 0; d.taps[a].bk = a * 64; }
    d.act = xs2d; d.aN = N; d.aH = H2; d.aW = W2; d.aC = 64; d.acs = 16; d.act_stride = 1; d.stem = 1;
    d.ntaps = 4; d.kchunks = 1;
    d.w = wp; d.w_rows = K; d.w_k = 256; d.ncols = K;
    d.Nl = N; d.Pl = H2; d.Ql = W2;
    d.out_n_stride = (long long)H2 * W2 * ycs; d.out_p_stride = (long long)W2 * ycs; d.out_q_stride = ycs;
    d.k_real = K; d.k_store = K;
    d.sum = sum; d.sumsq = sumsq; d.out = y;
    d.bias = bias; d.relu = relu;
    d.ws = ws; d.ws_floats = ws_floats;
    return convv2::launch(d, (cudaStream_t)stream);
}

extern "C" int tsb_conv_stem_fprop(const void* xs2d, int N, int H, int W, const void* wp, int K, void* y, int ycs,
                                   float* sum, float* sumsq, float* ws, long long ws_floats, tsb_stream_t stream) {
    return stem_fprop_impl(xs2d, N, H, W, wp, K, y, ycs, sum, sumsq, ws, ws_floats, nullptr, 0, stream);
}

extern "C" int tsb_conv_stem_fprop_fused(const void* xs2d, int N, int H, int W, const void* wp, int K, const float* bias,
                                         int relu, void* y, int ycs, tsb_stream_t stream) {
    return stem_fprop_impl(xs2d, N, H, W, wp, K, y, ycs, nullptr, nullptr, nullptr, 0, bias, relu != 0, stream);
}

extern "C" int tsb_conv_stem_wgrad(const void* xs2d, int N, int H, int W, const void* dy, int dycs, int K, float* dwp,
                                   float* ws, long long ws_floats, tsb_stream_t stream) {
    TSB_REQUIRE(xs2d && dy && dwp && N > 0 && H > 0 && W > 0 && K > 0, "tsb_conv_stem_wgrad: bad args");
    TSB_REQUIRE(H % 2 == 0 && W % 2 == 0 && dycs % 8 == 0 && K % 8 == 0, "tsb_conv_stem_wgrad: H,W even; K, dycs multiples of 8");
    const int H2 = H / 2, W2 = W / 2;
    WgParams prm;
    memset(&prm, 0, sizeof(prm));
    int TW, TH;
    pick_tile(W2, 64, &TW, &TH);
    prm.TW = TW; prm.TH = TH; prm.tw_shift = ilog2(TW);
    int rc = encode_4d(&prm.mapA, dy, K, W2, H2, N, (uint64_t)dycs * 2, (uint64_t)W2 * dycs * 2, (uint64_t)H2 * W2 * dycs * 2, 64, TW, TH, 1);
    if (rc) return rc;
    rc = encode_stem_map(&prm.mapB[0], xs2d, N, H2, W2, TW, TH);
    if (rc) return rc;
    for (int a = 0; a < 4; ++a) { prm.taps[a].dh = a - 2; prm.taps[a].dw = 0; prm.taps[a].map = 0; prm.taps[a].bk = 0; }
    prm.ntaps = 4;
    prm.cchunks = 1;
    prm.K = K;
    prm.C = 64;             // each tap row contributes 64 packed elements
    prm.dw_row_stride = 256;  // dwp [K][4][64]
    prm.dw = dwp;
    return wgrad_common(prm, N, H2, W2, K, ws, ws_floats, (cudaStream_t)stream);
}
