// im2col-free implicit-GEMM convolution on Hopper wgmma tensor cores (sm_90a): the C ABI entry points.
//
//   fprop / dgrad / stem : the persistent kernel of conv_v2.cu;
//   transposed fprop     : the dgrad-form launches with the fprop epilogue (bias, ReLU, bf16/fp32, BN statistics);
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
    // input prologue (flat 1x1 only): X = bf16(relu(x·in_scale[c] + in_shift[c])) over the pro_q pixels
    const float* in_scale;
    const float* in_shift;
    int pro_q;
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

// PRO: the input prologue of tsb_conv1x1_bnrelu_wgrad (flat launches only). Both consumer warpgroups read every X box
// of a stage, so the 256 consumer threads normalise the landed boxes together (bnrelu_box), fence them into the async
// proxy and meet at named barrier 1 before the wgmmas.
template <bool PRO>
__device__ __forceinline__ void wgrad_mnmajor_body(const WgParams& p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kWgBarOff);
    StageRing ring(full_bar, full_bar + kWgStages, kWgStages);

    const int warp = warp_uniform_idx(), lane = threadIdx.x & 31;
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
        ring.init(kWgConsumers * 4);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == kProducer) {
        if (lane == 0) {
            for (int it = 0; it < total_iters; ++it) {
                ring.acquire();
                const int t = t_begin + it;
                const int tw_i = t % p.tiles_w;
                const int th_i = (t / p.tiles_w) % p.tiles_h;
                const int n_img = t / (p.tiles_w * p.tiles_h);
                const int q0 = tw_i * p.TW, p0 = th_i * p.TH;
                uint8_t* a_s = smem + ring.slot * kWgStageBytes;
                uint8_t* b_s = a_s + 2 * kWgBoxBytes;
                mbar_arrive_expect_tx(ring.full_bar(), (uint32_t)((2 + nb) * kWgBoxBytes));
                tma_load_4d(a_s, &p.mapA, ring.full_bar(), co0, q0, p0, n_img);
                tma_load_4d(a_s + kWgBoxBytes, &p.mapA, ring.full_bar(), co0 + 64, q0, p0, n_img);  // OOB → zeros
                for (int j = 0; j < nb; ++j) {
                    const int b = box0 + j;
                    const int tap = b / p.cchunks, cc = b - tap * p.cchunks;
                    const Tap T = p.taps[tap];
                    tma_load_4d(b_s + j * kWgBoxBytes, &p.mapB[T.map], ring.full_bar(), cc * 64, q0 + T.dw, p0 + T.dh, n_img);
                }
                ring.advance();
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
#pragma unroll
        for (int j = 0; j < 4; ++j) fence_operands(acc[j]);
        for (int it = 0; it < total_iters; ++it) {
            ring.wait_full();
            if constexpr (PRO) {
                const int rows = min(64, p.pro_q - (t_begin + it) * 64);   // flat: tile t holds pixels [64 t, 64 t + 64)
                uint8_t* b_s = smem + ring.slot * kWgStageBytes + 2 * kWgBoxBytes;
                for (int j = 0; j < nb; ++j) {   // one tap: box b holds channel chunk b
                    bnrelu_box<64, kWgConsumers * 128>(b_s + j * kWgBoxBytes, rows, threadIdx.x, p.in_scale + (box0 + j) * 64,
                                                       p.in_shift + (box0 + j) * 64);
                }
                fence_proxy_async();
                asm volatile("bar.sync 1, %0;" ::"n"(kWgConsumers * 128) : "memory");
            }
            const uint32_t a_lo = base_lo + (uint32_t)(ring.slot * (kWgStageBytes >> 4)) + (uint32_t)c * (kWgBoxBytes >> 4);
            const uint32_t b_lo = base_lo + (uint32_t)(ring.slot * (kWgStageBytes >> 4)) + ((2 * kWgBoxBytes) >> 4);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (j < nb) {
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        wgmma_m64n64<1, 1>(acc[j], desc_at(desc_hi, a_lo + 128 * k),
                                           desc_at(desc_hi, b_lo + (uint32_t)j * (kWgBoxBytes >> 4) + 128 * k), 1u);
                }
            }
            ring.commit_release_prev();
        }
        ring.drain();
#pragma unroll
        for (int j = 0; j < 4; ++j) fence_operands(acc[j]);
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

__global__ void __launch_bounds__(kWgThreads, 1) wgrad_mnmajor_kernel(const __grid_constant__ WgParams p) {
    wgrad_mnmajor_body<false>(p);
}
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_mnmajor_bnrelu_kernel(const __grid_constant__ WgParams p) {
    wgrad_mnmajor_body<true>(p);
}

int launch_wg(const WgParams& prm, int splits, int co_tiles, int groups, cudaStream_t st) {
    const void* k = prm.in_scale ? reinterpret_cast<const void*>(wgrad_mnmajor_bnrelu_kernel)
                                 : reinterpret_cast<const void*>(wgrad_mnmajor_kernel);
    { int rc_ = tsb_ensure_dyn_smem(k, kWgSmemTotal); if (rc_) return rc_; }
    if (prm.in_scale) wgrad_mnmajor_bnrelu_kernel<<<dim3(splits, co_tiles, groups), kWgThreads, kWgSmemTotal, st>>>(prm);
    else wgrad_mnmajor_kernel<<<dim3(splits, co_tiles, groups), kWgThreads, kWgSmemTotal, st>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("wgrad_mnmajor");
    return TSB_OK;
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
static int fprop_impl(const tsb_conv_shape* s, const void* x, int xcs, const void* w, const float* bias, void* y, int ydtype,
                      int ycs, float* sum, float* sumsq, float* ws, long long ws_floats, const void* res, int relu,
                      tsb_stream_t stream, const float* in_scale = nullptr, const float* in_shift = nullptr) {
    int rc = check_conv_shape(s, "tsb_conv2d_fprop");
    if (rc) return rc;
    TSB_REQUIRE(x && w && y, "tsb_conv2d_fprop: null pointer");
    TSB_REQUIRE(s->C % 64 == 0, "tsb_conv2d_fprop: C must be a multiple of 64 (got %d)", s->C);
    TSB_REQUIRE(xcs % 8 == 0 && xcs >= s->C && tsb_aligned16(x) && tsb_aligned16(w), "tsb_conv2d_fprop: x alignment");
    TSB_REQUIRE(ydtype == TSB_BF16 || ydtype == TSB_F32, "tsb_conv2d_fprop: bad ydtype");
    TSB_REQUIRE(ycs % 8 == 0 && ycs >= s->K && tsb_aligned16(y),
                "tsb_conv2d_fprop: y channel stride must be a multiple of 8 and at least K (got ycs %d, K %d)", ycs, s->K);
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
    const int nt = forward_taps(s, d.taps);
    const int kst = (s->K + 7) / 8 * 8;   // <= ycs: ycs is a multiple of 8 and at least K
    d.act = x; d.aN = N; d.aH = H; d.aW = W; d.aC = s->C; d.acs = xcs; d.act_stride = s->stride; d.flat = flat;
    d.ntaps = nt; d.kchunks = s->C / 64;
    d.w = w; d.w_rows = s->K; d.w_k = (long long)s->R * s->S * s->C; d.ncols = kst;
    d.Nl = N; d.Pl = P; d.Ql = Q;
    d.out_n_stride = (long long)P * Q * ycs; d.out_p_stride = (long long)Q * ycs; d.out_q_stride = ycs; d.out_base = 0;
    d.k_real = s->K; d.k_store = kst; d.out_f32 = (ydtype == TSB_F32); d.accumulate = 0;
    d.bias = bias; d.sum = sum; d.sumsq = sumsq; d.out = y;
    d.relu = relu; d.res = res;
    d.ws = ws; d.ws_floats = ws_floats;
    d.in_scale = in_scale; d.in_shift = in_shift;
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

// The input-prologue checks of the two tsb_conv1x1_bnrelu_* entry points: a 1x1 stride-1 unpadded geometry (anything
// else is TSB_ERR_UNSUPPORTED), C % 64 == 0, 16-byte aligned per-channel vectors.
static int check_bnrelu_1x1(const tsb_conv_shape* s, const float* in_scale, const float* in_shift, const char* who) {
    int rc = check_conv_shape(s, who);
    if (rc) return rc;
    if (!(s->R == 1 && s->S == 1 && s->stride == 1 && s->pad == 0))
        TSB_FAIL(TSB_ERR_UNSUPPORTED, "%s: only 1x1 stride-1 convolutions without padding (got R %d, stride %d, pad %d)", who,
                 s->R, s->stride, s->pad);
    TSB_REQUIRE(in_scale && in_shift, "%s: null in_scale / in_shift", who);
    TSB_REQUIRE(tsb_aligned16(in_scale) && tsb_aligned16(in_shift), "%s: in_scale and in_shift must be 16-byte aligned", who);
    TSB_REQUIRE(s->C % 64 == 0, "%s: C must be a multiple of 64 (got %d)", who, s->C);
    return TSB_OK;
}

extern "C" int tsb_conv1x1_bnrelu_fprop(const tsb_conv_shape* s, const void* x, int xcs, const float* in_scale,
                                        const float* in_shift, const void* w, const float* bias, int relu, void* y,
                                        int ydtype, int ycs, float* sum, float* sumsq, float* ws, long long ws_floats,
                                        tsb_stream_t stream) {
    const char* who = "tsb_conv1x1_bnrelu_fprop";
    int rc = check_bnrelu_1x1(s, in_scale, in_shift, who);
    if (rc) return rc;
    TSB_REQUIRE(x && w && y, "%s: null pointer", who);
    TSB_REQUIRE(xcs % 8 == 0 && xcs >= s->C && tsb_aligned16(x) && tsb_aligned16(w),
                "%s: x channel stride must be a multiple of 8 and at least C, x and w 16-byte aligned (got xcs %d, C %d)", who,
                xcs, s->C);
    TSB_REQUIRE(ycs % 8 == 0 && ycs >= s->K && tsb_aligned16(y),
                "%s: y channel stride must be a multiple of 8 and at least K (got ycs %d, K %d)", who, ycs, s->K);
    TSB_REQUIRE(!(sum && relu), "%s: the statistics epilogue (training) takes no ReLU", who);
    return fprop_impl(s, x, xcs, w, bias, y, ydtype, ycs, sum, sumsq, ws, ws_floats, nullptr, relu != 0, stream, in_scale,
                      in_shift);
}

// The dgrad-form launches of conv geometry `s`: out[N,H,W,·] (channel stride ocs) = the transposed convolution of
// act[N,P,Q,K] (channel stride acs) by the conv's weight, read through the flipped pack wt [C][R][S][K]. Stride 1 is one
// launch; stride 2 is one launch per parity class (ph, pw) of the output, over that class's strided sub-grid, with the
// taps that reach it. A class no tap reaches (a 1x1 kernel at stride 2) runs with no taps, so its positions receive
// the epilogue of a zero accumulator. `epi` carries the epilogue fields (bias, relu, out_f32, k_store, accumulate,
// sum/sumsq, ws). With statistics each launch leaves its per-CTA slots in the workspace after those of the previous
// class, and all slots are added in class order, then CTA order, at the end: the result repeats bit for bit.
static int adjoint_launches(const tsb_conv_shape* s, const void* act, int acs, const void* wt, void* out, int ocs,
                            const convv2::Desc& epi, const char* who, cudaStream_t st) {
    const int classes = (s->stride == 1) ? 1 : 4;
    int slots = 0;   // statistics slots written so far, 2 * C floats each
    for (int cls = 0; cls < classes; ++cls) {
        const int ph = cls >> 1, pw = cls & 1;
        convv2::Desc d = epi;
        int N = s->N, P = s->P, Q = s->Q;          // act geometry (the A operand)
        int Hl, Wl;                                 // launch output grid
        const bool flat = (s->R == 1 && s->stride == 1 && s->pad == 0);
        if (s->stride == 1) { Hl = s->H; Wl = s->W; }
        else { Hl = (s->H - ph + 1) / 2; Wl = (s->W - pw + 1) / 2; }
        if (Hl <= 0 || Wl <= 0) continue;
        if (flat) {
            long long npix = (long long)N * P * Q;
            TSB_REQUIRE(npix < (1ll << 31), "%s: too many pixels", who);
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
            d.out_n_stride = 0; d.out_p_stride = 0; d.out_q_stride = ocs; d.out_base = 0;
        } else if (s->stride == 1) {
            d.out_n_stride = (long long)s->H * s->W * ocs;
            d.out_p_stride = (long long)s->W * ocs;
            d.out_q_stride = ocs;
            d.out_base = 0;
        } else {
            d.out_n_stride = (long long)s->H * s->W * ocs;
            d.out_p_stride = (long long)2 * s->W * ocs;
            d.out_q_stride = (long long)2 * ocs;
            d.out_base = ((long long)ph * s->W + pw) * ocs;
        }
        d.act = act; d.aN = N; d.aH = P; d.aW = Q; d.aC = s->K; d.acs = acs; d.act_stride = 1; d.flat = flat;
        d.ntaps = nt; d.kchunks = s->K / 64;
        d.w = wt; d.w_rows = s->C; d.w_k = (long long)s->R * s->S * s->K; d.ncols = s->C;
        d.Nl = N; d.Pl = Hl; d.Ql = Wl;
        d.k_real = s->C;
        d.out = out;
        int used = 0;
        if (epi.sum != nullptr) {
            const long long off = (long long)slots * 2 * s->C;
            TSB_REQUIRE(epi.ws && off < epi.ws_floats, "%s: statistics workspace too small", who);
            d.ws = epi.ws + off; d.ws_floats = epi.ws_floats - off;
        }
        const int rc = convv2::launch(d, st, epi.sum != nullptr ? &used : nullptr);
        if (rc) return rc;
        slots += used;
    }
    if (epi.sum == nullptr || slots == 0) return TSB_OK;
    // the sumsq slots follow the sum slots of the same CTA: a stride of 2·C between slots
    return tsb_det_reduce_pair(epi.sum, epi.sumsq, epi.ws, slots, s->C, st);
}

extern "C" int tsb_conv2d_dgrad(const tsb_conv_shape* s, const void* dy, int dycs, const void* wt, void* dx, int dxcs,
                                int accumulate, tsb_stream_t stream) {
    int rc = check_conv_shape(s, "tsb_conv2d_dgrad");
    if (rc) return rc;
    TSB_REQUIRE(dy && wt && dx, "tsb_conv2d_dgrad: null pointer");
    TSB_REQUIRE(s->K % 64 == 0, "tsb_conv2d_dgrad: K must be a multiple of 64 (pad the classifier to 64), got %d", s->K);
    TSB_REQUIRE(s->C % 8 == 0 && dycs % 8 == 0 && dycs >= s->K && dxcs % 8 == 0 && dxcs >= s->C && tsb_aligned16(dy) && tsb_aligned16(dx) && tsb_aligned16(wt),
                "tsb_conv2d_dgrad: alignment");
    convv2::Desc epi;
    memset(&epi, 0, sizeof(epi));
    epi.k_store = s->C; epi.accumulate = accumulate;
    return adjoint_launches(s, dy, dycs, wt, dx, dxcs, epi, "tsb_conv2d_dgrad", (cudaStream_t)stream);
}

extern "C" int tsb_conv_transpose2d_fprop(const tsb_conv_shape* s, const void* x, int xcs, const void* wt, const float* bias,
                                          int relu, void* y, int ydtype, int ycs, float* sum, float* sumsq, float* ws,
                                          long long ws_floats, tsb_stream_t stream) {
    int rc = check_conv_shape(s, "tsb_conv_transpose2d_fprop");
    if (rc) return rc;
    TSB_REQUIRE(x && wt && y, "tsb_conv_transpose2d_fprop: null pointer");
    TSB_REQUIRE(s->K % 64 == 0, "tsb_conv_transpose2d_fprop: input channels (K of the adjoint conv) must be a multiple of 64, got %d", s->K);
    TSB_REQUIRE(s->C % 8 == 0, "tsb_conv_transpose2d_fprop: output channels (C of the adjoint conv) must be a multiple of 8, got %d", s->C);
    TSB_REQUIRE(xcs % 8 == 0 && xcs >= s->K && tsb_aligned16(x) && tsb_aligned16(wt),
                "tsb_conv_transpose2d_fprop: x channel stride must be a multiple of 8 and at least K (got xcs %d, K %d)", xcs, s->K);
    TSB_REQUIRE(ydtype == TSB_BF16 || ydtype == TSB_F32, "tsb_conv_transpose2d_fprop: bad ydtype");
    TSB_REQUIRE(ycs % 8 == 0 && ycs >= s->C && tsb_aligned16(y),
                "tsb_conv_transpose2d_fprop: y channel stride must be a multiple of 8 and at least C (got ycs %d, C %d)", ycs, s->C);
    TSB_REQUIRE((sum == nullptr) == (sumsq == nullptr), "tsb_conv_transpose2d_fprop: sum and sumsq go together");
    TSB_REQUIRE(!(sum && ydtype != TSB_BF16), "tsb_conv_transpose2d_fprop: statistics need bf16 output");
    convv2::Desc epi;
    memset(&epi, 0, sizeof(epi));
    epi.k_store = s->C; epi.out_f32 = (ydtype == TSB_F32);
    epi.bias = bias; epi.relu = relu != 0; epi.sum = sum; epi.sumsq = sumsq;
    epi.ws = ws; epi.ws_floats = ws_floats;
    return adjoint_launches(s, x, xcs, wt, y, ycs, epi, "tsb_conv_transpose2d_fprop", (cudaStream_t)stream);
}

namespace {
int pick_nb(int nboxes) {
    if (nboxes % 4 == 0) return 4;
    if (nboxes % 3 == 0) return 3;
    if (nboxes % 2 == 0) return 2;
    return 1;
}
// the generic kernel; prm comes with its maps, taps, tiling, K, C, dw_row_stride, and dw = dW
int wgrad_common(WgParams& prm, int N, int P, int Q, int K, float* ws, long long ws_floats, cudaStream_t st) {
    prm.tiles_w = (Q + prm.TW - 1) / prm.TW;
    prm.tiles_h = (P + prm.TH - 1) / prm.TH;
    prm.total_tiles = prm.tiles_w * prm.tiles_h * N;
    prm.nboxes = prm.ntaps * prm.cchunks;
    prm.nb = pick_nb(prm.nboxes);
    const int groups = prm.nboxes / prm.nb;
    const int co_tiles = (K + 127) / 128;
    // about two waves of CTAs, at least 8 tiles per split
    float* dw = prm.dw;
    const SplitPlan sp = plan_splits(wave_splits(groups * co_tiles, prm.total_tiles, 8), prm.total_tiles,
                                     (long long)K * prm.dw_row_stride, dw, ws, ws_floats);
    prm.tiles_per_split = sp.tiles_per_split;
    prm.add = sp.add; prm.dw = sp.dst; prm.part_stride = sp.part_stride;
    int rc = launch_wg(prm, sp.splits, co_tiles, groups, st);
    return rc ? rc : finish_splits(sp, dw, st);
}
}  // namespace

static int wgrad_impl(const tsb_conv_shape* s, const void* x, int xcs, const void* dy, int dycs, float* dw, float* ws,
                      long long ws_floats, tsb_stream_t stream, const char* who, const float* in_scale = nullptr,
                      const float* in_shift = nullptr) {
    int rc = check_conv_shape(s, who);
    if (rc) return rc;
    TSB_REQUIRE(x && dy && dw, "%s: null pointer", who);
    TSB_REQUIRE(s->C % 64 == 0, "%s: C must be a multiple of 64 (got %d)", who, s->C);
    TSB_REQUIRE(xcs % 8 == 0 && xcs >= s->C && dycs % 8 == 0 && dycs >= s->K && tsb_aligned16(x) && tsb_aligned16(dy) &&
                tsb_aligned16(dw), "%s: layout (xcs >= C, dycs >= K, multiples of 8, 16-byte aligned)", who);
    cudaStream_t st = (cudaStream_t)stream;
    int N = s->N, H = s->H, W = s->W, P = s->P, Q = s->Q;
    const bool flat = (s->R == 1 && s->stride == 1 && s->pad == 0);
    if (flat) {
        long long npix = (long long)N * H * W;
        TSB_REQUIRE(npix < (1ll << 31), "tsb_conv2d_wgrad: too many pixels");
        W = (int)npix; H = 1; N = 1; P = 1; Q = W;
    }
    const long long dw_row_stride = (long long)s->R * s->S * s->C;
    if (!flat && s->R > 1) {
        convv2::WgradDesc d;
        memset(&d, 0, sizeof(d));
        d.x = x; d.dy = dy; d.N = N; d.H = H; d.W = W; d.C = s->C; d.xcs = xcs; d.P = P; d.Q = Q; d.K = s->K; d.dycs = dycs;
        d.stride = s->stride;
        d.ntaps = forward_taps(s, d.taps);
        d.dw_row_stride = dw_row_stride; d.dw = dw;
        d.ws = ws; d.ws_floats = ws_floats;
        rc = convv2::launch_wgrad_taps(d, s->R, s->pad, s->dil, st);   // 3x3 stride 1: all nine taps in one CTA
        if (rc != TSB_ERR_UNSUPPORTED) return rc;
        rc = convv2::launch_wgrad_rows(d, st);
        if (rc != TSB_ERR_UNSUPPORTED) return rc;
    }
    WgParams prm;
    memset(&prm, 0, sizeof(prm));
    int TW, TH;
    if (flat) { TW = 64; TH = 1; } else pick_tile(Q, 64, &TW, &TH);
    prm.TW = TW; prm.TH = TH; prm.tw_shift = ilog2(TW);
    rc = encode_4d(&prm.mapA, dy, s->K, Q, P, N, (uint64_t)dycs * 2, (uint64_t)Q * dycs * 2, (uint64_t)P * Q * dycs * 2, 64, TW, TH, 1);
    if (rc) return rc;
    const int box_w[4] = {TW, TW, TW, TW};
    rc = encode_act_maps(prm.mapB, x, N, H, W, s->C, xcs, s->stride, box_w, TH);
    if (rc) return rc;
    prm.ntaps = forward_taps(s, prm.taps);
    prm.cchunks = s->C / 64;
    prm.K = s->K;
    prm.C = s->C;
    prm.dw_row_stride = dw_row_stride;
    prm.dw = dw;
    prm.in_scale = in_scale; prm.in_shift = in_shift; prm.pro_q = Q;   // set only for flat launches
    return wgrad_common(prm, N, P, Q, s->K, ws, ws_floats, st);
}

extern "C" int tsb_conv2d_wgrad(const tsb_conv_shape* s, const void* x, int xcs, const void* dy, int dycs, float* dw,
                                float* ws, long long ws_floats, tsb_stream_t stream) {
    return wgrad_impl(s, x, xcs, dy, dycs, dw, ws, ws_floats, stream, "tsb_conv2d_wgrad");
}

extern "C" int tsb_conv1x1_bnrelu_wgrad(const tsb_conv_shape* s, const void* x, int xcs, const float* in_scale,
                                        const float* in_shift, const void* dy, int dycs, float* dw, float* ws,
                                        long long ws_floats, tsb_stream_t stream) {
    const char* who = "tsb_conv1x1_bnrelu_wgrad";
    int rc = check_bnrelu_1x1(s, in_scale, in_shift, who);
    return rc ? rc : wgrad_impl(s, x, xcs, dy, dycs, dw, ws, ws_floats, stream, who, in_scale, in_shift);
}

// ---------------------------------------------------------------------------------- 7x7/2 stem
static int stem_fprop_impl(const void* xs2d, int N, int H, int W, const void* wp, int K, void* y, int ycs, float* sum,
                           float* sumsq, float* ws, long long ws_floats, const float* bias, int relu, tsb_stream_t stream) {
    TSB_REQUIRE(xs2d && wp && y && N > 0 && H > 0 && W > 0 && K > 0, "tsb_conv_stem_fprop: bad args");
    TSB_REQUIRE(H % 2 == 0 && W % 2 == 0 && ycs % 8 == 0 && K % 8 == 0 && ycs >= K,
                "tsb_conv_stem_fprop: H,W even; K, ycs multiples of 8; ycs >= K");
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
    TSB_REQUIRE(H % 2 == 0 && W % 2 == 0 && dycs % 8 == 0 && K % 8 == 0 && dycs >= K,
                "tsb_conv_stem_wgrad: H,W even; K, dycs multiples of 8; dycs >= K");
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
