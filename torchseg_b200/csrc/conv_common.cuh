// Host-side helpers shared by the implicit-GEMM convolution translation units: tensor-map encoding through the
// driver entry point (no link-time libcuda dependency), tiling choices, NHWC activation views.
#pragma once
#include <cuda.h>
#include <mutex>

#include "tsb_common.cuh"

namespace convhost {

constexpr int kMaxTaps = 16;
struct Tap {
    int dh, dw;  // offset of the TMA box origin relative to the output-tile origin (map coordinates)
    int map;     // which A tensor map (stride-2 parity view)
    int bk;      // offset of this tap along the K dimension of B
};

// ------------------------------------------------------------------------------------------------
// host side: tensor-map encoding through the driver entry point (no link-time libcuda dependency)
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &f, 12000, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(f);
    });
    // The encode call goes to the DRIVER API, which needs a context current on the calling thread. A fresh thread
    // (autograd's backward worker) that has not yet made a context-binding runtime call gets CUDA_ERROR_INVALID_CONTEXT
    // (201); cudaFree(0) binds the device's primary context to this thread once.
    static thread_local bool t_bound = false;
    if (!t_bound) {
        cudaFree(0);
        t_bound = true;
    }
    return fn;
}

// rank-4 bf16 map; strides in BYTES for dims 1..3; zero OOB fill; 128B swizzle
static inline int encode_4d(CUtensorMap* m, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3, uint64_t s1,
              uint64_t s2, uint64_t s3, uint32_t b0, uint32_t b1, uint32_t b2, uint32_t b3) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) TSB_FAIL(TSB_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    cuuint64_t dims[4] = {d0, d1, d2, d3};
    cuuint64_t strides[3] = {s1, s2, s3};
    cuuint32_t box[4] = {b0, b1, b2, b3};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        TSB_FAIL(TSB_ERR_CUDA, "cuTensorMapEncodeTiled(4d) failed: %d dims=(%llu,%llu,%llu,%llu) strides=(%llu,%llu,%llu) box=(%u,%u,%u,%u)",
                 (int)r, (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, (unsigned long long)d3,
                 (unsigned long long)s1, (unsigned long long)s2, (unsigned long long)s3, b0, b1, b2, b3);
    return TSB_OK;
}
// rank-3 bf16 map; strides in BYTES for dims 1..2; zero OOB fill; 128B swizzle
static inline int encode_3d(CUtensorMap* m, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t s1,
                            uint64_t s2, uint32_t b0, uint32_t b1, uint32_t b2) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) TSB_FAIL(TSB_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    cuuint64_t dims[3] = {d0, d1, d2};
    cuuint64_t strides[2] = {s1, s2};
    cuuint32_t box[3] = {b0, b1, b2};
    cuuint32_t es[3] = {1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        TSB_FAIL(TSB_ERR_CUDA, "cuTensorMapEncodeTiled(3d) failed: %d dims=(%llu,%llu,%llu) strides=(%llu,%llu) box=(%u,%u,%u)",
                 (int)r, (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, (unsigned long long)s1,
                 (unsigned long long)s2, b0, b1, b2);
    return TSB_OK;
}
static inline int encode_2d(CUtensorMap* m, const void* base, uint64_t d0, uint64_t d1, uint64_t s1, uint32_t b0, uint32_t b1) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) TSB_FAIL(TSB_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    cuuint64_t dims[2] = {d0, d1};
    cuuint64_t strides[1] = {s1};
    cuuint32_t box[2] = {b0, b1};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        TSB_FAIL(TSB_ERR_CUDA, "cuTensorMapEncodeTiled(2d) failed: %d dims=(%llu,%llu) stride=%llu box=(%u,%u)", (int)r,
                 (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)s1, b0, b1);
    return TSB_OK;
}

inline int floordiv(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }
inline int posmod(int a, int b) { int m = a % b; return m < 0 ? m + b : m; }
inline int pow2ceil(int v) { int p = 1; while (p < v) p <<= 1; return p; }
inline int ilog2(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }

// spatial tile of `npx` (128 or 64) pixels: TW x TH with TW a power of two
static inline void pick_tile(int Q, int npx, int* TW, int* TH) {
    int tw = pow2ceil(Q);
    int pref = (npx == 128) ? 16 : 8;
    if (tw > pref) tw = pref;
    if (tw > npx) tw = npx;
    *TW = tw;
    *TH = npx / tw;
}

// A-operand maps over an NHWC bf16 tensor [N,H,W,Cs] (channel count Cc, channel stride cs), for a conv of
// stride `st`: st==1 → 1 map; st==2 → 4 parity views (ph,pw) of dims ceil((H-ph)/2) x ceil((W-pw)/2).
// Map m loads boxes of 64 channels x box_w[m] pixels x TH rows.
static inline int encode_act_maps(CUtensorMap* maps, const void* base, int N, int H, int W, int Cc, int cs, int st,
                                  const int box_w[4], int TH) {
    const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(base);
    if (st == 1) {
        return encode_4d(&maps[0], b, Cc, W, H, N, (uint64_t)cs * 2, (uint64_t)W * cs * 2, (uint64_t)H * W * cs * 2, 64,
                         box_w[0], TH, 1);
    }
    for (int ph = 0; ph < 2; ++ph)
        for (int pw = 0; pw < 2; ++pw) {
            int Hh = (H - ph + 1) / 2, Ww = (W - pw + 1) / 2;
            if (Hh <= 0 || Ww <= 0) { Hh = Hh > 0 ? Hh : 1; Ww = Ww > 0 ? Ww : 1; }
            int rc = encode_4d(&maps[ph * 2 + pw], b + ((long long)ph * W + pw) * cs, Cc, Ww, Hh, N, (uint64_t)2 * cs * 2,
                               (uint64_t)2 * W * cs * 2, (uint64_t)H * W * cs * 2, 64, box_w[ph * 2 + pw], TH, 1);
            if (rc) return rc;
        }
    return TSB_OK;
}

// Overlapped-window view of the 7x7/2 stem's s2d image: coordinate (e, ow, oh, n) → xs2d[n][oh][ow .. ow+3][0..15]
static inline int encode_stem_map(CUtensorMap* m, const void* xs2d, int N, int H2, int W2, int box_w, int TH) {
    const uint64_t row = (uint64_t)(W2 + 4) * 16 * 2;
    return encode_4d(m, xs2d, 64, (uint64_t)W2, (uint64_t)H2, (uint64_t)N, 32, row, row * H2, 64, box_w, TH, 1);
}

// Forward taps of a conv in (r, s) order: the box origin relative to the output-tile origin, in the coordinates of the
// tap's map (a stride-2 parity view), and the tap's K offset in the packed [K][R][S][C] weights. Returns the count.
static inline int forward_taps(const tsb_conv_shape* s, Tap* taps) {
    int nt = 0;
    for (int r = 0; r < s->R; ++r)
        for (int ss = 0; ss < s->S; ++ss) {
            Tap& T = taps[nt++];
            int th = r * s->dil - s->pad, tw = ss * s->dil - s->pad;
            if (s->stride == 1) { T.dh = th; T.dw = tw; T.map = 0; }
            else {
                int ph = posmod(th, 2), pw = posmod(tw, 2);
                T.dh = (th - ph) / 2; T.dw = (tw - pw) / 2; T.map = ph * 2 + pw;
            }
            T.bk = (r * s->S + ss) * s->C;
        }
    return nt;
}

// How a weight-gradient launch splits its pixel tiles over CTAs (blockIdx.x). Every split stores a dW-shaped slice into
// the workspace and finish_splits adds the slices in split order; one split adds into dW in place, as does a workspace
// too small for two slices. The split count sets the fp32 summation order, so each kernel keeps its own policy for
// `want`, the split count it asks for.
struct SplitPlan {
    int tiles_per_split, splits;
    int add;                 // one split: the kernel adds into dW
    float* dst;              // dW (add) or the workspace slices
    long long part_stride;   // elements between the slices of consecutive splits (0 when add)
    long long n_dw;          // elements of dW
};
static inline SplitPlan plan_splits(int want, int total_tiles, long long n_dw, float* dw, float* ws, long long ws_floats) {
    const long long fit = ws ? ws_floats / n_dw : 0;
    if (want > fit) want = (int)fit;
    if (want < 1) want = 1;
    SplitPlan sp;
    sp.tiles_per_split = (total_tiles + want - 1) / want;
    sp.splits = (total_tiles + sp.tiles_per_split - 1) / sp.tiles_per_split;
    sp.add = sp.splits == 1;
    sp.dst = sp.add ? dw : ws;
    sp.part_stride = sp.add ? 0 : n_dw;
    sp.n_dw = n_dw;
    return sp;
}
static inline int finish_splits(const SplitPlan& sp, float* dw, cudaStream_t st) {
    return sp.add ? TSB_OK : tsb_det_reduce(dw, sp.dst, sp.splits, sp.n_dw, sp.n_dw, st);
}
// Split count for about kWgradWaves waves of `ctas_per_split` CTAs, keeping at least `min_tiles` tiles per split.
constexpr int kWgradWaves = 2;
static inline int wave_splits(int ctas_per_split, int total_tiles, int min_tiles) {
    const int want = (kWgradWaves * tsb_num_sms() + ctas_per_split - 1) / ctas_per_split;
    const int max_splits = (total_tiles + min_tiles - 1) / min_tiles;
    return want < max_splits ? want : max_splits;
}


static inline int check_conv_shape(const tsb_conv_shape* s, const char* who) {
    TSB_REQUIRE(s != nullptr, "%s: null shape", who);
    TSB_REQUIRE(s->N > 0 && s->H > 0 && s->W > 0 && s->C > 0 && s->K > 0, "%s: bad sizes", who);
    TSB_REQUIRE(s->R == s->S && s->R >= 1 && s->R * s->S <= kMaxTaps, "%s: filter must be square with R*S <= %d", who, kMaxTaps);
    TSB_REQUIRE(s->stride == 1 || s->stride == 2, "%s: stride must be 1 or 2", who);
    TSB_REQUIRE(s->dil >= 1 && s->pad >= 0, "%s: bad pad/dil", who);
    int P = (s->H + 2 * s->pad - s->dil * (s->R - 1) - 1) / s->stride + 1;
    int Q = (s->W + 2 * s->pad - s->dil * (s->S - 1) - 1) / s->stride + 1;
    TSB_REQUIRE(P == s->P && Q == s->Q, "%s: P,Q (%d,%d) inconsistent with geometry (%d,%d)", who, s->P, s->Q, P, Q);
    return TSB_OK;
}

}  // namespace convhost
