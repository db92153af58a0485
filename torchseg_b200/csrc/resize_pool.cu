// Bilinear resize (align_corners=True), adaptive average pooling and 3x3/2 max pooling on NHWC tensors.
// HBM-bound: 16-byte vector loads/stores over the channel dimension, grid sized to the SM count.
// Reference call sites: F.interpolate  model/bisenet/cityscapes.bisenet.R18/network.py:82-84,93-94,164-166;
// nn.AdaptiveAvgPool2d furnace/seg_opr/seg_oprs.py:200,223; nn.MaxPool2d furnace/base_model/resnet.py:132.
#include "nhwc_vec.cuh"

namespace {

// pixel index → (n, row, col). One 64-bit division costs ~100 issue slots; activations have < 2^31 pixels, so the
// common case runs on 32-bit unsigned divisions.
__device__ __forceinline__ void split_pix(long long pix, int W, int H, int& w, int& h, int& n) {
    if (pix < 0x7fffffffLL) {
        const unsigned u = (unsigned)pix;
        const unsigned t = u / (unsigned)W;
        w = (int)(u - t * (unsigned)W);
        const unsigned nn = t / (unsigned)H;
        h = (int)(t - nn * (unsigned)H);
        n = (int)nn;
    } else {
        w = (int)(pix % W);
        const long long t = pix / W;
        h = (int)(t % H);
        n = (int)(t / H);
    }
}
constexpr int kThreads = 256;

__host__ __device__ __forceinline__ float area_scale(int in_size, int out_size) {
    return out_size > 1 ? (float)(in_size - 1) / (float)(out_size - 1) : 0.0f;
}
struct Lerp { int i0, i1; float l0, l1; };
__device__ __forceinline__ Lerp make_lerp(float scale, int dst, int in_size) {
    Lerp r;
    float src = __fmul_rn(scale, (float)dst);
    r.i0 = (int)src;
    if (r.i0 > in_size - 1) r.i0 = in_size - 1;
    r.i1 = r.i0 + ((r.i0 < in_size - 1) ? 1 : 0);
    r.l1 = __fsub_rn(src, (float)r.i0);
    r.l0 = __fsub_rn(1.0f, r.l1);
    return r;
}

// ---------------------------------------------------------------- bilinear forward (NHWC → NHWC)
template <typename TI, typename TO>
__global__ void __launch_bounds__(kThreads)
bilinear_fwd_kernel(const TI* __restrict__ in, int ics, TO* __restrict__ out, int ocs, int N, int C8, int Hi, int Wi,
                    int Ho, int Wo) {
    const float ry = area_scale(Hi, Ho), rx = area_scale(Wi, Wo);
    const long long total = (long long)N * Ho * Wo * C8;
    const long long stride_ = (long long)gridDim.x * kThreads;
    VecWalk wk_(C8, (long long)blockIdx.x * kThreads + threadIdx.x, stride_);   // no 64-bit division per vector
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += stride_, wk_.next()) {
        const int c8 = wk_.c8;
        const long long pix = wk_.p;
        int x, y, n;
        split_pix(pix, Wo, Ho, x, y, n);
        Lerp ly = make_lerp(ry, y, Hi), lx = make_lerp(rx, x, Wi);
        const TI* b = in + (long long)n * Hi * Wi * ics + c8 * 8;
        float a[8], bb[8], c[8], d[8], o[8];
        Vec8<TI>::load(b + ((long long)ly.i0 * Wi + lx.i0) * ics, a);
        Vec8<TI>::load(b + ((long long)ly.i0 * Wi + lx.i1) * ics, bb);
        Vec8<TI>::load(b + ((long long)ly.i1 * Wi + lx.i0) * ics, c);
        Vec8<TI>::load(b + ((long long)ly.i1 * Wi + lx.i1) * ics, d);
#pragma unroll
        for (int k = 0; k < 8; ++k)
            o[k] = ly.l0 * (lx.l0 * a[k] + lx.l1 * bb[k]) + ly.l1 * (lx.l0 * c[k] + lx.l1 * d[k]);
        Vec8<TO>::store(out + pix * ocs + c8 * 8, o);
    }
}

// scalar-channel variant (C not a multiple of 8, e.g. 19-class logits) with NHWC or NCHW output
template <typename TI, typename TO, bool kOutNCHW>
__global__ void __launch_bounds__(kThreads)
bilinear_fwd_scalar_kernel(const TI* __restrict__ in, int ics, TO* __restrict__ out, int ocs, int N, int C, int Hi,
                           int Wi, int Ho, int Wo) {
    const float ry = area_scale(Hi, Ho), rx = area_scale(Wi, Wo);
    const long long total = (long long)N * C * Ho * Wo;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        int x, y, c, n;
        if (kOutNCHW) {
            x = (int)(i % Wo); long long t = i / Wo; y = (int)(t % Ho); t /= Ho; c = (int)(t % C); n = (int)(t / C);
        } else {
            c = (int)(i % C); long long t = i / C; x = (int)(t % Wo); t /= Wo; y = (int)(t % Ho); n = (int)(t / Ho);
        }
        Lerp ly = make_lerp(ry, y, Hi), lx = make_lerp(rx, x, Wi);
        const TI* b = in + (long long)n * Hi * Wi * ics + c;
        float a = ld_as_float<TI>(b + ((long long)ly.i0 * Wi + lx.i0) * ics);
        float bb = ld_as_float<TI>(b + ((long long)ly.i0 * Wi + lx.i1) * ics);
        float cc = ld_as_float<TI>(b + ((long long)ly.i1 * Wi + lx.i0) * ics);
        float d = ld_as_float<TI>(b + ((long long)ly.i1 * Wi + lx.i1) * ics);
        // same op order as the OHEM fused path / oracle (no FMA contraction)
        float t0 = __fadd_rn(__fmul_rn(lx.l0, a), __fmul_rn(lx.l1, bb));
        float t1 = __fadd_rn(__fmul_rn(lx.l0, cc), __fmul_rn(lx.l1, d));
        float o = __fadd_rn(__fmul_rn(ly.l0, t0), __fmul_rn(ly.l1, t1));
        if (kOutNCHW) st_from_float<TO>(out + i, o);
        else st_from_float<TO>(out + (((long long)n * Ho + y) * Wo + x) * ocs + c, o);
    }
}

// ---------------------------------------------------------------- bilinear backward (gather form)
// din[n,i,j,c] = Σ_{y,x} wy(y,i) wx(x,j) dout[n,y,x,c]; deterministic, no atomics.
template <typename TO, typename TI>
__global__ void __launch_bounds__(kThreads)
bilinear_bwd_kernel(const TO* __restrict__ dout, int ocs, TI* __restrict__ din, int ics, int N, int C8, int Hi, int Wi,
                    int Ho, int Wo, int accumulate) {
    const float ry = area_scale(Hi, Ho), rx = area_scale(Wi, Wo);
    const long long total = (long long)N * Hi * Wi * C8;
    constexpr int kMaxCand = 12;  // candidate output columns kept in registers (up-scale factors >= 1/4 per side)
    const long long stride_ = (long long)gridDim.x * kThreads;
    VecWalk wk_(C8, (long long)blockIdx.x * kThreads + threadIdx.x, stride_);   // no 64-bit division per vector
    for (long long idx = (long long)blockIdx.x * kThreads + threadIdx.x; idx < total; idx += stride_, wk_.next()) {
        const int c8 = wk_.c8;
        const long long pix = wk_.p;
        int j, i, n;
        split_pix(pix, Wi, Hi, j, i, n);
        int y_lo, y_hi, x_lo, x_hi;
        if (ry > 0.f) { y_lo = max(0, (int)floorf((float)(i - 1) / ry) - 1); y_hi = min(Ho - 1, (int)ceilf((float)(i + 1) / ry) + 1); }
        else { y_lo = 0; y_hi = Ho - 1; }
        if (rx > 0.f) { x_lo = max(0, (int)floorf((float)(j - 1) / rx) - 1); x_hi = min(Wo - 1, (int)ceilf((float)(j + 1) / rx) + 1); }
        else { x_lo = 0; x_hi = Wo - 1; }
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
        const TO* base = dout + (long long)n * Ho * Wo * ocs + c8 * 8;
        const bool small = (x_hi - x_lo + 1) <= kMaxCand;
        float wxs[kMaxCand];
        if (small) {
#pragma unroll
            for (int k = 0; k < kMaxCand; ++k) {
                int x = x_lo + k;
                Lerp lx = make_lerp(rx, min(x, Wo - 1), Wi);
                wxs[k] = (x <= x_hi) ? ((lx.i0 == j ? lx.l0 : 0.f) + (lx.i1 == j ? lx.l1 : 0.f)) : 0.f;
            }
        }
        for (int y = y_lo; y <= y_hi; ++y) {
            Lerp ly = make_lerp(ry, y, Hi);
            float wy = (ly.i0 == i ? ly.l0 : 0.f) + (ly.i1 == i ? ly.l1 : 0.f);
            if (wy == 0.f) continue;
            if (small) {
#pragma unroll
                for (int k = 0; k < kMaxCand; ++k) {
                    if (wxs[k] != 0.f) {
                        float g[8];
                        Vec8<TO>::load(base + ((long long)y * Wo + x_lo + k) * ocs, g);
                        float wgt = wy * wxs[k];
#pragma unroll
                        for (int e = 0; e < 8; ++e) acc[e] += wgt * g[e];
                    }
                }
            } else {
                for (int x = x_lo; x <= x_hi; ++x) {
                    Lerp lx = make_lerp(rx, x, Wi);
                    float wx = (lx.i0 == j ? lx.l0 : 0.f) + (lx.i1 == j ? lx.l1 : 0.f);
                    if (wx == 0.f) continue;
                    float g[8];
                    Vec8<TO>::load(base + ((long long)y * Wo + x) * ocs, g);
                    float wgt = wy * wx;
#pragma unroll
                    for (int e = 0; e < 8; ++e) acc[e] += wgt * g[e];
                }
            }
        }
        TI* dst = din + pix * ics + c8 * 8;
        if (accumulate) {
            float old[8];
            Vec8<TI>::load(dst, old);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += old[k];
        }
        Vec8<TI>::store(dst, acc);
    }
}

// ---------------------------------------------------------------- adaptive average pool
// grid = (N*S*S, chunks). Threads: (pixel lane, channel group of 8). Each chunk stores its bin sums into workspace slot blockIdx.y.
__global__ void __launch_bounds__(kThreads)
adaptive_avgpool_fwd_kernel(const __nv_bfloat16* __restrict__ in, int ics, int N, int C, int H, int W, int S,
                            float* __restrict__ out) {
    extern __shared__ float s_acc[];  // [lanes][C]
    const int C8 = C / 8;
    const int groups_per_pass = min(C8, kThreads);
    const int lanes = kThreads / groups_per_pass;
    const int bin = blockIdx.x;
    const int n = bin / (S * S), bi = (bin / S) % S, bj = bin % S;
    const int h0 = (bi * H) / S, h1 = ((bi + 1) * H + S - 1) / S;
    const int w0 = (bj * W) / S, w1 = ((bj + 1) * W + S - 1) / S;
    const int bw = w1 - w0, npix = (h1 - h0) * bw;
    const float inv_area = 1.0f / (float)npix;
    const int chunk = (npix + gridDim.y - 1) / gridDim.y;
    const int p_begin = blockIdx.y * chunk, p_end = min(npix, p_begin + chunk);
    const int g = threadIdx.x % groups_per_pass, lane = threadIdx.x / groups_per_pass;
    for (int g0 = 0; g0 < C8; g0 += groups_per_pass) {
        const int cg = g0 + g;
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
        if (cg < C8 && lane < lanes) {
            for (int pp = p_begin + lane; pp < p_end; pp += lanes) {
                int hh = h0 + pp / bw, ww = w0 + pp % bw;
                float v[8];
                Vec8<__nv_bfloat16>::load(in + (((long long)n * H + hh) * W + ww) * ics + cg * 8, v);
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[k] += v[k];
            }
        }
        // reduce over pixel lanes through shared memory
        if (lane < lanes) {
#pragma unroll
            for (int k = 0; k < 8; ++k) s_acc[(lane * groups_per_pass + g) * 8 + k] = acc[k];
        }
        __syncthreads();
        if (lane == 0 && cg < C8) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                float s = 0.f;
                for (int l = 0; l < lanes; ++l) s += s_acc[(l * groups_per_pass + g) * 8 + k];
                // slot blockIdx.y of the deterministic workspace; the chunks are summed in order afterwards
                out[(long long)blockIdx.y * gridDim.x * C + (long long)bin * C + cg * 8 + k] = s * inv_area;
            }
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kThreads)
adaptive_avgpool_bwd_kernel(const float* __restrict__ dout, int N, int C8, int H, int W, int S,
                            __nv_bfloat16* __restrict__ din, int ics, int accumulate) {
    const long long total = (long long)N * H * W * C8;
    const long long stride_ = (long long)gridDim.x * kThreads;
    VecWalk wk_(C8, (long long)blockIdx.x * kThreads + threadIdx.x, stride_);   // no 64-bit division per vector
    for (long long idx = (long long)blockIdx.x * kThreads + threadIdx.x; idx < total; idx += stride_, wk_.next()) {
        const int c8 = wk_.c8;
        const long long pix = wk_.p;
        int w, h, n;
        split_pix(pix, W, H, w, h, n);
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
        // bins containing (h,w): adaptive bins may overlap by one row/col when H % S != 0
        int bi_lo = (h * S) / H, bj_lo = (w * S) / W;
        for (int bi = max(0, bi_lo - 1); bi <= min(S - 1, bi_lo + 1); ++bi) {
            int h0 = (bi * H) / S, h1 = ((bi + 1) * H + S - 1) / S;
            if (h < h0 || h >= h1) continue;
            for (int bj = max(0, bj_lo - 1); bj <= min(S - 1, bj_lo + 1); ++bj) {
                int w0 = (bj * W) / S, w1 = ((bj + 1) * W + S - 1) / S;
                if (w < w0 || w >= w1) continue;
                float inv_area = 1.0f / (float)((h1 - h0) * (w1 - w0));
                float g[8];
                ldg8f(dout + (((long long)n * S + bi) * S + bj) * (C8 * 8) + c8 * 8, g);
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[k] += g[k] * inv_area;
            }
        }
        __nv_bfloat16* dst = din + pix * ics + c8 * 8;
        if (accumulate) {
            float old[8];
            Vec8<__nv_bfloat16>::load(dst, old);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += old[k];
        }
        Vec8<__nv_bfloat16>::store(dst, acc);
    }
}

// ---------------------------------------------------------------- max pool 3x3 stride 2 pad 1
// forward also records the arg-max window position r*3+s (first maximum in scan order, strict '>' — ATen
// max_pool2d semantics) as one byte per output element, so the backward is a pure gather.
__global__ void __launch_bounds__(kThreads)
maxpool_fwd_kernel(const __nv_bfloat16* __restrict__ in, int ics, __nv_bfloat16* __restrict__ out, int ocs,
                   uint8_t* __restrict__ idx, int N, int C8, int H, int W, int P, int Q) {
    const long long total = (long long)N * P * Q * C8;
    const long long stride_ = (long long)gridDim.x * kThreads;
    VecWalk wk_(C8, (long long)blockIdx.x * kThreads + threadIdx.x, stride_);   // no 64-bit division per vector
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += stride_, wk_.next()) {
        const int c8 = wk_.c8;
        const long long pix = wk_.p;
        int q, p, n;
        split_pix(pix, Q, P, q, p, n);
        float m[8];
        uint32_t am[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) { m[k] = -INFINITY; am[k] = 0; }
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            int h = 2 * p - 1 + r;
            if (h < 0 || h >= H) continue;
#pragma unroll
            for (int s = 0; s < 3; ++s) {
                int w = 2 * q - 1 + s;
                if (w < 0 || w >= W) continue;
                float v[8];
                Vec8<__nv_bfloat16>::load(in + (((long long)n * H + h) * W + w) * ics + c8 * 8, v);
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    if (v[k] > m[k]) { m[k] = v[k]; am[k] = r * 3 + s; }
            }
        }
        Vec8<__nv_bfloat16>::store(out + pix * ocs + c8 * 8, m);
        if (idx) {
            uint2 pk;
            pk.x = am[0] | (am[1] << 8) | (am[2] << 16) | (am[3] << 24);
            pk.y = am[4] | (am[5] << 8) | (am[6] << 16) | (am[7] << 24);
            *reinterpret_cast<uint2*>(idx + pix * (long long)(C8 * 8) + c8 * 8) = pk;
        }
    }
}

// backward, gather form. One thread owns a 2x2 block of input pixels (h = 2a+dh, w = 2b+dw) x 8 channels: the
// block only touches the four windows (a..a+1) x (b..b+1), so each argmax / gradient vector is loaded once per
// four outputs (1.5x read amplification instead of 6x). Input pixel (h,w) receives dout[p,q] iff idx[p,q] names it.
__global__ void __launch_bounds__(kThreads)
maxpool_bwd_kernel(const uint8_t* __restrict__ idx, const __nv_bfloat16* __restrict__ dout, int ocs,
                   __nv_bfloat16* __restrict__ din, int dcs, int N, int C8, int H, int W, int P, int Q) {
    const int HB = (H + 1) / 2, WB = (W + 1) / 2;
    const long long total = (long long)N * HB * WB * C8;
    const long long stride_ = (long long)gridDim.x * kThreads;
    VecWalk wk_(C8, (long long)blockIdx.x * kThreads + threadIdx.x, stride_);   // no 64-bit division per vector
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += stride_, wk_.next()) {
        const int c8 = wk_.c8;
        const long long blk = wk_.p;
        int b, a, n;
        split_pix(blk, WB, HB, b, a, n);
        uint2 pk[4];
        uint4 gv[4];
        bool ok[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {  // window (a + k/2, b + k%2)
            const int p = a + (k >> 1), q = b + (k & 1);
            ok[k] = (p < P) && (q < Q);
            const long long opix = ((long long)n * P + (ok[k] ? p : 0)) * Q + (ok[k] ? q : 0);
            pk[k] = __ldg(reinterpret_cast<const uint2*>(idx + opix * (long long)(C8 * 8) + c8 * 8));
            gv[k] = __ldg(reinterpret_cast<const uint4*>(dout + opix * ocs + c8 * 8));
        }
        float g[4][8];
#pragma unroll
        for (int k = 0; k < 4; ++k) unpack8(gv[k], g[k]);
#pragma unroll
        for (int dh = 0; dh < 2; ++dh) {
            const int h = 2 * a + dh;
            if (h >= H) continue;
#pragma unroll
            for (int dw = 0; dw < 2; ++dw) {
                const int w = 2 * b + dw;
                if (w >= W) continue;
                float acc[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    // pixel (h,w) lies in window (p,q) iff 2p-1 <= h <= 2p+1: dh=0 → only p=a; dh=1 → p in {a, a+1}
                    const int kp = k >> 1, kq = k & 1;
                    if ((kp == 1 && dh == 0) || (kq == 1 && dw == 0) || !ok[k]) continue;
                    const int p = a + kp, q = b + kq;
                    const uint32_t code = (uint32_t)((h - (2 * p - 1)) * 3 + (w - (2 * q - 1)));
#pragma unroll
                    for (int e = 0; e < 8; ++e) {
                        uint32_t am = ((e < 4 ? pk[k].x : pk[k].y) >> ((e & 3) * 8)) & 0xffu;
                        acc[e] += (am == code) ? g[k][e] : 0.f;
                    }
                }
                Vec8<__nv_bfloat16>::store(din + (((long long)n * H + h) * W + w) * dcs + c8 * 8, acc);
            }
        }
    }
}

template <typename A, typename B> struct SameT { static constexpr bool v = false; };
template <typename A> struct SameT<A, A> { static constexpr bool v = true; };


// S = 1 (global average pool: ARM / FFM / global-context squeezes, seg_oprs.py:200,223, bisenet network.py:35): the backward is
// a broadcast of dout[n, c] / (H·W) over the map. The generic kernel spends ~10 integer divisions per 16-byte vector on the bin
// search (ncu: 437 GB/s for a pure 71 MB write); this one is a plain vector store walk.
__global__ void __launch_bounds__(kThreads)
global_avgpool_bwd_kernel(const float* __restrict__ dout, int C8, long long hw, long long total, float inv_area,
                          __nv_bfloat16* __restrict__ din, int ics, int accumulate) {
    const long long stride_ = (long long)gridDim.x * kThreads;
    VecWalk wk_(C8, (long long)blockIdx.x * kThreads + threadIdx.x, stride_);
    for (long long idx = (long long)blockIdx.x * kThreads + threadIdx.x; idx < total; idx += stride_, wk_.next()) {
        const int c8 = wk_.c8;
        const long long pix = wk_.p;
        const long long n = pix / hw;
        float g[8];
        ldg8f(dout + (n * C8 + c8) * 8, g);
#pragma unroll
        for (int k = 0; k < 8; ++k) g[k] *= inv_area;
        __nv_bfloat16* dst = din + pix * ics + c8 * 8;
        if (accumulate) {
            float old[8];
            Vec8<__nv_bfloat16>::load(dst, old);
#pragma unroll
            for (int k = 0; k < 8; ++k) g[k] += old[k];
        }
        Vec8<__nv_bfloat16>::store(dst, g);
    }
}

}  // namespace

#define TSB_DT_OK(dt) ((dt) == TSB_F32 || (dt) == TSB_BF16)

extern "C" int tsb_bilinear_fwd(const void* in, int idtype, int ics, void* out, int odtype, int ocs, int N, int C,
                                int Hi, int Wi, int Ho, int Wo, tsb_stream_t stream) {
    TSB_REQUIRE(in && out, "tsb_bilinear_fwd: null pointer");
    TSB_REQUIRE(TSB_DT_OK(idtype) && TSB_DT_OK(odtype), "tsb_bilinear_fwd: bad dtype");
    TSB_REQUIRE(N > 0 && C > 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0 && ics >= C && ocs >= C, "tsb_bilinear_fwd: bad shape");
    cudaStream_t st = (cudaStream_t)stream;
    const bool vec = (C % 8 == 0) && (ics % 8 == 0) && (ocs % 8 == 0) && tsb_aligned16(in) && tsb_aligned16(out);
    if (vec) {
        long long total = (long long)N * Ho * Wo * (C / 8);
        int grid = tsb_grid_for(total, kThreads, 8);
#define L(TI, TO) bilinear_fwd_kernel<TI, TO><<<grid, kThreads, 0, st>>>((const TI*)in, ics, (TO*)out, ocs, N, C / 8, Hi, Wi, Ho, Wo)
        if (idtype == TSB_BF16 && odtype == TSB_BF16) L(__nv_bfloat16, __nv_bfloat16);
        else if (idtype == TSB_BF16 && odtype == TSB_F32) L(__nv_bfloat16, float);
        else if (idtype == TSB_F32 && odtype == TSB_BF16) L(float, __nv_bfloat16);
        else L(float, float);
#undef L
    } else {
        long long total = (long long)N * Ho * Wo * C;
        int grid = tsb_grid_for(total, kThreads, 8);
#define L(TI, TO) bilinear_fwd_scalar_kernel<TI, TO, false><<<grid, kThreads, 0, st>>>((const TI*)in, ics, (TO*)out, ocs, N, C, Hi, Wi, Ho, Wo)
        if (idtype == TSB_BF16 && odtype == TSB_BF16) L(__nv_bfloat16, __nv_bfloat16);
        else if (idtype == TSB_BF16 && odtype == TSB_F32) L(__nv_bfloat16, float);
        else if (idtype == TSB_F32 && odtype == TSB_BF16) L(float, __nv_bfloat16);
        else L(float, float);
#undef L
    }
    TSB_CUDA_CHECK_LAUNCH("bilinear_fwd");
    return TSB_OK;
}

extern "C" int tsb_bilinear_fwd_nhwc_to_nchw(const void* in, int idtype, int ics, float* out, int N, int C, int Hi,
                                             int Wi, int Ho, int Wo, tsb_stream_t stream) {
    TSB_REQUIRE(in && out && TSB_DT_OK(idtype), "tsb_bilinear_fwd_nhwc_to_nchw: bad args");
    long long total = (long long)N * Ho * Wo * C;
    int grid = tsb_grid_for(total, kThreads, 8);
    cudaStream_t st = (cudaStream_t)stream;
    if (idtype == TSB_BF16)
        bilinear_fwd_scalar_kernel<__nv_bfloat16, float, true><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)in, ics, out, 0, N, C, Hi, Wi, Ho, Wo);
    else
        bilinear_fwd_scalar_kernel<float, float, true><<<grid, kThreads, 0, st>>>((const float*)in, ics, out, 0, N, C, Hi, Wi, Ho, Wo);
    TSB_CUDA_CHECK_LAUNCH("bilinear_fwd_nhwc_to_nchw");
    return TSB_OK;
}

extern "C" int tsb_bilinear_bwd(const void* dout, int odtype, int ocs, void* din, int idtype, int ics, int N, int C,
                                int Hi, int Wi, int Ho, int Wo, int accumulate, tsb_stream_t stream) {
    TSB_REQUIRE(dout && din && TSB_DT_OK(idtype) && TSB_DT_OK(odtype), "tsb_bilinear_bwd: bad args");
    TSB_REQUIRE((C % 8 == 0) && (ics % 8 == 0) && (ocs % 8 == 0) && tsb_aligned16(dout) && tsb_aligned16(din),
                "tsb_bilinear_bwd: C and channel strides must be multiples of 8, pointers 16B aligned");
    long long total = (long long)N * Hi * Wi * (C / 8);
    int grid = tsb_grid_for(total, kThreads, 8);
    cudaStream_t st = (cudaStream_t)stream;
#define L(TO, TI) bilinear_bwd_kernel<TO, TI><<<grid, kThreads, 0, st>>>((const TO*)dout, ocs, (TI*)din, ics, N, C / 8, Hi, Wi, Ho, Wo, accumulate)
    if (odtype == TSB_BF16 && idtype == TSB_BF16) L(__nv_bfloat16, __nv_bfloat16);
    else if (odtype == TSB_BF16 && idtype == TSB_F32) L(__nv_bfloat16, float);
    else if (odtype == TSB_F32 && idtype == TSB_BF16) L(float, __nv_bfloat16);
    else L(float, float);
#undef L
    TSB_CUDA_CHECK_LAUNCH("bilinear_bwd");
    return TSB_OK;
}

extern "C" int tsb_adaptive_avgpool_fwd(const void* in, int ics, int N, int C, int H, int W, int S, float* out, float* ws,
                                        long long ws_floats, tsb_stream_t stream) {
    TSB_REQUIRE(in && out, "tsb_adaptive_avgpool_fwd: null pointer");
    TSB_REQUIRE(C % 8 == 0 && ics % 8 == 0 && tsb_aligned16(in), "tsb_adaptive_avgpool_fwd: C, ics must be multiples of 8");
    TSB_REQUIRE(S >= 1 && S <= H && S <= W, "tsb_adaptive_avgpool_fwd: bad S");
    cudaStream_t st = (cudaStream_t)stream;
    TSB_CUDA_CALL(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)N * S * S * C, st));
    const int bins = N * S * S;
    const int max_bin_pix = ((H + S - 1) / S + 1) * ((W + S - 1) / S + 1);
    int chunks = (2 * tsb_num_sms() + bins - 1) / bins;
    const int C8 = C / 8;
    const int groups = C8 < kThreads ? C8 : kThreads;
    const int lanes = kThreads / groups;
    int max_chunks = (max_bin_pix + lanes * 4 - 1) / (lanes * 4);
    if (chunks > max_chunks) chunks = max_chunks;
    if (chunks < 1) chunks = 1;
    size_t smem = sizeof(float) * (size_t)lanes * groups * 8;
    TSB_REQUIRE(ws && (long long)chunks * bins * C <= ws_floats, "tsb_adaptive_avgpool_fwd: workspace needs %lld floats",
                (long long)chunks * bins * C);
    adaptive_avgpool_fwd_kernel<<<dim3(bins, chunks), kThreads, smem, st>>>((const __nv_bfloat16*)in, ics, N, C, H, W, S, ws);
    TSB_CUDA_CHECK_LAUNCH("adaptive_avgpool_fwd");
    return tsb_det_reduce(out, ws, chunks, (long long)bins * C, (long long)bins * C, st);
}

extern "C" int tsb_adaptive_avgpool_bwd(const float* dout, int N, int C, int H, int W, int S, void* din, int ics,
                                        int accumulate, tsb_stream_t stream) {
    TSB_REQUIRE(dout && din, "tsb_adaptive_avgpool_bwd: null pointer");
    TSB_REQUIRE(C % 8 == 0 && ics % 8 == 0 && tsb_aligned16(din) && tsb_aligned16(dout), "tsb_adaptive_avgpool_bwd: C, ics multiples of 8");
    long long total = (long long)N * H * W * (C / 8);
    int grid = tsb_grid_for(total, kThreads, 8);
    if (S == 1) {
        global_avgpool_bwd_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(dout, C / 8, (long long)H * W, total, 1.0f / (float)(H * W),
                                                                               (__nv_bfloat16*)din, ics, accumulate);
        TSB_CUDA_CHECK_LAUNCH("global_avgpool_bwd");
        return TSB_OK;
    }
    adaptive_avgpool_bwd_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(dout, N, C / 8, H, W, S, (__nv_bfloat16*)din, ics, accumulate);
    TSB_CUDA_CHECK_LAUNCH("adaptive_avgpool_bwd");
    return TSB_OK;
}

extern "C" int tsb_maxpool3x3s2_fwd(const void* in, int ics, void* out, int ocs, void* argmax, int N, int C, int H,
                                    int W, tsb_stream_t stream) {
    TSB_REQUIRE(in && out && C % 8 == 0 && ics % 8 == 0 && ocs % 8 == 0, "tsb_maxpool3x3s2_fwd: bad args");
    const int P = (H + 2 - 3) / 2 + 1, Q = (W + 2 - 3) / 2 + 1;
    long long total = (long long)N * P * Q * (C / 8);
    int grid = tsb_grid_for(total, kThreads, 8);
    maxpool_fwd_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)in, ics, (__nv_bfloat16*)out, ocs, (uint8_t*)argmax, N, C / 8, H, W, P, Q);
    TSB_CUDA_CHECK_LAUNCH("maxpool_fwd");
    return TSB_OK;
}

extern "C" int tsb_maxpool3x3s2_bwd(const void* argmax, const void* dout, int ocs, void* din, int dcs, int N, int C,
                                    int H, int W, tsb_stream_t stream) {
    TSB_REQUIRE(argmax && dout && din && C % 8 == 0 && ocs % 8 == 0 && dcs % 8 == 0, "tsb_maxpool3x3s2_bwd: bad args");
    const int P = (H + 2 - 3) / 2 + 1, Q = (W + 2 - 3) / 2 + 1;
    long long total = (long long)N * ((H + 1) / 2) * ((W + 1) / 2) * (C / 8);
    int grid = tsb_grid_for(total, kThreads, 8);
    maxpool_bwd_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>((const uint8_t*)argmax, (const __nv_bfloat16*)dout, ocs, (__nv_bfloat16*)din, dcs, N, C / 8, H, W, P, Q);
    TSB_CUDA_CHECK_LAUNCH("maxpool_bwd");
    return TSB_OK;
}
