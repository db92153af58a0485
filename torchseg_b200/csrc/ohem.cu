// OHEM cross-entropy for sm_90a — replaces ProbOhemCrossEntropy2d.forward
// (TorchSeg furnace/seg_opr/loss_opr.py:68-98).  HBM-bound byte work: coalesced loads,
// warp-shuffle / shared-memory histogram reductions, an exact radix *select* instead of the full sort.
#include "tsb_common.cuh"
#include "band.cuh"

namespace {
using namespace band;

constexpr int kThreads = 256;
constexpr int ST_HIST = 0;  // 4096 bins
constexpr int ST_NUM_VALID = TSB_OHEM_ST_NUM_VALID;
constexpr int ST_COUNT_LE = TSB_OHEM_ST_COUNT_LE;
constexpr int ST_ACTIVE = TSB_OHEM_ST_ACTIVE;
constexpr int ST_THRESH = TSB_OHEM_ST_THRESH;
constexpr int ST_KEPT = TSB_OHEM_ST_KEPT;
constexpr int ST_LOSS = TSB_OHEM_ST_LOSS;
constexpr int ST_INVDEN = TSB_OHEM_ST_INVDEN;
constexpr int ST_DONE = 4103;
constexpr int ST_PREFIX = 4104;
constexpr int ST_KREM = 4105;
constexpr int ST_LOSS_SUM = 4108;  // double
constexpr int ST_W_SUM = 4110;     // double
constexpr int ST_KEPT_ACC = 4112;

// p_target + nll from the C logits of one pixel held in registers (C <= CMAX).
template <int CMAX>
__device__ __forceinline__ void softmax_target(const float (&x)[CMAX], int C, int t, float& p_t, float& nll) {
    float m = x[0];
#pragma unroll
    for (int c = 1; c < CMAX; ++c)
        if (c < C) m = fmaxf(m, x[c]);
    float s = 0.f, et = 0.f, xt = 0.f;
#pragma unroll
    for (int c = 0; c < CMAX; ++c) {
        if (c < C) {
            float e = tsb_exp_det(__fsub_rn(x[c], m));
            s = __fadd_rn(s, e);
            if (c == t) { et = e; xt = x[c]; }
        }
    }
    p_t = __fdiv_rn(et, s);
    nll = logf(s) - (xt - m);
}

// shared tail of the two p_target kernels: writes p/nll and counts num_valid / count(p <= thresh).
// The radix histogram is NOT built here: it is only needed when count(p<=thresh) < k (tsb_ohem_select then
// runs a level-0 histogram pass over p, 4 bytes/pixel), the common case skips it entirely.
struct PtAccum {
    unsigned int num_valid = 0, count_le = 0;
};
__device__ __forceinline__ void pt_emit(long long i, bool valid, float p_t, float nll_v, float thresh, float* p,
                                        float* nll, PtAccum& acc) {
    float pv = valid ? p_t : 1.0f;  // loss_opr.py:81 masked_fill_(~valid, 1) then gather of class 0
    p[i] = pv;
    nll[i] = valid ? nll_v : 0.f;
    acc.num_valid += valid ? 1u : 0u;
    acc.count_le += (pv <= thresh) ? 1u : 0u;
}
__device__ __forceinline__ void pt_flush(const PtAccum& acc, uint32_t* state, float* s_red) {
    float nv = block_sum<kThreads>((float)acc.num_valid, s_red);
    float cl = block_sum<kThreads>((float)acc.count_le, s_red);
    if (threadIdx.x == 0) {
        // per-block partial counts are < 2^24, exact in float
        atomicAdd(&state[ST_NUM_VALID], (unsigned int)nv);
        atomicAdd(&state[ST_COUNT_LE], (unsigned int)cl);
    }
}

template <typename T, int CMAX>
__global__ void __launch_bounds__(kThreads)
ohem_ptarget_kernel(const T* __restrict__ logits, long long sn, long long sc, long long sy, long long sx,
                    const int64_t* __restrict__ labels, int N, int C, int H, int W, int ignore_label, float thresh,
                    float* __restrict__ p, float* __restrict__ nll, uint32_t* state) {
    __shared__ float s_red[33];
    PtAccum acc;
    const long long total = (long long)N * H * W;
    const long long hw = (long long)H * W;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        int n = (int)(i / hw);
        long long r = i - (long long)n * hw;
        int y = (int)(r / W), x = (int)(r - (long long)y * W);
        long long lab = labels[i];
        bool valid = lab != (long long)ignore_label;
        int t = valid ? (int)lab : 0;
        const T* base = logits + n * sn + y * sy + x * sx;
        float v[CMAX];
#pragma unroll
        for (int c = 0; c < CMAX; ++c)
            if (c < C) v[c] = ld_as_float<T>(base + c * sc);
        float p_t, nl;
        softmax_target<CMAX>(v, C, t, p_t, nl);
        pt_emit(i, valid, p_t, nl, thresh, p, nll, acc);
    }
    pt_flush(acc, state, s_red);
}

// generic-C variant (C > 32, e.g. ADE 150 classes): two passes over the pixel's logits
template <typename T>
__global__ void __launch_bounds__(kThreads)
ohem_ptarget_kernel_anyc(const T* __restrict__ logits, long long sn, long long sc, long long sy, long long sx,
                         const int64_t* __restrict__ labels, int N, int C, int H, int W, int ignore_label,
                         float thresh, float* __restrict__ p, float* __restrict__ nll, uint32_t* state) {
    __shared__ float s_red[33];
    PtAccum acc;
    const long long total = (long long)N * H * W;
    const long long hw = (long long)H * W;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        int n = (int)(i / hw);
        long long r = i - (long long)n * hw;
        int y = (int)(r / W), x = (int)(r - (long long)y * W);
        long long lab = labels[i];
        bool valid = lab != (long long)ignore_label;
        int t = valid ? (int)lab : 0;
        const T* base = logits + n * sn + y * sy + x * sx;
        float m = ld_as_float<T>(base);
        for (int c = 1; c < C; ++c) m = fmaxf(m, ld_as_float<T>(base + c * sc));
        float s = 0.f, et = 0.f, xt = 0.f;
        for (int c = 0; c < C; ++c) {
            float xv = ld_as_float<T>(base + c * sc);
            float e = tsb_exp_det(__fsub_rn(xv, m));
            s = __fadd_rn(s, e);
            if (c == t) { et = e; xt = xv; }
        }
        float p_t = __fdiv_rn(et, s);
        float nl = logf(s) - (xt - m);
        pt_emit(i, valid, p_t, nl, thresh, p, nll, acc);
    }
    pt_flush(acc, state, s_red);
}

// ---------------------------------------------------------------------------------------------
// Fused bilinear-upsample kernels work on BANDS: CTA = (x-strip of kStrip hi-res columns, low-res row i,
// image n). All hi-res rows y with floor(ry*y) == i share the two low-res source rows (i, i1), which are
// staged once in shared memory together with the per-column lerp coefficients.
// ---------------------------------------------------------------------------------------------
constexpr int kStrip = 256;          // hi-res columns per CTA (== kThreads)
// low-res columns a strip can touch: kStrip*w/W + 3; the two staged source rows live in DYNAMIC shared memory
// sized by the host from the actual scale (s_lo[2][maxcols][CMAX])

template <int CMAX, bool kHoist>
__global__ void __launch_bounds__(kThreads, kHoist ? 2 : 1)
ohem_ptarget_up_kernel(const float* __restrict__ lo, int cs, int h, int w, const int64_t* __restrict__ labels, int N,
                       int C, int H, int W, int ignore_label, float thresh, float* __restrict__ p,
                       float* __restrict__ nll, uint32_t* state, int maxcols) {
    __shared__ float s_red[33];
    extern __shared__ float s_lo_dyn[];  // [2][maxcols][CMAX]: the two low-res source rows of this band
    PtAccum acc;
    const float ry = area_scale(h, H), rx = area_scale(w, W);
    const int n = blockIdx.z, ci = blockIdx.y, x0 = blockIdx.x * kStrip, x1 = min(W, x0 + kStrip);
    const int i1 = ci + (ci < h - 1 ? 1 : 0);
    const BandGeom g = band_geom(ry, rx, ci, x0, x1, H, w);
    if (g.ncols > maxcols) __trap();
    float* s_lo0 = s_lo_dyn;
    float* s_lo1 = s_lo_dyn + maxcols * CMAX;
    for (int q = threadIdx.x; q < 2 * g.ncols * C; q += kThreads) {
        int c = q % C, t2 = q / C, col = t2 % g.ncols, row = t2 / g.ncols;
        (row ? s_lo1 : s_lo0)[col * CMAX + c] = __ldg(lo + (((long long)n * h + (row ? i1 : ci)) * w + g.jbase + col) * cs + c);
    }
    __syncthreads();
    const int x = x0 + threadIdx.x;
    const bool xin = x < x1;
    const Lerp lx = make_lerp(rx, xin ? x : x0, w);
    const int j0 = lx.i0 - g.jbase, j1 = lx.i1 - g.jbase;
    float t0[CMAX], t1[CMAX];   // horizontally blended source rows of this thread's column (row-invariant)
#pragma unroll
    for (int c = 0; c < CMAX; ++c) {
        t0[c] = 0.f; t1[c] = 0.f;
        if (kHoist && c < C) {
            t0[c] = lerp_h(lx, s_lo0[j0 * CMAX + c], s_lo0[j1 * CMAX + c]);
            t1[c] = lerp_h(lx, s_lo1[j0 * CMAX + c], s_lo1[j1 * CMAX + c]);
        }
    }
    // software pipeline: the label of row y+1 is requested before row y is evaluated (the row body is ~900 issue
    // slots, enough to cover the global-load latency at 8-16 resident warps)
    long long lab_next = xin ? labels[((long long)n * H + g.y_lo) * W + x] : 0;
    for (int y = g.y_lo; y <= g.y_hi; ++y) {
        const long long lab = lab_next;
        if (xin && y < g.y_hi) lab_next = labels[((long long)n * H + y + 1) * W + x];
        const Lerp ly = make_lerp(ry, y, h);
        if (ly.i0 != ci || !xin) continue;  // uniform in y across the CTA
        const long long i = ((long long)n * H + y) * W + x;
        bool valid = lab != (long long)ignore_label;
        int t = valid ? (int)lab : 0;
        float v[CMAX];
#pragma unroll
        for (int c = 0; c < CMAX; ++c)
            if (c < C)
                v[c] = kHoist ? lerp_v(ly, t0[c], t1[c])
                              : lerp_v(ly, lerp_h(lx, s_lo0[j0 * CMAX + c], s_lo0[j1 * CMAX + c]),
                                       lerp_h(lx, s_lo1[j0 * CMAX + c], s_lo1[j1 * CMAX + c]));
        float p_t, nl;
        softmax_target<CMAX>(v, C, t, p_t, nl);
        pt_emit(i, valid, p_t, nl, thresh, p, nll, acc);
    }
    pt_flush(acc, state, s_red);
}

// ---------------------------------------------------------------------------------------------
// radix select: decide kernel (1 block of 1024 threads) + histogram kernels for levels 1 and 2
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) ohem_decide_kernel(uint32_t* state, long long n, long long min_kept,
                                                            float thresh, int level) {
    __shared__ unsigned long long s_warp[32];
    __shared__ int s_bin;
    __shared__ unsigned long long s_before;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (level < 0) {  // initial decision from the counters alone
        if (tid == 0) {
            unsigned int num_valid = state[ST_NUM_VALID];
            unsigned int count_le = state[ST_COUNT_LE];
            // loss_opr.py:78-85: skip when min_kept > num_valid; kept mask only if num_valid>0 and min_kept>0
            bool active = !((long long)min_kept > (long long)num_valid) && num_valid > 0 && min_kept > 0;
            long long k = min_kept < n ? min_kept : n;
            unsigned int done = 1;
            float T = thresh;
            if (active && (long long)count_le < k) done = 0;  // k-th smallest p exceeds thresh → need it
            state[ST_ACTIVE] = active ? 1u : 0u;
            state[ST_THRESH] = __float_as_uint(T);
            state[ST_DONE] = done;
            state[ST_PREFIX] = 0;
            state[ST_KREM] = (unsigned int)k;
        }
        return;
    }
    const bool done = state[ST_DONE] != 0;
    if (!done) {
        const unsigned int krem = state[ST_KREM];
        // each thread owns 4 consecutive bins
        unsigned int h0 = state[ST_HIST + tid * 4 + 0], h1 = state[ST_HIST + tid * 4 + 1];
        unsigned int h2 = state[ST_HIST + tid * 4 + 2], h3 = state[ST_HIST + tid * 4 + 3];
        unsigned long long mine = (unsigned long long)h0 + h1 + h2 + h3;
        unsigned long long incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) s_warp[wid] = incl;
        __syncthreads();
        if (wid == 0) {
            unsigned long long wv = s_warp[lane];
            unsigned long long wi = wv;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                unsigned long long v = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += v;
            }
            s_warp[lane] = wi - wv;  // exclusive prefix of warp totals
        }
        __syncthreads();
        unsigned long long excl = s_warp[wid] + incl - mine;  // elements strictly before my 4 bins
        if (excl < krem && excl + mine >= krem) {
            unsigned long long c = excl;
            int b = tid * 4;
            if (c + h0 >= krem) { b += 0; }
            else { c += h0; if (c + h1 >= krem) { b += 1; } else { c += h1; if (c + h2 >= krem) { b += 2; } else { c += h2; b += 3; } } }
            s_bin = b;
            s_before = c;
        }
        __syncthreads();
        if (tid == 0) {
            unsigned int prefix = state[ST_PREFIX];
            int b = s_bin;
            unsigned int newk = krem - (unsigned int)s_before;
            if (level < 2) {
                state[ST_PREFIX] = (level == 0) ? (unsigned int)b : ((prefix << 12) | (unsigned int)b);
                state[ST_KREM] = newk;
            } else {
                unsigned int bits = (prefix << 8) | (unsigned int)b;
                state[ST_THRESH] = bits;  // T = k-th smallest p (> thresh, loss_opr.py:88-89)
                state[ST_DONE] = 1;
            }
        }
    }
    __syncthreads();
    // leave a clean histogram for the next level / next use
    for (int b = tid; b < 4096; b += 1024) state[ST_HIST + b] = 0;
}

__global__ void __launch_bounds__(kThreads) ohem_hist_kernel(const float* __restrict__ p, long long n, uint32_t* state,
                                                              int level) {
    if (state[ST_DONE] != 0) return;
    __shared__ unsigned int s_hist[4096];
    for (int b = threadIdx.x; b < 4096; b += kThreads) s_hist[b] = 0;
    __syncthreads();
    const unsigned int prefix = state[ST_PREFIX];
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        unsigned int u = __float_as_uint(p[i]);
        if (level == 0) {
            unsigned int bin = u >> 20;
            atomicAdd(&s_hist[bin > 4095u ? 4095u : bin], 1u);
        } else if (level == 1) {
            if ((u >> 20) == prefix) atomicAdd(&s_hist[(u >> 8) & 0xfffu], 1u);
        } else {
            if ((u >> 8) == prefix) atomicAdd(&s_hist[u & 0xffu], 1u);
        }
    }
    __syncthreads();
    for (int b = threadIdx.x; b < 4096; b += kThreads) {
        unsigned int v = s_hist[b];
        if (v) atomicAdd(&state[ST_HIST + b], v);
    }
}

// ---------------------------------------------------------------------------------------------
// loss over kept pixels
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) ohem_loss_kernel(const float* __restrict__ p, const float* __restrict__ nll,
                                                              const int64_t* __restrict__ labels, long long n,
                                                              int ignore_label, const float* __restrict__ cw,
                                                              uint32_t* state) {
    __shared__ float s_red[33];
    const bool active = state[ST_ACTIVE] != 0;
    const float T = __uint_as_float(state[ST_THRESH]);
    float ls = 0.f, ws = 0.f, kc = 0.f;
    auto one = [&](long long lab, float pv, float nl) {
        const bool kept = (lab != (long long)ignore_label) && (!active || pv <= T);
        if (kept) {
            const float wt = cw ? __ldg(cw + (int)lab) : 1.f;
            ls += wt * nl;
            ws += wt;
            kc += 1.f;
        }
    };
    // four pixels per thread and trip: 2 x 16 B of labels + 16 B of p + 16 B of nll in flight per thread
    const long long n4 = n / 4;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(nll) | reinterpret_cast<uintptr_t>(labels)) & 15u) == 0;
    long long done = 0;
    if (vec_ok) {
        for (long long q = (long long)blockIdx.x * kThreads + threadIdx.x; q < n4; q += (long long)gridDim.x * kThreads) {
            const longlong2 l01 = *reinterpret_cast<const longlong2*>(labels + q * 4);
            const longlong2 l23 = *reinterpret_cast<const longlong2*>(labels + q * 4 + 2);
            const float4 pv = *reinterpret_cast<const float4*>(p + q * 4);
            const float4 nv = *reinterpret_cast<const float4*>(nll + q * 4);
            one(l01.x, pv.x, nv.x);
            one(l01.y, pv.y, nv.y);
            one(l23.x, pv.z, nv.z);
            one(l23.y, pv.w, nv.w);
        }
        done = n4 * 4;
    }
    for (long long i = done + (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads)
        one(labels[i], p[i], nll[i]);
    ls = block_sum<kThreads>(ls, s_red);
    ws = block_sum<kThreads>(ws, s_red);
    kc = block_sum<kThreads>(kc, s_red);
    if (threadIdx.x == 0) {
        atomicAdd(reinterpret_cast<double*>(state + ST_LOSS_SUM), (double)ls);
        atomicAdd(reinterpret_cast<double*>(state + ST_W_SUM), (double)ws);
        atomicAdd(&state[ST_KEPT_ACC], (unsigned int)kc);
    }
}
__global__ void ohem_finalize_kernel(uint32_t* state, float* loss_out) {
    double ls = *reinterpret_cast<double*>(state + ST_LOSS_SUM);
    double ws = *reinterpret_cast<double*>(state + ST_W_SUM);
    float loss = (float)(ls / ws);  // 0/0 → NaN, as CrossEntropyLoss over zero pixels
    state[ST_KEPT] = state[ST_KEPT_ACC];
    state[ST_LOSS] = __float_as_uint(loss);
    state[ST_INVDEN] = __float_as_uint((float)(1.0 / ws));
    if (loss_out) *loss_out = loss;
}

// ---------------------------------------------------------------------------------------------
// gradient, materialised logits
// ---------------------------------------------------------------------------------------------
template <typename T, int CMAX>
__global__ void __launch_bounds__(kThreads)
ohem_grad_kernel(const T* __restrict__ logits, long long sn, long long sc, long long sy, long long sx,
                 const int64_t* __restrict__ labels, const float* __restrict__ p, int N, int C, int H, int W,
                 int ignore_label, const float* __restrict__ cw, const uint32_t* __restrict__ state,
                 const float* __restrict__ gscale, T* __restrict__ dlogits) {
    const bool active = state[ST_ACTIVE] != 0;
    const float Tth = __uint_as_float(state[ST_THRESH]);
    const float scale = __uint_as_float(state[ST_INVDEN]) * (gscale ? *gscale : 1.f);
    const long long total = (long long)N * H * W;
    const long long hw = (long long)H * W;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        int n = (int)(i / hw);
        long long r = i - (long long)n * hw;
        int y = (int)(r / W), x = (int)(r - (long long)y * W);
        long long lab = labels[i];
        bool kept = (lab != (long long)ignore_label) && (!active || p[i] <= Tth);
        long long off = n * sn + y * sy + x * sx;
        if (!kept) {
            for (int c = 0; c < C; ++c) st_from_float<T>(dlogits + off + c * sc, 0.f);
            continue;
        }
        int t = (int)lab;
        float wt = (cw ? __ldg(cw + t) : 1.f) * scale;
        if (CMAX > 0) {
            float v[CMAX > 0 ? CMAX : 1];
            float m = -INFINITY;
#pragma unroll
            for (int c = 0; c < CMAX; ++c)
                if (c < C) { v[c] = ld_as_float<T>(logits + off + c * sc); m = fmaxf(m, v[c]); }
            float s = 0.f;
#pragma unroll
            for (int c = 0; c < CMAX; ++c)
                if (c < C) { v[c] = __expf(v[c] - m); s += v[c]; }
            float inv = 1.f / s;
#pragma unroll
            for (int c = 0; c < CMAX; ++c)
                if (c < C) st_from_float<T>(dlogits + off + c * sc, (v[c] * inv - (c == t ? 1.f : 0.f)) * wt);
        } else {
            float m = -INFINITY;
            for (int c = 0; c < C; ++c) m = fmaxf(m, ld_as_float<T>(logits + off + c * sc));
            float s = 0.f;
            for (int c = 0; c < C; ++c) s += __expf(ld_as_float<T>(logits + off + c * sc) - m);
            float inv = 1.f / s;
            for (int c = 0; c < C; ++c) {
                float e = __expf(ld_as_float<T>(logits + off + c * sc) - m);
                st_from_float<T>(dlogits + off + c * sc, (e * inv - (c == t ? 1.f : 0.f)) * wt);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// gradient, fused-upsample form (band structure as above).  Per hi-res row of the band:
//   phase 1: thread x computes g[c] = (softmax_c - onehot_c) * w_t * scale for its pixel → smem s_g[c][x]
//   phase 2: thread (j,c) forms s = Σ_x wx(x,j) g[c][x] over the <= ~2*scale columns that touch low-res
//            column j and accumulates top += l0(y)*s, bot += l1(y)*s in registers.
// After the band: red.global.add of top → row i, bot → row i1.  No shuffles, no per-pixel atomics.
// ---------------------------------------------------------------------------------------------
template <int CMAX, bool kHoist>
__global__ void __launch_bounds__(kThreads, kHoist ? 2 : 1)
ohem_grad_up_kernel(const float* __restrict__ lo, int cs, int h, int w, const int64_t* __restrict__ labels,
                    const float* __restrict__ p, int N, int C, int H, int W, int ignore_label,
                    const float* __restrict__ cw, const uint32_t* __restrict__ state,
                    const float* __restrict__ gscale, float* __restrict__ dlo, int maxcols) {
    constexpr int kPitch = kStrip + 1;  // odd pitch → conflict-free column walks in phase 2
    extern __shared__ float s_dyn[];    // s_g0[CMAX][kPitch], s_g1[CMAX][kPitch], s_lo[2][maxcols][CMAX]
    float (*s_g0)[kPitch] = reinterpret_cast<float (*)[kPitch]>(s_dyn);
    float (*s_g1)[kPitch] = reinterpret_cast<float (*)[kPitch]>(s_dyn + CMAX * kPitch);
    float* s_lo0 = s_dyn + 2 * CMAX * kPitch;
    float* s_lo1 = s_lo0 + maxcols * CMAX;
    __shared__ float s_l0[kStrip], s_l1[kStrip];
    __shared__ short s_seg[kStrip + 8];  // s_seg[j] = first strip column whose left stencil column is >= j
    const bool active = state[ST_ACTIVE] != 0;
    const float Tth = __uint_as_float(state[ST_THRESH]);
    const float scale = __uint_as_float(state[ST_INVDEN]) * (gscale ? *gscale : 1.f);
    const float ry = area_scale(h, H), rx = area_scale(w, W);
    const int n = blockIdx.z, ci = blockIdx.y, x0 = blockIdx.x * kStrip, x1 = min(W, x0 + kStrip);
    const int nx = x1 - x0;
    const int i1 = ci + (ci < h - 1 ? 1 : 0);
    const BandGeom g = band_geom(ry, rx, ci, x0, x1, H, w);
    if (g.ncols > maxcols) __trap();
    for (int q = threadIdx.x; q < 2 * g.ncols * C; q += kThreads) {
        int c = q % C, t2 = q / C, col = t2 % g.ncols, row = t2 / g.ncols;
        (row ? s_lo1 : s_lo0)[col * CMAX + c] = __ldg(lo + (((long long)n * h + (row ? i1 : ci)) * w + g.jbase + col) * cs + c);
    }
    const int x = x0 + threadIdx.x;
    const bool xin = x < x1;
    const Lerp lx = make_lerp(rx, xin ? x : x0, w);
    const int j0 = lx.i0 - g.jbase, j1 = lx.i1 - g.jbase;
    s_l0[threadIdx.x] = xin ? lx.l0 : 0.f;
    s_l1[threadIdx.x] = xin ? lx.l1 : 0.f;
    // segment starts: columns with left stencil index j form the contiguous range [s_seg[j], s_seg[j+1])
    for (int q = threadIdx.x; q < g.ncols + 2; q += kThreads) s_seg[q] = (short)nx;
    __syncthreads();
    if (xin) {
        const int jprev = (threadIdx.x == 0) ? -1 : (make_lerp(rx, x - 1, w).i0 - g.jbase);
        for (int jj = jprev + 1; jj <= j0; ++jj) s_seg[jj] = (short)threadIdx.x;
    }
    // ---- phase 1: per-thread accumulation over the rows of the band (registers only)
    float G0[CMAX], G1[CMAX], t0[CMAX], t1[CMAX];
#pragma unroll
    for (int c = 0; c < CMAX; ++c) {
        G0[c] = 0.f; G1[c] = 0.f; t0[c] = 0.f; t1[c] = 0.f;
        if (kHoist && c < C && xin) {   // horizontally blended source rows: row-invariant, formed once per band
            t0[c] = lerp_h(lx, s_lo0[j0 * CMAX + c], s_lo0[j1 * CMAX + c]);
            t1[c] = lerp_h(lx, s_lo1[j0 * CMAX + c], s_lo1[j1 * CMAX + c]);
        }
    }
    // software pipeline: label and p of row y+1 are requested before row y is evaluated
    long long lab_next = 0;
    float p_next = 0.f;
    if (xin) {
        const long long q0 = ((long long)n * H + g.y_lo) * W + x;
        lab_next = labels[q0];
        p_next = active ? p[q0] : 0.f;
    }
    for (int y = g.y_lo; y <= g.y_hi; ++y) {
        const long long lab = lab_next;
        const float pv = p_next;
        if (xin && y < g.y_hi) {
            const long long q1 = ((long long)n * H + y + 1) * W + x;
            lab_next = labels[q1];
            p_next = active ? p[q1] : 0.f;
        }
        const Lerp ly = make_lerp(ry, y, h);
        if (ly.i0 != ci || !xin) continue;
        const bool kept = (lab != (long long)ignore_label) && (!active || pv <= Tth);
        if (!kept) continue;
        const int t = (int)lab;
        const float wt = (cw ? __ldg(cw + t) : 1.f) * scale;
        float v[CMAX];
        float m = -INFINITY;
#pragma unroll
        for (int c = 0; c < CMAX; ++c)
            if (c < C) {
                v[c] = kHoist ? lerp_v(ly, t0[c], t1[c])
                              : lerp_v(ly, lerp_h(lx, s_lo0[j0 * CMAX + c], s_lo0[j1 * CMAX + c]),
                                       lerp_h(lx, s_lo1[j0 * CMAX + c], s_lo1[j1 * CMAX + c]));
                m = fmaxf(m, v[c]);
            }
        float ssum = 0.f;
#pragma unroll
        for (int c = 0; c < CMAX; ++c)
            if (c < C) { v[c] = __expf(v[c] - m); ssum += v[c]; }
        const float inv = wt / ssum;
#pragma unroll
        for (int c = 0; c < CMAX; ++c)
            if (c < C) {
                const float gg = v[c] * inv - (c == t ? wt : 0.f);
                G0[c] = fmaf(ly.l0, gg, G0[c]);
                G1[c] = fmaf(ly.l1, gg, G1[c]);
            }
    }
#pragma unroll
    for (int c = 0; c < CMAX; ++c)
        if (c < C) { s_g0[c][threadIdx.x] = G0[c]; s_g1[c][threadIdx.x] = G1[c]; }
    __syncthreads();
    // ---- phase 2 (once per band): low-res column j receives the l0x-weighted sum of its own segment and the
    //      l1x-weighted sum of the previous segment (or of its own when the stencil is clamped at the last column)
    const int npairs = g.ncols * C;
    for (int q = threadIdx.x; q < npairs; q += kThreads) {
        const int j = q / C, c = q - j * C;
        const int a0 = s_seg[j], a1 = s_seg[j + 1];
        float top = 0.f, bot = 0.f;
        for (int xx = a0; xx < a1; ++xx) {
            const float wl = s_l0[xx];
            top = fmaf(wl, s_g0[c][xx], top);
            bot = fmaf(wl, s_g1[c][xx], bot);
        }
        const bool clamped = (g.jbase + j == w - 1);
        const int b0 = clamped ? a0 : (j > 0 ? (int)s_seg[j - 1] : 0);
        const int b1 = clamped ? a1 : (j > 0 ? a0 : 0);
        for (int xx = b0; xx < b1; ++xx) {
            const float wr = s_l1[xx];
            top = fmaf(wr, s_g0[c][xx], top);
            bot = fmaf(wr, s_g1[c][xx], bot);
        }
        if (clamped && j > 0) {  // the previous segment still points at this (last) column with its right weight
            for (int xx = s_seg[j - 1]; xx < a0; ++xx) {
                const float wr = s_l1[xx];
                top = fmaf(wr, s_g0[c][xx], top);
                bot = fmaf(wr, s_g1[c][xx], bot);
            }
        }
        if (top != 0.f) atomicAdd(dlo + (((long long)n * h + ci) * w + g.jbase + j) * cs + c, top);
        if (bot != 0.f) atomicAdd(dlo + (((long long)n * h + i1) * w + g.jbase + j) * cs + c, bot);
    }
}


// =============================================================================================
// Exact-class-count band kernels (CX = 19 Cityscapes, 21 VOC): second generation of the fused-upsample pair.
// ncu (profiles/r02_hot): the generic p_target kernel was ISSUE bound at 1005 warp-instructions per pixel, 40 % of them
// run-time `c < C` guards, `c == t` selects, the branch inside exp_det and the four-tap blend redone for every row; the
// gradient kernel ran at 54 % issue utilisation with 128 registers (2 CTAs / SM) and 105 ISETP per pixel.
//   * CX is a compile-time constant: no class guards, full unrolling;
//   * the horizontally blended source rows T0/T1[c][x] (row-invariant) are staged ONCE per band in shared memory, each
//     thread in its own column (no synchronisation): a row costs 2 LDS + 3 flops per class instead of 4 LDS + 9;
//   * the target class is fetched by ONE dynamic shared-memory read pair (its exp is recomputed: bit-identical, same
//     inputs) instead of CX compare-selects;
//   * gradient: softmax minus one-hot accumulates in the thread's own registers, and the bands run in four (row parity,
//     strip parity) launches that add to the low-res gradient without atomics: the gradient is the same on every run;
//     the accumulators' hand-over to phase 2 re-uses the T arrays in place (thread-private
//     columns), which leaves ~80 registers and 3 CTAs / SM.
// Arithmetic (operation order, roundings) is unchanged: p, T and the kept set stay bit-exact against the oracle.
// =============================================================================================
constexpr int kPitchX = kStrip + 1;

template <int CX>
__global__ void __launch_bounds__(kThreads, 3)
ohem_ptarget_up_x_kernel(const float* __restrict__ lo, int cs, int h, int w, const int64_t* __restrict__ labels, int N,
                         int H, int W, int ignore_label, float thresh, float* __restrict__ p, float* __restrict__ nll,
                         uint32_t* state, int maxcols) {
    __shared__ float s_red[33];
    extern __shared__ float s_dyn_x[];           // sT0[CX][kPitchX] | sT1[CX][kPitchX] | s_lo0[maxcols][CX] | s_lo1[...]
    float* sT0 = s_dyn_x;
    float* sT1 = s_dyn_x + CX * kPitchX;
    float* s_lo0 = s_dyn_x + 2 * CX * kPitchX;
    float* s_lo1 = s_lo0 + maxcols * CX;
    PtAccum acc;
    const float ry = area_scale(h, H), rx = area_scale(w, W);
    const int n = blockIdx.z, ci = blockIdx.y, x0 = blockIdx.x * kStrip, x1 = min(W, x0 + kStrip);
    const int i1 = ci + (ci < h - 1 ? 1 : 0);
    const BandGeom g = band_geom(ry, rx, ci, x0, x1, H, w);
    if (g.ncols > maxcols) __trap();
    for (int q = threadIdx.x; q < 2 * g.ncols * CX; q += kThreads) {
        const int c = q % CX, t2 = q / CX, col = t2 % g.ncols, row = t2 / g.ncols;
        (row ? s_lo1 : s_lo0)[col * CX + c] = __ldg(lo + (((long long)n * h + (row ? i1 : ci)) * w + g.jbase + col) * cs + c);
    }
    __syncthreads();
    const int tid = threadIdx.x;
    const int x = x0 + tid;
    const bool xin = x < x1;
    const Lerp lx = make_lerp(rx, xin ? x : x0, w);
    const int j0 = lx.i0 - g.jbase, j1 = lx.i1 - g.jbase;
#pragma unroll
    for (int c = 0; c < CX; ++c) {
        sT0[c * kPitchX + tid] = lerp_h(lx, s_lo0[j0 * CX + c], s_lo0[j1 * CX + c]);
        sT1[c * kPitchX + tid] = lerp_h(lx, s_lo1[j0 * CX + c], s_lo1[j1 * CX + c]);
    }
    long long lab_next = xin ? labels[((long long)n * H + g.y_lo) * W + x] : 0;
    for (int y = g.y_lo; y <= g.y_hi; ++y) {
        const long long lab = lab_next;
        if (xin && y < g.y_hi) lab_next = labels[((long long)n * H + y + 1) * W + x];
        const Lerp ly = make_lerp(ry, y, h);
        if (ly.i0 != ci || !xin) continue;  // uniform in y across the CTA
        const long long i = ((long long)n * H + y) * W + x;
        const bool valid = lab != (long long)ignore_label;
        const int t = valid ? (int)lab : 0;
        float v[CX];
#pragma unroll
        for (int c = 0; c < CX; ++c) v[c] = lerp_v(ly, sT0[c * kPitchX + tid], sT1[c * kPitchX + tid]);
        float m = v[0];
#pragma unroll
        for (int c = 1; c < CX; ++c) m = fmaxf(m, v[c]);
        float ssum = 0.f;
#pragma unroll
        for (int c = 0; c < CX; ++c) ssum = __fadd_rn(ssum, tsb_exp_det(__fsub_rn(v[c], m)));
        // target class: same operands, same operations as v[t] above → identical bits
        const float xt = lerp_v(ly, sT0[t * kPitchX + tid], sT1[t * kPitchX + tid]);
        const float et = tsb_exp_det(__fsub_rn(xt, m));
        const float p_t = __fdiv_rn(et, ssum);
        const float nl = logf(ssum) - (xt - m);
        pt_emit(i, valid, p_t, nl, thresh, p, nll, acc);
    }
    pt_flush(acc, state, s_red);
}

template <int CX>
__global__ void __launch_bounds__(kThreads, 3)
ohem_grad_up_x_kernel(const float* __restrict__ lo, int cs, int h, int w, const int64_t* __restrict__ labels,
                      const float* __restrict__ p, int N, int H, int W, int ignore_label, const float* __restrict__ cw,
                      const uint32_t* __restrict__ state, const float* __restrict__ gscale, float* __restrict__ dlo,
                      int maxcols, int phase) {
    extern __shared__ float s_dyn_x[];   // sT0 / s_g0 [CX][kPitchX] | sT1 / s_g1 | s_lo0 | s_lo1
    float* sT0 = s_dyn_x;
    float* sT1 = s_dyn_x + CX * kPitchX;
    float* s_lo0 = s_dyn_x + 2 * CX * kPitchX;
    float* s_lo1 = s_lo0 + maxcols * CX;
    __shared__ float s_l0[kStrip], s_l1[kStrip];
    __shared__ short s_seg[kStrip + 8];
    const bool active = state[ST_ACTIVE] != 0;
    const float Tth = __uint_as_float(state[ST_THRESH]);
    const float scale = __uint_as_float(state[ST_INVDEN]) * (gscale ? *gscale : 1.f);
    const float ry = area_scale(h, H), rx = area_scale(w, W);
    // launch `phase` (0..3) runs the bands of one (row parity, strip parity): bands of one launch never add to the same
    // low-res cell, and the four launches run in a fixed order, so every cell is summed in the same order on every run
    const int n = blockIdx.z, ci = 2 * blockIdx.y + (phase & 1), x0 = (2 * blockIdx.x + (phase >> 1)) * kStrip;
    if (ci >= h || x0 >= W) return;
    const int x1 = min(W, x0 + kStrip);
    const int nx = x1 - x0;
    const int i1 = ci + (ci < h - 1 ? 1 : 0);
    const BandGeom g = band_geom(ry, rx, ci, x0, x1, H, w);
    if (g.ncols > maxcols) __trap();
    for (int q = threadIdx.x; q < 2 * g.ncols * CX; q += kThreads) {
        const int c = q % CX, t2 = q / CX, col = t2 % g.ncols, row = t2 / g.ncols;
        (row ? s_lo1 : s_lo0)[col * CX + c] = __ldg(lo + (((long long)n * h + (row ? i1 : ci)) * w + g.jbase + col) * cs + c);
    }
    const int tid = threadIdx.x;
    const int x = x0 + tid;
    const bool xin = x < x1;
    const Lerp lx = make_lerp(rx, xin ? x : x0, w);
    const int j0 = lx.i0 - g.jbase, j1 = lx.i1 - g.jbase;
    s_l0[tid] = xin ? lx.l0 : 0.f;
    s_l1[tid] = xin ? lx.l1 : 0.f;
    for (int q = tid; q < g.ncols + 2; q += kThreads) s_seg[q] = (short)nx;
    __syncthreads();
    if (xin) {
        const int jprev = (tid == 0) ? -1 : (make_lerp(rx, x - 1, w).i0 - g.jbase);
        for (int jj = jprev + 1; jj <= j0; ++jj) s_seg[jj] = (short)tid;
    }
#pragma unroll
    for (int c = 0; c < CX; ++c) {
        sT0[c * kPitchX + tid] = lerp_h(lx, s_lo0[j0 * CX + c], s_lo0[j1 * CX + c]);
        sT1[c * kPitchX + tid] = lerp_h(lx, s_lo1[j0 * CX + c], s_lo1[j1 * CX + c]);
    }
    // ---- phase 1: per-thread accumulation over the rows of the band
    float G0[CX], G1[CX];
#pragma unroll
    for (int c = 0; c < CX; ++c) { G0[c] = 0.f; G1[c] = 0.f; }
    long long lab_next = 0;
    float p_next = 0.f;
    if (xin) {
        const long long q0 = ((long long)n * H + g.y_lo) * W + x;
        lab_next = labels[q0];
        p_next = active ? p[q0] : 0.f;
    }
    for (int y = g.y_lo; y <= g.y_hi; ++y) {
        const long long lab = lab_next;
        const float pv = p_next;
        if (xin && y < g.y_hi) {
            const long long q1 = ((long long)n * H + y + 1) * W + x;
            lab_next = labels[q1];
            p_next = active ? p[q1] : 0.f;
        }
        const Lerp ly = make_lerp(ry, y, h);
        if (ly.i0 != ci || !xin) continue;
        const bool kept = (lab != (long long)ignore_label) && (!active || pv <= Tth);
        if (!kept) continue;
        const int t = (int)lab;
        const float wt = (cw ? __ldg(cw + t) : 1.f) * scale;
        float v[CX];
#pragma unroll
        for (int c = 0; c < CX; ++c) v[c] = lerp_v(ly, sT0[c * kPitchX + tid], sT1[c * kPitchX + tid]);
        float m = v[0];
#pragma unroll
        for (int c = 1; c < CX; ++c) m = fmaxf(m, v[c]);
        float ssum = 0.f;
#pragma unroll
        for (int c = 0; c < CX; ++c) { v[c] = __expf(v[c] - m); ssum += v[c]; }
        const float inv = wt / ssum;
#pragma unroll
        for (int c = 0; c < CX; ++c) {
            // softmax minus one-hot, in this thread's own accumulators: the column sums of phase 2 add them in a fixed
            // order (shared-memory atomics would make the gradient's rounding vary from run to run)
            const float gg = v[c] * inv - (c == t ? wt : 0.f);
            G0[c] = fmaf(ly.l0, gg, G0[c]);
            G1[c] = fmaf(ly.l1, gg, G1[c]);
        }
    }
    // hand-over to phase 2 in place: column `tid` of sT0 / sT1 was only ever read by this thread
#pragma unroll
    for (int c = 0; c < CX; ++c) { sT0[c * kPitchX + tid] = G0[c]; sT1[c * kPitchX + tid] = G1[c]; }
    __syncthreads();
    // ---- phase 2 (once per band): low-res column j receives the l0x-weighted sum of its own segment and the
    //      l1x-weighted sum of the previous segment (or of its own when the stencil is clamped at the last column)
    const int npairs = g.ncols * CX;
    for (int q = tid; q < npairs; q += kThreads) {
        const int j = q / CX, c = q - j * CX;
        const float* g0 = sT0 + c * kPitchX;
        const float* g1 = sT1 + c * kPitchX;
        const int a0 = s_seg[j], a1 = s_seg[j + 1];
        float top = 0.f, bot = 0.f;
        for (int xx = a0; xx < a1; ++xx) {
            const float wl = s_l0[xx];
            top = fmaf(wl, g0[xx], top);
            bot = fmaf(wl, g1[xx], bot);
        }
        const bool clamped = (g.jbase + j == w - 1);
        const int b0 = clamped ? a0 : (j > 0 ? (int)s_seg[j - 1] : 0);
        const int b1 = clamped ? a1 : (j > 0 ? a0 : 0);
        for (int xx = b0; xx < b1; ++xx) {
            const float wr = s_l1[xx];
            top = fmaf(wr, g0[xx], top);
            bot = fmaf(wr, g1[xx], bot);
        }
        if (clamped && j > 0) {
            for (int xx = s_seg[j - 1]; xx < a0; ++xx) {
                const float wr = s_l1[xx];
                top = fmaf(wr, g0[xx], top);
                bot = fmaf(wr, g1[xx], bot);
            }
        }
        if (top != 0.f) dlo[(((long long)n * h + ci) * w + g.jbase + j) * cs + c] += top;
        if (bot != 0.f) dlo[(((long long)n * h + i1) * w + g.jbase + j) * cs + c] += bot;
    }
}

}  // namespace

// A/B switch (tsb_debug_set key 6): band kernels keep the horizontally blended source rows in registers; bit 0 =
// gradient kernel (measured 2.16 -> 1.85 ms/step), bit 1 = p_target kernel (measured slower: 111 registers halve the
// occupancy of an issue-bound kernel, 1.72 -> 1.85 ms) — default 1.
int g_tsb_ohem_hoist = 1;
int g_tsb_ohem_exact = 1;   // tsb_debug_set key 10: exact-class-count band kernels (C = 19 / 21)

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" int tsb_ohem_begin(uint32_t* state, tsb_stream_t stream) {
    TSB_REQUIRE(state != nullptr, "tsb_ohem_begin: null state");
    TSB_CUDA_CALL(cudaMemsetAsync(state, 0, sizeof(uint32_t) * TSB_OHEM_STATE_WORDS, (cudaStream_t)stream));
    return TSB_OK;
}

extern "C" int tsb_ohem_ptarget(const void* logits, int dtype, long long sn, long long sc, long long sy, long long sx,
                                const int64_t* labels, int N, int C, int H, int W, int ignore_label, float thresh,
                                float* p, float* nll, uint32_t* state, tsb_stream_t stream) {
    TSB_REQUIRE(logits && labels && p && nll && state, "tsb_ohem_ptarget: null pointer");
    TSB_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0, "tsb_ohem_ptarget: bad shape");
    TSB_REQUIRE(dtype == TSB_F32 || dtype == TSB_BF16, "tsb_ohem_ptarget: bad dtype");
    long long total = (long long)N * H * W;
    int grid = tsb_grid_for(total, kThreads, 8);
    cudaStream_t st = (cudaStream_t)stream;
    if (C <= 32) {
        if (dtype == TSB_F32)
            ohem_ptarget_kernel<float, 32><<<grid, kThreads, 0, st>>>((const float*)logits, sn, sc, sy, sx, labels, N, C, H, W, ignore_label, thresh, p, nll, state);
        else
            ohem_ptarget_kernel<__nv_bfloat16, 32><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)logits, sn, sc, sy, sx, labels, N, C, H, W, ignore_label, thresh, p, nll, state);
    } else {
        if (dtype == TSB_F32)
            ohem_ptarget_kernel_anyc<float><<<grid, kThreads, 0, st>>>((const float*)logits, sn, sc, sy, sx, labels, N, C, H, W, ignore_label, thresh, p, nll, state);
        else
            ohem_ptarget_kernel_anyc<__nv_bfloat16><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)logits, sn, sc, sy, sx, labels, N, C, H, W, ignore_label, thresh, p, nll, state);
    }
    TSB_CUDA_CHECK_LAUNCH("ohem_ptarget");
    return TSB_OK;
}

namespace {
// low-res columns one strip can touch
inline int band_maxcols(int w, int W) { return (int)(((long long)kStrip * w + W - 1) / W) + 3; }
}

extern "C" int tsb_ohem_ptarget_up(const float* logits_lo, int cs, int h, int w, const int64_t* labels, int N, int C,
                                   int H, int W, int ignore_label, float thresh, float* p, float* nll, uint32_t* state,
                                   tsb_stream_t stream) {
    TSB_REQUIRE(logits_lo && labels && p && nll && state, "tsb_ohem_ptarget_up: null pointer");
    TSB_REQUIRE(N > 0 && C > 0 && C <= 32 && cs >= C && H > 0 && W > 0 && h > 0 && w > 0,
                "tsb_ohem_ptarget_up: bad shape (C must be <= 32)");
    TSB_REQUIRE(N <= 65535 && h <= 65535, "tsb_ohem_ptarget_up: N and h must fit a grid dimension");
    const int maxcols = band_maxcols(w, W);
    dim3 grid((W + kStrip - 1) / kStrip, h, N);
    if (g_tsb_ohem_exact && (C == 19 || C == 21)) {      // exact-class-count kernels (Cityscapes / VOC)
        const size_t smx = sizeof(float) * (2 * (size_t)C * kPitchX + 2 * (size_t)maxcols * C);
        if (smx <= 100 * 1024) {
#define LX(CX)                                                                                                      \
    do {                                                                                                            \
        int rc_ = tsb_ensure_dyn_smem(reinterpret_cast<const void*>(ohem_ptarget_up_x_kernel<CX>), smx);            \
        if (rc_) return rc_;                                                                                        \
        ohem_ptarget_up_x_kernel<CX><<<grid, kThreads, smx, (cudaStream_t)stream>>>(logits_lo, cs, h, w, labels, N, H, W, ignore_label, thresh, p, nll, state, maxcols); \
    } while (0)
            if (C == 19) LX(19); else LX(21);
#undef LX
            TSB_CUDA_CHECK_LAUNCH("ohem_ptarget_up_x");
            return TSB_OK;
        }
    }
    const int cmax = C <= 20 ? 20 : 32;
    const size_t smem = sizeof(float) * 2 * (size_t)maxcols * cmax;
    TSB_REQUIRE(smem <= 28 * 1024, "tsb_ohem_ptarget_up: up-scale factor W/w too small for the band kernel");
#define L(CM, HO) ohem_ptarget_up_kernel<CM, HO><<<grid, kThreads, smem, (cudaStream_t)stream>>>(logits_lo, cs, h, w, labels, N, C, H, W, ignore_label, thresh, p, nll, state, maxcols)
    if (C <= 20) { if (g_tsb_ohem_hoist & 2) L(20, true); else L(20, false); }
    else { if (g_tsb_ohem_hoist & 2) L(32, true); else L(32, false); }
#undef L
    TSB_CUDA_CHECK_LAUNCH("ohem_ptarget_up");
    return TSB_OK;
}

extern "C" int tsb_ohem_select(const float* p, long long n, long long min_kept, float thresh, uint32_t* state,
                               tsb_stream_t stream) {
    TSB_REQUIRE(p && state && n > 0, "tsb_ohem_select: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    int grid = tsb_grid_for(n, kThreads, 8);
    ohem_decide_kernel<<<1, 1024, 0, st>>>(state, n, min_kept, thresh, -1);
    TSB_CUDA_CHECK_LAUNCH("ohem_decide_init");
    for (int level = 0; level < 3; ++level) {  // every kernel early-exits on the device-side done flag
        ohem_hist_kernel<<<grid, kThreads, 0, st>>>(p, n, state, level);
        TSB_CUDA_CHECK_LAUNCH("ohem_hist");
        ohem_decide_kernel<<<1, 1024, 0, st>>>(state, n, min_kept, thresh, level);
        TSB_CUDA_CHECK_LAUNCH("ohem_decide");
    }
    return TSB_OK;
}

extern "C" int tsb_ohem_loss(const float* p, const float* nll, const int64_t* labels, long long n, int ignore_label,
                             const float* class_weight, uint32_t* state, float* loss_out, tsb_stream_t stream) {
    TSB_REQUIRE(p && nll && labels && state && n > 0, "tsb_ohem_loss: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    int grid = tsb_grid_for(n, kThreads, 8);
    ohem_loss_kernel<<<grid, kThreads, 0, st>>>(p, nll, labels, n, ignore_label, class_weight, state);
    TSB_CUDA_CHECK_LAUNCH("ohem_loss");
    ohem_finalize_kernel<<<1, 1, 0, st>>>(state, loss_out);
    TSB_CUDA_CHECK_LAUNCH("ohem_finalize");
    return TSB_OK;
}

extern "C" int tsb_ohem_grad(const void* logits, int dtype, long long sn, long long sc, long long sy, long long sx,
                             const int64_t* labels, const float* p, int N, int C, int H, int W, int ignore_label,
                             const float* class_weight, const uint32_t* state, const float* gscale, void* dlogits,
                             tsb_stream_t stream) {
    TSB_REQUIRE(logits && labels && p && state && dlogits, "tsb_ohem_grad: null pointer");
    TSB_REQUIRE(dtype == TSB_F32 || dtype == TSB_BF16, "tsb_ohem_grad: bad dtype");
    long long total = (long long)N * H * W;
    int grid = tsb_grid_for(total, kThreads, 8);
    cudaStream_t st = (cudaStream_t)stream;
#define TSB_LAUNCH_GRAD(T, CM)                                                                                   \
    ohem_grad_kernel<T, CM><<<grid, kThreads, 0, st>>>((const T*)logits, sn, sc, sy, sx, labels, p, N, C, H, W,  \
                                                       ignore_label, class_weight, state, gscale, (T*)dlogits)
    if (C <= 32) {
        if (dtype == TSB_F32) TSB_LAUNCH_GRAD(float, 32); else TSB_LAUNCH_GRAD(__nv_bfloat16, 32);
    } else {
        if (dtype == TSB_F32) TSB_LAUNCH_GRAD(float, 0); else TSB_LAUNCH_GRAD(__nv_bfloat16, 0);
    }
#undef TSB_LAUNCH_GRAD
    TSB_CUDA_CHECK_LAUNCH("ohem_grad");
    return TSB_OK;
}

extern "C" int tsb_ohem_grad_up(const float* logits_lo, int cs, int h, int w, const int64_t* labels, const float* p,
                                int N, int C, int H, int W, int ignore_label, const float* class_weight,
                                const uint32_t* state, const float* gscale, float* dlogits_lo, tsb_stream_t stream) {
    TSB_REQUIRE(logits_lo && labels && p && state && dlogits_lo, "tsb_ohem_grad_up: null pointer");
    TSB_REQUIRE(C > 0 && C <= 32 && cs >= C, "tsb_ohem_grad_up: C must be <= 32");
    TSB_REQUIRE(N <= 65535 && h <= 65535, "tsb_ohem_grad_up: N and h must fit a grid dimension");
    const int maxcols = band_maxcols(w, W);
    TSB_REQUIRE(maxcols <= kStrip, "tsb_ohem_grad_up: up-scale factor W/w too small for the band kernel");
    if (g_tsb_ohem_exact && (C == 19 || C == 21)) {
        const size_t smx = sizeof(float) * (2 * (size_t)C * kPitchX + 2 * (size_t)maxcols * C);
        if (smx <= 72 * 1024) {
            dim3 gridx(((W + kStrip - 1) / kStrip + 1) / 2, (h + 1) / 2, N);
#define GX(CX)                                                                                                      \
    do {                                                                                                            \
        int rc_ = tsb_ensure_dyn_smem(reinterpret_cast<const void*>(ohem_grad_up_x_kernel<CX>), smx);               \
        if (rc_) return rc_;                                                                                        \
        for (int ph = 0; ph < 4; ++ph) {                                                                            \
            ohem_grad_up_x_kernel<CX><<<gridx, kThreads, smx, (cudaStream_t)stream>>>(logits_lo, cs, h, w, labels, p, N, H, W, ignore_label, class_weight, state, gscale, dlogits_lo, maxcols, ph); \
            TSB_CUDA_CHECK_LAUNCH("ohem_grad_up_x");                                                               \
        }                                                                                                           \
    } while (0)
            if (C == 19) GX(19); else GX(21);
#undef GX
            return TSB_OK;
        }
    }
    const int cmax = C <= 20 ? 20 : 32;
    const size_t smem = sizeof(float) * (2 * (size_t)cmax * (kStrip + 1) + 2 * (size_t)maxcols * cmax);
    TSB_REQUIRE(smem <= 96 * 1024, "tsb_ohem_grad_up: shared memory budget exceeded");
    dim3 grid((W + kStrip - 1) / kStrip, h, N);
    cudaStream_t st = (cudaStream_t)stream;
#define L(CM, HO)                                                                                                       \
    do {                                                                                                                \
        { int rc_ = tsb_ensure_dyn_smem(reinterpret_cast<const void*>(ohem_grad_up_kernel<CM, HO>), smem); if (rc_) return rc_; } \
        ohem_grad_up_kernel<CM, HO><<<grid, kThreads, smem, st>>>(logits_lo, cs, h, w, labels, p, N, C, H, W, ignore_label, class_weight, state, gscale, dlogits_lo, maxcols); \
    } while (0)
    if (C <= 20) { if (g_tsb_ohem_hoist & 1) L(20, true); else L(20, false); }
    else { if (g_tsb_ohem_hoist & 1) L(32, true); else L(32, false); }
#undef L
    TSB_CUDA_CHECK_LAUNCH("ohem_grad_up");
    return TSB_OK;
}
