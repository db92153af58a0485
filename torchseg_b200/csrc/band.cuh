// Bilinear (align_corners=True) interpolation coefficients and the BAND decomposition shared by the fused
// upsample + loss kernels (ohem.cu, ce_up.cu): CTA = (strip of hi-res columns, low-res row ci, image n); all hi-res rows y
// with floor(ry*y) == ci share the two low-res source rows (ci, i1). The pieces every band kernel runs are here once:
//   band_geom     the rows and low-res columns a band touches (band_maxcols bounds the columns on the host)
//   stage_rows    the two source rows into shared memory
//   blend_rows    their horizontal blend T0 / T1 at the thread's column (row-invariant, formed once per band)
//   seg_init/fill the segment table of the backward's column reduction
//   col_sums      the backward's phase 2: the per-(low-res column, class) weighted column sums
// Each kernel keeps its own shared-memory layout (passed in as pitches and index functions), thread-to-column mapping,
// barriers and stores.
#pragma once
#include "tsb_common.cuh"

namespace band {

// bilinear source coordinate, align_corners=True, exactly ATen's float recipe:
// scale = float(in-1)/float(out-1) (0 if out==1); src = scale*dst; i0 = (int)src; lambda = src - i0
struct Lerp {
    int i0, i1;
    float l0, l1;
};
static __device__ __forceinline__ Lerp make_lerp(float scale, int dst, int in_size) {
    Lerp r;
    float src = __fmul_rn(scale, (float)dst);
    r.i0 = (int)src;
    if (r.i0 > in_size - 1) r.i0 = in_size - 1;
    r.i1 = r.i0 + ((r.i0 < in_size - 1) ? 1 : 0);
    r.l1 = __fsub_rn(src, (float)r.i0);
    r.l0 = __fsub_rn(1.0f, r.l1);
    return r;
}
// 4-tap bilinear blend in the oracle's operation order (no FMA contraction: separate multiply / add roundings),
// split at its own intermediate values: t = horizontal blend of one source row (depends on the column only, so a band
// kernel forms it ONCE per thread), v = vertical blend per hi-res row.
static __device__ __forceinline__ float lerp_h(const Lerp& lx, float a, float b) {
    return __fadd_rn(__fmul_rn(lx.l0, a), __fmul_rn(lx.l1, b));
}
static __device__ __forceinline__ float lerp_v(const Lerp& ly, float t0, float t1) {
    return __fadd_rn(__fmul_rn(ly.l0, t0), __fmul_rn(ly.l1, t1));
}
static __host__ __device__ __forceinline__ float area_scale(int in_size, int out_size) {
    return out_size > 1 ? (float)(in_size - 1) / (float)(out_size - 1) : 0.0f;
}

struct BandGeom {
    int i1;           // second low-res source row (ci + 1, clamped to the last row)
    int y_lo, y_hi;   // candidate hi-res rows (membership re-checked exactly)
    int jbase, ncols; // low-res columns [jbase, jbase+ncols) touched by this strip
};
static __device__ __forceinline__ BandGeom band_geom(float ry, float rx, int ci, int x0, int x1 /*exclusive*/, int h, int H,
                                                     int w) {
    BandGeom g;
    g.i1 = ci + (ci < h - 1 ? 1 : 0);
    if (ry > 0.f) {
        g.y_lo = max(0, (int)floorf((float)ci / ry) - 1);
        g.y_hi = min(H - 1, (int)ceilf((float)(ci + 1) / ry) + 1);
    } else { g.y_lo = 0; g.y_hi = H - 1; }
    Lerp a = make_lerp(rx, x0, w), b = make_lerp(rx, x1 - 1, w);
    g.jbase = a.i0;
    g.ncols = b.i1 - a.i0 + 1;
    return g;
}
// low-res columns a strip of `strip` hi-res columns can touch (bounds BandGeom::ncols; sizes the staged rows)
static inline int band_maxcols(int strip, int w, int W) { return (int)(((long long)strip * w + W - 1) / W) + 3; }

// the band's two low-res source rows (ci, g.i1), columns [g.jbase, g.jbase + g.ncols), classes [0, C) of the NHWC
// low-res logits (pixel stride cs) into s_lo0 / s_lo1[column * pitch + class]; NT threads. With kClear, the same pass
// also clears s_clear[0, 2 * ncols * C).
template <int NT, bool kClear = false>
static __device__ __forceinline__ void stage_rows(const float* __restrict__ lo, int cs, int h, int w, int n, int ci,
                                                  const BandGeom& g, int C, int pitch, float* s_lo0, float* s_lo1,
                                                  float* s_clear = nullptr) {
    for (int q = threadIdx.x; q < 2 * g.ncols * C; q += NT) {
        const int c = q % C, t2 = q / C, col = t2 % g.ncols, row = t2 / g.ncols;
        (row ? s_lo1 : s_lo0)[col * pitch + c] = __ldg(lo + (((long long)n * h + (row ? g.i1 : ci)) * w + g.jbase + col) * cs + c);
        if (kClear) s_clear[q] = 0.f;
    }
}

// T0 / T1 of the thread's column (stencil lx at staged columns j0 / j1): the staged rows blended horizontally, for the
// classes c = c0 + dc * k < C, k in [0, nk), into sT0 / sT1[at(c)]
template <class At>
static __device__ __forceinline__ void blend_rows(const Lerp& lx, int j0, int j1, const float* s_lo0, const float* s_lo1,
                                                  int pitch, int nk, int c0, int dc, int C, float* sT0, float* sT1, At at) {
#pragma unroll
    for (int k = 0; k < nk; ++k) {
        const int c = c0 + dc * k;
        if (c < C) {
            sT0[at(c)] = lerp_h(lx, s_lo0[j0 * pitch + c], s_lo0[j1 * pitch + c]);
            sT1[at(c)] = lerp_h(lx, s_lo1[j0 * pitch + c], s_lo1[j1 * pitch + c]);
        }
    }
}

// Segment table of the backward's column reduction: the strip columns whose left stencil column is j form the range
// [s_seg[j], s_seg[j+1]); s_l0 / s_l1 hold each strip column's horizontal weights (0 past the image edge). Built in two
// steps around a barrier of the caller: seg_init, __syncthreads, seg_fill. `col` is the thread's strip column (image
// column x, stencil lx, left staged column j0) and `owner` whether this thread writes it: one thread per column.
template <int NT>
static __device__ __forceinline__ void seg_init(float* s_l0, float* s_l1, short* s_seg, int col, bool owner, bool xin,
                                                const Lerp& lx, int ncols, int nx) {
    if (owner) {
        s_l0[col] = xin ? lx.l0 : 0.f;
        s_l1[col] = xin ? lx.l1 : 0.f;
    }
    for (int q = threadIdx.x; q < ncols + 2; q += NT) s_seg[q] = (short)nx;
}
static __device__ __forceinline__ void seg_fill(short* s_seg, int col, bool owner, bool xin, float rx, int x, int w,
                                                int jbase, int j0) {
    if (xin && owner) {
        const int jprev = (col == 0) ? -1 : (make_lerp(rx, x - 1, w).i0 - jbase);
        for (int jj = jprev + 1; jj <= j0; ++jj) s_seg[jj] = (short)col;
    }
}

// Phase 2 for one (low-res column j, class): top / bot (starting from the caller's values) gain the l0x-weighted sum of
// the accumulators sG0 / sG1[at(xx)] over segment j, then the l1x-weighted sum over segment j-1, or over segment j itself
// when j is the clamped last image column, followed by segment j-1, which still points at that column with its right
// weight. Returns (top, bot); the caller stores them.
template <class At>
static __device__ __forceinline__ float2 col_sums(const float* sG0, const float* sG1, At at, const short* s_seg,
                                                  const float* s_l0, const float* s_l1, const BandGeom& g, int w, int j,
                                                  float top, float bot) {
    const int a0 = s_seg[j], a1 = s_seg[j + 1];
    for (int xx = a0; xx < a1; ++xx) {
        const float wl = s_l0[xx];
        top = fmaf(wl, sG0[at(xx)], top);
        bot = fmaf(wl, sG1[at(xx)], bot);
    }
    const bool clamped = (g.jbase + j == w - 1);
    const int b0 = clamped ? a0 : (j > 0 ? (int)s_seg[j - 1] : 0);
    const int b1 = clamped ? a1 : (j > 0 ? a0 : 0);
    for (int xx = b0; xx < b1; ++xx) {
        const float wr = s_l1[xx];
        top = fmaf(wr, sG0[at(xx)], top);
        bot = fmaf(wr, sG1[at(xx)], bot);
    }
    if (clamped && j > 0) {
        for (int xx = s_seg[j - 1]; xx < a0; ++xx) {
            const float wr = s_l1[xx];
            top = fmaf(wr, sG0[at(xx)], top);
            bot = fmaf(wr, sG1[at(xx)], bot);
        }
    }
    return make_float2(top, bot);
}

}  // namespace band
