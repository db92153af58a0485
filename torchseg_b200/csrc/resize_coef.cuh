// OpenCV INTER_LINEAR resize coefficients (imgproc/src/resize.cpp), shared by the training input pipeline
// (data_pipeline.cu) and the evaluator (eval.cu). Every operation is an explicit IEEE double / float op (no FMA contraction),
// so the taps and weights are cv2's bit for bit.
//
// `inv_scale` is cv2's inv_scale: destination over source. cv2.resize(img, dsize) takes dsize / ssize; cv2.resize(img, None,
// fx=s) takes s itself, which differs from dsize / ssize once dsize = rint(ssize · s) is rounded.
#pragma once
#include <cuda_runtime.h>

struct LinearTap {           // source pixels i0, i1 (clamped) and the weight f of i1
    int i0, i1;
    float f;
};
// resize.cpp: fx = (float)((dx + 0.5) * scale - 0.5); sx = cvFloor(fx); fx -= sx; [x only: clamp at the borders with fx = 0]
__device__ __forceinline__ LinearTap linear_tap(int d, int src, double inv_scale, bool border_zero) {
    const double scale = __ddiv_rn(1.0, inv_scale);
    float f = (float)__dadd_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), -0.5);
    int s = (int)floorf(f);
    f = __fsub_rn(f, (float)s);
    if (border_zero) {
        if (s < 0) { f = 0.f; s = 0; }
        if (s >= src - 1) { f = 0.f; s = src - 1; }
    }
    LinearTap t;
    t.f = f;
    t.i0 = min(max(s, 0), src - 1);
    t.i1 = min(max(s + 1, 0), src - 1);
    return t;
}

struct Coef {                // 8-bit path: 11-bit fixed-point weights (INTER_RESIZE_COEF_SCALE = 2048)
    int i0, i1, w0, w1;
};
__device__ __forceinline__ Coef linear_coef(int d, int src, double inv_scale, bool border_zero) {
    const LinearTap t = linear_tap(d, src, inv_scale, border_zero);
    Coef c;
    c.w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, t.f), 2048.f));
    c.w1 = __float2int_rn(__fmul_rn(t.f, 2048.f));
    c.i0 = t.i0;
    c.i1 = t.i1;
    return c;
}

// 8-bit vertical pass (VResizeLinear<uchar, int, short, FixedPtCast<int, uchar, INTER_RESIZE_COEF_BITS*2>>) of two
// horizontal sums s0 (row i0) and s1 (row i1)
__device__ __forceinline__ int linear_u8(const Coef& cy, int s0, int s1) {
    const int v = (((cy.w0 * (s0 >> 4)) >> 16) + ((cy.w1 * (s1 >> 4)) >> 16) + 2) >> 2;
    return min(max(v, 0), 255);
}
