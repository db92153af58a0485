// Evaluator on the device (SURVEY §8 f2): everything `Evaluator.sliding_eval` / `scale_process` / `whole_eval`
// (engine/evaluator.py) do around the network forward, bit-identical to the numpy / cv2 / torch host path.
//
//   tsb_eval_windows     uint8 HWC frame → cv2.resize(fx=s) → centred pad → normalise → [n, 3, wh, ww] fp32 windows
//   tsb_eval_accumulate  network log-probs (+ the mirrored pass) → exp → windows SUMMED into the [C, PH, PW] canvas
//   tsb_eval_resize_add  margin-cropped canvas → cv2.resize to the frame size (fp32) → += the fp64 total [, → arg-max]
//
// cv2 facts the kernels restate (imgproc/src/resize.cpp, OpenCV 4.x; tests/eval_oracle.py has the numpy form):
// - fx=s takes dsize = rint(ssize · s) and coefficient scale 1/s; dsize == ssize is a copy;
// - INTER_LINEAR at an exact scale of 2 in both directions is INTER_AREA (resizeAreaFast): uint8 (a+b+c+d+2) >> 2 over
//   full 2x2 blocks and rint((float)sum / count) over blocks cut by an odd border; float ((a00+a01)+a10)+a11 times 0.25;
// - float INTER_LINEAR rounds both products and the sum of each pass separately (no FMA); 8-bit is fixed point.
// The sums keep the host order: windows in raster order per pixel (no atomics), scales in list order in fp64.
#include <float.h>
#include <math.h>

#include "tsb_common.cuh"
#include "resize_coef.cuh"

namespace {

enum { RS_COPY = 0, RS_LINEAR = 1, RS_AREA2 = 2 };

// cv2.resize's choice of path for INTER_LINEAR: same size → copy; both scales (1 / inv_scale) exactly 2 → area fast
int resize_mode(int src_h, int src_w, int dst_h, int dst_w, double inv_y, double inv_x) {
    if (src_h == dst_h && src_w == dst_w) return RS_COPY;
    const double sx = 1.0 / inv_x, sy = 1.0 / inv_y;
    if (fabs(sx - 2.0) < DBL_EPSILON && fabs(sy - 2.0) < DBL_EPSILON) return RS_AREA2;
    return RS_LINEAR;
}

// one pixel (y, x) of cv2.resize(src, None, fx=s, fy=s, INTER_LINEAR) for uint8 HWC with cin channels; grey frames
// (cin = 1) are replicated to the three output planes
__device__ __forceinline__ void scaled_pixel_u8(const uint8_t* __restrict__ src, int H, int W, int cin, int mode, double inv,
                                                int y, int x, int v[3]) {
    if (mode == RS_COPY) {
        const uint8_t* p = src + ((size_t)y * W + x) * cin;
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = p[cin == 3 ? c : 0];
    } else if (mode == RS_AREA2) {
        const int y0 = 2 * y, x0 = 2 * x;
        if (y0 + 2 <= H && x0 + 2 <= W) {           // full block (resizeAreaFast's vector and scalar fast loops)
            const uint8_t* p = src + ((size_t)y0 * W + x0) * cin;
            const size_t r = (size_t)W * cin;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const int k = cin == 3 ? c : 0;
                v[c] = ((int)p[k] + (int)p[cin + k] + (int)p[r + k] + (int)p[r + cin + k] + 2) >> 2;
            }
        } else {                                    // block cut by the bottom / right border of an odd frame
            const bool two_y = y0 + 2 <= H, two_x = x0 + 2 <= W;
            const uint8_t* p = src + ((size_t)y0 * W + x0) * cin;
            const size_t r = (size_t)W * cin;
            const float cnt = (float)((two_y ? 2 : 1) * (two_x ? 2 : 1));
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const int k = cin == 3 ? c : 0;
                int sum = p[k];
                if (two_x) sum += p[cin + k];
                if (two_y) sum += p[r + k] + (two_x ? p[r + cin + k] : 0);
                v[c] = min(max(__float2int_rn(__fdiv_rn((float)sum, cnt)), 0), 255);
            }
        }
    } else {
        const Coef cx = linear_coef(x, W, inv, true), cy = linear_coef(y, H, inv, false);
        const uint8_t* r0 = src + (size_t)cy.i0 * W * cin;
        const uint8_t* r1 = src + (size_t)cy.i1 * W * cin;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int k = cin == 3 ? c : 0;
            const int s0 = (int)r0[cx.i0 * cin + k] * cx.w0 + (int)r0[cx.i1 * cin + k] * cx.w1;
            const int s1 = (int)r1[cx.i0 * cin + k] * cx.w0 + (int)r1[cx.i1 * cin + k] * cx.w1;
            v[c] = linear_u8(cy, s0, s1);
        }
    }
}

// one thread per window pixel: the scaled frame sits at (top, left) of the canvas, everything else is padding
__global__ void __launch_bounds__(256)
eval_windows_kernel(const uint8_t* __restrict__ src, int H, int W, int cin, int mode, double inv, int sh, int sw, int top,
                    int left, const float* __restrict__ lut, int pad_zero, const int* __restrict__ corners, int wh, int ww,
                    int mirror, float* __restrict__ out) {
    const int n = blockIdx.z, wy = blockIdx.y, wx = blockIdx.x * blockDim.x + threadIdx.x;
    if (wx >= ww) return;
    const size_t plane = (size_t)wh * ww;
    float* o = out + (size_t)n * 3 * plane + (size_t)wy * ww + wx;
    const int y = __ldg(corners + 2 * n) + wy - top;
    const int x = __ldg(corners + 2 * n + 1) + (mirror ? ww - 1 - wx : wx) - left;
    if (y < 0 || y >= sh || x < 0 || x >= sw) {
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c * plane] = pad_zero ? 0.f : __ldg(lut + c * 256);
        return;
    }
    int v[3];
    scaled_pixel_u8(src, H, W, cin, mode, inv, y, x, v);
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c * plane] = __ldg(lut + c * 256 + v[c]);
}

// one thread per canvas element (x, y, class): the windows covering it, in order, each adding exp(lp + mirror(lp_flip))
__global__ void __launch_bounds__(256)
eval_accumulate_kernel(const float* __restrict__ lp, const float* __restrict__ lpf, const int* __restrict__ corners, int n,
                       int C, int wh, int ww, float* __restrict__ acc, int ah, int aw) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, c = blockIdx.z;
    if (x >= aw) return;
    float* a = acc + ((size_t)c * ah + y) * aw + x;
    float v = 0.f;
    bool hit = false;
    for (int k = 0; k < n; ++k) {
        const int ly = y - __ldg(corners + 2 * k), lx = x - __ldg(corners + 2 * k + 1);
        if (ly < 0 || ly >= wh || lx < 0 || lx >= ww) continue;
        if (!hit) { v = *a; hit = true; }
        const size_t row = (((size_t)k * C + c) * wh + ly) * ww;
        float s = __ldg(lp + row + lx);
        if (lpf) s = __fadd_rn(s, __ldg(lpf + row + (ww - 1 - lx)));
        v = __fadd_rn(v, expf(s));                  // accurate expf: torch.exp's libdevice function (no fast-math)
    }
    if (hit) *a = v;
}

// one thread per output pixel: every class resized, added to the fp64 total; with `pred`, the first maximum of the
// updated total is written instead of the total itself (numpy argmax: the first NaN wins, else the first maximum)
__global__ void __launch_bounds__(128)
eval_resize_add_kernel(const float* __restrict__ src, int C, int h, int w, long long cstride, long long rstride, int mode,
                       double inv_y, double inv_x, double* __restrict__ total, int H, int W, int64_t* __restrict__ pred) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    size_t o00, o01 = 0, o10 = 0, o11 = 0;
    float a0 = 1.f, a1 = 0.f, b0 = 1.f, b1 = 0.f;
    if (mode == RS_COPY) {
        o00 = (size_t)y * rstride + x;
    } else if (mode == RS_AREA2) {
        o00 = (size_t)(2 * y) * rstride + 2 * x;
        o01 = o00 + 1;
        o10 = o00 + rstride;
        o11 = o10 + 1;
    } else {
        const LinearTap tx = linear_tap(x, w, inv_x, true), ty = linear_tap(y, h, inv_y, false);
        a0 = __fsub_rn(1.f, tx.f); a1 = tx.f;
        b0 = __fsub_rn(1.f, ty.f); b1 = ty.f;
        o00 = (size_t)ty.i0 * rstride + tx.i0;
        o01 = (size_t)ty.i0 * rstride + tx.i1;
        o10 = (size_t)ty.i1 * rstride + tx.i0;
        o11 = (size_t)ty.i1 * rstride + tx.i1;
    }
    const size_t plane = (size_t)H * W;
    double* t = total + (size_t)y * W + x;
    double best = 0.0;
    int arg = 0;
    for (int c = 0; c < C; ++c) {
        const float* s = src + (size_t)c * cstride;
        float r;
        if (mode == RS_COPY) {
            r = __ldg(s + o00);
        } else if (mode == RS_AREA2) {
            r = __fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(__ldg(s + o00), __ldg(s + o01)), __ldg(s + o10)), __ldg(s + o11)), 0.25f);
        } else {
            const float h0 = __fadd_rn(__fmul_rn(__ldg(s + o00), a0), __fmul_rn(__ldg(s + o01), a1));
            const float h1 = __fadd_rn(__fmul_rn(__ldg(s + o10), a0), __fmul_rn(__ldg(s + o11), a1));
            r = __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, b1));
        }
        const double v = __dadd_rn(t[(size_t)c * plane], (double)r);
        if (pred) {
            if (c == 0 || v > best || (isnan(v) && !isnan(best))) { best = v; arg = c; }
        } else {
            t[(size_t)c * plane] = v;
        }
    }
    if (pred) pred[(size_t)y * W + x] = arg;
}

}  // namespace

extern "C" int tsb_eval_windows(const uint8_t* src, int H, int W, int cin, double fx, int sh, int sw, int top, int left,
                                const float* lut, int pad_zero, const int* corners, int n, int wh, int ww, int mirror,
                                float* out, tsb_stream_t stream) {
    TSB_REQUIRE(src && lut && corners && out, "tsb_eval_windows: null pointer");
    TSB_REQUIRE(cin == 1 || cin == 3, "tsb_eval_windows: cin must be 1 or 3");
    TSB_REQUIRE(H > 0 && W > 0 && sh > 0 && sw > 0 && top >= 0 && left >= 0, "tsb_eval_windows: bad frame sizes");
    TSB_REQUIRE(n > 0 && n <= 65535 && wh > 0 && wh <= 65535 && ww > 0, "tsb_eval_windows: bad window sizes");
    const bool same = sh == H && sw == W;
    TSB_REQUIRE(same || (fx > 0 && sh == (int)nearbyint(H * fx) && sw == (int)nearbyint(W * fx)),
                "tsb_eval_windows: (sh, sw) must be cv2's dsize (rint(H * fx), rint(W * fx))");
    const int mode = same ? RS_COPY : resize_mode(H, W, sh, sw, fx, fx);
    dim3 grid((ww + 255) / 256, wh, n);
    eval_windows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, H, W, cin, mode, fx, sh, sw, top, left, lut, pad_zero,
                                                                corners, wh, ww, mirror, out);
    TSB_CUDA_CHECK_LAUNCH("eval_windows");
    return TSB_OK;
}

extern "C" int tsb_eval_accumulate(const float* lp, const float* lp_flip, const int* corners, int n, int C, int wh, int ww,
                                   float* acc, int acc_h, int acc_w, tsb_stream_t stream) {
    TSB_REQUIRE(lp && corners && acc, "tsb_eval_accumulate: null pointer");
    TSB_REQUIRE(n > 0 && C > 0 && C <= 65535 && wh > 0 && ww > 0, "tsb_eval_accumulate: bad sizes");
    TSB_REQUIRE(acc_h > 0 && acc_h <= 65535 && acc_w > 0, "tsb_eval_accumulate: bad accumulator size");
    dim3 grid((acc_w + 255) / 256, acc_h, C);
    eval_accumulate_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(lp, lp_flip, corners, n, C, wh, ww, acc, acc_h, acc_w);
    TSB_CUDA_CHECK_LAUNCH("eval_accumulate");
    return TSB_OK;
}

extern "C" int tsb_eval_resize_add(const float* src, int C, int h, int w, long long plane_stride, long long row_stride,
                                   double* total, int H, int W, int64_t* pred, tsb_stream_t stream) {
    TSB_REQUIRE(src && total, "tsb_eval_resize_add: null pointer");
    TSB_REQUIRE(C > 0 && h > 0 && w > 0 && H > 0 && H <= 65535 && W > 0, "tsb_eval_resize_add: bad sizes");
    TSB_REQUIRE(row_stride >= w && plane_stride >= (long long)(h - 1) * row_stride + w,
                "tsb_eval_resize_add: strides overlap the [C, h, w] view");
    const double inv_y = (double)H / h, inv_x = (double)W / w;
    const int mode = resize_mode(h, w, H, W, inv_y, inv_x);
    dim3 grid((W + 127) / 128, H);
    eval_resize_add_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(src, C, h, w, plane_stride, row_stride, mode, inv_y, inv_x,
                                                                   total, H, W, pred);
    TSB_CUDA_CHECK_LAUNCH("eval_resize_add");
    return TSB_OK;
}
