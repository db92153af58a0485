// Training-time input pipeline on the device (SURVEY §8 f4): random mirror → random scale (cv2.resize INTER_LINEAR for the
// image, INTER_NEAREST for the label) → normalize → random crop + centred constant pad → HWC→CHW, fused into ONE pass
// from the decoded uint8 image to the fp32 NCHW batch and the int64 label batch the train loop consumes.
// Replaces TrainPre.__call__ (TorchSeg model/bisenet/cityscapes.bisenet.R18/dataloader.py:16-33) and the
// img_utils functions it calls (TorchSeg furnace/utils/img_utils.py:24-78,118-125,140-145,181-187); the random draws
// stay on the host (torchseg_b200/utils/gpu_pipeline.py) in the reference's order.
//
// Bit-exact by construction: OpenCV's 8-bit INTER_LINEAR is FIXED POINT (11-bit coefficients, int32 horizontal pass,
// (((b0*(S0>>4))>>16) + ((b1*(S1>>4))>>16) + 2) >> 2 vertically — imgproc/src/resize.cpp); the coefficient arithmetic below
// uses explicit IEEE double / float operations (no FMA contraction), and normalisation is a 3 x 256 table built on the host
// with the reference's own float32 / float64 sequence. HBM-bound byte work: one thread per output pixel, coalesced
// plane-wise stores (the 6 MB uint8 source of a Cityscapes frame replaces 20 MB of fp32 image + int64 label on the H2D path).
#include "tsb_common.cuh"

namespace {

struct PreSample {           // mirror of the 10 x int64 descriptor row (include/tsb.h)
    long long img, gt, H, W, flip, sh, sw, pos_h, pos_w, reserved;
};

struct Coef {
    int i0, i1, w0, w1;
};
// resize.cpp: fx = (float)((dx + 0.5) * scale - 0.5); sx = cvFloor(fx); fx -= sx; [x only: clamp at the borders with fx = 0]
__device__ __forceinline__ Coef linear_coef(int d, int src, int dst, bool border_zero) {
    const double scale = __ddiv_rn(1.0, __ddiv_rn((double)dst, (double)src));
    float f = (float)__dadd_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), -0.5);
    int s = (int)floorf(f);
    f = __fsub_rn(f, (float)s);
    if (border_zero) {
        if (s < 0) { f = 0.f; s = 0; }
        if (s >= src - 1) { f = 0.f; s = src - 1; }
    }
    Coef c;
    c.w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
    c.w1 = __float2int_rn(__fmul_rn(f, 2048.f));
    c.i0 = min(max(s, 0), src - 1);
    c.i1 = min(max(s + 1, 0), src - 1);
    return c;
}
__device__ __forceinline__ int nearest_index(int d, int src, int dst) {   // x_ofs = min(cvFloor(x * ifx), size - 1)
    const double scale = __ddiv_rn(1.0, __ddiv_rn((double)dst, (double)src));
    const int s = (int)floor(__dmul_rn((double)d, scale));
    return min(s, src - 1);
}

__global__ void __launch_bounds__(256)
train_preprocess_kernel(const PreSample* __restrict__ samples, int crop_h, int crop_w, int reverse_channels,
                        const float* __restrict__ lut, float img_pad, int gt_pad, float* __restrict__ out_img,
                        long long* __restrict__ out_gt) {
    const int n = blockIdx.z;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= crop_w) return;
    const PreSample S = samples[n];
    const int H = (int)S.H, W = (int)S.W, sh = (int)S.sh, sw = (int)S.sw;
    // random_crop_pad_to_shape: the crop [pos, pos + crop) ∩ image, centred in the target, constant border
    const int c_h = min(crop_h, sh - (int)S.pos_h), c_w = min(crop_w, sw - (int)S.pos_w);
    const int top = (crop_h - c_h) / 2, left = (crop_w - c_w) / 2;
    const int yy = y - top, xx = x - left;
    const size_t plane = (size_t)crop_h * crop_w;
    float* o = out_img + (size_t)n * 3 * plane + (size_t)y * crop_w + x;
    long long* og = out_gt + (size_t)n * plane + (size_t)y * crop_w + x;
    if (yy < 0 || yy >= c_h || xx < 0 || xx >= c_w) {
        o[0] = img_pad; o[plane] = img_pad; o[2 * plane] = img_pad;
        *og = (long long)gt_pad;
        return;
    }
    const int ys = (int)S.pos_h + yy, xs = (int)S.pos_w + xx;      // coordinates in the (mirrored, scaled) image
    const bool flip = S.flip != 0;
    // label: INTER_NEAREST
    {
        const int gy = nearest_index(ys, H, sh), gx = nearest_index(xs, W, sw);
        const uint8_t* g = reinterpret_cast<const uint8_t*>(S.gt);
        *og = (long long)g[(size_t)gy * W + (flip ? W - 1 - gx : gx)];
    }
    // image: INTER_LINEAR, fixed point
    const Coef cx = linear_coef(xs, W, sw, true), cy = linear_coef(ys, H, sh, false);
    const int xa = flip ? W - 1 - cx.i0 : cx.i0, xb = flip ? W - 1 - cx.i1 : cx.i1;
    const uint8_t* p = reinterpret_cast<const uint8_t*>(S.img);
    const uint8_t* r0a = p + ((size_t)cy.i0 * W + xa) * 3;
    const uint8_t* r0b = p + ((size_t)cy.i0 * W + xb) * 3;
    const uint8_t* r1a = p + ((size_t)cy.i1 * W + xa) * 3;
    const uint8_t* r1b = p + ((size_t)cy.i1 * W + xb) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int cs = reverse_channels ? 2 - c : c;
        const int s0 = (int)r0a[cs] * cx.w0 + (int)r0b[cs] * cx.w1;
        const int s1 = (int)r1a[cs] * cx.w0 + (int)r1b[cs] * cx.w1;
        int v = (((cy.w0 * (s0 >> 4)) >> 16) + ((cy.w1 * (s1 >> 4)) >> 16) + 2) >> 2;
        v = min(max(v, 0), 255);
        o[(size_t)c * plane] = __ldg(lut + c * 256 + v);
    }
}


// ------------------------------------------------------------------------------------------------
// DFN border labels (TorchSeg model/dfn/cityscapes.dfn.R101_v1c/dataloader.py:15-29): Canny(apertureSize 7, thresholds
// 5 → 0 after OpenCV's /16) of the scaled label map with 255 → 0, dilated by a 7x7 rectangle, 255 → 1, cropped / padded like
// the label. All integer arithmetic (imgproc/src/canny.cpp restated): Sobel-7 sums are exact ints, /16 with round-half-even,
// L1 magnitude with a ZERO border, fixed-point tangent test for the non-maximum suppression; low == high, so hysteresis adds
// nothing. Only the crop window (+7 pixels of halo) of every sample is computed:
//   G   [ch+14][cw+14] u8   label (255 → 0), coordinates CLAMPED into the scaled image (= BORDER_REPLICATE)
//   DXY [ch+8][cw+8]  2xi16 + MAG i32, zero outside the image
//   E   [ch+6][cw+6]  u8    edge map, zero outside the image
// ------------------------------------------------------------------------------------------------
struct EdgeGeom {
    int H, W, sh, sw, flip, r0, c0, c_h, c_w, top, left;
};
__device__ __forceinline__ EdgeGeom edge_geom(const PreSample& S, int crop_h, int crop_w) {
    EdgeGeom g;
    g.H = (int)S.H; g.W = (int)S.W; g.sh = (int)S.sh; g.sw = (int)S.sw; g.flip = S.flip != 0;
    g.r0 = (int)S.pos_h; g.c0 = (int)S.pos_w;
    g.c_h = min(crop_h, g.sh - g.r0); g.c_w = min(crop_w, g.sw - g.c0);
    g.top = (crop_h - g.c_h) / 2; g.left = (crop_w - g.c_w) / 2;
    return g;
}

__global__ void __launch_bounds__(256)
edge_stage_kernel(const PreSample* __restrict__ samples, int crop_h, int crop_w, uint8_t* __restrict__ G) {
    const int n = blockIdx.z, yy = blockIdx.y, xx = blockIdx.x * blockDim.x + threadIdx.x;
    const int GW = crop_w + 14, GH = crop_h + 14;
    if (xx >= GW) return;
    const PreSample S = samples[n];
    const EdgeGeom g = edge_geom(S, crop_h, crop_w);
    const int ys = min(max(g.r0 - 7 + yy, 0), g.sh - 1), xs = min(max(g.c0 - 7 + xx, 0), g.sw - 1);
    const int gy = nearest_index(ys, g.H, g.sh), gx = nearest_index(xs, g.W, g.sw);
    const uint8_t v = reinterpret_cast<const uint8_t*>(S.gt)[(size_t)gy * g.W + (g.flip ? g.W - 1 - gx : gx)];
    G[((size_t)n * GH + yy) * GW + xx] = (v == 255) ? 0 : v;
}

__device__ __forceinline__ int div16_rne(int v) {      // cvRound(v / 16.0)
    const int q = v >> 4, rem = v - (q << 4);
    return q + ((rem > 8 || (rem == 8 && (q & 1))) ? 1 : 0);
}

__global__ void __launch_bounds__(256)
edge_sobel_kernel(const PreSample* __restrict__ samples, int crop_h, int crop_w, const uint8_t* __restrict__ G,
                  short2* __restrict__ DXY, int* __restrict__ MAG) {
    const int n = blockIdx.z, yy = blockIdx.y, xx = blockIdx.x * blockDim.x + threadIdx.x;
    const int GW = crop_w + 14, GH = crop_h + 14, MW = crop_w + 8, MH = crop_h + 8;
    if (xx >= MW) return;
    const PreSample S = samples[n];
    const EdgeGeom g = edge_geom(S, crop_h, crop_w);
    const int ys = g.r0 - 4 + yy, xs = g.c0 - 4 + xx;
    const size_t o = ((size_t)n * MH + yy) * MW + xx;
    if (ys < 0 || ys >= g.sh || xs < 0 || xs >= g.sw) { MAG[o] = 0; DXY[o] = make_short2(0, 0); return; }
    const int sm[7] = {1, 6, 15, 20, 15, 6, 1}, dv[7] = {-1, -4, -5, 0, 5, 4, 1};
    const uint8_t* base = G + ((size_t)n * GH + yy) * GW + xx;    // G row of (ys - 3) is yy, column of (xs - 3) is xx
    int dx = 0, dy = 0;
#pragma unroll
    for (int i = 0; i < 7; ++i) {
        int rx = 0, ry = 0;
#pragma unroll
        for (int j = 0; j < 7; ++j) {
            const int v = base[(size_t)i * GW + j];
            rx += dv[j] * v;
            ry += sm[j] * v;
        }
        dx += sm[i] * rx;
        dy += dv[i] * ry;
    }
    dx = div16_rne(dx);
    dy = div16_rne(dy);
    DXY[o] = make_short2((short)dx, (short)dy);
    MAG[o] = abs(dx) + abs(dy);
}

__global__ void __launch_bounds__(256)
edge_nms_kernel(const PreSample* __restrict__ samples, int crop_h, int crop_w, const short2* __restrict__ DXY,
                const int* __restrict__ MAG, uint8_t* __restrict__ E) {
    const int n = blockIdx.z, yy = blockIdx.y, xx = blockIdx.x * blockDim.x + threadIdx.x;
    const int MW = crop_w + 8, MH = crop_h + 8, EW = crop_w + 6, EH = crop_h + 6;
    if (xx >= EW) return;
    const PreSample S = samples[n];
    const EdgeGeom g = edge_geom(S, crop_h, crop_w);
    const int ys = g.r0 - 3 + yy, xs = g.c0 - 3 + xx;
    uint8_t e = 0;
    if (ys >= 0 && ys < g.sh && xs >= 0 && xs < g.sw) {
        const int* mrow = MAG + ((size_t)n * MH + yy + 1) * MW + xx + 1;     // MAG origin is one pixel further out
        const int m = mrow[0];
        if (m > 0) {                                                        // low = floor(5 / 16) = 0
            const short2 d = DXY[((size_t)n * MH + yy + 1) * MW + xx + 1];
            const int xs_ = d.x, ys_ = d.y;
            const int x = abs(xs_), y = abs(ys_) << 15;
            const int TG22 = 13573;                                          // (int)(0.41421356237 * 2^15 + 0.5)
            const int tg22x = x * TG22;
            if (y < tg22x) {
                e = (m > mrow[-1] && m >= mrow[1]) ? 255 : 0;
            } else {
                const int tg67x = tg22x + (x << 16);
                if (y > tg67x) {
                    e = (m > mrow[-MW] && m >= mrow[MW]) ? 255 : 0;
                } else {
                    const int s = ((xs_ ^ ys_) < 0) ? -1 : 1;
                    e = (m > mrow[-MW - s] && m > mrow[MW + s]) ? 255 : 0;
                }
            }
        }
    }
    E[((size_t)n * EH + yy) * EW + xx] = e;
}

__global__ void __launch_bounds__(256)
edge_dilate_kernel(const PreSample* __restrict__ samples, int crop_h, int crop_w, const uint8_t* __restrict__ E, int gt_pad,
                   long long* __restrict__ out) {
    const int n = blockIdx.z, y = blockIdx.y, x = blockIdx.x * blockDim.x + threadIdx.x;
    const int EW = crop_w + 6, EH = crop_h + 6;
    if (x >= crop_w) return;
    const PreSample S = samples[n];
    const EdgeGeom g = edge_geom(S, crop_h, crop_w);
    const int yy = y - g.top, xx = x - g.left;
    long long v = gt_pad;
    if (yy >= 0 && yy < g.c_h && xx >= 0 && xx < g.c_w) {
        const uint8_t* e = E + ((size_t)n * EH + yy) * EW + xx;             // E row of (ys - 3) is yy
        int any = 0;
#pragma unroll
        for (int i = 0; i < 7; ++i)
#pragma unroll
            for (int j = 0; j < 7; ++j) any |= e[(size_t)i * EW + j];
        v = any ? 1 : 0;
    }
    out[((size_t)n * crop_h + y) * crop_w + x] = v;
}

}  // namespace

extern "C" int tsb_train_preprocess(const long long* samples_dev, int n, int crop_h, int crop_w, int reverse_channels,
                                    const float* lut, float img_pad, int gt_pad, float* out_img, long long* out_gt,
                                    tsb_stream_t stream) {
    TSB_REQUIRE(samples_dev && lut && out_img && out_gt, "tsb_train_preprocess: null pointer");
    TSB_REQUIRE(n > 0 && n <= 65535 && crop_h > 0 && crop_h <= 65535 && crop_w > 0, "tsb_train_preprocess: bad sizes");
    dim3 grid((crop_w + 255) / 256, crop_h, n);
    train_preprocess_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const PreSample*>(samples_dev), crop_h, crop_w,
                                                                    reverse_channels, lut, img_pad, gt_pad, out_img, out_gt);
    TSB_CUDA_CHECK_LAUNCH("train_preprocess");
    return TSB_OK;
}

extern "C" size_t tsb_edge_labels_workspace_bytes(int n, int crop_h, int crop_w) {
    if (n <= 0 || crop_h <= 0 || crop_w <= 0) return 0;
    const size_t g = (size_t)(crop_h + 14) * (crop_w + 14), m = (size_t)(crop_h + 8) * (crop_w + 8), e = (size_t)(crop_h + 6) * (crop_w + 6);
    auto up = [](size_t v) { return (v + 255) / 256 * 256; };
    return up(g * n) + up(m * n * 4) + up(m * n * 4) + up(e * n);
}

extern "C" int tsb_edge_labels(const long long* samples_dev, int n, int crop_h, int crop_w, int gt_pad, void* workspace,
                               size_t workspace_bytes, long long* out_aux, tsb_stream_t stream) {
    TSB_REQUIRE(samples_dev && workspace && out_aux, "tsb_edge_labels: null pointer");
    TSB_REQUIRE(n > 0 && n <= 65535 && crop_h > 0 && crop_h + 14 <= 65535 && crop_w > 0, "tsb_edge_labels: bad sizes");
    TSB_REQUIRE(workspace_bytes >= tsb_edge_labels_workspace_bytes(n, crop_h, crop_w) && (reinterpret_cast<uintptr_t>(workspace) & 255u) == 0,
                "tsb_edge_labels: workspace too small or not 256-byte aligned");
    const size_t g = (size_t)(crop_h + 14) * (crop_w + 14), m = (size_t)(crop_h + 8) * (crop_w + 8);
    auto up = [](size_t v) { return (v + 255) / 256 * 256; };
    uint8_t* G = reinterpret_cast<uint8_t*>(workspace);
    short2* DXY = reinterpret_cast<short2*>(G + up(g * n));
    int* MAG = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(DXY) + up(m * n * 4));
    uint8_t* E = reinterpret_cast<uint8_t*>(MAG) + up(m * n * 4);
    const PreSample* S = reinterpret_cast<const PreSample*>(samples_dev);
    cudaStream_t st = (cudaStream_t)stream;
    edge_stage_kernel<<<dim3((crop_w + 14 + 255) / 256, crop_h + 14, n), 256, 0, st>>>(S, crop_h, crop_w, G);
    TSB_CUDA_CHECK_LAUNCH("edge_stage");
    edge_sobel_kernel<<<dim3((crop_w + 8 + 255) / 256, crop_h + 8, n), 256, 0, st>>>(S, crop_h, crop_w, G, DXY, MAG);
    TSB_CUDA_CHECK_LAUNCH("edge_sobel");
    edge_nms_kernel<<<dim3((crop_w + 6 + 255) / 256, crop_h + 6, n), 256, 0, st>>>(S, crop_h, crop_w, DXY, MAG, E);
    TSB_CUDA_CHECK_LAUNCH("edge_nms");
    edge_dilate_kernel<<<dim3((crop_w + 255) / 256, crop_h, n), 256, 0, st>>>(S, crop_h, crop_w, E, gt_pad, out_aux);
    TSB_CUDA_CHECK_LAUNCH("edge_dilate");
    return TSB_OK;
}
