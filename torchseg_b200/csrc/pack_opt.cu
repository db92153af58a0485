// Layout/precision packing, elementwise glue, fused flat-buffer SGD and the sigmoid focal loss.
// All HBM-bound streaming kernels (vectorised where the layout allows), sm_90a.
#include "nhwc_vec.cuh"

namespace {
// NCHW fp32 [N,3,H,W] → s2d NHWC16 bf16 [N, H/2, W/2+4, 16]; pixel column 0,1 and W/2+2, W/2+3 are zero
// padding; channel (py*2+px)*3+c. One thread per packed pixel (32 bytes = two 16-byte stores).
__global__ void __launch_bounds__(kThreads)
pack_image_s2d_kernel(const float* __restrict__ img, int N, int H, int W, __nv_bfloat16* __restrict__ out) {
    const int H2 = H / 2, W2 = W / 2, WP = W2 + 4;
    const long long total = (long long)N * H2 * WP;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        int xp = (int)(i % WP);
        long long t = i / WP;
        int y2 = (int)(t % H2), n = (int)(t / H2);
        float v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) v[k] = 0.f;
        int x2 = xp - 2;
        if (x2 >= 0 && x2 < W2) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float* pl = img + ((long long)n * 3 + c) * H * W;
                float2 r0 = __ldg(reinterpret_cast<const float2*>(pl + (long long)(2 * y2) * W + 2 * x2));
                float2 r1 = __ldg(reinterpret_cast<const float2*>(pl + (long long)(2 * y2 + 1) * W + 2 * x2));
                v[0 * 3 + c] = r0.x; v[1 * 3 + c] = r0.y; v[2 * 3 + c] = r1.x; v[3 * 3 + c] = r1.y;
            }
        }
        __nv_bfloat16* dst = out + i * 16;
        Vec8<__nv_bfloat16>::store(dst, v);
        Vec8<__nv_bfloat16>::store(dst + 8, v + 8);
    }
}

// fp32 KRSC → bf16 KRSC and bf16 flipped-transposed [C][R-1-r][S-1-s][K]
__global__ void __launch_bounds__(kThreads)
pack_weight_kernel(const float* __restrict__ w, int K, int R, int S, int C, __nv_bfloat16* __restrict__ wb,
                   __nv_bfloat16* __restrict__ wt) {
    const long long total = (long long)K * R * S * C;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        float v = __ldg(w + i);
        __nv_bfloat16 b = __float2bfloat16_rn(v);
        if (wb) wb[i] = b;
        if (wt) {
            int c = (int)(i % C);
            long long t = i / C;
            int s = (int)(t % S); t /= S;
            int r = (int)(t % R);
            int k = (int)(t / R);
            wt[(((long long)c * R + (R - 1 - r)) * S + (S - 1 - s)) * K + k] = b;
        }
    }
}

// stem: w [K,R,R,3] (KRSC fp32, stride-2 conv with pad = (R-1)/2, R = 7 or 3) → wp [K,4(a),4(b),16] bf16.
// conv: out(oh,ow) = Σ_{r,s} W[r,s]·X[2oh+r-pad, 2ow+s-pad];  r-pad = 2*(a-2)+py, a∈[0,4), py∈{0,1}
//   → r = 2a + py - (4 - pad)   (R=7,pad=3: r = 2a+py-1;  R=3,pad=1: r = 2a+py-3, only a ∈ {1,2} carry weights)
__device__ __forceinline__ bool stem_map(int a, int b, int e, int R, int pad, int& r, int& s, int& c) {
    if (e >= 12) return false;
    int q = e / 3;
    c = e % 3;
    int py = q >> 1, px = q & 1;
    r = 2 * a + py - (4 - pad);
    s = 2 * b + px - (4 - pad);
    return r >= 0 && r < R && s >= 0 && s < R;
}
__global__ void pack_stem_weight_kernel(const float* __restrict__ w, int K, int R, int pad, __nv_bfloat16* __restrict__ wp) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= K * 256) return;
    int e = i & 15, b = (i >> 4) & 3, a = (i >> 6) & 3, k = i >> 8;
    int r, s, c;
    float v = 0.f;
    if (stem_map(a, b, e, R, pad, r, s, c)) v = w[((k * R + r) * R + s) * 3 + c];
    wp[i] = __float2bfloat16_rn(v);
}
__global__ void unpack_stem_wgrad_kernel(const float* __restrict__ dwp, int K, int R, int pad, float* __restrict__ dw) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= K * 256) return;
    int e = i & 15, b = (i >> 4) & 3, a = (i >> 6) & 3, k = i >> 8;
    int r, s, c;
    if (stem_map(a, b, e, R, pad, r, s, c)) dw[((k * R + r) * R + s) * 3 + c] += dwp[i];  // (a,b,e) ↔ (r,s,c) is 1:1
}

template <typename TS, typename TD>
__global__ void __launch_bounds__(kThreads)
cast_scale_kernel(const TS* __restrict__ src, int scs, TD* __restrict__ dst, int dcs, long long npix, int C8,
                  const float* __restrict__ scale_dev) {
    const float sc = scale_dev ? *scale_dev : 1.f;
    for_each_vec(npix * C8, C8, [&](long long p, int c8) {
        float v[8];
        Vec8<TS>::load(src + p * scs + c8 * 8, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] *= sc;
        Vec8<TD>::store(dst + p * dcs + c8 * 8, v);
    });
}

// y = a + b; y = relu(a + b), the tail of RefineResidual / BNRefine (seg_oprs.py:158-162,184-188); and the ReLU
// backward dx = (y > 0) ? dy : 0 with a = dy, b = y
struct AddOp { __device__ float operator()(float a, float b) const { return a + b; } };
struct AddReluOp { __device__ float operator()(float a, float b) const { return fmaxf(a + b, 0.f); } };
struct ReluBwdOp { __device__ float operator()(float a, float b) const { return b > 0.f ? a : 0.f; } };

template <typename Op>
__global__ void __launch_bounds__(kThreads)
binary_kernel(const __nv_bfloat16* __restrict__ a, int acs, const __nv_bfloat16* __restrict__ b, int bcs,
              __nv_bfloat16* __restrict__ y, int ycs, long long npix, int C8) {
    for_each_vec(npix * C8, C8, [&](long long p, int c8) {
        float u[8], v[8];
        Vec8<__nv_bfloat16>::load(a + p * acs + c8 * 8, u);
        Vec8<__nv_bfloat16>::load(b + p * bcs + c8 * 8, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) u[k] = Op()(u[k], v[k]);
        Vec8<__nv_bfloat16>::store(y + p * ycs + c8 * 8, u);
    });
}

template <typename Op>
int binary_launch(const char* fn, const void* a, int acs, const void* b, int bcs, void* y, int ycs, long long npix,
                  int C, tsb_stream_t stream) {
    TSB_REQUIRE(a && b && y && npix > 0, "%s: bad args", fn);
    TSB_REQUIRE(TSB_VEC_OK(C, acs, a) && TSB_VEC_OK(C, bcs, b) && TSB_VEC_OK(C, ycs, y),
                "%s: C and channel strides must be multiples of 8, strides >= C, pointers 16B aligned", fn);
    const int C8 = C / 8;
    binary_kernel<Op><<<tsb_grid_for(npix * C8, kThreads, 8), kThreads, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)a, acs, (const __nv_bfloat16*)b, bcs, (__nv_bfloat16*)y, ycs, npix, C8);
    TSB_CUDA_CHECK_LAUNCH(fn);
    return TSB_OK;
}

// dst[pix, 0..Kp) (bf16) = src[pix, 0..K) zero-extended: gradient of a K-class head (K = 19, 150, 1 ...) into the
// 64-multiple GEMM-K layout the dgrad / wgrad kernels read. Any K, any source channel stride; one pass, no memset.
template <typename TS>
__global__ void __launch_bounds__(kThreads)
cast_pad_kernel(const TS* __restrict__ src, int scs, int K, __nv_bfloat16* __restrict__ dst, int dcs, int Kp8,
                long long npix) {
    for_each_vec(npix * Kp8, Kp8, [&](long long p, int c8) {
        const int c0 = c8 * 8;
        const TS* s = src + p * scs + c0;
        float v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = (c0 + k < K) ? (float)s[k] : 0.f;
        Vec8<__nv_bfloat16>::store(dst + p * dcs + c0, v);
    });
}

// db[k] += Σ_pix dy[pix,k]; one warp per pixel stripe, lanes over channels (K <= 64 typical: 19 padded). Each CTA
// writes its partial sums to its own slot of the deterministic workspace (`db` here), summed in CTA order afterwards.
__global__ void __launch_bounds__(kThreads)
bias_grad_kernel(const __nv_bfloat16* __restrict__ dy, int dycs, long long npix, int K, float* __restrict__ db) {
    __shared__ float s_acc[kThreads];
    const int kk = threadIdx.x % 64, lane = threadIdx.x / 64;  // 4 pixel lanes x 64 channels
    for (int k0 = 0; k0 < K; k0 += 64) {
        int k = k0 + kk;
        float acc = 0.f;
        if (k < K)
            for (long long p = (long long)blockIdx.x * 4 + lane; p < npix; p += (long long)gridDim.x * 4)
                acc += __bfloat162float(dy[p * dycs + k]);
        s_acc[threadIdx.x] = acc;
        __syncthreads();
        if (lane == 0 && k < K) db[(long long)blockIdx.x * K + k] = s_acc[kk] + s_acc[64 + kk] + s_acc[128 + kk] + s_acc[192 + kk];
        __syncthreads();
    }
}

// fused momentum SGD on flat buffers; segment lookup by binary search over seg_end (nseg <= a few dozen)
__global__ void __launch_bounds__(kThreads)
sgd_flat_kernel(float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ mom, long long n,
                const long long* __restrict__ seg_end, const float* __restrict__ seg_lr,
                const float* __restrict__ seg_wd, int nseg, float momentum, float gscale, int first_step,
                __nv_bfloat16* __restrict__ param_bf16) {
    for (long long i4 = ((long long)blockIdx.x * kThreads + threadIdx.x) * 4; i4 < n; i4 += (long long)gridDim.x * kThreads * 4) {
        // all four elements may straddle a segment boundary → per-element lookup only when needed
        int lo = 0, hi = nseg - 1;
        while (lo < hi) { int mid = (lo + hi) >> 1; if (seg_end[mid] > i4) hi = mid; else lo = mid + 1; }
        int seg = lo;
        if (i4 + 4 <= n && seg_end[seg] >= i4 + 4) {
            float lr = seg_lr[seg], wd = seg_wd[seg];
            float4 p = *reinterpret_cast<float4*>(param + i4);
            float4 g = *reinterpret_cast<const float4*>(grad + i4);
            float4 b = first_step ? make_float4(0.f, 0.f, 0.f, 0.f) : *reinterpret_cast<float4*>(mom + i4);
            float gx = fmaf(wd, p.x, g.x * gscale), gy = fmaf(wd, p.y, g.y * gscale);
            float gz = fmaf(wd, p.z, g.z * gscale), gw = fmaf(wd, p.w, g.w * gscale);
            b.x = first_step ? gx : fmaf(momentum, b.x, gx);
            b.y = first_step ? gy : fmaf(momentum, b.y, gy);
            b.z = first_step ? gz : fmaf(momentum, b.z, gz);
            b.w = first_step ? gw : fmaf(momentum, b.w, gw);
            p.x -= lr * b.x; p.y -= lr * b.y; p.z -= lr * b.z; p.w -= lr * b.w;
            *reinterpret_cast<float4*>(mom + i4) = b;
            *reinterpret_cast<float4*>(param + i4) = p;
            if (param_bf16)   // bf16 KRSC operand copy of the updated weights: the next step's convs read this directly
                *reinterpret_cast<uint2*>(param_bf16 + i4) = make_uint2(pack_bf16(p.x, p.y), pack_bf16(p.z, p.w));
        } else {
            for (long long i = i4; i < i4 + 4 && i < n; ++i) {
                while (seg < nseg - 1 && seg_end[seg] <= i) ++seg;
                float lr = seg_lr[seg], wd = seg_wd[seg];
                float g = fmaf(wd, param[i], grad[i] * gscale);
                float b = first_step ? g : fmaf(momentum, mom[i], g);
                mom[i] = b;
                param[i] -= lr * b;
                if (param_bf16) param_bf16[i] = __float2bfloat16_rn(param[i]);
            }
        }
    }
}

// all dgrad weight operands in ONE launch: for every listed conv weight, wt[c][R-1-r][S-1-s][k] = wb[k][r][s][c]
// (bf16 → bf16, both inside flat buffers at the same offset). 32x32 (k, c) tiles per filter tap through smem so
// that both the read (along c) and the write (along k) are contiguous.
struct WtDesc {
    long long off;
    int K, RS, C, tiles_k, tiles_c, pad;
};
__global__ void __launch_bounds__(256)
pack_wt_multi_kernel(const __nv_bfloat16* __restrict__ wb, __nv_bfloat16* __restrict__ wt, const WtDesc* __restrict__ desc,
                     const int* __restrict__ bstart, int nt) {
    __shared__ unsigned short tile[32][33];
    int lo = 0, hi = nt - 1;
    const int b = blockIdx.x;
    while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (bstart[mid] <= b) lo = mid; else hi = mid - 1; }
    const WtDesc d = desc[lo];
    int local = b - bstart[lo];
    const int tc = local % d.tiles_c; local /= d.tiles_c;
    const int tk = local % d.tiles_k;
    const int rs = local / d.tiles_k;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const unsigned short* src = reinterpret_cast<const unsigned short*>(wb) + d.off;
    unsigned short* dst = reinterpret_cast<unsigned short*>(wt) + d.off;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int k = tk * 32 + ty + j * 8, c = tc * 32 + tx;
        if (k < d.K && c < d.C) tile[ty + j * 8][tx] = src[((long long)k * d.RS + rs) * d.C + c];
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int c = tc * 32 + ty + j * 8, k = tk * 32 + tx;
        if (c < d.C && k < d.K) dst[((long long)c * d.RS + (d.RS - 1 - rs)) * d.K + k] = tile[tx][ty + j * 8];
    }
}

// SigmoidFocalLoss.forward (loss_opr.py:23-45) reproduced literally; also its analytic derivative
// dLossMean/dpred (unit upstream gradient).
template <typename T>
__global__ void __launch_bounds__(kThreads)
focal_kernel(const T* __restrict__ pred, const int64_t* __restrict__ target, long long n, int ignore_label, float gamma,
             float alpha, float* __restrict__ loss_sum, T* __restrict__ dpred) {
    __shared__ float s_red[33];
    float acc = 0.f;
    const float inv_n = 1.0f / (float)n;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        float x = ld_as_float<T>(pred + i);
        float tg = (float)target[i];
        float mask = (tg != (float)ignore_label) ? 1.f : 0.f;
        float yv = mask * tg;
        float s = 1.f / (1.f + expf(-x));
        // max_val = clamp(-s, min=0) = 0 since s > 0  (loss_opr.py:33)
        float one_m = 1.f - s;
        float pw1 = powf(one_m, gamma), pw2 = powf(s, gamma);
        float pos = pw1 * (s - s * yv);
        float lse = logf(1.f + expf(-s));
        float neg = pw2 * lse;
        float l = -(alpha * pos + (1.f - alpha) * neg) * mask;
        acc += l;
        if (dpred) {
            // derivative wrt s
            float dpos = -gamma * powf(one_m, gamma - 1.f) * (s - s * yv) + pw1 * (1.f - yv);
            float dneg = gamma * powf(s, gamma - 1.f) * lse + pw2 * (-expf(-s) / (1.f + expf(-s)));
            float dl_ds = -(alpha * dpos + (1.f - alpha) * dneg) * mask;
            st_from_float<T>(dpred + i, dl_ds * s * (1.f - s) * inv_n);
        }
    }
    acc = block_sum<kThreads>(acc, s_red);
    if (threadIdx.x == 0) atomicAdd(loss_sum, acc * inv_n);
}
}  // namespace

extern "C" int tsb_pack_image_s2d(const float* img, int N, int H, int W, void* out, tsb_stream_t stream) {
    TSB_REQUIRE(img && out && N > 0 && H > 0 && W > 0, "tsb_pack_image_s2d: bad args");
    TSB_REQUIRE(H % 2 == 0 && W % 2 == 0, "tsb_pack_image_s2d: H and W must be even");
    TSB_REQUIRE((reinterpret_cast<uintptr_t>(img) & 7u) == 0 && tsb_aligned16(out), "tsb_pack_image_s2d: alignment");
    long long total = (long long)N * (H / 2) * (W / 2 + 4);
    int grid = tsb_grid_for(total, kThreads, 8);
    pack_image_s2d_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(img, N, H, W, (__nv_bfloat16*)out);
    TSB_CUDA_CHECK_LAUNCH("pack_image_s2d");
    return TSB_OK;
}

extern "C" int tsb_pack_weight(const float* w, int K, int R, int S, int C, void* w_bf16, void* wt_bf16, tsb_stream_t stream) {
    TSB_REQUIRE(w && (w_bf16 || wt_bf16) && K > 0 && R > 0 && S > 0 && C > 0, "tsb_pack_weight: bad args");
    long long total = (long long)K * R * S * C;
    int grid = tsb_grid_for(total, kThreads, 8);
    pack_weight_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(w, K, R, S, C, (__nv_bfloat16*)w_bf16, (__nv_bfloat16*)wt_bf16);
    TSB_CUDA_CHECK_LAUNCH("pack_weight");
    return TSB_OK;
}

extern "C" int tsb_pack_stem_weight(const float* w, int K, int R, void* wp_bf16, tsb_stream_t stream) {
    TSB_REQUIRE(w && wp_bf16 && K > 0, "tsb_pack_stem_weight: bad args");
    TSB_REQUIRE(R == 7 || R == 3, "tsb_pack_stem_weight: R must be 7 (pad 3) or 3 (pad 1)");
    pack_stem_weight_kernel<<<(K * 256 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(w, K, R, (R - 1) / 2, (__nv_bfloat16*)wp_bf16);
    TSB_CUDA_CHECK_LAUNCH("pack_stem_weight");
    return TSB_OK;
}

extern "C" int tsb_unpack_stem_wgrad(const float* dwp, int K, int R, float* dw, tsb_stream_t stream) {
    TSB_REQUIRE(dwp && dw && K > 0, "tsb_unpack_stem_wgrad: bad args");
    TSB_REQUIRE(R == 7 || R == 3, "tsb_unpack_stem_wgrad: R must be 7 (pad 3) or 3 (pad 1)");
    unpack_stem_wgrad_kernel<<<(K * 256 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(dwp, K, R, (R - 1) / 2, dw);
    TSB_CUDA_CHECK_LAUNCH("unpack_stem_wgrad");
    return TSB_OK;
}

extern "C" int tsb_cast_scale(const void* src, int sdtype, int scs, void* dst, int ddtype, int dcs, long long npix, int C,
                              const float* scale_dev, tsb_stream_t stream) {
    TSB_REQUIRE(src && dst && npix > 0, "tsb_cast_scale: bad args");
    TSB_REQUIRE(TSB_VEC_OK(C, scs, src) && TSB_VEC_OK(C, dcs, dst),
                "tsb_cast_scale: C and channel strides must be multiples of 8, strides >= C, pointers 16B aligned");
    int C8 = C / 8;
    int grid = tsb_grid_for(npix * C8, kThreads, 8);
    const bool ok = dispatch_dtype_pair(sdtype, ddtype, [&](auto ts, auto td) {
        using TS = typename decltype(ts)::type;
        using TD = typename decltype(td)::type;
        cast_scale_kernel<TS, TD><<<grid, kThreads, 0, (cudaStream_t)stream>>>((const TS*)src, scs, (TD*)dst, dcs, npix, C8, scale_dev);
    });
    TSB_REQUIRE(ok, "tsb_cast_scale: bad dtype");
    TSB_CUDA_CHECK_LAUNCH("cast_scale");
    return TSB_OK;
}

extern "C" int tsb_cast_pad(const void* src, int sdtype, int scs, int K, void* dst_bf16, int dcs, int Kp, long long npix,
                            tsb_stream_t stream) {
    TSB_REQUIRE(src && dst_bf16 && npix > 0 && K > 0 && Kp >= K, "tsb_cast_pad: bad args");
    TSB_REQUIRE(TSB_VEC_OK(Kp, dcs, dst_bf16) && scs >= K, "tsb_cast_pad: Kp, dcs multiples of 8, dcs >= Kp, scs >= K, dst 16B aligned");
    TSB_REQUIRE(sdtype == TSB_F32 || sdtype == TSB_BF16, "tsb_cast_pad: bad dtype");
    int grid = tsb_grid_for(npix * (Kp / 8), kThreads, 8);
    if (sdtype == TSB_F32)
        cast_pad_kernel<float><<<grid, kThreads, 0, (cudaStream_t)stream>>>((const float*)src, scs, K, (__nv_bfloat16*)dst_bf16, dcs, Kp / 8, npix);
    else
        cast_pad_kernel<__nv_bfloat16><<<grid, kThreads, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)src, scs, K, (__nv_bfloat16*)dst_bf16, dcs, Kp / 8, npix);
    TSB_CUDA_CHECK_LAUNCH("cast_pad");
    return TSB_OK;
}

extern "C" int tsb_add(const void* a, int acs, const void* b, int bcs, void* y, int ycs, long long npix, int C,
                       tsb_stream_t stream) {
    return binary_launch<AddOp>("tsb_add", a, acs, b, bcs, y, ycs, npix, C, stream);
}

extern "C" int tsb_add_relu(const void* a, int acs, const void* b, int bcs, void* y, int ycs, long long npix, int C,
                            tsb_stream_t stream) {
    return binary_launch<AddReluOp>("tsb_add_relu", a, acs, b, bcs, y, ycs, npix, C, stream);
}

extern "C" int tsb_relu_bwd(const void* dy, int dycs, const void* y, int ycs, void* dx, int dxcs, long long npix, int C,
                            tsb_stream_t stream) {
    return binary_launch<ReluBwdOp>("tsb_relu_bwd", dy, dycs, y, ycs, dx, dxcs, npix, C, stream);
}

extern "C" int tsb_bias_grad(const void* dy, int dycs, long long npix, int K, float* db, float* ws, long long ws_floats,
                             tsb_stream_t stream) {
    TSB_REQUIRE(dy && db && npix > 0 && K > 0, "tsb_bias_grad: bad args");
    TSB_REQUIRE(dycs >= K, "tsb_bias_grad: dycs must be >= K");
    int grid = tsb_grid_for(npix, 64, 4);
    TSB_REQUIRE(ws && (long long)grid * K <= ws_floats, "tsb_bias_grad: workspace needs %lld floats", (long long)grid * K);
    bias_grad_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)dy, dycs, npix, K, ws);
    TSB_CUDA_CHECK_LAUNCH("bias_grad");
    return tsb_det_reduce(db, ws, grid, K, K, (cudaStream_t)stream);
}

extern "C" int tsb_sgd_flat(float* param, const float* grad, float* mom_buf, long long n, const long long* seg_end,
                            const float* seg_lr, const float* seg_wd, int nseg, float momentum, float gscale,
                            int first_step, tsb_stream_t stream) {
    TSB_REQUIRE(param && grad && mom_buf && seg_end && seg_lr && seg_wd && n > 0 && nseg > 0, "tsb_sgd_flat: bad args");
    TSB_REQUIRE(tsb_aligned16(param) && tsb_aligned16(grad) && tsb_aligned16(mom_buf), "tsb_sgd_flat: buffers must be 16B aligned");
    int grid = tsb_grid_for((n + 3) / 4, kThreads, 8);
    sgd_flat_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(param, grad, mom_buf, n, seg_end, seg_lr, seg_wd, nseg, momentum, gscale, first_step, nullptr);
    TSB_CUDA_CHECK_LAUNCH("sgd_flat");
    return TSB_OK;
}

extern "C" int tsb_sgd_flat_pack(float* param, const float* grad, float* mom_buf, long long n, const long long* seg_end,
                                 const float* seg_lr, const float* seg_wd, int nseg, float momentum, float gscale,
                                 int first_step, void* param_bf16, tsb_stream_t stream) {
    TSB_REQUIRE(param && grad && mom_buf && seg_end && seg_lr && seg_wd && param_bf16 && n > 0 && nseg > 0, "tsb_sgd_flat_pack: bad args");
    TSB_REQUIRE(tsb_aligned16(param) && tsb_aligned16(grad) && tsb_aligned16(mom_buf) && tsb_aligned16(param_bf16),
                "tsb_sgd_flat_pack: buffers must be 16B aligned");
    int grid = tsb_grid_for((n + 3) / 4, kThreads, 8);
    sgd_flat_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(param, grad, mom_buf, n, seg_end, seg_lr, seg_wd, nseg, momentum, gscale, first_step, (__nv_bfloat16*)param_bf16);
    TSB_CUDA_CHECK_LAUNCH("sgd_flat_pack");
    return TSB_OK;
}

extern "C" int tsb_pack_wt_multi(const void* wb_flat, void* wt_flat, const void* desc, const int* block_start, int ntensors,
                                 int nblocks, tsb_stream_t stream) {
    TSB_REQUIRE(wb_flat && wt_flat && desc && block_start && ntensors > 0 && nblocks > 0, "tsb_pack_wt_multi: bad args");
    pack_wt_multi_kernel<<<nblocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)wb_flat, (__nv_bfloat16*)wt_flat, (const WtDesc*)desc, block_start, ntensors);
    TSB_CUDA_CHECK_LAUNCH("pack_wt_multi");
    return TSB_OK;
}

extern "C" int tsb_sigmoid_focal_fwd_bwd(const void* pred, int dtype, const int64_t* target, long long n,
                                         int ignore_label, float gamma, float alpha, float* loss_mean,
                                         void* dpred_unit, tsb_stream_t stream) {
    TSB_REQUIRE(pred && target && loss_mean && n > 0, "tsb_sigmoid_focal_fwd_bwd: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    TSB_CUDA_CALL(cudaMemsetAsync(loss_mean, 0, sizeof(float), st));
    int grid = tsb_grid_for(n, kThreads, 8);
    if (dtype == TSB_F32)
        focal_kernel<float><<<grid, kThreads, 0, st>>>((const float*)pred, target, n, ignore_label, gamma, alpha, loss_mean, (float*)dpred_unit);
    else if (dtype == TSB_BF16)
        focal_kernel<__nv_bfloat16><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)pred, target, n, ignore_label, gamma, alpha, loss_mean, (__nv_bfloat16*)dpred_unit);
    else
        TSB_FAIL(TSB_ERR_ARG, "tsb_sigmoid_focal_fwd_bwd: bad dtype");
    TSB_CUDA_CHECK_LAUNCH("focal");
    return TSB_OK;
}
