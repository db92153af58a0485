// Training-mode BatchNorm pieces on NHWC bf16 activations (fp32 statistics), sm_90a.
// Replaces norm_layer(...) of ConvBnRelu (TorchSeg furnace/seg_opr/seg_oprs.py:34,42), the
// BasicBlock bn1/bn2 + residual add + ReLU (TorchSeg furnace/base_model/resnet.py:33-53) and the
// statistics half of apex SyncBatchNorm (train.py:54-55).  All HBM-bound: 16-byte vector accesses,
// per-channel reductions through shared memory + one workspace slot per CTA, summed in CTA order (tsb_det_reduce).
#include "nhwc_vec.cuh"

namespace {
// Per-CTA partial sums go to slot blockIdx.x of the deterministic workspace (tsb_det_reduce sums the slots in order).
__device__ __forceinline__ void store_part_v4(float* base, long long stride, float a, float b, float c, float d) {
    *reinterpret_cast<float4*>(base + blockIdx.x * stride) = make_float4(a, b, c, d);
}

// Generic per-channel column reduction over [npix, C] with NACC accumulators per channel.
// Functor: f(pix, c8, float acc[NACC][8]) accumulates one 8-channel vector of one pixel.
template <int NACC, typename F>
__device__ __forceinline__ void column_reduce(long long npix, int C8, float* const (&outs)[NACC], long long part_stride, F f) {
    extern __shared__ float s_buf[];  // [lanes][groups][NACC][8]
    const int groups = min(C8, kThreads);
    const int lanes = kThreads / groups;
    const int g = threadIdx.x % groups, lane = threadIdx.x / groups;
    const long long chunk = (npix + gridDim.x - 1) / gridDim.x;
    const long long p0 = (long long)blockIdx.x * chunk;
    const long long p1 = (p0 + chunk < npix) ? p0 + chunk : npix;
    for (int g0 = 0; g0 < C8; g0 += groups) {
        const int cg = g0 + g;
        float acc[NACC][8];
#pragma unroll
        for (int a = 0; a < NACC; ++a)
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[a][k] = 0.f;
        if (cg < C8 && lane < lanes)
            for (long long pp = p0 + lane; pp < p1; pp += lanes) f(pp, cg, acc);
        if (lane < lanes) {
#pragma unroll
            for (int a = 0; a < NACC; ++a)
#pragma unroll
                for (int k = 0; k < 8; ++k) s_buf[((lane * groups + g) * NACC + a) * 8 + k] = acc[a][k];
        }
        __syncthreads();
        // thread (lane, g) sums accumulator quads striped over lanes and stores each into this CTA's workspace slot
        if (cg < C8 && lane < lanes) {
            for (int quad = lane; quad < NACC * 2; quad += lanes) {
                float s[4] = {0.f, 0.f, 0.f, 0.f};
                for (int l = 0; l < lanes; ++l) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) s[k] += s_buf[(l * groups + g) * NACC * 8 + quad * 4 + k];
                }
                store_part_v4(outs[quad / 2] + cg * 8 + (quad % 2) * 4, part_stride, s[0], s[1], s[2], s[3]);
            }
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kThreads)
bn_stats_kernel(const __nv_bfloat16* __restrict__ x, int cs, long long npix, int C8, float* sum, float* sumsq, long long part_stride) {
    float* const outs[2] = {sum, sumsq};
    column_reduce<2>(npix, C8, outs, part_stride, [&](long long p, int cg, float (&acc)[2][8]) {
        float v[8];
        Vec8<__nv_bfloat16>::load(x + p * cs + cg * 8, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) { acc[0][k] += v[k]; acc[1][k] += v[k] * v[k]; }
    });
}

__global__ void bn_finalize_kernel(const float* __restrict__ sum, const float* __restrict__ sumsq, double count, int C,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                   float momentum, float* mean, float* invstd, float* scale, float* shift,
                                   float* running_mean, float* running_var) {
    int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double m = (double)sum[c] / count;
    double var = (double)sumsq[c] / count - m * m;  // biased (normalisation)
    if (var < 0.0) var = 0.0;
    float is = (float)(1.0 / sqrt(var + (double)eps));
    float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
    if (mean) mean[c] = (float)m;
    if (invstd) invstd[c] = is;
    if (scale) scale[c] = g * is;
    if (shift) shift[c] = b - (float)m * g * is;
    if (running_mean) running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)m;
    if (running_var) {
        double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
    }
}

// Elementwise kernels below are launched with gridDim.x*kThreads a multiple of C8 whenever C8 divides kThreads
// (all power-of-two channel counts): a thread then keeps the SAME 8-channel group for its whole grid-stride loop and
// the per-channel parameters are loaded into registers once (otherwise the LSU, not HBM, bounds the kernel).
template <bool kRelu, bool kRes>
__global__ void __launch_bounds__(kThreads)
bn_apply_kernel(const __nv_bfloat16* __restrict__ x, int xcs, const float* __restrict__ scale,
                const float* __restrict__ shift, const __nv_bfloat16* __restrict__ res, int rcs,
                __nv_bfloat16* __restrict__ y, int ycs, long long npix, int C8) {
    const long long total = npix * C8;
    const bool hoist = (kThreads % C8) == 0;
    float sc[8], sh[8];
    if (hoist) {
        const int c8 = threadIdx.x % C8;
        ldg8f(scale + c8 * 8, sc);
        ldg8f(shift + c8 * 8, sh);
    }
    // two independent vectors per trip (loads issued back to back before the math); (pixel, channel-group) indices
    // come from a VecWalk — no 64-bit division in the loop
    constexpr int kU = 2;
    const long long stride = (long long)gridDim.x * kThreads;
    const long long start = (long long)blockIdx.x * kThreads + threadIdx.x;
    VecWalk wk(C8, start, stride);
    for (long long i0 = start; i0 < total; i0 += kU * stride) {
        uint4 xq[kU], rq[kU];
        long long off_y[kU];
        int c8s[kU];
        bool ok[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            ok[u] = i0 + u * stride < total;
            c8s[u] = wk.c8;
            const long long p = wk.p;
            wk.next();
            if (ok[u]) {
                xq[u] = *reinterpret_cast<const uint4*>(x + p * xcs + c8s[u] * 8);
                if (kRes) rq[u] = *reinterpret_cast<const uint4*>(res + p * rcs + c8s[u] * 8);
            } else {
                xq[u] = make_uint4(0u, 0u, 0u, 0u);
                if (kRes) rq[u] = make_uint4(0u, 0u, 0u, 0u);
            }
            off_y[u] = p * ycs + c8s[u] * 8;
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            float v[8];
            unpack8(xq[u], v);
            if (!hoist) {
                ldg8f(scale + c8s[u] * 8, sc);
                ldg8f(shift + c8s[u] * 8, sh);
            }
            float r[8];
            if (kRes) unpack8(rq[u], r);
            bn_act8<kRelu, kRes>(v, sc, sh, r);
            if (ok[u]) Vec8<__nv_bfloat16>::store(y + off_y[u], v);
        }
    }
}

// kRelu: 0 = no activation, 1 = ReLU mask read from y (y > 0), 2 = mask recomputed as fma(x, scale, shift) > 0 —
// exact for layers without a residual (bf16 rounding keeps the sign), and saves the whole read of y.
template <int kRelu>
__global__ void __launch_bounds__(kThreads)
bn_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ dy, int dycs, const __nv_bfloat16* __restrict__ y, int ycs,
                     const __nv_bfloat16* __restrict__ x, int xcs, const float* __restrict__ mean,
                     const float* __restrict__ invstd, const float* __restrict__ scale, const float* __restrict__ shift,
                     long long npix, int C8, float* sum_dz, float* sum_dz_xhat, long long part_stride) {
    // inner loop: acc0 += dz, acc1 += dz*x (no per-pixel parameter loads); Σ dz·x̂ = invstd·(acc1 − mean·acc0) is
    // formed once per (block, channel) when the partial sums are flushed.
    extern __shared__ float s_buf[];  // [lanes][groups][2][8]
    const int groups = min(C8, kThreads);
    const int lanes = kThreads / groups;
    const int g = threadIdx.x % groups, lane = threadIdx.x / groups;
    const long long chunk = (npix + gridDim.x - 1) / gridDim.x;
    const long long p0 = (long long)blockIdx.x * chunk;
    const long long p1 = (p0 + chunk < npix) ? p0 + chunk : npix;
    for (int g0 = 0; g0 < C8; g0 += groups) {
        const int cg = g0 + g;
        float a0[8], a1[8], sc[8], sh[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) { a0[k] = 0.f; a1[k] = 0.f; sc[k] = 0.f; sh[k] = 0.f; }
        if (cg < C8 && lane < lanes) {
            if (kRelu == 2) { ldg8f(scale + cg * 8, sc); ldg8f(shift + cg * 8, sh); }
            // kU independent pixel rows per trip: all 2-3 x kU 16-byte loads are issued before the first use, so each
            // thread keeps >= 128 B in flight (the pass is pure HBM streaming; one load pair per trip left the memory
            // pipe at ~3.4 TB/s)
            constexpr int kU = 4;
            long long pp = p0 + lane;
            for (; pp + (long long)(kU - 1) * lanes < p1; pp += (long long)kU * lanes) {
                uint4 gq[kU], xq[kU], yq[kU];
#pragma unroll
                for (int u = 0; u < kU; ++u) {
                    const long long q = pp + (long long)u * lanes;
                    gq[u] = *reinterpret_cast<const uint4*>(dy + q * dycs + cg * 8);
                    xq[u] = *reinterpret_cast<const uint4*>(x + q * xcs + cg * 8);
                    if (kRelu == 1) yq[u] = *reinterpret_cast<const uint4*>(y + q * ycs + cg * 8);
                }
#pragma unroll
                for (int u = 0; u < kU; ++u) {
                    float gv[8], xv[8];
                    unpack8(gq[u], gv);
                    unpack8(xq[u], xv);
                    if (kRelu == 1) {
                        float yv[8];
                        unpack8(yq[u], yv);
#pragma unroll
                        for (int k = 0; k < 8; ++k) gv[k] = yv[k] > 0.f ? gv[k] : 0.f;
                    } else if (kRelu == 2) {
#pragma unroll
                        for (int k = 0; k < 8; ++k) gv[k] = fmaf(xv[k], sc[k], sh[k]) > 0.f ? gv[k] : 0.f;
                    }
#pragma unroll
                    for (int k = 0; k < 8; ++k) { a0[k] += gv[k]; a1[k] = fmaf(gv[k], xv[k], a1[k]); }
                }
            }
            for (; pp < p1; pp += lanes) {
                float gv[8], xv[8];
                Vec8<__nv_bfloat16>::load(dy + pp * dycs + cg * 8, gv);
                Vec8<__nv_bfloat16>::load(x + pp * xcs + cg * 8, xv);
                if (kRelu == 1) {
                    float yv[8];
                    Vec8<__nv_bfloat16>::load(y + pp * ycs + cg * 8, yv);
#pragma unroll
                    for (int k = 0; k < 8; ++k) gv[k] = yv[k] > 0.f ? gv[k] : 0.f;
                } else if (kRelu == 2) {
#pragma unroll
                    for (int k = 0; k < 8; ++k) gv[k] = fmaf(xv[k], sc[k], sh[k]) > 0.f ? gv[k] : 0.f;
                }
#pragma unroll
                for (int k = 0; k < 8; ++k) { a0[k] += gv[k]; a1[k] = fmaf(gv[k], xv[k], a1[k]); }
            }
        }
        if (lane < lanes) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                s_buf[((lane * groups + g) * 2 + 0) * 8 + k] = a0[k];
                s_buf[((lane * groups + g) * 2 + 1) * 8 + k] = a1[k];
            }
        }
        __syncthreads();
        // flush: one 16-byte store per 4 channels and accumulator into this CTA's workspace slot
        if (cg < C8 && lane < lanes) {
            for (int h = lane; h < 2; h += lanes) {
                float t0[4] = {0.f, 0.f, 0.f, 0.f}, t1[4] = {0.f, 0.f, 0.f, 0.f};
                for (int l = 0; l < lanes; ++l) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        t0[k] += s_buf[((l * groups + g) * 2 + 0) * 8 + h * 4 + k];
                        t1[k] += s_buf[((l * groups + g) * 2 + 1) * 8 + h * 4 + k];
                    }
                }
                const int c = cg * 8 + h * 4;
                const float4 m = __ldg(reinterpret_cast<const float4*>(mean + c));
                const float4 is = __ldg(reinterpret_cast<const float4*>(invstd + c));
                store_part_v4(sum_dz + c, part_stride, t0[0], t0[1], t0[2], t0[3]);
                store_part_v4(sum_dz_xhat + c, part_stride, is.x * (t1[0] - m.x * t0[0]), is.y * (t1[1] - m.y * t0[1]),
                           is.z * (t1[2] - m.z * t0[2]), is.w * (t1[3] - m.w * t0[3]));
            }
        }
        __syncthreads();
    }
}

// kAdd: dx = bf16(float(dx) + r) with r the fp32 value stored without it (tsb_bn_bwd_apply_add)
template <int kRelu, bool kDres, bool kAdd>
__device__ __forceinline__ void
bn_bwd_apply_body(const __nv_bfloat16* __restrict__ dy, int dycs, const __nv_bfloat16* __restrict__ y, int ycs,
                  const __nv_bfloat16* __restrict__ x, int xcs, const float* __restrict__ mean,
                  const float* __restrict__ invstd, const float* __restrict__ gamma,
                  const float* __restrict__ sum_dz, const float* __restrict__ sum_dz_xhat, float inv_count,
                  __nv_bfloat16* __restrict__ dx, int dxcs, __nv_bfloat16* __restrict__ dres, int drcs,
                  long long npix, int C8, float* dgamma_acc, float* dbeta_acc, const float* __restrict__ scale,
                  const float* __restrict__ shift) {
    if (dgamma_acc != nullptr && blockIdx.x == 0) {  // fold the parameter-gradient accumulation into this pass
        for (int c = threadIdx.x; c < C8 * 8; c += kThreads) {
            dgamma_acc[c] += sum_dz_xhat[c];
            dbeta_acc[c] += sum_dz[c];
        }
    }
    // dx = γ·σ⁻¹·(dz − Σdz/n − x̂·Σdz·x̂/n), x̂ = (x−μ)σ⁻¹   ⇒   dx = A·dz + B·x + C  with per-channel
    //   A = γσ⁻¹,  B = −γσ⁻²·Σdz·x̂/n,  C = −A·Σdz/n − B·μ
    auto coeffs = [&](int c8, float (&A)[8], float (&B)[8], float (&Cc)[8], float (&sc)[8], float (&sh)[8]) {
        float m[8], is[8], ga[8], s1[8], s2[8];
        ldg8f(mean + c8 * 8, m); ldg8f(invstd + c8 * 8, is); ldg8f(gamma + c8 * 8, ga);
        ldg8f(sum_dz + c8 * 8, s1); ldg8f(sum_dz_xhat + c8 * 8, s2);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            A[k] = ga[k] * is[k];
            B[k] = -A[k] * is[k] * s2[k] * inv_count;
            Cc[k] = -A[k] * s1[k] * inv_count - B[k] * m[k];
        }
        if (kRelu == 2) { ldg8f(scale + c8 * 8, sc); ldg8f(shift + c8 * 8, sh); }
    };
    const long long total = npix * C8;
    const bool hoist = (kThreads % C8) == 0;
    float A[8], B[8], Cc[8], sc[8], sh[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { sc[k] = 0.f; sh[k] = 0.f; }
    if (hoist) coeffs(threadIdx.x % C8, A, B, Cc, sc, sh);
    constexpr int kU = 2;   // two independent vectors per trip: 4-6 loads in flight per thread before the math
    const long long stride = (long long)gridDim.x * kThreads;
    const long long start = (long long)blockIdx.x * kThreads + threadIdx.x;
    VecWalk wk(C8, start, stride);
    for (long long i0 = start; i0 < total; i0 += kU * stride) {
        uint4 gq[kU], xq[kU], yq[kU], dq[kU];
        long long pix[kU];
        int c8s[kU];
        bool ok[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            ok[u] = i0 + u * stride < total;
            c8s[u] = wk.c8;
            pix[u] = wk.p;
            wk.next();
            if (ok[u]) {
                gq[u] = *reinterpret_cast<const uint4*>(dy + pix[u] * dycs + c8s[u] * 8);
                xq[u] = *reinterpret_cast<const uint4*>(x + pix[u] * xcs + c8s[u] * 8);
                if (kRelu == 1) yq[u] = *reinterpret_cast<const uint4*>(y + pix[u] * ycs + c8s[u] * 8);
                if (kAdd) dq[u] = *reinterpret_cast<const uint4*>(dx + pix[u] * dxcs + c8s[u] * 8);
            } else {
                gq[u] = xq[u] = yq[u] = dq[u] = make_uint4(0u, 0u, 0u, 0u);
            }
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            if (!hoist) coeffs(c8s[u], A, B, Cc, sc, sh);
            float g[8], xv[8], o[8];
            unpack8(gq[u], g);
            unpack8(xq[u], xv);
            if (kRelu == 1) {
                float yv[8];
                unpack8(yq[u], yv);
#pragma unroll
                for (int k = 0; k < 8; ++k) g[k] = yv[k] > 0.f ? g[k] : 0.f;
            } else if (kRelu == 2) {
#pragma unroll
                for (int k = 0; k < 8; ++k) g[k] = fmaf(xv[k], sc[k], sh[k]) > 0.f ? g[k] : 0.f;
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) o[k] = fmaf(A[k], g[k], fmaf(B[k], xv[k], Cc[k]));
            if (kAdd) {
                float d[8];
                unpack8(dq[u], d);
#pragma unroll
                for (int k = 0; k < 8; ++k) o[k] = d[k] + o[k];
            }
            if (ok[u]) {
                Vec8<__nv_bfloat16>::store(dx + pix[u] * dxcs + c8s[u] * 8, o);
                if (kDres) Vec8<__nv_bfloat16>::store(dres + pix[u] * drcs + c8s[u] * 8, g);
            }
        }
    }
}

#define TSB_BN_BWD_APPLY_ARGS                                                                                          \
    const __nv_bfloat16* __restrict__ dy, int dycs, const __nv_bfloat16* __restrict__ y, int ycs,                      \
        const __nv_bfloat16* __restrict__ x, int xcs, const float* __restrict__ mean, const float* __restrict__ invstd, \
        const float* __restrict__ gamma, const float* __restrict__ sum_dz, const float* __restrict__ sum_dz_xhat,      \
        float inv_count, __nv_bfloat16* __restrict__ dx, int dxcs, __nv_bfloat16* __restrict__ dres, int drcs,         \
        long long npix, int C8, float *dgamma_acc, float *dbeta_acc, const float *__restrict__ scale,                  \
        const float *__restrict__ shift
#define TSB_BN_BWD_APPLY_PASS \
    dy, dycs, y, ycs, x, xcs, mean, invstd, gamma, sum_dz, sum_dz_xhat, inv_count, dx, dxcs, dres, drcs, npix, C8, \
        dgamma_acc, dbeta_acc, scale, shift
template <int kRelu, bool kDres>
__global__ void __launch_bounds__(kThreads, 3) bn_bwd_apply_kernel(TSB_BN_BWD_APPLY_ARGS) {
    bn_bwd_apply_body<kRelu, kDres, false>(TSB_BN_BWD_APPLY_PASS);
}
template <int kRelu, bool kDres>   // the read of dx costs registers: two CTAs per SM keep it free of spills
__global__ void __launch_bounds__(kThreads, 2) bn_bwd_apply_add_kernel(TSB_BN_BWD_APPLY_ARGS) {
    bn_bwd_apply_body<kRelu, kDres, true>(TSB_BN_BWD_APPLY_PASS);
}
#undef TSB_BN_BWD_APPLY_ARGS
#undef TSB_BN_BWD_APPLY_PASS

// ---------------------------------------------------------------- channel attention scale (ARM / FFM)
template <bool kAdd>
__global__ void __launch_bounds__(kThreads)
chan_scale_fwd_kernel(const __nv_bfloat16* __restrict__ x, int xcs, const float* __restrict__ a, float base,
                      const __nv_bfloat16* __restrict__ add, int acs, __nv_bfloat16* __restrict__ y, int ycs, int HW,
                      int C8, long long total) {
    for_each_vec(total, C8, [&](long long p, int c8) {
        int n = (int)(p / HW);
        float v[8], av[8];
        Vec8<__nv_bfloat16>::load(x + p * xcs + c8 * 8, v);
        ldg8f(a + (long long)n * C8 * 8 + c8 * 8, av);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] *= base + 1.f / (1.f + __expf(-av[k]));
        if (kAdd) {
            float r[8];
            Vec8<__nv_bfloat16>::load(add + p * acs + c8 * 8, r);
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] += r[k];
        }
        Vec8<__nv_bfloat16>::store(y + p * ycs + c8 * 8, v);
    });
}

// grid = (chunks, N): per image column reduction for da plus elementwise dx
__global__ void __launch_bounds__(kThreads)
chan_scale_bwd_kernel(const __nv_bfloat16* __restrict__ dy, int dycs, const __nv_bfloat16* __restrict__ x, int xcs,
                      const float* __restrict__ a, float base, __nv_bfloat16* __restrict__ dx, int dxcs, float* da,
                      int HW, int C8) {
    extern __shared__ float s_buf[];
    const int n = blockIdx.y;
    const int groups = min(C8, kThreads);
    const int lanes = kThreads / groups;
    const int g = threadIdx.x % groups, lane = threadIdx.x / groups;
    const int chunk = (HW + gridDim.x - 1) / gridDim.x;
    const int p0 = blockIdx.x * chunk, p1 = min(HW, p0 + chunk);
    for (int g0 = 0; g0 < C8; g0 += groups) {
        const int cg = g0 + g;
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
        if (cg < C8 && lane < lanes) {
            float av[8], sg[8];
            ldg8f(a + (long long)n * C8 * 8 + cg * 8, av);
#pragma unroll
            for (int k = 0; k < 8; ++k) sg[k] = 1.f / (1.f + __expf(-av[k]));
            for (int pp = p0 + lane; pp < p1; pp += lanes) {
                long long p = (long long)n * HW + pp;
                float gv[8], xv[8], o[8];
                Vec8<__nv_bfloat16>::load(dy + p * dycs + cg * 8, gv);
                Vec8<__nv_bfloat16>::load(x + p * xcs + cg * 8, xv);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    o[k] = gv[k] * (base + sg[k]);
                    acc[k] += gv[k] * xv[k];
                }
                Vec8<__nv_bfloat16>::store(dx + p * dxcs + cg * 8, o);
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] *= sg[k] * (1.f - sg[k]);
        }
        if (lane < lanes) {
#pragma unroll
            for (int k = 0; k < 8; ++k) s_buf[(lane * groups + g) * 8 + k] = acc[k];
        }
        __syncthreads();
        if (cg < C8 && lane < lanes) {
            for (int slot = lane; slot < 8; slot += lanes) {
                float s = 0.f;
                for (int l = 0; l < lanes; ++l) s += s_buf[(l * groups + g) * 8 + slot];
                da[blockIdx.x * (long long)gridDim.y * C8 * 8 + (long long)n * C8 * 8 + cg * 8 + slot] = s;   // workspace slot
            }
        }
        __syncthreads();
    }
}

}  // namespace

extern "C" int tsb_bn_stats(const void* x, int cs, long long npix, int C, float* sum, float* sumsq, float* ws,
                            long long ws_floats, tsb_stream_t stream) {
    TSB_REQUIRE(x && sum && sumsq && npix > 0, "tsb_bn_stats: bad args");
    TSB_REQUIRE(TSB_VEC_OK(C, cs, x), "tsb_bn_stats: C and cs must be multiples of 8, cs >= C, x 16B aligned");
    int C8 = C / 8;
    const int grid = colred_grid(npix, C8, 16, tsb_num_sms() * 8LL);
    TSB_REQUIRE(ws && (long long)grid * 2 * C <= ws_floats, "tsb_bn_stats: workspace needs %lld floats", (long long)grid * 2 * C);
    TSB_REQUIRE(tsb_aligned16(ws), "tsb_bn_stats: ws must be 16B aligned");
    bn_stats_kernel<<<grid, kThreads, colred_smem(C8, 2), (cudaStream_t)stream>>>((const __nv_bfloat16*)x, cs, npix, C8, ws, ws + C, 2LL * C);
    TSB_CUDA_CHECK_LAUNCH("bn_stats");
    return tsb_det_reduce_pair(sum, sumsq, ws, grid, C, (cudaStream_t)stream);
}

extern "C" int tsb_bn_finalize(const float* sum, const float* sumsq, double count, int C, const float* gamma,
                               const float* beta, float eps, float momentum, float* mean, float* invstd, float* scale,
                               float* shift, float* running_mean, float* running_var, tsb_stream_t stream) {
    TSB_REQUIRE(sum && sumsq && count > 0 && C > 0, "tsb_bn_finalize: bad args");
    bn_finalize_kernel<<<(C + 127) / 128, 128, 0, (cudaStream_t)stream>>>(sum, sumsq, count, C, gamma, beta, eps, momentum, mean, invstd, scale, shift, running_mean, running_var);
    TSB_CUDA_CHECK_LAUNCH("bn_finalize");
    return TSB_OK;
}

extern "C" int tsb_bn_apply(const void* x, int xcs, const float* scale, const float* shift, const void* residual,
                            int rcs, int relu, void* y, int ycs, long long npix, int C, tsb_stream_t stream) {
    TSB_REQUIRE(x && scale && shift && y && npix > 0, "tsb_bn_apply: bad args");
    TSB_REQUIRE(TSB_VEC_OK(C, xcs, x) && TSB_VEC_OK(C, ycs, y) && (!residual || TSB_VEC_OK(C, rcs, residual)),
                "tsb_bn_apply: C and channel strides must be multiples of 8, strides >= C, pointers 16B aligned");
    TSB_REQUIRE(tsb_aligned16(scale) && tsb_aligned16(shift), "tsb_bn_apply: scale and shift must be 16B aligned");
    int C8 = C / 8;
    int grid = tsb_grid_for(npix * C8, kThreads, 8);
    cudaStream_t st = (cudaStream_t)stream;
#define L(R, S) bn_apply_kernel<R, S><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)x, xcs, scale, shift, (const __nv_bfloat16*)residual, rcs, (__nv_bfloat16*)y, ycs, npix, C8)
    if (relu) { if (residual) L(true, true); else L(true, false); }
    else { if (residual) L(false, true); else L(false, false); }
#undef L
    TSB_CUDA_CHECK_LAUNCH("bn_apply");
    return TSB_OK;
}

extern "C" int tsb_bn_bwd_reduce(const void* dy, int dycs, const void* y, int ycs, const void* x, int xcs,
                                 const float* mean, const float* invstd, int relu, long long npix, int C, float* sum_dz,
                                 float* sum_dz_xhat, const float* scale, const float* shift, float* ws, long long ws_floats,
                                 tsb_stream_t stream) {
    TSB_REQUIRE(dy && x && mean && invstd && sum_dz && sum_dz_xhat && npix > 0, "tsb_bn_bwd_reduce: bad args");
    const int mode = !relu ? 0 : (y ? 1 : 2);
    TSB_REQUIRE(mode != 2 || (scale && shift), "tsb_bn_bwd_reduce: relu without y needs scale and shift");
    TSB_REQUIRE(TSB_VEC_OK(C, dycs, dy) && TSB_VEC_OK(C, xcs, x) && (mode != 1 || TSB_VEC_OK(C, ycs, y)), "tsb_bn_bwd_reduce: C and channel strides must be multiples of 8, strides >= C, pointers 16B aligned");
    TSB_REQUIRE(tsb_aligned16(mean) && tsb_aligned16(invstd) && (mode != 2 || (tsb_aligned16(scale) && tsb_aligned16(shift))),
                "tsb_bn_bwd_reduce: per-channel vectors must be 16B aligned");
    int C8 = C / 8;
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = colred_grid(npix, C8, 16, tsb_num_sms() * 8LL);
    TSB_REQUIRE(ws && (long long)grid * 2 * C <= ws_floats, "tsb_bn_bwd_reduce: workspace needs %lld floats", (long long)grid * 2 * C);
    TSB_REQUIRE(tsb_aligned16(ws), "tsb_bn_bwd_reduce: ws must be 16B aligned");
#define L(M) bn_bwd_reduce_kernel<M><<<grid, kThreads, colred_smem(C8, 2), st>>>((const __nv_bfloat16*)dy, dycs, (const __nv_bfloat16*)y, ycs, (const __nv_bfloat16*)x, xcs, mean, invstd, scale, shift, npix, C8, ws, ws + C, 2LL * C)
    if (mode == 0) L(0); else if (mode == 1) L(1); else L(2);
#undef L
    TSB_CUDA_CHECK_LAUNCH("bn_bwd_reduce");
    return tsb_det_reduce_pair(sum_dz, sum_dz_xhat, ws, grid, C, st);
}

template <bool kAdd>
static int bn_bwd_apply_impl(const void* dy, int dycs, const void* y, int ycs, const void* x, int xcs,
                             const float* mean, const float* invstd, const float* gamma, const float* sum_dz,
                             const float* sum_dz_xhat, double count, int relu, void* dx, int dxcs, void* dres,
                             int drcs, long long npix, int C, float* dgamma_acc, float* dbeta_acc,
                             const float* scale, const float* shift, tsb_stream_t stream, const char* who) {
    TSB_REQUIRE(dy && x && mean && invstd && gamma && sum_dz && sum_dz_xhat && dx && npix > 0 && count > 0, "%s: bad args", who);
    TSB_REQUIRE((dgamma_acc == nullptr) == (dbeta_acc == nullptr), "%s: dgamma_acc and dbeta_acc go together", who);
    const int mode = !relu ? 0 : (y ? 1 : 2);
    TSB_REQUIRE(mode != 2 || (scale && shift), "%s: relu without y needs scale and shift", who);
    TSB_REQUIRE(TSB_VEC_OK(C, dycs, dy) && TSB_VEC_OK(C, xcs, x) && TSB_VEC_OK(C, dxcs, dx) &&
                (mode != 1 || TSB_VEC_OK(C, ycs, y)) && (!dres || TSB_VEC_OK(C, drcs, dres)), "%s: C and channel strides must be multiples of 8, strides >= C, pointers 16B aligned", who);
    TSB_REQUIRE(tsb_aligned16(mean) && tsb_aligned16(invstd) && tsb_aligned16(gamma) && tsb_aligned16(sum_dz) &&
                tsb_aligned16(sum_dz_xhat) && (mode != 2 || (tsb_aligned16(scale) && tsb_aligned16(shift))),
                "%s: per-channel vectors must be 16B aligned", who);
    int C8 = C / 8;
    int grid = tsb_grid_for(npix * C8, kThreads, 8);
    cudaStream_t st = (cudaStream_t)stream;
    float inv_count = (float)(1.0 / count);
#define K_(R, D) (kAdd ? bn_bwd_apply_add_kernel<R, D> : bn_bwd_apply_kernel<R, D>)
#define L(R, D) K_(R, D)<<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)dy, dycs, (const __nv_bfloat16*)y, ycs, (const __nv_bfloat16*)x, xcs, mean, invstd, gamma, sum_dz, sum_dz_xhat, inv_count, (__nv_bfloat16*)dx, dxcs, (__nv_bfloat16*)dres, drcs, npix, C8, dgamma_acc, dbeta_acc, scale, shift)
    if (mode == 0) { if (dres) L(0, true); else L(0, false); }
    else if (mode == 1) { if (dres) L(1, true); else L(1, false); }
    else { if (dres) L(2, true); else L(2, false); }
#undef L
#undef K_
    TSB_CUDA_CHECK_LAUNCH(kAdd ? "bn_bwd_apply_add" : "bn_bwd_apply");
    return TSB_OK;
}

extern "C" int tsb_bn_bwd_apply(const void* dy, int dycs, const void* y, int ycs, const void* x, int xcs,
                                const float* mean, const float* invstd, const float* gamma, const float* sum_dz,
                                const float* sum_dz_xhat, double count, int relu, void* dx, int dxcs, void* dres,
                                int drcs, long long npix, int C, float* dgamma_acc, float* dbeta_acc,
                                const float* scale, const float* shift, tsb_stream_t stream) {
    return bn_bwd_apply_impl<false>(dy, dycs, y, ycs, x, xcs, mean, invstd, gamma, sum_dz, sum_dz_xhat, count, relu, dx,
                                    dxcs, dres, drcs, npix, C, dgamma_acc, dbeta_acc, scale, shift, stream,
                                    "tsb_bn_bwd_apply");
}

extern "C" int tsb_bn_bwd_apply_add(const void* dy, int dycs, const void* y, int ycs, const void* x, int xcs,
                                    const float* mean, const float* invstd, const float* gamma, const float* sum_dz,
                                    const float* sum_dz_xhat, double count, int relu, void* dx, int dxcs, void* dres,
                                    int drcs, long long npix, int C, float* dgamma_acc, float* dbeta_acc,
                                    const float* scale, const float* shift, tsb_stream_t stream) {
    return bn_bwd_apply_impl<true>(dy, dycs, y, ycs, x, xcs, mean, invstd, gamma, sum_dz, sum_dz_xhat, count, relu, dx,
                                   dxcs, dres, drcs, npix, C, dgamma_acc, dbeta_acc, scale, shift, stream,
                                   "tsb_bn_bwd_apply_add");
}

extern "C" int tsb_chan_scale_fwd(const void* x, int xcs, const float* a, float base, const void* add, int acs, void* y,
                                  int ycs, int N, int HW, int C, tsb_stream_t stream) {
    TSB_REQUIRE(x && a && y && N > 0 && HW > 0, "tsb_chan_scale_fwd: bad args");
    TSB_REQUIRE(TSB_VEC_OK(C, xcs, x) && TSB_VEC_OK(C, ycs, y) && (!add || TSB_VEC_OK(C, acs, add)) && tsb_aligned16(a), "tsb_chan_scale_fwd: C and channel strides must be multiples of 8, strides >= C, pointers 16B aligned");
    int C8 = C / 8;
    long long total = (long long)N * HW * C8;
    int grid = tsb_grid_for(total, kThreads, 8);
    cudaStream_t st = (cudaStream_t)stream;
    if (add)
        chan_scale_fwd_kernel<true><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)x, xcs, a, base, (const __nv_bfloat16*)add, acs, (__nv_bfloat16*)y, ycs, HW, C8, total);
    else
        chan_scale_fwd_kernel<false><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)x, xcs, a, base, nullptr, 0, (__nv_bfloat16*)y, ycs, HW, C8, total);
    TSB_CUDA_CHECK_LAUNCH("chan_scale_fwd");
    return TSB_OK;
}

extern "C" int tsb_chan_scale_bwd(const void* dy, int dycs, const void* x, int xcs, const float* a, float base, void* dx,
                                  int dxcs, float* da, int N, int HW, int C, float* ws, long long ws_floats,
                                  tsb_stream_t stream) {
    TSB_REQUIRE(dy && x && a && dx && da && N > 0 && HW > 0, "tsb_chan_scale_bwd: bad args");
    TSB_REQUIRE(TSB_VEC_OK(C, dycs, dy) && TSB_VEC_OK(C, xcs, x) && TSB_VEC_OK(C, dxcs, dx) && tsb_aligned16(a), "tsb_chan_scale_bwd: C and channel strides must be multiples of 8, strides >= C, pointers 16B aligned");
    int C8 = C / 8;
    const int chunks = colred_grid(HW, C8, 16, (tsb_num_sms() * 8 + N - 1) / N);
    TSB_REQUIRE(ws && (long long)chunks * N * C <= ws_floats, "tsb_chan_scale_bwd: workspace needs %lld floats", (long long)chunks * N * C);
    chan_scale_bwd_kernel<<<dim3(chunks, N), kThreads, colred_smem(C8, 1), (cudaStream_t)stream>>>((const __nv_bfloat16*)dy, dycs, (const __nv_bfloat16*)x, xcs, a, base, (__nv_bfloat16*)dx, dxcs, ws, HW, C8);
    TSB_CUDA_CHECK_LAUNCH("chan_scale_bwd");
    return tsb_det_reduce(da, ws, chunks, (long long)N * C, (long long)N * C, (cudaStream_t)stream);
}
