// Soft-max over the pixels of each image, per class: OCRNet's soft object regions (Yuan, Chen & Wang, "Object-Contextual
// Representations for Semantic Segmentation", ECCV 2020, the SpatialGather module):
//
//   P[b, n, k] = exp(l[b, n, k] − M[b, k]) / S[b, k],   M = max_n l,   S = Σ_n exp(l − M),   n < N, k < K
//
// and its gradient dl = P ⊙ (dP − Σ_n P·dP). The logits are the fp32 NHWC aux logits; P is written as a bf16
// [B·N][Kp] operand (Kp = K rounded up to 64, channels K..Kp−1 exactly 0) of the per-image wgmma GEMMs that form the
// object-region proxy. The backward recomputes P in fp32 from the logits and the saved (M, S).
//
// Determinism: the pixels of an image are cut into `chunks` fixed ranges that depend on N and K only (not on B). A
// chunk's CTA reduces its range lane by lane and then over its lanes in lane order into a workspace slot; the apply
// kernels add an image's slots in chunk order. No atomics, so every result is bit-identical from run to run and does
// not depend on the other images of the batch.
#include "nhwc_vec.cuh"

namespace {

constexpr int kMaxK = 256;
constexpr int kPixPerLane = 4;    // the least pixels per lane of a chunk
constexpr int kMaxChunks = 64;    // per image, before a lane takes more than kPixPerLane pixels

struct Plan {
    int C8, lanes, per_cta, chunks;
};

// the column-reduction geometry (nhwc_vec.cuh) of K channels: one 8-channel group per thread, 256 / C8 pixel lanes
Plan make_plan(int N, int K) {
    Plan pl;
    pl.C8 = (K + 7) / 8;
    pl.lanes = kThreads / colred_groups(pl.C8);
    long long ppl = ((long long)N + (long long)pl.lanes * kMaxChunks - 1) / ((long long)pl.lanes * kMaxChunks);
    if (ppl < kPixPerLane) ppl = kPixPerLane;
    pl.per_cta = (int)(ppl * pl.lanes);
    pl.chunks = (int)(((long long)N + pl.per_cta - 1) / pl.per_cta);
    return pl;
}

// 8 logits of channels [8·c8, 8·c8 + 8); channels >= K read as −∞ (they may hold anything)
__device__ __forceinline__ void load_logits(const float* row, int c8, int K, float x[8]) {
    Vec8<float>::load(row + 8 * c8, x);
#pragma unroll
    for (int e = 0; e < 8; ++e)
        if (8 * c8 + e >= K) x[e] = -INFINITY;
}

// forward, per chunk: the running (max, Σ exp(l − max)) of each lane, then of the CTA over its lanes in lane order, into
// ws[((b · chunks + chunk) · 2 + {0, 1}) · K + k]. grid (chunks, B)
__global__ void __launch_bounds__(kThreads) ssm_partial_kernel(const float* __restrict__ logits, int lcs, int N, int K,
                                                               int C8, int lanes, int per_cta, float* __restrict__ ws) {
    __shared__ float s_m[kThreads * 8], s_s[kThreads * 8];
    const int b = blockIdx.y, chunk = blockIdx.x, c8 = threadIdx.x % C8, lane = threadIdx.x / C8;
    const int n0 = chunk * per_cta, n1 = min(N, n0 + per_cta);
    float m[8], s[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { m[e] = -INFINITY; s[e] = 0.f; }
    if (lane < lanes) {
        for (int n = n0 + lane; n < n1; n += lanes) {
            float x[8];
            load_logits(logits + ((long long)b * N + n) * lcs, c8, K, x);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                if (x[e] > m[e]) {
                    s[e] = s[e] * expf(m[e] - x[e]) + 1.f;
                    m[e] = x[e];
                } else {
                    s[e] += expf(x[e] - m[e]);
                }
            }
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            s_m[lane * C8 * 8 + 8 * c8 + e] = m[e];
            s_s[lane * C8 * 8 + 8 * c8 + e] = s[e];
        }
    }
    __syncthreads();
    const int k = threadIdx.x;
    if (k >= K) return;
    float M = -INFINITY;
    for (int l = 0; l < lanes; ++l) M = fmaxf(M, s_m[l * C8 * 8 + k]);
    float S = 0.f;
    for (int l = 0; l < lanes; ++l) {
        const float ml = s_m[l * C8 * 8 + k];
        if (ml != -INFINITY) S += s_s[l * C8 * 8 + k] * expf(ml - M);
    }
    float* slot = ws + ((long long)b * gridDim.x + chunk) * 2 * K;
    slot[k] = M;
    slot[K + k] = S;
}

// (M, 1/S) of channel k < K of image b from its chunk slots, added in chunk order
__device__ __forceinline__ void combine_chunks(const float* ws, int b, int chunks, int K, int k, float& M, float& S) {
    const float* base = ws + (long long)b * chunks * 2 * K;
    M = -INFINITY;
    for (int c = 0; c < chunks; ++c) M = fmaxf(M, base[c * 2 * K + k]);
    S = 0.f;
    for (int c = 0; c < chunks; ++c) {
        const float mc = base[c * 2 * K + k];
        if (mc != -INFINITY) S += base[c * 2 * K + K + k] * expf(mc - M);
    }
}

// P (fp32) of the 8 channels of group c8 from the logits and the image's (M, 1/S) in shared memory; 0 for channels >= K
__device__ __forceinline__ void probs(const float* row, int c8, int K, const float* s_M, const float* s_inv, float p[8]) {
    load_logits(row, c8, K, p);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const int k = 8 * c8 + e;
        p[e] = k < K ? expf(p[e] - s_M[k]) * s_inv[k] : 0.f;
    }
}

// forward, per chunk: combine the image's slots into (M, S) (chunk 0 stores them as stats[b][2][K]), then write the
// chunk's rows of P, all Kp channels. grid (chunks, B)
__global__ void __launch_bounds__(kThreads) ssm_apply_kernel(const float* __restrict__ logits, int lcs, int N, int K,
                                                             int C8, int Kp8, int per_cta, const float* __restrict__ ws,
                                                             __nv_bfloat16* __restrict__ P, float* __restrict__ stats) {
    __shared__ float s_M[kMaxK], s_inv[kMaxK];
    const int b = blockIdx.y, chunk = blockIdx.x, k = threadIdx.x;
    if (k < K) {
        float M, S;
        combine_chunks(ws, b, gridDim.x, K, k, M, S);
        s_M[k] = M;
        s_inv[k] = 1.f / S;
        if (chunk == 0) {
            stats[(long long)b * 2 * K + k] = M;
            stats[(long long)b * 2 * K + K + k] = S;
        }
    }
    __syncthreads();
    const int n0 = chunk * per_cta, n1 = min(N, n0 + per_cta);
    const long long total = (long long)(n1 - n0) * Kp8;
    VecWalk wk(Kp8, threadIdx.x, kThreads);
    for (long long i = threadIdx.x; i < total; i += kThreads, wk.next()) {
        const long long row = (long long)b * N + n0 + wk.p;
        float p[8];
        if (wk.c8 < C8) {
            probs(logits + row * lcs, wk.c8, K, s_M, s_inv, p);
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e) p[e] = 0.f;
        }
        Vec8<__nv_bfloat16>::store(P + row * Kp8 * 8 + 8 * wk.c8, p);
    }
}

// backward, per chunk: Σ P·dP of each lane, then of the CTA over its lanes in lane order, into ws[(b · chunks + chunk)
// · K + k]. grid (chunks, B)
__global__ void __launch_bounds__(kThreads) ssm_bwd_partial_kernel(const float* __restrict__ logits, int lcs,
                                                                   const float* __restrict__ stats,
                                                                   const float* __restrict__ dP, int dpcs, int N, int K,
                                                                   int C8, int lanes, int per_cta,
                                                                   float* __restrict__ ws) {
    __shared__ float s_acc[kThreads * 8];
    __shared__ float s_M[kMaxK], s_inv[kMaxK];
    const int b = blockIdx.y, chunk = blockIdx.x, c8 = threadIdx.x % C8, lane = threadIdx.x / C8;
    if (threadIdx.x < K) {
        s_M[threadIdx.x] = stats[(long long)b * 2 * K + threadIdx.x];
        s_inv[threadIdx.x] = 1.f / stats[(long long)b * 2 * K + K + threadIdx.x];
    }
    __syncthreads();
    const int n0 = chunk * per_cta, n1 = min(N, n0 + per_cta);
    if (lane < lanes) {
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
        for (int n = n0 + lane; n < n1; n += lanes) {
            const long long row = (long long)b * N + n;
            float p[8], g[8];
            probs(logits + row * lcs, c8, K, s_M, s_inv, p);
            Vec8<float>::load(dP + row * dpcs + 8 * c8, g);
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (8 * c8 + e < K) acc[e] = fmaf(p[e], g[e], acc[e]);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) s_acc[lane * C8 * 8 + 8 * c8 + e] = acc[e];
    }
    __syncthreads();
    const int k = threadIdx.x;
    if (k >= K) return;
    float r = 0.f;
    for (int l = 0; l < lanes; ++l) r += s_acc[l * C8 * 8 + k];
    ws[((long long)b * gridDim.x + chunk) * K + k] = r;
}

// backward, per chunk: r = the image's slots added in chunk order, then dl = P ⊙ (dP − r) on channels < K (the
// logits' other channels are not written). grid (chunks, B)
__global__ void __launch_bounds__(kThreads) ssm_bwd_apply_kernel(const float* __restrict__ logits, int lcs,
                                                                 const float* __restrict__ stats,
                                                                 const float* __restrict__ dP, int dpcs,
                                                                 float* __restrict__ dl, int dlcs, int N, int K, int C8,
                                                                 int per_cta, const float* __restrict__ ws) {
    __shared__ float s_M[kMaxK], s_inv[kMaxK], s_r[kMaxK];
    const int b = blockIdx.y, chunk = blockIdx.x, k = threadIdx.x;
    if (k < K) {
        s_M[k] = stats[(long long)b * 2 * K + k];
        s_inv[k] = 1.f / stats[(long long)b * 2 * K + K + k];
        const float* base = ws + (long long)b * gridDim.x * K;
        float r = 0.f;
        for (int c = 0; c < (int)gridDim.x; ++c) r += base[(long long)c * K + k];
        s_r[k] = r;
    }
    __syncthreads();
    const int n0 = chunk * per_cta, n1 = min(N, n0 + per_cta);
    const long long total = (long long)(n1 - n0) * C8;
    VecWalk wk(C8, threadIdx.x, kThreads);
    for (long long i = threadIdx.x; i < total; i += kThreads, wk.next()) {
        const long long row = (long long)b * N + n0 + wk.p;
        float p[8], g[8];
        probs(logits + row * lcs, wk.c8, K, s_M, s_inv, p);
        Vec8<float>::load(dP + row * dpcs + 8 * wk.c8, g);
        const int k0 = 8 * wk.c8;
#pragma unroll
        for (int e = 0; e < 8; ++e) p[e] = k0 + e < K ? p[e] * (g[e] - s_r[k0 + e]) : 0.f;
        float* dst = dl + row * dlcs + k0;
        if (k0 + 8 <= K) {
            Vec8<float>::store(dst, p);
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (k0 + e < K) dst[e] = p[e];
        }
    }
}

int check_args(const char* who, const float* logits, int lcs, int B, int N, int K) {
    TSB_REQUIRE(B >= 1 && N >= 1 && B <= 65535, "%s: bad shape B=%d N=%d", who, B, N);
    TSB_REQUIRE((long long)B * N < (1LL << 31), "%s: B*N must be below 2^31", who);
    TSB_REQUIRE(K >= 1 && K <= kMaxK, "%s: K=%d, 1 <= K <= %d is supported", who, K, kMaxK);
    TSB_REQUIRE(logits != nullptr, "%s: null logits", who);
    TSB_REQUIRE(TSB_VEC_OK((K + 7) / 8 * 8, lcs, logits),
                "%s: logits must be 16-byte aligned with a channel stride that is a multiple of 8 and >= K rounded up to 8 "
                "(got %d)", who,
                lcs);
    return TSB_OK;
}

int check_ws(const char* who, const float* ws, long long ws_floats, long long need) {
    TSB_REQUIRE(ws != nullptr && need <= ws_floats, "%s: workspace needs %lld floats", who, need);
    return TSB_OK;
}

#define SSM_CHECK(expr) do { int rc_ = (expr); if (rc_) return rc_; } while (0)

}  // namespace

extern "C" int tsb_spatial_softmax_fwd(const float* logits, int lcs, void* P, float* stats, int B, int N, int K, float* ws,
                                       long long ws_floats, tsb_stream_t stream) {
    const char* who = "tsb_spatial_softmax_fwd";
    SSM_CHECK(check_args(who, logits, lcs, B, N, K));
    TSB_REQUIRE(P != nullptr && stats != nullptr, "%s: null P or stats", who);
    TSB_REQUIRE(tsb_aligned16(P), "%s: P must be 16-byte aligned", who);
    const Plan pl = make_plan(N, K);
    SSM_CHECK(check_ws(who, ws, ws_floats, (long long)B * pl.chunks * 2 * K));
    const int Kp8 = (K + 63) / 64 * 8;
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid(pl.chunks, B);
    ssm_partial_kernel<<<grid, kThreads, 0, st>>>(logits, lcs, N, K, pl.C8, pl.lanes, pl.per_cta, ws);
    TSB_CUDA_CHECK_LAUNCH("spatial_softmax_partial");
    ssm_apply_kernel<<<grid, kThreads, 0, st>>>(logits, lcs, N, K, pl.C8, Kp8, pl.per_cta, ws, (__nv_bfloat16*)P,
                                                stats);
    TSB_CUDA_CHECK_LAUNCH("spatial_softmax_apply");
    return TSB_OK;
}

extern "C" int tsb_spatial_softmax_bwd(const float* logits, int lcs, const float* stats, const float* dP, int dpcs,
                                       float* dl, int dlcs, int B, int N, int K, float* ws, long long ws_floats,
                                       tsb_stream_t stream) {
    const char* who = "tsb_spatial_softmax_bwd";
    SSM_CHECK(check_args(who, logits, lcs, B, N, K));
    TSB_REQUIRE(stats != nullptr && dP != nullptr && dl != nullptr, "%s: null stats, dP or dl", who);
    const int K8 = (K + 7) / 8 * 8;
    TSB_REQUIRE(TSB_VEC_OK(K8, dpcs, dP) && TSB_VEC_OK(K8, dlcs, dl),
                "%s: dP and dl must be 16-byte aligned with channel strides that are multiples of 8 and >= K rounded up "
                "to 8", who);
    const Plan pl = make_plan(N, K);
    SSM_CHECK(check_ws(who, ws, ws_floats, (long long)B * pl.chunks * K));
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid(pl.chunks, B);
    ssm_bwd_partial_kernel<<<grid, kThreads, 0, st>>>(logits, lcs, stats, dP, dpcs, N, K, pl.C8, pl.lanes, pl.per_cta,
                                                      ws);
    TSB_CUDA_CHECK_LAUNCH("spatial_softmax_bwd_partial");
    ssm_bwd_apply_kernel<<<grid, kThreads, 0, st>>>(logits, lcs, stats, dP, dpcs, dl, dlcs, N, K, pl.C8, pl.per_cta, ws);
    TSB_CUDA_CHECK_LAUNCH("spatial_softmax_bwd_apply");
    return TSB_OK;
}
