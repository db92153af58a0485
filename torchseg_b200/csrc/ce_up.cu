// Fused bilinear up-sampling (align_corners=True, to an explicit output size) + cross-entropy with ignore index for MANY
// classes (32 < C <= 152: ADE20K's 150) — replaces `F.interpolate(...)` → `log_softmax` → `nn.CrossEntropyLoss` of the PSPNet /
// PSANet heads (TorchSeg model/pspnet/ade.pspnet.R101_v1c/network.py:46-57, psanet network.py:46-55) without ever
// writing the [B,150,H,W] fp32 logits: materialised, those cost ~24 GB of HBM traffic per head and step at 16 x 713 x 713
// (write, two reads, gradient write, gradient read).
//
// Band decomposition (band.cuh): CTA = (64 hi-res columns, low-res row i, image n), 256 threads = 64 columns x 4 class lanes;
// lane q of a pixel owns the classes c = 4j + q. The horizontally blended source rows live in shared memory as
// T[j][column][q] (consecutive lanes → consecutive words: conflict-free), staged once per band; a hi-res row then costs 2 LDS
// + 3 flops per class for the value, and the 4 lanes of a pixel combine max / sum with two shuffles.
//   forward : lse[pixel] = logsumexp_c v_c (kept for the backward), loss = mean over valid pixels of lse − v_target
//   backward: d lo[i, j, c] += Σ_pixels w_y·w_x·(exp(v_c − lse) − [c = target])·g/count — the softmax part through per-thread
//             register accumulators reduced per band in shared memory (phase 2: band.cuh col_sums, shared with the OHEM
//             gradient kernels), the one-hot part through a low-resolution shared-memory tile (4 RED.shared per pixel) that
//             phase 2 starts from
#include "band.cuh"

namespace {
using namespace band;

constexpr int kT = 256;
constexpr int kXS = 64;        // hi-res columns per CTA
constexpr int kJMax = 38;      // class quads: C <= 152

// state words: [0..1] double loss sum, [2] valid count, [3] float loss, [4] float 1/count
// T[j][column][q], class quads padded to kXS + 1 columns: row loop (fixed j, consecutive lanes = consecutive (column, q)) and
// phase 2 of the backward (fixed column, consecutive lanes = consecutive classes: quad stride 260 words = 4 banks) are both
// conflict-free
constexpr int kTQ = (kXS + 1) * 4;
__device__ __forceinline__ int t_index(int c, int xloc) { return (c >> 2) * kTQ + (xloc << 2) + (c & 3); }

__global__ void __launch_bounds__(kT, 2)
ce_up_fwd_kernel(const float* __restrict__ lo, int cs, int h, int w, const int64_t* __restrict__ labels, int C, int H, int W,
                 int ignore_label, float* __restrict__ lse_out, uint32_t* state, int maxcols) {
    extern __shared__ float s_dyn[];       // sT0[J][65][4] | sT1[J][65][4] | s_lo0[maxcols][C] | s_lo1[maxcols][C]
    __shared__ float s_red[33];
    const int J = (C + 3) >> 2;
    float* sT0 = s_dyn;
    float* sT1 = s_dyn + J * kTQ;
    float* s_lo0 = s_dyn + 2 * J * kTQ;
    float* s_lo1 = s_lo0 + maxcols * C;
    const float ry = area_scale(h, H), rx = area_scale(w, W);
    const int n = blockIdx.z, ci = blockIdx.y, x0 = blockIdx.x * kXS, x1 = min(W, x0 + kXS);
    const BandGeom g = band_geom(ry, rx, ci, x0, x1, h, H, w);
    if (g.ncols > maxcols) __trap();
    stage_rows<kT>(lo, cs, h, w, n, ci, g, C, C, s_lo0, s_lo1);
    __syncthreads();
    const int xloc = threadIdx.x >> 2, qd = threadIdx.x & 3;
    const int x = x0 + xloc;
    const bool xin = x < x1;
    const Lerp lx = make_lerp(rx, xin ? x : x0, w);
    const int j0 = lx.i0 - g.jbase, j1 = lx.i1 - g.jbase;
    blend_rows(lx, j0, j1, s_lo0, s_lo1, C, J, qd, 4, C, sT0, sT1, [&](int c) { return t_index(c, xloc); });
    // (thread-private entries: no barrier needed before the row loop; lanes of one pixel only read each other's entries for
    //  the TARGET class, so make the quad's writes visible to the quad)
    __syncwarp();
    float loss_acc = 0.f, cnt = 0.f;
    long long lab_next = xin ? labels[((long long)n * H + g.y_lo) * W + x] : 0;
    for (int y = g.y_lo; y <= g.y_hi; ++y) {
        const long long lab = lab_next;
        if (xin && y < g.y_hi) lab_next = labels[((long long)n * H + y + 1) * W + x];
        const Lerp ly = make_lerp(ry, y, h);
        if (ly.i0 != ci) continue;              // uniform across the CTA
        // (lanes with x outside the image run along on column x0's data and store nothing: the shuffles stay convergent)
        float v[kJMax];
        float m = -INFINITY;
#pragma unroll
        for (int j = 0; j < kJMax; ++j) {
            const int c = 4 * j + qd;
            v[j] = -INFINITY;
            if (c < C) {
                v[j] = lerp_v(ly, sT0[t_index(c, xloc)], sT1[t_index(c, xloc)]);
                m = fmaxf(m, v[j]);
            }
        }
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        float ssum = 0.f;
#pragma unroll
        for (int j = 0; j < kJMax; ++j)
            if (4 * j + qd < C) ssum += __expf(v[j] - m);
        ssum += __shfl_xor_sync(0xffffffffu, ssum, 1);
        ssum += __shfl_xor_sync(0xffffffffu, ssum, 2);
        const float lse = m + logf(ssum);
        const bool valid = xin && lab != (long long)ignore_label;
        if (qd == 0 && xin) {
            lse_out[((long long)n * H + y) * W + x] = lse;
            if (valid) {
                const int t = (int)lab;
                const float xt = lerp_v(ly, sT0[t_index(t, xloc)], sT1[t_index(t, xloc)]);
                loss_acc += lse - xt;
                cnt += 1.f;
            }
        }
    }
    loss_acc = block_sum<kT>(loss_acc, s_red);
    cnt = block_sum<kT>(cnt, s_red);
    if (threadIdx.x == 0 && cnt > 0.f) {
        atomicAdd(reinterpret_cast<double*>(state), (double)loss_acc);
        atomicAdd(&state[2], (unsigned int)cnt);
    }
}

__global__ void ce_up_finalize_kernel(uint32_t* state, float* loss_out) {
    const double s = *reinterpret_cast<double*>(state);
    const double c = (double)state[2];
    const float loss = (float)(s / c);           // 0/0 → NaN, as CrossEntropyLoss over zero valid pixels
    state[3] = __float_as_uint(loss);
    state[4] = __float_as_uint((float)(1.0 / c));
    if (loss_out) *loss_out = loss;
}

__global__ void __launch_bounds__(kT, 2)
ce_up_bwd_kernel(const float* __restrict__ lo, int cs, int h, int w, const int64_t* __restrict__ labels,
                 const float* __restrict__ lse_in, int C, int H, int W, int ignore_label, const uint32_t* __restrict__ state,
                 const float* __restrict__ gscale, float* __restrict__ dlo, int maxcols) {
    extern __shared__ float s_dyn[];       // sT0 / G0 | sT1 / G1 | s_lo0 | s_lo1 | s_oh[2][maxcols][C]
    __shared__ float s_l0[kXS], s_l1[kXS];
    __shared__ short s_seg[kXS + 8];
    const int J = (C + 3) >> 2;
    float* sT0 = s_dyn;
    float* sT1 = s_dyn + J * kTQ;
    float* s_lo0 = s_dyn + 2 * J * kTQ;
    float* s_lo1 = s_lo0 + maxcols * C;
    float* s_oh = s_lo1 + maxcols * C;
    const float wgt = __uint_as_float(state[4]) * (gscale ? *gscale : 1.f);
    const float ry = area_scale(h, H), rx = area_scale(w, W);
    const int n = blockIdx.z, ci = blockIdx.y, x0 = blockIdx.x * kXS, x1 = min(W, x0 + kXS);
    const int nx = x1 - x0;
    const BandGeom g = band_geom(ry, rx, ci, x0, x1, h, H, w);
    if (g.ncols > maxcols) __trap();
    stage_rows<kT, true>(lo, cs, h, w, n, ci, g, C, C, s_lo0, s_lo1, s_oh);   // and clear the one-hot tile
    const int xloc = threadIdx.x >> 2, qd = threadIdx.x & 3;
    const int x = x0 + xloc;
    const bool xin = x < x1;
    const Lerp lx = make_lerp(rx, xin ? x : x0, w);
    const int j0 = lx.i0 - g.jbase, j1 = lx.i1 - g.jbase;
    seg_init<kT>(s_l0, s_l1, s_seg, xloc, qd == 0, xin, lx, g.ncols, nx);
    __syncthreads();
    seg_fill(s_seg, xloc, qd == 0, xin, rx, x, w, g.jbase, j0);
    blend_rows(lx, j0, j1, s_lo0, s_lo1, C, J, qd, 4, C, sT0, sT1, [&](int c) { return t_index(c, xloc); });
    float G0[kJMax], G1[kJMax];
#pragma unroll
    for (int j = 0; j < kJMax; ++j) { G0[j] = 0.f; G1[j] = 0.f; }
    long long lab_next = 0;
    float lse_next = 0.f;
    if (xin) {
        const long long q0 = ((long long)n * H + g.y_lo) * W + x;
        lab_next = labels[q0];
        lse_next = lse_in[q0];
    }
    for (int y = g.y_lo; y <= g.y_hi; ++y) {
        const long long lab = lab_next;
        const float lse = lse_next;
        if (xin && y < g.y_hi) {
            const long long q1 = ((long long)n * H + y + 1) * W + x;
            lab_next = labels[q1];
            lse_next = lse_in[q1];
        }
        const Lerp ly = make_lerp(ry, y, h);
        if (ly.i0 != ci || !xin) continue;
        if (lab == (long long)ignore_label) continue;
#pragma unroll
        for (int j = 0; j < kJMax; ++j) {
            const int c = 4 * j + qd;
            if (c < C) {
                const float v = lerp_v(ly, sT0[t_index(c, xloc)], sT1[t_index(c, xloc)]);
                const float p = __expf(v - lse) * wgt;
                G0[j] = fmaf(ly.l0, p, G0[j]);
                G1[j] = fmaf(ly.l1, p, G1[j]);
            }
        }
        if (qd == 0) {
            const int t = (int)lab;
            const float a0 = -wgt * ly.l0, a1 = -wgt * ly.l1;
            atomicAdd(s_oh + j0 * C + t, a0 * lx.l0);
            atomicAdd(s_oh + j1 * C + t, a0 * lx.l1);
            atomicAdd(s_oh + (g.ncols + j0) * C + t, a1 * lx.l0);
            atomicAdd(s_oh + (g.ncols + j1) * C + t, a1 * lx.l1);
        }
    }
    // hand-over in place: entry (c, xloc) of sT0 / sT1 was only ever read by this thread (and its quad for the target class
    // in the forward kernel — not here)
#pragma unroll
    for (int j = 0; j < kJMax; ++j) {
        const int c = 4 * j + qd;
        if (c < C) { sT0[t_index(c, xloc)] = G0[j]; sT1[t_index(c, xloc)] = G1[j]; }
    }
    __syncthreads();
    // phase 2, starting from the one-hot tile
    const int npairs = g.ncols * C;
    for (int q = threadIdx.x; q < npairs; q += kT) {
        const int j = q / C, c = q - j * C;
        const float2 s = col_sums(sT0, sT1, [&](int xx) { return t_index(c, xx); }, s_seg, s_l0, s_l1, g, w, j,
                                  s_oh[j * C + c], s_oh[(g.ncols + j) * C + c]);
        if (s.x != 0.f) atomicAdd(dlo + (((long long)n * h + ci) * w + g.jbase + j) * cs + c, s.x);
        if (s.y != 0.f) atomicAdd(dlo + (((long long)n * h + g.i1) * w + g.jbase + j) * cs + c, s.y);
    }
}

// dynamic shared memory of the backward kernel, or 0 when it cannot run this geometry. The forward refuses those
// geometries too, so that a loss it accepts can always be differentiated.
static size_t bwd_smem(int C, int w, int W) {
    const int maxcols = band_maxcols(kXS, w, W);
    const size_t smem = sizeof(float) * (2 * (size_t)((C + 3) / 4) * kTQ + 4 * (size_t)maxcols * C);
    return maxcols <= kXS && smem <= 110 * 1024 ? smem : 0;
}

}  // namespace

extern "C" int tsb_ce_up_fwd(const float* logits_lo, int cs, int h, int w, const int64_t* labels, int N, int C, int H, int W,
                             int ignore_label, float* lse, uint32_t* state, float* loss_out, tsb_stream_t stream) {
    TSB_REQUIRE(logits_lo && labels && lse && state, "tsb_ce_up_fwd: null pointer");
    TSB_REQUIRE(N > 0 && N <= 65535 && h > 0 && h <= 65535 && w > 0 && H > 0 && W > 0, "tsb_ce_up_fwd: bad shape");
    TSB_REQUIRE(C >= 1 && C <= 4 * kJMax && cs >= C, "tsb_ce_up_fwd: 1 <= C <= %d", 4 * kJMax);
    TSB_REQUIRE(bwd_smem(C, w, W) != 0, "tsb_ce_up_fwd: up-scale factor W/w too small for the backward band kernel");
    const int maxcols = band_maxcols(kXS, w, W);
    const int J = (C + 3) / 4;
    const size_t smem = sizeof(float) * (2 * (size_t)J * kTQ + 2 * (size_t)maxcols * C);
    TSB_REQUIRE(smem <= 110 * 1024, "tsb_ce_up_fwd: up-scale factor W/w too small for the band kernel");
    cudaStream_t st = (cudaStream_t)stream;
    TSB_CUDA_CALL(cudaMemsetAsync(state, 0, sizeof(uint32_t) * 8, st));
    int rc = tsb_ensure_dyn_smem(reinterpret_cast<const void*>(ce_up_fwd_kernel), smem);
    if (rc) return rc;
    ce_up_fwd_kernel<<<dim3((W + kXS - 1) / kXS, h, N), kT, smem, st>>>(logits_lo, cs, h, w, labels, C, H, W, ignore_label, lse, state, maxcols);
    TSB_CUDA_CHECK_LAUNCH("ce_up_fwd");
    ce_up_finalize_kernel<<<1, 1, 0, st>>>(state, loss_out);
    TSB_CUDA_CHECK_LAUNCH("ce_up_finalize");
    return TSB_OK;
}

extern "C" int tsb_ce_up_bwd(const float* logits_lo, int cs, int h, int w, const int64_t* labels, const float* lse, int N, int C,
                             int H, int W, int ignore_label, const uint32_t* state, const float* gscale, float* dlogits_lo,
                             tsb_stream_t stream) {
    TSB_REQUIRE(logits_lo && labels && lse && state && dlogits_lo, "tsb_ce_up_bwd: null pointer");
    TSB_REQUIRE(N > 0 && N <= 65535 && h > 0 && h <= 65535 && w > 0 && H > 0 && W > 0, "tsb_ce_up_bwd: bad shape");
    TSB_REQUIRE(C >= 1 && C <= 4 * kJMax && cs >= C, "tsb_ce_up_bwd: 1 <= C <= %d", 4 * kJMax);
    const int maxcols = band_maxcols(kXS, w, W);
    TSB_REQUIRE(maxcols <= kXS, "tsb_ce_up_bwd: up-scale factor W/w too small for the band kernel");
    const size_t smem = bwd_smem(C, w, W);
    TSB_REQUIRE(smem != 0, "tsb_ce_up_bwd: shared memory budget exceeded");
    int rc = tsb_ensure_dyn_smem(reinterpret_cast<const void*>(ce_up_bwd_kernel), smem);
    if (rc) return rc;
    ce_up_bwd_kernel<<<dim3((W + kXS - 1) / kXS, h, N), kT, smem, (cudaStream_t)stream>>>(logits_lo, cs, h, w, labels, lse, C, H, W, ignore_label, state, gscale, dlogits_lo, maxcols);
    TSB_CUDA_CHECK_LAUNCH("ce_up_bwd");
    return TSB_OK;
}
