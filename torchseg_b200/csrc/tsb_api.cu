// libtsb: library-level entry points (error string, version, launch counter).
#include <stdarg.h>
#include <atomic>
#include <map>
#include <mutex>
#include <utility>

#include "tsb_common.cuh"

static thread_local char g_err[512] = "";
std::atomic<long long> g_tsb_launches{0};

void tsb_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

void tsb_count_launch(int n) { g_tsb_launches.fetch_add(n, std::memory_order_relaxed); }

// out[i] += slot[0][i] + slot[1][i] + ... in slot order: s = 0; s += slot[0][i]; s += slot[1][i]; ...; out[i] += s.
// Both kernels below run exactly this chain per output, so they give the same bits.
//
// Grid-wide form, for large n (weight-gradient split slices: n ~ 10^4-10^6, few slots) and for calls of at most kBatch
// slots: one thread per output, the slots loaded kBatch at a time ahead of the adds.
__global__ void det_reduce_kernel(float* __restrict__ out, const float* __restrict__ parts, int nparts, long long n,
                                  long long stride) {
    constexpr int kBatch = 32;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float s = 0.f;
        int b = 0;
        for (; b + kBatch <= nparts; b += kBatch) {
            float v[kBatch];
#pragma unroll
            for (int u = 0; u < kBatch; ++u) v[u] = __ldg(parts + (long long)(b + u) * stride + i);
#pragma unroll
            for (int u = 0; u < kBatch; ++u) s += v[u];
        }
        for (; b < nparts; ++b) s += parts[(long long)b * stride + i];
        out[i] += s;
    }
}

// Column form, for small n (BatchNorm and conv-epilogue statistics: n = C or 2C = 64-1024 outputs, up to 8 x 132
// slots). One thread per output cannot be fed by the grid-wide form there: 1-4 CTAs, each thread ~33 dependent L2 round
// trips. Here a CTA owns kColG consecutive outputs (one 32-byte sector of every slot row), so a 2 x 64-channel pair runs
// on 16 CTAs. All its threads stage kColRows slot rows at a time into shared memory with cp.async (many loads in
// flight, the next chunk landing while the current one is summed), and thread j < kColG adds column j in slot order
// from shared memory: the time is about one L2 round trip plus the 4-cycle add chain of nparts slots. kVec is the
// floats per copy: 4 when every row of the group is 16-byte aligned, else 1.
constexpr int kColG = 8, kColThreads = 256, kColRows = 256;

template <int kVec>
__global__ void __launch_bounds__(kColThreads) det_reduce_cols_kernel(float* __restrict__ out, const float* __restrict__ parts,
                                                                      int nparts, long long n, long long stride) {
    __shared__ __align__(16) float buf[2][kColRows][kColG];
    constexpr int kPerRow = kColG / kVec;
    const long long i0 = (long long)blockIdx.x * kColG;
    const int width = (int)min((long long)kColG, n - i0);   // outputs of this group (< kColG only in the last)
    const int nchunks = (nparts + kColRows - 1) / kColRows;
    auto stage = [&](int c) {
        const int r0 = c * kColRows, rows = min(kColRows, nparts - r0);
        float(*dst)[kColG] = buf[c & 1];
        for (int e = threadIdx.x; e < rows * kPerRow; e += kColThreads) {
            const int r = e / kPerRow, v = (e % kPerRow) * kVec;
            const float* row = parts + (long long)(r0 + r) * stride + i0;
            const int bytes = 4 * max(0, min(kVec, width - v));   // columns past n are zero-filled, never read
            const uint32_t s = (uint32_t)__cvta_generic_to_shared(&dst[r][v]);
            if (kVec == 4)
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(bytes ? row + v : row), "r"(bytes) : "memory");
            else
                asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(s), "l"(bytes ? row + v : row), "r"(bytes) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    float sum = 0.f;
    stage(0);
    for (int c = 0; c < nchunks; ++c) {
        if (c + 1 < nchunks) {
            stage(c + 1);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();   // chunk c landed for every thread
        if (threadIdx.x < width) {
            const float(*src)[kColG] = buf[c & 1];
            const int rows = min(kColRows, nparts - c * kColRows);
#pragma unroll 16
            for (int r = 0; r < rows; ++r) sum += src[r][threadIdx.x];
        }
        __syncthreads();   // buffer c & 1 is free for chunk c + 2
    }
    if (threadIdx.x < width) out[i0 + threadIdx.x] += sum;
}

int tsb_det_reduce(float* out, const float* parts, int nparts, long long n, long long stride, cudaStream_t st) {
    // The column form wins when the chains are long (more than the one batch of 32 loads the grid-wide form issues per
    // dependent round trip) and the outputs few. Measured per call on an H100: the grid-wide form stays ahead at <= 32
    // slots and at 1024 column CTAs (8192 outputs, 256 slots), the column form is ahead at 608 CTAs (4864 outputs).
    const long long groups = (n + kColG - 1) / kColG;
    if (nparts > 32 && groups <= 5LL * tsb_num_sms()) {
        if (tsb_aligned16(parts) && stride % 4 == 0)
            det_reduce_cols_kernel<4><<<(int)groups, kColThreads, 0, st>>>(out, parts, nparts, n, stride);
        else
            det_reduce_cols_kernel<1><<<(int)groups, kColThreads, 0, st>>>(out, parts, nparts, n, stride);
    } else {
        det_reduce_kernel<<<tsb_grid_for(n, 256, 8), 256, 0, st>>>(out, parts, nparts, n, stride);
    }
    TSB_CUDA_CHECK_LAUNCH("det_reduce");
    return TSB_OK;
}

int tsb_det_reduce_pair(float* out_a, float* out_b, const float* parts, int nparts, long long C, cudaStream_t st) {
    if (out_b == out_a + C) return tsb_det_reduce(out_a, parts, nparts, 2 * C, 2 * C, st);
    const int rc = tsb_det_reduce(out_a, parts, nparts, C, 2 * C, st);
    return rc ? rc : tsb_det_reduce(out_b, parts + C, nparts, C, 2 * C, st);
}

extern "C" const char* tsb_last_error(void) { return g_err; }
extern "C" int tsb_version(void) { return 100; }
extern "C" long long tsb_launch_count(void) { return g_tsb_launches.load(); }

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-(device, function) property: remember what was already raised for
// each pair under a mutex (autograd's backward thread and the forward thread both launch kernels; a process may drive
// several devices).
int tsb_ensure_dyn_smem(const void* func, size_t bytes) {
    static std::mutex mu;
    static std::map<std::pair<int, const void*>, size_t> done;
    int dev = 0;
    TSB_CUDA_CALL(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(mu);
    size_t& have = done[std::make_pair(dev, func)];
    if (bytes > have) {   // monotonic: exactly what is asked for (static + dynamic shared memory must fit 227 KB)
        TSB_CUDA_CALL(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        have = bytes;
    }
    return TSB_OK;
}
