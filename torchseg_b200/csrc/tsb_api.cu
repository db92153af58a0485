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

// out[i] += slot[0][i] + slot[1][i] + ... in slot order. n is a channel count (often 64-512: one CTA), so each thread
// walks ~1000 slots alone; the slots are loaded kBatch at a time ahead of the adds, which stay one chain in slot order
// (same bits), instead of the few loads per L2 round trip the plain loop kept in flight.
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

int tsb_det_reduce(float* out, const float* parts, int nparts, long long n, long long stride, cudaStream_t st) {
    det_reduce_kernel<<<tsb_grid_for(n, 256, 8), 256, 0, st>>>(out, parts, nparts, n, stride);
    TSB_CUDA_CHECK_LAUNCH("det_reduce");
    return TSB_OK;
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
