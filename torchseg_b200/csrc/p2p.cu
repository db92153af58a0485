// Device-initiated all-reduce of SMALL fp32 vectors over NVLink peer memory — the SyncBatchNorm statistics exchange
// (replaces apex SyncBatchNorm's per-layer all-reduce, TorchSeg model/bisenet/cityscapes.bisenet.R18/train.py:54-55).
//
// A BiSeNet step has ~70 of these exchanges ([Σx | Σx²] forward, [Σdz | Σdz·x̂] backward; 128..8192 floats each): with NCCL
// every one costs a launch + protocol latency of 25-40 us on the compute stream, i.e. the whole weak-scaling loss of the
// step. Here ONE small kernel per exchange writes the local partial sums straight into every peer's symmetric buffer
// (NVLink stores), waits for the partials of all peers to land in its own buffer and reduces the `world` partials in rank
// order (identical result bits on every rank, run-to-run deterministic).
//
// Protocol ("LL": the flag travels WITH the data, no memory fences): every fp32 value is stored as an 8-byte pair
// {value bits, seq}; 8-byte stores are single transactions over NVLink, so a reader that sees seq in a pair has the value.
// The alternative (data stores + __threadfence_system + st.release.sys / ld.acquire.sys flags) pays system-scope fences
// with peer writes in flight on every exchange; the fence-free form needs one NVLink store latency.
//
// Symmetric buffer of every rank (allocated and exchanged by the caller, e.g. torch symmetric memory):
//   [nslots] x { uint2 pair[world][slot_floats] }
// Exchange number `seq` (1, 2, 3, ... identical on all ranks: every rank executes the same layer sequence) uses slot
// seq % nslots; pairs of an older use of the slot carry an older seq and never match, so nothing is ever reset. A slot is
// re-used only after nslots-1 other exchanges, each of which orders all ranks, so a writer can never overtake a reader.
#include "tsb_common.cuh"

namespace {

constexpr int kXThreads = 1024;

__device__ __forceinline__ void st_volatile_v4(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint4 ld_volatile_v4(const void* p) {
    uint4 v;
    asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}

struct XchgParams {
    float* vals;                 // [n] local partial sums in, global sums out (n % 4 == 0)
    int n;
    unsigned long long peers[TSB_P2P_MAX_WORLD];   // symmetric buffer base address on every rank (peer-mapped)
    int rank, world;
    unsigned int seq;
    unsigned int* seq_dev;       // optional device-resident exchange counter (pre-incremented here): lets a captured CUDA
                                 // graph replay the exchange with a fresh sequence number every time
    int nslots, slot_floats;
    float* acc_hi;               // optional: acc_hi[c] += vals[half + c]  (LOCAL Σdz·x̂ → dgamma) before the exchange
    float* acc_lo;               //           acc_lo[c] += vals[c]         (LOCAL Σdz   → dbeta)
    int half;
};

__global__ void __launch_bounds__(kXThreads, 1) p2p_allreduce_kernel(XchgParams p) {
    if (p.seq_dev != nullptr) {      // exchanges are serialised on the stream: a plain read-modify-write by one thread
        __shared__ unsigned int s_seq;
        if (threadIdx.x == 0) {
            unsigned int v = *p.seq_dev + 1u;
            if (v == 0u) v = 1u;     // 0 is the "never written" value of a fresh buffer
            *p.seq_dev = v;
            s_seq = v;
        }
        __syncthreads();
        p.seq = s_seq;
    }
    const size_t slot_bytes = (size_t)p.world * p.slot_floats * 8;
    const size_t slot_off = (size_t)(p.seq % (unsigned)p.nslots) * slot_bytes;
    const int n2 = p.n >> 1;     // one thread-iteration = two values = one 16-byte {v0, seq, v1, seq} store
    // 1. my partials → region [rank] of the slot on every rank (own copy included); local dgamma / dbeta first
    for (int i = threadIdx.x; i < n2; i += kXThreads) {
        const float2 v = *reinterpret_cast<const float2*>(p.vals + 2 * i);
        if (p.acc_hi != nullptr) {
            float* acc = (2 * i < p.half) ? p.acc_lo + 2 * i : p.acc_hi + (2 * i - p.half);
            acc[0] += v.x;
            acc[1] += v.y;
        }
        for (int r = 0; r < p.world; ++r) {
            uint8_t* dst = reinterpret_cast<uint8_t*>(p.peers[r] + slot_off) + ((size_t)p.rank * p.slot_floats + 2 * i) * 8;
            st_volatile_v4(dst, __float_as_uint(v.x), p.seq, __float_as_uint(v.y), p.seq);
        }
    }
    // 2. every thread waits for ITS pairs from every rank in my buffer and reduces them in rank order (identical bits on
    //    all ranks). Bounded: a dead or diverged peer traps after ~20 s instead of hanging the box.
    const uint8_t* mine = reinterpret_cast<const uint8_t*>(p.peers[p.rank] + slot_off);
    const long long t0 = clock64();
    for (int i = threadIdx.x; i < n2; i += kXThreads) {
        float s0 = 0.f, s1 = 0.f;
        for (int r = 0; r < p.world; ++r) {
            const uint8_t* src = mine + ((size_t)r * p.slot_floats + 2 * i) * 8;
            uint4 q = ld_volatile_v4(src);
            unsigned int spins = 0;
            while (q.y != p.seq || q.w != p.seq) {
                if ((++spins & 0x3ffu) == 0 && clock64() - t0 > 40000000000ll) __trap();
                q = ld_volatile_v4(src);
            }
            s0 += __uint_as_float(q.x);
            s1 += __uint_as_float(q.z);
        }
        *reinterpret_cast<float2*>(p.vals + 2 * i) = make_float2(s0, s1);
    }
}

}  // namespace

extern "C" size_t tsb_p2p_buffer_bytes(int world, int nslots, int slot_floats) {
    if (world < 1 || nslots < 2 || slot_floats < 4) return 0;
    return (size_t)world * slot_floats * 8 * (size_t)nslots;   // {value, seq} pairs
}

extern "C" int tsb_p2p_allreduce_sum(float* vals, int n, const unsigned long long* peer_bases, int rank, int world,
                                     unsigned int seq, unsigned int* seq_dev, int nslots, int slot_floats, float* acc_hi,
                                     float* acc_lo, tsb_stream_t stream) {
    TSB_REQUIRE(vals && peer_bases, "tsb_p2p_allreduce_sum: null pointer");
    TSB_REQUIRE(world >= 1 && world <= TSB_P2P_MAX_WORLD && rank >= 0 && rank < world, "tsb_p2p_allreduce_sum: bad rank/world");
    TSB_REQUIRE(n > 0 && n % 4 == 0 && n <= slot_floats && slot_floats % 4 == 0, "tsb_p2p_allreduce_sum: n must be a multiple of 4 and fit a slot (n=%d, slot=%d)", n, slot_floats);
    TSB_REQUIRE(nslots >= 2 && (seq != 0 || seq_dev != nullptr), "tsb_p2p_allreduce_sum: nslots >= 2, seq >= 1 (or a device counter)");
    TSB_REQUIRE((acc_hi == nullptr) == (acc_lo == nullptr) && (acc_hi == nullptr || n % 2 == 0), "tsb_p2p_allreduce_sum: accumulators go together");
    TSB_REQUIRE(tsb_aligned16(vals), "tsb_p2p_allreduce_sum: vals must be 16-byte aligned");
    XchgParams prm;
    memset(&prm, 0, sizeof(prm));
    prm.vals = vals; prm.n = n;
    for (int r = 0; r < world; ++r) {
        TSB_REQUIRE(peer_bases[r] != 0 && peer_bases[r] % 128 == 0, "tsb_p2p_allreduce_sum: peer base %d missing / not 128-byte aligned", r);
        prm.peers[r] = peer_bases[r];
    }
    prm.rank = rank; prm.world = world; prm.seq = seq; prm.seq_dev = seq_dev; prm.nslots = nslots; prm.slot_floats = slot_floats;
    prm.acc_hi = acc_hi; prm.acc_lo = acc_lo; prm.half = n / 2;
    p2p_allreduce_kernel<<<1, kXThreads, 0, (cudaStream_t)stream>>>(prm);
    TSB_CUDA_CHECK_LAUNCH("p2p_allreduce");
    return TSB_OK;
}
