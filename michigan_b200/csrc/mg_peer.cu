// michigan_b200 — one-shot small all-reduce over NVLink peer memory (sm_90a).
//
// The SyncBN statistics exchange of the reference (batchnorm.py:105-126: every replica sends [sum | sum of squares]
// to the master through Python queues, comm.py:49-133; the master reduce-adds and broadcasts mean / inv_std) is a
// 2*C-double message, C <= 1024.  Here every rank PUSHES its vector into a slot of every peer's symmetric buffer
// (plain stores over NVLink / NVSwitch), publishes a sequence number with a system-scope release store, waits for the
// sequence numbers of all peers in its OWN memory (local polling), and then sums the world_size vectors in rank order
// - every rank performs the same additions in the same order, so the result is bit-identical on all ranks (the
// reference's broadcast guarantee) without a second exchange.  One kernel, one CTA, no host round trip, no NCCL call.
//
// Buffer (same layout on every rank, allocated by the host as symmetric / peer-mapped memory):
//     data : kSlots x world x kMaxN doubles        slot = seq % kSlots, row = source rank
//     flags: kSlots x world unsigned long long     sequence number of the last vector written into (slot, source)
// Slot reuse is safe with kSlots >= 2: a rank starts exchange s+1 only after it has read every peer's vector of
// exchange s, and a peer can only be one exchange ahead of the slowest rank it waits for.
#include <cuda_runtime.h>
#include "mg_internal.h"

namespace mg {

constexpr int kPeerSlots = 4;
constexpr int kPeerMaxN = 2 * 1024 + 8;
constexpr int kPeerMaxWorld = 16;

struct PeerParams {
    double* data;
    int n, world, rank;
    unsigned long long seq;
    unsigned char* bufs[kPeerMaxWorld];
    int* status;
    long long timeout_cycles;
    double tail;      // set_tail: data[n-1] = tail before the push (the per-rank sample count travelling with the sums)
    int set_tail;
};

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_sys_f64(double* p, double v) {
    asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ double ld_relaxed_sys_f64(const double* p) {
    double v;
    asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
    return v;
}

__host__ __device__ inline size_t peer_flags_offset(int world) { return (size_t)kPeerSlots * world * kPeerMaxN * sizeof(double); }

__global__ void __launch_bounds__(512, 1) peer_allreduce_kernel(const PeerParams p) {
    const int tid = threadIdx.x;
    const int slot = (int)(p.seq % kPeerSlots);
    const size_t row = ((size_t)slot * p.world + p.rank) * kPeerMaxN;
    // 1. push this rank's vector into row `rank` of slot `slot` on every rank (own buffer included)
    for (int i = tid; i < p.n; i += blockDim.x) {
        const double v = (p.set_tail && i == p.n - 1) ? p.tail : p.data[i];
        for (int r = 0; r < p.world; ++r) st_relaxed_sys_f64(reinterpret_cast<double*>(p.bufs[r]) + row + i, v);
    }
    __syncthreads();
    // 2. publish: release at system scope orders the CTA's stores (observed through the barrier) before the flag
    if (tid < p.world) {
        unsigned long long* f = reinterpret_cast<unsigned long long*>(p.bufs[tid] + peer_flags_offset(p.world)) + (size_t)slot * p.world + p.rank;
        __threadfence_system();
        st_release_sys(f, p.seq);
    }
    // 3. wait for every rank's vector of THIS exchange in local memory
    if (tid < p.world) {
        const unsigned long long* f = reinterpret_cast<const unsigned long long*>(p.bufs[p.rank] + peer_flags_offset(p.world)) + (size_t)slot * p.world + tid;
        const long long t0 = clock64();
        while (ld_acquire_sys(f) != p.seq) {
            if (clock64() - t0 > p.timeout_cycles) {   // a peer died or the call sequences diverged: report, do not hang the GPU
                atomicExch(p.status, 1);
                break;
            }
            __nanosleep(64);
        }
    }
    __syncthreads();
    // 4. rank-ordered sum (identical on every rank)
    const double* mine = reinterpret_cast<const double*>(p.bufs[p.rank]) + (size_t)slot * p.world * kPeerMaxN;
    for (int i = tid; i < p.n; i += blockDim.x) {
        double s = 0.0;
        for (int r = 0; r < p.world; ++r) s += ld_relaxed_sys_f64(mine + (size_t)r * kPeerMaxN + i);
        p.data[i] = s;
    }
}

}  // namespace mg

extern "C" long long mg_peer_buffer_bytes(int world) {
    if (world < 1 || world > mg::kPeerMaxWorld) return -1;
    return (long long)(mg::peer_flags_offset(world) + (size_t)mg::kPeerSlots * world * sizeof(unsigned long long));
}

extern "C" int mg_peer_max_elems(void) { return mg::kPeerMaxN; }

extern "C" int mg_peer_allreduce_f64(double* data, int n, const void* const* peer_bufs, int world, int rank, unsigned long long seq,
                                     int set_tail, double tail, int* status_dev, void* stream) {
    using namespace mg;
    if (!data || !peer_bufs || !status_dev) return set_error(-1, "mg_peer_allreduce_f64: null pointer");
    if (world < 2 || world > kPeerMaxWorld || rank < 0 || rank >= world)
        return set_error(-2, "mg_peer_allreduce_f64: bad world/rank %d/%d (2 <= world <= %d)", world, rank, kPeerMaxWorld);
    if (n < 1 || n > kPeerMaxN) return set_error(-3, "mg_peer_allreduce_f64: n = %d outside [1, %d]", n, kPeerMaxN);
    if (seq == 0) return set_error(-4, "mg_peer_allreduce_f64: sequence numbers start at 1 (the flags are zero-initialised)");
    PeerParams p;
    p.data = data; p.n = n; p.world = world; p.rank = rank; p.seq = seq; p.status = status_dev;
    p.timeout_cycles = 8000000000LL;   // ~4 s at 1.9 GHz
    p.tail = tail; p.set_tail = set_tail;
    for (int r = 0; r < kPeerMaxWorld; ++r) p.bufs[r] = r < world ? (unsigned char*)peer_bufs[r] : nullptr;
    for (int r = 0; r < world; ++r)
        if (!p.bufs[r]) return set_error(-5, "mg_peer_allreduce_f64: null peer buffer %d", r);
    peer_allreduce_kernel<<<1, 512, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return check_launch("mg_peer_allreduce_f64");
}
