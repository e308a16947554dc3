// michigan_b200 — C-ABI glue: error strings, launch counter, driver entry points.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <mutex>
#include <cstdlib>
#include <cstring>
#include "mg_internal.h"

namespace mg {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

int set_error(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int num_sms() {
    static thread_local int cached_dev = -1, cached = 0;
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev != cached_dev) {
        cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, dev);
        cached_dev = dev;
    }
    return cached;
}

// ---------------------------------------------------------------------------------------------- tuning knobs
struct KnobDef { const char* env; int dflt; };
static const KnobDef kKnobs[TK_COUNT] = {
    {"MG_DUAL", 2}, {"MG_MERGE", 1}, {"MG_HALO", 0}, {"MG_HALO_PW", 10}, {"MG_EPI_IMPL", 1}, {"MG_EPI_IMPL_SPADE", -1},
    {"MG_EPI_CW16", 1}, {"MG_EPI_CW_SPADE", 16}, {"MG_STAGES", 0}, {"MG_WGRAD_DUAL", 1}, {"MG_THIN_GEMM", 1},
    {"MG_THIN_WGRAD_LEGACY", 0}, {"MG_GROUP3", 1}, {"MG_SEG_TMA", 1}, {"MG_WGRAD_HALO", 1}, {"MG_EPI_TMA", 2}, {"MG_BN_FILL", 1}, {"MG_EPI_EARLY", 0},
};
static std::atomic<int> g_knob[TK_COUNT];
static std::once_flag g_knob_once;

static void knobs_init() {
    std::call_once(g_knob_once, [] {
        for (int i = 0; i < TK_COUNT; ++i) {
            const char* v = getenv(kKnobs[i].env);
            g_knob[i].store(v ? atoi(v) : kKnobs[i].dflt, std::memory_order_relaxed);
        }
        if (g_knob[TK_EPI_IMPL_SPADE].load() < 0) g_knob[TK_EPI_IMPL_SPADE].store(g_knob[TK_EPI_IMPL].load());
    });
}

int tune(int knob) {
    knobs_init();
    return g_knob[knob].load(std::memory_order_relaxed);
}

#ifdef MG_PROBES
int probe_bits() {
    const char* e = getenv("MG_DBG");   // probe build only: re-read on every launch so that a tool can switch probes in-process
    return e ? atoi(e) : 0;
}
#endif

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
        if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

int encode_tensor_map(CUtensorMap* map, void* gaddr, CUtensorMapDataType dtype, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                      const cuuint32_t* box, const cuuint32_t* estrides, CUtensorMapSwizzle swizzle) {
    // Per-thread direct-mapped cache: a layer re-launched on the same buffers (the caching allocator hands the same
    // addresses back every iteration) reuses its 128-byte descriptor instead of calling into the driver.
    struct Key {
        void* gaddr; int dtype, rank, swizzle;
        cuuint64_t dims[4], strides[3];
        cuuint32_t box[4], estr[4];
    };
    struct Entry { Key key; CUtensorMap map; bool valid; };
    constexpr int kSlots = 1024;
    static thread_local Entry* cache = nullptr;
    if (!cache) cache = static_cast<Entry*>(calloc(kSlots, sizeof(Entry)));
    Key k;
    memset(&k, 0, sizeof(k));
    k.gaddr = gaddr; k.dtype = (int)dtype; k.rank = rank; k.swizzle = (int)swizzle;
    for (int i = 0; i < rank; ++i) { k.dims[i] = dims[i]; k.box[i] = box[i]; k.estr[i] = estrides[i]; }
    for (int i = 0; i + 1 < rank; ++i) k.strides[i] = strides[i];
    unsigned long long h = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(Key) / 8; ++i) h = (h ^ reinterpret_cast<const unsigned long long*>(&k)[i]) * 1099511628211ull;
    Entry* e = cache ? &cache[(h ^ (h >> 29)) & (kSlots - 1)] : nullptr;
    if (e && e->valid && memcmp(&e->key, &k, sizeof(Key)) == 0) { *map = e->map; return 0; }
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return set_error(-100, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    CUresult r = fn(map, dtype, (cuuint32_t)rank, gaddr, dims, strides, box, estrides,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return set_error(-101, "cuTensorMapEncodeTiled failed: CUresult %d (rank %d, dims %llu %llu, box %u %u)", (int)r,
                         rank, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    if (e) { e->key = k; e->map = *map; e->valid = true; }
    return 0;
}

// ---------------------------------------------------------------------------------------------- order-independent sums
// The buffers come from a memory pool of this library (one per device, created on first use) that keeps freed blocks
// cached: the train step allocates a few MB per backward kernel, and a pool that trimmed at every synchronisation would
// hand them back to the driver each step.  Allocation stays stream-ordered, so concurrent streams never share a buffer.
static cudaMemPool_t acc64_pool(int dev) {
    static std::mutex mu;
    static cudaMemPool_t pools[64] = {};
    std::lock_guard<std::mutex> lock(mu);
    if (dev < 0 || dev >= 64) return nullptr;
    if (!pools[dev]) {
        cudaMemPoolProps props = {};
        props.allocType = cudaMemAllocationTypePinned;
        props.location.type = cudaMemLocationTypeDevice;
        props.location.id = dev;
        cudaMemPool_t pool = nullptr;
        if (cudaMemPoolCreate(&pool, &props) != cudaSuccess) return nullptr;
        unsigned long long keep = ~0ull;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        pools[dev] = pool;
    }
    return pools[dev];
}

int acc64_alloc(double** acc, size_t n, cudaStream_t stream) {
    *acc = nullptr;
    int dev = 0;
    cudaGetDevice(&dev);
    cudaMemPool_t pool = acc64_pool(dev);
    if (!pool) return set_error(-1, "acc64_alloc: no memory pool for device %d", dev);
    cudaError_t e = cudaMallocFromPoolAsync(reinterpret_cast<void**>(acc), n * sizeof(double), pool, stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(*acc, 0, n * sizeof(double), stream);
    if (e != cudaSuccess) return set_error((int)e, "acc64_alloc: %s", cudaGetErrorString(e));
    return 0;
}

__global__ void acc64_fold_kernel(const double* __restrict__ acc, float* __restrict__ dst, long long n, int add) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        dst[i] = (add ? dst[i] : 0.f) + (float)acc[i];
}

int acc64_fold(const double* acc, float* dst, size_t n, int add, cudaStream_t stream) {
    long long blocks = ((long long)n + 255) / 256;
    if (blocks > 4096) blocks = 4096;
    if (blocks < 1) blocks = 1;
    acc64_fold_kernel<<<(int)blocks, 256, 0, stream>>>(acc, dst, (long long)n, add);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error((int)e, "acc64_fold: %s", cudaGetErrorString(e));
    return 0;
}

int acc64_free(double* acc, cudaStream_t stream) {
    cudaError_t e = cudaFreeAsync(acc, stream);
    if (e != cudaSuccess) return set_error((int)e, "acc64_free: %s", cudaGetErrorString(e));
    return 0;
}

}  // namespace mg

extern "C" int mg_version(void) { return MG_ABI_VERSION; }
extern "C" const char* mg_last_error(void) { return mg::g_err; }
extern "C" long long mg_launch_count(void) { return mg::g_launches.load(); }

extern "C" int mg_set_tuning(const char* name, int value) {
    if (!name) return mg::set_error(-1, "mg_set_tuning: null name");
    mg::knobs_init();
    for (int i = 0; i < mg::TK_COUNT; ++i)
        if (strcmp(name, mg::kKnobs[i].env) == 0) { mg::g_knob[i].store(value); return 0; }
    return mg::set_error(-2, "mg_set_tuning: unknown knob %s", name);
}

extern "C" int mg_get_tuning(const char* name) {
    if (!name) return -1;
    for (int i = 0; i < mg::TK_COUNT; ++i)
        if (strcmp(name, mg::kKnobs[i].env) == 0) return mg::tune(i);
    return -1;
}
