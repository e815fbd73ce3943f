// tooncrafter_b200 — error state, launch counter, TMA descriptor cache.
#include <stdlib.h>
#include "tc_host.h"

#include <atomic>
#include <cstring>
#include <mutex>
#include <unordered_map>
#include <vector>

namespace tc_host {

static thread_local std::string g_err;
static std::atomic<unsigned long long> g_launches{0};

void set_error(const std::string& msg) { g_err = msg; }
int fail(int code, const std::string& msg) {
    g_err = msg;
    return code;
}
int check_cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return 0;
    g_err = std::string(what) + ": " + cudaGetErrorString(e);
    return TC_ERR_CUDA;
}
void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

int sm_count() {
    static int cached = 0;
    if (cached == 0) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) == cudaSuccess &&
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
            cached = n;
        else
            cached = 132;
    }
    return cached;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

struct MapKey {
    uint64_t v[15];
    bool operator==(const MapKey& o) const { return std::memcmp(v, o.v, sizeof(v)) == 0; }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        uint64_t h = 1469598103934665603ull;
        for (int i = 0; i < 15; ++i) {
            h ^= k.v[i];
            h *= 1099511628211ull;
        }
        return (size_t)h;
    }
};

static std::mutex g_map_mu;
// node-based container: pointers to values stay valid across inserts
static std::unordered_map<MapKey, CUtensorMap*, MapKeyHash> g_maps;

const CUtensorMap* get_tensor_map(const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                                  const uint32_t* box, int swizzle_bytes) {
    MapKey key;
    std::memset(&key, 0, sizeof(key));
    key.v[0] = reinterpret_cast<uint64_t>(base);
    key.v[1] = (uint64_t)rank;
    for (int i = 0; i < rank; ++i) key.v[2 + i] = dims[i];
    for (int i = 0; i + 1 < rank; ++i) key.v[6 + i] = strides_bytes[i];
    for (int i = 0; i < rank; ++i) key.v[10 + i] = box[i];
    key.v[14] = (uint64_t)swizzle_bytes;

    std::lock_guard<std::mutex> lk(g_map_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) return it->second;

    EncodeTiledFn enc = get_encode_fn();
    if (!enc) {
        set_error("cuTensorMapEncodeTiled entry point unavailable");
        return nullptr;
    }
    void* mem = nullptr;
    if (posix_memalign(&mem, 64, sizeof(CUtensorMap)) != 0) {
        set_error("posix_memalign failed");
        return nullptr;
    }
    CUtensorMap* m = reinterpret_cast<CUtensorMap*>(mem);
    cuuint64_t gdim[4];
    cuuint64_t gstr[3];
    cuuint32_t bx[4];
    cuuint32_t es[4];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bx[i] = box[i];
        es[i] = 1;
    }
    for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx,
                     es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swizzle_bytes == 32   ? CU_TENSOR_MAP_SWIZZLE_32B
                     : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                           : CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char buf[256];
        snprintf(buf, sizeof(buf),
                 "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu] strides [%llu %llu %llu] "
                 "box [%u %u %u %u]",
                 (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
                 (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
                 (unsigned long long)(rank > 1 ? strides_bytes[0] : 0),
                 (unsigned long long)(rank > 2 ? strides_bytes[1] : 0),
                 (unsigned long long)(rank > 3 ? strides_bytes[2] : 0), box[0], rank > 1 ? box[1] : 0,
                 rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
        set_error(buf);
        free(mem);
        return nullptr;
    }
    g_maps.emplace(key, m);
    return m;
}

bool pdl_enabled() {
    static const bool on = [] {
        const char* e = getenv("TC_PDL");
        return !(e && e[0] == '0');
    }();
    return on;
}

}  // namespace tc_host

extern "C" {
const char* tc_last_error(void) { return tc_host::g_err.c_str(); }
int tc_version(void) { return 102; }
unsigned long long tc_launch_count(void) { return tc_host::g_launches.load(); }
int tc_sm_count(void) { return tc_host::sm_count(); }
}
