// tooncrafter_b200 — host-side helpers shared by the C-ABI translation units.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <string>
#include <utility>

#include "../../include/tooncrafter_b200.h"

namespace tc_host {

void set_error(const std::string& msg);
int fail(int code, const std::string& msg);
int check_cuda(cudaError_t e, const char* what);
void count_launch(int n = 1);
int sm_count();

// Cached cuTensorMapEncodeTiled: fp16 tensor of `rank` dims (dim 0 contiguous), 128B (or 64B / 32B) swizzle,
// zero fill out of bounds.  strides are in BYTES for dims 1..rank-1.
const CUtensorMap* get_tensor_map(const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                                  const uint32_t* box, int swizzle_bytes = 128);

// TC_PDL=0 in the environment turns programmatic dependent launch off (A/B testing)
bool pdl_enabled();

// Every kernel launch of the library: programmatic stream serialization (the kernel's prologue and launch latency
// overlap the predecessor's tail; all kernels call griddepcontrol.wait before touching global memory), optional
// 2-CTA cluster.  The result is reported through cudaGetLastError() like a <<<>>> launch.
template <typename... KArgs, typename... Args>
inline void launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, int cluster_x,
                   Args&&... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    int n = 0;
    if (pdl_enabled()) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (cluster_x > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = (unsigned)cluster_x;
        attr[n].val.clusterDim.y = 1;
        attr[n].val.clusterDim.z = 1;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = (unsigned)n;
    (void)cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...);
}

}  // namespace tc_host

#define TC_CHECK_ARG(cond, msg)                                      \
    do {                                                             \
        if (!(cond)) return tc_host::fail(TC_ERR_INVALID, (msg));    \
    } while (0)

#define TC_CHECK_LAUNCH(what)                                        \
    do {                                                             \
        int _rc = tc_host::check_cuda(cudaGetLastError(), (what));   \
        if (_rc) return _rc;                                         \
    } while (0)
