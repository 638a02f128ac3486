// Host-side helpers shared by the C-ABI translation units: error reporting and TMA descriptor encoding.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aniportrait_b200.h"

namespace ap {

// printf-style; stores the message in a thread-local buffer read by ap_last_error(). Returns `code`.
int fail(int code, const char* fmt, ...);

// cuTensorMapEncodeTiled resolved through cudaGetDriverEntryPoint (no link-time libcuda dependency, so the
// library also loads on a CPU-only box for symbol checks).
// dims/box are innermost-first; strides_bytes has rank-1 entries (stride of dim 1..rank-1).
int encode_tmap(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                const uint32_t* box, bool swizzle128, int elem_bytes = 2, int swizzle_bytes = 0);

int num_sms();

// Programmatic dependent launch (PDL): every kernel of the library is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization and starts with griddepcontrol.launch_dependents (the next kernel of the
// stream may be scheduled as soon as all CTAs of this one are running) followed — after its data-independent prologue
// (barrier init, descriptor prefetch) — by griddepcontrol.wait (blocks until the previous kernel has
// completed and its writes are visible). Launch latency and prologues of the ~700 kernels of a UNet call then overlap the
// tail of their predecessors, also inside CUDA graphs (captured as programmatic dependency edges). Opt-in (AP_PDL=1): the
// full GPU suite passes with it.
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              int cluster, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  unsigned n = 0;
  if (cluster > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = (unsigned)cluster;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

#define AP_LAUNCH(kernel, grid, block, smem, stream, ...)                                                              \
  do {                                                                                                                 \
    cudaError_t _le = ap::launch_pdl(kernel, dim3(grid), dim3(block), (size_t)(smem), (cudaStream_t)(stream), 1,       \
                                     __VA_ARGS__);                                                                     \
    if (_le != cudaSuccess) return ap::fail(AP_ERR_CUDA, "launch " #kernel ": %s", cudaGetErrorString(_le));           \
  } while (0)

#define AP_CHECK_CUDA(expr)                                                                       \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) return ap::fail(AP_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

#define AP_REQUIRE(cond, ...)                                  \
  do {                                                         \
    if (!(cond)) return ap::fail(AP_ERR_INVALID, __VA_ARGS__); \
  } while (0)

// true for NULL and for any address on the 16-byte grid (the kernels' uint4 / float4 accesses need it)
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace ap
