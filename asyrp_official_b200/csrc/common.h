// Host-side helpers shared by the .cu translation units of libasyrp_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <string>

#define ASYRP_API __attribute__((visibility("default")))

namespace asyrp {

// Error codes returned through the C ABI (0 = success). Mirrors include/asyrp_b200.h.
enum : int {
  ASYRP_OK = 0,
  ASYRP_ERR_INVALID = -1,   // bad argument / unsupported shape
  ASYRP_ERR_CUDA = -2,      // CUDA runtime / driver error
  ASYRP_ERR_NO_DEVICE = -3, // no sm_90 device available
};

void set_error(const char* fmt, ...);
const char* get_error();

#define ASYRP_CHECK_CUDA(expr)                                                                   \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      ::asyrp::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return ::asyrp::ASYRP_ERR_CUDA;                                                            \
    }                                                                                            \
  } while (0)

#define ASYRP_REQUIRE(cond, ...)            \
  do {                                      \
    if (!(cond)) {                          \
      ::asyrp::set_error(__VA_ARGS__);      \
      return ::asyrp::ASYRP_ERR_INVALID;    \
    }                                       \
  } while (0)

// kernel<<<grid, block, smem, stream>>>(args...) with the PDL launch attribute (see launch() below); returns
// ASYRP_ERR_CUDA from the enclosing C-ABI function on failure
#define ASYRP_LAUNCH(kernel, grid, block, smem, stream, ...)                                              \
  do {                                                                                                    \
    cudaError_t _le = ::asyrp::launch(kernel, grid, block, smem, stream, __VA_ARGS__);                    \
    if (_le != cudaSuccess) {                                                                             \
      ::asyrp::set_error("%s:%d: launch of %s failed: %s", __FILE__, __LINE__, #kernel, cudaGetErrorString(_le)); \
      return ::asyrp::ASYRP_ERR_CUDA;                                                                     \
    }                                                                                                     \
  } while (0)

// cuTensorMapEncodeTiled resolved at run time (no link-time dependency on libcuda, so the library loads
// on a machine without a driver and simply fails loudly when an op is created).
int encode_tensor_map(CUtensorMap* out, CUtensorMapDataType dt, uint32_t rank, const void* gaddr,
                      const uint64_t* dims, const uint64_t* strides_bytes /* rank-1 */, const uint32_t* box,
                      CUtensorMapSwizzle swz);

int sm_count();

// Programmatic dependent launch (PDL).  Every kernel of the library starts with `griddepcontrol.launch_dependents`
// and executes `griddepcontrol.wait` before its first global-memory access; launched with the
// programmaticStreamSerialization attribute, kernel i+1 is scheduled (and runs its prologue: barrier init,
// descriptor prefetch) while kernel i drains, instead of after it — inside a captured graph too.  Inside a CUDA graph
// the launch gaps are already hidden and a conv CTA with ~227 KB of shared memory cannot become resident before its
// predecessor on the same SM has exited, so there is little to overlap.  Hence OFF by default; asyrp_set_pdl(1) /
// ASYRP_PDL=1 enables it (eager, launch-bound callers of the C ABI benefit).
int pdl_enabled();

template <typename... Exp, typename... Act>
inline cudaError_t launch(void (*kernel)(Exp...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Act&&... args) {
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.attrs = attr;
  cfg.numAttrs = 0;
  if (pdl_enabled()) {
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.numAttrs = 1;
  }
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<Exp>(args)...);
}

}  // namespace asyrp
