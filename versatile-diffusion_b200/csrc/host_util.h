// Host-side helpers shared by the vdb200 translation units: error reporting, launch counting,
// SM count, TMA tensor-map construction through the driver entry point (no libcuda link needed).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <cstdlib>

namespace vdb {

int set_error(int code, const char* fmt, ...);   // records message, returns code
bool pdl_enabled();                               // VDB_PDL=1 enables programmatic dependent launch (default off)
int num_sms();
void count_launch(int n = 1);

#define VDB_CUDA_CHECK(expr)                                                                       \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      return ::vdb::set_error(2, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// bf16 tensor maps, SWIZZLE_128B, zero OOB fill. Strides in bytes (dim0 is contiguous).
int make_tmap_2d(CUtensorMap* m, const void* ptr, uint64_t d0, uint64_t d1, uint64_t stride1, uint32_t box0,
                 uint32_t box1);
int make_tmap_4d(CUtensorMap* m, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3,
                 uint64_t stride1, uint64_t stride2, uint64_t stride3, uint32_t box0, uint32_t box1,
                 uint32_t box2, uint32_t box3);

int make_tmap_4d_sw64(CUtensorMap* m, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3,
                      uint64_t stride1, uint64_t stride2, uint64_t stride3, uint32_t box0, uint32_t box1,
                      uint32_t box2, uint32_t box3);   // SWIZZLE_64B (epilogue store tiles: 64-byte rows)

// Launch with the programmatic-stream-serialization attribute: the kernel's prologue may overlap the tail of
// the previous kernel in the stream; every kernel launched this way calls pdl_wait() before reading its inputs.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                              Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace vdb
