// Host-side helpers shared by the vdb200 translation units: error reporting, checked and counted kernel launches,
// SM count, TMA tensor-map construction through the driver entry point (no libcuda link needed).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <utility>

namespace vdb {

int set_error(int code, const char* fmt, ...);   // records message, returns code
int num_sms();
void count_launch();

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

namespace detail {
template <typename... KArgs, typename... Args>
inline int launch(const dim3* cluster, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, void* stream,
                  Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr{};
  if (cluster) {
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = cluster->x; attr.val.clusterDim.y = cluster->y; attr.val.clusterDim.z = cluster->z;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
  }
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
  if (e != cudaSuccess) {
    const char* name = nullptr;
    if (cudaFuncGetName(&name, reinterpret_cast<const void*>(kernel)) != cudaSuccess || !name) name = "kernel";
    return set_error(2, "launch of %s (grid %u x %u x %u, block %u, %zu B shared memory) failed: %s", name, grid.x, grid.y,
                     grid.z, block.x * block.y * block.z, smem, cudaGetErrorString(e));
  }
  count_launch();
  return 0;
}
}  // namespace detail

// Every kernel launch of the library goes through launch(): `kernel` on a grid x block grid with `smem` bytes of dynamic
// shared memory, on the C ABI's stream handle, or, given `cluster`, as thread-block clusters of that shape.  Returns 0 and
// counts the launch (vdb_launch_count), or records this launch's own error and returns 2 (VDB_ERR_CUDA) without counting it.
template <typename... KArgs, typename... Args>
inline int launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, void* stream, Args&&... args) {
  return detail::launch(nullptr, kernel, grid, block, smem, stream, std::forward<Args>(args)...);
}
template <typename... KArgs, typename... Args>
inline int launch(dim3 cluster, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, void* stream, Args&&... args) {
  return detail::launch(&cluster, kernel, grid, block, smem, stream, std::forward<Args>(args)...);
}

}  // namespace vdb
