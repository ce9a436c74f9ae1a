#include "host_util.h"
#include <cstdarg>
#include <atomic>
#include <mutex>

namespace vdb {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int num_sms() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static int encode(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                  const cuuint32_t* box, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn fn = get_encode();
  if (!fn) return set_error(2, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if (reinterpret_cast<uintptr_t>(ptr) & 15) return set_error(1, "tensor map: base pointer must be 16-byte aligned");
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  for (int i = 0; i < rank - 1; ++i)
    if (strides[i] % 16) return set_error(1, "tensor map: stride %d (%llu B) not a multiple of 16", i, (unsigned long long)strides[i]);
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(2, "cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu box %u,%u)", (int)r, rank,
                     (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
  return 0;
}

int make_tmap_2d(CUtensorMap* m, const void* ptr, uint64_t d0, uint64_t d1, uint64_t stride1, uint32_t box0,
                 uint32_t box1) {
  cuuint64_t dims[2] = {d0, d1};
  cuuint64_t strides[1] = {stride1};
  cuuint32_t box[2] = {box0, box1};
  return encode(m, ptr, 2, dims, strides, box);
}

int make_tmap_4d(CUtensorMap* m, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3,
                 uint64_t stride1, uint64_t stride2, uint64_t stride3, uint32_t box0, uint32_t box1, uint32_t box2,
                 uint32_t box3) {
  cuuint64_t dims[4] = {d0, d1, d2, d3};
  cuuint64_t strides[3] = {stride1, stride2, stride3};
  cuuint32_t box[4] = {box0, box1, box2, box3};
  return encode(m, ptr, 4, dims, strides, box);
}

// store-side map of an epilogue staging box: 32 bf16 columns (64 B) x 16 rows, SWIZZLE_64B
int make_tmap_4d_sw64(CUtensorMap* m, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3,
                      uint64_t stride1, uint64_t stride2, uint64_t stride3, uint32_t box0, uint32_t box1, uint32_t box2,
                      uint32_t box3) {
  cuuint64_t dims[4] = {d0, d1, d2, d3};
  cuuint64_t strides[3] = {stride1, stride2, stride3};
  cuuint32_t box[4] = {box0, box1, box2, box3};
  return encode(m, ptr, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B);
}

}  // namespace vdb

extern "C" {
const char* vdb_last_error(void) { return vdb::g_err; }
long long vdb_launch_count(void) { return vdb::g_launches.load(); }
void vdb_reset_launch_count(void) { vdb::g_launches.store(0); }
int vdb_num_sms(void) { return vdb::num_sms(); }
const char* vdb_version(void) { return "vdb200 0.1 (sm_90a)"; }
}
