// Library-level entry points of the C ABI: version, thread-local error text, launch counter; and the host helpers the
// kernels share: the tensor-map encoder and the per-device scratch buffers.
#include <stdarg.h>

#include <map>
#include <mutex>

#include "../../include/pfd_b200.h"
#include "common.h"

namespace pfd {
thread_local std::string g_last_error;
std::atomic<int64_t> g_launches{0};

int set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return 1;
}
}  // namespace pfd

namespace pfd {
static std::mutex g_opt_mu;
static std::map<std::string, int>& opt_table() {
  static std::map<std::string, int> t;
  return t;
}
int option(const char* name, int dflt) {
  std::lock_guard<std::mutex> lk(g_opt_mu);
  auto it = opt_table().find(name);
  return it == opt_table().end() ? dflt : it->second;
}

// PFD_DETERMINISTIC=1 in the environment when the library is loaded makes deterministic mode the default, so that
// unmodified programs can run in either mode; pfd_set_option("deterministic", v) overrides it, a reset restores it.
static const int g_det_default = [] {
  const char* e = getenv("PFD_DETERMINISTIC");
  return (e && e[0] == '1') ? 1 : 0;
}();
bool deterministic() { return option("deterministic", g_det_default) != 0; }

int encode_tensor_map_f16(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims,
                          const cuuint64_t* strides_bytes, const cuuint32_t* box, const cuuint32_t* elem_strides,
                          const char* what) {
  typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static const EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    const bool ok = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
                    q == cudaDriverEntryPointSuccess;
    return ok ? reinterpret_cast<EncodeTiledFn>(p) : nullptr;
  }();
  if (!fn) return set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  const CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(ptr), dims, strides_bytes, box,
                        elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_SUCCESS) return 0;
  const bool r4 = rank > 3;
  return set_error("tensor map (%s) encode failed: CUresult %d rank %d dims[%llu,%llu,%llu,%llu] "
                   "strides[%llu,%llu,%llu] box[%u,%u,%u,%u] ptr %p",
                   what, (int)r, rank, (unsigned long long)dims[0], (unsigned long long)dims[1],
                   (unsigned long long)dims[2], (unsigned long long)(r4 ? dims[3] : 0),
                   (unsigned long long)strides_bytes[0], (unsigned long long)strides_bytes[1],
                   (unsigned long long)(r4 ? strides_bytes[2] : 0), box[0], box[1], box[2], r4 ? box[3] : 0, ptr);
}

void* device_scratch(ScratchSlot slot, size_t bytes, size_t zero_bytes, cudaStream_t st) {
  constexpr int MAX_DEV = 64;
  static std::mutex mu;
  static void* buf[SCRATCH_SLOTS][MAX_DEV] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MAX_DEV) return nullptr;
  std::lock_guard<std::mutex> lk(mu);
  if (buf[slot][dev]) return buf[slot][dev];
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) {
    (void)cudaGetLastError();
    return nullptr;
  }
  void* p = nullptr;
  if (cudaMalloc(&p, bytes) != cudaSuccess) {
    (void)cudaGetLastError();
    return nullptr;
  }
  if (zero_bytes && (cudaMemset(p, 0, zero_bytes) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess)) {
    (void)cudaGetLastError();
    cudaFree(p);
    return nullptr;
  }
  buf[slot][dev] = p;
  return p;
}
}  // namespace pfd

extern "C" PFD_API int pfd_set_option(const char* name, int32_t value) {
  std::lock_guard<std::mutex> lk(pfd::g_opt_mu);
  if (!name) {
    pfd::opt_table().clear();          // NULL: back to the built-in defaults
    return 0;
  }
  pfd::opt_table()[name] = value;
  return 0;
}

extern "C" PFD_API int pfd_version(void) { return PFD_ABI_VERSION; }
extern "C" PFD_API const char* pfd_last_error(void) { return pfd::g_last_error.c_str(); }
extern "C" PFD_API int64_t pfd_launch_count(void) { return pfd::g_launches.load(); }
