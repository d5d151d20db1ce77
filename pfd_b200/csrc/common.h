// Shared helpers for the C-ABI translation units (error text, launch counter, launch geometry, kernel entry,
// shared-memory opt-in, tensor maps, per-device scratch).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <atomic>
#include <string>

namespace pfd {

extern thread_local std::string g_last_error;
extern std::atomic<int64_t> g_launches;

int set_error(const char* fmt, ...);
// run-time tuning switch set through pfd_set_option (A/B measurements inside one process); dflt when unset
int option(const char* name, int dflt);

inline int check_launch(const char* what) {
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return 0;
}

// Programmatic dependent launch: every pfd kernel begins with griddepcontrol.wait (see pdl_enter() below
// and pdl_wait() in ptx.cuh) so its CTAs may be scheduled while the previous kernel of the stream drains;
// set PFD_NO_PDL=1 to launch with plain stream ordering.
inline bool use_pdl() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("PFD_NO_PDL");
    v = (e && e[0] == '1') ? 0 : 1;
  }
  return v == 1;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                            Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = use_pdl() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

#ifdef __CUDACC__
// Programmatic dependent launch at a kernel's entry: block until the producer kernel has completed, then let the
// consumer kernel start scheduling its CTAs (see launch_k).  The GEMM and attention kernels place the two halves
// separately (pdl_wait / pdl_launch_dependents in ptx.cuh).
__device__ __forceinline__ void pdl_enter() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// ToPILImage on a float tensor: pic.mul(255).byte() - the product is rounded in the tensor's dtype, then truncated
// (torchvision ToPILImage, controlnet.py:339; shared by the Canny and HED annotators)
template <typename T>
__device__ __forceinline__ uint32_t to_u8(T v);
template <>
__device__ __forceinline__ uint32_t to_u8<float>(float v) {
  const float m = v * 255.f;
  return (uint32_t)(unsigned char)(int)m;
}
template <>
__device__ __forceinline__ uint32_t to_u8<__half>(__half v) {
  const float m = __half2float(__hmul(v, __float2half_rn(255.f)));
  return (uint32_t)(unsigned char)(int)m;
}
#endif

inline int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// Grid of a grid-stride kernel: ceil(work / per_block) blocks, at most 16 per SM, at least 1.
inline int grid_cap(long long work, int per_block) {
  long long g = (work + per_block - 1) / per_block;
  const long long cap = (long long)num_sms() * 16;
  if (g > cap) g = cap;
  return (int)(g < 1 ? 1 : g);
}

inline bool misaligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

// Lets `kernel` use `bytes` of dynamic shared memory (beyond the default 48 KiB), once per process.  The flag is per
// kernel instance: the kernel is a template argument, not a function pointer, whose type template instances share.
template <auto kernel>
inline int smem_opt_in(int bytes, const char* what) {
  static bool done = false;
  if (done) return 0;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return set_error("cudaFuncSetAttribute(%s, %d bytes): %s", what, bytes, cudaGetErrorString(e));
  done = true;
  return 0;
}

// fp16 TMA tensor map of rank 3 or 4 with 128-byte swizzle and 256-byte L2 promotion; elements outside `dims` read as
// zero.  dims, box and elem_strides have `rank` entries, strides_bytes rank - 1.  `what` names the operand in the error.
int encode_tensor_map_f16(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims,
                          const cuuint64_t* strides_bytes, const cuuint32_t* box, const cuuint32_t* elem_strides,
                          const char* what);

// Per-device scratch buffers.  Each slot holds one buffer per device, allocated by the first call on that device and
// then shared by every later call, eager or captured, so a graph replay makes the same choices as the eager run.
// cudaMalloc is illegal inside a stream capture: the first call must be eager (every graph-captured path of the
// package runs eagerly first).  The launches of one device are stream-ordered by the callers (one request at a time),
// so one buffer per device is enough.
enum ScratchSlot { SCRATCH_SPLITK, SCRATCH_GN_DET, SCRATCH_SLOTS };
// The slot's buffer for the current device: `bytes` long, the first `zero_bytes` zeroed when it is allocated.  Null
// when it cannot be allocated, or when it is not allocated yet and `st` is capturing; the caller reports the error.
void* device_scratch(ScratchSlot slot, size_t bytes, size_t zero_bytes, cudaStream_t st);

// Deterministic mode (pfd_set_option "deterministic"; default from PFD_DETERMINISTIC=1 at load, see api.cu): every
// summation order depends only on a sample's own shapes, never on the batch, the SM count or a race between CTAs.
bool deterministic();
// SM count the GEMM and GroupNorm plan their grids and split-K with: the device's, or the smaller "plan_sms" option
// (lets one card reproduce the plan of a smaller one).
inline int plan_sms() {
  const int dev = num_sms();
  const int p = option("plan_sms", 0);
  return (p > 0 && p < dev) ? p : dev;
}

}  // namespace pfd
