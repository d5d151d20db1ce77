// Host-side shared helpers for the C-ABI translation units (error text, launch counter).
#pragma once
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

// Programmatic dependent launch: every pfd kernel begins with griddepcontrol.wait (see pdl_wait() in
// ptx.cuh / elementwise.cu) so its CTAs may be scheduled while the previous kernel of the stream drains;
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

}  // namespace pfd
