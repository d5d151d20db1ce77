// Counter-based Gaussian noise for the samplers: every element's value is a pure function of
// (sample seed, stream, draw index, element index), so a sample's noise does not depend on its batch, its position in
// the batch or the GPU it runs on, and a captured CUDA graph can draw fresh noise per step from a device-side counter.
//   Philox4x32-10: key = (seed lo, seed hi), counter = (g lo, g hi, draw, stream) with g = element / 4
//   Box-Muller over the word pairs (w0, w1) and (w2, w3), in fp32 with the accurate logf / sqrtf / sincospif
// The exact definition is in include/pfd_b200.h (pfd_randn_f16).
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "../../include/pfd_b200.h"
#include "common.h"

namespace pfd {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

// (w_a, w_b) -> two N(0, 1) values; u1 = fp32(fp32(w_a) + 1) * 2^-32 lies in (0, 1], u2 = fp32(w_b) * 2^-32
__device__ __forceinline__ float2 box_muller(uint32_t wa, uint32_t wb) {
  const float u1 = ((float)wa + 1.0f) * 2.3283064365386963e-10f;
  const float u2 = (float)wb * 2.3283064365386963e-10f;
  const float r = sqrtf(-2.0f * logf(u1));
  float s, c;
  sincospif(2.0f * u2, &s, &c);
  return make_float2(r * c, r * s);
}

__global__ void randn_f16_kernel(__half* __restrict__ out, int B, long long n, const unsigned long long* __restrict__ seeds,
                                 uint32_t stream_id, int draw, const int* __restrict__ draw_dev, float scale) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const uint32_t d = (uint32_t)(draw + (draw_dev ? *draw_dev : 0));
  const long long groups = (n + 3) / 4;
  const long long items = groups * B;
  for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < items;
       it += (long long)gridDim.x * blockDim.x) {
    const long long b = it / groups, g = it - b * groups;
    const unsigned long long seed = seeds[b];
    const uint4 w = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)((unsigned long long)g >> 32), d, stream_id),
                                  (uint32_t)seed, (uint32_t)(seed >> 32));
    const float2 z01 = box_muller(w.x, w.y), z23 = box_muller(w.z, w.w);
    const __half2 h01 = __floats2half2_rn(scale * z01.x, scale * z01.y);
    const __half2 h23 = __floats2half2_rn(scale * z23.x, scale * z23.y);
    const long long e = 4 * g;
    __half* p = out + b * n + e;
    if (e + 4 <= n && ((reinterpret_cast<uintptr_t>(p) & 7) == 0)) {
      uint2 v;
      v.x = *reinterpret_cast<const uint32_t*>(&h01);
      v.y = *reinterpret_cast<const uint32_t*>(&h23);
      *reinterpret_cast<uint2*>(p) = v;   // 8-byte store of 4 halves
    } else {                              // the sample's last partial group, or a sample start not 8-byte aligned
      const __half h[4] = {__low2half(h01), __high2half(h01), __low2half(h23), __high2half(h23)};
      for (int j = 0; j < 4 && e + j < n; ++j) p[j] = h[j];
    }
  }
}

}  // namespace pfd

using namespace pfd;

extern "C" PFD_API int pfd_randn_f16(void* out, int32_t B, int64_t n, const uint64_t* seeds, uint32_t stream_id,
                                     int32_t draw, const int32_t* draw_dev, float scale, void* stream) {
  if (!out || !seeds || B <= 0 || n <= 0) return set_error("pfd_randn_f16: null/empty argument");
  const long long items = ((long long)n + 3) / 4 * B;
  long long g = (items + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  if (g > cap) g = cap;
  launch_k(randn_f16_kernel, dim3((unsigned)g), dim3(256), (size_t)0, static_cast<cudaStream_t>(stream),
           static_cast<__half*>(out), (int)B, (long long)n, reinterpret_cast<const unsigned long long*>(seeds),
           stream_id, (int)draw, reinterpret_cast<const int*>(draw_dev), scale);
  return check_launch("randn_f16");
}
