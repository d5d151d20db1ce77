// k-diffusion samplers (Euler ancestral, DPM-Solver++(2M)) on the device: the per-step update and the device-side
// loop header.  Every step of every sampler type is the same affine update
//   D  = x - sigma * eps                       (eps-prediction denoiser, CFG combined in fp32)
//   x' = a*x + b*D + c*D_prev + u*noise
// with the per-step row {sigma, a, b, c, u, c_in_next} computed on the host in float64 (pfd_b200/sampler.py), so the
// kernel has no knowledge of the sampler type and one captured graph can hold a whole deterministic loop.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "../../include/pfd_b200.h"
#include "common.h"

namespace pfd {

// *step += 1; t_out[0..nb) = ttab[*step]  (the index is clamped to the table)
__global__ void ksampler_begin_step_kernel(int* __restrict__ step, const float* __restrict__ ttab, int nsteps,
                                           float* __restrict__ t_out, int nb) {
  pdl_enter();
  int idx = *step + 1;
  idx = idx < 0 ? 0 : (idx >= nsteps ? nsteps - 1 : idx);
  __syncthreads();
  for (int i = threadIdx.x; i < nb; i += blockDim.x) t_out[i] = ttab[idx];
  if (threadIdx.x == 0) *step = idx;
}

__global__ void ksampler_step_kernel(const __half* __restrict__ eps, int cfg, float guidance, long long half_n,
                                     const float* __restrict__ coef, const int* __restrict__ step, int last_step,
                                     float* __restrict__ x, float* __restrict__ d_prev,
                                     const __half* __restrict__ noise, __half* __restrict__ unet_in,
                                     __half* __restrict__ out, const int* __restrict__ log_tab,
                                     __half* __restrict__ log_xt, __half* __restrict__ log_x0) {
  pdl_enter();
  const int st = *step;
  const float* row = coef + (long long)st * PFD_KSAMPLER_NCOEF;
  const float sigma = row[0], a = row[1], b = row[2], c = row[3], u = row[4], cin_next = row[5];
  const bool use_noise = noise != nullptr && u != 0.f;
  __half* o = st == last_step ? out : nullptr;
  const int slot = log_tab ? log_tab[st] : -1;
  __half* lxt = slot >= 0 ? log_xt + (long long)slot * half_n : nullptr;
  __half* lx0 = slot >= 0 ? log_x0 + (long long)slot * half_n : nullptr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < half_n;
       i += (long long)gridDim.x * blockDim.x) {
    float e;
    if (cfg) {
      const float eu = __half2float(eps[i]);
      e = eu + guidance * (__half2float(eps[half_n + i]) - eu);
    } else {
      e = guidance * __half2float(eps[i]);  // e_t = eps * scale without the CFG batch, as in the DDIM sampler
    }
    const float xv = x[i];
    const float d = xv - sigma * e;
    float xn = a * xv + b * d + c * d_prev[i];
    if (use_noise) xn += u * __half2float(noise[i]);
    x[i] = xn;
    d_prev[i] = d;
    const __half xin = __float2half_rn(xn * cin_next);
    unet_in[i] = xin;
    if (cfg) unet_in[half_n + i] = xin;
    if (o) o[i] = __float2half_rn(xn);
    if (lxt) {
      lxt[i] = xin;
      lx0[i] = __float2half_rn(d);
    }
  }
}

}  // namespace pfd

using namespace pfd;

extern "C" PFD_API int pfd_ksampler_begin_step(int32_t* step, const float* ttab, int32_t nsteps, float* t_out,
                                               int32_t nb, void* stream) {
  if (!step || !ttab || !t_out || nsteps <= 0 || nb <= 0)
    return set_error("pfd_ksampler_begin_step: null/empty argument");
  launch_k(ksampler_begin_step_kernel, dim3(1), dim3(64), (size_t)0, static_cast<cudaStream_t>(stream),
           reinterpret_cast<int*>(step), ttab, (int)nsteps, t_out, (int)nb);
  return check_launch("ksampler_begin_step");
}

extern "C" PFD_API int pfd_ksampler_step_f32(const void* eps, int32_t cfg, float guidance, int64_t half_n,
                                             const float* coef, const int32_t* step, int32_t last_step, float* x,
                                             float* d_prev, const void* noise, void* unet_in, void* out,
                                             const int32_t* log_tab, void* log_xt, void* log_x0, void* stream) {
  if (!eps || !coef || !step || !x || !d_prev || !unet_in || !out || half_n <= 0)
    return set_error("pfd_ksampler_step_f32: null/empty argument");
  if (log_tab && (!log_xt || !log_x0)) return set_error("pfd_ksampler_step_f32: log_tab without log buffers");
  launch_k(ksampler_step_kernel, dim3(grid_cap(half_n, 256)), dim3(256), (size_t)0, static_cast<cudaStream_t>(stream),
           static_cast<const __half*>(eps), (int)(cfg != 0), guidance, (long long)half_n, coef,
           reinterpret_cast<const int*>(step), (int)last_step, x, d_prev, static_cast<const __half*>(noise),
           static_cast<__half*>(unet_in), static_cast<__half*>(out), reinterpret_cast<const int*>(log_tab),
           static_cast<__half*>(log_xt), static_cast<__half*>(log_x0));
  return check_launch("ksampler_step");
}
