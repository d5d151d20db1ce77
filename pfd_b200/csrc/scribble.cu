// Scribble annotators of ControlNet.preprocess(type='scribble') on the GPU (controlnet.py:432-491).
//
// method='hed': make_scribble (controlnet.py:436-454) on the uint8 HED levels of pfd_hed_fuse_f32's output:
//   scribble_nms_kernel    g = cv2.GaussianBlur(float32(u8), (0,0), 3) (ksize 25, BORDER_REFLECT_101), then the
//                          non-maximum suppression of the four 3-tap cv2.dilate lines (g is kept where it equals the
//                          dilation along at least one line; out-of-image neighbours are ignored) and `> 127` -> 0/255;
//   scribble_blur_u8_kernel cv2.GaussianBlur of that uint8 map with sigma 3 (ksize 19) on cv2's bit-exact fixed-point
//                          path, then `> 4` -> 1.0 in all three output channels (ToTensor + repeat).
// method='xdog' (controlnet.py:476-482): scribble_xdog_kernel quantises like ToPILImage, blurs every colour channel
//   with sigma 0.5 (ksize 5) and sigma 5 (ksize 41) in float32, dog = uint8(clip(255 - min_c(g2 - g1), 0, 255)) and
//   edge = uint8(2 * uint8(255 - dog)) > threshold, with the uint8 wrap of the numpy expression kept.
//
// The uint8 blur is integer arithmetic and bit-exact.  The float blurs follow OpenCV's kernels (getGaussianKernel's
// bit-exact float64 taps rounded to float32) and its pass structure (rows, then columns), but not its exact operation
// order, so results differ from cv2 by float32 rounding; only decisions at near-ties can differ (README, scribble).
// Every kernel is a function of one image's pixels: 32x32 output tiles, one batch image per grid.z, halos in shared
// memory with the reflect-101 index computed per halo pixel (it folds repeatedly on images smaller than the radius).
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/pfd_b200.h"
#include "common.h"

namespace pfd {

// cv2.borderInterpolate(BORDER_REFLECT_101): ... 2 1 | 0 1 2 ... n-1 | n-2 ..., folded until inside
__device__ __forceinline__ int reflect101(int i, int n) {
  if (n == 1) return 0;
  while ((unsigned)i >= (unsigned)n) i = i < 0 ? -i : 2 * (n - 1) - i;
  return i;
}

constexpr int ST = 32;                     // output tile side
constexpr int SB_R = 12;                   // sigma 3 float blur radius (ksize 25)
constexpr int SU_R = 9;                    // sigma 3 uint8 blur radius (ksize 19)
constexpr int SX1_R = 2, SX2_R = 20;       // xdog: sigma 0.5 (ksize 5) and sigma 5 (ksize 41)

struct Taps25 { float k[2 * SB_R + 1]; };
struct Taps5 { float k[2 * SX1_R + 1]; };
struct Taps41 { float k[2 * SX2_R + 1]; };
struct Fixed19 { int k[2 * SU_R + 1]; };

// make_scribble's nms(): float blur of the tile plus a 1-pixel halo, then the directional maxima and `> 127`.
__global__ void __launch_bounds__(256)
scribble_nms_kernel(const float* __restrict__ hed, long long img_stride, int H, int W, Taps25 kt,
                    unsigned char* __restrict__ z) {
  constexpr int G = ST + 2;                // blurred region: tile + NMS halo
  constexpr int IN = G + 2 * SB_R;         // input region
  __shared__ float s_in[IN][IN];
  __shared__ float s_row[IN][G];
  __shared__ float s_g[G][G + 1];
  pdl_enter();
  const int n = blockIdx.z;
  const int x0 = blockIdx.x * ST, y0 = blockIdx.y * ST;
  const float* src = hed + (long long)n * img_stride;
  for (int k = threadIdx.x; k < IN * IN; k += blockDim.x) {
    const int ly = k / IN, lx = k % IN;
    const int gy = reflect101(y0 - 1 - SB_R + ly, H), gx = reflect101(x0 - 1 - SB_R + lx, W);
    s_in[ly][lx] = rintf(src[(long long)gy * W + gx] * 255.f);   // the uint8 level behind ToTensor's level / 255
  }
  __syncthreads();
  for (int k = threadIdx.x; k < IN * G; k += blockDim.x) {       // rows: sequential taps
    const int ly = k / G, lx = k % G;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 2 * SB_R + 1; ++j) acc = fmaf(kt.k[j], s_in[ly][lx + j], acc);
    s_row[ly][lx] = acc;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < G * G; k += blockDim.x) {        // columns: symmetric pairs
    const int ly = k / G, lx = k % G;
    float acc = kt.k[SB_R] * s_row[ly + SB_R][lx];
#pragma unroll
    for (int i = 1; i <= SB_R; ++i) acc = fmaf(kt.k[SB_R + i], s_row[ly + SB_R - i][lx] + s_row[ly + SB_R + i][lx], acc);
    s_g[ly][lx] = acc;
  }
  __syncthreads();
  const int ty = threadIdx.x / ST;
  const int tx = threadIdx.x % ST;
  for (int r = ty; r < ST; r += blockDim.x / ST) {
    const int gy = y0 + r, gx = x0 + tx;
    if (gy >= H || gx >= W) continue;
    const float c = s_g[r + 1][tx + 1];
    // cv2.dilate(g, line) == g  <=>  g >= every in-image neighbour on the line
    auto ge = [&](int dy, int dx) {
      const int ya = gy - dy, xa = gx - dx, yb = gy + dy, xb = gx + dx;
      const bool a = ya < 0 || ya >= H || xa < 0 || xa >= W || c >= s_g[r + 1 - dy][tx + 1 - dx];
      const bool b = yb < 0 || yb >= H || xb < 0 || xb >= W || c >= s_g[r + 1 + dy][tx + 1 + dx];
      return a && b;
    };
    const bool kept = ge(0, 1) || ge(1, 0) || ge(1, 1) || ge(1, -1);
    z[((long long)n * H + gy) * W + gx] = (kept && c > 127.f) ? 255 : 0;
  }
}

// cv2.GaussianBlur(u8, (0,0), 3) on OpenCV's fixed-point path: 8-fractional-bit taps, integer row and column sums,
// (sum + 2^15) >> 16.  Writes the blurred map (blurred != nullptr) and / or the thresholded control map (out).
__global__ void __launch_bounds__(256)
scribble_blur_u8_kernel(const unsigned char* __restrict__ z, int H, int W, Fixed19 kt,
                        unsigned char* __restrict__ blurred, float* __restrict__ out) {
  constexpr int IN = ST + 2 * SU_R;
  __shared__ int s_in[IN][IN];
  __shared__ int s_row[IN][ST];
  pdl_enter();
  const int n = blockIdx.z;
  const int x0 = blockIdx.x * ST, y0 = blockIdx.y * ST;
  const unsigned char* src = z + (long long)n * H * W;
  for (int k = threadIdx.x; k < IN * IN; k += blockDim.x) {
    const int ly = k / IN, lx = k % IN;
    s_in[ly][lx] = src[(long long)reflect101(y0 - SU_R + ly, H) * W + reflect101(x0 - SU_R + lx, W)];
  }
  __syncthreads();
  for (int k = threadIdx.x; k < IN * ST; k += blockDim.x) {
    const int ly = k / ST, lx = k % ST;
    int acc = 0;
#pragma unroll
    for (int j = 0; j < 2 * SU_R + 1; ++j) acc += kt.k[j] * s_in[ly][lx + j];
    s_row[ly][lx] = acc;
  }
  __syncthreads();
  const long long hw = (long long)H * W;
  const int ty = threadIdx.x / ST;
  const int tx = threadIdx.x % ST;
  for (int r = ty; r < ST; r += blockDim.x / ST) {
    const int gy = y0 + r, gx = x0 + tx;
    if (gy >= H || gx >= W) continue;
    int acc = 0;
#pragma unroll
    for (int i = 0; i < 2 * SU_R + 1; ++i) acc += kt.k[i] * s_row[r + i][tx];
    const int b = (acc + (1 << 15)) >> 16;                          // taps sum to 256: at most 255, no saturation
    const long long p = (long long)gy * W + gx;
    if (blurred) blurred[n * hw + p] = (unsigned char)b;
    if (out) {
      const float v = b > 4 ? 1.f : 0.f;                            // 255 / 255 (ToTensor), repeated to RGB
      float* o = out + (long long)n * 3 * hw + p;
      o[0] = v;
      o[hw] = v;
      o[2 * hw] = v;
    }
  }
}

// apply_scribble_xdog on one 32x32 tile: the colour channels are blurred one after the other and the running
// min_c(g2 - g1) stays in registers (4 output pixels per thread).
template <typename T>
__global__ void __launch_bounds__(256)
scribble_xdog_kernel(const T* __restrict__ x, int H, int W, int threshold, Taps5 k1, Taps41 k2,
                     float* __restrict__ out) {
  constexpr int IN = ST + 2 * SX2_R;
  constexpr int IN1 = ST + 2 * SX1_R;
  constexpr int PER = ST * ST / 256;
  __shared__ unsigned char s_in[3][IN][IN];
  __shared__ float s_r2[IN][ST];
  __shared__ float s_r1[IN1][ST];
  pdl_enter();
  const int n = blockIdx.z;
  const int x0 = blockIdx.x * ST, y0 = blockIdx.y * ST;
  const long long hw = (long long)H * W;
  const T* img = x + (long long)n * 3 * hw;
  for (int k = threadIdx.x; k < IN * IN; k += blockDim.x) {
    const int ly = k / IN, lx = k % IN;
    const long long p = (long long)reflect101(y0 - SX2_R + ly, H) * W + reflect101(x0 - SX2_R + lx, W);
#pragma unroll
    for (int c = 0; c < 3; ++c) s_in[c][ly][lx] = (unsigned char)to_u8<T>(img[c * hw + p]);   // ToPILImage
  }
  float mn[PER];
#pragma unroll
  for (int q = 0; q < PER; ++q) mn[q] = INFINITY;
  for (int c = 0; c < 3; ++c) {
    __syncthreads();                                                // s_in ready / previous channel's columns done
    for (int k = threadIdx.x; k < IN * ST; k += blockDim.x) {
      const int ly = k / ST, lx = k % ST;
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 2 * SX2_R + 1; ++j) acc = fmaf(k2.k[j], (float)s_in[c][ly][lx + j], acc);
      s_r2[ly][lx] = acc;
    }
    for (int k = threadIdx.x; k < IN1 * ST; k += blockDim.x) {
      const int ly = k / ST, lx = k % ST;
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 2 * SX1_R + 1; ++j)
        acc = fmaf(k1.k[j], (float)s_in[c][ly + SX2_R - SX1_R][lx + SX2_R - SX1_R + j], acc);
      s_r1[ly][lx] = acc;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      const int pix = threadIdx.x + q * 256;
      const int r = pix / ST, cx = pix % ST;
      float g2 = k2.k[SX2_R] * s_r2[r + SX2_R][cx];
#pragma unroll
      for (int i = 1; i <= SX2_R; ++i) g2 = fmaf(k2.k[SX2_R + i], s_r2[r + SX2_R - i][cx] + s_r2[r + SX2_R + i][cx], g2);
      float g1 = k1.k[SX1_R] * s_r1[r + SX1_R][cx];
#pragma unroll
      for (int i = 1; i <= SX1_R; ++i) g1 = fmaf(k1.k[SX1_R + i], s_r1[r + SX1_R - i][cx] + s_r1[r + SX1_R + i][cx], g1);
      mn[q] = fminf(mn[q], g2 - g1);
    }
  }
#pragma unroll
  for (int q = 0; q < PER; ++q) {
    const int pix = threadIdx.x + q * 256;
    const int gy = y0 + pix / ST, gx = x0 + pix % ST;
    if (gy >= H || gx >= W) continue;
    const float v = fminf(fmaxf(255.f - mn[q], 0.f), 255.f);
    const unsigned dog = (unsigned)v;                               // astype(uint8) truncates
    const unsigned e = (2u * ((255u - dog) & 255u)) & 255u;         // uint8 arithmetic: 2 * (255 - dog) wraps mod 256
    const float o = (int)e > threshold ? 1.f : 0.f;
    float* op = out + (long long)n * 3 * hw + (long long)gy * W + gx;
    op[0] = o;
    op[hw] = o;
    op[2 * hw] = o;
  }
}

// getGaussianKernel(n, sigma) as OpenCV computes it (float64, symmetric halves, normalised by the reciprocal sum)
static void gaussian_taps(int n, double sigma, double* k) {
  const double scale2 = -0.125 / (sigma * sigma);
  const int h = (n - 1) / 2;
  double sum = 0.0;
  for (int i = 0, xx = 1 - n; i < h; ++i, xx += 2) {
    k[i] = exp((double)(xx * xx) * scale2);
    sum += k[i];
  }
  sum = sum * 2.0 + 1.0;
  const double mul = 1.0 / sum;
  for (int i = 0; i < h; ++i) k[n - 1 - i] = k[i] = k[i] * mul;
  k[h] = mul;
}

template <int N>
static void float_taps(double sigma, float* out) {
  double k[N];
  gaussian_taps(N, sigma, k);
  for (int i = 0; i < N; ++i) out[i] = (float)k[i];
}

// OpenCV's 8-bit fixed-point taps: the float64 taps times 256, rounded from the outside in with the rounding error
// carried to the next tap, and the centre tap taking what is left of 256.
static Fixed19 fixed_taps19(double sigma) {
  constexpr int N = 2 * SU_R + 1;
  double k[N];
  gaussian_taps(N, sigma, k);
  Fixed19 f;
  double err = 0.0;
  int sum = 0;
  for (int i = 0; i < N / 2; ++i) {
    const double a = k[i] * 256.0 + err;
    const int v = (int)nearbyint(a);
    err = a - v;
    f.k[i] = f.k[N - 1 - i] = v;
    sum += v;
  }
  f.k[N / 2] = 256 - 2 * sum;
  return f;
}

}  // namespace pfd

using namespace pfd;

extern "C" PFD_API int pfd_scribble_blur_u8(const uint8_t* z, int32_t B, int32_t H, int32_t W, uint8_t* blurred,
                                            float* out, void* stream) {
  if (!z || (!blurred && !out) || B <= 0 || H <= 0 || W <= 0 || B > 65535)
    return set_error("pfd_scribble_blur_u8: bad arguments (B=%d H=%d W=%d)", B, H, W);
  static const Fixed19 kt = fixed_taps19(3.0);
  launch_k(scribble_blur_u8_kernel, dim3((W + ST - 1) / ST, (H + ST - 1) / ST, B), dim3(256), (size_t)0,
           static_cast<cudaStream_t>(stream), (const unsigned char*)z, (int)H, (int)W, kt, (unsigned char*)blurred, out);
  return check_launch("scribble_blur_u8");
}

extern "C" PFD_API int pfd_scribble_hed_f32(const float* hed, int64_t img_stride, int32_t B, int32_t H, int32_t W,
                                            uint8_t* nms, float* out, void* stream) {
  if (!hed || !nms || !out || B <= 0 || H <= 0 || W <= 0 || B > 65535 || img_stride < (int64_t)H * W)
    return set_error("pfd_scribble_hed_f32: bad arguments (B=%d H=%d W=%d stride=%lld)", B, H, W,
                     (long long)img_stride);
  static const Taps25 kt = [] { Taps25 t; float_taps<2 * SB_R + 1>(3.0, t.k); return t; }();
  launch_k(scribble_nms_kernel, dim3((W + ST - 1) / ST, (H + ST - 1) / ST, B), dim3(256), (size_t)0,
           static_cast<cudaStream_t>(stream), hed, (long long)img_stride, (int)H, (int)W, kt, (unsigned char*)nms);
  if (int rc = check_launch("scribble_nms")) return rc;
  return pfd_scribble_blur_u8(nms, B, H, W, nullptr, out, stream);
}

extern "C" PFD_API int pfd_scribble_xdog_f32(const void* x, int32_t src_is_f32, int32_t B, int32_t H, int32_t W,
                                             int32_t threshold, float* out, void* stream) {
  if (!x || !out || B <= 0 || H <= 0 || W <= 0 || B > 65535)
    return set_error("pfd_scribble_xdog_f32: bad arguments (B=%d H=%d W=%d)", B, H, W);
  static const Taps5 k1 = [] { Taps5 t; float_taps<2 * SX1_R + 1>(0.5, t.k); return t; }();
  static const Taps41 k2 = [] { Taps41 t; float_taps<2 * SX2_R + 1>(5.0, t.k); return t; }();
  const dim3 grid((W + ST - 1) / ST, (H + ST - 1) / ST, B);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (src_is_f32)
    launch_k(scribble_xdog_kernel<float>, grid, dim3(256), (size_t)0, st, static_cast<const float*>(x), (int)H, (int)W,
             (int)threshold, k1, k2, out);
  else
    launch_k(scribble_xdog_kernel<__half>, grid, dim3(256), (size_t)0, st, static_cast<const __half*>(x), (int)H,
             (int)W, (int)threshold, k1, k2, out);
  return check_launch("scribble_xdog");
}
