// HED soft-edge annotator of ControlNet.preprocess(type='hed' / 'softedge_v11p') on the GPU.
//
// Replaces controlnet.py:370-376 -> controlnet_annotator/hed/__init__.py:102-128 (apply_hed) around the VGG network
// ControlNetHED_Apache2 (hed/__init__.py:23-59).  The 13 3x3 convolutions (+ ReLU) run on the implicit-GEMM kernel;
// this file holds the glue around them:
//   hed_input_kernel      ToPILImage quantisation (x.mul(255).byte()), `x - norm` (hed/__init__.py:52) and the
//                         NCHW -> channel-last fp16 layout, all times the activation scale;
//   hed_pool_side_kernel  one read of a block's output gives both the 1x1 side projection (hed/__init__.py:38) and
//                         the 2x2 max-pool that feeds the next block (hed/__init__.py:34);
//   hed_fuse_kernel       cv2.resize(INTER_LINEAR) of the five side maps to the image size, np.mean, sigmoid in
//                         float64, (edge*255).clip(0,255).astype(uint8), ToTensor and repeat to RGB
//                         (hed/__init__.py:119-127, controlnet.py:372-374).
// The network runs at activation scale s (ReLU convs and max-pool are positively homogeneous when the conv biases are
// scaled by s too): every activation and side map is s times the reference's, and the fuse kernel multiplies by 1/s.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/pfd_b200.h"
#include "common.h"

namespace pfd {

// out[n, y, x, c] = (u8(x[n, c, y, x]) - norm[c]) * scale for c < 3, 0 for the pad channels
template <typename T>
__global__ void hed_input_kernel(const T* __restrict__ x, int B, int H, int W, int Cpad, const float* __restrict__ norm,
                                 float scale, __half* __restrict__ out) {
  pdl_enter();
  const float n0 = norm[0], n1 = norm[1], n2 = norm[2];
  const long long hw = (long long)H * W;
  const long long total = (long long)B * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / hw, p = i % hw;
    const T* src = x + n * 3 * hw + p;
    __half* o = out + i * Cpad;
    o[0] = __float2half_rn(((float)to_u8<T>(src[0]) - n0) * scale);
    o[1] = __float2half_rn(((float)to_u8<T>(src[hw]) - n1) * scale);
    o[2] = __float2half_rn(((float)to_u8<T>(src[2 * hw]) - n2) * scale);
    for (int c = 3; c < Cpad; ++c) o[c] = __float2half_rn(0.f);
  }
}

// A segment of L lanes (L = power of two >= C/8, at most 32) owns one 2x2 cell of the [B,h,w,C] block output; each lane
// reads 16-byte channel vectors of the (up to) four pixels once and uses them for both products:
//   side[n, y, x]    = sum_c x[n, y, x, c] * proj_w[c] + proj_b      (fp32, lane partials then a shuffle tree)
//   pooled[n, y, x]  = max of the 2x2 window (F.max_pool2d floor semantics: the cells of an odd last row / column
//                      only produce side values)
__global__ void __launch_bounds__(256)
hed_pool_side_kernel(const __half* __restrict__ x, int B, int h, int w, int C, int L, const float* __restrict__ proj_w,
                     const float* __restrict__ proj_b, float* __restrict__ side, __half* __restrict__ pooled) {
  extern __shared__ float s_w[];
  pdl_enter();
  for (int c = threadIdx.x; c < C; c += blockDim.x) s_w[c] = proj_w[c];
  __syncthreads();
  const float bias = *proj_b;
  const int vecs = C / 8;
  const int ncy = (h + 1) / 2, ncx = (w + 1) / 2, ph = h / 2, pw = w / 2;
  const long long ncells = (long long)B * ncy * ncx;
  const int lane = threadIdx.x & 31, seg = lane / L, sl = lane % L;
  const int segs_per_warp = 32 / L;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const long long nwarps = (long long)gridDim.x * blockDim.x / 32;
  // the loop bound is uniform across the warp: every lane reaches the shuffles
  for (long long base = warp0 * segs_per_warp; base < ncells; base += nwarps * segs_per_warp) {
    const long long cell = base + seg;
    const bool live = cell < ncells;
    int n = 0, cy = 0, cx = 0;
    if (live) {
      n = (int)(cell / ((long long)ncy * ncx));
      const int r = (int)(cell % ((long long)ncy * ncx));
      cy = r / ncx;
      cx = r % ncx;
    }
    const int y0 = 2 * cy, x0 = 2 * cx;
    const bool has_r = x0 + 1 < w, has_d = y0 + 1 < h;
    const bool pool = live && pooled != nullptr && cy < ph && cx < pw;
    const __half* px = x + (((long long)n * h + y0) * w + x0) * C;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (live) {
      for (int v = sl; v < vecs; v += L) {
        const uint4 z = make_uint4(0u, 0u, 0u, 0u);
        uint4 q[4];
        q[0] = __ldg(reinterpret_cast<const uint4*>(px) + v);
        q[1] = has_r ? __ldg(reinterpret_cast<const uint4*>(px + C) + v) : z;
        q[2] = has_d ? __ldg(reinterpret_cast<const uint4*>(px + (long long)w * C) + v) : z;
        q[3] = (has_r && has_d) ? __ldg(reinterpret_cast<const uint4*>(px + (long long)w * C + C) + v) : z;
        const float* wv = s_w + 8 * v;
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const __half2* hp = reinterpret_cast<const __half2*>(&q[p]);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(hp[j]);
            acc[p] = fmaf(f.x, wv[2 * j], acc[p]);
            acc[p] = fmaf(f.y, wv[2 * j + 1], acc[p]);
          }
        }
        if (pool) {
          uint4 m;
          const __half2* a = reinterpret_cast<const __half2*>(&q[0]);
          const __half2* b = reinterpret_cast<const __half2*>(&q[1]);
          const __half2* c = reinterpret_cast<const __half2*>(&q[2]);
          const __half2* d = reinterpret_cast<const __half2*>(&q[3]);
          __half2* mo = reinterpret_cast<__half2*>(&m);
#pragma unroll
          for (int j = 0; j < 4; ++j) mo[j] = __hmax2(__hmax2(a[j], b[j]), __hmax2(c[j], d[j]));
          reinterpret_cast<uint4*>(pooled + (((long long)n * ph + cy) * pw + cx) * C)[v] = m;
        }
      }
    }
#pragma unroll
    for (int p = 0; p < 4; ++p)
      for (int o = L / 2; o > 0; o >>= 1) acc[p] += __shfl_xor_sync(0xffffffffu, acc[p], o);
    if (live && sl == 0) {
      float* so = side + ((long long)n * h + y0) * w + x0;
      so[0] = acc[0] + bias;
      if (has_r) so[1] = acc[1] + bias;
      if (has_d) so[w] = acc[2] + bias;
      if (has_r && has_d) so[w + 1] = acc[3] + bias;
    }
  }
}

struct HedSides {
  const float* p[PFD_HED_MAX_SIDES];
  int h[PFD_HED_MAX_SIDES], w[PFD_HED_MAX_SIDES];
  double sy[PFD_HED_MAX_SIDES], sx[PFD_HED_MAX_SIDES];  // cv2's scale = 1 / (dsize / ssize), in double
  int n;
};

// cv2.resize(src, (W, H), INTER_LINEAR) of a float32 map, sampled at (y, x): source position (d + 0.5) * scale - 0.5 in
// double, its floor and fraction (fraction rounded to float), the column clamped to the borders with a zero fraction,
// the rows clipped to the image; horizontal pass, then vertical, as separate float products and sums (no FMA).
// dsize == ssize is a copy (cv2 special-cases it; the weights below would give the same values).
__device__ __forceinline__ float resize_linear(const float* __restrict__ s, int h, int w, double sy, double sx, int H,
                                               int W, int y, int x) {
  if (h == H && w == W) return s[(long long)y * w + x];
  const double fyd = (y + 0.5) * sy - 0.5, fxd = (x + 0.5) * sx - 0.5;
  const double iyd = floor(fyd), ixd = floor(fxd);
  int iy = (int)iyd, ix = (int)ixd;
  const float fy = (float)(fyd - iyd);
  float fx = (float)(fxd - ixd);
  if (ix < 0) {
    ix = 0;
    fx = 0.f;
  }
  if (ix >= w - 1) {
    ix = w - 1;
    fx = 0.f;
  }
  const int ix1 = min(ix + 1, w - 1);
  const int r0 = min(max(iy, 0), h - 1), r1 = min(max(iy + 1, 0), h - 1);
  const float a0 = __fsub_rn(1.f, fx), b0 = __fsub_rn(1.f, fy);
  const float* s0 = s + (long long)r0 * w;
  const float* s1 = s + (long long)r1 * w;
  const float t0 = __fadd_rn(__fmul_rn(s0[ix], a0), __fmul_rn(s0[ix1], fx));
  const float t1 = __fadd_rn(__fmul_rn(s1[ix], a0), __fmul_rn(s1[ix1], fx));
  return __fadd_rn(__fmul_rn(t0, b0), __fmul_rn(t1, fy));
}

__global__ void hed_fuse_kernel(HedSides sd, int B, int H, int W, float inv_scale, float* __restrict__ out) {
  pdl_enter();
  const long long hw = (long long)H * W;
  const long long total = (long long)B * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i / hw);
    const long long p = i % hw;
    const int y = (int)(p / W), x = (int)(p % W);
    float acc = 0.f;
    for (int k = 0; k < sd.n; ++k) {                       // np.mean over a float32 axis: sequential sum, then / n
      const float* s = sd.p[k] + (long long)n * sd.h[k] * sd.w[k];
      const float v = __fmul_rn(resize_linear(s, sd.h[k], sd.w[k], sd.sy[k], sd.sx[k], H, W, y, x), inv_scale);
      acc = k == 0 ? v : __fadd_rn(acc, v);
    }
    const float m = __fdiv_rn(acc, (float)sd.n);
    const double e = 1.0 / (1.0 + exp(-(double)m));
    const double q = fmin(fmax(e * 255.0, 0.0), 255.0);
    const float v = __fdiv_rn((float)(unsigned)q, 255.f);  // astype(uint8) truncates; ToTensor divides by 255
    float* o = out + (long long)n * 3 * hw + p;
    o[0] = v;
    o[hw] = v;
    o[2 * hw] = v;
  }
}

}  // namespace pfd

using namespace pfd;

extern "C" PFD_API int pfd_hed_input_f16(const void* x, int32_t src_is_f32, int32_t B, int32_t H, int32_t W,
                                         int32_t Cpad, const float* norm, float scale, void* out, void* stream) {
  if (!x || !norm || !out || B <= 0 || H <= 0 || W <= 0 || Cpad < 3)
    return set_error("pfd_hed_input_f16: bad arguments (B=%d H=%d W=%d Cpad=%d)", B, H, W, Cpad);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int g = grid_cap((long long)B * H * W, 256);
  if (src_is_f32)
    launch_k(hed_input_kernel<float>, dim3(g), dim3(256), (size_t)0, st, static_cast<const float*>(x), (int)B, (int)H,
             (int)W, (int)Cpad, norm, scale, static_cast<__half*>(out));
  else
    launch_k(hed_input_kernel<__half>, dim3(g), dim3(256), (size_t)0, st, static_cast<const __half*>(x), (int)B, (int)H,
             (int)W, (int)Cpad, norm, scale, static_cast<__half*>(out));
  return check_launch("hed_input");
}

extern "C" PFD_API int pfd_hed_pool_side_f16(const void* x, int32_t B, int32_t h, int32_t w, int32_t C,
                                             const float* proj_w, const float* proj_b, float* side, void* pooled,
                                             void* stream) {
  if (!x || !proj_w || !proj_b || !side || B <= 0 || h <= 0 || w <= 0 || C <= 0 || C % 8 || C > 8192)
    return set_error("pfd_hed_pool_side_f16: bad arguments (B=%d h=%d w=%d C=%d)", B, h, w, C);
  if (misaligned(x) || misaligned(pooled))
    return set_error("pfd_hed_pool_side_f16: x and pooled must be 16-byte aligned");
  int L = 1;
  while (L < C / 8 && L < 32) L <<= 1;
  const long long cells = (long long)B * ((h + 1) / 2) * ((w + 1) / 2);
  const int g = grid_cap(cells, 256 / L);
  launch_k(hed_pool_side_kernel, dim3(g), dim3(256), (size_t)C * sizeof(float), static_cast<cudaStream_t>(stream),
           static_cast<const __half*>(x), (int)B, (int)h, (int)w, (int)C, L, proj_w, proj_b, side,
           static_cast<__half*>(pooled));
  return check_launch("hed_pool_side");
}

extern "C" PFD_API int pfd_hed_fuse_f32(const float* const* sides, const int32_t* side_h, const int32_t* side_w,
                                        int32_t nsides, int32_t B, int32_t H, int32_t W, float inv_scale, float* out,
                                        void* stream) {
  if (!sides || !side_h || !side_w || !out || nsides < 1 || nsides > PFD_HED_MAX_SIDES || B <= 0 || H <= 0 || W <= 0)
    return set_error("pfd_hed_fuse_f32: bad arguments (n=%d B=%d H=%d W=%d)", nsides, B, H, W);
  HedSides sd = {};
  sd.n = nsides;
  for (int k = 0; k < nsides; ++k) {
    if (!sides[k] || side_h[k] <= 0 || side_w[k] <= 0)
      return set_error("pfd_hed_fuse_f32: side map %d is empty", k);
    sd.p[k] = sides[k];
    sd.h[k] = side_h[k];
    sd.w[k] = side_w[k];
    sd.sy[k] = 1.0 / ((double)H / side_h[k]);
    sd.sx[k] = 1.0 / ((double)W / side_w[k]);
  }
  launch_k(hed_fuse_kernel, dim3(grid_cap((long long)B * H * W, 256)), dim3(256), (size_t)0,
           static_cast<cudaStream_t>(stream), sd, (int)B, (int)H, (int)W, inv_scale, out);
  return check_launch("hed_fuse");
}
