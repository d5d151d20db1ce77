// M-LSD line annotator behind ControlNet.preprocess(type='mlsd' / 'mlsd_v11p') on the GPU.
//
// Replaces controlnet.py:378-386 -> controlnet_annotator/mlsd/__init__.py:56-81 (apply_mlsd) -> utils.py:49-88
// (pred_lines, deccode_output_score_and_ptss) around MobileV2_MLSD_Large (models/mbv2_mlsd_large.py).  Every 3x3 and
// 1x1 conv of the network runs on pfd_gemm_f16 (BN folded into the weights at pack time; the dilation-5 conv as 25
// polyphase 3x3 convs on strided views).  This file holds the rest:
//   mlsd_input_kernel     ToPILImage quantisation and concat(rgb, ones): channel-last fp16 [u8 - 127.5 (x3), -126.5,
//                         0 (x12)]; the 1 / 127.5 of the reference's normalisation is folded into the stem weights, so
//                         every input value is exact in fp16 and the TFLite zero pad stays zero (utils.py:56-61);
//   mlsd_dw_kernel        the depthwise 3x3 ConvBNReLU6 of an inverted residual, stride 1 (padding 1) or 2 (TFLite:
//                         pad (0,1,0,1), padding 0), with ReLU6 applied to its input too (the expand GEMM before it
//                         only has ReLU; min(fp16 relu(v), 6) == fp16 relu6(v) because rounding is monotone and 6 is
//                         exact);
//   mlsd_upsample_kernel  F.interpolate(scale_factor=2, bilinear, align_corners=True) into a channel slice of the
//                         BlockTypeA concat buffer (mbv2_mlsd_large.py:27-29);
//   mlsd_head_kernel      block23.conv3 rows 7..11 (the 1x1 that feeds the decode) in fp32, planar fp32 output;
//   mlsd_nms_kernel       sigmoid, the 3x3 max-pool NMS and the thr_v test -> one sortable key per map cell;
//   mlsd_select_kernel    one CTA per image: top-200 of the keys (radix select, ties to the lowest flat index), the
//                         thr_d test in float32 and the float64 endpoints, compacted in flat-index order;
//   mlsd_draw_kernel      cv2.line(..., 1, LINE_8) of every segment: OpenCV's clipLine, then its 8-connected
//                         LineIterator (left to right) in closed form, one warp per segment.
// Every kernel computes an image's values from that image only (no float atomics, no batch-dependent order), so a
// batch gives the same bits as single images.  Segment counts stay on the device: nothing synchronises the host.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/pfd_b200.h"
#include "common.h"
#include "cvdraw.cuh"

namespace pfd {

constexpr int MLSD_TOPK = PFD_MLSD_TOPK;
constexpr int MLSD_CIN = 16;         // stem input channels: rgb, ones, 12 zero pads (the GEMM's 3x3 path needs >= 16)
constexpr int SEL_THREADS = 1024;

// out[n, y, x, :] = [u8(r) - 127.5, u8(g) - 127.5, u8(b) - 127.5, 1 - 127.5, 0 x 12]
template <typename T>
__global__ void __launch_bounds__(256)
mlsd_input_kernel(const T* __restrict__ x, int B, int H, int W, __half* __restrict__ out) {
  pdl_enter();
  const long long hw = (long long)H * W, total = (long long)B * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / hw, p = i % hw;
    const T* src = x + n * 3 * hw + p;
    __align__(16) __half v[8];
    v[0] = __float2half_rn((float)to_u8<T>(src[0]) - 127.5f);
    v[1] = __float2half_rn((float)to_u8<T>(src[hw]) - 127.5f);
    v[2] = __float2half_rn((float)to_u8<T>(src[2 * hw]) - 127.5f);
    v[3] = __float2half_rn(-126.5f);
#pragma unroll
    for (int c = 4; c < 8; ++c) v[c] = __float2half_rn(0.f);
    uint4* o = reinterpret_cast<uint4*>(out + i * MLSD_CIN);
    o[0] = *reinterpret_cast<const uint4*>(v);
    o[1] = make_uint4(0, 0, 0, 0);
  }
}

// One thread per (output pixel, 8-channel vector).  x: [B,H,W,C] fp16 (a ReLU output); w: fp32 [9][C] (tap-major, BN
// folded); b: fp32 [C].  out[n,y,x,c] = clamp(sum_t w[t][c] * min(x[n, S*y+dy, S*x+dx, c], 6) + b[c], 0, 6) with
// (dy, dx) in {-1,0,1}^2 for stride 1 and {0,1,2}^2 for stride 2 (zero outside the image).
template <int S>
__global__ void __launch_bounds__(256)
mlsd_dw_kernel(const __half* __restrict__ x, int B, int H, int W, int C, const float* __restrict__ wt,
               const float* __restrict__ bias, __half* __restrict__ out) {
  pdl_enter();
  const int Ho = S == 1 ? H : H / 2, Wo = S == 1 ? W : W / 2;
  const int V = C / 8;
  const long long total = (long long)B * Ho * Wo * V;
  const int off = S == 1 ? -1 : 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % V);
    long long r = i / V;
    const int ox = (int)(r % Wo);
    r /= Wo;
    const int oy = (int)(r % Ho);
    const long long n = r / Ho;
    const int c0 = v * 8;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int iy = S * oy + t / 3 + off, ix = S * ox + t % 3 + off;
      if (iy < 0 || iy >= H || ix < 0 || ix >= W) continue;
      const uint4 q = *reinterpret_cast<const uint4*>(x + (((n * H + iy) * W + ix) * C + c0));
      const __half* h = reinterpret_cast<const __half*>(&q);
      const float4 w0 = *reinterpret_cast<const float4*>(wt + t * C + c0);
      const float4 w1 = *reinterpret_cast<const float4*>(wt + t * C + c0 + 4);
      const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaf(wv[j], fminf(__half2float(h[j]), 6.f), acc[j]);
    }
    __align__(16) __half o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = __float2half_rn(fminf(fmaxf(acc[j] + bias[c0 + j], 0.f), 6.f));
    *reinterpret_cast<uint4*>(out + (((n * Ho + oy) * Wo + ox) * C + c0)) = *reinterpret_cast<const uint4*>(o);
  }
}

// x: [B,h,w,C] fp16 -> out pixel (n, Y, X) at out + ((n*2h + Y)*2w + X) * pitch, C channels: PyTorch's bilinear rule
// with align_corners=True (scale = (in - 1) / (out - 1) in float32, source = scale * dst, second index clamped).
__global__ void __launch_bounds__(256)
mlsd_upsample_kernel(const __half* __restrict__ x, int B, int h, int w, int C, __half* __restrict__ out, long long pitch) {
  pdl_enter();
  const int Ho = 2 * h, Wo = 2 * w, V = C / 8;
  const float sy = Ho > 1 ? (float)(h - 1) / (float)(Ho - 1) : 0.f;
  const float sx = Wo > 1 ? (float)(w - 1) / (float)(Wo - 1) : 0.f;
  const long long total = (long long)B * Ho * Wo * V;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % V);
    long long r = i / V;
    const int X = (int)(r % Wo);
    r /= Wo;
    const int Y = (int)(r % Ho);
    const long long n = r / Ho;
    const float fy = sy * (float)Y, fx = sx * (float)X;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < h - 1 ? 1 : 0), x1 = x0 + (x0 < w - 1 ? 1 : 0);
    const float ly1 = fy - (float)y0, lx1 = fx - (float)x0, ly0 = 1.f - ly1, lx0 = 1.f - lx1;
    const __half* base = x + n * h * w * C + v * 8;
    const uint4 q00 = *reinterpret_cast<const uint4*>(base + ((long long)y0 * w + x0) * C);
    const uint4 q01 = *reinterpret_cast<const uint4*>(base + ((long long)y0 * w + x1) * C);
    const uint4 q10 = *reinterpret_cast<const uint4*>(base + ((long long)y1 * w + x0) * C);
    const uint4 q11 = *reinterpret_cast<const uint4*>(base + ((long long)y1 * w + x1) * C);
    const __half* a = reinterpret_cast<const __half*>(&q00);
    const __half* b = reinterpret_cast<const __half*>(&q01);
    const __half* c = reinterpret_cast<const __half*>(&q10);
    const __half* d = reinterpret_cast<const __half*>(&q11);
    __align__(16) __half o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      o[j] = __float2half_rn(ly0 * (lx0 * __half2float(a[j]) + lx1 * __half2float(b[j])) +
                             ly1 * (lx0 * __half2float(c[j]) + lx1 * __half2float(d[j])));
    *reinterpret_cast<uint4*>(out + ((n * Ho + Y) * Wo + X) * pitch + v * 8) = *reinterpret_cast<const uint4*>(o);
  }
}

// One thread per pixel: out[n, k, y, x] = b[k] + sum_c w[k][c] * x[n, y, x, c] in fp32, k < 5 (planar output).
__global__ void __launch_bounds__(128)
mlsd_head_kernel(const __half* __restrict__ x, int B, int h, int w, int C, const float* __restrict__ wt,
                 const float* __restrict__ bias, float* __restrict__ out) {
  extern __shared__ float s_w[];
  pdl_enter();
  for (int i = threadIdx.x; i < 5 * C; i += blockDim.x) s_w[i] = wt[i];
  __syncthreads();
  const long long hw = (long long)h * w, total = (long long)B * hw;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
    float acc[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) acc[k] = bias[k];
    const __half* src = x + p * C;
    for (int c0 = 0; c0 < C; c0 += 8) {
      const uint4 q = *reinterpret_cast<const uint4*>(src + c0);
      const __half* hv = reinterpret_cast<const __half*>(&q);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float v = __half2float(hv[j]);
#pragma unroll
        for (int k = 0; k < 5; ++k) acc[k] = fmaf(s_w[k * C + c0 + j], v, acc[k]);
      }
    }
    const long long n = p / hw, q = p % hw;
#pragma unroll
    for (int k = 0; k < 5; ++k) out[(n * 5 + k) * hw + q] = acc[k];
  }
}

__device__ __forceinline__ float mlsd_sigmoid(float v) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-v))); }

// key[n, i] = bits(heat) + 1 when map cell i is a 3x3 maximum of heat = sigmoid(centre) (max_pool2d's padding never
// wins) and heat > thr_v, else 0.  Positive floats order like their bit patterns, so keys order like scores.
__global__ void __launch_bounds__(256)
mlsd_nms_kernel(const float* __restrict__ maps, int B, int h, int w, float thr_v, uint32_t* __restrict__ keys) {
  pdl_enter();
  const long long hw = (long long)h * w, total = (long long)B * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / hw, p = i % hw;
    const int y = (int)(p / w), x = (int)(p % w);
    const float* c = maps + n * 5 * hw;
    const float v = mlsd_sigmoid(c[p]);
    bool keep = true;
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int yy = y + dy, xx = x + dx;
        if ((dy || dx) && yy >= 0 && yy < h && xx >= 0 && xx < w && mlsd_sigmoid(c[(long long)yy * w + xx]) > v)
          keep = false;
      }
    keys[i] = (keep && v > thr_v) ? __float_as_uint(v) + 1u : 0u;
  }
}

// Exclusive block-wide prefix sum of v over SEL_THREADS threads; *total gets the sum.  s: 32 ints of shared memory.
__device__ __forceinline__ int block_scan(int v, int* s, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int t = s[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += y;
    }
    s[lane] = t;
  }
  __syncthreads();
  const int pre = (warp ? s[warp - 1] : 0) + x - v;
  *total = s[31];
  __syncthreads();
  return pre;
}

// One CTA per image.  The top-200 keys (radix select over the key bits, 8 bits per pass; among equal keys the lowest
// flat indices), then for each selected cell in flat-index order the reference's distance test
// sqrt((sx - ex)^2 + (sy - ey)^2) > thr_d in float32 and the endpoints int(2 * (x + d)) in float64 (truncated toward
// zero; clamped to +-2^30, far outside any image).  segs: int32 [B, 200, 4] (x0, y0, x1, y1); count: int32 [B].
__global__ void __launch_bounds__(SEL_THREADS)
mlsd_select_kernel(const uint32_t* __restrict__ keys, const float* __restrict__ maps, int h, int w, float thr_d,
                   int* __restrict__ segs, int* __restrict__ count) {
  __shared__ int hist[256];
  __shared__ int s_scan[32];
  __shared__ uint32_t s_prefix, s_mask;
  __shared__ int s_rem, s_all;
  pdl_enter();
  const int n = blockIdx.x;
  const long long hw = (long long)h * w;
  const uint32_t* K = keys + n * hw;
  const float* M = maps + n * 5 * hw;
  if (threadIdx.x == 0) {
    s_prefix = 0;
    s_mask = 0;
    s_rem = MLSD_TOPK;
    s_all = 0;
  }
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    for (int i = threadIdx.x; i < 256; i += SEL_THREADS) hist[i] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix, mask = s_mask;
    for (long long i = threadIdx.x; i < hw; i += SEL_THREADS) {
      const uint32_t k = K[i];
      if (k && (k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      if (pass == 0) {
        int tot = 0;
        for (int b = 0; b < 256; ++b) tot += hist[b];
        if (tot <= MLSD_TOPK) s_all = 1;
      }
      if (!s_all) {
        int cum = 0;
        for (int b = 255; b >= 0; --b) {
          if (cum + hist[b] >= s_rem) {
            s_prefix |= (uint32_t)b << shift;
            s_mask |= 255u << shift;
            s_rem -= cum;
            break;
          }
          cum += hist[b];
        }
      }
    }
    __syncthreads();
    if (s_all) break;
  }
  // every key > T is taken, and the first `rem` keys == T in flat-index order; with <= 200 candidates, all of them
  const uint32_t T = s_all ? 0u : s_prefix;
  const int rem = s_all ? 0 : s_rem;
  int eq_base = 0, out_base = 0;
  for (long long c0 = 0; c0 < hw; c0 += SEL_THREADS) {
    const long long i = c0 + threadIdx.x;
    const uint32_t k = i < hw ? K[i] : 0u;
    if (!__syncthreads_or(k != 0u && k >= T)) continue;       // nothing selected in this chunk
    const int eq = (k != 0u && k == T) ? 1 : 0;
    int tot_eq;
    const int r = block_scan(eq, s_scan, &tot_eq);
    const bool sel = k > T || (eq && eq_base + r < rem);
    eq_base += tot_eq;
    int ok = 0;
    float d0 = 0.f, d1 = 0.f, d2 = 0.f, d3 = 0.f;
    if (sel) {
      d0 = M[hw + i];
      d1 = M[2 * hw + i];
      d2 = M[3 * hw + i];
      d3 = M[4 * hw + i];
      const float ex = __fsub_rn(d0, d2), ey = __fsub_rn(d1, d3);
      const float dist = __fsqrt_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)));
      ok = dist > thr_d ? 1 : 0;
    }
    int tot_ok;
    const int j = out_base + block_scan(ok, s_scan, &tot_ok);
    if (ok && j < MLSD_TOPK) {
      const double x = (double)(i % w), y = (double)(i / w);
      const double e[4] = {__dmul_rn(2.0, __dadd_rn(x, (double)d0)), __dmul_rn(2.0, __dadd_rn(y, (double)d1)),
                           __dmul_rn(2.0, __dadd_rn(x, (double)d2)), __dmul_rn(2.0, __dadd_rn(y, (double)d3))};
      int* o = segs + ((long long)n * MLSD_TOPK + j) * 4;
#pragma unroll
      for (int q = 0; q < 4; ++q) o[q] = (int)fmin(fmax(trunc(e[q]), -1073741824.0), 1073741824.0);
    }
    out_base += tot_ok;
  }
  if (threadIdx.x == 0) count[n] = out_base < MLSD_TOPK ? out_base : MLSD_TOPK;
}

// One warp per segment slot (blockIdx.y = image).  out: [B,3,H,W], 1.0 on the line.
__global__ void __launch_bounds__(256)
mlsd_draw_kernel(const int* __restrict__ segs, const int* __restrict__ count, int H, int W, float* __restrict__ out) {
  pdl_enter();
  const int n = blockIdx.y;
  const int s = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (s >= count[n]) return;
  const int* sg = segs + ((long long)n * MLSD_TOPK + s) * 4;
  const long long hw = (long long)H * W;
  float* o = out + (long long)n * 3 * hw;
  for_each_line_pixel(W, H, sg[0], sg[1], sg[2], sg[3], lane, [&](long long x, long long y) {
    const long long p = y * W + x;
    o[p] = 1.f;
    o[hw + p] = 1.f;
    o[2 * hw + p] = 1.f;
  });
}

}  // namespace pfd

using namespace pfd;


extern "C" PFD_API int pfd_mlsd_input_f16(const void* x, int32_t x_f32, int32_t B, int32_t H, int32_t W, void* out,
                                          void* stream) {
  if (!x || !out || B <= 0 || H <= 0 || W <= 0)
    return set_error("pfd_mlsd_input_f16: bad arguments (B=%d H=%d W=%d)", B, H, W);
  if (misaligned(out)) return set_error("pfd_mlsd_input_f16: out must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int g = grid_cap((long long)B * H * W, 256);
  if (x_f32)
    launch_k(mlsd_input_kernel<float>, dim3(g), dim3(256), (size_t)0, st, static_cast<const float*>(x), (int)B, (int)H,
             (int)W, static_cast<__half*>(out));
  else
    launch_k(mlsd_input_kernel<__half>, dim3(g), dim3(256), (size_t)0, st, static_cast<const __half*>(x), (int)B,
             (int)H, (int)W, static_cast<__half*>(out));
  return check_launch("mlsd_input");
}

extern "C" PFD_API int pfd_mlsd_dw_f16(const void* x, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride,
                                       const float* w, const float* b, void* out, void* stream) {
  if (!x || !w || !b || !out || B <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8 || (stride != 1 && stride != 2) ||
      (stride == 2 && (H < 2 || W < 2)))
    return set_error("pfd_mlsd_dw_f16: bad arguments (B=%d H=%d W=%d C=%d stride=%d)", B, H, W, C, stride);
  if (misaligned(x) || misaligned(w) || misaligned(out))
    return set_error("pfd_mlsd_dw_f16: x, w and out must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long work = (long long)B * (H / stride) * (W / stride) * (C / 8);
  const int g = grid_cap(work, 256);
  if (stride == 1)
    launch_k(mlsd_dw_kernel<1>, dim3(g), dim3(256), (size_t)0, st, static_cast<const __half*>(x), (int)B, (int)H,
             (int)W, (int)C, w, b, static_cast<__half*>(out));
  else
    launch_k(mlsd_dw_kernel<2>, dim3(g), dim3(256), (size_t)0, st, static_cast<const __half*>(x), (int)B, (int)H,
             (int)W, (int)C, w, b, static_cast<__half*>(out));
  return check_launch("mlsd_dw");
}

extern "C" PFD_API int pfd_mlsd_upsample_f16(const void* x, int32_t B, int32_t h, int32_t w, int32_t C, void* out,
                                             int64_t pitch, void* stream) {
  if (!x || !out || B <= 0 || h <= 0 || w <= 0 || C <= 0 || C % 8 || pitch < C || pitch % 8)
    return set_error("pfd_mlsd_upsample_f16: bad arguments (B=%d h=%d w=%d C=%d pitch=%lld)", B, h, w, C,
                     (long long)pitch);
  if (misaligned(x) || misaligned(out)) return set_error("pfd_mlsd_upsample_f16: x and out must be 16-byte aligned");
  const int g = grid_cap((long long)B * 4 * h * w * (C / 8), 256);
  launch_k(mlsd_upsample_kernel, dim3(g), dim3(256), (size_t)0, static_cast<cudaStream_t>(stream),
           static_cast<const __half*>(x), (int)B, (int)h, (int)w, (int)C, static_cast<__half*>(out), (long long)pitch);
  return check_launch("mlsd_upsample");
}

extern "C" PFD_API int pfd_mlsd_head_f32(const void* x, int32_t B, int32_t h, int32_t w, int32_t C, const float* wt,
                                         const float* b, float* out, void* stream) {
  if (!x || !wt || !b || !out || B <= 0 || h <= 0 || w <= 0 || C <= 0 || C % 8 || C > 256)
    return set_error("pfd_mlsd_head_f32: bad arguments (B=%d h=%d w=%d C=%d)", B, h, w, C);
  if (misaligned(x)) return set_error("pfd_mlsd_head_f32: x must be 16-byte aligned");
  launch_k(mlsd_head_kernel, dim3(grid_cap((long long)B * h * w, 128)), dim3(128), (size_t)5 * C * sizeof(float),
           static_cast<cudaStream_t>(stream), static_cast<const __half*>(x), (int)B, (int)h, (int)w, (int)C, wt, b, out);
  return check_launch("mlsd_head");
}

extern "C" PFD_API int pfd_mlsd_decode_f32(const float* maps, int32_t B, int32_t h, int32_t w, float thr_v, float thr_d,
                                           uint32_t* keys, int32_t* segs, int32_t* count, void* stream) {
  if (!maps || !keys || !segs || !count || B <= 0 || h <= 0 || w <= 0 || (long long)h * w < MLSD_TOPK)
    return set_error("pfd_mlsd_decode_f32: bad arguments (B=%d h=%d w=%d; h*w must be >= %d)", B, h, w, MLSD_TOPK);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  launch_k(mlsd_nms_kernel, dim3(grid_cap((long long)B * h * w, 256)), dim3(256), (size_t)0, st, maps, (int)B,
           (int)h, (int)w, thr_v, keys);
  if (int rc = check_launch("mlsd_nms")) return rc;
  launch_k(mlsd_select_kernel, dim3(B), dim3(SEL_THREADS), (size_t)0, st, static_cast<const uint32_t*>(keys), maps,
           (int)h, (int)w, thr_d, static_cast<int*>(segs), static_cast<int*>(count));
  return check_launch("mlsd_select");
}

extern "C" PFD_API int pfd_mlsd_draw_f32(const int32_t* segs, const int32_t* count, int32_t B, int32_t H, int32_t W,
                                         float* out, void* stream) {
  if (!segs || !count || !out || B <= 0 || H <= 0 || W <= 0 || B > 65535)
    return set_error("pfd_mlsd_draw_f32: bad arguments (B=%d H=%d W=%d)", B, H, W);
  const dim3 grid((MLSD_TOPK + 7) / 8, B);
  launch_k(mlsd_draw_kernel, grid, dim3(256), (size_t)0, static_cast<cudaStream_t>(stream),
           static_cast<const int*>(segs), static_cast<const int*>(count), (int)H, (int)W, out);
  return check_launch("mlsd_draw");
}
