// PiDiNet soft-edge annotator behind ControlNet.preprocess(type='scribble') (default method 'pidinet') on the GPU.
//
// Replaces controlnet.py:465-472 -> controlnet_annotator/pidinet/__init__.py:67-96 (apply_pidinet) around the network
// pidinet() of pidinet/model.py:441-666 ('carv4', 60 channels, dil=24, sa=True).  The input step reuses
// pfd_hed_input_f16 + im2col3x3 + pfd_gemm_f16, and every 1x1 conv of the trunk (conv2 + x, or conv2 + shortcut as a
// two-segment K) runs on pfd_gemm_f16.  This file holds the rest:
//   pidinet_dw_kernel      the depthwise pixel-difference conv of a block (weights converted to a plain 3x3 / 5x5 at
//                          pack time), fp32 accumulation, ReLU fused; for the first block of a stage the 2x2 max-pool
//                          is fused in front and the pooled tensor is written too (model.py:454-463);
//   pidinet_reduce_kernel  CDCM's ReLU + 1x1 conv to 24 channels with bias (model.py:418-420);
//   pidinet_cdcm_kernel    the sum of CDCM's four dilated 3x3 convs 24 -> 24 (dilation 5, 7, 9, 11, model.py:421-425)
//                          as one implicit GEMM on the tensor cores (mma.sync m16n8k16, fp16 in, fp32 accumulation);
//   pidinet_side_kernel    CSAM (model.py:395-401) and MapReduce (model.py:437-438) to the stage's side map;
//   pidinet_fuse_kernel    F.interpolate(bilinear, align_corners=False) of the four side maps, the classifier 1x1 conv,
//                          sigmoid, (edge*255).clip(0,255).astype(uint8), ToTensor and repeat to RGB (model.py:626-645,
//                          pidinet/__init__.py:88-96, controlnet.py:469-471).
// Every kernel computes an output pixel from its own image only, so a batch gives the same bits as single images.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/pfd_b200.h"
#include "common.h"

namespace pfd {

__device__ __forceinline__ uint4 hmax4(uint4 a, uint4 b) {
  uint4 r;
  const __half2* x = reinterpret_cast<const __half2*>(&a);
  const __half2* y = reinterpret_cast<const __half2*>(&b);
  __half2* o = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int j = 0; j < 4; ++j) o[j] = __hmax2(x[j], y[j]);
  return r;
}

// One thread per (output pixel, 8-channel vector).  x: [B,Hin,Win,C] fp16; w: fp32 [KS*KS][C] (tap-major);
// out = relu(depthwise conv of the input, zero padding KS/2) [B,h,w,C] fp16.  POOL: the conv input is the 2x2 / stride 2
// max-pool of x (h = Hin/2, w = Win/2, floor), also written to pooled; otherwise h = Hin, w = Win.
template <int KS, bool POOL>
__global__ void __launch_bounds__(256)
pidinet_dw_kernel(const __half* __restrict__ x, int B, int Hin, int Win, int C, const float* __restrict__ wt,
                  __half* __restrict__ out, __half* __restrict__ pooled) {
  pdl_enter();
  const int h = POOL ? Hin / 2 : Hin, w = POOL ? Win / 2 : Win;
  const int V = C / 8;
  const long long total = (long long)B * h * w * V;
  constexpr int R = KS / 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % V);
    const long long pix = i / V;
    const int px = (int)(pix % w);
    const int py = (int)((pix / w) % h);
    const int n = (int)(pix / ((long long)w * h));
    const __half* xn = x + (long long)n * Hin * Win * C + 8 * v;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int ky = 0; ky < KS; ++ky) {
      const int yy = py + ky - R;
      if (yy < 0 || yy >= h) continue;
#pragma unroll
      for (int kx = 0; kx < KS; ++kx) {
        const int xx = px + kx - R;
        if (xx < 0 || xx >= w) continue;
        uint4 q;
        if (POOL) {
          const __half* p0 = xn + ((long long)(2 * yy) * Win + 2 * xx) * C;
          q = hmax4(hmax4(__ldg(reinterpret_cast<const uint4*>(p0)), __ldg(reinterpret_cast<const uint4*>(p0 + C))),
                    hmax4(__ldg(reinterpret_cast<const uint4*>(p0 + (long long)Win * C)),
                          __ldg(reinterpret_cast<const uint4*>(p0 + (long long)Win * C + C))));
          if (ky == R && kx == R)
            *reinterpret_cast<uint4*>(pooled + (((long long)n * h + py) * w + px) * C + 8 * v) = q;
        } else {
          q = __ldg(reinterpret_cast<const uint4*>(xn + ((long long)yy * Win + xx) * C));
        }
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(wt + (ky * KS + kx) * C + 8 * v));
        const float4 w1 = __ldg(reinterpret_cast<const float4*>(wt + (ky * KS + kx) * C + 8 * v + 4));
        const __half2* hq = reinterpret_cast<const __half2*>(&q);
        const float2 f0 = __half22float2(hq[0]), f1 = __half22float2(hq[1]);
        const float2 f2 = __half22float2(hq[2]), f3 = __half22float2(hq[3]);
        acc[0] = fmaf(f0.x, w0.x, acc[0]);
        acc[1] = fmaf(f0.y, w0.y, acc[1]);
        acc[2] = fmaf(f1.x, w0.z, acc[2]);
        acc[3] = fmaf(f1.y, w0.w, acc[3]);
        acc[4] = fmaf(f2.x, w1.x, acc[4]);
        acc[5] = fmaf(f2.y, w1.y, acc[5]);
        acc[6] = fmaf(f3.x, w1.z, acc[6]);
        acc[7] = fmaf(f3.y, w1.w, acc[7]);
      }
    }
    uint4 o;
    __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) ho[j] = __floats2half2_rn(fmaxf(acc[2 * j], 0.f), fmaxf(acc[2 * j + 1], 0.f));
    *reinterpret_cast<uint4*>(out + pix * C + 8 * v) = o;
  }
}

constexpr int PIDI_D = 24;  // CDCM / CSAM / MapReduce width (dil=24)

// One thread per pixel: m[p, o] = b[o] + sum_c relu(x[p, c]) * w[c, o], o < 24.  x: [P, C] fp16; w: fp32 [C][24] in
// shared memory; m: [P, 24] fp16.
__global__ void __launch_bounds__(128)
pidinet_reduce_kernel(const __half* __restrict__ x, long long P, int C, const float* __restrict__ wg,
                      const float* __restrict__ bg, __half* __restrict__ m) {
  extern __shared__ float s_w[];
  pdl_enter();
  for (int i = threadIdx.x; i < C * PIDI_D; i += blockDim.x) s_w[i] = wg[i];
  __syncthreads();
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (long long)gridDim.x * blockDim.x) {
    float acc[PIDI_D];
#pragma unroll
    for (int o = 0; o < PIDI_D; ++o) acc[o] = __ldg(bg + o);
    const uint4* xp = reinterpret_cast<const uint4*>(x + p * C);
    for (int v = 0; v < C / 8; ++v) {
      const uint4 q = __ldg(xp + v);
      const __half2* hq = reinterpret_cast<const __half2*>(&q);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(hq[j]);
        const float a = fmaxf(f.x, 0.f), b = fmaxf(f.y, 0.f);
        const float* w0 = s_w + (8 * v + 2 * j) * PIDI_D;
#pragma unroll
        for (int o = 0; o < PIDI_D; ++o) acc[o] = fmaf(a, w0[o], acc[o]);
#pragma unroll
        for (int o = 0; o < PIDI_D; ++o) acc[o] = fmaf(b, w0[PIDI_D + o], acc[o]);
      }
    }
    uint4 r[3];
    __half2* hr = reinterpret_cast<__half2*>(r);
#pragma unroll
    for (int o = 0; o < PIDI_D / 2; ++o) hr[o] = __floats2half2_rn(acc[2 * o], acc[2 * o + 1]);
    uint4* mp = reinterpret_cast<uint4*>(m + p * PIDI_D);
    mp[0] = r[0];
    mp[1] = r[1];
    mp[2] = r[2];
  }
}

// CDCM dilated convs: u[n,y,x,:] = sum_{d in 5,7,9,11} sum_{ky,kx} W_d[:, :, ky, kx] . m[n, y+(ky-1)d, x+(kx-1)d, :]
// (zero padding), an implicit GEMM with M = pixels, N = 24, K = 4 * 9 * 24 = 864.  K is walked in 108 halves of 8
// channels (tap-major, then channel group 0..2 of the tap); two consecutive halves form one k16 step, so a step may
// straddle two taps and no K is padded.  A CTA owns a 16x16 pixel tile: the 24-channel input with an 11-pixel halo
// (38x38 pixels, zero outside the image) is staged once in shared memory, the weights arrive pre-arranged in the B
// fragment order of mma.m16n8k16 ([54 steps][3 n-tiles][32 lanes] x 2 words).  Warp w computes tile rows 4w..4w+3,
// one m16 tile (16 pixels of a row) each.  Pixel rows are 12 words apart, so the 8 fragment rows x 4 lanes of an A load
// hit 32 distinct banks.
constexpr int CD_T = 16, CD_HALO = 11, CD_S = CD_T + 2 * CD_HALO, CD_STEPS = 54;
constexpr int CD_THREADS = 128;
constexpr size_t CD_SMEM_TILE = (size_t)CD_S * CD_S * PIDI_D * 2;
constexpr size_t CD_SMEM_W = (size_t)CD_STEPS * 3 * 32 * 8;
constexpr size_t CD_SMEM = CD_SMEM_TILE + CD_SMEM_W;

__device__ __forceinline__ void mma16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// word offset (relative to the tile origin) of half hh's channel group at its tap's displacement
__device__ __forceinline__ int cd_half_off(int hh) {
  const int tap = hh / 3, cg = hh - 3 * (hh / 3);
  const int di = tap / 9, t9 = tap - 9 * di;
  const int d = 5 + 2 * di;
  const int dy = (t9 / 3 - 1) * d, dx = (t9 % 3 - 1) * d;
  return (dy * CD_S + dx) * (PIDI_D / 2) + cg * 4;
}

__global__ void __launch_bounds__(CD_THREADS, 2)
pidinet_cdcm_kernel(const __half* __restrict__ m, int h, int w, const uint2* __restrict__ wpk, float* __restrict__ u) {
  extern __shared__ __align__(16) unsigned char cd_smem[];
  uint4* s_tile = reinterpret_cast<uint4*>(cd_smem);
  const uint32_t* s_tw = reinterpret_cast<const uint32_t*>(cd_smem);
  uint2* s_b = reinterpret_cast<uint2*>(cd_smem + CD_SMEM_TILE);
  pdl_enter();
  const int n = blockIdx.z, ty0 = blockIdx.y * CD_T, tx0 = blockIdx.x * CD_T;
  for (int i = threadIdx.x; i < CD_STEPS * 3 * 32; i += CD_THREADS) s_b[i] = __ldg(wpk + i);
  const __half* mn = m + (long long)n * h * w * PIDI_D;
  for (int i = threadIdx.x; i < CD_S * CD_S * 3; i += CD_THREADS) {
    const int c = i % 3, p = i / 3;
    const int yy = ty0 - CD_HALO + p / CD_S, xx = tx0 - CD_HALO + p % CD_S;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (yy >= 0 && yy < h && xx >= 0 && xx < w)
      v = __ldg(reinterpret_cast<const uint4*>(mn + ((long long)yy * w + xx) * PIDI_D) + c);
    s_tile[i] = v;
  }
  __syncthreads();
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32, g = lane / 4, t = lane % 4;
  float acc[4][3][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[r][j][e] = 0.f;
  // word index of (tile row 4*warp, column g, channel 2t) in the staged tile
  const int base = ((4 * warp + CD_HALO) * CD_S + g + CD_HALO) * (PIDI_D / 2) + t;
#pragma unroll 2
  for (int s = 0; s < CD_STEPS; ++s) {
    const int o0 = base + cd_half_off(2 * s), o1 = base + cd_half_off(2 * s + 1);
    uint2 b[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) b[j] = s_b[(s * 3 + j) * 32 + lane];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int ro = r * CD_S * (PIDI_D / 2);
      uint32_t a[4];
      a[0] = s_tw[o0 + ro];
      a[1] = s_tw[o0 + ro + 8 * (PIDI_D / 2)];
      a[2] = s_tw[o1 + ro];
      a[3] = s_tw[o1 + ro + 8 * (PIDI_D / 2)];
#pragma unroll
      for (int j = 0; j < 3; ++j) mma16816(acc[r][j], a, b[j].x, b[j].y);
    }
  }
  float* un = u + (long long)n * h * w * PIDI_D;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int yy = ty0 + 4 * warp + r;
    if (yy >= h) continue;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int xx = tx0 + g + 8 * half;
      if (xx >= w) continue;
      float* up = un + ((long long)yy * w + xx) * PIDI_D + 2 * t;
#pragma unroll
      for (int j = 0; j < 3; ++j)
        *reinterpret_cast<float2*>(up + 8 * j) = make_float2(acc[r][j][2 * half], acc[r][j][2 * half + 1]);
    }
  }
}

// CSAM + MapReduce of one stage, one thread per pixel.  u: [B,h,w,24] fp32 (the CDCM output);
// prm: fp32 [PFD_PIDINET_SIDE_PARAMS] = csam conv1 weight [4][24], conv1 bias [4], conv2 weight [4][9] (tap-major
// within a channel), MapReduce weight [24], MapReduce bias [1].
//   a    = sigmoid(sum_{tap, c} conv2[c, tap] * y_c(p + tap)),  y_c(q) = conv1_b[c] + conv1_w[c] . relu(u(q)) inside the
//          image and 0 outside (conv2 zero-pads y);
//   side = conv_reduce(u * a) = a * (mr_w . u(p)) + mr_b: a is one scalar per pixel, so the product with u commutes with
//          the 1x1 conv.
__global__ void __launch_bounds__(256)
pidinet_side_kernel(const float* __restrict__ u, int B, int h, int w, const float* __restrict__ prm,
                    float* __restrict__ side) {
  __shared__ float s_p[PFD_PIDINET_SIDE_PARAMS];
  pdl_enter();
  for (int i = threadIdx.x; i < PFD_PIDINET_SIDE_PARAMS; i += blockDim.x) s_p[i] = prm[i];
  __syncthreads();
  const float* w1 = s_p;
  const float* b1 = s_p + 4 * PIDI_D;
  const float* w2 = b1 + 4;
  const float* wr = w2 + 36;
  const float br = wr[PIDI_D];
  const long long total = (long long)B * h * w;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % w), y = (int)((i / w) % h);
    const long long n = i / ((long long)w * h);
    const float* un = u + n * h * w * PIDI_D;
    float z = 0.f;
    for (int tap = 0; tap < 9; ++tap) {
      const int yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
      if (yy < 0 || yy >= h || xx < 0 || xx >= w) continue;
      const float4* q = reinterpret_cast<const float4*>(un + ((long long)yy * w + xx) * PIDI_D);
      float yc[4] = {b1[0], b1[1], b1[2], b1[3]};
#pragma unroll
      for (int v = 0; v < PIDI_D / 4; ++v) {
        const float4 f = __ldg(q + v);
        const float r[4] = {fmaxf(f.x, 0.f), fmaxf(f.y, 0.f), fmaxf(f.z, 0.f), fmaxf(f.w, 0.f)};
#pragma unroll
        for (int c = 0; c < 4; ++c)
#pragma unroll
          for (int k = 0; k < 4; ++k) yc[c] = fmaf(w1[c * PIDI_D + 4 * v + k], r[k], yc[c]);
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) z = fmaf(w2[c * 9 + tap], yc[c], z);
    }
    const float a = 1.f / (1.f + expf(-z));
    const float4* q = reinterpret_cast<const float4*>(un + ((long long)y * w + x) * PIDI_D);
    float e = 0.f;
#pragma unroll
    for (int v = 0; v < PIDI_D / 4; ++v) {
      const float4 f = __ldg(q + v);
      e = fmaf(wr[4 * v], f.x, e);
      e = fmaf(wr[4 * v + 1], f.y, e);
      e = fmaf(wr[4 * v + 2], f.z, e);
      e = fmaf(wr[4 * v + 3], f.w, e);
    }
    side[i] = fmaf(a, e, br);
  }
}

struct PidiSides {
  const float* p[4];
  int h[4], w[4];
  float sy[4], sx[4];  // PyTorch's scale = float(in) / out
};

// F.interpolate(bilinear, align_corners=False) source position: max(0, fma(d + 0.5, scale, -0.5)), index = floor,
// lambda = pos - index, second index clamped at the edge.
__device__ __forceinline__ void bil_coord(int d, float scale, int n, int& i0, int& i1, float& lam) {
  const float pos = fmaxf(fmaf((float)d + 0.5f, scale, -0.5f), 0.f);
  i0 = (int)pos;
  lam = pos - (float)i0;
  i1 = min(i0 + 1, n - 1);
}

__device__ __forceinline__ float bil_lerp(float a0, float a1, float lam) {
  return fmaf(a0, 1.f - lam, __fmul_rn(a1, lam));
}

// PyTorch's CPU kernel for outputs with H + W > 128: a pass along the width, then along the height, each skipped when
// its size does not change (restated in oracle/pidinet_oracle.resize_bilinear).
__device__ __forceinline__ float resize_bilinear_pt(const float* __restrict__ s, int h, int w, float sy, float sx,
                                                    int H, int W, int y, int x) {
  int x0 = x, x1 = x, y0 = y, y1 = y;
  float lx = 0.f, ly = 0.f;
  if (w != W) bil_coord(x, sx, w, x0, x1, lx);
  if (h != H) bil_coord(y, sy, h, y0, y1, ly);
  const float* r0 = s + (long long)y0 * w;
  const float* r1 = s + (long long)y1 * w;
  const float t0 = w != W ? bil_lerp(r0[x0], r0[x1], lx) : r0[x];
  if (h == H) return t0;
  const float t1 = w != W ? bil_lerp(r1[x0], r1[x1], lx) : r1[x];
  return bil_lerp(t0, t1, ly);
}

__global__ void pidinet_fuse_kernel(PidiSides sd, int B, int H, int W, const float* __restrict__ cls,
                                    float* __restrict__ out) {
  pdl_enter();
  const double c0 = cls[0], c1 = cls[1], c2 = cls[2], c3 = cls[3], cb = cls[4];
  const long long hw = (long long)H * W;
  const long long total = (long long)B * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i / hw);
    const long long p = i % hw;
    const int y = (int)(p / W), x = (int)(p % W);
    float e[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      e[k] = resize_bilinear_pt(sd.p[k] + (long long)n * sd.h[k] * sd.w[k], sd.h[k], sd.w[k], sd.sy[k], sd.sx[k], H, W,
                                y, x);
    const double a = cb + c0 * e[0] + c1 * e[1] + c2 * e[2] + c3 * e[3];
    const double q = fmin(fmax(255.0 / (1.0 + exp(-a)), 0.0), 255.0);
    const float v = __fdiv_rn((float)(unsigned)q, 255.f);  // astype(uint8) truncates; ToTensor divides by 255
    float* o = out + (long long)n * 3 * hw + p;
    o[0] = v;
    o[hw] = v;
    o[2 * hw] = v;
  }
}

}  // namespace pfd

using namespace pfd;

extern "C" PFD_API int pfd_pidinet_dw_f16(const void* x, int32_t B, int32_t Hin, int32_t Win, int32_t C, int32_t ks,
                                          int32_t pool, const float* w, void* out, void* pooled, void* stream) {
  if (!x || !w || !out || B <= 0 || Hin <= 0 || Win <= 0 || C <= 0 || C % 8 || (ks != 3 && ks != 5) ||
      (pool && (!pooled || ks != 3 || Hin < 2 || Win < 2)))
    return set_error("pfd_pidinet_dw_f16: bad arguments (B=%d H=%d W=%d C=%d ks=%d pool=%d)", B, Hin, Win, C, ks, pool);
  if (misaligned(x) || misaligned(out) || misaligned(pooled) || misaligned(w))
    return set_error("pfd_pidinet_dw_f16: x, w, out and pooled must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long work = (long long)B * (pool ? Hin / 2 : Hin) * (pool ? Win / 2 : Win) * (C / 8);
  const int g = grid_cap(work, 256);
  const __half* xi = static_cast<const __half*>(x);
  __half* o = static_cast<__half*>(out);
  __half* p = static_cast<__half*>(pooled);
  if (pool)
    launch_k(pidinet_dw_kernel<3, true>, dim3(g), dim3(256), (size_t)0, st, xi, (int)B, (int)Hin, (int)Win, (int)C, w,
             o, p);
  else if (ks == 3)
    launch_k(pidinet_dw_kernel<3, false>, dim3(g), dim3(256), (size_t)0, st, xi, (int)B, (int)Hin, (int)Win, (int)C,
             w, o, p);
  else
    launch_k(pidinet_dw_kernel<5, false>, dim3(g), dim3(256), (size_t)0, st, xi, (int)B, (int)Hin, (int)Win, (int)C,
             w, o, p);
  return check_launch("pidinet_dw");
}

extern "C" PFD_API int pfd_pidinet_reduce_f16(const void* x, int64_t P, int32_t C, const float* w, const float* b,
                                              void* m, void* stream) {
  if (!x || !w || !b || !m || P <= 0 || C <= 0 || C % 8 || C > 512)
    return set_error("pfd_pidinet_reduce_f16: bad arguments (P=%lld C=%d)", (long long)P, C);
  if (misaligned(x) || misaligned(m))
    return set_error("pfd_pidinet_reduce_f16: x and m must be 16-byte aligned");
  launch_k(pidinet_reduce_kernel, dim3(grid_cap(P, 128)), dim3(128), (size_t)C * PIDI_D * sizeof(float),
           static_cast<cudaStream_t>(stream), static_cast<const __half*>(x), (long long)P, (int)C, w, b,
           static_cast<__half*>(m));
  return check_launch("pidinet_reduce");
}

extern "C" PFD_API int pfd_pidinet_cdcm_f16(const void* m, int32_t B, int32_t h, int32_t w, const void* wpk, float* u,
                                            void* stream) {
  if (!m || !wpk || !u || B <= 0 || h <= 0 || w <= 0 || B > 65535)
    return set_error("pfd_pidinet_cdcm_f16: bad arguments (B=%d h=%d w=%d)", B, h, w);
  if (misaligned(m) || misaligned(wpk) || misaligned(u))
    return set_error("pfd_pidinet_cdcm_f16: m, wpk and u must be 16-byte aligned");
  if (int rc = smem_opt_in<pidinet_cdcm_kernel>((int)CD_SMEM, "pidinet_cdcm_kernel")) return rc;
  const dim3 grid((w + CD_T - 1) / CD_T, (h + CD_T - 1) / CD_T, B);
  launch_k(pidinet_cdcm_kernel, grid, dim3(CD_THREADS), CD_SMEM, static_cast<cudaStream_t>(stream),
           static_cast<const __half*>(m), (int)h, (int)w, static_cast<const uint2*>(wpk), u);
  return check_launch("pidinet_cdcm");
}

extern "C" PFD_API int pfd_pidinet_side_f32(const float* u, int32_t B, int32_t h, int32_t w, const float* params,
                                            float* side, void* stream) {
  if (!u || !params || !side || B <= 0 || h <= 0 || w <= 0)
    return set_error("pfd_pidinet_side_f32: bad arguments (B=%d h=%d w=%d)", B, h, w);
  if (misaligned(u)) return set_error("pfd_pidinet_side_f32: u must be 16-byte aligned");
  launch_k(pidinet_side_kernel, dim3(grid_cap((long long)B * h * w, 256)), dim3(256), (size_t)0,
           static_cast<cudaStream_t>(stream), u, (int)B, (int)h, (int)w, params, side);
  return check_launch("pidinet_side");
}

extern "C" PFD_API int pfd_pidinet_fuse_f32(const float* const* sides, const int32_t* side_h, const int32_t* side_w,
                                            int32_t B, int32_t H, int32_t W, const float* cls, float* out,
                                            void* stream) {
  if (!sides || !side_h || !side_w || !cls || !out || B <= 0 || H <= 0 || W <= 0)
    return set_error("pfd_pidinet_fuse_f32: bad arguments (B=%d H=%d W=%d)", B, H, W);
  PidiSides sd = {};
  for (int k = 0; k < 4; ++k) {
    if (!sides[k] || side_h[k] <= 0 || side_w[k] <= 0 || side_h[k] > H || side_w[k] > W)
      return set_error("pfd_pidinet_fuse_f32: side map %d is empty or larger than the output", k);
    sd.p[k] = sides[k];
    sd.h[k] = side_h[k];
    sd.w[k] = side_w[k];
    sd.sy[k] = (float)side_h[k] / (float)H;
    sd.sx[k] = (float)side_w[k] / (float)W;
  }
  launch_k(pidinet_fuse_kernel, dim3(grid_cap((long long)B * H * W, 256)), dim3(256), (size_t)0,
           static_cast<cudaStream_t>(stream), sd, (int)B, (int)H, (int)W, cls, out);
  return check_launch("pidinet_fuse");
}
