// HBM-bound kernels of the Prompt-Free-Diffusion hot path (channel-last fp16, fp32 math):
// GroupNorm(+SiLU, optional two-source concat), LayerNorm(+residual), row softmax with the
// reference's fp16 score rounding, timestep embedding, nearest 2x upsample, layout converts,
// small-Cin im2col, fused CFG + DDIM update, Swin window gather/scatter and patch-merge gather.
// All loads/stores are 128-bit vectorised where the layout allows; reductions use warp shuffles.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>

#include <mutex>

#include "../../include/pfd_b200.h"
#include "common.h"

namespace pfd {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __half22float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 u;
  __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  return u;
}
__device__ __forceinline__ float rh(float v) { return __half2float(__float2half_rn(v)); }

// ------------------------------------------------------------------------------------ GroupNorm
// Thread mapping shared by both passes: blockDim is a multiple of the number of 8-channel vectors
// (vecs = C/8) so a thread always owns the same channel vector and strides over pixels ->
// consecutive threads read consecutive 16-byte vectors of one pixel (fully coalesced), per-channel
// partial sums / affine coefficients live in registers, and nothing is recomputed per element.
//   pass 1 (gn_stats): per-(image, group) sum / sum of squares of d = x - K_g -> fp64 atomics (one per group per CTA)
//   pass 2 (gn_apply): y = x * a[c] + b[c] (a = rstd*gamma, b = beta - mean*a) [+ SiLU] -> fp16
// K_g, the pivot, is the group's first channel at pixel 0 of the image.  Variance does not change under a shift, and
// the one-pass E[d^2] - E[d]^2 loses only (E[d] / std)^2 of the fp32 partial sums' precision instead of (mean / std)^2:
// activations with a large common offset (VAE decoder, real checkpoints) keep a full-precision rstd.
constexpr int GN_MAX_GROUPS = 32;

__device__ __forceinline__ uint4 gn_load(const __half* __restrict__ x1, int c1, const __half* __restrict__ x2,
                                         int c2, long long pixn, int c) {
  if (c < c1) return __ldg(reinterpret_cast<const uint4*>(x1 + pixn * c1 + c));
  return __ldg(reinterpret_cast<const uint4*>(x2 + pixn * c2 + (c - c1)));
}

// pivot K_g of the group holding channel c of image n (HW pixels per image)
__device__ __forceinline__ float gn_pivot(const __half* __restrict__ x1, int c1, const __half* __restrict__ x2,
                                          int c2, long long HW, int n, int cpg, int c) {
  const int gc = c / cpg * cpg;
  const long long pixn = (long long)n * HW;
  return __half2float(gc < c1 ? __ldg(x1 + pixn * c1 + gc) : __ldg(x2 + pixn * c2 + (gc - c1)));
}

// pivots of the groups a thread's 8-channel vector at channel c touches (two loads when a group spans >= 8 channels)
__device__ __forceinline__ void gn_pivots(const __half* __restrict__ x1, int c1, const __half* __restrict__ x2, int c2,
                                          long long HW, int n, int cpg, int c, float (&kp)[8]) {
  if (cpg >= 8) {
    const int gb = (c / cpg + 1) * cpg;     // first channel of the next group
    const float k0 = gn_pivot(x1, c1, x2, c2, HW, n, cpg, c);
    const float k1 = gb < c + 8 ? gn_pivot(x1, c1, x2, c2, HW, n, cpg, gb) : k0;
#pragma unroll
    for (int i = 0; i < 8; ++i) kp[i] = c + i < gb ? k0 : k1;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) kp[i] = gn_pivot(x1, c1, x2, c2, HW, n, cpg, c + i);
  }
}

// fold a thread's 8 per-channel sums into (at most eight) group bins, then one shared atomic per bin
__device__ __forceinline__ void gn_fold_bins(const float (&sm)[8], const float (&sq)[8], int c, int cpg, float* s_sum,
                                             float* s_sq) {
  int g_prev = c / cpg;
  float as = 0.f, aq = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int g = (c + i) / cpg;
    if (g != g_prev) {
      atomicAdd(&s_sum[g_prev], as);
      atomicAdd(&s_sq[g_prev], aq);
      as = aq = 0.f;
      g_prev = g;
    }
    as += sm[i];
    aq += sq[i];
  }
  atomicAdd(&s_sum[g_prev], as);
  atomicAdd(&s_sq[g_prev], aq);
}

// at least 3 CTAs per SM: keeps this HBM-bound pass at 64 registers (the pivots and the wide-row branch add pressure)
__global__ void __launch_bounds__(320, 3)
gn_stats_kernel(const __half* __restrict__ x1, int c1, const __half* __restrict__ x2, int c2,
                long long HW, int groups, long long pix_per_cta, double* __restrict__ ws) {
  pdl_enter();
  const int C = c1 + c2;
  const int cpg = C / groups;
  const int vecs = C / 8;
  const int n = blockIdx.y;
  const long long p0 = (long long)blockIdx.x * pix_per_cta;
  long long p1 = p0 + pix_per_cta;
  if (p1 > HW) p1 = HW;
  __shared__ float s_sum[GN_MAX_GROUPS];
  __shared__ float s_sq[GN_MAX_GROUPS];
  if (threadIdx.x < GN_MAX_GROUPS) {
    s_sum[threadIdx.x] = 0.f;
    s_sq[threadIdx.x] = 0.f;
  }
  __syncthreads();
  const int lanes = blockDim.x / vecs;      // pixel lanes per CTA (blockDim % vecs == 0, or vecs > blockDim)
  if (lanes >= 1) {
    const int v = threadIdx.x % vecs;
    const int c = v * 8;
    float sm[8], sq[8], kp[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) sm[i] = sq[i] = 0.f;
    gn_pivots(x1, c1, x2, c2, HW, n, cpg, c, kp);
    long long pix = p0 + threadIdx.x / vecs;
    for (; pix + 3 * lanes < p1; pix += 4 * lanes) {
      uint4 u[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) u[k] = gn_load(x1, c1, x2, c2, (long long)n * HW + pix + k * lanes, c);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float f[8];
        unpack8(u[k], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = f[i] - kp[i];
          sm[i] += d;
          sq[i] += d * d;
        }
      }
    }
    for (; pix < p1; pix += lanes) {
      float f[8];
      unpack8(gn_load(x1, c1, x2, c2, (long long)n * HW + pix, c), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d = f[i] - kp[i];
        sm[i] += d;
        sq[i] += d * d;
      }
    }
    gn_fold_bins(sm, sq, c, cpg, s_sum, s_sq);
  } else {
    // very wide rows (vecs > blockDim): a thread owns vectors v, v + blockDim, ... and walks the chunk for each, so
    // its sums stay per-thread in registers as on the narrow path (not one shared fp32 sum of the whole chunk)
    for (int v = threadIdx.x; v < vecs; v += blockDim.x) {
      const int c = v * 8;
      float sm[8], sq[8], kp[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) sm[i] = sq[i] = 0.f;
      gn_pivots(x1, c1, x2, c2, HW, n, cpg, c, kp);
      for (long long pix = p0; pix < p1; ++pix) {
        float f[8];
        unpack8(gn_load(x1, c1, x2, c2, (long long)n * HW + pix, c), f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = f[i] - kp[i];
          sm[i] += d;
          sq[i] += d * d;
        }
      }
      gn_fold_bins(sm, sq, c, cpg, s_sum, s_sq);
    }
  }
  __syncthreads();
  if (threadIdx.x < groups) {
    atomicAdd(&ws[((long long)n * groups + threadIdx.x) * 2 + 0], (double)s_sum[threadIdx.x]);
    atomicAdd(&ws[((long long)n * groups + threadIdx.x) * 2 + 1], (double)s_sq[threadIdx.x]);
  }
}

// Deterministic statistics (deterministic mode).  Same per-thread accumulation as gn_stats_kernel; then
//   1. every thread stores its 8 per-channel fp32 sums in shared memory, red[lane][channel];
//   2. warp w folds group g (g = w, w + warps, ...): lane l adds items l, l + 32, ... of the group's (lane, channel)
//      list in fp64, then a fixed xor butterfly -> one fp64 (sum, sumsq) partial per (image, group, chunk) in part;
//   3. the last CTA of an image to arrive (integer counter) adds that image's partials in chunk order the same way and
//      writes the final (sum, sumsq) to ws; it resets the counter for the next call.
// The chunk size comes from (HW, C) alone (see pfd_groupnorm_f16), so no order depends on NB or on the SM count.
constexpr int GN_DET_MAX_CHUNKS = 128;     // per image; ppc >= HW / 128
constexpr int GN_DET_MAX_NB = 64;

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(320)
gn_stats_det_kernel(const __half* __restrict__ x1, int c1, const __half* __restrict__ x2, int c2, long long HW,
                    int groups, long long pix_per_cta, double2* __restrict__ part, int* __restrict__ arrivals,
                    double* __restrict__ ws) {
  pdl_enter();
  extern __shared__ float red[];            // [2][lanes][C]: sums, then sums of squares
  __shared__ int s_last;
  const int C = c1 + c2;
  const int cpg = C / groups;
  const int vecs = C / 8;
  const int n = blockIdx.y;
  const int chunks = gridDim.x;
  const long long p0 = (long long)blockIdx.x * pix_per_cta;
  long long p1 = p0 + pix_per_cta;
  if (p1 > HW) p1 = HW;
  const int lanes = blockDim.x / vecs;
  const int nl = lanes >= 1 ? lanes : 1;
  float* red_s = red;
  float* red_q = red + (long long)nl * C;
  const long long base = (long long)n * HW;
  if (lanes >= 1) {
    if (threadIdx.x < lanes * vecs) {
      const int v = threadIdx.x % vecs, lane = threadIdx.x / vecs;
      const int c = v * 8;
      float sm[8], sq[8], kp[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) sm[i] = sq[i] = 0.f;
      gn_pivots(x1, c1, x2, c2, HW, n, cpg, c, kp);
      long long pix = p0 + lane;
      for (; pix + 3 * lanes < p1; pix += 4 * lanes) {
        uint4 u[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) u[k] = gn_load(x1, c1, x2, c2, base + pix + k * lanes, c);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float f[8];
          unpack8(u[k], f);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float d = f[i] - kp[i];
            sm[i] += d;
            sq[i] += d * d;
          }
        }
      }
      for (; pix < p1; pix += lanes) {
        float f[8];
        unpack8(gn_load(x1, c1, x2, c2, base + pix, c), f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = f[i] - kp[i];
          sm[i] += d;
          sq[i] += d * d;
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        red_s[lane * C + c + i] = sm[i];
        red_q[lane * C + c + i] = sq[i];
      }
    }
  } else {
    // very wide rows (vecs > blockDim): a thread owns vectors v, v + blockDim, ... and walks the chunk for each
    for (int v = threadIdx.x; v < vecs; v += blockDim.x) {
      const int c = v * 8;
      float sm[8], sq[8], kp[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) sm[i] = sq[i] = 0.f;
      gn_pivots(x1, c1, x2, c2, HW, n, cpg, c, kp);
      for (long long pix = p0; pix < p1; ++pix) {
        float f[8];
        unpack8(gn_load(x1, c1, x2, c2, base + pix, c), f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = f[i] - kp[i];
          sm[i] += d;
          sq[i] += d * d;
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        red_s[c + i] = sm[i];
        red_q[c + i] = sq[i];
      }
    }
  }
  __syncthreads();
  // only whole warps fold (blockDim is a multiple of vecs, not always of 32): the shuffles need all 32 lanes
  const int warp = threadIdx.x >> 5, lid = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int items = nl * cpg;                // item j = (lane j / cpg, channel g * cpg + j % cpg)
  for (int g = warp; warp < nwarps && g < groups; g += nwarps) {
    double s = 0.0, q = 0.0;
    for (int j = lid; j < items; j += 32) {
      const int idx = (j / cpg) * C + g * cpg + j % cpg;
      s += (double)red_s[idx];
      q += (double)red_q[idx];
    }
    s = warp_sum_d(s);
    q = warp_sum_d(q);
    if (lid == 0) {
      part[((long long)n * groups + g) * chunks + blockIdx.x] = make_double2(s, q);
      __threadfence();                       // the partial is visible device-wide before this CTA is counted in
    }
  }
  // count this CTA in; the last arrival of image n reduces the image's partials
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(&arrivals[n], 1) == chunks - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int g = warp; warp < nwarps && g < groups; g += nwarps) {
    const double2* pg = part + ((long long)n * groups + g) * chunks;
    double s = 0.0, q = 0.0;
    for (int j = lid; j < chunks; j += 32) {
      const double2 t = __ldcg(pg + j);
      s += t.x;
      q += t.y;
    }
    s = warp_sum_d(s);
    q = warp_sum_d(q);
    if (lid == 0) {
      ws[((long long)n * groups + g) * 2 + 0] = s;
      ws[((long long)n * groups + g) * 2 + 1] = q;
    }
  }
  if (threadIdx.x == 0) arrivals[n] = 0;
}

__global__ void __launch_bounds__(320)
gn_apply_kernel(const __half* __restrict__ x1, int c1, const __half* __restrict__ x2, int c2,
                long long HW, int groups, const __half* __restrict__ gamma,
                const __half* __restrict__ beta, float eps, int silu,
                const double* __restrict__ ws, __half* __restrict__ out, long long pix_per_cta,
                double inv_cnt) {
  pdl_enter();
  const int C = c1 + c2;
  const int cpg = C / groups;
  const int vecs = C / 8;
  const int n = blockIdx.y;
  const long long p0 = (long long)blockIdx.x * pix_per_cta;
  long long p1 = p0 + pix_per_cta;
  if (p1 > HW) p1 = HW;
  const int lanes = blockDim.x / vecs;
  const int vstep = lanes >= 1 ? vecs : blockDim.x;
  const int pstep = lanes >= 1 ? lanes : 1;
  for (int v = threadIdx.x % vstep; v < vecs; v += vstep) {
    const int c = v * 8;
    float a8[8], b8[8];
    {
      float g8[8], be8[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + c)), g8);
      unpack8(__ldg(reinterpret_cast<const uint4*>(beta + c)), be8);
      int gprev = -1;
      float mean = 0.f, rstd = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int g = (c + i) / cpg;
        if (g != gprev) {
          // ws holds the sums of d = x - K_g: mean = K_g + E[d], var = E[d^2] - E[d]^2 (fp64, no DP division)
          const double s_sum = ws[((long long)n * groups + g) * 2 + 0];
          const double s_sq = ws[((long long)n * groups + g) * 2 + 1];
          const double m = s_sum * inv_cnt;
          double var = s_sq * inv_cnt - m * m;
          if (var < 0) var = 0;
          mean = (float)((double)gn_pivot(x1, c1, x2, c2, HW, n, cpg, c + i) + m);
          rstd = rsqrtf((float)var + eps);
          gprev = g;
        }
        a8[i] = rstd * g8[i];
        b8[i] = be8[i] - mean * a8[i];
      }
    }
    auto emit = [&](long long pixn, const uint4& u) {
      float f[8];
      unpack8(u, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float y = fmaf(f[i], a8[i], b8[i]);
        if (silu) {
          y = rh(y);  // reference materialises the GroupNorm output in fp16 before SiLU
          y = __fdividef(y, 1.f + __expf(-y));
        }
        f[i] = y;
      }
      *reinterpret_cast<uint4*>(out + pixn * C + c) = pack8(f);
    };
    long long pix = p0 + (lanes >= 1 ? threadIdx.x / vecs : 0);
    const long long base = (long long)n * HW;
    for (; pix + 3 * pstep < p1; pix += 4 * pstep) {
      uint4 u[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) u[k] = gn_load(x1, c1, x2, c2, base + pix + k * pstep, c);
#pragma unroll
      for (int k = 0; k < 4; ++k) emit(base + pix + k * pstep, u[k]);
    }
    for (; pix < p1; pix += pstep) emit(base + pix, gn_load(x1, c1, x2, c2, base + pix, c));
  }
}

// ------------------------------------------------------------------------------------ LayerNorm
// one warp per row; C % 8 == 0; row cached in registers (C <= 8*32*MAXV).
template <int MAXV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const __half* __restrict__ x, const __half* __restrict__ res, long long rows, int C,
                 const __half* __restrict__ gamma, const __half* __restrict__ beta, float eps,
                 __half* __restrict__ out) {
  pdl_enter();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + warp;
  if (row >= rows) return;
  const int vecs = C / 8;
  float f[MAXV][8];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int v = lane + k * 32;
    if (v < vecs) {
      unpack8(__ldg(reinterpret_cast<const uint4*>(x + row * C + v * 8)), f[k]);
      if (res) {
        float r8[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(res + row * C + v * 8)), r8);
#pragma unroll
        for (int i = 0; i < 8; ++i) f[k][i] = rh(f[k][i] + r8[i]);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) s += f[k][i];
    }
  }
  s = warp_sum(s);
  const float mean = s / C;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int v = lane + k * 32;
    if (v < vecs) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d = f[k][i] - mean;
        q += d * d;
      }
    }
  }
  q = warp_sum(q);
  const float rstd = rsqrtf(q / C + eps);
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int v = lane + k * 32;
    if (v < vecs) {
      float g8[8], b8[8], o[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + v * 8)), g8);
      unpack8(__ldg(reinterpret_cast<const uint4*>(beta + v * 8)), b8);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = (f[k][i] - mean) * rstd * g8[i] + b8[i];
      *reinterpret_cast<uint4*>(out + row * C + v * 8) = pack8(o);
    }
  }
}

// ------------------------------------------------------------------------------------ softmax
// one warp per row (cols <= 32*MAXE) or one CTA per row for long rows.
__global__ void __launch_bounds__(256)
softmax_rows_kernel(__half* __restrict__ s, long long batch, int rows, int cols, long long ld,
                    float scale, const __half* __restrict__ bias, int nheads,
                    const __half* __restrict__ mask, int nwin) {
  pdl_enter();
  // CTA per row, threads stride over columns; values cached in shared memory as fp32.
  extern __shared__ float sv[];
  const long long r = blockIdx.x;  // global row = b*rows + i
  const long long b = r / rows;
  const int i = (int)(r % rows);
  __half* row = s + r * ld;
  const __half* brow = bias ? bias + ((long long)(b % nheads) * rows + i) * cols : nullptr;
  const __half* mrow = mask ? mask + ((long long)((b / nheads) % nwin) * rows + i) * cols : nullptr;
  __shared__ float red[32];
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) {
    float v = __half2float(row[c]);
    v = rh(v * scale);  // reference: fp16 score * scale stays an fp16 tensor
    if (brow) v = rh(v + __half2float(brow[c]));
    if (mrow) v = rh(v + __half2float(mrow[c]));
    sv[c] = v;
    mx = fmaxf(mx, v);
  }
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : -INFINITY;
    t = warp_max(t);
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  mx = red[0];
  __syncthreads();
  float sum = 0.f;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) {
    const float e = __expf(sv[c] - mx);
    sv[c] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  const float inv = 1.f / red[0];
  for (int c = threadIdx.x; c < cols; c += blockDim.x) row[c] = __float2half_rn(sv[c] * inv);
}

// ------------------------------------------------------------------------------------ misc
// T = long long (integer DDIM timesteps) or float (fractional k-sampler timesteps); (float)t is exact for t <= 2^24,
// so both agree bit for bit at integer t
template <typename T>
__global__ void timestep_embedding_kernel(const T* __restrict__ t, int n, int dim,
                                          float max_period, __half* __restrict__ out) {
  pdl_enter();
  const int half_d = dim / 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * half_d) return;
  const int b = idx / half_d, i = idx % half_d;
  // diffusion_utils.py:141-146: freqs = exp(-ln(max_period) * i / half) in fp32
  const float freq = expf(-logf(max_period) * (float)i / (float)half_d);
  const float arg = (float)t[b] * freq;
  out[(long long)b * dim + i] = __float2half_rn(cosf(arg));
  out[(long long)b * dim + half_d + i] = __float2half_rn(sinf(arg));
  if ((dim & 1) && i == 0) out[(long long)b * dim + dim - 1] = __float2half_rn(0.f);
}

__global__ void upsample2x_kernel(const uint4* __restrict__ x, int NB, int H, int W, int vecs,
                                  uint4* __restrict__ out) {
  pdl_enter();
  const long long total = (long long)NB * (2 * H) * (2 * W) * vecs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vecs);
    long long p = i / vecs;
    const int ox = (int)(p % (2 * W));
    p /= (2 * W);
    const int oy = (int)(p % (2 * H));
    const int n = (int)(p / (2 * H));
    out[i] = __ldg(&x[(((long long)n * H + (oy >> 1)) * W + (ox >> 1)) * vecs + v]);
  }
}

template <typename T>
__global__ void nchw_to_nhwc_kernel(const T* __restrict__ x, int NB, int C, int H, int W, int Cpad,
                                    float mul, float add, __half* __restrict__ out) {
  pdl_enter();
  const long long total = (long long)NB * H * W * Cpad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cpad);
    long long p = i / Cpad;
    const int xw = (int)(p % W);
    p /= W;
    const int y = (int)(p % H);
    const int n = (int)(p / H);
    float v = 0.f;
    if (c < C) v = fmaf((float)x[(((long long)n * C + c) * H + y) * W + xw], mul, add);
    out[i] = __float2half_rn(v);
  }
}

__global__ void nhwc_to_nchw_kernel(const __half* __restrict__ x, int NB, int C, int H, int W,
                                    int Cpad, float mul, float add, float lo, float hi,
                                    __half* __restrict__ out) {
  pdl_enter();
  const long long total = (long long)NB * C * H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int xw = (int)(i % W);
    long long p = i / W;
    const int y = (int)(p % H);
    p /= H;
    const int c = (int)(p % C);
    const int n = (int)(p / C);
    float v = __half2float(x[(((long long)n * H + y) * W + xw) * Cpad + c]);
    v = rh(v * mul + add);
    v = fminf(fmaxf(v, lo), hi);
    out[i] = __float2half_rn(v);
  }
}

__global__ void im2col3x3_kernel(const __half* __restrict__ x, int NB, int H, int W, int C,
                                 int stride, int Ho, int Wo, int Kpad, __half* __restrict__ out) {
  pdl_enter();
  const long long total = (long long)NB * Ho * Wo * Kpad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % Kpad);
    long long p = i / Kpad;
    const int ox = (int)(p % Wo);
    p /= Wo;
    const int oy = (int)(p % Ho);
    const int n = (int)(p / Ho);
    __half v = __float2half_rn(0.f);
    if (k < 9 * C) {
      const int tap = k / C, c = k % C;
      const int iy = oy * stride + tap / 3 - 1;
      const int ix = ox * stride + tap % 3 - 1;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = x[(((long long)n * H + iy) * W + ix) * C + c];
    }
    out[i] = v;
  }
}

__global__ void axpby_kernel(const __half* __restrict__ a, float sa, const __half* __restrict__ b,
                             float sb, long long n, __half* __restrict__ out) {
  pdl_enter();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float v = __half2float(a[i]) * sa;
    if (b) v += __half2float(b[i]) * sb;
    out[i] = __float2half_rn(v);
  }
}

__global__ void add_rowvec_kernel(const uint4* __restrict__ a, const uint4* __restrict__ row,
                                  long long rows, int vecs, uint4* __restrict__ out) {
  pdl_enter();
  const long long total = rows * vecs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    float f[8], r[8];
    unpack8(__ldg(&a[i]), f);
    unpack8(__ldg(&row[i % vecs]), r);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] += r[k];
    out[i] = pack8(f);
  }
}

// DiagonalGaussianDistribution of the VAE encoder (distributions.py:24-37, autokl.py:33-42): moments are the
// channel-last [B, H, W, 2*zc] quant_conv output (mean | logvar); logvar is clamped to [-30, 20], std = exp(0.5 *
// logvar); sample = scale * (mean + std * noise).  Outputs are NCHW [B, zc, H, W]; any output may be NULL.
__global__ void vae_posterior_kernel(const __half* __restrict__ mom, int B, int zc, int H, int W, int cpad,
                                     const float* __restrict__ noise, float scale, __half* __restrict__ mean,
                                     __half* __restrict__ logvar, __half* __restrict__ stdv,
                                     __half* __restrict__ sample) {
  pdl_enter();
  const long long total = (long long)B * zc * H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int xw = (int)(i % W);
    long long p = i / W;
    const int y = (int)(p % H);
    p /= H;
    const int c = (int)(p % zc);
    const int n = (int)(p / zc);
    const __half* m = mom + (((long long)n * H + y) * W + xw) * cpad;
    const float mu = __half2float(m[c]);
    const float lv = fminf(fmaxf(__half2float(m[zc + c]), -30.f), 20.f);
    const float sd = rh(__expf(0.5f * lv));
    if (mean) mean[i] = __float2half_rn(mu);
    if (logvar) logvar[i] = __float2half_rn(lv);
    if (stdv) stdv[i] = __float2half_rn(sd);
    if (sample) sample[i] = __float2half_rn(scale * fmaf(sd, noise ? noise[i] : 0.f, mu));
  }
}

// Start of one DDIM step inside a replayed CUDA graph: the device-side step counter walks the schedule backwards
// (ddim.py:108-112: index = total - i - 1) and the timestep of that index is broadcast to the UNet's t input
// (ddim.py:113 torch.full((bs,), step)), so a graph holding any number of steps needs no host work between steps.
// The counter stops at 0, so a header run once too often leaves the next ddim_step on schedule index 0, not on -1.
__global__ void ddim_begin_step_kernel(int* __restrict__ step, const long long* __restrict__ ttab,
                                       long long* __restrict__ t_out, int nb) {
  pdl_enter();
  const int idx = max(*step - 1, 0);
  __syncthreads();
  for (int i = threadIdx.x; i < nb; i += blockDim.x) t_out[i] = ttab[idx];
  if (threadIdx.x == 0) *step = idx;
}

// CFG combine + DDIM update with the reference's fp16 rounding sequence (ddim.py:150-171).
// noise (optional, eta > 0): x_prev = a_prev.sqrt()*pred_x0 + dir_xt + sigma_t*noise*temperature, every product /
// sum rounded to fp16 in the reference's evaluation order (ddim.py:166-170).  guidance and temperature are python
// floats there: torch multiplies an fp16 tensor by a python scalar held in fp32, so neither is rounded to fp16.
// log_tab (optional): slot per schedule index (-1 = not logged) of the `intermediates` lists (ddim.py:122-124);
// the step's x_prev / pred_x0 are also written to log_xt / log_x0 [slot] so multi-step graphs need no host copy.
__global__ void ddim_step_kernel(const __half* __restrict__ eps, const __half* __restrict__ x,
                                 long long half_n, float guidance, const float* __restrict__ coef,
                                 const int* __restrict__ step, __half* __restrict__ x_prev,
                                 __half* __restrict__ pred_x0, const __half* __restrict__ noise,
                                 float temperature, const int* __restrict__ log_tab,
                                 __half* __restrict__ log_xt, __half* __restrict__ log_x0) {
  pdl_enter();
  const int st = step ? *step : 0;
  // torch.full(..., dtype=fp16) rounds each coefficient to fp16 first (ddim.py:160-163)
  const float a_t = rh(coef[st * 4 + 0]);
  const float a_prev = rh(coef[st * 4 + 1]);
  const float sigma = rh(coef[st * 4 + 2]);
  const float s1m = rh(coef[st * 4 + 3]);
  const float sqrt_at = rh(sqrtf(a_t));
  const float sqrt_ap = rh(sqrtf(a_prev));
  const float dir_c = rh(sqrtf(rh(rh(1.f - a_prev) - rh(sigma * sigma))));
  const float temp = temperature;
  const int slot = log_tab ? log_tab[st] : -1;
  __half* lxt = slot >= 0 ? log_xt + (long long)slot * half_n : nullptr;
  __half* lx0 = slot >= 0 ? log_x0 + (long long)slot * half_n : nullptr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < half_n;
       i += (long long)gridDim.x * blockDim.x) {
    const float eu = __half2float(eps[i]);
    const float ec = __half2float(eps[half_n + i]);
    // e_t = e_u + s * (e_c - e_u), each op rounded to fp16 like the eager reference
    const float e = rh(eu + rh(guidance * rh(ec - eu)));
    const float xv = __half2float(x[i]);
    const float p0 = rh(rh(xv - rh(s1m * e)) / sqrt_at);
    const float dir = rh(dir_c * e);
    float xp = rh(rh(sqrt_ap * p0) + dir);
    if (noise) xp = rh(xp + rh(rh(sigma * __half2float(noise[i])) * temp));
    const __half xh = __float2half_rn(xp), p0h = __float2half_rn(p0);
    x_prev[i] = xh;
    if (pred_x0) pred_x0[i] = p0h;
    if (lxt) {
      lxt[i] = xh;
      lx0[i] = p0h;
    }
  }
}

// Swin: pad to multiples of ws, cyclic shift by -shift, partition into windows (swin.py:269-287).
// out[(b*nWh + wy)*nWw + wx][iy*ws+ix][c] = xpad[b, (wy*ws+iy+shift)%Hp, (wx*ws+ix+shift)%Wp, c]
__global__ void window_gather_kernel(const uint4* __restrict__ x, int B, int H, int W, int vecs,
                                     int ws, int shift, int Hp, int Wp, uint4* __restrict__ out) {
  pdl_enter();
  const long long total = (long long)B * Hp * Wp * vecs;
  const int nWw = Wp / ws, nWh = Hp / ws;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vecs);
    long long p = i / vecs;
    const int t = (int)(p % (ws * ws));
    p /= (ws * ws);
    const int wx = (int)(p % nWw);
    p /= nWw;
    const int wy = (int)(p % nWh);
    const int b = (int)(p / nWh);
    const int sy = (wy * ws + t / ws + shift) % Hp;
    const int sx = (wx * ws + t % ws + shift) % Wp;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (sy < H && sx < W) u = __ldg(&x[(((long long)b * H + sy) * W + sx) * vecs + v]);
    out[i] = u;
  }
}
// inverse: out[b,y,x,:] = residual[b,y,x,:] + win[window(y,x)]   (swin.py:289-304,307)
__global__ void window_scatter_kernel(const uint4* __restrict__ win, int B, int H, int W, int vecs,
                                      int ws, int shift, int Hp, int Wp,
                                      const uint4* __restrict__ residual, uint4* __restrict__ out) {
  pdl_enter();
  const long long total = (long long)B * H * W * vecs;
  const int nWw = Wp / ws, nWh = Hp / ws;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vecs);
    long long p = i / vecs;
    const int xw = (int)(p % W);
    p /= W;
    const int y = (int)(p % H);
    const int b = (int)(p / H);
    // x[y] = shifted[(y - shift) mod Hp]
    const int sy = (y - shift + Hp) % Hp;
    const int sx = (xw - shift + Wp) % Wp;
    const int wy = sy / ws, iy = sy % ws, wx = sx / ws, ix = sx % ws;
    const long long widx = (((long long)b * nWh + wy) * nWw + wx) * (ws * ws) + iy * ws + ix;
    float f[8];
    unpack8(__ldg(&win[widx * vecs + v]), f);
    if (residual) {
      float r[8];
      unpack8(__ldg(&residual[i]), r);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] += r[k];
    }
    out[i] = pack8(f);
  }
}

// PatchMerging gather (swin.py:336-346): pad odd H/W with zeros, concat [x0,x1,x2,x3] =
// [(0,0),(1,0),(0,1),(1,1)] (dy,dx) along channels.
__global__ void patch_merge_kernel(const uint4* __restrict__ x, int B, int H, int W, int vecs,
                                   uint4* __restrict__ out) {
  pdl_enter();
  const int H2 = (H + 1) / 2, W2 = (W + 1) / 2;
  const long long total = (long long)B * H2 * W2 * 4 * vecs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vecs);
    long long p = i / vecs;
    const int qd = (int)(p % 4);
    p /= 4;
    const int ox = (int)(p % W2);
    p /= W2;
    const int oy = (int)(p % H2);
    const int b = (int)(p / H2);
    const int dy = qd & 1, dx = qd >> 1;  // x0:(0,0) x1:(1,0) x2:(0,1) x3:(1,1)
    const int y = 2 * oy + dy, xw = 2 * ox + dx;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (y < H && xw < W) u = __ldg(&x[(((long long)b * H + y) * W + xw) * vecs + v]);
    out[i] = u;
  }
}


// PatchEmbed gather (swin.py:479-489): zero-pad H,W to multiples of P, then
// out[b, py, px, (c*P + dy)*P + dx] = img[b, c, py*P+dy, px*P+dx]  (K order == flattened conv weight)
template <typename T>
__global__ void patchify_kernel(const T* __restrict__ x, int B, int C, int H, int W, int P, int Kpad,
                                __half* __restrict__ out) {
  pdl_enter();
  const int Hp = (H + P - 1) / P, Wp = (W + P - 1) / P;
  const long long total = (long long)B * Hp * Wp * Kpad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % Kpad);
    long long p = i / Kpad;
    const int px = (int)(p % Wp);
    p /= Wp;
    const int py = (int)(p % Hp);
    const int b = (int)(p / Hp);
    float v = 0.f;
    if (k < C * P * P) {
      const int dx = k % P, dy = (k / P) % P, c = k / (P * P);
      const int y = py * P + dy, xx = px * P + dx;
      if (y < H && xx < W) v = (float)x[(((long long)b * C + c) * H + y) * W + xx];
    }
    out[i] = __float2half_rn(v);
  }
}

// Scratch of the deterministic GroupNorm statistics, one per device: GN_DET_MAX_NB arrival counters, then the fp64
// partials [NB][groups][chunks].  Allocated (and the counters zeroed) by the first deterministic call on the device,
// which must not be inside a stream capture - every graph-captured path of the package runs eagerly first.  The
// counters return to zero at the end of every call, and the calls of one device are stream-ordered (like the GEMM's
// split-K workspace), so one buffer serves them all.
constexpr size_t GN_DET_COUNTER_BYTES = 256;
constexpr size_t GN_DET_SCRATCH_BYTES =
    GN_DET_COUNTER_BYTES + sizeof(double) * 2 * GN_DET_MAX_NB * GN_MAX_GROUPS * GN_DET_MAX_CHUNKS;
static_assert(GN_DET_MAX_NB * sizeof(int) <= GN_DET_COUNTER_BYTES, "arrival counters overflow their slot");

static char* gn_det_scratch(cudaStream_t st) {
  constexpr int MAX_DEV = 64;
  static std::mutex mu;
  static char* buf[MAX_DEV] = {nullptr};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MAX_DEV) return nullptr;
  std::lock_guard<std::mutex> lk(mu);
  if (buf[dev]) return buf[dev];
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) {
    (void)cudaGetLastError();
    return nullptr;
  }
  char* p = nullptr;
  if (cudaMalloc(&p, GN_DET_SCRATCH_BYTES) != cudaSuccess) {
    (void)cudaGetLastError();
    return nullptr;
  }
  if (cudaMemset(p, 0, GN_DET_COUNTER_BYTES) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) {
    (void)cudaGetLastError();
    cudaFree(p);
    return nullptr;
  }
  buf[dev] = p;
  return p;
}

}  // namespace pfd

using namespace pfd;

extern "C" PFD_API int pfd_groupnorm_f16(const void* x1, int32_t c1, const void* x2, int32_t c2, int32_t NB,
                                 int64_t HW, int32_t groups, const void* gamma, const void* beta,
                                 float eps, int32_t silu, void* out, float* ws, int32_t zero_ws, void* stream) {
  const int C = c1 + (x2 ? c2 : 0);
  if (!x2) c2 = 0;
  if (groups <= 0 || groups > GN_MAX_GROUPS || C % groups) return set_error("pfd_groupnorm_f16: C=%d groups=%d", C, groups);
  if (c1 % 8 || c2 % 8) return set_error("pfd_groupnorm_f16: channel counts must be multiples of 8 (%d,%d)", c1, c2);
  if (!ws) return set_error("pfd_groupnorm_f16: workspace required");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  double* dws = reinterpret_cast<double*>(ws);
  const int vecs = C / 8;
  // block = largest multiple of vecs that fits 256 threads (or 320 for C = 2560); wide rows fall back to 256
  int threads = vecs <= 320 ? (vecs <= 256 ? (256 / vecs) * vecs : vecs) : 256;
  if (threads < 64) threads = vecs * ((64 + vecs - 1) / vecs);
  const double inv_cnt = 1.0 / ((double)HW * (C / groups));
  const bool det = deterministic();
  const long long min_ppc = 16LL * (threads / vecs > 0 ? threads / vecs : 1);
  long long ppc;
  if (det) {
    // chunk size from (HW, C) only: 16 pixels per pixel-lane, but at most GN_DET_MAX_CHUNKS chunks per image
    ppc = (HW + GN_DET_MAX_CHUNKS - 1) / GN_DET_MAX_CHUNKS;
  } else {
    if (zero_ws) cudaMemsetAsync(dws, 0, sizeof(double) * 2 * NB * groups, st);
    // ~3 CTAs per SM, but at least 16 pixels per pixel-lane so the per-CTA setup is amortised
    const long long c0 = (3LL * plan_sms() + NB - 1) / NB;
    ppc = (HW + c0 - 1) / c0;
  }
  if (ppc < min_ppc) ppc = min_ppc;
  const long long chunks = (HW + ppc - 1) / ppc;
  dim3 grid((unsigned)chunks, (unsigned)NB);
  if (det) {
    const int lanes = threads / vecs > 0 ? threads / vecs : 1;
    const size_t smem = sizeof(float) * 2 * lanes * C;
    if (NB > GN_DET_MAX_NB || smem > 48 * 1024)
      return set_error("pfd_groupnorm_f16: deterministic statistics support NB <= %d and C <= 6144 (NB=%d, C=%d)",
                       GN_DET_MAX_NB, NB, C);
    char* dscr = gn_det_scratch(st);
    if (!dscr) return set_error("pfd_groupnorm_f16: deterministic statistics scratch unavailable (the first "
                                "deterministic call on a device must not be inside a stream capture)");
    launch_k(gn_stats_det_kernel, grid, dim3(threads), smem, st, static_cast<const __half*>(x1), (int)c1,
             static_cast<const __half*>(x2), (int)c2, (long long)HW, (int)groups, (long long)ppc,
             reinterpret_cast<double2*>(dscr + GN_DET_COUNTER_BYTES), reinterpret_cast<int*>(dscr), dws);
    if (int rc = check_launch("gn_stats_det")) return rc;
  } else {
    launch_k(gn_stats_kernel, dim3(grid), dim3(threads), (size_t)(0), st, static_cast<const __half*>(x1), c1, static_cast<const __half*>(x2), c2,
                                              HW, groups, ppc, dws);
    if (int rc = check_launch("gn_stats")) return rc;
  }
  launch_k(gn_apply_kernel, dim3(grid), dim3(threads), (size_t)(0), st, static_cast<const __half*>(x1), (int)c1,
           static_cast<const __half*>(x2), (int)c2, (long long)HW, (int)groups, static_cast<const __half*>(gamma),
           static_cast<const __half*>(beta), eps, (int)silu, (const double*)dws, static_cast<__half*>(out), (long long)ppc,
           inv_cnt);
  return check_launch("gn_apply");
}

extern "C" PFD_API int pfd_layernorm_f16(const void* x, const void* res, int64_t rows, int32_t C,
                                 const void* gamma, const void* beta, float eps, void* out,
                                 void* stream) {
  if (C % 8 || C > 8 * 32 * 16) return set_error("pfd_layernorm_f16: C=%d unsupported", C);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int wpb = 8;
  const unsigned grid = (unsigned)((rows + wpb - 1) / wpb);
  const int vecs = C / 8;
  const __half* xp = static_cast<const __half*>(x);
  const __half* rp = static_cast<const __half*>(res);
  const __half* gp = static_cast<const __half*>(gamma);
  const __half* bp = static_cast<const __half*>(beta);
  __half* op = static_cast<__half*>(out);
  if (vecs <= 32) launch_k(layernorm_kernel<1>, dim3(grid), dim3(256), (size_t)(0), st, xp, rp, rows, C, gp, bp, eps, op);
  else if (vecs <= 64) launch_k(layernorm_kernel<2>, dim3(grid), dim3(256), (size_t)(0), st, xp, rp, rows, C, gp, bp, eps, op);
  else if (vecs <= 128) launch_k(layernorm_kernel<4>, dim3(grid), dim3(256), (size_t)(0), st, xp, rp, rows, C, gp, bp, eps, op);
  else if (vecs <= 256) launch_k(layernorm_kernel<8>, dim3(grid), dim3(256), (size_t)(0), st, xp, rp, rows, C, gp, bp, eps, op);
  else launch_k(layernorm_kernel<16>, dim3(grid), dim3(256), (size_t)(0), st, xp, rp, rows, C, gp, bp, eps, op);
  return check_launch("layernorm");
}

extern "C" PFD_API int pfd_softmax_f16(void* s, int64_t batch, int32_t rows, int32_t cols, int64_t ld,
                               float scale, const void* bias, int32_t nheads, const void* mask,
                               int32_t nwin, void* stream) {
  // the row is cached as fp32 in shared memory: up to 50176 columns (196 KB; 1536x1536 VAE mid attention = 36864)
  if (cols <= 0 || cols > 50176) return set_error("pfd_softmax_f16: cols=%d unsupported", cols);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long nrows = batch * rows;
  if (nheads <= 0) nheads = 1;
  if (nwin <= 0) nwin = 1;
  int threads = cols >= 1024 ? 256 : (cols >= 256 ? 128 : 64);
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(softmax_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 50176 * 4);
    attr = true;
  }
  launch_k(softmax_rows_kernel, dim3((unsigned)nrows), dim3(threads), (size_t)(cols * sizeof(float)), st, 
      static_cast<__half*>(s), batch, rows, cols, ld, scale, static_cast<const __half*>(bias), nheads,
      static_cast<const __half*>(mask), nwin);
  return check_launch("softmax");
}

extern "C" PFD_API int pfd_timestep_embedding_f16(const int64_t* t, int32_t n, int32_t dim, float max_period,
                                          void* out, void* stream) {
  const int total = n * (dim / 2);
  launch_k(timestep_embedding_kernel<long long>, dim3((total + 127) / 128), dim3(128), (size_t)(0), static_cast<cudaStream_t>(stream),
      reinterpret_cast<const long long*>(t), n, dim, max_period, static_cast<__half*>(out));
  return check_launch("timestep_embedding");
}

extern "C" PFD_API int pfd_timestep_embedding_ft_f16(const float* t, int32_t n, int32_t dim, float max_period,
                                                     void* out, void* stream) {
  if (!t || !out || n <= 0 || dim <= 0) return set_error("pfd_timestep_embedding_ft_f16: null/empty argument");
  const int total = n * (dim / 2);
  launch_k(timestep_embedding_kernel<float>, dim3((total + 127) / 128), dim3(128), (size_t)(0),
           static_cast<cudaStream_t>(stream), t, n, dim, max_period, static_cast<__half*>(out));
  return check_launch("timestep_embedding_ft");
}

extern "C" PFD_API int pfd_upsample2x_f16(const void* x, int32_t NB, int32_t H, int32_t W, int32_t C, void* out,
                                  void* stream) {
  if (C % 8) return set_error("pfd_upsample2x_f16: C=%d", C);
  const long long total = (long long)NB * 4 * H * W * (C / 8);
  launch_k(upsample2x_kernel, dim3(grid_cap(total, 256)), dim3(256), (size_t)(0), static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(x), NB, H, W, C / 8, static_cast<uint4*>(out));
  return check_launch("upsample2x");
}

extern "C" PFD_API int pfd_nchw_to_nhwc_f16(const void* x, int32_t src_is_f32, int32_t NB, int32_t C, int32_t H,
                                    int32_t W, int32_t Cpad, float mul, float add, void* out, void* stream) {
  const long long total = (long long)NB * H * W * Cpad;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (src_is_f32)
    launch_k(nchw_to_nhwc_kernel<float>, dim3(grid_cap(total, 256)), dim3(256), (size_t)(0), st, static_cast<const float*>(x), NB, C, H, W, Cpad, mul, add, static_cast<__half*>(out));
  else
    launch_k(nchw_to_nhwc_kernel<__half>, dim3(grid_cap(total, 256)), dim3(256), (size_t)(0), st, static_cast<const __half*>(x), NB, C, H, W, Cpad, mul, add, static_cast<__half*>(out));
  return check_launch("nchw_to_nhwc");
}

extern "C" PFD_API int pfd_nhwc_to_nchw_f16(const void* x, int32_t NB, int32_t C, int32_t H, int32_t W, int32_t Cpad,
                                    float mul, float add, float lo, float hi, void* out, void* stream) {
  const long long total = (long long)NB * C * H * W;
  launch_k(nhwc_to_nchw_kernel, dim3(grid_cap(total, 256)), dim3(256), (size_t)(0), static_cast<cudaStream_t>(stream), 
      static_cast<const __half*>(x), NB, C, H, W, Cpad, mul, add, lo, hi, static_cast<__half*>(out));
  return check_launch("nhwc_to_nchw");
}

extern "C" PFD_API int pfd_im2col3x3_f16(const void* x, int32_t NB, int32_t H, int32_t W, int32_t C, int32_t stride,
                                 int32_t Kpad, void* out, void* stream) {
  if (Kpad < 9 * C || Kpad % 8) return set_error("pfd_im2col3x3_f16: Kpad=%d for C=%d", Kpad, C);
  const int Ho = (H + 2 - 3) / stride + 1, Wo = (W + 2 - 3) / stride + 1;
  const long long total = (long long)NB * Ho * Wo * Kpad;
  launch_k(im2col3x3_kernel, dim3(grid_cap(total, 256)), dim3(256), (size_t)(0), static_cast<cudaStream_t>(stream), 
      static_cast<const __half*>(x), NB, H, W, C, stride, Ho, Wo, Kpad, static_cast<__half*>(out));
  return check_launch("im2col3x3");
}

extern "C" PFD_API int pfd_axpby_f16(const void* a, float sa, const void* b, float sb, int64_t n, void* out,
                             void* stream) {
  launch_k(axpby_kernel, dim3(grid_cap(n, 256)), dim3(256), (size_t)(0), static_cast<cudaStream_t>(stream), 
      static_cast<const __half*>(a), sa, static_cast<const __half*>(b), sb, n, static_cast<__half*>(out));
  return check_launch("axpby");
}

extern "C" PFD_API int pfd_add_rowvec_f16(const void* a, const void* row, int64_t rows, int32_t C, void* out,
                                  void* stream) {
  if (C % 8) return set_error("pfd_add_rowvec_f16: C=%d", C);
  launch_k(add_rowvec_kernel, dim3(grid_cap(rows * (C / 8), 256)), dim3(256), (size_t)(0), static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(a), static_cast<const uint4*>(row), rows, C / 8, static_cast<uint4*>(out));
  return check_launch("add_rowvec");
}

extern "C" PFD_API int pfd_ddim_step_f16(const void* eps, const void* x, int64_t half_n, float guidance,
                                 const float* coef, const int32_t* step, void* x_prev, void* pred_x0,
                                 const void* noise, float temperature, const int32_t* log_tab, void* log_xt,
                                 void* log_x0, void* stream) {
  if (!eps || !x || !x_prev || !coef || half_n <= 0) return set_error("pfd_ddim_step_f16: null/empty argument");
  if (log_tab && (!log_xt || !log_x0)) return set_error("pfd_ddim_step_f16: log_tab without log buffers");
  launch_k(ddim_step_kernel, dim3(grid_cap(half_n, 256)), dim3(256), (size_t)(0), static_cast<cudaStream_t>(stream),
      static_cast<const __half*>(eps), static_cast<const __half*>(x), half_n, guidance, coef, step,
      static_cast<__half*>(x_prev), static_cast<__half*>(pred_x0), static_cast<const __half*>(noise), temperature,
      log_tab, static_cast<__half*>(log_xt), static_cast<__half*>(log_x0));
  return check_launch("ddim_step");
}

extern "C" PFD_API int pfd_vae_posterior_f16(const void* moments, int32_t B, int32_t zc, int32_t H, int32_t W,
                                             int32_t cpad, const float* noise, float scale, void* mean,
                                             void* logvar, void* stdv, void* sample, void* stream) {
  if (!moments || B <= 0 || zc <= 0 || cpad < 2 * zc) return set_error("pfd_vae_posterior_f16: bad arguments");
  const long long total = (long long)B * zc * H * W;
  launch_k(vae_posterior_kernel, dim3(grid_cap(total, 256)), dim3(256), (size_t)(0), static_cast<cudaStream_t>(stream),
      static_cast<const __half*>(moments), (int)B, (int)zc, (int)H, (int)W, (int)cpad, noise, scale,
      static_cast<__half*>(mean), static_cast<__half*>(logvar), static_cast<__half*>(stdv), static_cast<__half*>(sample));
  return check_launch("vae_posterior");
}

extern "C" PFD_API int pfd_ddim_begin_step(int32_t* step, const int64_t* ttab, int64_t* t_out, int32_t nb,
                                           void* stream) {
  if (!step || !ttab || !t_out || nb <= 0) return set_error("pfd_ddim_begin_step: null/empty argument");
  launch_k(ddim_begin_step_kernel, dim3(1), dim3(64), (size_t)(0), static_cast<cudaStream_t>(stream),
      reinterpret_cast<int*>(step), reinterpret_cast<const long long*>(ttab), reinterpret_cast<long long*>(t_out),
      (int)nb);
  return check_launch("ddim_begin_step");
}

extern "C" PFD_API int pfd_window_gather_f16(const void* x, int32_t B, int32_t H, int32_t W, int32_t C, int32_t ws,
                                     int32_t shift, void* out, void* stream) {
  if (C % 8) return set_error("pfd_window_gather_f16: C=%d", C);
  const int Hp = (H + ws - 1) / ws * ws, Wp = (W + ws - 1) / ws * ws;
  const long long total = (long long)B * Hp * Wp * (C / 8);
  launch_k(window_gather_kernel, dim3(grid_cap(total, 256)), dim3(256), (size_t)(0), static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(x), B, H, W, C / 8, ws, shift, Hp, Wp, static_cast<uint4*>(out));
  return check_launch("window_gather");
}

extern "C" PFD_API int pfd_window_scatter_f16(const void* win, int32_t B, int32_t H, int32_t W, int32_t C,
                                      int32_t ws, int32_t shift, const void* residual, void* out,
                                      void* stream) {
  if (C % 8) return set_error("pfd_window_scatter_f16: C=%d", C);
  const int Hp = (H + ws - 1) / ws * ws, Wp = (W + ws - 1) / ws * ws;
  const long long total = (long long)B * H * W * (C / 8);
  launch_k(window_scatter_kernel, dim3(grid_cap(total, 256)), dim3(256), (size_t)(0), static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(win), B, H, W, C / 8, ws, shift, Hp, Wp,
      static_cast<const uint4*>(residual), static_cast<uint4*>(out));
  return check_launch("window_scatter");
}

extern "C" PFD_API int pfd_patch_merge_gather_f16(const void* x, int32_t B, int32_t H, int32_t W, int32_t C,
                                          void* out, void* stream) {
  if (C % 8) return set_error("pfd_patch_merge_gather_f16: C=%d", C);
  const long long total = (long long)B * ((H + 1) / 2) * ((W + 1) / 2) * 4 * (C / 8);
  launch_k(patch_merge_kernel, dim3(grid_cap(total, 256)), dim3(256), (size_t)(0), static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(x), B, H, W, C / 8, static_cast<uint4*>(out));
  return check_launch("patch_merge");
}

extern "C" PFD_API int pfd_patchify_f16(const void* x, int32_t src_is_f32, int32_t B, int32_t C, int32_t H,
                                        int32_t W, int32_t P, int32_t Kpad, void* out, void* stream) {
  if (Kpad < C * P * P || Kpad % 8) return set_error("pfd_patchify_f16: Kpad=%d for C=%d P=%d", Kpad, C, P);
  const long long total = (long long)B * ((H + P - 1) / P) * ((W + P - 1) / P) * Kpad;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (src_is_f32)
    launch_k(patchify_kernel<float>, dim3(grid_cap(total, 256)), dim3(256), (size_t)(0), st, static_cast<const float*>(x), B, C, H, W, P, Kpad, static_cast<__half*>(out));
  else
    launch_k(patchify_kernel<__half>, dim3(grid_cap(total, 256)), dim3(256), (size_t)(0), st, static_cast<const __half*>(x), B, C, H, W, P, Kpad, static_cast<__half*>(out));
  return check_launch("patchify");
}
