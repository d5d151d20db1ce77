// OpenPose body annotator behind ControlNet.preprocess(type='openpose' / 'openpose_v11p') on the GPU.
//
// Replaces controlnet.py:396-406 -> controlnet_annotator/openpose (OpenposeDetector with the body network only:
// Body.__call__, body.py:43-229, and util.draw_bodypose, util.py:70-124).  The VGG/CPM network's 3x3 and 1x1 convs
// run on pfd_gemm_f16 and its 7x7 convs on pfd_im2col7x7_f16 + pfd_gemm_f16.  This file holds the rest:
//   op_input_kernel     ToPILImage quantisation, the BGR flip, cv2.resize of the uint8 image (INTER_AREA or
//                       INTER_LANCZOS4, on OpenCV's own tables and fixed-point rounding, built by openpose_tables.py),
//                       the 128 pad to a multiple of 8 and u8 / 256 - 0.5 (exact in fp16; the pad is exactly 0);
//   op_pool_kernel      2x2 / stride 2 max pool (channel-last fp16);
//   op_im2col7_kernel   7x7 / pad 3 im2col (channel-last fp16, K = 49 * C, k = tap * C + c);
//   op_head_kernel      the stage-6 1x1 heads in fp32 (ReLU on the heatmap head, none on the PAF head: the reference's
//                       no_relu_layers lists Mconv7_stage6_L1 twice and never Mconv7_stage6_L2), planar fp32 output;
//   op_resize_kernel    cv2.resize of float32 maps on the same tables (LANCZOS4 x8 then crop, then to the image size);
//   op_gauss_kernel     scipy.ndimage.gaussian_filter(sigma=3) in float64 ('reflect', radius 12, axis 0 then 1, in
//                       scipy's symmetric-kernel operation order, outermost tap first);
//   op_peak_count / op_peak_emit   4-neighbour peaks > 0.1 in np.nonzero (raster) order, at most PFD_OPENPOSE_MAX_PEAKS
//                       per (image, part); the rest are dropped and counted;
//   op_paf_kernel       one thread per (limb, candidate pair): 10 linspace samples of the PAF (evaluated pointwise
//                       through the final resize), the distance prior and both criteria, in float64;
//   op_assemble_kernel  one CTA per image: the greedy matching of each limb (highest score first, ties in (i, j) order)
//                       and the reference's sequential person assembly and row deletion;
//   op_draw_kernel      one warp per primitive: cv2.ellipse2Poly + fillConvexPoly (shift 0, LINE_8) per limb and the
//                       filled cv2.circle(r=4) per keypoint; the last primitive in drawing order wins each pixel
//                       (atomicMax of the primitive's index), then op_color_kernel writes the canvas / 255.
// Every kernel computes an image's values from that image only, so a batch gives the same bits as single images.  No
// count leaves the device.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/pfd_b200.h"
#include "common.h"

namespace pfd {

constexpr int OP_CAP = PFD_OPENPOSE_MAX_PEAKS;
constexpr int OP_ROWS = PFD_OPENPOSE_MAX_PERSONS;
constexpr int OP_PRIMS = 35;          // per person: 17 limbs, then 18 keypoints
constexpr int OP_CIN = 16;            // network input channels: b, g, r and 13 zero pads (the GEMM's 3x3 path)
constexpr int OP_RADIUS = 12;         // int(4.0 * 3 + 0.5)

__device__ __forceinline__ void pdl_enter_o() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

static inline int grid_cap_o(long long work, int per_block) {
  long long g = (work + per_block - 1) / per_block;
  const long long cap = (long long)num_sms() * 16;
  if (g > cap) g = cap;
  return (int)(g < 1 ? 1 : g);
}

// limbSeq (1-based parts) and mapIdx (PAF channels + 19) of body.py:115-121
__constant__ int8_t c_limb_a[19] = {2, 2, 3, 4, 6, 7, 2, 9, 10, 2, 12, 13, 2, 1, 15, 1, 16, 3, 6};
__constant__ int8_t c_limb_b[19] = {3, 6, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 1, 15, 17, 16, 18, 17, 18};
__constant__ int8_t c_paf_x[19] = {31, 39, 33, 35, 41, 43, 19, 21, 23, 25, 27, 29, 47, 49, 53, 51, 55, 37, 45};

// ------------------------------------------------------------------------------------------------------------------
// separable resize tables: idx int32 [D, T], weights [D, T] (float32, or int32 for the uint8 LANCZOS4 path)
struct OpAxis {
  const int* idx;
  const void* w;
  int taps;
};

// uint8 image sample (ToPILImage quantisation of x's element)
template <typename T>
__device__ __forceinline__ int op_u8(const T* x, long long off) { return (int)to_u8<T>(x[off]); }

// out[n, y, x, 0..15] for the padded network input.  mode 0: copy, 1: integer block mean (fy x fx), 2: LANCZOS4
// (int16 weights, int sums, (v + 2^21) >> 22), 3: INTER_AREA (float weights, sum, cvRound).
template <typename T>
__global__ void __launch_bounds__(256)
op_input_kernel(const T* __restrict__ x, int B, int H, int W, int h, int w, int hp, int wp, int mode, int fy, int fx,
                OpAxis ay, OpAxis ax, __half* __restrict__ out) {
  pdl_enter_o();
  const long long total = (long long)B * hp * wp;
  const long long hw = (long long)H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(i % wp);
    const long long r = i / wp;
    const int Y = (int)(r % hp);
    const long long n = r / hp;
    __align__(16) __half v[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) v[c] = __float2half_rn(0.f);
    if (Y < h && X < w) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const long long base = (n * 3 + (2 - c)) * hw;      // BGR
        int u = 0;
        if (mode == 0) {
          u = op_u8(x, base + (long long)Y * W + X);
        } else if (mode == 1) {
          int s = 0;
          for (int a = 0; a < fy; ++a)
            for (int b = 0; b < fx; ++b) s += op_u8(x, base + (long long)(Y * fy + a) * W + X * fx + b);
          if (fy == 2 && fx == 2) u = (s + 2) >> 2;
          else u = min(max(__float2int_rn(__fmul_rn((float)s, 1.f / (float)(fy * fx))), 0), 255);
        } else if (mode == 2) {
          const int* iy = ay.idx + Y * 8;
          const int* ix = ax.idx + X * 8;
          const int* wy = static_cast<const int*>(ay.w) + Y * 8;
          const int* wx = static_cast<const int*>(ax.w) + X * 8;
          int acc = 0;
          for (int k = 0; k < 8; ++k) {
            int row = 0;
            for (int j = 0; j < 8; ++j) row += op_u8(x, base + (long long)iy[k] * W + ix[j]) * wx[j];
            acc += row * wy[k];
          }
          u = min(max((acc + (1 << 21)) >> 22, 0), 255);
        } else {
          const int* iy = ay.idx + Y * ay.taps;
          const int* ix = ax.idx + X * ax.taps;
          const float* wy = static_cast<const float*>(ay.w) + Y * ay.taps;
          const float* wx = static_cast<const float*>(ax.w) + X * ax.taps;
          float acc = 0.f;
          for (int k = 0; k < ay.taps; ++k) {
            float row = 0.f;
            for (int j = 0; j < ax.taps; ++j)
              row = __fadd_rn(row, __fmul_rn((float)op_u8(x, base + (long long)iy[k] * W + ix[j]), wx[j]));
            acc = __fadd_rn(acc, __fmul_rn(wy[k], row));
          }
          u = min(max(__float2int_rn(acc), 0), 255);
        }
        v[c] = __float2half_rn((float)u * (1.f / 256.f) - 0.5f);
      }
    }
    uint4* o = reinterpret_cast<uint4*>(out + i * OP_CIN);
    o[0] = reinterpret_cast<const uint4*>(v)[0];
    o[1] = reinterpret_cast<const uint4*>(v)[1];
  }
}

__global__ void __launch_bounds__(256)
op_pool_kernel(const __half* __restrict__ x, int B, int H, int W, int C, __half* __restrict__ out) {
  pdl_enter_o();
  const int Ho = H / 2, Wo = W / 2, V = C / 8;
  const long long total = (long long)B * Ho * Wo * V;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % V);
    long long r = i / V;
    const int ox = (int)(r % Wo);
    r /= Wo;
    const int oy = (int)(r % Ho);
    const long long n = r / Ho;
    const __half* p = x + ((n * H + 2 * oy) * W + 2 * ox) * C + v * 8;
    uint4 q[4] = {*reinterpret_cast<const uint4*>(p), *reinterpret_cast<const uint4*>(p + C),
                  *reinterpret_cast<const uint4*>(p + (long long)W * C),
                  *reinterpret_cast<const uint4*>(p + (long long)W * C + C)};
    __half2* m = reinterpret_cast<__half2*>(&q[0]);
#pragma unroll
    for (int t = 1; t < 4; ++t) {
      const __half2* o = reinterpret_cast<const __half2*>(&q[t]);
#pragma unroll
      for (int j = 0; j < 4; ++j) m[j] = __hmax2(m[j], o[j]);
    }
    *reinterpret_cast<uint4*>(out + ((n * Ho + oy) * Wo + ox) * C + v * 8) = q[0];
  }
}

// out[(n*H + y)*W + x][tap * C + c] = x[n, y + tap/7 - 3, x + tap%7 - 3, c] (0 outside); one thread per 8 channels
__global__ void __launch_bounds__(256)
op_im2col7_kernel(const __half* __restrict__ x, int B, int H, int W, int C, __half* __restrict__ out) {
  pdl_enter_o();
  const int V = C / 8;
  const long long total = (long long)B * H * W * 49 * V;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % V);
    long long r = i / V;
    const int tap = (int)(r % 49);
    r /= 49;
    const int ox = (int)(r % W);
    r /= W;
    const int oy = (int)(r % H);
    const long long n = r / H;
    const int iy = oy + tap / 7 - 3, ix = ox + tap % 7 - 3;
    uint4 q = make_uint4(0, 0, 0, 0);
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) q = *reinterpret_cast<const uint4*>(x + ((n * H + iy) * W + ix) * C + v * 8);
    *reinterpret_cast<uint4*>(out + i * 8) = q;
  }
}

// out[n, o + k, y, x] = act(b[k] + sum_c w[k][c] * x[n, y, x, c]) in fp32, one thread per (pixel, k)
__global__ void __launch_bounds__(256)
op_head_kernel(const __half* __restrict__ x, int B, int h, int w, int C, const float* __restrict__ wt,
               const float* __restrict__ bias, int N, int relu, float* __restrict__ out, int out_c, int out_off) {
  pdl_enter_o();
  const long long hw = (long long)h * w, total = (long long)B * hw * N;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i % (B * hw);
    const int k = (int)(i / (B * hw));
    const __half* src = x + p * C;
    const float* wk = wt + (long long)k * C;
    float acc = bias[k];
    for (int c0 = 0; c0 < C; c0 += 8) {
      const uint4 q = *reinterpret_cast<const uint4*>(src + c0);
      const __half* hv = reinterpret_cast<const __half*>(&q);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc = fmaf(wk[c0 + j], __half2float(hv[j]), acc);
    }
    if (relu) acc = fmaxf(acc, 0.f);
    const long long n = p / hw, q = p % hw;
    out[(n * out_c + out_off + k) * hw + q] = acc;
  }
}

// value of the resized float map at (Y, X): mode 0 copy, 1 block mean (fy x fx), 2 separable table
__device__ __forceinline__ float op_resample(const float* __restrict__ s, int ws, int mode, int fy, int fx,
                                             const OpAxis ay, const OpAxis ax, int Y, int X) {
  if (mode == 0) return s[(long long)Y * ws + X];
  if (mode == 1) {
    float acc = 0.f;
    for (int a = 0; a < fy; ++a)
      for (int b = 0; b < fx; ++b) acc = __fadd_rn(acc, s[(long long)(Y * fy + a) * ws + X * fx + b]);
    return __fmul_rn(acc, 1.f / (float)(fy * fx));
  }
  const int* iy = ay.idx + Y * ay.taps;
  const int* ix = ax.idx + X * ax.taps;
  const float* wy = static_cast<const float*>(ay.w) + Y * ay.taps;
  const float* wx = static_cast<const float*>(ax.w) + X * ax.taps;
  float acc = 0.f;
  for (int k = 0; k < ay.taps; ++k) {
    const float* row = s + (long long)iy[k] * ws;
    float r = 0.f;
    for (int j = 0; j < ax.taps; ++j) r = __fadd_rn(r, __fmul_rn(row[ix[j]], wx[j]));
    acc = __fadd_rn(acc, __fmul_rn(wy[k], r));
  }
  return acc;
}

// out[n, c, Y, X] (Y < H, X < W) = resample of src[n, c0 + c] (planar, src_c channels of hs x ws)
__global__ void __launch_bounds__(256)
op_resize_kernel(const float* __restrict__ src, int B, int src_c, int c0, int C, int hs, int ws, int H, int W, int mode,
                 int fy, int fx, OpAxis ay, OpAxis ax, float* __restrict__ out) {
  pdl_enter_o();
  const long long HW = (long long)H * W, total = (long long)B * C * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(i % W);
    const int Y = (int)((i / W) % H);
    const long long nc = i / HW;
    const int c = (int)(nc % C);
    const long long n = nc / C;
    out[i] = op_resample(src + (n * src_c + c0 + c) * (long long)hs * ws, ws, mode, fy, fx, ay, ax, Y, X);
  }
}

__device__ __forceinline__ int op_reflect(int i, int n) {
  const int p = 2 * n;
  i %= p;
  if (i < 0) i += p;
  return i < n ? i : p - 1 - i;
}

// one 1-D pass of the Gaussian along y (axis 0) or x (axis 1), scipy's symmetric correlate1d (NI_Correlate1D):
// t = s[0] * g[0]; t += (s[-l] + s[l]) * g[l], outermost tap first (l = 12..1)
template <typename TI>
__global__ void __launch_bounds__(256)
op_gauss_kernel(const TI* __restrict__ in, long long planes, int H, int W, int axis, const double* __restrict__ g,
                double* __restrict__ out) {
  pdl_enter_o();
  const long long HW = (long long)H * W, total = planes * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(i % W);
    const int Y = (int)((i / W) % H);
    const TI* p = in + (i / HW) * HW;
    double t;
    if (axis == 0) {
      t = __dmul_rn((double)p[(long long)Y * W + X], g[0]);
      for (int l = OP_RADIUS; l >= 1; --l)
        t = __dadd_rn(t, __dmul_rn(__dadd_rn((double)p[(long long)op_reflect(Y + l, H) * W + X],
                                             (double)p[(long long)op_reflect(Y - l, H) * W + X]), g[l]));
    } else {
      const TI* row = p + (long long)Y * W;
      t = __dmul_rn((double)row[X], g[0]);
      for (int l = OP_RADIUS; l >= 1; --l)
        t = __dadd_rn(t, __dmul_rn(__dadd_rn((double)row[op_reflect(X + l, W)], (double)row[op_reflect(X - l, W)]), g[l]));
    }
    out[i] = t;
  }
}

__device__ __forceinline__ bool op_is_peak(const double* __restrict__ m, int H, int W, int y, int x) {
  const double v = m[(long long)y * W + x];
  const double l = y > 0 ? m[(long long)(y - 1) * W + x] : 0.0;
  const double r = y < H - 1 ? m[(long long)(y + 1) * W + x] : 0.0;
  const double u = x > 0 ? m[(long long)y * W + x - 1] : 0.0;
  const double d = x < W - 1 ? m[(long long)y * W + x + 1] : 0.0;
  return v >= l && v >= r && v >= u && v >= d && v > 0.1;
}

// one warp per (image, part, row): rowcnt[plane * H + y] = number of peaks in the row
__global__ void __launch_bounds__(256)
op_peak_count_kernel(const double* __restrict__ blur, long long planes, int H, int W, int* __restrict__ rowcnt) {
  pdl_enter_o();
  const long long row = (long long)blockIdx.x * 8 + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (row >= planes * H) return;
  const double* m = blur + (row / H) * (long long)H * W;
  const int y = (int)(row % H);
  int cnt = 0;
  for (int x0 = 0; x0 < W; x0 += 32) {
    const int x = x0 + lane;
    cnt += __popc(__ballot_sync(0xffffffffu, x < W && op_is_peak(m, H, W, y, x)));
  }
  if (lane == 0) rowcnt[row] = cnt;
}

// one warp per row: the row's peaks at their raster rank (ranks >= OP_CAP dropped).  xy int32 [planes, CAP, 2],
// score float64 [planes, CAP] (the unblurred map value), total int32 [planes] (all peaks, kept or not).
__global__ void __launch_bounds__(256)
op_peak_emit_kernel(const double* __restrict__ blur, const float* __restrict__ maps, long long planes, int H, int W,
                    const int* __restrict__ rowcnt, int* __restrict__ xy, double* __restrict__ score,
                    int* __restrict__ total) {
  pdl_enter_o();
  const long long row = (long long)blockIdx.x * 8 + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (row >= planes * H) return;
  const long long plane = row / H;
  const int y = (int)(row % H);
  int off = 0;
  for (int r = lane; r < y; r += 32) off += rowcnt[plane * H + r];
#pragma unroll
  for (int o = 16; o; o >>= 1) off += __shfl_xor_sync(0xffffffffu, off, o);
  if (y == H - 1 && lane == 0) total[plane] = off + rowcnt[row];
  if (rowcnt[row] == 0 || off >= OP_CAP) return;
  const double* m = blur + plane * (long long)H * W;
  for (int x0 = 0; x0 < W && off < OP_CAP; x0 += 32) {
    const int x = x0 + lane;
    const bool pk = x < W && op_is_peak(m, H, W, y, x);
    const unsigned b = __ballot_sync(0xffffffffu, pk);
    const int k = off + __popc(b & ((1u << lane) - 1u));
    if (pk && k < OP_CAP) {
      xy[(plane * OP_CAP + k) * 2] = x;
      xy[(plane * OP_CAP + k) * 2 + 1] = y;
      score[plane * OP_CAP + k] = (double)maps[plane * (long long)H * W + (long long)y * W + x];
    }
    off += __popc(b);
  }
}

// numpy's round-half-to-even of a float64, as int
__device__ __forceinline__ int op_round(double v) { return (int)rint(v); }

// conn[n, k, i * CAP + j]: score_with_dist_prior of candidate pair (i, j) of limb k, NaN when a criterion fails
__global__ void __launch_bounds__(256)
op_paf_kernel(const float* __restrict__ up, int up_c, int hs, int ws, int H, int W, int mode, int fy, int fx, OpAxis ay,
              OpAxis ax, const int* __restrict__ total, const int* __restrict__ xy, double* __restrict__ conn) {
  pdl_enter_o();
  const int n = blockIdx.z, k = blockIdx.y;
  const int pair = blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= OP_CAP * OP_CAP) return;
  const int i = pair / OP_CAP, j = pair % OP_CAP;
  const int pa = c_limb_a[k] - 1, pb = c_limb_b[k] - 1;
  const int nA = min(total[n * 18 + pa], OP_CAP), nB = min(total[n * 18 + pb], OP_CAP);
  double* o = conn + ((long long)n * 19 + k) * OP_CAP * OP_CAP + pair;
  if (i >= nA || j >= nB) {
    *o = __longlong_as_double(0x7ff8000000000000LL);
    return;
  }
  const int* A = xy + ((long long)(n * 18 + pa) * OP_CAP + i) * 2;
  const int* Bp = xy + ((long long)(n * 18 + pb) * OP_CAP + j) * 2;
  const double ax0 = A[0], ay0 = A[1], bx0 = Bp[0], by0 = Bp[1];
  const double vx = bx0 - ax0, vy = by0 - ay0;
  double norm = __dsqrt_rn(__dadd_rn(__dmul_rn(vx, vx), __dmul_rn(vy, vy)));
  norm = fmax(0.001, norm);
  const double ux = __ddiv_rn(vx, norm), uy = __ddiv_rn(vy, norm);
  const double sx = __ddiv_rn(vx, 9.0), sy = __ddiv_rn(vy, 9.0);
  const float* cx = up + ((long long)n * up_c + (c_paf_x[k] - 19)) * hs * ws;
  const float* cy = cx + (long long)hs * ws;
  double sum = 0.0;
  int above = 0;
  for (int t = 0; t < 10; ++t) {
    // np.linspace: start + t * step (start when the step is 0), the last sample exactly the end point
    const double px = t == 9 ? bx0 : (sx == 0.0 ? ax0 : __dadd_rn(__dmul_rn((double)t, sx), ax0));
    const double py = t == 9 ? by0 : (sy == 0.0 ? ay0 : __dadd_rn(__dmul_rn((double)t, sy), ay0));
    const int X = op_round(px), Y = op_round(py);
    const double fxv = op_resample(cx, ws, mode, fy, fx, ay, ax, Y, X);
    const double fyv = op_resample(cy, ws, mode, fy, fx, ay, ax, Y, X);
    const double s = __dadd_rn(__dmul_rn(fxv, ux), __dmul_rn(fyv, uy));
    sum = __dadd_rn(sum, s);
    above += s > 0.05 ? 1 : 0;
  }
  const double prior = fmin(__dsub_rn(__ddiv_rn(__dmul_rn(0.5, (double)H), norm), 1.0), 0.0);
  const double sc = __dadd_rn(__ddiv_rn(sum, 10.0), prior);
  *o = (above > 8 && sc > 0.0) ? sc : __longlong_as_double(0x7ff8000000000000LL);
}

// One CTA (256 threads) per image.  rows: float64 workspace [B, OP_ROWS, 20] (18 candidate ids, score, parts, as
// the reference's subset); persons int32 [B, OP_ROWS, 18] (per part the peak's index within its part, or -1) and
// pscore float64 [B, OP_ROWS, 2] (total score, parts) of the kept rows; npersons int32 [B].
__global__ void __launch_bounds__(256)
op_assemble_kernel(const int* __restrict__ total, const double* __restrict__ score, const double* __restrict__ conn,
                   double* __restrict__ rows, int* __restrict__ persons, double* __restrict__ pscore,
                   int* __restrict__ npersons) {
  __shared__ int s_base[19];
  __shared__ unsigned char s_usedA[OP_CAP], s_usedB[OP_CAP];
  __shared__ double s_bs[8];
  __shared__ int s_bi[8];
  __shared__ int s_conn_i[OP_CAP], s_conn_j[OP_CAP];
  __shared__ double s_conn_s[OP_CAP];
  __shared__ int s_nconn, s_nrows;
  pdl_enter_o();
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    int b = 0;
    for (int p = 0; p < 18; ++p) {
      s_base[p] = b;
      b += min(total[n * 18 + p], OP_CAP);
    }
    s_base[18] = b;
    s_nrows = 0;
  }
  __syncthreads();
  double* R = rows + (long long)n * OP_ROWS * 20;
  const double* S = score + (long long)n * 18 * OP_CAP;
  for (int k = 0; k < 19; ++k) {
    const int pa = c_limb_a[k] - 1, pb = c_limb_b[k] - 1;
    const int nA = s_base[pa + 1] - s_base[pa], nB = s_base[pb + 1] - s_base[pb];
    if (nA == 0 || nB == 0) continue;
    const double* C = conn + ((long long)n * 19 + k) * OP_CAP * OP_CAP;
    for (int t = tid; t < OP_CAP; t += blockDim.x) s_usedA[t] = s_usedB[t] = 0;
    if (tid == 0) s_nconn = 0;
    __syncthreads();
    // greedy: repeatedly the best remaining pair whose i and j are both unused (== the reference's walk over the
    // stably sorted candidates); ties go to the lower i * CAP + j, the stable sort's order
    for (;;) {
      double best = -INFINITY;
      int bi = -1;
      for (int i = 0; i < nA; ++i) {
        if (s_usedA[i]) continue;
        for (int j = tid; j < nB; j += blockDim.x) {
          const double v = C[i * OP_CAP + j];
          if (!s_usedB[j] && !isnan(v) && v > best) best = v, bi = i * OP_CAP + j;
        }
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (oi >= 0 && (bi < 0 || ob > best || (ob == best && oi < bi))) best = ob, bi = oi;
      }
      if (lane == 0) s_bs[warp] = best, s_bi[warp] = bi;
      __syncthreads();
      if (tid == 0) {
        double b = -INFINITY;
        int id = -1;
        for (int w = 0; w < 8; ++w)
          if (s_bi[w] >= 0 && (id < 0 || s_bs[w] > b || (s_bs[w] == b && s_bi[w] < id))) b = s_bs[w], id = s_bi[w];
        if (id >= 0) {
          s_usedA[id / OP_CAP] = 1;
          s_usedB[id % OP_CAP] = 1;
          s_conn_i[s_nconn] = id / OP_CAP;
          s_conn_j[s_nconn] = id % OP_CAP;
          s_conn_s[s_nconn] = b;
          s_nconn++;
        }
        s_bi[0] = id;
      }
      __syncthreads();
      const bool done = s_bi[0] < 0;
      __syncthreads();
      if (done) break;
    }
    // sequential assembly (body.py:179-219), warp 0; rows with parts == 0 are deleted merges
    if (warp == 0) {
      for (int c = 0; c < s_nconn; ++c) {
        const double idA = (double)(s_base[pa] + s_conn_i[c]), idB = (double)(s_base[pb] + s_conn_j[c]);
        const double cs = s_conn_s[c];
        int found = 0, j1 = -1, j2 = -1;
        const int nr = s_nrows;
        for (int r0 = 0; r0 < nr && found < 2; r0 += 32) {
          const int r = r0 + lane;
          const bool m = r < nr && R[r * 20 + 19] != 0.0 && (R[r * 20 + pa] == idA || R[r * 20 + pb] == idB);
          unsigned b = __ballot_sync(0xffffffffu, m);
          while (b && found < 2) {
            const int f = r0 + __ffs(b) - 1;
            if (found == 0) j1 = f; else j2 = f;
            ++found;
            b &= b - 1;
          }
        }
        if (lane == 0) {
          const double sB = S[pb * OP_CAP + s_conn_j[c]];
          if (found == 1) {
            double* row = R + j1 * 20;
            if (row[pb] != idB) {
              row[pb] = idB;
              row[19] += 1.0;
              row[18] = __dadd_rn(row[18], __dadd_rn(sB, cs));
            }
          } else if (found == 2) {
            double* r1 = R + j1 * 20;
            double* r2 = R + j2 * 20;
            bool disjoint = true;
            for (int p = 0; p < 18; ++p) disjoint &= !(r1[p] >= 0.0 && r2[p] >= 0.0);
            if (disjoint) {
              for (int p = 0; p < 18; ++p) r1[p] = __dadd_rn(r1[p], __dadd_rn(r2[p], 1.0));
              r1[18] = __dadd_rn(r1[18], r2[18]);
              r1[19] = __dadd_rn(r1[19], r2[19]);
              r1[18] = __dadd_rn(r1[18], cs);
              r2[19] = 0.0;                                   // np.delete(subset, j2): never matched again
            } else {
              r1[pb] = idB;
              r1[19] += 1.0;
              r1[18] = __dadd_rn(r1[18], __dadd_rn(sB, cs));
            }
          } else if (k < 17 && nr < OP_ROWS) {
            double* row = R + nr * 20;
            for (int p = 0; p < 18; ++p) row[p] = -1.0;
            row[pa] = idA;
            row[pb] = idB;
            row[19] = 2.0;
            row[18] = __dadd_rn(__dadd_rn(S[pa * OP_CAP + s_conn_i[c]], sB), cs);
            s_nrows = nr + 1;
          }
        }
        __syncwarp();
      }
    }
    __syncthreads();
  }
  // delete rows with < 4 parts or score / parts < 0.4; compact in order
  if (tid == 0) {
    int m = 0;
    for (int r = 0; r < s_nrows; ++r) {
      const double* row = R + r * 20;
      if (row[19] == 0.0 || row[19] < 4.0 || __ddiv_rn(row[18], row[19]) < 0.4) continue;
      for (int p = 0; p < 18; ++p) {
        const int id = (int)row[p];
        persons[((long long)n * OP_ROWS + m) * 18 + p] = id < 0 ? -1 : id - s_base[p];
      }
      pscore[((long long)n * OP_ROWS + m) * 2] = row[18];
      pscore[((long long)n * OP_ROWS + m) * 2 + 1] = row[19];
      ++m;
    }
    npersons[n] = m;
  }
}

__device__ __forceinline__ void op_put(int* idx, int H, int W, long long x, long long y, int prim) {
  if (x >= 0 && x < W && y >= 0 && y < H) atomicMax(idx + y * W + x, prim);
}

// OpenCV's clipLine(Size(W, H), pt1, pt2) in int64 (drawing.cpp): false when the segment misses the image
__device__ bool op_clip(long long W, long long H, long long& x1, long long& y1, long long& x2, long long& y2) {
  const long long right = W - 1, bottom = H - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    long long a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += (long long)__ddiv_rn(__dmul_rn((double)(a - y1), (double)(x2 - x1)), (double)(y2 - y1));
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += (long long)__ddiv_rn(__dmul_rn((double)(a - y2), (double)(x2 - x1)), (double)(y2 - y1));
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += (long long)__ddiv_rn(__dmul_rn((double)(a - x1), (double)(y2 - y1)), (double)(x2 - x1));
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += (long long)__ddiv_rn(__dmul_rn((double)(a - x2), (double)(y2 - y1)), (double)(x2 - x1));
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// cv2.line(..., 1, LINE_8) pixels, warp-parallel: clipLine, then the 8-connected LineIterator in closed form
__device__ void op_line(int* idx, int H, int W, long long x1, long long y1, long long x2, long long y2, int prim,
                        int lane) {
  if (!op_clip(W, H, x1, y1, x2, y2)) return;
  if (x2 < x1) {
    long long t = x1; x1 = x2; x2 = t;
    t = y1; y1 = y2; y2 = t;
  }
  const long long dx = x2 - x1, ady = y2 >= y1 ? y2 - y1 : y1 - y2;
  const long long sy = y2 >= y1 ? 1 : -1;
  const bool vert = ady > dx;
  const long long D = vert ? ady : dx, d = vert ? dx : ady;
  for (long long i = lane; i <= D; i += 32) {
    const long long a = 2 * d * i - D;
    const long long m = D == 0 ? 0 : (a >= 0 ? (a + 2 * D - 1) / (2 * D) : -((-a) / (2 * D)));
    op_put(idx, H, W, vert ? x1 + m : x1 + i, vert ? y1 + sy * i : y1 + sy * m, prim);
  }
}

constexpr int OP_WARPS = 4;
constexpr int OP_DRAW_BLOCKS = 64;   // per image: 256 warps share the primitives

// One primitive, drawn by one warp: its pixels get atomicMax(prim).  pts: the warp's ellipse2Poly buffer.
__device__ void op_draw_prim(const int* __restrict__ persons, const int* __restrict__ xy, int H, int W,
                             const float* __restrict__ sintab, int* __restrict__ idx, int (*pts)[2], int n, int prim,
                             int lane) {
  const int p = prim / OP_PRIMS, s = prim % OP_PRIMS;
  const int* person = persons + ((long long)n * OP_ROWS + p) * 18;
  int* canvas = idx + (long long)n * H * W;
  const double fW = W, fH = H;
  // keypoint (x / W) * W and (y / H) * H in float64, as the reference stores and draws them
  auto kp = [&](int part, double& kx, double& ky) -> bool {
    const int c = person[part];
    if (c < 0) return false;
    const int* q = xy + ((long long)(n * 18 + part) * OP_CAP + c) * 2;
    kx = __dmul_rn(__ddiv_rn((double)q[0], fW), fW);
    ky = __dmul_rn(__ddiv_rn((double)q[1], fH), fH);
    return true;
  };
  if (s >= 17) {
    double kx, ky;
    if (!kp(s - 17, kx, ky)) return;
    const long long cx = (long long)kx, cy = (long long)ky;
    // cv2.circle(r=4, filled): the spans of OpenCV's Circle() for radius 4
    int err = 0, dx = 4, dy = 0, plus = 1, minus = 7;
    while (dx >= dy) {
      for (int t = lane; t < 4 * 9; t += 32) {
        const int span = t / 9, o = t % 9 - 4;
        const int half = span < 2 ? dx : dy, yo = span == 0 ? -dy : span == 1 ? dy : span == 2 ? -dx : dx;
        if (o >= -half && o <= half) op_put(canvas, H, W, cx + o, cy + yo, prim);
      }
      dy++;
      err += plus;
      plus += 2;
      const int mask = (err <= 0) - 1;
      err -= minus & mask;
      dx += mask;
      minus -= mask & 2;
    }
    return;
  }
  double x1, y1, x2, y2;
  if (!kp(c_limb_a[s] - 1, x1, y1) || !kp(c_limb_b[s] - 1, x2, y2)) return;
  // util.py:106-113: X = y coordinates, Y = x coordinates
  const double mX = __ddiv_rn(__dadd_rn(y1, y2), 2.0), mY = __ddiv_rn(__dadd_rn(x1, x2), 2.0);
  const double ex = __dsub_rn(y1, y2), ey = __dsub_rn(x1, x2);
  const double length = __dsqrt_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)));
  // math.degrees(math.atan2(.)) is exactly 0, +-45, +-90, +-135 or 180 on the axes and diagonals; int() of CUDA's atan2
  // (up to 2 ulp) could land one degree low there, so those cases are taken exactly
  double angle;
  if (ex == 0.0 || ey == 0.0 || fabs(ex) == fabs(ey)) {
    const double q = ex == 0.0 ? (ey < 0.0 ? 180.0 : 0.0) : ey == 0.0 ? 90.0 : (ey > 0.0 ? 45.0 : 135.0);
    angle = ex < 0.0 ? -q : q;
  } else {
    angle = __dmul_rn(atan2(ex, ey), 180.0 / 3.141592653589793);
  }
  const long long ccx = (long long)mY, ccy = (long long)mX;
  const int axw = (int)__ddiv_rn(length, 2.0), axh = 4;
  int ang = (int)angle;
  while (ang < 0) ang += 360;
  while (ang > 360) ang -= 360;
  const double alpha = sintab[450 - ang], beta = sintab[ang];     // cos, sin
  // ellipse2Poly(center, axes, angle, 0, 360, 1): 361 points, cvRound, consecutive duplicates removed
  int np = 0;
  for (int i0 = 0; i0 <= 360; i0 += 32) {
    const int i = i0 + lane;
    long long px = 0, py = 0;
    if (i <= 360) {
      const double x = __dmul_rn((double)axw, (double)sintab[450 - i]);
      const double y = __dmul_rn((double)axh, (double)sintab[i]);
      px = __double2ll_rn(__dsub_rn(__dadd_rn((double)ccx, __dmul_rn(x, alpha)), __dmul_rn(y, beta)));
      py = __double2ll_rn(__dadd_rn(__dadd_rn((double)ccy, __dmul_rn(x, beta)), __dmul_rn(y, alpha)));
    }
    long long qx = __shfl_up_sync(0xffffffffu, px, 1), qy = __shfl_up_sync(0xffffffffu, py, 1);
    if (lane == 0) {
      qx = np ? (long long)pts[np - 1][0] : LLONG_MIN;
      qy = np ? (long long)pts[np - 1][1] : LLONG_MIN;
    }
    const bool keep = i <= 360 && (px != qx || py != qy);
    const unsigned b = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      const int k = np + __popc(b & ((1u << lane) - 1u));
      pts[k][0] = (int)px;
      pts[k][1] = (int)py;
    }
    np += __popc(b);
    __syncwarp();
  }
  if (np == 1) {
    pts[1][0] = pts[0][0] = (int)ccx;
    pts[1][1] = pts[0][1] = (int)ccy;
    np = 2;
  }
  __syncwarp();
  // fillConvexPoly(shift 0, LINE_8): the outline as lines, then spans between the two edge walkers
  for (int i = 0; i < np; ++i) {
    const int a = i == 0 ? np - 1 : i - 1;
    op_line(canvas, H, W, pts[a][0], pts[a][1], pts[i][0], pts[i][1], prim, lane);
  }
  long long xmin = pts[0][0], xmax = pts[0][0], ymin = pts[0][1], ymax = pts[0][1];
  int imin = 0;
  for (int i = 0; i < np; ++i) {
    if (pts[i][1] < ymin) ymin = pts[i][1], imin = i;
    ymax = max(ymax, (long long)pts[i][1]);
    xmax = max(xmax, (long long)pts[i][0]);
    xmin = min(xmin, (long long)pts[i][0]);
  }
  if (np < 3 || xmax < 0 || ymax < 0 || xmin >= W || ymin >= H) return;
  const long long ONE = 1LL << 16, HALF = ONE >> 1;
  ymax = min(ymax, (long long)H - 1);
  int e_idx[2] = {imin, imin}, e_di[2] = {1, np - 1}, e_ye[2] = {(int)ymin, (int)ymin};
  long long e_x[2] = {-ONE, -ONE}, e_dx[2] = {0, 0};
  int edges = np;
  long long y = ymin;
  do {
    for (int e = 0; e < 2; ++e) {
      if (y >= e_ye[e]) {
        int i0 = e_idx[e], di = e_di[e];
        int ii = i0 + di;
        if (ii >= np) ii -= np;
        for (; edges-- > 0;) {
          const int ty = pts[ii][1];
          if (ty > y) {
            const long long xs = (long long)pts[i0][0] << 16, xe = (long long)pts[ii][0] << 16;
            e_ye[e] = ty;
            e_dx[e] = ((xe - xs) * 2 + (ty - y)) / (2 * (ty - y));
            e_x[e] = xs;
            e_idx[e] = ii;
            break;
          }
          i0 = ii;
          ii += di;
          if (ii >= np) ii -= np;
        }
      }
    }
    if (edges < 0) break;
    if (y >= 0) {
      const int l = e_x[0] > e_x[1] ? 1 : 0, r = 1 - l;
      long long xx1 = (e_x[l] + HALF) >> 16, xx2 = (e_x[r] + HALF) >> 16;
      if (xx2 >= 0 && xx1 < W) {
        xx1 = max(xx1, 0LL);
        xx2 = min(xx2, (long long)W - 1);
        for (long long x = xx1 + lane; x <= xx2; x += 32) op_put(canvas, H, W, x, y, prim);
      }
    }
    e_x[0] += e_dx[0];
    e_x[1] += e_dx[1];
  } while (++y <= ymax);
}

// Warps loop over the primitives of the image's persons (blockIdx.y = image): person p = prim / 35, slot s = prim % 35
// (limb s < 17, else keypoint s - 17); the grid does not depend on the person count, which stays on the device.  idx: int32 [B, H, W], -1 where nothing is drawn.
__global__ void __launch_bounds__(OP_WARPS * 32)
op_draw_kernel(const int* __restrict__ persons, const int* __restrict__ npersons, const int* __restrict__ xy, int H,
               int W, const float* __restrict__ sintab, int* __restrict__ idx) {
  __shared__ int s_pts[OP_WARPS][362][2];
  pdl_enter_o();
  const int n = blockIdx.y, warp = threadIdx.x / 32, lane = threadIdx.x & 31;
  const int nprim = npersons[n] * OP_PRIMS;
  for (int prim = blockIdx.x * OP_WARPS + warp; prim < nprim; prim += gridDim.x * OP_WARPS)
    op_draw_prim(persons, xy, H, W, sintab, idx, s_pts[warp], n, prim, lane);
}

// out[n, c, y, x] = colour[idx % 35][c] / 255 (0 where idx < 0)
__global__ void __launch_bounds__(256)
op_color_kernel(const int* __restrict__ idx, int B, int H, int W, const unsigned char* __restrict__ colors,
                float* __restrict__ out) {
  pdl_enter_o();
  const long long HW = (long long)H * W, total = (long long)B * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = idx[i];
    const long long n = i / HW, p = i % HW;
#pragma unroll
    for (int c = 0; c < 3; ++c)
      out[(n * 3 + c) * HW + p] = v < 0 ? 0.f : __fdiv_rn((float)colors[(v % OP_PRIMS) * 3 + c], 255.f);
  }
}

}  // namespace pfd

using namespace pfd;

static bool misaligned_o(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

static bool axis_ok(const int32_t* idx, const void* w, int32_t taps) { return idx && w && taps > 0; }

extern "C" PFD_API int pfd_openpose_input_f16(const void* x, int32_t x_f32, int32_t B, int32_t H, int32_t W, int32_t h,
                                              int32_t w, int32_t hp, int32_t wp, int32_t mode, int32_t fy, int32_t fx,
                                              const int32_t* iy, const void* wy, int32_t ty, const int32_t* ix,
                                              const void* wx, int32_t tx, void* out, void* stream) {
  if (!x || !out || B <= 0 || H <= 0 || W <= 0 || h <= 0 || w <= 0 || hp < h || wp < w || mode < 0 || mode > 3 ||
      (mode == 1 && (fy <= 0 || fx <= 0 || h * fy > H || w * fx > W)) ||
      (mode >= 2 && (!axis_ok(iy, wy, ty) || !axis_ok(ix, wx, tx) || (mode == 2 && (ty != 8 || tx != 8)))) ||
      (mode == 0 && (h != H || w != W)))
    return set_error("pfd_openpose_input_f16: bad arguments (B=%d H=%d W=%d h=%d w=%d mode=%d)", B, H, W, h, w, mode);
  if (misaligned_o(out)) return set_error("pfd_openpose_input_f16: out must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const OpAxis ay{iy, wy, ty}, ax{ix, wx, tx};
  const int g = grid_cap_o((long long)B * hp * wp, 256);
  if (x_f32)
    launch_k(op_input_kernel<float>, dim3(g), dim3(256), (size_t)0, st, static_cast<const float*>(x), (int)B, (int)H,
             (int)W, (int)h, (int)w, (int)hp, (int)wp, (int)mode, (int)fy, (int)fx, ay, ax, static_cast<__half*>(out));
  else
    launch_k(op_input_kernel<__half>, dim3(g), dim3(256), (size_t)0, st, static_cast<const __half*>(x), (int)B, (int)H,
             (int)W, (int)h, (int)w, (int)hp, (int)wp, (int)mode, (int)fy, (int)fx, ay, ax, static_cast<__half*>(out));
  return check_launch("openpose_input");
}

extern "C" PFD_API int pfd_openpose_pool_f16(const void* x, int32_t B, int32_t H, int32_t W, int32_t C, void* out,
                                             void* stream) {
  if (!x || !out || B <= 0 || H < 2 || W < 2 || C <= 0 || C % 8)
    return set_error("pfd_openpose_pool_f16: bad arguments (B=%d H=%d W=%d C=%d)", B, H, W, C);
  if (misaligned_o(x) || misaligned_o(out)) return set_error("pfd_openpose_pool_f16: x and out must be 16-byte aligned");
  launch_k(op_pool_kernel, dim3(grid_cap_o((long long)B * (H / 2) * (W / 2) * (C / 8), 256)), dim3(256), (size_t)0,
           static_cast<cudaStream_t>(stream), static_cast<const __half*>(x), (int)B, (int)H, (int)W, (int)C,
           static_cast<__half*>(out));
  return check_launch("openpose_pool");
}

extern "C" PFD_API int pfd_im2col7x7_f16(const void* x, int32_t B, int32_t H, int32_t W, int32_t C, void* out,
                                         void* stream) {
  if (!x || !out || B <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8)
    return set_error("pfd_im2col7x7_f16: bad arguments (B=%d H=%d W=%d C=%d)", B, H, W, C);
  if (misaligned_o(x) || misaligned_o(out)) return set_error("pfd_im2col7x7_f16: x and out must be 16-byte aligned");
  launch_k(op_im2col7_kernel, dim3(grid_cap_o((long long)B * H * W * 49 * (C / 8), 256)), dim3(256), (size_t)0,
           static_cast<cudaStream_t>(stream), static_cast<const __half*>(x), (int)B, (int)H, (int)W, (int)C,
           static_cast<__half*>(out));
  return check_launch("im2col7x7");
}

extern "C" PFD_API int pfd_openpose_head_f32(const void* x, int32_t B, int32_t h, int32_t w, int32_t C, const float* wt,
                                             const float* b, int32_t N, int32_t relu, float* out, int32_t out_c,
                                             int32_t out_off, void* stream) {
  if (!x || !wt || !b || !out || B <= 0 || h <= 0 || w <= 0 || C <= 0 || C % 8 || N <= 0 || out_off < 0 ||
      out_off + N > out_c)
    return set_error("pfd_openpose_head_f32: bad arguments (B=%d h=%d w=%d C=%d N=%d)", B, h, w, C, N);
  if (misaligned_o(x)) return set_error("pfd_openpose_head_f32: x must be 16-byte aligned");
  launch_k(op_head_kernel, dim3(grid_cap_o((long long)B * h * w * N, 256)), dim3(256), (size_t)0,
           static_cast<cudaStream_t>(stream), static_cast<const __half*>(x), (int)B, (int)h, (int)w, (int)C, wt, b,
           (int)N, (int)relu, out, (int)out_c, (int)out_off);
  return check_launch("openpose_head");
}

extern "C" PFD_API int pfd_openpose_resize_f32(const float* src, int32_t B, int32_t src_c, int32_t c0, int32_t C,
                                               int32_t hs, int32_t ws, int32_t H, int32_t W, int32_t mode, int32_t fy,
                                               int32_t fx, const int32_t* iy, const float* wy, int32_t ty,
                                               const int32_t* ix, const float* wx, int32_t tx, float* out, void* stream) {
  if (!src || !out || B <= 0 || C <= 0 || c0 < 0 || c0 + C > src_c || hs <= 0 || ws <= 0 || H <= 0 || W <= 0 ||
      mode < 0 || mode > 2 || (mode == 0 && (H > hs || W > ws)) ||
      (mode == 1 && (fy <= 0 || fx <= 0 || H * fy > hs || W * fx > ws)) ||
      (mode == 2 && (!axis_ok(iy, wy, ty) || !axis_ok(ix, wx, tx))))
    return set_error("pfd_openpose_resize_f32: bad arguments (B=%d C=%d %dx%d -> %dx%d mode=%d)", B, C, hs, ws, H, W,
                     mode);
  const OpAxis ay{iy, wy, ty}, ax{ix, wx, tx};
  launch_k(op_resize_kernel, dim3(grid_cap_o((long long)B * C * H * W, 256)), dim3(256), (size_t)0,
           static_cast<cudaStream_t>(stream), src, (int)B, (int)src_c, (int)c0, (int)C, (int)hs, (int)ws, (int)H,
           (int)W, (int)mode, (int)fy, (int)fx, ay, ax, out);
  return check_launch("openpose_resize");
}

extern "C" PFD_API int pfd_openpose_peaks_f32(const float* maps, int32_t B, int32_t H, int32_t W, const double* gauss,
                                              double* tmp, double* blur, int32_t* rowcnt, int32_t* xy, double* score,
                                              int32_t* total, void* stream) {
  if (!maps || !gauss || !tmp || !blur || !rowcnt || !xy || !score || !total || B <= 0 || H <= 0 || W <= 0)
    return set_error("pfd_openpose_peaks_f32: bad arguments (B=%d H=%d W=%d)", B, H, W);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long planes = (long long)B * 18, px = planes * H * W;
  launch_k(op_gauss_kernel<float>, dim3(grid_cap_o(px, 256)), dim3(256), (size_t)0, st, maps, planes, (int)H, (int)W,
           0, gauss, tmp);
  if (int rc = check_launch("openpose_gauss_y")) return rc;
  launch_k(op_gauss_kernel<double>, dim3(grid_cap_o(px, 256)), dim3(256), (size_t)0, st,
           static_cast<const double*>(tmp), planes, (int)H, (int)W, 1, gauss, blur);
  if (int rc = check_launch("openpose_gauss_x")) return rc;
  const long long rowsn = planes * H;
  const unsigned g = (unsigned)((rowsn + 7) / 8);
  launch_k(op_peak_count_kernel, dim3(g), dim3(256), (size_t)0, st, static_cast<const double*>(blur), planes, (int)H,
           (int)W, static_cast<int*>(rowcnt));
  if (int rc = check_launch("openpose_peak_count")) return rc;
  launch_k(op_peak_emit_kernel, dim3(g), dim3(256), (size_t)0, st, static_cast<const double*>(blur), maps, planes,
           (int)H, (int)W, static_cast<const int*>(rowcnt), static_cast<int*>(xy), score, static_cast<int*>(total));
  return check_launch("openpose_peak_emit");
}

extern "C" PFD_API int pfd_openpose_assemble_f32(const float* up, int32_t B, int32_t up_c, int32_t hs, int32_t ws,
                                                 int32_t H, int32_t W, int32_t mode, int32_t fy, int32_t fx,
                                                 const int32_t* iy, const float* wy, int32_t ty, const int32_t* ix,
                                                 const float* wx, int32_t tx, const int32_t* total, const int32_t* xy,
                                                 const double* score, double* conn, double* rows, int32_t* persons,
                                                 double* pscore, int32_t* npersons, void* stream) {
  if (!up || !total || !xy || !score || !conn || !rows || !persons || !pscore || !npersons || B <= 0 || B > 65535 ||
      up_c != 57 || mode < 0 || mode > 2 || (mode == 2 && (!axis_ok(iy, wy, ty) || !axis_ok(ix, wx, tx))))
    return set_error("pfd_openpose_assemble_f32: bad arguments (B=%d up_c=%d mode=%d)", B, up_c, mode);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const OpAxis ay{iy, wy, ty}, ax{ix, wx, tx};
  launch_k(op_paf_kernel, dim3(OP_CAP * OP_CAP / 256, 19, B), dim3(256), (size_t)0, st, up, (int)up_c, (int)hs,
           (int)ws, (int)H, (int)W, (int)mode, (int)fy, (int)fx, ay, ax, static_cast<const int*>(total),
           static_cast<const int*>(xy), conn);
  if (int rc = check_launch("openpose_paf")) return rc;
  launch_k(op_assemble_kernel, dim3(B), dim3(256), (size_t)0, st, static_cast<const int*>(total), score,
           static_cast<const double*>(conn), rows, static_cast<int*>(persons), pscore, static_cast<int*>(npersons));
  return check_launch("openpose_assemble");
}

extern "C" PFD_API int pfd_openpose_draw_f32(const int32_t* persons, const int32_t* npersons, const int32_t* xy,
                                             int32_t B, int32_t H, int32_t W, const float* sintab,
                                             const uint8_t* colors, int32_t* idx, float* out, void* stream) {
  if (!persons || !npersons || !xy || !sintab || !colors || !idx || !out || B <= 0 || B > 65535 || H <= 0 || W <= 0)
    return set_error("pfd_openpose_draw_f32: bad arguments (B=%d H=%d W=%d)", B, H, W);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (cudaMemsetAsync(idx, 0xff, sizeof(int32_t) * (size_t)B * H * W, st) != cudaSuccess)
    return set_error("pfd_openpose_draw_f32: memset failed");
  launch_k(op_draw_kernel, dim3(OP_DRAW_BLOCKS, B), dim3(OP_WARPS * 32), (size_t)0, st,
           static_cast<const int*>(persons), static_cast<const int*>(npersons), static_cast<const int*>(xy), (int)H,
           (int)W, sintab, static_cast<int*>(idx));
  if (int rc = check_launch("openpose_draw")) return rc;
  launch_k(op_color_kernel, dim3(grid_cap_o((long long)B * H * W, 256)), dim3(256), (size_t)0, st,
           static_cast<const int*>(idx), (int)B, (int)H, (int)W, static_cast<const unsigned char*>(colors), out);
  return check_launch("openpose_color");
}
