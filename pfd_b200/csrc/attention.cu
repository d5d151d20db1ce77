// Fused attention for sm_90a (wgmma + TMA + mbarrier) of the UNet / ControlNet / SeeCoder self- and cross-attention
// (attention.py:178-201):  O = softmax(Q K^T * scale) V  per (batch, head), the [N, Nk] score matrix never reaches HBM.
//
// flash_attn_kernel (any Nk, d <= 192):
//   CTA = 128 query rows of one (batch, head); keys processed in blocks of 64.
//   warps 0..7 : two consumer warpgroups, 64 query rows each:
//                S_j = Q K_j^T        wgmma, A = Q and B = K_j from shared memory, fp32 logits in registers;
//                online softmax       row max / sum over the 4 threads of a row (2 shuffles), p = 2^(s*scale*log2e - m)
//                                     rounded to fp16, the running output rescaled in registers when m moves;
//                O += P_j V_j         wgmma with A = P straight from registers (the S accumulator fragment is the A
//                                     operand fragment), B = the V^T block (d rows x 64 keys, K-major) from shared memory.
//   warp 8     : TMA producer (Q once; K and V^T blocks through 2-stage rings released by the consumer warps).
//   The row sum l accumulates the fp16-rounded probabilities, the values the PV product actually uses.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include "../../include/pfd_b200.h"
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace pfd {

constexpr int FA_BQ = 128;
constexpr int FA_BKV = 64;
constexpr int FA_THREADS = 288;       // 2 consumer warpgroups + 1 producer warp

__device__ __forceinline__ float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct alignas(64) FlashParams {
  CUtensorMap tmQ, tmK, tmV;
  int Nq, Nk, heads, d;
  int nblk;
  float scale;
  __half* out;
  long long o_sb, o_sq, o_sh;  // element strides: batch, query row, head
};

// DCH: 64-wide chunks of the head dim (Q / K tiles); DP: head dim padded to the wgmma N granule of 16 (V^T rows)
template <int DCH, int DP>
struct FlashCfg {
  static constexpr int Q_BYTES = DCH * FA_BQ * 128;
  static constexpr int K_BYTES = DCH * FA_BKV * 128;
  static constexpr int V_BYTES = DP * 128;
  static constexpr int SMEM_BYTES = Q_BYTES + 2 * K_BYTES + 2 * V_BYTES + 1024 + 128;
  static_assert(DP % 16 == 0 && DP <= 64 * DCH, "V^T rows");
};

template <int DCH, int DP>
__global__ void __launch_bounds__(FA_THREADS, DCH == 1 ? 2 : 1)
flash_attn_kernel(const __grid_constant__ FlashParams p) {
  using Cfg = FlashCfg<DCH, DP>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - raw_addr);
  const int d = p.d;
  const uint32_t sQ = base;
  const uint32_t sK = sQ + Cfg::Q_BYTES;                  // [2][K_BYTES]
  const uint32_t sV = sK + 2 * Cfg::K_BYTES;              // [2][V_BYTES]
  const uint32_t bars = sV + 2 * Cfg::V_BYTES;
  const uint32_t bar_q = bars;
  auto k_full = [&](int s) { return bars + 8u * (1 + s); };
  auto k_empty = [&](int s) { return bars + 8u * (3 + s); };
  auto v_full = [&](int s) { return bars + 8u * (5 + s); };
  auto v_empty = [&](int s) { return bars + 8u * (7 + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * FA_BQ;
  const int bh = blockIdx.y;
  const int hb = bh % p.heads, bb = bh / p.heads;
  const int nblk = p.nblk;

  if (threadIdx.x == 256) {
    tma_prefetch_desc(&p.tmQ);
    tma_prefetch_desc(&p.tmK);
    tma_prefetch_desc(&p.tmV);
    mbar_init(bar_q, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(k_full(s), 1);
      mbar_init(k_empty(s), 8);            // one arrival per consumer warp
      mbar_init(v_full(s), 1);
      mbar_init(v_empty(s), 8);
    }
    mbar_fence_init();
  }
  if (DP > d && warp < 8) {
    // rows d..DP-1 of the V^T stages are never written by TMA (its box has d rows): zero, so the padded output
    // columns stay finite
    const int per_stage = (DP - d) * 8;               // 16-byte granules
    for (int i = threadIdx.x; i < 2 * per_stage; i += 256) {
      const int st = i / per_stage, g = i % per_stage;
      *reinterpret_cast<uint4*>(gbase + Cfg::Q_BYTES + 2 * Cfg::K_BYTES + st * Cfg::V_BYTES + d * 128 + g * 16) =
          make_uint4(0, 0, 0, 0);
    }
    fence_proxy_async_smem();
  }
  __syncthreads();
  pdl_wait();                  // q / k / v are produced by the preceding projection GEMMs
  pdl_launch_dependents();

  if (warp == 8) {
    if (lane == 0) {
      mbar_expect_tx(bar_q, Cfg::Q_BYTES);
      for (int c = 0; c < DCH; ++c) tma_load_4d(sQ + c * FA_BQ * 128, &p.tmQ, bar_q, c * 64, q0, hb, bb);
      for (int j = 0; j < nblk; ++j) {
        const int st = j & 1, u = j >> 1;
        if (u >= 1) mbar_wait(k_empty(st), (u - 1) & 1);          // S of block j - 2 has read the stage
        mbar_expect_tx(k_full(st), Cfg::K_BYTES);
        for (int c = 0; c < DCH; ++c)
          tma_load_4d(sK + st * Cfg::K_BYTES + c * FA_BKV * 128, &p.tmK, k_full(st), c * 64, j * FA_BKV, hb, bb);
        if (u >= 1) mbar_wait(v_empty(st), (u - 1) & 1);          // PV of block j - 2 has read the stage
        mbar_expect_tx(v_full(st), d * 128);
        tma_load_4d(sV + st * Cfg::V_BYTES, &p.tmV, v_full(st), j * FA_BKV, 0, hb, bb);
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumer warpgroups
  const int cw = warp >> 2;                  // rows [64 cw, 64 cw + 64) of the query tile
  const int wl = warp & 3;
  const int tq = lane & 3;
  const float c2 = p.scale * 1.4426950408889634f;   // logits in log2 units: t = s * c2
  float o[DP / 2];
#pragma unroll
  for (int i = 0; i < DP / 2; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  mbar_wait(bar_q, 0);
  for (int j = 0; j < nblk; ++j) {
    const int st = j & 1;
    const uint32_t ph = (j >> 1) & 1;
    mbar_wait(k_full(st), ph);
    float s[FA_BKV / 2];
#pragma unroll
    for (int i = 0; i < FA_BKV / 2; ++i) s[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < DCH; ++c) {
      const uint64_t ad = make_sw128_kmajor_desc(sQ + c * FA_BQ * 128 + cw * 64 * 128);
      const uint64_t bd = make_sw128_kmajor_desc(sK + st * Cfg::K_BYTES + c * FA_BKV * 128);
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (c * 64 + k * 16 < d) Wgmma<FA_BKV>::ss(s, ad + 2u * k, bd + 2u * k, (c | k) != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(k_empty(st));
    // mask keys beyond Nk (their K rows are TMA zero fill): column 8 jj + 2 tq + e of the block
    const int kvalid = p.Nk - j * FA_BKV;
    if (kvalid < FA_BKV) {
#pragma unroll
      for (int jj = 0; jj < FA_BKV / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * jj + 2 * tq + e >= kvalid) {
            s[4 * jj + e] = -INFINITY;
            s[4 * jj + 2 + e] = -INFINITY;
          }
    }
    // row maxima (rows r0 = 16 wl + lane / 4 and r0 + 8): 16 values per thread, then across the 4 threads of the row
    float mx[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float a = fmax3(s[2 * i], s[2 * i + 1], s[4 + 2 * i]);
      float b = fmax3(s[4 + 2 * i + 1], s[8 + 2 * i], s[8 + 2 * i + 1]);
#pragma unroll
      for (int jj = 3; jj < FA_BKV / 8; ++jj) {
        if (jj & 1) b = fmax3(b, s[4 * jj + 2 * i], s[4 * jj + 2 * i + 1]);
        else a = fmax3(a, s[4 * jj + 2 * i], s[4 * jj + 2 * i + 1]);
      }
      mx[i] = fmaxf(a, b);
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
    }
    float nm[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float mnew = fmaxf(m[i], mx[i] * c2);
      const float alpha = fast_exp2(m[i] - mnew);       // j == 0: exp2(-inf) = 0 (o and l are still 0)
      m[i] = mnew;
      nm[i] = -mnew;
      l[i] *= alpha;
#pragma unroll
      for (int jj = 0; jj < DP / 8; ++jj) {
        o[4 * jj + 2 * i] *= alpha;
        o[4 * jj + 2 * i + 1] *= alpha;
      }
    }
    // P = 2^(s c2 - m) in fp16, laid out as the A fragments of the four k16 steps of the PV product
    uint32_t pa[4][4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = r & 1;                    // row r0 (i = 0) or r0 + 8
        const int idx = 8 * k + 4 * (r >> 1) + 2 * i;
        const __half2 h = __floats2half2_rn(fast_exp2(fmaf(s[idx], c2, nm[i])), fast_exp2(fmaf(s[idx + 1], c2, nm[i])));
        const float2 hf = __half22float2(h);
        l[i] += hf.x + hf.y;
        pa[k][r] = *reinterpret_cast<const uint32_t*>(&h);
      }
    }
    mbar_wait(v_full(st), ph);
    wgmma_fence();
    const uint64_t vd = make_sw128_kmajor_desc(sV + st * Cfg::V_BYTES);
#pragma unroll
    for (int k = 0; k < 4; ++k) Wgmma<DP>::rs(o, pa[k], vd + 2u * k, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(v_empty(st));
  }
  // ---- epilogue: O / l -> [B, Nq, heads*d]
  const int b = bh / p.heads, h = bh % p.heads;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float li = l[i];
    li += __shfl_xor_sync(0xffffffffu, li, 1);
    li += __shfl_xor_sync(0xffffffffu, li, 2);
    const float inv = li > 0.f ? 1.f / li : 0.f;
    const int q = q0 + cw * 64 + wl * 16 + (lane >> 2) + 8 * i;
    if (q >= p.Nq) continue;
    __half* orow = p.out + (long long)b * p.o_sb + (long long)q * p.o_sq + (long long)h * p.o_sh;
#pragma unroll
    for (int jj = 0; jj < DP / 8; ++jj) {
      const int col = 8 * jj + 2 * tq;
      if (col < d)
        *reinterpret_cast<__half2*>(orow + col) = __floats2half2_rn(o[4 * jj + 2 * i] * inv, o[4 * jj + 2 * i + 1] * inv);
    }
  }
}

// [B, heads, rows, inner] operand at element strides (sb, sh, sr), read in boxes of 64 x box_rows
static int encode4d(CUtensorMap* m, const void* ptr, cuuint64_t inner, cuuint64_t rows, cuuint64_t heads,
                    cuuint64_t B, long long sr, long long sh, long long sb, cuuint32_t box_rows, const char* what) {
  const cuuint64_t dims[4] = {inner, rows, heads, B};
  const cuuint64_t strides[3] = {(cuuint64_t)sr * 2, (cuuint64_t)sh * 2, (cuuint64_t)sb * 2};
  const cuuint32_t box[4] = {64, box_rows, 1, 1};
  const cuuint32_t es[4] = {1, 1, 1, 1};
  return encode_tensor_map_f16(m, ptr, 4, dims, strides, box, es, what);
}

template <int DCH, int DP>
static int launch_flash(const FlashParams& p, dim3 grid, cudaStream_t st) {
  using Cfg = FlashCfg<DCH, DP>;
  if (int rc = smem_opt_in<flash_attn_kernel<DCH, DP>>(Cfg::SMEM_BYTES, "flash_attn_kernel")) return rc;
  launch_k(flash_attn_kernel<DCH, DP>, grid, dim3(FA_THREADS), (size_t)Cfg::SMEM_BYTES, st, p);
  return check_launch("pfd_flash_attn_f16");
}

}  // namespace pfd

using namespace pfd;

extern "C" PFD_API int pfd_flash_attn_strided_f16(const void* q, const void* k, const void* vt, void* out,
                                                  int32_t B, int32_t heads, int32_t Nq, int32_t Nk, int32_t d,
                                                  const int64_t* q_strides, const int64_t* k_strides,
                                                  const int64_t* vt_strides, float scale, int64_t o_sb,
                                                  int64_t o_sq, void* stream) {
  if (d % 8 || d <= 0 || d > 192) return set_error("pfd_flash_attn_f16: head dim %d unsupported", d);
  if (Nq <= 0 || Nk <= 0) return set_error("pfd_flash_attn_f16: empty problem");
  for (int i = 0; i < 3; ++i)
    if (q_strides[i] % 8 || k_strides[i] % 8 || vt_strides[i] % 8)
      return set_error("pfd_flash_attn_f16: strides must be multiples of 8 elements");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  FlashParams p;
  memset(&p, 0, sizeof(p));
  // strides = {batch, head, row} in elements; q/k rows run over d, vt rows (one per channel) run over the keys
  if (int rc = encode4d(&p.tmQ, q, d, Nq, heads, B, q_strides[2], q_strides[1], q_strides[0], FA_BQ, "Q")) return rc;
  if (int rc = encode4d(&p.tmK, k, d, Nk, heads, B, k_strides[2], k_strides[1], k_strides[0], FA_BKV, "K")) return rc;
  if (int rc = encode4d(&p.tmV, vt, Nk, d, heads, B, vt_strides[2], vt_strides[1], vt_strides[0], (cuuint32_t)d, "V^T")) return rc;
  p.Nq = Nq; p.Nk = Nk; p.heads = heads; p.d = d;
  p.nblk = (Nk + FA_BKV - 1) / FA_BKV;
  p.scale = scale;
  p.out = static_cast<__half*>(out);
  p.o_sb = o_sb; p.o_sq = o_sq; p.o_sh = d;
  dim3 grid((Nq + FA_BQ - 1) / FA_BQ, (unsigned)((long long)B * heads));
  switch ((d + 15) / 16) {
    case 1: return launch_flash<1, 16>(p, grid, st);
    case 2: return launch_flash<1, 32>(p, grid, st);
    case 3: return launch_flash<1, 48>(p, grid, st);
    case 4: return launch_flash<1, 64>(p, grid, st);
    case 5: return launch_flash<2, 80>(p, grid, st);
    case 6: return launch_flash<2, 96>(p, grid, st);
    case 7: return launch_flash<2, 112>(p, grid, st);
    case 8: return launch_flash<2, 128>(p, grid, st);
    case 9: return launch_flash<3, 144>(p, grid, st);
    case 10: return launch_flash<3, 160>(p, grid, st);
    case 11: return launch_flash<3, 176>(p, grid, st);
    default: return launch_flash<3, 192>(p, grid, st);
  }
}

extern "C" PFD_API int pfd_flash_attn_f16(const void* q, const void* k, const void* vt, void* out, int32_t B,
                                          int32_t heads, int32_t Nq, int32_t Nk, int32_t d, int32_t q_rows,
                                          int32_t k_rows, float scale, int64_t vt_pitch, int64_t o_sb,
                                          int64_t o_sq, int32_t reserved, void* stream) {
  (void)reserved;
  // packed layouts: q [B*heads, q_rows, d], k [B*heads, k_rows, d], vt [B*heads, d, vt_pitch]
  const int64_t qs[3] = {(int64_t)heads * q_rows * d, (int64_t)q_rows * d, d};
  const int64_t ks[3] = {(int64_t)heads * k_rows * d, (int64_t)k_rows * d, d};
  const int64_t vs[3] = {(int64_t)heads * d * vt_pitch, (int64_t)d * vt_pitch, vt_pitch};
  return pfd_flash_attn_strided_f16(q, k, vt, out, B, heads, Nq, Nk, d, qs, ks, vs, scale, o_sb, o_sq, stream);
}
