// wgmma tensor-core contraction for sm_90a: one persistent, warp-specialised kernel that serves
// every Linear / 1x1 conv / 3x3 conv (implicit GEMM; TMA performs the im2col gather with
// zero-filled halos) / batched QK^T and PV product on the Prompt-Free-Diffusion hot path.
//
//   D[128 x BN] (fp32, registers)  +=  A[128 x 64] (fp16, smem, TMA 4-D box)  x  B[BN x 64]^T (fp16, smem)
//
// Roles (384 threads): warpgroup 0 = TMA producer (thread 0) and three store warps (warps 1-3); warpgroups 1 and 2 =
// wgmma consumers, each owning 64 rows of the tile.  After a tile's MMAs the consumers apply the fused epilogue
// (bias / time-embedding / activation / GEGLU) and write the fp16 tile to a shared-memory staging buffer, then go on
// to the next tile's K blocks; the store warps add the residual and write the tile to global memory with 16-byte
// stores while those MMAs run (gemm_stage_tile / gemm_store_tile, barriers c_full / c_empty).  Split-K partials and
// element-strided outputs keep the direct epilogue from the registers (gemm_epilogue).  The producer runs ahead
// through a ring of shared-memory stages, so the loads of tile i+1 overlap the epilogue of tile i.  See
// include/pfd_b200.h (pfd_gemm_f16) for the reference call sites this replaces.
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

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int WG_K = 16;
constexpr int GEMM_THREADS = 384;           // producer warpgroup + 2 consumer warpgroups
constexpr int STAGE_A_BYTES = BM * BK * 2;  // 16 KiB
constexpr int SMEM_BUDGET = 232448;         // 227 KiB opt-in limit per CTA
constexpr int SMEM_FIXED = 1024 + 256;      // alignment slack + barriers

struct alignas(64) GemmParams {
  CUtensorMap tmA[PFD_MAX_SEG];
  CUtensorMap tmB;
  int nseg;
  int taps[PFD_MAX_SEG];
  int chunks[PFD_MAX_SEG];
  int a_c[PFD_MAX_SEG];
  int stride;
  int tap_off;
  int bw, bh, bn;
  int tiles_w, tiles_h, tiles_nb, n_tiles;
  int W, H, NB, N;
  int b_batched;
  int num_kb;
  int splits;        // split-K factor (1 = off); work items = tiles * splits
  int kb_per_split;
  float* ws;         // fp32 partials [splits][m_tiles*128][N] when splits > 1
  float alpha;
  int act;
  const __half* bias;
  const __half* rowadd;
  const __half* residual;
  __half* out;
  long long so_n1, so_n0, so_y, so_x, so_c1, so_c0;
  long long rowadd_ld;
  int ndiv, cdiv;
  int vec_ok;
};

constexpr int STORE_THREADS = 96;           // warps 1-3 of the producer warpgroup

template <int BN>
struct GemmCfg {
  static constexpr int STAGE_B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = STAGE_A_BYTES + STAGE_B_BYTES;
  // staged fp16 output tile: rows padded by 16 B, so the 8 rows x 4 lanes of a warp's half2 fragment writes fall on
  // 32 distinct banks; followed by the store warps' output row offsets of two consecutive tiles
  static constexpr int C_PITCH = BN * 2 + 16;
  static constexpr int C_BYTES = BM * C_PITCH + 2 * BM * 8;
  static constexpr int RAW_STAGES = (SMEM_BUDGET - SMEM_FIXED - C_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = RAW_STAGES > 8 ? 8 : RAW_STAGES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + C_BYTES + SMEM_FIXED;
  // Register budgets (setmaxnreg) of the two roles.  The CTA starts with 168 per thread (__launch_bounds__(384, 1)),
  // so 128 PRODUCER_REGS + 256 CONSUMER_REGS = 384 x 168.  The producer warpgroup's budget bounds the store warps'
  // STORE_BATCH (16-byte chunks per thread whose residual loads are in flight at once); the 256-wide tile's consumers
  // hold 128 fp32 accumulators, so they get the larger budget.
  static constexpr int CONSUMER_REGS = BN >= 256 ? 224 : 208;
  static constexpr int PRODUCER_REGS = BN >= 256 ? 56 : 88;
  static constexpr int STORE_BATCH = BN >= 256 ? 4 : 8;
  // The consumers load a tile's bias before its K loop, so the latency lies under the MMAs.  Not at BN = 256: 128
  // accumulators plus 32 bias registers spill within CONSUMER_REGS, so there the loads follow the MMAs.
  static constexpr bool BIAS_EARLY = BN < 256;
  static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS == GEMM_THREADS * 168, "register budgets");
  static_assert(STAGE_B_BYTES % 1024 == 0, "B stage must keep 1024-B swizzle alignment");
  static_assert(BN % 16 == 0 && BN >= 16 && BN <= 256, "wgmma N constraint");
  static_assert(STAGES == (BN <= 64 ? 8 : BN <= 160 ? 5 : BN <= 192 ? 4 : 3), "pipeline depth per N tile");
};

// erf to ~1.5e-7 absolute (Abramowitz & Stegun 7.1.26) with MUFU rcp/ex2: about half the
// instructions of erff(), far below the fp16 output resolution of the GELU / GEGLU epilogues.
__device__ __forceinline__ float fast_erf(float x) {
  const float ax = fabsf(x);
  const float t = __fdividef(1.f, fmaf(0.3275911f, ax, 1.f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  const float y = 1.f - poly * __expf(-ax * ax);
  return copysignf(y, x);
}

// GELU as x * sigmoid(x * (a + b x^2 + c x^4)), coefficients fitted to the exact erf form on [-8, 8]
// (max |error| 2.5e-5, tools/fit_gelu.py; fp16 resolution near 1 is 4.9e-4).  The polynomial is evaluated on
// clamp(x, +-10) because c < 0 would flip its sign beyond |x| = 11.1; at |x| = 10 the sigmoid is already 0 / 1
// to 3e-9.  9 FMA-pipe instructions + 2 MUFU per element against ~17 + 2 for the A&S erf form.
// Outside [-8, 8] the error of x * sigmoid(...) against the exact GELU is below 3e-8 up to |x| = 10; beyond, the
// clamped sigmoid is off by at most 3e-9, so the error is below 3e-9 |x| (1.9e-4 at x = -65504, where GELU is 0).
__device__ __forceinline__ float gelu_sig(float x) {
  const float xc = fminf(fmaxf(x, -10.f), 10.f);
  const float x2 = xc * xc;
  // coefficients pre-multiplied by -log2(e)
  const float pl = fmaf(x2, fmaf(x2, 1.01426305e-3f, -1.06775723e-1f), -2.30112135f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(xc * pl));
  return __fdividef(x, 1.f + e);
}

__device__ __forceinline__ float act_apply(float v, int act) {
  if (act == PFD_ACT_SILU) return __fdividef(v, 1.f + __expf(-v));
  if (act == PFD_ACT_GELU) return 0.5f * v * (1.f + fast_erf(v * 0.70710678118654752f));
  if (act == PFD_ACT_RELU) return fmaxf(v, 0.f);
  return v;
}

__device__ __forceinline__ float h2lo(uint32_t u) { return __low2float(*reinterpret_cast<const __half2*>(&u)); }
__device__ __forceinline__ float h2hi(uint32_t u) { return __high2float(*reinterpret_cast<const __half2*>(&u)); }
__device__ __forceinline__ uint32_t ldg_h2(const __half* p) { return __ldg(reinterpret_cast<const unsigned int*>(p)); }

// The epilogue arithmetic of every output path (staged tile, direct epilogue, split-K finish).  Each path rounds these
// values to fp16 before it adds the residual in fp16.
//
// act(acc * alpha + bias [+ row add]) of an adjacent column pair (lo, hi), in fp32.  The per-image row add (time
// embedding) comes after the bias and before the activation, the reference's (conv + bias) + emb -> act.
// bias and ra hold the fp16 pairs of the bias and the row add.
__device__ __forceinline__ void epi_pair(float& lo, float& hi, float alpha, uint32_t bias, bool rowadd, uint32_t ra,
                                         int act) {
  lo = fmaf(lo, alpha, h2lo(bias));
  hi = fmaf(hi, alpha, h2hi(bias));
  if (rowadd) {
    lo += h2lo(ra);
    hi += h2hi(ra);
  }
  if (act != PFD_ACT_NONE) {
    lo = act_apply(lo, act);
    hi = act_apply(hi, act);
  }
}

// GEGLU output pair fp16(value) * fp16(gelu(fp16(gate))), value and gate each acc * alpha + bias.  The reference's
// x, gate = proj(x).chunk(2) are fp16 tensors, and it computes x * gelu(gate) in fp16 (attention.py:50-51).
// bv and bg hold the fp16 bias pairs of value and gate.
__device__ __forceinline__ __half2 geglu_pair(const float* v, const float* g, float alpha, uint32_t bv, uint32_t bg) {
  const __half2 a = __floats2half2_rn(fmaf(v[0], alpha, h2lo(bv)), fmaf(v[1], alpha, h2hi(bv)));
  const float2 gf = __half22float2(__floats2half2_rn(fmaf(g[0], alpha, h2lo(bg)), fmaf(g[1], alpha, h2hi(bg))));
  return __hmul2(a, __floats2half2_rn(gelu_sig(gf.x), gelu_sig(gf.y)));
}

// One unit of work of a persistent CTA: K blocks [kb0, kb1) of output tile `tile`, the whole contraction of the tile
// or, with split-K, slice `slot`.
struct WorkItem {
  int tile, kb0, kb1, slot;
};
__device__ __forceinline__ bool gemm_work(const GemmParams& p, int wi, int total_tiles, WorkItem& w) {
  const int G = gridDim.x, c = blockIdx.x;
  const int work = c + wi * G;
  if (work >= total_tiles * p.splits) return false;
  w.tile = work % total_tiles;
  w.slot = work / total_tiles;
  w.kb0 = w.slot * p.kb_per_split;
  w.kb1 = min(p.num_kb, w.kb0 + p.kb_per_split);
  return true;
}

// Origin of an M tile in the output raster.  The 128 rows of a tile are a bw x bh x bn box of pixels, all three
// powers of two (pfd_gemm_f16), so a tile row splits into (x, y, image) with shifts: lbw = log2(bw), lbh = log2(bh).
struct TileOrigin {
  int x0, y0, n0, lbw, lbh;
};
__device__ __forceinline__ TileOrigin tile_origin(const GemmParams& p, int m_tile) {
  TileOrigin o;
  o.x0 = (m_tile % p.tiles_w) * p.bw;
  o.y0 = ((m_tile / p.tiles_w) % p.tiles_h) * p.bh;
  o.n0 = (m_tile / (p.tiles_w * p.tiles_h)) * p.bn;
  o.lbw = __ffs(p.bw) - 1;
  o.lbh = __ffs(p.bh) - 1;
  return o;
}
// Position of a tile row in the output raster: (x, y, image n) and whether it lies inside the raster.
struct TileRow {
  int x, y, n;
  bool valid;
};
__device__ __forceinline__ TileRow tile_row(const GemmParams& p, const TileOrigin& o, int row) {
  TileRow r;
  r.x = o.x0 + (row & (p.bw - 1));
  r.y = o.y0 + ((row >> o.lbw) & (p.bh - 1));
  r.n = o.n0 + (row >> (o.lbw + o.lbh));
  r.valid = (r.x < p.W) && (r.y < p.H) && (r.n < p.NB);
  return r;
}
__device__ __forceinline__ long long out_row_off(const GemmParams& p, const TileRow& r) {
  return (long long)(r.n / p.ndiv) * p.so_n1 + (long long)(r.n % p.ndiv) * p.so_n0 + (long long)r.y * p.so_y +
         (long long)r.x * p.so_x;
}
__device__ __forceinline__ long long out_col_off(const GemmParams& p, int c) {
  return p.cdiv >= p.N ? (long long)c * p.so_c0 : (long long)(c / p.cdiv) * p.so_c1 + (long long)(c % p.cdiv) * p.so_c0;
}

// Accumulator fragment of a consumer warpgroup (rows [64 cw, 64 cw + 64) of the tile): thread (warp wl, lane l) holds
// rows 16 wl + l/4 (+ 8) and, for every 8-column group j, the column pair 8j + 2 (l % 4) (+ 1): acc[4j + {0, 1}] for
// the first row, acc[4j + {2, 3}] for the second.
//
// Bias of a thread's BN / 8 column pairs of tile `tile`.  The consumers issue these loads before the tile's K loop, so
// their latency lies under the MMAs.  A GEGLU tile is packed [value(BN/2) | gate(BN/2)] in weights and bias alike
// (pack_geglu), so element j is the value bias of pair j for j < BN / 16 and the gate bias of pair j - BN / 16 after.
template <int BN>
__device__ __forceinline__ void gemm_load_bias(const GemmParams& p, int tile, uint32_t (&bias)[BN / 8]) {
  const int col0 = (tile % p.n_tiles) * BN + 2 * (threadIdx.x & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) bias[j] = (p.bias && col0 + 8 * j < p.N) ? ldg_h2(p.bias + col0 + 8 * j) : 0u;
}

// Staged epilogue (every tile with 16-byte addressable output columns, vec_ok, and no split-K): the consumers write
// the tile's fp16 values into the shared-memory buffer `cbuf` (row pitch C_PITCH) and go on to the next tile; the
// store warps (gemm_store_tile) add the residual and write the rows to global memory.
//   * GEGLU: fp16(value) * fp16(gelu(fp16(gate))) in columns [0, BN/2) of the buffer;
//   * otherwise fp16(act(acc * alpha + bias + row add)).
// The row-add loads of a block of column groups are all issued before any of them is used.
template <int BN, bool GEGLU>
__device__ __forceinline__ void gemm_stage_tile(const GemmParams& p, const float (&acc)[BN / 2],
                                                const uint32_t (&bias)[BN / 8], int cw, int tile, uint8_t* cbuf) {
  constexpr int C_PITCH = GemmCfg<BN>::C_PITCH;
  const int wl = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int n_tile = tile % p.n_tiles;
  const TileOrigin org = tile_origin(p, tile / p.n_tiles);
  const int n_out = GEGLU ? p.N / 2 : p.N;
  const int col_base = n_tile * (GEGLU ? BN / 2 : BN);
  const int cq = 2 * (lane & 3);
  int rows[2];
  bool valid[2];
  const __half* rowadd_row[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    rows[i] = cw * 64 + wl * 16 + (lane >> 2) + 8 * i;
    const TileRow r = tile_row(p, org, rows[i]);
    valid[i] = r.valid;
    rowadd_row[i] = (p.rowadd && r.valid) ? p.rowadd + (long long)r.n * p.rowadd_ld : nullptr;
  }
  auto put = [&](int i, int c, __half2 h) {
    *reinterpret_cast<__half2*>(cbuf + rows[i] * C_PITCH + c * 2) = h;
  };
  const float alpha = p.alpha;
  if (GEGLU) {
#pragma unroll
    for (int j = 0; j < BN / 16; ++j) {
      const int c = 8 * j + cq;               // value column inside the tile; its gate is column c + BN / 2
      if (col_base + c >= n_out) continue;
      const uint32_t bv = bias[j], bg = bias[j + BN / 16];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (!valid[i]) continue;
        put(i, c, geglu_pair(&acc[4 * j + 2 * i], &acc[4 * (j + BN / 16) + 2 * i], alpha, bv, bg));
      }
    }
    return;
  }
  const int act = p.act;
  constexpr int JB = (BN / 8) % 8 == 0 ? 8 : 4;   // column groups per block of loads
#pragma unroll
  for (int j0 = 0; j0 < BN / 8; j0 += JB) {
    uint32_t ra[2][JB];
#pragma unroll
    for (int jj = 0; jj < JB; ++jj) {
      const int col = col_base + 8 * (j0 + jj) + cq;
#pragma unroll
      for (int i = 0; i < 2; ++i) ra[i][jj] = (rowadd_row[i] && col < n_out) ? ldg_h2(rowadd_row[i] + col) : 0u;
    }
#pragma unroll
    for (int jj = 0; jj < JB; ++jj) {
      const int j = j0 + jj;
      if (col_base + 8 * j + cq >= n_out) continue;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (!valid[i]) continue;
        float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
        epi_pair(v0, v1, alpha, bias[j], rowadd_row[i] != nullptr, ra[i][jj], act);
        put(i, 8 * j + cq, __floats2half2_rn(v0, v1));
      }
    }
  }
}

// Store warps (warps 1-3 of warpgroup 0): write one staged tile from `cbuf` to its output rows in 16-byte chunks and
// add the residual in fp16 - the reference's `x + f(h)` on fp16 tensors.  A row has CPR chunks, a compile-time number,
// and a thread keeps ONE chunk column for the whole tile: CPR threads share a row, a pass covers 96 / CPR rows, and the
// 96 % CPR threads left over idle (16 of 96 at BN = 160, 6 at its GEGLU half).  So the column offset - with the head
// split's division - is computed once per tile, and the rows of a thread advance by a constant step.  When the tile
// is 128 consecutive pixels of one raster line (bw = 128: every Linear), a row's offset is the tile's plus row * so_x;
// other tiles (convolutions) look it up in `rowoff`, filled first (one of two buffers used by alternate tiles).
// Each thread issues the residual loads of STORE_BATCH passes before any of their stores; the first batch is loaded
// before waiting for the consumers to fill the buffer (`c_full`, phase `parity`).
template <int BN, bool GEGLU>
__device__ __forceinline__ void gemm_store_tile(const GemmParams& p, int tile, const uint8_t* cbuf, long long* rowoff,
                                                uint32_t c_full, uint32_t parity) {
  constexpr int C_PITCH = GemmCfg<BN>::C_PITCH;
  constexpr int STORE_BATCH = GemmCfg<BN>::STORE_BATCH;
  constexpr int CPR = (GEGLU ? BN / 2 : BN) / 8;      // 16-byte chunks per tile row
  constexpr int RPP = STORE_THREADS / CPR;            // rows per pass
  constexpr int NPASS = (BM + RPP - 1) / RPP;
  const int t = threadIdx.x - 32;
  const int n_tile = tile % p.n_tiles;
  const TileOrigin org = tile_origin(p, tile / p.n_tiles);
  const bool line_tile = p.bw == BM;    // bh = bn = 1: the tile lies on raster line y0 of image n0, both in the raster
  if (!line_tile) {
#pragma unroll 1
    for (int row = t; row < BM; row += STORE_THREADS) {
      const TileRow r = tile_row(p, org, row);
      rowoff[row] = r.valid ? out_row_off(p, r) : -1;
    }
    asm volatile("bar.sync 2, %0;" ::"n"(STORE_THREADS) : "memory");
  }
  const int ch = t % CPR, r0 = t / CPR;
  const int col = n_tile * CPR * 8 + 8 * ch;
  const bool col_ok = r0 < RPP && col < (GEGLU ? p.N / 2 : p.N);
  const long long col_off = out_col_off(p, col);
  const bool add_res = p.residual && !GEGLU;
  const uint8_t* const src = cbuf + r0 * C_PITCH + ch * 16;

  // row_off(row): element offset of (row, this thread's chunk) in the output, or -1 outside the raster.  It is cheap
  // enough to be evaluated again at the store, which keeps the offsets of a batch out of the registers.
  auto store_rows = [&](auto row_off) {
    uint4 res[STORE_BATCH];
    auto load_batch = [&](int pass0) {
#pragma unroll
      for (int b = 0; b < STORE_BATCH; ++b) {
        const int row = r0 + (pass0 + b) * RPP;
        const long long off = (col_ok && row < BM) ? row_off(row) : -1;
        if (off >= 0) res[b] = __ldg(reinterpret_cast<const uint4*>(p.residual + off));
      }
    };
    if (add_res) load_batch(0);
    mbar_wait(c_full, parity);
#pragma unroll 1
    for (int pass0 = 0; pass0 < NPASS; pass0 += STORE_BATCH) {
#pragma unroll
      for (int b = 0; b < STORE_BATCH; ++b) {
        const int row = r0 + (pass0 + b) * RPP;
        const long long off = (col_ok && row < BM) ? row_off(row) : -1;
        if (off < 0) continue;
        uint4 v = *reinterpret_cast<const uint4*>(src + (pass0 + b) * (RPP * C_PITCH));
        if (add_res) {
          __half2* h = reinterpret_cast<__half2*>(&v);
          const __half2* r = reinterpret_cast<const __half2*>(&res[b]);
#pragma unroll
          for (int k = 0; k < 4; ++k) h[k] = __hadd2(h[k], r[k]);
        }
        *reinterpret_cast<uint4*>(p.out + off) = v;
      }
      if (add_res && pass0 + STORE_BATCH < NPASS) load_batch(pass0 + STORE_BATCH);
    }
  };

  if (line_tile) {
    const int rows_in = p.W - org.x0;
    TileRow first;
    first.x = org.x0; first.y = org.y0; first.n = org.n0;
    const long long base = out_row_off(p, first) + col_off;
    const long long so_x = p.so_x;
    store_rows([&](int row) { return row < rows_in ? base + row * so_x : -1ll; });
  } else {
    store_rows([&](int row) {
      const long long ro = rowoff[row];
      return ro >= 0 ? ro + col_off : -1ll;
    });
  }
}

// Direct epilogue from the accumulator registers, for the tiles the staged epilogue does not take:
//   * split-K slice: raw fp32 partials -> workspace (bias etc. in splitk_finish_kernel);
//   * element-strided outputs (V^T, !vec_ok): as gemm_stage_tile + gemm_store_tile, with scalar stores.
template <int BN>
__device__ __forceinline__ void gemm_epilogue(const GemmParams& p, const float (&acc)[BN / 2], int cw, int tile,
                                              int split, int m_tiles) {
  const int wl = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int n_tile = tile % p.n_tiles;
  const int m_tile = tile / p.n_tiles;
  const TileOrigin org = tile_origin(p, m_tile);
  const bool geglu = (p.act == PFD_ACT_GEGLU);
  const int n_out = geglu ? p.N / 2 : p.N;
  const int col_base = n_tile * (geglu ? BN / 2 : BN);
  const int cq = 2 * (lane & 3);
  int rows[2];
  bool valid[2];
  long long row_off[2];
  const __half* rowadd_row[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = cw * 64 + wl * 16 + (lane >> 2) + 8 * i;
    rows[i] = row;
    const TileRow r = tile_row(p, org, row);
    valid[i] = r.valid;
    row_off[i] = out_row_off(p, r);
    rowadd_row[i] = (p.rowadd && valid[i]) ? p.rowadd + (long long)r.n * p.rowadd_ld : nullptr;
  }
  // (lo, hi) -> fp16 output columns c, c + 1 of row i; the residual is added to the fp16 values, as the store warps do
  auto store2 = [&](int i, int c, float lo, float hi) {
    const long long o0 = row_off[i] + out_col_off(p, c);
    const long long o1 = row_off[i] + out_col_off(p, c + 1);
    __half h0 = __float2half_rn(lo), h1 = __float2half_rn(hi);
    if (p.residual) {
      h0 = __hadd(h0, p.residual[o0]);
      h1 = __hadd(h1, p.residual[o1]);
    }
    p.out[o0] = h0;
    p.out[o1] = h1;
  };

  if (p.splits > 1) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float* wrow = p.ws + ((long long)split * m_tiles * BM + (long long)m_tile * BM + rows[i]) * p.N;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = col_base + 8 * j + cq;
        if (col < p.N) *reinterpret_cast<float2*>(wrow + col) = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
      }
    }
    return;
  }
  const float alpha = p.alpha;
  if (geglu) {
#pragma unroll
    for (int j = 0; j < BN / 16; ++j) {
      const int c = 8 * j + cq;               // value column inside the tile; its gate is column c + BN / 2
      const int col = col_base + c;
      if (col >= n_out) continue;
      uint32_t bv = 0u, bg = 0u;
      if (p.bias) {
        bv = ldg_h2(p.bias + (long long)n_tile * BN + c);
        bg = ldg_h2(p.bias + (long long)n_tile * BN + BN / 2 + c);
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (!valid[i]) continue;
        const float2 of = __half22float2(
            geglu_pair(&acc[4 * j + 2 * i], &acc[4 * (j + BN / 16) + 2 * i], alpha, bv, bg));
        store2(i, col, of.x, of.y);
      }
    }
    return;
  }
  const int act = p.act;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = col_base + 8 * j + cq;
    if (col >= n_out) continue;
    const uint32_t b = p.bias ? ldg_h2(p.bias + col) : 0u;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (!valid[i]) continue;
      const uint32_t r = rowadd_row[i] ? ldg_h2(rowadd_row[i] + col) : 0u;
      float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
      epi_pair(v0, v1, alpha, b, rowadd_row[i] != nullptr, r, act);
      store2(i, col, v0, v1);
    }
  }
}

template <int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ GemmParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];

  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;
  const uint32_t smemA = base;                                        // [STAGES][A tile]
  const uint32_t smemB = base + STAGES * STAGE_A_BYTES;               // [STAGES][B tile]
  const uint32_t cbuf_off = base - raw_addr + STAGES * Cfg::STAGE_BYTES;
  uint8_t* const cbuf = smem_raw + cbuf_off;                          // staged output tile [BM][C_PITCH]
  long long* const rowoff = reinterpret_cast<long long*>(cbuf + BM * Cfg::C_PITCH);   // [2][BM]
  const uint32_t bars = base + STAGES * Cfg::STAGE_BYTES + Cfg::C_BYTES;
  // barrier layout: full[STAGES] | empty[STAGES] | c_full | c_empty
  auto full_bar = [&](int s) { return bars + 8u * s; };
  auto empty_bar = [&](int s) { return bars + 8u * (STAGES + s); };
  const uint32_t c_full = bars + 16u * STAGES, c_empty = c_full + 8u;

  const int wg = threadIdx.x >> 7;
  // staged epilogue for every tile of the launch (see gemm_stage_tile)
  const bool staged = p.vec_ok && p.splits == 1;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nseg; ++s) tma_prefetch_desc(&p.tmA[s]);
    tma_prefetch_desc(&p.tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);           // one arrival per consumer warp
    }
    mbar_init(c_full, 8);                   // one arrival per consumer warp
    mbar_init(c_empty, STORE_THREADS / 32); // one arrival per store warp
    mbar_fence_init();
  }
  __syncthreads();
  // prologue above overlapped the previous kernel's tail; global data may only be touched from here on
  pdl_wait();
  pdl_launch_dependents();

  const int m_tiles = p.tiles_w * p.tiles_h * p.tiles_nb;
  const int total_tiles = m_tiles * p.n_tiles;

  if (wg == 0) {
    // ------------------------------------------------------------ TMA producer (thread 0) + store warps (warps 1-3)
    setmaxnreg_dec<Cfg::PRODUCER_REGS>();
    if (threadIdx.x >= 32 && staged) {
      uint32_t c_phase = 0;
      WorkItem w;
      for (int wi = 0; gemm_work(p, wi, total_tiles, w); ++wi) {
        if (p.act == PFD_ACT_GEGLU) gemm_store_tile<BN, true>(p, w.tile, cbuf, rowoff + (c_phase ? BM : 0), c_full, c_phase);
        else gemm_store_tile<BN, false>(p, w.tile, cbuf, rowoff + (c_phase ? BM : 0), c_full, c_phase);
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mbar_arrive(c_empty);
        c_phase ^= 1u;
      }
    } else if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      WorkItem w;
      for (int wi = 0; gemm_work(p, wi, total_tiles, w); ++wi) {
        const int tile = w.tile, kb_begin = w.kb0, kb_end = w.kb1;
        const int n_tile = tile % p.n_tiles;
        const int m_tile = tile / p.n_tiles;
        const int tx = m_tile % p.tiles_w;
        const int ty = (m_tile / p.tiles_w) % p.tiles_h;
        const int tn = m_tile / (p.tiles_w * p.tiles_h);
        const int x0 = tx * p.bw * p.stride;
        const int y0 = ty * p.bh * p.stride;
        const int n0 = tn * p.bn;
        const int bcoord = p.b_batched ? n0 : 0;
        int kofs = 0;
        int kbi = 0;
        for (int s = 0; s < p.nseg; ++s) {
          const int ntap = p.taps[s];
          for (int t = 0; t < ntap; ++t) {
            const int dy = (ntap == 9) ? (t / 3 - 1 + p.tap_off) : 0;
            const int dx = (ntap == 9) ? (t % 3 - 1 + p.tap_off) : 0;
            for (int j = 0; j < p.chunks[s]; ++j, ++kbi) {
              if (kbi < kb_begin || kbi >= kb_end) continue;
              mbar_wait(empty_bar(stage), phase ^ 1u);
              mbar_expect_tx(full_bar(stage), Cfg::STAGE_BYTES);
              tma_load_4d(smemA + stage * STAGE_A_BYTES, &p.tmA[s], full_bar(stage), j * BK, x0 + dx, y0 + dy, n0);
              tma_load_3d(smemB + stage * Cfg::STAGE_B_BYTES, &p.tmB, full_bar(stage), kofs + j * BK, n_tile * BN,
                          bcoord);
              if (++stage == STAGES) {
                stage = 0;
                phase ^= 1u;
              }
            }
            kofs += p.a_c[s];
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------ wgmma consumers (64 rows each) + epilogue
    setmaxnreg_inc<Cfg::CONSUMER_REGS>();
    const int cw = wg - 1;
    const bool arrive_lane = (threadIdx.x & 31) == 0;
    int stage = 0;
    uint32_t phase = 0, c_phase = 0;
    float acc[BN / 2];
    WorkItem w;
    for (int wi = 0; gemm_work(p, wi, total_tiles, w); ++wi) {
      const int nkb = w.kb1 - w.kb0;
      uint32_t bias[BN / 8];
      if (Cfg::BIAS_EARLY && staged) gemm_load_bias<BN>(p, w.tile, bias);
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(full_bar(stage), phase);
        const uint64_t adesc = make_sw128_kmajor_desc(smemA + stage * STAGE_A_BYTES + cw * 64 * 128);
        const uint64_t bdesc = make_sw128_kmajor_desc(smemB + stage * Cfg::STAGE_B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / WG_K; ++k)
          Wgmma<BN>::ss(acc, adesc + 2u * k, bdesc + 2u * k, (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        // keep one group in flight: the stage read by the previous group may now be refilled
        wgmma_wait<1>();
        if (prev >= 0 && arrive_lane) mbar_arrive(empty_bar(prev));
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1u;
        }
      }
      wgmma_wait<0>();
      if (prev >= 0 && arrive_lane) mbar_arrive(empty_bar(prev));
      if (staged) {
        if (!Cfg::BIAS_EARLY) gemm_load_bias<BN>(p, w.tile, bias);
        mbar_wait(c_empty, c_phase ^ 1u);   // the store warps have read the previous tile out of the buffer
        if (p.act == PFD_ACT_GEGLU) gemm_stage_tile<BN, true>(p, acc, bias, cw, w.tile, cbuf);
        else gemm_stage_tile<BN, false>(p, acc, bias, cw, w.tile, cbuf);
        __syncwarp();
        if (arrive_lane) mbar_arrive(c_full);
        c_phase ^= 1u;
      } else {
        gemm_epilogue<BN>(p, acc, cw, w.tile, w.slot, m_tiles);
      }
    }
  }
}

// Split-K second pass: sum the fp32 partials of all splits and apply the fused epilogue
// (bias, per-image row add, activation, residual) with the same generic output addressing.
__global__ void __launch_bounds__(256)
splitk_finish_kernel(const __grid_constant__ GemmParams p) {
  pdl_wait();
  pdl_launch_dependents();
  const int m_tiles = p.tiles_w * p.tiles_h * p.tiles_nb;
  const long long rows_pad = (long long)m_tiles * BM;
  const int vecs = p.N / 8;
  const long long total = rows_pad * vecs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vecs);
    const long long prow = i / vecs;
    const TileRow r = tile_row(p, tile_origin(p, (int)(prow / BM)), (int)(prow % BM));
    if (!r.valid) continue;
    const int col = v * 8;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int s = 0; s < p.splits; ++s) {
      const float4* src = reinterpret_cast<const float4*>(p.ws + ((long long)s * rows_pad + prow) * p.N + col);
      const float4 a = __ldg(src), b = __ldg(src + 1);
      acc[0] += a.x; acc[1] += a.y; acc[2] += a.z; acc[3] += a.w;
      acc[4] += b.x; acc[5] += b.y; acc[6] += b.z; acc[7] += b.w;
    }
    uint4 bv = make_uint4(0, 0, 0, 0), rv = bv;
    if (p.bias) bv = __ldg(reinterpret_cast<const uint4*>(p.bias + col));
    if (p.rowadd) rv = __ldg(reinterpret_cast<const uint4*>(p.rowadd + (long long)r.n * p.rowadd_ld + col));
    const uint32_t* b2 = &bv.x;
    const uint32_t* r2 = &rv.x;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      epi_pair(acc[2 * k], acc[2 * k + 1], p.alpha, b2[k], p.rowadd != nullptr, r2[k], p.act);
    // fp16(act(...)), then the residual added in fp16: the same rounding as the staged epilogue
    const long long row_off = out_row_off(p, r);
    if (p.vec_ok) {
      const long long off = row_off + out_col_off(p, col);
      uint4 o;
      __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
      for (int k = 0; k < 4; ++k) oh[k] = __floats2half2_rn(acc[2 * k], acc[2 * k + 1]);
      if (p.residual) {
        const uint4 res = __ldg(reinterpret_cast<const uint4*>(p.residual + off));
        const __half2* rh = reinterpret_cast<const __half2*>(&res);
#pragma unroll
        for (int k = 0; k < 4; ++k) oh[k] = __hadd2(oh[k], rh[k]);
      }
      *reinterpret_cast<uint4*>(p.out + off) = o;
    } else {
      // column by column: a head width (cdiv) that is not a multiple of 8 splits the 8 columns between two heads
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const long long off = row_off + out_col_off(p, col + k);
        __half h = __float2half_rn(acc[k]);
        if (p.residual) h = __hadd(h, p.residual[off]);
        p.out[off] = h;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ host
// Size of the split-K workspace, which also bounds the partials of a split-K plan.  It decides which shapes are split
// and so the bits of their results: keep it at 64 MiB - 4 KiB.
constexpr size_t SPLITK_WS_BYTES = (64ull << 20) - 4096;

static inline long long cdivll(long long a, long long b) { return (a + b - 1) / b; }

template <int BN>
static int launch_gemm(const GemmParams& p, int grid, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  static int trace = -1;
  if (trace < 0) {
    const char* e = getenv("PFD_GEMM_TRACE");
    trace = (e && e[0] == '1') ? 1 : 0;
  }
  if (trace)   // one line per launch
    fprintf(stderr, "GEMMTRACE M=%lld N=%d K=%d nseg=%d taps=%d stride=%d act=%d bias=%d res=%d rowadd=%d BN=%d "
            "splits=%d grid=%d batched=%d vec=%d plain=%d\n", (long long)p.W * p.H * p.NB, p.N, p.num_kb * BK,
            p.nseg, p.taps[0], p.stride, p.act, p.bias != nullptr, p.residual != nullptr, p.rowadd != nullptr, BN,
            p.splits, grid, p.b_batched, p.vec_ok, (int)(p.cdiv >= p.N));
  if (int rc = smem_opt_in<gemm_wgmma_kernel<BN>>(Cfg::SMEM_BYTES, "gemm_wgmma_kernel")) return rc;
  launch_k(gemm_wgmma_kernel<BN>, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, stream, p);
  return check_launch("pfd_gemm_f16");
}

}  // namespace pfd

using namespace pfd;

extern "C" PFD_API int pfd_gemm_f16(const pfd_gemm_desc* d) {
  if (!d) return set_error("pfd_gemm_f16: null descriptor");
  if (d->nseg < 1 || d->nseg > PFD_MAX_SEG) return set_error("pfd_gemm_f16: nseg %d out of range", d->nseg);
  if (d->N <= 0 || d->N % 8) return set_error("pfd_gemm_f16: N=%d must be a positive multiple of 8", d->N);
  if (d->K % 8) return set_error("pfd_gemm_f16: K pitch %lld must be a multiple of 8", (long long)d->K);
  if (d->W <= 0 || d->H <= 0 || d->NB <= 0) return set_error("pfd_gemm_f16: empty output raster");
  if (d->stride != 1 && d->stride != 2) return set_error("pfd_gemm_f16: stride %d unsupported", d->stride);
  if (d->tap_off != 0 && d->tap_off != 1) return set_error("pfd_gemm_f16: tap_off %d unsupported", d->tap_off);
  if (!d->out || !d->b_ptr) return set_error("pfd_gemm_f16: null out/b pointer");
  long long ktot = 0;
  for (int s = 0; s < d->nseg; ++s) {
    if (d->taps[s] != 1 && d->taps[s] != 9) return set_error("pfd_gemm_f16: taps[%d]=%d", s, d->taps[s]);
    if (d->a_c[s] <= 0 || d->a_c[s] % 8) return set_error("pfd_gemm_f16: a_c[%d]=%d must be a multiple of 8", s, d->a_c[s]);
    if (!d->a_ptr[s]) return set_error("pfd_gemm_f16: a_ptr[%d] is null", s);
    if ((reinterpret_cast<uintptr_t>(d->a_ptr[s]) & 15) || (d->a_sx[s] % 8) || (d->a_sy[s] % 8) || (d->a_sn[s] % 8))
      return set_error("pfd_gemm_f16: A segment %d not 16-byte aligned/strided", s);
    ktot += (long long)d->taps[s] * d->a_c[s];
  }
  if (ktot > d->K) return set_error("pfd_gemm_f16: segments cover K=%lld > pitch %lld", ktot, (long long)d->K);
  if (reinterpret_cast<uintptr_t>(d->b_ptr) & 15) return set_error("pfd_gemm_f16: B not 16-byte aligned");
  const bool geglu = d->act == PFD_ACT_GEGLU;

  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.nseg = d->nseg;
  p.stride = d->stride;
  p.tap_off = d->tap_off;
  p.W = d->W; p.H = d->H; p.NB = d->NB; p.N = d->N;
  p.b_batched = d->b_batch_stride != 0;
  p.alpha = d->alpha;
  p.act = d->act;
  p.bias = static_cast<const __half*>(d->bias);
  p.rowadd = static_cast<const __half*>(d->rowadd);
  p.residual = static_cast<const __half*>(d->residual);
  p.rowadd_ld = d->rowadd_ld > 0 ? d->rowadd_ld : d->N;
  p.out = static_cast<__half*>(d->out);
  p.so_n1 = d->so_n1; p.so_n0 = d->so_n0; p.so_y = d->so_y; p.so_x = d->so_x;
  p.so_c1 = d->so_c1; p.so_c0 = d->so_c0;
  p.ndiv = d->ndiv > 0 ? d->ndiv : 1;
  p.cdiv = d->cdiv > 0 ? d->cdiv : (1 << 30);
  p.vec_ok = (d->so_c0 == 1) && (p.cdiv % 8 == 0) && (d->so_n1 % 8 == 0) && (d->so_n0 % 8 == 0) &&
             (d->so_y % 8 == 0) && (d->so_x % 8 == 0) && (d->so_c1 % 8 == 0) &&
             ((reinterpret_cast<uintptr_t>(d->out) & 15) == 0) &&
             ((reinterpret_cast<uintptr_t>(d->residual) & 15) == 0);
  if ((reinterpret_cast<uintptr_t>(d->bias) & 15) || (reinterpret_cast<uintptr_t>(d->rowadd) & 15) || (d->rowadd_ld % 8))
    return set_error("pfd_gemm_f16: bias/rowadd must be 16-byte aligned");

  // ---- output raster tiling: 128 rows = bw x bh x bn pixels, minimise padded work
  int bw = 128, bh = 1, bn = 1;
  if (!p.b_batched) {
    long long best = -1;
    for (int cw = 128; cw >= 1; cw >>= 1) {
      if (cw * d->stride > 256) continue;
      for (int ch = 128 / cw; ch >= 1; ch >>= 1) {
        if (ch * d->stride > 256) continue;
        int cn = 128 / (cw * ch);
        long long cost = cdivll(d->W, cw) * cdivll(d->H, ch) * cdivll(d->NB, cn);
        if (best < 0 || cost < best) {
          best = cost; bw = cw; bh = ch; bn = cn;
        }
      }
    }
  }
  p.bw = bw; p.bh = bh; p.bn = bn;
  p.tiles_w = (int)cdivll(d->W, bw);
  p.tiles_h = (int)cdivll(d->H, bh);
  p.tiles_nb = (int)cdivll(d->NB, bn);
  const long long m_tiles = (long long)p.tiles_w * p.tiles_h * p.tiles_nb;

  // ---- N tile: minimise (waves x per-tile cost)
  // Plain GEMMs with short K (every segment 1x1, at most 40 K blocks of 64, one B for all rows) take 128 x 64 tiles.
  // There a tile's time grows much faster than its width, so the wave model below ranks the wide tiles too well:
  // on H100 the UNet's K = 320 ... 2560 Linears run 1.2x to 1.6x faster with 64-wide than with the 160-wide tiles it
  // picks (tools/gemm_sweep.py).  Longer K (convolutions, K = 5120) keeps the model.
  bool short_k_plain = !p.b_batched && !geglu;
  int kb_count = 0;
  for (int s = 0; s < d->nseg; ++s) {
    if (d->taps[s] != 1) short_k_plain = false;
    kb_count += d->taps[s] * ((d->a_c[s] + BK - 1) / BK);
  }
  short_k_plain = short_k_plain && kb_count <= 40;
  const int cands[5] = {256, 192, 160, 128, 64};
  int BNsel = 128;
  double best_cost = -1;
  const int sms = plan_sms();
  for (int i = 0; i < 5; ++i) {
    const int bn_c = cands[i];
    if (geglu && (d->N % bn_c)) continue;
    if (d->bn_force && d->bn_force != bn_c) continue;
    if (short_k_plain && !d->bn_force && bn_c != 64) continue;
    const long long nt = cdivll(d->N, bn_c);
    const long long tiles = m_tiles * nt;
    const double waves = (double)cdivll(tiles, sms);
    const double cost = waves * (bn_c + 24);
    if (best_cost < 0 || cost < best_cost - 1e-9) {
      best_cost = cost; BNsel = bn_c;
    }
  }
  if (best_cost < 0) return set_error("pfd_gemm_f16: no valid N tile (bn_force=%d, N=%d, geglu=%d)", d->bn_force, d->N, (int)geglu);
  p.n_tiles = (int)cdivll(d->N, BNsel);
  p.splits = 1;

  // ---- tensor maps
  int num_kb = 0;
  for (int s = 0; s < d->nseg; ++s) {
    p.taps[s] = d->taps[s];
    p.a_c[s] = d->a_c[s];
    p.chunks[s] = (d->a_c[s] + BK - 1) / BK;
    num_kb += p.taps[s] * p.chunks[s];
    cuuint64_t dims[4] = {(cuuint64_t)d->a_c[s], (cuuint64_t)d->in_w, (cuuint64_t)d->in_h, (cuuint64_t)d->NB};
    cuuint64_t strides[3] = {(cuuint64_t)d->a_sx[s] * 2, (cuuint64_t)d->a_sy[s] * 2, (cuuint64_t)d->a_sn[s] * 2};
    cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)(bw * d->stride), (cuuint32_t)(bh * d->stride), (cuuint32_t)bn};
    cuuint32_t estr[4] = {1, (cuuint32_t)d->stride, (cuuint32_t)d->stride, 1};
    if (int rc = encode_tensor_map_f16(&p.tmA[s], d->a_ptr[s], 4, dims, strides, box, estr, "A")) return rc;
  }
  p.num_kb = num_kb;
  p.kb_per_split = num_kb;
  cudaStream_t st = static_cast<cudaStream_t>(d->stream);
  float* const skws = static_cast<float*>(device_scratch(SCRATCH_SPLITK, SPLITK_WS_BYTES, 0, st));
  // ---- split-K for long-K problems that cannot fill the machine (8x8-level convs): fewer, wider N tiles
  //      (less A re-read through L2) x several K slices, fp32 partials reduced by splitk_finish_kernel.
  //      Never in deterministic mode: whether it fires depends on M and the SM count, and it regroups the K sum.
  if (!geglu && !d->bn_force && num_kb >= 32 && !deterministic()) {
    int bn_sk = 128;
    const int sk_cands[4] = {256, 192, 160, 128};
    for (int i = 0; i < 4; ++i)
      if (d->N % sk_cands[i] == 0) {
        bn_sk = sk_cands[i];
        break;
      }
    const long long nt_sk = cdivll(d->N, bn_sk);
    const long long tiles_sk = m_tiles * nt_sk;
    if (tiles_sk * 2 <= sms) {
      int splits = (int)(sms / tiles_sk);
      if (splits > 8) splits = 8;
      if (splits > num_kb / 8) splits = num_kb / 8;
      const size_t need = (size_t)splits * (size_t)m_tiles * BM * (size_t)d->N * sizeof(float);
      if (splits >= 2 && need <= SPLITK_WS_BYTES) {
        float* ws = skws;
        if (ws) {
          BNsel = bn_sk;
          p.n_tiles = (int)nt_sk;
          p.splits = splits;
          p.kb_per_split = (num_kb + splits - 1) / splits;
          p.splits = (num_kb + p.kb_per_split - 1) / p.kb_per_split;
          p.ws = ws;
        }
      }
    }
  }
  {
    const long long nbatch = p.b_batched ? d->NB : 1;
    cuuint64_t dims[3] = {(cuuint64_t)d->K, (cuuint64_t)d->N, (cuuint64_t)nbatch};
    const long long bs = p.b_batched ? d->b_batch_stride : (long long)d->K * d->N;
    cuuint64_t strides[2] = {(cuuint64_t)d->K * 2, (cuuint64_t)bs * 2};
    cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)BNsel, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    if (int rc = encode_tensor_map_f16(&p.tmB, d->b_ptr, 3, dims, strides, box, estr, "B")) return rc;
  }
  const long long total = m_tiles * p.n_tiles * p.splits;
  int grid = (int)(total < sms ? total : sms);
  int rc;
  switch (BNsel) {
    case 64: rc = launch_gemm<64>(p, grid, st); break;
    case 128: rc = launch_gemm<128>(p, grid, st); break;
    case 160: rc = launch_gemm<160>(p, grid, st); break;
    case 192: rc = launch_gemm<192>(p, grid, st); break;
    default: rc = launch_gemm<256>(p, grid, st); break;
  }
  if (rc || p.splits == 1) return rc;
  const long long vec_items = m_tiles * BM * (long long)(d->N / 8);
  long long fgrid = (vec_items + 255) / 256;
  if (fgrid > 8LL * sms) fgrid = 8LL * sms;
  launch_k(splitk_finish_kernel, dim3((unsigned)fgrid), dim3(256), 0, st, p);
  return check_launch("pfd_gemm_f16(split-K finish)");
}
