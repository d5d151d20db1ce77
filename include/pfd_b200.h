/*
 * pfd_b200 — C ABI of the H100 (sm_90a) kernel library behind the Prompt-Free-Diffusion hot path.
 *
 * The reference (SHI-Labs/Prompt-Free-Diffusion) has NO native boundary: every op on the path is a
 * torch/ATen library call made from lib/model_zoo/*.py.  This header is therefore the boundary a
 * maintainer would bind (via ctypes, see INTEGRATION.md) to replace those call sites.  Each entry
 * point cites the reference call site(s) it replaces.
 *
 * Conventions
 *   - plain C types only: device pointers as void*, sizes as int32/int64, cudaStream_t as void*.
 *   - every function returns 0 on success; non-zero = error, text via pfd_last_error().
 *   - no ownership transfer: the caller allocates every buffer (e.g. through torch) and keeps it
 *     alive until the stream has executed the call.
 *   - all activations are fp16, channel-last ("NHWC" / token-major [B, N, C]); all reductions and
 *     accumulations are fp32.
 *   - thread safety: calls on distinct streams are independent; pfd_last_error is thread-local.
 */
#ifndef PFD_B200_H_
#define PFD_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PFD_ABI_VERSION 2
#if defined(__GNUC__)
#define PFD_API __attribute__((visibility("default")))
#else
#define PFD_API
#endif
#define PFD_MAX_SEG 3

/* activation codes for pfd_gemm_desc.act */
enum {
  PFD_ACT_NONE = 0,
  PFD_ACT_SILU = 1,   /* x*sigmoid(x)          (openaimodel.py:203 nn.SiLU, autokl_modules.py:33) */
  PFD_ACT_GELU = 2,   /* exact erf GELU        (swin.py:84 nn.GELU)                               */
  PFD_ACT_RELU = 3,   /* seecoder.py:24 F.relu                                                    */
  PFD_ACT_GEGLU = 4   /* value*gelu(gate), weights packed [value|gate] per N tile (attention.py:44-51) */
};

PFD_API int pfd_version(void);
PFD_API const char* pfd_last_error(void);
/* number of kernels launched by this library in this process so far (bench.py: gpu_launches) */
PFD_API int64_t pfd_launch_count(void);
/* Run-time tuning switches, so that variants can be A/B-timed inside one process (tools/ab_unet.py); name == NULL
 * resets all of them to the built-in defaults.  Unknown names are stored and ignored.  Known names (default):
 *   deterministic (0)  1 = deterministic mode: with the same build on the same GPU architecture, every output of the
 *                      library is a bitwise function of the sample's own inputs - the same across runs and processes,
 *                      batch compositions (sample i of a batch equals the sample computed alone), GPU counts and SM
 *                      counts.  GroupNorm adds its statistics in a fixed order (no float atomics; chunks sized from
 *                      HW and C only), and the GEMM never splits K.  Results stay within
 *                      rounding of the default mode but are not bit-equal to it.  The default is 1 when the
 *                      environment variable PFD_DETERMINISTIC=1 is set when the library is loaded; a reset
 *                      (name == NULL) returns to that default.  CUDA graphs captured before the switch keep the
 *                      mode they were captured in: the Python package's set_deterministic() also drops its cached
 *                      graphs, setting this option directly does not.
 *   plan_sms (0)       test only: SM count the GEMM and GroupNorm plan their grids and split-K with; 0 = the
 *                      device's, otherwise min(value, the device's). */
PFD_API int pfd_set_option(const char* name, int32_t value);

/*
 * pfd_gemm_f16 — the wgmma tensor-core contraction used for every Linear, 1x1 conv, 3x3 conv
 * (implicit GEMM, TMA does the im2col) and batched QK^T / PV product on the path.
 *
 *   out[n, y, x, :] = act( alpha * sum_seg sum_tap sum_c A_seg[n, y*s+dy-1+o, x*s+dx-1+o, c] * Wt[:, k(seg,tap,c)]
 *                          + bias + rowadd[n, :] ) + residual[n, y, x, :]
 *
 * Rounding: the sum is accumulated in fp32; acc*alpha + bias + rowadd and the activation are evaluated in fp32 and
 *   rounded to fp16 once, y = fp16(act(...)); the residual is then added in fp16, out = fp16(y + residual) - the
 *   reference's `x + f(h)` on fp16 tensors.  Every path (staged or direct epilogue, split-K finish) rounds
 *   at these two points, so the plan changes only the fp32 summation order of the accumulator.
 *
 * Replaces: torch.nn.functional.conv2d / F.linear / torch.einsum / torch.bmm at
 *   openaimodel.py:203,229,240 (ResBlock convs + skip), :150 (Downsample), :105 (Upsample conv),
 *   attention.py:169-176,186-201 (to_q/k/v/out, QK^T, PV), :47,67 (GEGLU proj, ff out),
 *   attention.py:329,343 (proj_in/out), openaimodel.py:217-223,2629-2633 (emb_layers, time_embed),
 *   controlnet.py:165-181,299, autokl_modules.py:92-106,162-202,487,529, autokl.py:27,
 *   swin.py:88-90,171-173,322, seecoder.py:70-76,111,161,215-217,358,381.
 *
 * A operand: up to PFD_MAX_SEG channel-last fp16 tensors sharing the output raster (W,H,NB);
 *   segment s contributes taps[s] (1 or 9) x a_c[s] entries of K, in that order, so the weight
 *   matrix Wt is [N, K] row-major with K = sum_s taps[s]*a_c[s] (k = base_s + tap*a_c[s] + c).
 *   A plain [M,K] GEMM is W=M, H=1, NB=1 (or NB=batch for a batched GEMM with b_batch_stride!=0).
 * Requirements: a_c[s] % 8 == 0, K % 8 == 0, N % 8 == 0, all pointers 16-byte aligned.
 */
typedef struct pfd_gemm_desc {
  int32_t nseg;
  int32_t taps[PFD_MAX_SEG];
  int32_t a_c[PFD_MAX_SEG];
  const void* a_ptr[PFD_MAX_SEG];
  int64_t a_sx[PFD_MAX_SEG]; /* element strides of A: pixel, row, image */
  int64_t a_sy[PFD_MAX_SEG];
  int64_t a_sn[PFD_MAX_SEG];
  int32_t in_w, in_h;        /* extent of the A raster (== W,H for stride 1; ~2W,2H for stride 2) */
  int32_t stride;            /* 1 or 2 (3x3 stride-2 conv, openaimodel.py:150) */
  int32_t W, H, NB;          /* output raster: width, height, images (or rows, 1, batches) */

  const void* b_ptr;         /* weights [N, K] fp16 (K contiguous) */
  int32_t N;
  int64_t K;                 /* row pitch of b in elements (>= sum of segment K) */
  int64_t b_batch_stride;    /* 0: weights shared; else elements between per-image B matrices */

  float alpha;
  int32_t act;
  const void* bias;          /* [N] fp16 or NULL */
  const void* rowadd;        /* [NB, >=N] fp16 or NULL: per-image broadcast add (time embedding) */
  int64_t rowadd_ld;         /* row pitch of rowadd in elements (0 = N) */
  const void* residual;      /* same addressing as out, or NULL */

  void* out;                 /* fp16 */
  /* out offset (elements) = (n/ndiv)*so_n1 + (n%ndiv)*so_n0 + y*so_y + x*so_x
   *                         + (c/cdiv)*so_c1 + (c%cdiv)*so_c0                     */
  int64_t so_n1, so_n0, so_y, so_x, so_c1, so_c0;
  int32_t ndiv, cdiv;
  int32_t bn_force;          /* 0 = library picks the N tile; else one of 64/128/160/192/256 (GEGLU packing) */
  int32_t tap_off;           /* 3x3 taps read A at (y*s + dy - 1 + tap_off): 0 = symmetric padding 1; 1 = the VAE
                                encoder's F.pad(x,(0,1,0,1)) + stride-2 conv with padding 0 (autokl_modules.py:69-76) */
  void* stream;
} pfd_gemm_desc;

PFD_API int pfd_gemm_f16(const pfd_gemm_desc* d);
/*
 * GroupNorm(32 groups) [+ SiLU] over channel-last fp16, optionally over the channel-concatenation
 * of two tensors (the UNet skip concat, pfd.py:356,519) — writes one contiguous [NB,H,W,C1+C2].
 * Replaces: diffusion_utils.py:175-191 (GroupNorm32, eps 1e-5) + nn.SiLU (openaimodel.py:201-203,
 *   224-229, 2732-2734), attention.py:83-84 (eps 1e-6), autokl_modules.py:33-39,
 *   seecoder.py:359,383.
 * ws: scratch of at least NB*groups*16 + NB*4 bytes (fp64 sum / sum-of-squares per (image, group) of x - K, where
 *     the pivot K is the group's first channel at the image's first pixel, then one 32-bit arrival counter per image
 *     for the single-pass kernel),
 *     16-byte aligned.  zero_ws != 0: the call zeroes it first (one extra memset node); zero_ws == 0: the
 *     caller guarantees it is already zero (e.g. one bulk memset of many slots per network evaluation).
 * Deterministic mode (pfd_set_option "deterministic"): each CTA's statistics are combined in a fixed order into one
 *     fp64 partial per (image, group, pixel chunk) in a library-owned per-device buffer, and the last CTA of each
 *     image adds them in chunk order and overwrites ws (which then need not be zero).  Limits: NB <= 64, C <= 6144.
 *     The first deterministic call on a device allocates that buffer and must not be inside a stream capture.
 */
PFD_API int pfd_groupnorm_f16(const void* x1, int32_t c1, const void* x2, int32_t c2, int32_t NB,
                      int64_t HW, int32_t groups, const void* gamma, const void* beta, float eps,
                      int32_t silu, void* out, float* ws, int32_t zero_ws, void* stream);

/* LayerNorm over the last dim of [rows, C] fp16 (attention.py:294-296, swin.py norms, seecoder.py norms).
 * Optional fused residual: out = LN(x + res) (post-norm layers of seecoder.py:85-90,135-136). */
PFD_API int pfd_layernorm_f16(const void* x, const void* res, int64_t rows, int32_t C, const void* gamma,
                      const void* beta, float eps, void* out, void* stream);

/*
 * Row softmax over fp16 scores [batch, rows, cols] (row pitch ld), in place or to out:
 *   p = softmax( round_fp16(s) * scale + bias[(b % bias_mod_h)...] + mask[...] )
 * reproducing the reference's fp16 score rounding (attention.py:188-197, autokl_modules.py:188-192,
 * swin.py:187-203).  bias: [nheads, rows, cols] fp16 or NULL, selected by (b % nheads);
 * mask: [nwin, rows, cols] fp16 or NULL, selected by ((b / nheads) % nwin).
 */
PFD_API int pfd_softmax_f16(void* s, int64_t batch, int32_t rows, int32_t cols, int64_t ld, float scale,
                    const void* bias, int32_t nheads, const void* mask, int32_t nwin, void* stream);

/* sinusoidal timestep embedding [cos | sin], fp32 math, fp16 out (diffusion_utils.py:131-151). */
PFD_API int pfd_timestep_embedding_f16(const int64_t* t, int32_t n, int32_t dim, float max_period,
                               void* out, void* stream);
/* the same embedding for float32 (fractional) timesteps t[n], as the k-diffusion samplers evaluate the UNet at
 * t(sigma) (diffusion_utils.py:131-146 accepts any float t); equals pfd_timestep_embedding_f16 at integer t. */
PFD_API int pfd_timestep_embedding_ft_f16(const float* t, int32_t n, int32_t dim, float max_period, void* out,
                                          void* stream);

/* nearest-neighbour 2x upsample, channel-last (openaimodel.py:114, autokl_modules.py:54). */
PFD_API int pfd_upsample2x_f16(const void* x, int32_t NB, int32_t H, int32_t W, int32_t C, void* out,
                       void* stream);

/* layout converts at the pipeline edges: NCHW fp16/fp32 <-> channel-last fp16 (with channel pad):
 * out[n,y,x,c] = x[n,c,y,x]*mul + add for c < C, 0 for the pad channels (autokl.py:34: x*2-1). */
PFD_API int pfd_nchw_to_nhwc_f16(const void* x, int32_t src_is_f32, int32_t NB, int32_t C, int32_t H,
                         int32_t W, int32_t Cpad, float mul, float add, void* out, void* stream);
/* out_nchw[n,c,y,x] = clamp(x[n,y,x,c]*mul + add, lo, hi) for c < C (autokl.py:47,53: (dec+1)/2, clamp) */
PFD_API int pfd_nhwc_to_nchw_f16(const void* x, int32_t NB, int32_t C, int32_t H, int32_t W, int32_t Cpad,
                         float mul, float add, float lo, float hi, void* out, void* stream);

/* explicit im2col for 3x3 convs whose Cin is too small for the TMA path (Cin<8: UNet/VAE conv_in,
 * ControlNet hint stem): out[n,y,x, tap*Cin + c] (K padded to Kpad with zeros). */
PFD_API int pfd_im2col3x3_f16(const void* x, int32_t NB, int32_t H, int32_t W, int32_t C, int32_t stride,
                      int32_t Kpad, void* out, void* stream);

/* out = a*sa + b*sb (elementwise fp16, fp32 math); b may be NULL. */
PFD_API int pfd_axpby_f16(const void* a, float sa, const void* b, float sb, int64_t n, void* out,
                  void* stream);
/* out[n, :] = a[n, :] + row[:]  (level/position embeddings, seecoder.py:402,513) */
PFD_API int pfd_add_rowvec_f16(const void* a, const void* row, int64_t rows, int32_t C, void* out,
                       void* stream);

/*
 * Fused classifier-free-guidance combine + DDIM update (ddim.py:150-151,159-171), fp16 in/out with
 * the reference's fp16 rounding points reproduced:
 *   e = e_u + s*(e_c - e_u); pred_x0 = (x - sqrt(1-a_t)*e)/sqrt(a_t);
 *   x_prev = sqrt(a_prev)*pred_x0 + sqrt(1-a_prev-sigma^2)*e   (eta = 0 path; sigma*noise added by caller)
 * eps: [2*B, ...] as [uncond | cond] halves of `half_n` elements each; coefficients are read from a
 * device table coef[step*4 + {0..3}] = {a_t, a_prev, sigma_t, sqrt_one_minus_at} (fp32) indexed by
 * the device-side int *step so that a captured CUDA graph can be replayed for every step.
 * noise (optional, eta > 0, ddim.py:168-170): x_prev += sigma_t * noise * temperature with the reference's fp16
 * rounding order (guidance and temperature stay fp32, as python scalars do in torch).  log_tab (optional): int32 slot per schedule index (-1 = none); the step's x_prev / pred_x0
 * are also stored at log_xt / log_x0 + slot*half_n (the `intermediates` lists, ddim.py:122-124).
 */
PFD_API int pfd_ddim_step_f16(const void* eps, const void* x, int64_t half_n, float guidance,
                      const float* coef, const int32_t* step, void* x_prev, void* pred_x0,
                      const void* noise, float temperature, const int32_t* log_tab, void* log_xt,
                      void* log_x0, void* stream);

/* VAE encoder posterior (distributions.py:24-37, autokl.py:33-42, pfd.py:266-273): moments = channel-last
 * [B,H,W,cpad] quant_conv output (mean | logvar in the first 2*zc channels); logvar clamped to [-30,20],
 * std = exp(logvar/2), sample = scale*(mean + std*noise) with caller-drawn fp32 noise [B,zc,H,W] (NULL: mode).
 * Outputs NCHW fp16 [B,zc,H,W]; each may be NULL. */
PFD_API int pfd_vae_posterior_f16(const void* moments, int32_t B, int32_t zc, int32_t H, int32_t W, int32_t cpad,
                                  const float* noise, float scale, void* mean, void* logvar, void* stdv,
                                  void* sample, void* stream);

/* Device-side loop header of one DDIM step (ddim.py:108-113): *step = max(*step - 1, 0); t_out[0..nb) = ttab[*step].
 * Lets one CUDA graph hold several (or all) steps of the sampling loop with no host work in between. */
PFD_API int pfd_ddim_begin_step(int32_t* step, const int64_t* ttab, int64_t* t_out, int32_t nb, void* stream);

/*
 * k-diffusion samplers: Euler ancestral and DPM-Solver++(2M) (sampler.py:19-27,84-104, whose `sample` (:56-82) never
 * wraps the eps-prediction UNet as a denoiser nor applies CFG).  Every step of either type is one affine update with a
 * host-computed row coef[step*PFD_KSAMPLER_NCOEF + {0..5}] = {sigma, a, b, c, u, c_in_next} (fp32):
 *   e  = e_u + guidance*(e_c - e_u)   (cfg != 0: eps = [uncond | cond] halves of half_n fp16 elements)
 *      = guidance*eps                 (cfg == 0: one half, as the DDIM sampler's e_t = eps * scale)
 *   D  = x - sigma*e                  (the denoised estimate; x is the fp32 state, UNet input x*c_in)
 *   x' = a*x + b*D + c*d_prev + u*noise   (noise: fp16, NULL = none; u = sigma_up of an ancestral step)
 * The call then stores x' to x, D to d_prev, and fp16(x'*c_in_next) to unet_in (both halves when cfg != 0), i.e. the
 * next step's UNet input; on step == last_step also fp16(x') to out [half_n].  log_tab (optional): int32 slot per step
 * (-1 = none); the step's fp16 UNet input and D are also stored at log_xt / log_x0 + slot*half_n.
 * The step index is read from the device int *step, so a captured CUDA graph can be replayed for every step.
 */
#define PFD_KSAMPLER_NCOEF 6
PFD_API int pfd_ksampler_step_f32(const void* eps, int32_t cfg, float guidance, int64_t half_n, const float* coef,
                                  const int32_t* step, int32_t last_step, float* x, float* d_prev, const void* noise,
                                  void* unet_in, void* out, const int32_t* log_tab, void* log_xt, void* log_x0,
                                  void* stream);
/* Device-side loop header of one k-sampler step: *step += 1 (clamped to [0, nsteps)); t_out[0..nb) = ttab[*step], the
 * step's float timestep t(sigma).  Starts from *step = -1. */
PFD_API int pfd_ksampler_begin_step(int32_t* step, const float* ttab, int32_t nsteps, float* t_out, int32_t nb,
                                    void* stream);

/*
 * Per-sample counter-based Gaussian noise (graph-capturable):
 *   out[b*n + e] = fp16(scale * z(seeds[b], stream_id, draw + (draw_dev ? *draw_dev : 0), e)),  b < B, e < n
 * z is a pure function of its arguments, so sample b's noise depends on its own seed only, never on the batch:
 *   Philox4x32-10 with key = (seed & 0xffffffff, seed >> 32) and counter = (g & 0xffffffff, g >> 32, draw, stream_id),
 *   g = e / 4, gives the words w0..w3; Box-Muller over (w0, w1) and (w2, w3) in fp32 with the accurate device functions:
 *     u1 = fp32(fp32(w0) + 1) * 2^-32  (in (0, 1]),   u2 = fp32(w1) * 2^-32,
 *     z0 = sqrtf(-2 logf(u1)) * cos(2 pi u2),   z1 = sqrtf(-2 logf(u1)) * sin(2 pi u2)   (sincospif(2 u2))
 *   and (z2, z3) likewise from (w2, w3); element e takes z_(e % 4) of group g.
 * seeds: device array of B uint64.  draw_dev (optional): device int32 added to draw, so a captured graph can use the
 * sampler's device-side step counter as the draw index.  Streams used by the samplers: 0 = x_T, 1 = per-step sampler
 * noise (draw = schedule position), 2 = img2img forward noise.  Grid-stride, one Philox call per 4 elements.
 */
PFD_API int pfd_randn_f16(void* out, int32_t B, int64_t n, const uint64_t* seeds, uint32_t stream_id, int32_t draw,
                          const int32_t* draw_dev, float scale, void* stream);

/* Swin window plumbing on channel-last [B,H,W,C] (swin.py:269-304): pad + cyclic shift + window
 * partition in one gather (fwd) and the inverse scatter + crop (bwd). */
PFD_API int pfd_window_gather_f16(const void* x, int32_t B, int32_t H, int32_t W, int32_t C, int32_t ws,
                          int32_t shift, void* out, void* stream);
PFD_API int pfd_window_scatter_f16(const void* win, int32_t B, int32_t H, int32_t W, int32_t C,
                           int32_t ws, int32_t shift, const void* residual, void* out,
                           void* stream);
/* PatchMerging 2x2 gather -> [B, H/2*W/2, 4C] in the reference's x0,x1,x2,x3 order (swin.py:341-346). */
PFD_API int pfd_patch_merge_gather_f16(const void* x, int32_t B, int32_t H, int32_t W, int32_t C,
                               void* out, void* stream);

/*
 * Fused flash attention (wgmma): out[b, i, h*d + :] = softmax_j( fp16(q_i . k_j) * scale ) @ v  per (b, h),
 * scores never leave the SM.  Replaces attention.py:186-201 (einsum -> softmax -> einsum) for the UNet /
 * ControlNet self- and cross-attention.
 *   q  [B*heads, q_rows, d]   (first Nq rows valid)      k [B*heads, k_rows, d] (first Nk rows valid)
 *   vt [B*heads, d, vt_pitch] (V transposed, first Nk columns valid)
 *   out element (b, i, h, c) at  b*o_sb + i*o_sq + h*d + c.       d % 8 == 0, d <= 192.
 * Nk <= 160 with d <= 48 (the cross-attention against the 148 SeeCoder context tokens at the UNet's d = 40 level,
 * attention.py:178-201 with `context`) runs a persistent kernel whose single score tile holds every key (exact row
 * maximum, no online softmax); everything else the 64-key-block flash kernel.
 */
PFD_API int pfd_flash_attn_f16(const void* q, const void* k, const void* vt, void* out, int32_t B,
                               int32_t heads, int32_t Nq, int32_t Nk, int32_t d, int32_t q_rows,
                               int32_t k_rows, float scale, int64_t vt_pitch, int64_t o_sb, int64_t o_sq,
                               int32_t reserved, void* stream);

/* Same kernel with arbitrary 4-D strided operands: q, k as [B, heads, N, d] views and vt as [B, heads, d, Nk]
 * views, strides {batch, head, row} in elements (rows contiguous).  Lets a fused q|k projection GEMM and a
 * "swapped" V^T = Wv . X^T GEMM ([C, B*N] row-major) feed the kernel without any re-layout. */
PFD_API int pfd_flash_attn_strided_f16(const void* q, const void* k, const void* vt, void* out, int32_t B,
                                       int32_t heads, int32_t Nq, int32_t Nk, int32_t d,
                                       const int64_t* q_strides, const int64_t* k_strides,
                                       const int64_t* vt_strides, float scale, int64_t o_sb, int64_t o_sq,
                                       void* stream);

/* PatchEmbed gather (swin.py:479-489): NCHW image (fp16/fp32) -> [B, ceil(H/P), ceil(W/P), Kpad] rows in
 * the K order of the flattened conv weight [O, C*P*P]; zero padding for ragged H/W and K..Kpad. */
PFD_API int pfd_patchify_f16(const void* x, int32_t src_is_f32, int32_t B, int32_t C, int32_t H,
                             int32_t W, int32_t P, int32_t Kpad, void* out, void* stream);

/*
 * ControlNet.preprocess(type='canny') on the GPU (controlnet.py:332-360 -> controlnet_annotator/canny/__init__.py:4-5,
 * i.e. cv2.Canny(rgb_u8, low, high) with aperture 3 / L1 gradient, bit-exact): x is an NCHW [B,3,H,W] image in
 * [0,1] (fp16 or fp32), quantised like ToPILImage (x.mul(255).byte()); out is float32 [B,3,H,W] with 1.0 on edge
 * pixels (ToTensor + repeat(1,3,1,1)).  workspace: pfd_canny_workspace_bytes(B,H,W) bytes of device memory.
 * The call synchronises `stream` (hysteresis runs until a host-visible fixed point): not graph-capturable.
 * sweeps_out (optional, host): number of hysteresis sweeps that were needed.
 */
PFD_API int64_t pfd_canny_workspace_bytes(int32_t B, int32_t H, int32_t W);
PFD_API int pfd_canny_f32(const void* x, int32_t src_is_f32, int32_t B, int32_t H, int32_t W, int32_t low,
                          int32_t high, void* workspace, float* out, int32_t* sweeps_out, void* stream);
/* ToTensor(ToPILImage(x)) = floor(x*255)/255 as float32 (controlnet.py:345-348, preprocess type 'input'). */
PFD_API int pfd_image_u8_roundtrip_f32(const void* x, int32_t src_is_f32, int64_t n, float* out, void* stream);

/*
 * ControlNet.preprocess(type='hed' / 'softedge_v11p') (controlnet.py:370-376 -> controlnet_annotator/hed/__init__.py:
 * 102-128): the glue around the 13 convolutions of ControlNetHED_Apache2 (hed/__init__.py:23-59), which run on
 * pfd_gemm_f16.  The network runs at an activation scale s: the input and every conv bias are multiplied by s, so each
 * activation and side map is s times the reference's (ReLU convs and max-pool are positively homogeneous).
 *
 * pfd_hed_input_f16: NCHW [B,3,H,W] image in [0,1] (fp16 or fp32) -> channel-last fp16 [B,H,W,Cpad],
 *   out = (u8 - norm[c]) * scale with u8 = x.mul(255).byte() (ToPILImage, rounded in x's dtype) and the
 *   `x - self.norm` of hed/__init__.py:52; channels 3..Cpad-1 are zero.  norm: device float[3].
 * pfd_hed_pool_side_f16: one read of a block output x [B,h,w,C] fp16 (C % 8 == 0, 16-byte aligned) writes
 *   side [B,h,w] fp32 = x . proj_w + *proj_b (the block's 1x1 projection, hed/__init__.py:38; fp32 accumulation) and,
 *   when pooled != NULL, pooled [B,h/2,w/2,C] fp16 = 2x2 stride-2 max-pool, floor for odd h / w (F.max_pool2d,
 *   hed/__init__.py:34).  proj_w: device float[C]; proj_b: device float[1].
 * pfd_hed_fuse_f32: apply_hed after the network (hed/__init__.py:119-127) for nsides <= PFD_HED_MAX_SIDES fp32 side
 *   maps [B,h_k,w_k] (host array of device pointers and sizes): cv2.resize(INTER_LINEAR) of each to H x W, times
 *   inv_scale, np.mean over the maps (sequential float32 sum / n), sigmoid in float64, trunc(clip(edge*255, 0, 255)),
 *   then /255 (ToTensor) -> float32 [B,3,H,W] with three equal channels.
 * All three are asynchronous on `stream` and graph-capturable.
 */
#define PFD_HED_MAX_SIDES 5
PFD_API int pfd_hed_input_f16(const void* x, int32_t src_is_f32, int32_t B, int32_t H, int32_t W, int32_t Cpad,
                              const float* norm, float scale, void* out, void* stream);
PFD_API int pfd_hed_pool_side_f16(const void* x, int32_t B, int32_t h, int32_t w, int32_t C, const float* proj_w,
                                  const float* proj_b, float* side, void* pooled, void* stream);
PFD_API int pfd_hed_fuse_f32(const float* const* sides, const int32_t* side_h, const int32_t* side_w, int32_t nsides,
                             int32_t B, int32_t H, int32_t W, float inv_scale, float* out, void* stream);

/*
 * ControlNet.preprocess(type='scribble') (controlnet.py:432-491) for a whole batch; out is float32 [B,3,H,W] with 1.0
 * on scribble pixels in all three channels (ToTensor + repeat).  Asynchronous on `stream` and graph-capturable.
 *
 * pfd_scribble_hed_f32: make_scribble (controlnet.py:436-454) of the HED levels round(255 * hed[n*img_stride + y*W+x])
 *   (channel 0 of pfd_hed_fuse_f32's output with img_stride = 3*H*W): float32 cv2.GaussianBlur sigma 3 (ksize 25,
 *   BORDER_REFLECT_101), kept where it equals cv2.dilate along one of the four 3-tap lines, `> 127` -> 255 into
 *   nms (device uint8 [B,H,W], caller-allocated), then pfd_scribble_blur_u8 of nms into out.
 * pfd_scribble_blur_u8: cv2.GaussianBlur(z, (0,0), 3) of a uint8 [B,H,W] map on OpenCV's fixed-point path (ksize 19,
 *   bit-exact); writes the blurred map to `blurred` and / or `> 4` -> 1.0 to `out` (either may be NULL, not both).
 * pfd_scribble_xdog_f32: the xdog branch (controlnet.py:476-482) on an NCHW [B,3,H,W] image in [0,1] (fp16 or fp32,
 *   quantised like ToPILImage): per channel float32 Gaussian blurs g1 (sigma 0.5, ksize 5) and g2 (sigma 5, ksize 41),
 *   dog = uint8(clip(255 - min_c(g2 - g1), 0, 255)) truncated, edge where uint8(2 * uint8(255 - dog)) > threshold
 *   (the product wraps mod 256, as in the numpy expression).
 * The float blurs use OpenCV's float32 taps but not its operation order: decisions within float32 rounding of a tie may
 * differ from cv2 (README, scribble annotators).
 */
PFD_API int pfd_scribble_hed_f32(const float* hed, int64_t img_stride, int32_t B, int32_t H, int32_t W, uint8_t* nms,
                                 float* out, void* stream);
PFD_API int pfd_scribble_blur_u8(const uint8_t* z, int32_t B, int32_t H, int32_t W, uint8_t* blurred, float* out,
                                 void* stream);
PFD_API int pfd_scribble_xdog_f32(const void* x, int32_t src_is_f32, int32_t B, int32_t H, int32_t W, int32_t threshold,
                                  float* out, void* stream);

/*
 * PiDiNet, the default method of ControlNet.preprocess(type='scribble') (controlnet.py:465-472 ->
 * controlnet_annotator/pidinet/__init__.py:67-96 around pidinet() of pidinet/model.py:441-666: 'carv4', 60 channels,
 * dil=24, sa=True).  The input step (exact u8 levels; the BGR flip and the / 255 are folded into the weights) is
 * pfd_hed_input_f16 + im2col + the init block's GEMM; the trunk's 1x1 convs run on pfd_gemm_f16.  The pixel-difference weights are converted to plain
 * depthwise kernels when they are packed.  All five are asynchronous on `stream` and graph-capturable, and each output
 * pixel depends on its own image only.
 *
 * pfd_pidinet_dw_f16: depthwise conv1 of a PDC block (model.py:450,457-458): x [B,Hin,Win,C] fp16 (C % 8 == 0,
 *   16-byte aligned), w fp32 [ks*ks][C] (ks 3 or 5, zero padding ks/2) -> out = relu(conv) fp16 [B,h,w,C].  pool != 0
 *   (ks 3 only): the conv input is the 2x2 stride-2 max-pool of x (model.py:455-456, floor), also written to pooled
 *   [B,h,w,C] with h = Hin/2, w = Win/2.
 * pfd_pidinet_reduce_f16: CDCM's relu + conv1 (model.py:419-420): x [P,C] fp16 (C % 8 == 0, C <= 512) -> m [P,24] fp16
 *   = relu(x) . w + b; w: device fp32 [C][24], b: device fp32 [24].
 * pfd_pidinet_cdcm_f16: CDCM's conv2_1..conv2_4 summed (model.py:421-425): m [B,h,w,24] fp16 -> u [B,h,w,24] fp32 =
 *   sum over dilation d in 5,7,9,11 of the 3x3 conv with dilation d and zero padding d, on the tensor cores.  wpk: the
 *   four weights [24,24,3,3] arranged as mma.m16n8k16 B fragments: [54 k16 steps][3 n-tiles][32 lanes][4 halves],
 *   where K runs over (dilation, ky, kx, channel) and a lane (g = lane/4, t = lane%4) of n-tile j holds output
 *   channel 8j+g at K offsets 2t, 2t+1, 2t+8, 2t+9 of the step.
 * pfd_pidinet_side_f32: CSAM then MapReduce of one stage (model.py:395-401, 437-438, 616, 626): u [B,h,w,24] fp32 ->
 *   side [B,h,w] fp32 = a * (mr_w . u) + mr_b with a = sigmoid(conv3x3_pad1(conv1x1_4(relu(u)) + b1)); params: device
 *   fp32 [PFD_PIDINET_SIDE_PARAMS] = conv1 w [4][24], conv1 b [4], conv2 w [4][9], MapReduce w [24], MapReduce b [1].
 * pfd_pidinet_fuse_f32: model.py:626-645 and pidinet/__init__.py:88-96 for four fp32 side maps [B,h_k,w_k] (host
 *   array of device pointers and sizes, h_k <= H, w_k <= W): F.interpolate(bilinear, align_corners=False) to H x W,
 *   classifier cls[0..3] . e + cls[4] (device fp32 [5]), sigmoid, trunc(clip(edge*255, 0, 255)) / 255 -> float32
 *   [B,3,H,W] with three equal channels.
 */
#define PFD_PIDINET_SIDE_PARAMS 161
PFD_API int pfd_pidinet_dw_f16(const void* x, int32_t B, int32_t Hin, int32_t Win, int32_t C, int32_t ks, int32_t pool,
                               const float* w, void* out, void* pooled, void* stream);
PFD_API int pfd_pidinet_reduce_f16(const void* x, int64_t P, int32_t C, const float* w, const float* b, void* m,
                                   void* stream);
PFD_API int pfd_pidinet_cdcm_f16(const void* m, int32_t B, int32_t h, int32_t w, const void* wpk, float* u,
                                 void* stream);
PFD_API int pfd_pidinet_side_f32(const float* u, int32_t B, int32_t h, int32_t w, const float* params, float* side,
                                 void* stream);
PFD_API int pfd_pidinet_fuse_f32(const float* const* sides, const int32_t* side_h, const int32_t* side_w, int32_t B,
                                 int32_t H, int32_t W, const float* cls, float* out, void* stream);

/*
 * M-LSD, ControlNet.preprocess(type='mlsd' / 'mlsd_v11p') (controlnet.py:378-386 -> controlnet_annotator/mlsd:
 * apply_mlsd, pred_lines and MobileV2_MLSD_Large).  Every conv of the network except the depthwise ones and the final
 * 1x1 runs on pfd_gemm_f16 with BN folded into its weights.  All six are asynchronous on `stream` and graph-capturable
 * (segment counts stay on the device), and each output depends on its own image only.
 *
 * pfd_mlsd_input_f16: NCHW [B,3,H,W] image in [0,1] (fp32 if x_f32, else fp16) -> channel-last fp16 [B,H,W,16] =
 *   [u8 - 127.5 for r, g, b; 1 - 127.5 for the ones channel; 0 x 12] with u8 = x.mul(255).byte() (ToPILImage).  The
 *   network's 1 / 127.5 belongs in the stem weights.
 * pfd_mlsd_dw_f16: depthwise 3x3 ConvBNReLU6 (mbv2_mlsd_large.py:92-121): x [B,H,W,C] fp16 (C % 8 == 0), w fp32 [9][C]
 *   (tap-major), b fp32 [C] -> out = clamp(conv(min(x, 6)) + b, 0, 6) fp16; stride 1: [B,H,W,C], padding 1; stride 2:
 *   [B,H/2,W/2,C], F.pad(x, (0,1,0,1)) then padding 0.
 * pfd_mlsd_upsample_f16: F.interpolate(scale_factor=2, bilinear, align_corners=True) of x [B,h,w,C] fp16 into out, an
 *   [B,2h,2w] raster of fp16 pixels `pitch` elements apart (a channel slice of a wider tensor).
 * pfd_mlsd_head_f32: x [B,h,w,C] fp16 (C % 8 == 0, C <= 256), w fp32 [5][C], b fp32 [5] -> out fp32 [B,5,h,w] =
 *   w . x + b (the rows 7..11 of block23.conv3 that the decode reads).
 * pfd_mlsd_decode_f32: deccode_output_score_and_ptss(maps, 200, 3) and the segment tests of pred_lines (utils.py:18-88):
 *   maps fp32 [B,5,h,w] (centre logit, start x, y, end x, y displacements; h*w >= PFD_MLSD_TOPK) -> segs int32
 *   [B,PFD_MLSD_TOPK,4] (x0, y0, x1, y1 image coordinates int(2 * (x + d)), float64, truncated) and count int32 [B].
 *   A cell is a candidate when sigmoid(centre) is a 3x3 maximum and > thr_v; the top PFD_MLSD_TOPK candidates by score
 *   (ties: lowest flat index) become segments when |start - end| > thr_d (float32), listed in flat-index order.  keys:
 *   uint32 workspace [B*h*w].
 * pfd_mlsd_draw_f32: cv2.line(img, p0, p1, 255, 1, LINE_8) of segs[n, 0..count[n]) on out, float32 [B,3,H,W], which
 *   the caller zeroes: 1.0 on every pixel of OpenCV's clipLine + 8-connected LineIterator, on all three planes.
 */
#define PFD_MLSD_TOPK 200
PFD_API int pfd_mlsd_input_f16(const void* x, int32_t x_f32, int32_t B, int32_t H, int32_t W, void* out, void* stream);
PFD_API int pfd_mlsd_dw_f16(const void* x, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride, const float* w,
                            const float* b, void* out, void* stream);
PFD_API int pfd_mlsd_upsample_f16(const void* x, int32_t B, int32_t h, int32_t w, int32_t C, void* out, int64_t pitch,
                                  void* stream);
PFD_API int pfd_mlsd_head_f32(const void* x, int32_t B, int32_t h, int32_t w, int32_t C, const float* wt,
                              const float* b, float* out, void* stream);
PFD_API int pfd_mlsd_decode_f32(const float* maps, int32_t B, int32_t h, int32_t w, float thr_v, float thr_d,
                                uint32_t* keys, int32_t* segs, int32_t* count, void* stream);
PFD_API int pfd_mlsd_draw_f32(const int32_t* segs, const int32_t* count, int32_t B, int32_t H, int32_t W, float* out,
                              void* stream);

/* OpenPose body annotator, ControlNet.preprocess(type='openpose' / 'openpose_v11p') (controlnet.py:396-406 ->
 * controlnet_annotator/openpose: Body.__call__ and util.draw_bodypose).  The network's 3x3 / 1x1 convs run on
 * pfd_gemm_f16, its 7x7 convs on pfd_im2col7x7_f16 + pfd_gemm_f16.  Resize tables (idx int32 [D, T], weights [D, T])
 * are OpenCV's, built on the host (pfd_b200/openpose_tables.py).
 * pfd_openpose_input_f16: NCHW [B,3,H,W] image in [0,1] -> channel-last fp16 [B,hp,wp,16]: x.mul(255).byte(), BGR,
 *   cv2.resize to h x w (mode 0 copy, 1 integer block mean fy x fx, 2 uint8 LANCZOS4 with int weights (8 taps), 3
 *   INTER_AREA with float weights), padded to hp x wp with 128, u8 / 256 - 0.5; channels 3..15 are zero.
 * pfd_openpose_pool_f16: 2x2 / stride 2 max pool of x [B,H,W,C] fp16 (C % 8 == 0).
 * pfd_im2col7x7_f16: x [B,H,W,C] fp16 (C % 8 == 0) -> out [B*H*W, 49*C], k = tap * C + c, zero padding 3.
 * pfd_openpose_head_f32: out[n, out_off + k, y, x] (planar fp32, out_c channels) = act(b[k] + w[k] . x[n,y,x,:]),
 *   k < N, w fp32 [N][C], act = ReLU when relu.
 * pfd_openpose_resize_f32: cv2.resize of channels c0..c0+C of planar fp32 src [B,src_c,hs,ws] to out [B,C,H,W]
 *   (mode 0 copy / crop, 1 block mean fy x fx, 2 separable float tables).
 * pfd_openpose_peaks_f32: heatmaps fp32 [B,18,H,W] -> scipy gaussian_filter(sigma 3) in float64 (gauss: 13 weights,
 *   centre first; tmp, blur: float64 [B,18,H,W]; rowcnt int32 [B*18*H]), then the peaks (>= their 4 neighbours, 0
 *   outside, and > 0.1) in raster order: xy int32 [B,18,PFD_OPENPOSE_MAX_PEAKS,2] (x, y), score float64 (the
 *   unblurred value) and total int32 [B,18], the number of peaks found.  Peaks past PFD_OPENPOSE_MAX_PEAKS in raster
 *   order are dropped; total - PFD_OPENPOSE_MAX_PEAKS of them when total exceeds it.
 * pfd_openpose_assemble_f32: PAF scoring, greedy limb matching and person assembly (body.py:127-229).  up: planar fp32
 *   [B,57,hs,ws] (38 PAF channels, then 19 heatmap channels) at the resized-image size, brought to H x W pointwise by
 *   (mode, fy, fx, tables) as in pfd_openpose_resize_f32; conn float64 [B,19,MAX_PEAKS^2] and rows float64
 *   [B,MAX_PERSONS,20] are workspaces.  persons int32 [B,MAX_PERSONS,18] (per part the peak's index in its part, or
 *   -1), pscore float64 [B,MAX_PERSONS,2] (total score, parts) and npersons int32 [B].  Where the reference would
 *   raise IndexError (a connection matching a third person row), the first two matching rows are used.
 * pfd_openpose_draw_f32: util.draw_bodypose of every person on a zero canvas: out float32 [B,3,H,W] = colour / 255
 *   (colors uint8 [35,3]: 17 limb colours, then 18 keypoint colours; sintab: OpenCV's 451-entry sine table; idx
 *   int32 [B,H,W] workspace).
 */
#define PFD_OPENPOSE_MAX_PEAKS 128
#define PFD_OPENPOSE_MAX_PERSONS (17 * PFD_OPENPOSE_MAX_PEAKS)
PFD_API int pfd_openpose_input_f16(const void* x, int32_t x_f32, int32_t B, int32_t H, int32_t W, int32_t h, int32_t w,
                                   int32_t hp, int32_t wp, int32_t mode, int32_t fy, int32_t fx, const int32_t* iy,
                                   const void* wy, int32_t ty, const int32_t* ix, const void* wx, int32_t tx, void* out,
                                   void* stream);
PFD_API int pfd_openpose_pool_f16(const void* x, int32_t B, int32_t H, int32_t W, int32_t C, void* out, void* stream);
PFD_API int pfd_im2col7x7_f16(const void* x, int32_t B, int32_t H, int32_t W, int32_t C, void* out, void* stream);
PFD_API int pfd_openpose_head_f32(const void* x, int32_t B, int32_t h, int32_t w, int32_t C, const float* wt,
                                  const float* b, int32_t N, int32_t relu, float* out, int32_t out_c, int32_t out_off,
                                  void* stream);
PFD_API int pfd_openpose_resize_f32(const float* src, int32_t B, int32_t src_c, int32_t c0, int32_t C, int32_t hs,
                                    int32_t ws, int32_t H, int32_t W, int32_t mode, int32_t fy, int32_t fx,
                                    const int32_t* iy, const float* wy, int32_t ty, const int32_t* ix, const float* wx,
                                    int32_t tx, float* out, void* stream);
PFD_API int pfd_openpose_peaks_f32(const float* maps, int32_t B, int32_t H, int32_t W, const double* gauss, double* tmp,
                                   double* blur, int32_t* rowcnt, int32_t* xy, double* score, int32_t* total,
                                   void* stream);
PFD_API int pfd_openpose_assemble_f32(const float* up, int32_t B, int32_t up_c, int32_t hs, int32_t ws, int32_t H,
                                      int32_t W, int32_t mode, int32_t fy, int32_t fx, const int32_t* iy,
                                      const float* wy, int32_t ty, const int32_t* ix, const float* wx, int32_t tx,
                                      const int32_t* total, const int32_t* xy, const double* score, double* conn,
                                      double* rows, int32_t* persons, double* pscore, int32_t* npersons, void* stream);
PFD_API int pfd_openpose_draw_f32(const int32_t* persons, const int32_t* npersons, const int32_t* xy, int32_t B,
                                  int32_t H, int32_t W, const float* sintab, const uint8_t* colors, int32_t* idx,
                                  float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PFD_B200_H_ */
