/* vdb200 — C ABI of the H100-native Versatile-Diffusion sampling hot path (libvdb200.so).
 *
 * The reference (SHI-Labs/Versatile-Diffusion) has no FFI/operator boundary: its hot path is eager
 * PyTorch inside lib/model_zoo.  This header is the boundary a maintainer binds
 * instead: every entry point replaces the arithmetic of one reference call site (cited per function),
 * takes raw device pointers + explicit sizes + a cudaStream_t (passed as void*), allocates nothing,
 * keeps no global state besides a thread-local error string and a launch counter, and returns an
 * int status (0 = ok).  Python binding: versatile-diffusion_b200/vdb200/_lib.py (ctypes); the
 * reference-side stubs are shown in INTEGRATION.md.
 *
 * Conventions
 *   - activations: bf16, NHWC / token-major ([B, H, W, C] == [B*H*W, C]); latents/images fp32.
 *   - weights: bf16 [N, K] row-major (K contiguous); conv weights repacked to [Cout, (ky,kx,ci)].
 *   - all device pointers 16-byte aligned; leading dimensions in ELEMENTS.
 *   - `stream` is a cudaStream_t; kernels are stream-ordered and CUDA-graph capturable.
 */
#ifndef VDB200_H_
#define VDB200_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { VDB_OK = 0, VDB_ERR_INVALID = 1, VDB_ERR_CUDA = 2, VDB_ERR_UNSUPPORTED = 3 };
enum { VDB_ACT_NONE = 0, VDB_ACT_SILU = 1, VDB_ACT_GELU = 2, VDB_ACT_QUICK_GELU = 3, VDB_ACT_GEGLU = 4,
       VDB_ACT_GELU_TANH = 5 /* GPT-2's tanh approximation; vdb_textdec_gemv only */,
       VDB_ACT_TANH = 6 /* BertPooler's tanh; vdb_textdec_gemv only */ };

/* ---- library state ------------------------------------------------------------------------- */
const char* vdb_version(void);
const char* vdb_last_error(void);        /* message of the last non-zero status on this thread */
long long vdb_launch_count(void);        /* kernels launched by this library since the last reset */
void vdb_reset_launch_count(void);
int vdb_num_sms(void);

/* ---- K4: CFG mix + DDIM update — DDIMSampler.p_sample_ddim, lib/model_zoo/ddim.py:144-171 ------
 * e = e_u + scale*(e_c - e_u); pred_x0 = (x - sqrt(1-a_t) e)/sqrt(a_t);
 * x_prev = sqrt(a_prev) pred_x0 + sqrt(1 - a_prev - sigma^2) e + sigma*noise*temperature.
 * coef: device fp32 {a_t, a_prev, sigma_t, sqrt_one_minus_a_t}[, more rows]; step_idx (device int,
 * may be NULL) selects the row, so one captured CUDA graph serves every step. e_uncond/noise/pred_x0
 * may be NULL (scale==1 path, eta==0, no pred_x0 wanted). x_prev may alias x (in place); x_prev_dup (may be
 * NULL) receives a second copy — the cond half of the next step's torch.cat([x]*2) (ddim.py:144).
 * fp32, bit-identical to the reference ops. */
int vdb_ddim_cfg_step(const float* e_uncond, const float* e_cond, const float* x, const float* noise,
                      const float* coef, const int* step_idx, float scale, float temperature, float* x_prev,
                      float* x_prev_dup, float* pred_x0, long long n, void* stream);
/* ---- CFG mix + one multistep DPM-Solver++ update — DPMSolverSampler, lib/model_zoo/dpm_solver.py (an addition: the reference
 * has no such sampler; the algorithm and the table are specified in that module's docstring) -------------------------------------
 * coef: device fp32 rows of 8 {P, Q, A, B, C, D, 0, 0}; row *step_idx (device int, required) is used, so one captured CUDA graph
 * serves every step, warm-up and lower-order final steps included.  hist: a ring of 3 x n fp32 (slot s at hist + s*n) holding
 * the data predictions of the last steps.  In this op order, fp32 with explicit round-to-nearest (no FMA contraction):
 *   e = e_u + scale*(e_c - e_u);  x0 = P*x + Q*e  (-> hist slot idx % 3, and pred_x0);
 *   x_next = ((A*x + B*x0) + C*h1) + D*h2,  h1 = slot (idx+1) % 3, h2 = slot (idx+2) % 3.
 * A C or D term whose coefficient is exactly 0 is skipped and its slot not read (the ring is uninitialised at the first steps).
 * e_uncond may be NULL (scale==1 path: e = e_c); pred_x0 and x_next_dup may be NULL.  x_next may alias x; x_next_dup receives a
 * second copy (the cond half of the next step's batch).  VDB_ERR_INVALID before any launch: a null e_cond / x / coef / step_idx /
 * hist / x_next, n <= 0, a pointer not 16-byte aligned, or hist overlapping x, x_next, x_next_dup or pred_x0. */
int vdb_dpmpp_cfg_step(const float* e_uncond, const float* e_cond, const float* x, const float* coef, const int* step_idx,
                       float scale, float* hist, float* x_next, float* x_next_dup, float* pred_x0, long long n, void* stream);
/* ---- CFG mix + one stochastic DPM-Solver++ (SDE) update — DPMSolverSDESampler, lib/model_zoo/dpm_solver.py ---------------------
 * vdb_dpmpp_cfg_step with the noise column of the row: coef rows of 8 {P, Q, A, B, C, D, N, 0} and, in this op order,
 *   x_next = (((A*x + B*x0) + C*h1) + D*h2) + N*z,
 * fp32 with explicit round-to-nearest.  z = noise (fp32, n elements) when non-NULL, else four normals per element quad from
 * Philox4x32-10 at counter (quad, *step_idx, 0x73646573 "sdes", 0) under the 64-bit key *seed (two Box-Muller pairs,
 * u = (b + 0.5) 2^-32, as vdb_inpaint_blend_f32).  A C, D or N term whose coefficient is exactly 0 is skipped: at N == 0 nothing
 * is drawn or read and the result is vdb_dpmpp_cfg_step's bit for bit.  VDB_ERR_INVALID before any launch: the refusals of
 * vdb_dpmpp_cfg_step, neither seed nor noise, a seed not 8-byte aligned, noise not 16-byte aligned, or noise overlapping hist,
 * x_next, x_next_dup or pred_x0. */
int vdb_dpmpp_sde_cfg_step(const float* e_uncond, const float* e_cond, const float* x, const float* coef, const int* step_idx,
                           float scale, float* hist, float* x_next, float* x_next_dup, float* pred_x0, long long n,
                           const unsigned long long* seed, const float* noise, void* stream);
/* ---- inpainting: blended latent diffusion — lib/model_zoo/inpaint.py (an addition: the reference has no inpainting; the
 * semantics are specified in that module's docstring) ------------------------------------------------------------------------------
 * vdb_inpaint_blend_f32, after each sampler step: x, x0, noise fp32 NHWC [bs, hw, c]; mask fp32 [bs, hw] (mask_per_item != 0) or
 * [1, hw] (broadcast over the batch), 1 = generate, 0 = keep, broadcast over c.  table: device fp32 rows {a, b}; row *step_idx
 * (device int, required) is used.  z = noise when non-NULL, else four normals per element quad from Philox4x32-10 at counter
 * (quad, *step_idx, 0x696e7074 "inpt", 0) under the 64-bit key *seed (two Box-Muller pairs, u = (b + 0.5) 2^-32).  Per element,
 * fp32 with explicit round-to-nearest:  k = a*x0 + b*z;  x = m == 1 ? x : m == 0 ? k : m*x + (1 - m)*k;  x_dup (may be NULL)
 * receives a copy.  VDB_ERR_INVALID before any launch: a null x / x0 / mask / table / step_idx, neither seed nor noise, a size
 * <= 0, a pointer not 16-byte aligned, or x0, mask or noise overlapping x or x_dup. */
int vdb_inpaint_blend_f32(float* x, float* x_dup, const float* x0, const float* mask, int mask_per_item, const float* table,
                          const int* step_idx, const unsigned long long* seed, const float* noise, int bs, long long hw, int c,
                          void* stream);
/* the blend's Philox draws of step *step_idx for elements [0, n) of a latent, into out (fp32) */
int vdb_inpaint_noise_f32(const unsigned long long* seed, const int* step_idx, long long n, float* out, void* stream);
/* pixel mask fp32 [n, H8, W8] -> latent mask [n, H8/8, W8/8]: the max over each 8x8 cell (max_pool2d's rule: NaN propagates);
 * H8 and W8 multiples of 8 */
int vdb_mask_to_latent(const float* mask, int n, int H8, int W8, float* out, void* stream);
/* post-decode paste-back, fp32 NCHW [n, c, hw]: out = m*decoded + (1 - m)*image per pixel (m == 1 and m == 0 select exactly),
 * mask [n, hw] (mask_per_item != 0) or [1, hw]; out may alias decoded or image */
int vdb_composite_f32(const float* decoded, const float* image, const float* mask, int mask_per_item, int n, int c, long long hw,
                      float* out, void* stream);
/* ---- editing: DDIM inversion and DiffEdit — lib/model_zoo/edit.py (an addition: the reference has no inversion and no
 * editing; the semantics are specified in that module's docstring) ------------------------------------------------------------------
 * vdb_latent_store_slot_f32: ring[s] = x with s = *step_idx + offset (device int, required), slot s at ring + s*n; x and the ring
 * fp32 of n and slots*n elements.  A slot outside [0, slots) is not written.  VDB_ERR_INVALID before any launch: a null x / ring /
 * step_idx, n <= 0 or slots <= 0, a pointer not 16-byte aligned, or x overlapping the ring. */
int vdb_latent_store_slot_f32(const float* x, float* ring, int slots, const int* step_idx, int offset, long long n, void* stream);
/* vdb_inversion_blend_f32, after each step of a walk from an inversion: x fp32 NHWC [bs, hw, c]; ring fp32 [slots, bs, hw, c], the
 * inversion's trajectory; mask fp32 [bs, hw] (mask_per_item != 0) or [1, hw], 1 = generate, 0 = keep, broadcast over c.  Per element,
 * with k = ring[*step_idx] (device int, required), fp32 with explicit round-to-nearest, the formula of vdb_inpaint_blend_f32:
 * x = m == 1 ? x : m == 0 ? k : m*x + (1 - m)*k;  x_dup (may be NULL) receives a copy.  A *step_idx outside [0, slots) reads
 * nothing and leaves x and x_dup as they are.  VDB_ERR_INVALID before any launch: a null
 * x / ring / mask / step_idx, a size <= 0, a pointer not 16-byte aligned, or the ring or mask overlapping x or x_dup. */
int vdb_inversion_blend_f32(float* x, float* x_dup, const float* ring, int slots, const float* mask, int mask_per_item,
                            const int* step_idx, int bs, long long hw, int c, void* stream);
/* vdb_diffedit_mask_f32: DiffEdit's mask of bs images from D noise draws.  e_* fp32 NHWC [D*bs, hw, c] (draw d of image b at row
 * d*bs + b); e_src_u / e_tgt_u may be NULL (that side has no CFG: E = e_c), else E = e_u + s*(e_c - e_u).  out fp32 [bs, hw]:
 * dist(p) = (sum over d, then c, of |E_tgt - E_src|) / (D c);  cap = ratio * mean_p dist;  out = cap > 0 && min(dist, cap)/cap >= 0.5
 * ? 1 : 0.  One CTA per image, every sum in an order fixed by the shape, so the result is bit-reproducible.  VDB_ERR_INVALID before
 * any launch: a null e_src_c / e_tgt_c / out, a size <= 0, ratio not finite and > 0, a pointer not 16-byte aligned, or out
 * overlapping an input. */
int vdb_diffedit_mask_f32(const float* e_src_u, const float* e_src_c, float s_src, const float* e_tgt_u, const float* e_tgt_c,
                          float s_tgt, int D, int bs, long long hw, int c, float ratio, float* out, void* stream);
/* ---- Prompt-to-Prompt editing — lib/model_zoo/prompt_edit.py (an addition: the reference has no prompt editing; the semantics are
 * specified in that module's docstring) ------------------------------------------------------------------------------------------
 * vdb_local_blend_f32, after each step: x fp32 NHWC [n, H, W, C], row 0 the source image; map fp32 [n, h, w], the word maps; flags
 * device int32 per step, read at *step_idx (device int, required): 0 leaves x untouched.  For each target b = 1 .. n-1 (one CTA each):
 * pooled_s = 3x3 max-pool (stride 1, pad 1) of map[s], mask_s(y, x) = max(pooled_s) > 0 && pooled_s[floor(y h / H), floor(x w / W)] /
 * max(pooled_s) > threshold (the division rounded to nearest), and x_b = (mask_b || mask_0) ? x_b : x_0 (a selection: the per-element
 * blend of vdb_inpaint_blend_f32 at m in {0, 1}).  x_dup (may be NULL) receives the rows written.  VDB_ERR_INVALID before any launch:
 * a null x / map / flags / step_idx, n < 2, a size <= 0, h * w > 4096, a threshold not finite, a pointer not 4-byte aligned, or x,
 * x_dup and map overlapping. */
int vdb_local_blend_f32(float* x, float* x_dup, const float* map, const int* flags, const int* step_idx, int n, int H, int W, int C,
                        int h, int w, float threshold, void* stream);
/* ---- region prompts and panoramas: MultiDiffusion on a window layout — lib/model_zoo/regions.py and lib/model_zoo/panorama.py
 * (additions: the reference has no region or panorama mode; the layout, the weights, the merge and the bootstrapping are specified
 * in those modules' docstrings) -------------------------------------------------------------------------------------------------
 * A panorama's window fusion is the walk with no regions, R = 0.  The canvas is fp32 NHWC [bs, H, W, C].  The layout has ny x nx
 * windows of h x w; window g = iy*nx + ix reads rows oy[iy] + r (r < h) and columns (ox[ix] + j) mod W (j < w); oy / ox are device
 * int32 tables, and only a circular layout has columns that wrap.  Region prompts without windows use one window equal to the
 * canvas.  The gather and the merge take a range [first, first + k) of windows, one UNet chunk.
 * masks: fp32 [R, bs, H, W] on the canvas, region r = 1..R at row r - 1, values in [0, 1]; 0 <= R <= 8.  Region 0 is the
 * background, of weight m_0 = max(0, 1 - S) with S = m_1 + ... + m_R summed in ascending r (S = 0 when R = 0), and D = m_0 + S
 * (fp32, rounded).
 * vdb_region_gather_f32: out = u_blocks + R + 1 blocks of [k*bs, h, w, C], u_blocks in {0, 1, R + 1}; block blk is region
 * blk - u_blocks of the c half, region 0 for the single u block, region blk for one of R + 1 u blocks; row j*bs + b of a block is
 * window first + j of image b.  Every block is an exact copy of the window unless rows is non-NULL and
 * row *step_idx of rows (fp32 {on, a, b, 0}) has on != 0: then region r >= 1 reads, per element of mask value m,
 * m == 1 ? x : m == 0 ? k : m*x + (1 - m)*k  with  k = a*bg + b*z  (fp32, round-to-nearest), bg = row floor(w*nb / 2^32) of the
 * backgrounds bg fp32 [nb, C], w the first word of Philox4x32-10 at counter ((r*bs + b), *step_idx, 0x72676e73 "rgns", 1) under the
 * key *seed, and z = noise (fp32 NHWC canvas) when non-NULL, else the canvas element's normal at counter (element quad, *step_idx,
 * "rgns", 0) by the Box-Muller of vdb_inpaint_blend_f32.  VDB_ERR_INVALID before any launch: a null x / out / table, a size <= 0,
 * a window larger than the canvas, a range outside the ny*nx windows, tables not 4-byte aligned, R outside [0, 8], u_blocks not
 * 0, 1 or R + 1, rows without step_idx / seed / nb > 0 backgrounds (or without masks when R >= 1), x / out / noise not 16-byte
 * aligned, masks / rows / bg / step_idx not 4-byte, seed not 8-byte, or out overlapping x, masks, noise or bg.
 * vdb_region_noise_f32: the gather's draws of step *step_idx: z [n] for canvas elements [0, n), picks int32 [R*bs], entry
 * (r - 1)*bs + b the background row of region r, image b; 1 <= R <= 8.
 * vdb_region_merge_f32: eps [halves*(R+1)*k*bs, h, w, C], block s*(R+1) + r (halves 1, or 2 for [u blocks; c blocks]) -> out
 * [halves*bs, H, W, C].  cover_y int32 [H, 2]: the windows covering row y are iy in [cover_y[2y], cover_y[2y+1]); cover_x int32
 * [W, 4]: those covering column x are ix in [cover_x[4x], cover_x[4x+1]) then [cover_x[4x+2], cover_x[4x+3]), ascending.  Per
 * element, over its covering windows in ascending window index and r = 0..R inside each, fp32 with round-to-nearest: each term
 * m_r*e of nonzero weight (a zero weight is skipped) is one product; the first sets out, later ones are added, and the call whose
 * range holds the last window divides by n*D (n covering windows, the product rounded).  Elements with no covering window in the
 * range are not touched, so calls over consecutive ranges compute exactly what one call over all windows does; a hard mask selects
 * its region's eps bit for bit.  With R = 0 (masks may be NULL) every product is 1*e = e and n*D = n, so the merge is the plain
 * window average and an element with one covering window gets that window's eps bit for bit.  No atomics: the result is
 * bit-reproducible.  VDB_ERR_INVALID before any launch: the gather's size, range and table refusals, a null cover table, a null
 * masks when R >= 1, halves not 1 or 2, R outside [0, 8], eps / out / cover_x not 16-byte aligned, cover_y / masks not 4-byte, or
 * eps or masks overlapping out. */
int vdb_region_gather_f32(const float* x, int bs, int H, int W, int C, const int* oy, const int* ox, int ny, int nx, int h, int w,
                          int first, int k, int R, int u_blocks, const float* masks, const float* rows, const int* step_idx,
                          const unsigned long long* seed, const float* bg, int nb, const float* noise, float* out, void* stream);
int vdb_region_noise_f32(const unsigned long long* seed, const int* step_idx, long long n, int R, int bs, int nb, float* z, int* picks,
                         void* stream);
int vdb_region_merge_f32(const float* eps, int halves, int bs, int H, int W, int C, const int* oy, const int* ox, const int* cover_y,
                         const int* cover_x, int ny, int nx, int h, int w, int first, int k, int R, const float* masks, float* out,
                         void* stream);
/* ---- self-attention guidance — lib/model_zoo/sag.py (an addition: the reference has no SAG; the semantics are specified in that
 * module's docstring) ----------------------------------------------------------------------------------------------------------------
 * vdb_sag_degrade_f32: x, e, out fp32 NHWC [bs, H, W, C]; mass fp32 [bs, hm*wm], the mid block's key mass; table device fp32 rows
 * {sqrt(a_t), sqrt(1 - a_t)}, row *step_idx (device int, required).  Per element, fp32 with explicit round-to-nearest:
 *   x0 = (x - s1*e) / sa;  v = M ? blur(x0) : x0;  out = sa*v + s1*e
 * with M = mass[b, (y*hm/H)*wm + x*wm/W] > 1 (integer division: nearest upsampling) and blur the depthwise 9x9 Gaussian of sigma 1
 * (taps exp(-k^2/2), k = -4..4, normalised in double) with reflect padding by 4, applied along rows then along columns, each sum
 * in tap order with fused multiply-adds.  VDB_ERR_INVALID before any launch: a null argument, a size <= 0, H or W < 5, a pointer not
 * 4-byte aligned, or out overlapping x, e or mass; VDB_ERR_UNSUPPORTED: C > 8, hm > H, wm > W or hm*wm > 4096.
 * vdb_sag_guide_f32, in place on n elements: d = s*(e_src - e_deg) with e_src = e_u when e_u is non-NULL (CFG), else e_c; then
 * e_c += d and e_u += d, fp32 with explicit round-to-nearest.  VDB_ERR_INVALID before any launch: a null e_c / e_deg, n <= 0, s not
 * finite, a pointer not 4-byte aligned, or any two of e_u, e_c, e_deg overlapping. */
int vdb_sag_degrade_f32(const float* x, const float* e, const float* mass, const float* table, const int* step_idx, int bs, int H,
                        int W, int C, int hm, int wm, float* out, void* stream);
int vdb_sag_guide_f32(float* e_u, float* e_c, const float* e_deg, float s, long long n, void* stream);
/* y = a*x + b*z, fp32 — VD_v2_0.q_sample (vd.py:221-224) for the img2img start (ddim.py:97-103) */
int vdb_axpby_f32(const float* x, const float* z, float a, float b, float* y, long long n, void* stream);
int vdb_add_int(int* p, int delta, void* stream); /* device-side step counter update */
/* y = c0*x0 + c1*x1 + c2*x2 + c3*x3 (x1..x3 may be NULL), fp32 — PLMS eps extrapolation (north-star addition: the
 * reference has no PLMS sampler; formula of Liu et al. 2022 / CompVis latent-diffusion plms.py) */
int vdb_lincomb4_f32(const float* x0, const float* x1, const float* x2, const float* x3, float c0, float c1, float c2,
                     float c3, float* y, long long n, void* stream);

/* ---- wgmma GEMM — nn.Linear / 1x1 conv call sites: attention.py:37-64,161-193,237,249;
 *      autokl_modules.py:150-202; HF CLIP q/k/v/out/fc1/fc2 (clip.py:58-61,92-100) ----------------
 * out[M,N] = act(alpha * ([A | A2] @ W^T + bias)) + resid.   A [M,K] (lda), optional A2 [M,K2] (lda2)
 * concatenated along K, W [N, K+K2] (ldw).  bias fp32 [N] (bias_bstride==0) or per-batch rows
 * [.., N] selected by row / rows_per_batch.  act = VDB_ACT_*; VDB_ACT_GEGLU expects W/bias rows packed
 * per 256-column tile as 128 value rows then their 128 gate rows and writes N/2 columns
 * (GEGLU.forward, attention.py:42-44).  out bf16 (out_f32==0) or fp32.  bn: 0 = auto, else force
 * tile N in {64,128,160,256} on a 128-row tile, or 160 | VDB_IGEMM_BM256 for the 256-row tile (bf16 out, act 0,
 * alpha 1, N % 32 == 0, one bias row per 256 rows, no split-K; the same in the other igemm entry points).  ksplit: 0 = auto, 1 = off; split-K needs workspace >= ksplit*M*N*4 B. */
#define VDB_IGEMM_BM256 0x1000
int vdb_gemm_bf16(const void* A, long long M, long long K, long long lda, const void* A2, long long K2,
                  long long lda2, const void* W, long long N, long long ldw, const float* bias,
                  long long bias_bstride, long long rows_per_batch, const void* resid, long long ldr, void* out,
                  long long ldo, int out_f32, int act, float alpha, int bn, int ksplit, void* workspace,
                  size_t ws_bytes, void* stream);

/* The tiling the last vdb_gemm_bf16 / vdb_gemm_ln_bf16 / vdb_conv3x3_bf16 call on this thread launched (host-side record, no
 * device work): out[0..n) receives {BN, STAGES, epilogue MODE, ksplit, grid, M tiles, N tiles} (as many as n
 * allows).  Returns the number of fields (7).  For tests and tools that need to know which kernel instantiation ran. */
int vdb_igemm_last_plan(int* out, int n);
/* The tile height BM (128 or 256 rows) of that same launch; 0 before the first one. */
int vdb_igemm_last_bm(void);
/* The order in which that same launch walked its output tiles: 0 = M tile index fastest, 1 = N tile index fastest (a single-pass
 * launch with several N tiles whose A operand outweighs W, so that a wave reads each band of A rows once). */
int vdb_igemm_last_n_fast(void);

/* ---- the same GEMM with a LayerNorm folded in — BasicTransformerBlock norm1/2/3, attention.py:206-208,214-218 -------------
 * CONSUMER (ln_stats != NULL):  out = act( LN(x) W0^T + b0 )  computed from the RAW x without ever forming LN(x):
 *     out[m,n] = act( rstd[m] * (x W^T - mean[m] * ln_colsum[n]) + bias[n] )
 *   with W = W0 * gamma (per input channel, rounded to bf16), ln_colsum[n] = sum_k float(W[n,k]), bias[n] = b0[n] + sum_k beta_k W0[n,k]
 *   prepared once by the caller.  mean / rstd come from ln_stats = [ln_parts][ln_rows][2] fp32 partial (sum, sum of squares) over
 *   disjoint column ranges of x's rows (written by a PRODUCER launch below, which reports ln_parts), ln_dim == K = the LayerNorm width,
 *   ln_eps its epsilon.
 *   ln_on_cols = 1: x is the W-side operand (out^T = W0 LN(x)^T, the transposed V^T projection): A holds the prepared weights, the
 *   statistics belong to the output COLUMNS, ln_colsum is indexed by the output ROW and ln_rowbias[m] (may be NULL) carries the beta term.
 *   act: VDB_ACT_NONE or VDB_ACT_GEGLU (packed as for vdb_gemm_bf16; ln_colsum packed like bias).  No residual.
 * PRODUCER (stats_out != NULL):  out = A W^T + bias + resid as vdb_gemm_bf16, and stats_out (room for [2 * ceil(N/64)][M][2] fp32)
 *   receives *stats_parts partial (sum, sum of squares) per output row (fp32 values before the bf16 rounding; one partial per N tile
 *   and epilogue warp, so *stats_parts = 2 * N tiles is known on the host when the call returns), N % 32 == 0.
 * Exactly one of ln_stats / stats_out; bf16 out, 16-byte aligned out / resid rows. */
int vdb_gemm_ln_bf16(const void* A, long long M, long long K, long long lda, const void* W, long long N, long long ldw,
                     const float* bias, const void* resid, long long ldr, void* out, long long ldo, int act,
                     const float* ln_stats, long long ln_rows, int ln_parts, int ln_dim, float ln_eps, const float* ln_colsum,
                     int ln_on_cols, const float* ln_rowbias, float* stats_out, int* stats_parts, int bn, void* stream);

/* ---- wgmma implicit-GEMM 3x3 conv on NHWC — ResBlock convs openaimodel.py:203,229; Downsample
 *      :150-152; Upsample.conv :105; VAE autokl_modules.py:48-76,93-111 ---------------------------
 * mode 0: stride 1 pad 1; mode 1: stride 2 pad 1; mode 2: stride 2 with pad (0,1,0,1) (VAE).
 * mode 3 + 2*py + px: parity (py,px) of "nearest 2x upsample then 3x3 conv" (Upsample.forward, openaimodel.py:107-117;
 *      autokl_modules.py:54-58) evaluated on the SOURCE image with the 9 taps folded into 2x2: X = source [B,H,W,C],
 *      out = [B,H,W,N] (that parity sub-lattice), Wt = [N, 4*C] (ty,tx,c) pre-summed on the host; no skip inputs.
 * mode 7 + 2*py + px: the same parity conv, but `out` is the full [B,2H,2W,N] tensor and the tile is stored straight into pixels
 *      (2y+py, 2x+px) through the output tensor map (no interleave pass, no parity temporaries); bf16 out, no residual / skips /
 *      split-K, N % 32 == 0.
 * Wt [N, 9*C + Cs1 + Cs2], K order (ky,kx,c) then the 1x1 skip_connection columns whose inputs
 * skip1/skip2 (raw NHWC at output resolution; the two halves of torch.cat([h, hs.pop()]),
 * vd.py:372) are accumulated into the same accumulator tile (ResBlock.skip_connection, openaimodel.py:240).
 * bias/resid/out/act as vdb_gemm_bf16 with rows_per_batch = Hout*Wout. C, Cs1, Cs2 multiples of 64. */
int vdb_conv3x3_bf16(const void* X, int B, int H, int W, int C, int mode, const void* Wt, int N, long long ldw,
                     const void* skip1, int Cs1, const void* skip2, int Cs2, const float* bias,
                     long long bias_bstride, const void* resid, long long ldr, void* out, long long ldo,
                     int out_f32, int act, int bn, int ksplit, void* workspace, size_t ws_bytes, void* stream);

/* ---- wgmma flash attention — CrossAttention.forward, attention.py:178-192 -----------------
 * O = softmax(Q K^T * scale) V per (batch, head), fp32 online softmax, nothing materialised.
 * Q [B*Nq, ldq] head h at columns q_col0 + h*DK; K [B*Nk, ldk] at k_col0 + h*DK;
 * Vt [H*DVP, ldv] row h*DVP + c, column b*kv_bstride + j; out [B*Nq, ldo] head h at columns h*d_head.
 * DK = vdb_attention_dk_pad(d_head), DVP = vdb_attention_dv_pad(d_head); the head pads must be
 * zero: Q / K columns d_head .. DK-1 of each head and Vt rows h*DVP + d_head .. h*DVP + DVP-1 (the
 * projection weights are zero-padded at pack time). causal != 0: CLIP text mask.
 * Batch b starts at row b*q_bstride of Q/out and at row (K) / column (Vt) b*kv_bstride; kv_bstride must be a
 * multiple of 8 (TMA: 16-byte aligned innermost coordinate), so ragged contexts (77, 257 tokens) are stored
 * padded to 80 / 264 per batch item; the pad keys are masked by Nk. 0 = dense (stride = count).
 * May hold any finite values: the pad keys (K rows / Vt columns b*kv_bstride + [Nk, kv_bstride)), the pad
 * query rows b*q_bstride + [Nq, q_bstride) of Q, and everything outside the given slices (other columns of
 * Q / K / Vt, Vt columns past B*kv_bstride).  Only rows b*q_bstride + [0, Nq), columns [0, H*d_head) of out
 * are written.
 * Three forms, picked by kv_len and items (both non-NULL: VDB_ERR_UNSUPPORTED, no such kernel):
 * - plain (kv_len and items NULL; Bq, Bkv, step_idx and accumulate 0 / NULL): the above.
 * - kv_len != NULL: a key count per batch item — BertSelfAttention.forward, optimus_bert.py:200-233, under the padding mask of
 *   BertForLatentConnector_XX.forward (:1404-1412): key j of item b is visible iff j < kv_len[b] (kv_len: device int32 [B],
 *   clamped to [0, Nk]).  The reference adds -10000 to the masked scores; exp of that underflows to exactly 0 in fp32 next to any
 *   visible key, so the hard mask computes the same function.  An item with kv_len[b] <= 0 gets zero output rows.  Masked K / V
 *   rows are never weighted (they may hold any finite values).  d_head 64 only (VDB_ERR_UNSUPPORTED otherwise); causal != 0 or a
 *   misaligned kv_len return VDB_ERR_INVALID.
 * - items != NULL: the operands of each output item chosen by a device table — Prompt-to-Prompt's attention injection,
 *   lib/model_zoo/prompt_edit.py.  items: device int32 [rows][3][B]; output item b reads Q from item bq = items[r][0][b], K from
 *   item bk = items[r][1][b] and V^T from item bv = items[r][2][b] of row r = *step_idx (device int), and writes item b of out.
 *   Entries must lie in [0, Bq) (bq) and [0, Bkv) (bk, bv), where Q holds Bq items and K / V^T hold Bkv items (the tensor maps are
 *   sized by them); bv < 0 skips item b: nothing is read or written for it.  accumulate != 0: out = bf16(float(out) + O).  With
 *   items[r][.][b] = b and accumulate 0 the output equals the plain form's bitwise.  A null or misaligned items / step_idx, or
 *   Bq / Bkv <= 0, return VDB_ERR_INVALID; so does any of Bq, Bkv, step_idx, accumulate given without items.
 * Refusals in order: the form's own (for the table: items / step_idx, then kv_len, then Bq / Bkv), then the checks common to all
 * three, then a d_head without a kernel (VDB_ERR_UNSUPPORTED). */
int vdb_attention_dk_pad(int d_head);
int vdb_attention_dv_pad(int d_head);
int vdb_attention_bf16(const void* Q, long long ldq, int q_col0, const void* K, long long ldk, int k_col0,
                       const void* Vt, long long ldv, void* out, long long ldo, int B, int H, int Nq, int Nk,
                       int q_bstride, int kv_bstride, int d_head, float scale, int causal,
                       const int* kv_len, int Bq, int Bkv, const int* items, const int* step_idx, int accumulate,
                       void* stream);
/* Prompt-to-Prompt's word maps from the operands of a cross-attention call, fp32 math: for r in [0, n) and query p in [0, N),
 *   map[r, p] += sum over heads h of sum over keys j < L of w[r, j] * softmax_j(scale * q . k)
 * with q = Q row (row0 + r) * N + p, k = K row (row0 + r) * kv_bstride + j, both at columns h*DK .. h*DK + d_head (DK =
 * vdb_attention_dk_pad(d_head)), bf16.  w, map fp32 [n, L], [n, N].  One CTA per (16 queries, r), sums in an order fixed by the
 * shape, one writer per entry: bit-reproducible.  L <= 80 (a text context) and d_head <= 160 a multiple of 8, else
 * VDB_ERR_UNSUPPORTED.  VDB_ERR_INVALID before any launch: a null Q / K / w / map, a size <= 0, row0 < 0, kv_bstride < L (0 = L),
 * odd or short ldq / ldk, a pointer not 4-byte aligned, or map overlapping w. */
int vdb_xattn_word_map_f32(const void* Q, long long ldq, const void* K, long long ldk, const float* w, float* map, int n, int row0,
                           int H, int N, int L, int kv_bstride, int d_head, float scale, void* stream);
/* Self-attention guidance's key mass (lib/model_zoo/sag.py) from the operands of a self-attention call, fp32 math: for r in
 * [0, n) and key j in [0, N),
 *   mass[r, j] += w * sum over heads h of sum over queries p < N of softmax_j(scale * q . k)
 * with q = Q row (row0 + r) * N + p at columns q_col0 + h*DK .., k = K row (row0 + r) * kv_bstride + j at columns k_col0 + h*DK ..
 * (DK = vdb_attention_dk_pad(d_head)), bf16: the fused q | k buffer of a self-attention layer, or its separate q and padded keys.
 * Two launches: the softmax max and sum of every (r, h, p) into stats (fp32 scratch of n*H*N*2), then one writer per mass entry
 * adding the heads in order and the queries in a fixed order: bit-reproducible, no atomics.  N <= 4096 and d_head <= 160 a multiple
 * of 8, else VDB_ERR_UNSUPPORTED.  VDB_ERR_INVALID before any launch: a null Q / K / stats / mass, a size <= 0, row0 < 0,
 * kv_bstride < N (0 = N), odd or negative column offsets, odd ldq / ldk or ldq < q_col0 + H*DK (ldk likewise), a pointer not 4-byte
 * aligned, or mass overlapping stats. */
int vdb_sattn_key_mass_f32(const void* Q, long long ldq, int q_col0, const void* K, long long ldk, int k_col0, float* stats,
                           float w, float* mass, int n, int row0, int H, int N, int kv_bstride, int d_head, float scale,
                           void* stream);

/* ---- GroupNorm(32) [+SiLU] [+channel concat] on NHWC — normalization()/Normalize():
 *      diffusion_utils.py:168-191 (eps 1e-5), attention.py:76-77 & autokl_modules.py:38-39 (1e-6) ----
 * y[B,HW,C1+C2] = act(GN32(cat(x1,x2))).  scratch: ZERO-INITIALISED device buffer of
 * vdb_groupnorm_scratch_floats(B,HW) floats (partial sums, finalised mean/rstd, per-batch arrival counters); it may
 * be reused by later calls on the same stream (the kernels leave the counters at zero). Deterministic: no float atomics. */
int vdb_groupnorm_nsplit(int B, int HW);
long long vdb_groupnorm_scratch_floats(int B, int HW);
int vdb_groupnorm_nhwc(const void* x1, int C1, const void* x2, int C2, int B, int HW, int groups, const float* gamma,
                       const float* beta, float eps, int act, float* scratch, void* y, void* stream);

/* ---- LayerNorm over the last dim — BasicTransformerBlock.norm1/2/3 attention.py:206-208 ---------- */
int vdb_layernorm(const void* x, long long rows, int C, const float* gamma, const float* beta, float eps, void* y,
                  void* stream);

/* The kernel the last vdb_groupnorm_nhwc / vdb_layernorm call on this thread launched (host-side record, no device work):
 * out[0..n) receives {family, T0, T1, G, S, nsplit, grid x, grid y, grid z} (as many as n allows).  family 1: gn_bundle_kernel
 * <T0 = NVMAX, T1 = THREADS>, G groups per CTA, cluster size S; 2: gn_fused_kernel<T0 = NV>, nsplit CTAs per image; 3:
 * gn_stats_kernel + gn_apply_kernel, nsplit statistics CTAs per image (grid: the statistics kernel's); 4: layernorm_rg_kernel
 * <T0 = VPL, T1 = LPR>; 5: layernorm_kernel<T0 = MAXV, T1 = R>; 0: none yet.  Returns the number of fields (9).  For tests
 * and tools that need to know which kernel instantiation ran. */
int vdb_norm_last_plan(int* out, int n);

/* ---- nearest 2x upsample NHWC — Upsample.forward openaimodel.py:114, autokl_modules.py:54 -------- */
int vdb_upsample2x_nhwc(const void* x, int B, int H, int W, int C, void* y, void* stream);

/* ---- CLIP image preprocessing on the device — replaces the host PIL round trip of CLIPImageContextEncoder._encode,
 *      clip.py:88-94 (ToPILImage + CLIPProcessor: bicubic resize of the shortest side to 224, centre crop, rescale, normalise).
 *      Bit-exact with torchvision.ToPILImage + Pillow's 8-bit two-pass bicubic resampling; the int32 coefficient tables
 *      (bounds [out,2] = first tap, tap count; kk [out,ksize], 22 fractional bits) come from the host.  mean3 / std3 are HOST arrays. */
int vdb_clip_to_u8_hwc(const float* x, int n, int H, int W, void* y /* u8 [n,H,W,3] */, void* stream);
int vdb_resample_h_u8(const void* x /* u8 [n,H,Win,3] */, int n, int H, int Win, int Wout, const int* bounds, const int* kk,
                      int ksize, void* y /* u8 [n,H,Wout,3] */, void* stream);
int vdb_resample_v_crop_norm(const void* x /* u8 [n,Hin,W,3] */, int n, int Hin, int W, const int* bounds, const int* kk,
                             int ksize /* 0: no vertical resize */, int top, int left, int S, const float* mean3,
                             const float* std3, float* y /* fp32 [n,3,S,S] */, void* stream);

/* ---- im2col for tiny-Cin 3x3 convs (latent 4ch / RGB 3ch inputs): fp32 NHWC -> bf16 [B*H*W, Kpad]
 *      (x*in_scale + in_shift applied first: AutoencoderKL.encode's x*2-1, autokl.py:34) ----------- */
int vdb_im2col3x3_small(const float* x, int B, int H, int W, int Cin, int Kpad, float in_scale, float in_shift,
                        void* y, void* stream);

/* ---- fp32 NCHW <-> NHWC permute with y = x*mul + add [clamped to [0,1]] (autokl.py:47) ------------ */
int vdb_permute_f32(const float* x, int B, int C, long long HW, int to_nhwc, float mul, float add, int clamp01,
                    float* y, void* stream);
/* DiagonalGaussianDistribution.sample (distributions.py:24-37) fused with the latent scale of vae_encode
 * (vd.py:282-289): z = (mean + exp(0.5*clamp(logvar,-30,20)) * noise) * post_mul on NHWC fp32 moments [npix,2C] */
int vdb_gaussian_sample(const float* moments, const float* noise, int C, long long npix, float post_mul, float* z,
                        void* stream);
int vdb_cast_f32_bf16(const float* x, void* y, long long n, void* stream);
/* tiny 1x1 conv on fp32 NHWC: y = W (x*pre_mul) + b — quant_conv / post_quant_conv, autokl.py:26-27,36,45 and
 * the 1/latent_scale_factor of VD_v2_0.vae_decode, vd.py:291-296 */
int vdb_pointwise_small(const float* x, long long npix, int Cin, int Cout, const float* Wm, const float* bias,
                        float pre_mul, float* y, void* stream);
int vdb_cast_bf16_f32(const void* x, float* y, long long n, void* stream);

/* ---- timestep_embedding [cos|sin] — diffusion_utils.py:131-151 ---------------------------------
 * ts: device int64 [B], or a table indexed by *step_idx (broadcast to all B rows) when step_idx != NULL.
 * neg_log_period = (float)(-ln(max_period)). */
int vdb_timestep_embedding(const long long* ts, const int* step_idx, int B, int dim, float neg_log_period,
                           float* out, void* stream);

/* ---- skinny linear (M <= 16) — time_embed openaimodel.py:2629-2633, ResBlock.emb_layers :217-223 --
 * out[M,N] = act_out(act_in(x)[M,K] @ W[N,K]^T + bias); x/out fp32, W bf16; act 0 none, 1 SiLU. */
int vdb_linear_small(const float* x, int M, int K, const void* Wt, int N, const float* bias, int act_in, int act_out,
                     float* out, void* stream);

/* ---- CLIP context-encoder front/back ends — CLIPTextContextEncoder.encode clip.py:53-62, CLIPImageContextEncoder
 *      ._encode / ._encode_wmask clip.py:88-143 (the arithmetic of transformers.CLIPModel around the encoder layers,
 *      which run on vdb_layernorm / vdb_gemm_bf16 / vdb_attention_bf16).  Token streams are bf16 [B, Lp, C] with
 *      Lp = L rounded up to a multiple of 8 and zero pad rows. ------------------------------------------------- */
/* x[b,n] = token_embedding[tokens[b,n]] + position_embedding[n] */
int vdb_clip_text_embed(const long long* tokens, const float* tok_emb, const float* pos_emb, int B, int L, int Lp, int C,
                        void* x, void* stream);
/* PxP patches of NCHW fp32 pixels -> bf16 [B*(HW/P)^2, Kpad] rows in the patch_embedding conv's (c,py,px) order */
int vdb_patchify(const float* pixels, int B, int Cin, int HW, int P, int Kpad, void* y, void* stream);
/* [class_embedding ; patch embeddings] + position_embedding, optional per-token scale (masked variant) */
int vdb_vit_assemble(const void* patches, const float* cls, const float* pos, const float* tok_scale, int B, int L, int Lp,
                     int C, void* x, void* stream);
/* out[b,n,:] = z[b,n,:] / ||z[b, idx[b], :]|| [* row_scale[b,n]], fp32 [B,L,C] (idx NULL = token 0) */
int vdb_scale_by_row_norm(const void* z, const int* idx, const float* row_scale, int B, int L, int Lp, int C, float* out,
                          void* stream);

/* ---- row softmax (VAE AttnBlock, autokl_modules.py:186-188) ------------------------------------- */
int vdb_softmax_rows(const void* x, long long rows, int n, long long ld, float scale, void* y, void* stream);

/* ---- per-position affine + activation (text-latent flow, SURVEY §8f rank 4): y[r,i] = act(x[r,i] * gamma[i] + beta[i]) on bf16
 *      rows with fp32 parameters — the affine half of FCBlock's GroupNorm32 (openaimodel.py:2100-2112), whose gamma / beta are
 *      indexed by the FLATTENED channel c*sdim + s while vdb_groupnorm_nhwc normalises per channel c.  act 0 none, 1 SiLU. ---- */
int vdb_affine_act_rows(const void* x, long long rows, int n, const float* gamma, const float* beta, int act, void* y, void* stream);

/* ---- load-time weight repack (SURVEY §8b `vdb_pack_conv_weight`): checkpoint tensors in the reference's layouts (fp32,
 *      contiguous: Conv2d [Cout,Cin,kh,kw], Linear [out,in]) -> the bf16 K-major layouts the kernels above consume, so a
 *      binder that keeps the reference's own nn.Modules needs none of this repo's Python.  All device pointers. ------------ */
/* Conv2d weight [Cout, Cin, kh, kw] -> out[n, col0 + (ky*kw + kx)*Cin + ci] (row stride ldo): 3x3 convs of ResBlock.in_layers[2] /
 * out_layers[3] / Downsample.op / Upsample.conv (openaimodel.py:89-274) with col0 = 0, ldo = 9*Cin [+ Cskip]; a channel-changing
 * ResBlock's 1x1 skip_connection (:233-240) is appended as extra K columns with kh = kw = 1, col0 = 9*Cout_of_conv1. */
int vdb_pack_conv_weight(const float* w, int Cout, int Cin, int kh, int kw, void* out, long long ldo, long long col0, void* stream);
/* GEGLU.proj (attention.py:37-45) weight [2*n2, K] + bias [2*n2] -> rows interleaved per 256-row tile (128 value rows, then
 * their 128 gate rows) as the ACT_GEGLU epilogue of vdb_gemm_bf16 expects; n2 % 128 == 0. */
int vdb_pack_geglu(const float* w, const float* b, int n2, int K, void* w_out, float* b_out, void* stream);
/* CrossAttention.to_q / to_k / to_v weight [H*d, K] (attention.py:152-168) -> [H*dpad, K] with zero rows after each head's d
 * rows; dpad = vdb_attention_dk_pad(d) for q / k, vdb_attention_dv_pad(d) for v. */
int vdb_pad_heads(const float* w, int H, int d, int dpad, int K, void* out, void* stream);

/* ---- Optimus GPT-2 text decoder, one token step for R <= 16 rows — optimus_vae_next.decode / sample_single_sequence_conditional
 *      (optimus.py:662-688, 746-763) over GPT2ForLatentConnector_XX (optimus_gpt2.py:870-994, 1025-1082).  The step index is a
 *      device int (`step` = the input token's index s, advanced with vdb_add_int), so one captured graph serves every step.
 *      Residual stream, activations, logits and the KV cache are fp32; weights bf16 [N, K] (Conv1D's [in, out] transposed). ---- */
/* out[r, n] = act( LN(x)[r, :] . W[n, :] + bias[n] ), or out += that (accumulate != 0: the in-place residual add of Block.forward,
 * optimus_gpt2.py:236-240).  LN = LayerNorm(gamma, beta, eps) of the fp32 row when ln_gamma != NULL (ln_1 / ln_2 / ln_f fused into
 * c_attn / c_fc / lm_head), else the identity.  act VDB_ACT_NONE, VDB_ACT_GELU_TANH (MLP.act) or VDB_ACT_TANH.  Replaces
 * Conv1D.forward (modeling_utils.py:420-424) for attn.c_attn / attn.c_proj / mlp.c_fc / mlp.c_proj, transformer.linear / linear_emb
 * and lm_head; on the encoder side, BertPooler.forward (optimus_bert.py:364-376, VDB_ACT_TANH on the [CLS] rows: ldx = the token
 * stream's batch stride) and the z_mu half of BertForLatentConnector_XX.linear (optimus.py:741).  1 <= R <= 16, K % 32 == 0, K <= 3072, W 16-byte aligned with ldw % 8 == 0, x != out.  Reads every weight once. */
int vdb_textdec_gemv(const float* x, int R, long long K, long long ldx, const float* ln_gamma, const float* ln_beta, float ln_eps,
                     const void* W, long long N, long long ldw, const float* bias, int act, int accumulate, float* out, long long ldo,
                     void* stream);
/* Attention.forward for the one new query of each row (optimus_gpt2.py:205-227, _attn :152-175), d_head 64.  qkv [R, ldq] holds
 * c_attn's q | k | v (H*64 each); this step's k / v are appended at slot *step of kcache / vcache ([R][H][T][64] fp32, this
 * layer); the keys are the layer's latent slice mem[r, h*64 ..] (key == value, position 0) then slots 0 .. *step.  out [R, H*64].
 * src (may be NULL; beam search): cache slot j < *step of row r is read from physical row src[r * T + j] (int32 [R, T], every
 * entry in [0, R)) instead of row r; this step's k / v are still written at row r, slot *step.  A physical (row, slot) is written
 * once, at step == slot, so permuting beams permutes src rows and never moves the cache.  With src[r, j] = r the output equals
 * src == NULL's bitwise.  src is checked for 4-byte alignment when given; the other argument checks do not depend on it. */
int vdb_textdec_attention(const float* qkv, long long ldq, const float* mem, long long ldm, float* kcache, float* vcache,
                          const int* src, int R, int H, int T, const int* step, float scale, float* out, long long ldo, void* stream);
/* h[r, :] = wte[tokens[r, s]] + wpe[s + pos_offset] + emb[r, :], s = *step: the embedding sum of GPT2Model_XX.forward
 * (optimus_gpt2.py:941-948) with emb = linear_emb(z); pos_offset 1 (the latent is position 0).  fp32 wte [V, D], wpe [P, D]. */
int vdb_textdec_embed(const int* tokens, int ldt, const int* step, const float* wte, int V, const float* wpe, int P, int pos_offset,
                      const float* emb, int R, int D, float* h, void* stream);
/* torch.multinomial(softmax(logits / temperature)) of sample_single_sequence_conditional (optimus.py:662-688), by inverse CDF of
 * u in [0, 1): u = uniforms[r * ldu + s] when uniforms != NULL, else a Philox4x32-10 draw keyed by *seed (device u64) at counter
 * (r, s).  forced != NULL takes token s+1 from forced[r * ldf + s + 1] instead (teacher forcing).  Writes tokens[r * ldt + s + 1];
 * == eos sets done[r] = 1 and lengths[r] = s + 2; when s + 1 == max_len - 2 a non-eos row also gets eos at s + 2 (the reference
 * overwrites the max_len-th token, so its last draw is skipped).  Rows with done[r] != 0 are left frozen.  record (may be NULL)
 * receives the step's logits at record[(s * R + r) * V ..].
 * The top-k / nucleus cuts of top_k_top_p_filtering (reference optimus.py:690-719) restrict the draw.  Per row, l = logits /
 * temperature (fp32):
 *   top_k > 0: k = min(top_k, V); every token with l < (the k-th largest l) is removed.  Ties with the k-th value are kept, so
 *     more than k tokens can survive.
 *   then, when 0 < top_p < 1: the survivors' softmax, ordered by descending l; a survivor is kept when the probability mass
 *     before it in that order is <= top_p (the first one always is).  Tied tokens are taken in ascending vocabulary index, as a
 *     stable descending sort orders them: with boundary value v, M(>v) the mass above it and q the mass of one tied token, the
 *     first min(#ties, 1 + floor((top_p - M(>v)) / q)) ties are kept.  (The reference's torch.sort is not stable, so this is the
 *     one case its order leaves open.)  Masses are exp(l - max) / Z with Z the survivors' fp64 sum, compared as 64-bit fixed-point
 *     integers (units of 2^-62), so the cut is exact and repeatable.
 * top_k == 0 (or >= V) turns the top-k cut off, top_p == 0 or 1 the nucleus cut; with both off, or with forced tokens, the full
 * softmax is sampled (reference top_k 0, top_p 1: no filtering).  top_k = 1 is greedy decoding.  With a cut on, the draw is the
 * inverse CDF over the kept tokens only, in vocabulary order, their mass renormalised, with the same u; the filter stages the row
 * in shared memory, so V <= 53248.  top_k < 0 or top_p NaN or outside [0, 1] return VDB_ERR_INVALID before any launch, as do
 * the other argument errors. */
int vdb_textdec_sample(const float* logits, int R, int V, long long ldl, float temperature, int top_k, float top_p,
                       const unsigned long long* seed, const double* uniforms, int ldu, const int* forced, int ldf, int* tokens, int ldt,
                       int* done, int* lengths, const int* step, int eos, int max_len, float* record, void* stream);
/* One beam-search step, s = *step.  It stands in for the reference's optimus_vae.decode(z, strategy='beam', K)
 * (optimus.py:196-213), whose beam_search_decode does not exist in the reference's GPT-2, so this definition is the specification.
 * Rows r = latent * K + beam, R = n * K <= 16, 1 <= K <= 16.  Per beam: tokens [R, ldt] (token 0 = <BOS>), src [R, lds] (the
 * slot-to-row table of vdb_textdec_attention), scores fp64 [R], done [R], lengths [R].  Before step 0 the caller sets
 * every score to -inf except beam 0's (0), so the first step does not produce K copies of one hypothesis.
 *   logp_r(v) = log softmax(logits[r] / temperature)(v), all in fp64 from the fp32 logits (the division, max, exp, sum and log).
 *   Candidates: each live beam b crossed with each token v, score S_b + logp_b(v); each finished beam b as itself, score S_b.
 *   The K best become beams 0 .. K-1 in rank order; ties go to the lower parent beam, then the lower token id.
 *   New beam j with parent p: tokens[j, 0 .. s+1] = tokens[p, 0 .. s+1], src[j, 0 .. s-1] = src[p, 0 .. s-1], src[j, s] = p's row,
 *   and for a live parent tokens[j, s+1] = v.  v == eos finishes it (lengths = s + 2); otherwise, when s + 1 == max_len - 2, <eos>
 *   is appended at s + 2 unscored and it finishes (lengths = s + 3).  A finished beam keeps its score and length.
 * A latent is finished when all K beams are; live scores only decrease, so no live beam could have beaten them.  A beam's
 * scored-token count is min(lengths - 1, max_len - 2) (a chosen <eos> counts, a forced one does not).  Two launches: one CTA per
 * row (K best tokens via the top-k radix select of vdb_textdec_sample, ties in vocabulary order; at most K of one
 * row's tokens can enter the K best), then one CTA per latent.  The per-row pick orders a row's tokens by their fp32 logit
 * (ties to the lower token id), which is the order of S_b + logp_b(v) except where the fp64 rounding of l / temperature - lse or
 * of S_b + logp makes two different logits score equal: there the larger logit is kept, where the rule above would keep the
 * lower token id.  cand_tok int32 [R * K] and cand_logp fp64 [R * K] are scratch.
 * record (may be NULL): this step's logits per physical row, before the permutation, at record[(s * R + r) * V ..].
 * trace (may be NULL): fp64 [steps][R][3], the new beam's (parent beam index, token or -1 for a finished beam, score).
 * Deterministic.  Returns VDB_ERR_INVALID before any launch unless R = n * K <= 16, 1 <= K <= 16, K <= V <= 53248, ldl >= V,
 * temperature > 0, max_len >= 2, ldt >= max_len, lds >= 1, the pointers are non-null, the fp32 / int32 buffers 4-byte aligned and
 * the fp64 buffers 8-byte aligned.
 * A step with s >= lds or s + 1 >= ldt does nothing. */
int vdb_textdec_beam_step(const float* logits, int R, int V, long long ldl, float temperature, int K, int* tokens, int ldt, int* src,
                          int lds, double* scores, int* done, int* lengths, const int* step, int eos, int max_len, int* cand_tok,
                          double* cand_logp, float* record, double* trace, void* stream);
/* The repetition logits processors, in place on the fp32 logits [R, ldl] of one token step, before vdb_textdec_sample
 * or vdb_textdec_beam_step reads them (so those see, and `record` holds, the edited logits).  Row r's history is
 * h = tokens[r, 0 .. s], s = *step: <BOS>, then every token so far, including this step's input token.
 *   Repetition penalty p (finite, > 0; 1 = off), as HF's RepetitionPenaltyLogitsProcessor: for each DISTINCT id v of h with
 *     0 <= v < V, l[v] = l[v] < 0 ? l[v] * p : l[v] / p, IEEE round-to-nearest fp32 (a true division, no reciprocal).  An id is
 *     penalised once however often it occurs; ids outside [0, V) are ignored.
 *   No-repeat n-gram n (0 = off), as HF's NoRepeatNGramLogitsProcessor: for every 0 <= j <= s - n + 1 with
 *     h[j .. j+n-2] == h[s-n+2 .. s] (the last n - 1 tokens), l[h[j+n-1]] = -inf (ids outside [0, V) ignored).  n = 1 bans every
 *     token of h; nothing is banned while s + 1 < n.
 * The penalty runs first; the two commute (the penalty maps -inf to -inf).  Both act on the raw logits, before the sampler's
 * division by temperature and its top-k / nucleus cuts.  Rows with done[r] != 0 are left untouched, and a step with s < 0 or
 * s + 1 >= ldt does nothing.  Beam search applies the edit to each beam's own row; the beam step's fp64 log-softmax then
 * renormalises over the edited logits (HF edits log-probabilities and does not renormalise).
 * Precondition for small vocabularies: a banned token is never drawn, and never extends a beam, only while a row keeps at least
 * one finite logit (beam search: at least K finite logits per live beam).  V = 50260 with at most 32 history tokens always does.
 * One launch, one CTA per row, reading only the row's history and at most 2 (s + 1) of its logits.  penalty == 1 and ngram == 0
 * return 0 without a launch.  Returns VDB_ERR_INVALID before any launch unless 1 <= R <= 16, V >= 1, ldl >= V, ldt >= 1, penalty
 * is finite and > 0, 0 <= ngram <= ldt, the pointers are non-null and 4-byte aligned. */
int vdb_textdec_repetition(float* logits, int R, int V, long long ldl, const int* tokens, int ldt, const int* done, const int* step,
                           float penalty, int ngram, void* stream);

/* ---- semantic/style disentanglement of the image context — decompose / adjust_rank of the reference app.py:48-127 -----------
 * For each item b < n_items of x [n_items, m, n] (fp32, contiguous):  X = x - rowmean(x);  the randomized PCA of torch.pca_lowrank
 * (X, q, center=False, niter) with the Gaussian start R [m, q] (fp32, shared by all items; the reference's torch.randn(m, q)) gives
 * X ~= U diag(S) V^T;  x_new = U diag(S * factors) V^T + rowmean(x) [+ X - U diag(S) V^T when keep_remainder != 0];
 * out = x_new / std(x_new) * std(x) (unbiased, over all m * n elements of the item).  factors: device fp32 [q].  s_out (may be NULL):
 * device fp32 [n_items, q], the unscaled S, descending; u_out [n_items, m, q] and v_out [n_items, n, q] (may be NULL): U and V.
 * U = X V diag(1 / S) is undefined where S = 0: such a column of u_out is written as zeros (an item whose rows are each constant,
 * X = 0, has S = 0, U = 0 and V = 0, so U diag(S) V^T = 0 = X as for torch.pca_lowrank).
 * One launch (one 8-CTA cluster per item, X resident in shared memory); the QRs are CholeskyQR2 in fp64, so U and V differ from
 * torch's by column signs only.  Deterministic for a given R.
 * NULL x / R / factors / out, n_items < 1, niter < 0 or a misaligned x / out return VDB_ERR_INVALID; shapes other than n = 768,
 * q = 20, 40 <= m <= 320 (n_items <= 65535) return VDB_ERR_UNSUPPORTED.  out must not alias x. */
int vdb_rank_adjust_f32(const float* x, int n_items, int m, int n, const float* R, int q, int niter, const float* factors,
                        int keep_remainder, float* out, float* s_out, float* u_out, float* v_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VDB200_H_ */
