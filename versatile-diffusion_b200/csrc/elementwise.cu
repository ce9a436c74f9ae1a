// vdb200 — HBM-bound kernels of the sampling path (sm_90a): DDIM/CFG update, GroupNorm statistics
// and apply(+SiLU, +channel concat), LayerNorm, nearest 2x upsample, small-Cin im2col, skinny
// (M <= 16) linears for the timestep-embedding MLP, sinusoidal timestep embedding, row softmax,
// layout permutes. All vectorised to 16-byte accesses on NHWC / token-major bf16 tensors.
#include <curand_philox4x32_x.h>

#include "common.cuh"
#include "host_util.h"

namespace vdb {

// ---------------------------------------------------------------------------------------------
// K4: classifier-free-guidance mix + DDIM x_{t-1} update        (reference ddim.py:144-171)
//   e      = e_u + s * (e_c - e_u)
//   pred_x0= (x - sqrt(1-a_t) * e) / sqrt(a_t)
//   dir    = sqrt(1 - a_prev - sigma^2) * e
//   x_prev = sqrt(a_prev) * pred_x0 + dir + sigma * noise * temperature
// Explicit _rn intrinsics keep the op order / rounding of the reference's separate ATen ops
// (no FMA contraction), so fp32 results are bit-identical to the CPU oracle.
// coef = {a_t, a_prev, sigma_t, sqrt_one_minus_at}; if step_idx != null, row *step_idx of coef.
// ---------------------------------------------------------------------------------------------
__global__ void ddim_cfg_step_kernel(const float* __restrict__ e_uncond, const float* __restrict__ e_cond,
                                     const float* __restrict__ x, const float* __restrict__ noise,
                                     const float* __restrict__ coef, const int* __restrict__ step_idx,
                                     float scale, float temperature, float* __restrict__ x_prev,
                                     float* __restrict__ x_prev_dup, float* __restrict__ pred_x0, long long n) {
  const float* c = coef + (step_idx ? 4 * (*step_idx) : 0);
  const float a_t = c[0], a_prev = c[1], sigma = c[2], s1m = c[3];
  const float sqrt_at = __fsqrt_rn(a_t);
  const float sqrt_aprev = __fsqrt_rn(a_prev);
  const float dir_c = __fsqrt_rn(__fsub_rn(__fsub_rn(1.0f, a_prev), __fmul_rn(sigma, sigma)));
  for (long long i = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) * 4; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x * 4) {
    float ec[4], eu[4], xv[4], nz[4] = {0.f, 0.f, 0.f, 0.f}, xp[4], p0[4];
    if (i + 3 < n) {
      *reinterpret_cast<float4*>(ec) = __ldg(reinterpret_cast<const float4*>(e_cond + i));
      if (e_uncond) *reinterpret_cast<float4*>(eu) = __ldg(reinterpret_cast<const float4*>(e_uncond + i));
      *reinterpret_cast<float4*>(xv) = __ldg(reinterpret_cast<const float4*>(x + i));
      if (noise) *reinterpret_cast<float4*>(nz) = __ldg(reinterpret_cast<const float4*>(noise + i));
    } else {
      for (int q = 0; q < 4; ++q)
        if (i + q < n) {
          ec[q] = e_cond[i + q];
          if (e_uncond) eu[q] = e_uncond[i + q];
          xv[q] = x[i + q];
          if (noise) nz[q] = noise[i + q];
        }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float e = ec[q];
      if (e_uncond) e = __fadd_rn(eu[q], __fmul_rn(scale, __fsub_rn(ec[q], eu[q])));
      const float px0 = __fdiv_rn(__fsub_rn(xv[q], __fmul_rn(s1m, e)), sqrt_at);
      const float dir = __fmul_rn(dir_c, e);
      const float nn = __fmul_rn(__fmul_rn(sigma, nz[q]), temperature);
      xp[q] = __fadd_rn(__fadd_rn(__fmul_rn(sqrt_aprev, px0), dir), nn);
      p0[q] = px0;
    }
    if (i + 3 < n) {
      *reinterpret_cast<float4*>(x_prev + i) = *reinterpret_cast<float4*>(xp);
      if (x_prev_dup) *reinterpret_cast<float4*>(x_prev_dup + i) = *reinterpret_cast<float4*>(xp);
      if (pred_x0) *reinterpret_cast<float4*>(pred_x0 + i) = *reinterpret_cast<float4*>(p0);
    } else {
      for (int q = 0; q < 4; ++q)
        if (i + q < n) {
          x_prev[i + q] = xp[q];
          if (x_prev_dup) x_prev_dup[i + q] = xp[q];
          if (pred_x0) pred_x0[i + q] = p0[q];
        }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// CFG mix + one multistep DPM-Solver++ update (lib/model_zoo/dpm_solver.py), row *step_idx of the 8-float table
// coef = {P, Q, A, B, C, D, 0, 0}, in this op order (explicit _rn: no FMA contraction, so an fp32 CPU restatement is bitwise):
//   e   = e_u + s * (e_c - e_u)
//   x0  = P*x + Q*e                                  -> hist slot idx % 3, pred_x0
//   x'  = ((A*x + B*x0) [+ C*h1]) [+ D*h2]           h1 = hist slot (idx+1) % 3, h2 = slot (idx+2) % 3
// A bracketed term is skipped (and its slot not read) when its coefficient is exactly 0: the ring holds no data yet at the
// first steps.  The slot pointers are 16-byte aligned only when n % 4 == 0, so the ring is accessed by vectors only then.
//
// The stochastic form (DPMSolverSDESampler) adds column 6 of the row, N, and one Gaussian term:
//   x'  = (((A*x + B*x0) [+ C*h1]) [+ D*h2]) [+ N*z]
// z is the explicit noise when given, else four normals per element quad from philox_normals at counter (quad, idx, "sdes", 0)
// under the 64-bit key *seed.  At N == 0 the term is skipped and nothing is drawn or read, so such a row gives the bits of the
// deterministic kernel, which is the same body without the noise term.
// ---------------------------------------------------------------------------------------------
constexpr unsigned kSdeTag = 0x73646573u;       // "sdes": distinct from "inpt", "rgns" and "text"

__device__ __forceinline__ void philox_normals(unsigned long long key, unsigned quad, int step, unsigned tag, float z[4]);

template <bool kNoise>
__device__ __forceinline__ void dpmpp_cfg_step_body(const float* __restrict__ e_uncond, const float* __restrict__ e_cond,
                                                    const float* x, const float* __restrict__ coef,
                                                    const int* __restrict__ step_idx, float scale, float* __restrict__ hist,
                                                    float* x_next, float* __restrict__ x_next_dup, float* __restrict__ pred_x0,
                                                    long long n, const unsigned long long* __restrict__ seed,
                                                    const float* __restrict__ noise) {
  const int idx = *step_idx;
  const float* c = coef + 8 * idx;
  const float P = c[0], Q = c[1], A = c[2], B = c[3], C = c[4], D = c[5];
  float N = 0.f;
  unsigned long long key = 0ull;
  if (kNoise) {
    N = c[6];
    if (N != 0.f && !noise) key = *seed;
  }
  float* h0 = hist + static_cast<long long>(idx % 3) * n;
  const float* h1 = hist + static_cast<long long>((idx + 1) % 3) * n;
  const float* h2 = hist + static_cast<long long>((idx + 2) % 3) * n;
  const bool hvec = (n & 3) == 0;
  for (long long i = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) * 4; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x * 4) {
    const bool full = i + 3 < n;
    float ec[4], eu[4], xv[4], a1[4] = {0.f, 0.f, 0.f, 0.f}, a2[4] = {0.f, 0.f, 0.f, 0.f}, xn[4], p0[4];
    if (full) {
      *reinterpret_cast<float4*>(ec) = __ldg(reinterpret_cast<const float4*>(e_cond + i));
      if (e_uncond) *reinterpret_cast<float4*>(eu) = __ldg(reinterpret_cast<const float4*>(e_uncond + i));
      *reinterpret_cast<float4*>(xv) = *reinterpret_cast<const float4*>(x + i);   // x may alias x_next: no __ldg
    } else {
      for (int q = 0; q < 4; ++q)
        if (i + q < n) {
          ec[q] = e_cond[i + q];
          if (e_uncond) eu[q] = e_uncond[i + q];
          xv[q] = x[i + q];
        }
    }
    if (full && hvec) {
      if (C != 0.f) *reinterpret_cast<float4*>(a1) = *reinterpret_cast<const float4*>(h1 + i);
      if (D != 0.f) *reinterpret_cast<float4*>(a2) = *reinterpret_cast<const float4*>(h2 + i);
    } else {
      for (int q = 0; q < 4; ++q)
        if (i + q < n) {
          if (C != 0.f) a1[q] = h1[i + q];
          if (D != 0.f) a2[q] = h2[i + q];
        }
    }
    float zv[4] = {0.f, 0.f, 0.f, 0.f};
    if (kNoise && N != 0.f) {
      if (!noise) {
        philox_normals(key, static_cast<unsigned>(i >> 2), idx, kSdeTag, zv);
      } else if (full) {
        *reinterpret_cast<float4*>(zv) = __ldg(reinterpret_cast<const float4*>(noise + i));
      } else {
        for (int q = 0; q < 4; ++q)
          if (i + q < n) zv[q] = noise[i + q];
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float e = ec[q];
      if (e_uncond) e = __fadd_rn(eu[q], __fmul_rn(scale, __fsub_rn(ec[q], eu[q])));
      const float px0 = __fadd_rn(__fmul_rn(P, xv[q]), __fmul_rn(Q, e));
      float v = __fadd_rn(__fmul_rn(A, xv[q]), __fmul_rn(B, px0));
      if (C != 0.f) v = __fadd_rn(v, __fmul_rn(C, a1[q]));
      if (D != 0.f) v = __fadd_rn(v, __fmul_rn(D, a2[q]));
      if (kNoise && N != 0.f) v = __fadd_rn(v, __fmul_rn(N, zv[q]));
      xn[q] = v;
      p0[q] = px0;
    }
    if (full) {
      *reinterpret_cast<float4*>(x_next + i) = *reinterpret_cast<float4*>(xn);
      if (x_next_dup) *reinterpret_cast<float4*>(x_next_dup + i) = *reinterpret_cast<float4*>(xn);
      if (pred_x0) *reinterpret_cast<float4*>(pred_x0 + i) = *reinterpret_cast<float4*>(p0);
    } else {
      for (int q = 0; q < 4; ++q)
        if (i + q < n) {
          x_next[i + q] = xn[q];
          if (x_next_dup) x_next_dup[i + q] = xn[q];
          if (pred_x0) pred_x0[i + q] = p0[q];
        }
    }
    if (full && hvec) {
      *reinterpret_cast<float4*>(h0 + i) = *reinterpret_cast<float4*>(p0);
    } else {
      for (int q = 0; q < 4; ++q)
        if (i + q < n) h0[i + q] = p0[q];
    }
  }
}

__global__ void dpmpp_cfg_step_kernel(const float* __restrict__ e_uncond, const float* __restrict__ e_cond,
                                      const float* x, const float* __restrict__ coef, const int* __restrict__ step_idx,
                                      float scale, float* __restrict__ hist, float* x_next, float* __restrict__ x_next_dup,
                                      float* __restrict__ pred_x0, long long n) {
  dpmpp_cfg_step_body<false>(e_uncond, e_cond, x, coef, step_idx, scale, hist, x_next, x_next_dup, pred_x0, n, nullptr, nullptr);
}

__global__ void dpmpp_sde_cfg_step_kernel(const float* __restrict__ e_uncond, const float* __restrict__ e_cond,
                                          const float* x, const float* __restrict__ coef, const int* __restrict__ step_idx,
                                          float scale, float* __restrict__ hist, float* x_next, float* __restrict__ x_next_dup,
                                          float* __restrict__ pred_x0, long long n, const unsigned long long* __restrict__ seed,
                                          const float* __restrict__ noise) {
  dpmpp_cfg_step_body<true>(e_uncond, e_cond, x, coef, step_idx, scale, hist, x_next, x_next_dup, pred_x0, n, seed, noise);
}

// ---------------------------------------------------------------------------------------------
// Inpainting (lib/model_zoo/inpaint.py): blended latent diffusion.  After every sampler step the kept region (mask 0) is
// overwritten with the original latent re-noised to the step's target point, row *step_idx of the table {a, b}:
//   k  = a*x0 + b*z                       (explicit _rn: an fp32 CPU restatement is bitwise)
//   x' = m == 1 ? x' : m == 0 ? k : m*x' + (1 - m)*k
// z is the explicit noise when given, else the Philox4x32-10 stream below.  The exact selects at m = 0 and m = 1 make a hard
// mask keep x0 bit for bit at the last row {1, 0} and leave the generated region bit for bit as the step wrote it.
// ---------------------------------------------------------------------------------------------
constexpr unsigned kInpaintTag = 0x696e7074u;   // "inpt": the text decoder's stream uses "text" (0x74657874)

// the per-element blend of the inpainting and the inversion blends: m x + (1 - m) k, selecting exactly at m = 1 and m = 0
__device__ __forceinline__ float mask_blend(float m, float x, float k) {
  return m == 1.f ? x : m == 0.f ? k : __fadd_rn(__fmul_rn(m, x), __fmul_rn(__fsub_rn(1.f, m), k));
}

// Four standard normals of counter (quad, step, tag, 0) under a 64-bit key: two Box-Muller pairs, u = (b + 0.5) 2^-32 in
// fp64 (never 0 or 1), (r cos 2 pi u', r sin 2 pi u') with r = sqrt(-2 ln u), rounded to fp32.
__device__ __forceinline__ void philox_normals(unsigned long long key, unsigned quad, int step, unsigned tag, float z[4]) {
  const uint4 b = curand_Philox4x32_10(make_uint4(quad, static_cast<unsigned>(step), tag, 0u),
                                       make_uint2(static_cast<unsigned>(key), static_cast<unsigned>(key >> 32)));
  const unsigned w[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    const double u0 = (static_cast<double>(w[2 * p]) + 0.5) * 0x1.0p-32;
    const double u1 = (static_cast<double>(w[2 * p + 1]) + 0.5) * 0x1.0p-32;
    const double r = sqrt(-2.0 * log(u0));
    double s, c;
    sincospi(2.0 * u1, &s, &c);
    z[2 * p] = static_cast<float>(r * c);
    z[2 * p + 1] = static_cast<float>(r * s);
  }
}

__device__ __forceinline__ void inpaint_normals(unsigned long long key, unsigned quad, int step, float z[4]) {
  philox_normals(key, quad, step, kInpaintTag, z);
}

// x, x0, noise: fp32 NHWC [bs, hw, c] flattened to n = bs*hw*c; mask [bs | 1, hw], broadcast over c.  Element quad i/4 draws
// counter quad i/4.  The slots are 16-byte aligned only when n % 4 == 0, so vectors are used on full quads only.
__global__ void inpaint_blend_kernel(float* x, float* __restrict__ x_dup, const float* __restrict__ x0,
                                     const float* __restrict__ mask, int mask_per_item, const float* __restrict__ table,
                                     const int* __restrict__ step_idx, const unsigned long long* __restrict__ seed,
                                     const float* __restrict__ noise, long long n, long long hw, int c) {
  const int idx = *step_idx;
  const float a = table[2 * idx], b = table[2 * idx + 1];
  const unsigned long long key = noise ? 0ull : *seed;
  for (long long i = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) * 4; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x * 4) {
    const bool full = i + 3 < n;
    float xv[4], kv[4], zv[4];
    if (full) {
      *reinterpret_cast<float4*>(xv) = *reinterpret_cast<const float4*>(x + i);
      *reinterpret_cast<float4*>(kv) = __ldg(reinterpret_cast<const float4*>(x0 + i));
      if (noise) *reinterpret_cast<float4*>(zv) = __ldg(reinterpret_cast<const float4*>(noise + i));
    } else {
      for (int q = 0; q < 4; ++q)
        if (i + q < n) {
          xv[q] = x[i + q];
          kv[q] = x0[i + q];
          if (noise) zv[q] = noise[i + q];
        }
    }
    if (!noise) inpaint_normals(key, static_cast<unsigned>(i >> 2), idx, zv);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (i + q >= n) break;
      const long long pix = (i + q) / c;
      const float m = mask[mask_per_item ? pix : pix % hw];
      const float k = __fadd_rn(__fmul_rn(a, kv[q]), __fmul_rn(b, zv[q]));
      xv[q] = mask_blend(m, xv[q], k);
    }
    if (full) {
      *reinterpret_cast<float4*>(x + i) = *reinterpret_cast<float4*>(xv);
      if (x_dup) *reinterpret_cast<float4*>(x_dup + i) = *reinterpret_cast<float4*>(xv);
    } else {
      for (int q = 0; q < 4; ++q)
        if (i + q < n) {
          x[i + q] = xv[q];
          if (x_dup) x_dup[i + q] = xv[q];
        }
    }
  }
}

// the blend kernel's draws of step *step_idx for elements [0, n)
__global__ void inpaint_noise_kernel(const unsigned long long* __restrict__ seed, const int* __restrict__ step_idx, long long n,
                                     float* __restrict__ out) {
  const unsigned long long key = *seed;
  const int idx = *step_idx;
  for (long long i = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) * 4; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x * 4) {
    float z[4];
    inpaint_normals(key, static_cast<unsigned>(i >> 2), idx, z);
    for (int q = 0; q < 4; ++q)
      if (i + q < n) out[i + q] = z[q];
  }
}

// pixel mask [n, H8, W8] -> latent mask [n, H8/8, W8/8]: max over each 8x8 cell, first maximum in row-major order, NaN wins
// (max_pool2d's rule, so the result is bitwise torch's)
__global__ void mask_to_latent_kernel(const float* __restrict__ mask, int n, int H8, int W8, float* __restrict__ out) {
  const int H = H8 / 8, W = W8 / 8;
  const long long total = static_cast<long long>(n) * H * W;
  for (long long o = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; o < total;
       o += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int xw = static_cast<int>(o % W), yh = static_cast<int>((o / W) % H);
    const long long b = o / (static_cast<long long>(W) * H);
    const float* p = mask + (b * H8 + 8LL * yh) * W8 + 8 * xw;
    float best = p[0];
    for (int r = 0; r < 8; ++r)
      for (int s = 0; s < 8; ++s) {
        const float v = p[static_cast<long long>(r) * W8 + s];
        if (v > best || v != v) best = v;
      }
    out[o] = best;
  }
}

// out = m*decoded + (1 - m)*image per pixel, NCHW [n, c, hw], mask [n | 1, hw]; exact selects at m = 0 and m = 1
__global__ void composite_kernel(const float* decoded, const float* image, const float* __restrict__ mask, int mask_per_item,
                                 int c, long long hw, long long total, float* out) {
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = e % hw;
    const float m = mask[(mask_per_item ? e / (hw * c) * hw : 0) + p];
    const float d = decoded[e], im = image[e];
    out[e] = m == 1.f ? d : m == 0.f ? im : __fadd_rn(__fmul_rn(m, d), __fmul_rn(__fsub_rn(1.f, m), im));
  }
}

// ---------------------------------------------------------------------------------------------
// Editing (lib/model_zoo/edit.py): DDIM inversion and DiffEdit.
// ring[*step_idx + offset] = x: the inversion walk records its trajectory from inside the captured step graph, where a memcpy
// node's destination would be fixed at capture time.  A slot outside [0, slots) is not written.  n = elements per slot.
// ---------------------------------------------------------------------------------------------
__global__ void latent_store_slot_kernel(const float* __restrict__ x, float* __restrict__ ring, int slots,
                                         const int* __restrict__ step_idx, int offset, long long n) {
  const int s = *step_idx + offset;
  if (s < 0 || s >= slots) return;
  float* dst = ring + static_cast<long long>(s) * n;
  const bool vec = (n & 3) == 0;
  for (long long i = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) * 4; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x * 4) {
    if (vec) {
      *reinterpret_cast<float4*>(dst + i) = __ldg(reinterpret_cast<const float4*>(x + i));
    } else {
      for (int q = 0; q < 4; ++q)
        if (i + q < n) dst[i + q] = x[i + q];
    }
  }
}

// After forward step *step_idx of a walk from an inversion: x = m x + (1 - m) slot, slot = ring + *step_idx * n, the
// trajectory's latent at the step's target level.  mask [bs | 1, hw] broadcast over c; x_dup (may be NULL) receives a copy.
// A slot outside [0, slots) is not read: x and x_dup are left as they are.
__global__ void inversion_blend_kernel(float* x, float* __restrict__ x_dup, const float* __restrict__ ring, int slots,
                                       const float* __restrict__ mask, int mask_per_item, const int* __restrict__ step_idx,
                                       long long n, long long hw, int c) {
  const int s = *step_idx;
  if (s < 0 || s >= slots) return;
  const float* slot = ring + static_cast<long long>(s) * n;
  const bool vec = (n & 3) == 0;
  for (long long i = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) * 4; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x * 4) {
    const bool full = i + 3 < n;
    float xv[4], kv[4];
    if (full) {
      *reinterpret_cast<float4*>(xv) = *reinterpret_cast<const float4*>(x + i);
    } else {
      for (int q = 0; q < 4; ++q)
        if (i + q < n) xv[q] = x[i + q];
    }
    if (full && vec) {
      *reinterpret_cast<float4*>(kv) = __ldg(reinterpret_cast<const float4*>(slot + i));
    } else {
      for (int q = 0; q < 4; ++q)
        if (i + q < n) kv[q] = slot[i + q];
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (i + q >= n) break;
      const long long pix = (i + q) / c;
      xv[q] = mask_blend(mask[mask_per_item ? pix : pix % hw], xv[q], kv[q]);
    }
    if (full) {
      *reinterpret_cast<float4*>(x + i) = *reinterpret_cast<float4*>(xv);
      if (x_dup) *reinterpret_cast<float4*>(x_dup + i) = *reinterpret_cast<float4*>(xv);
    } else {
      for (int q = 0; q < 4; ++q)
        if (i + q < n) {
          x[i + q] = xv[q];
          if (x_dup) x_dup[i + q] = xv[q];
        }
    }
  }
}

// DiffEdit's mask, one CTA per image b.  e_* fp32 NHWC [D*bs, hw, c], draw d of image b at row d*bs + b.  Per pixel p, in fp32:
//   E = e_u + s (e_c - e_u)  (e_c when e_u is NULL),  acc = sum over d, then c, of |E_tgt - E_src|,  dist = acc / (D c)
//   mu = (sum over p of dist) / hw  (per-thread sums in p order, then a fixed tree over the threads),  cap = ratio mu
//   out = cap > 0 && min(dist, cap) / cap >= 0.5 ? 1 : 0
// dist is parked in out between the two passes.  The order of every sum depends only on the shape: bit-reproducible.
constexpr int kDiffEditThreads = 256;

__global__ void __launch_bounds__(kDiffEditThreads) diffedit_mask_kernel(
    const float* __restrict__ es_u, const float* __restrict__ es_c, float s_src, const float* __restrict__ et_u,
    const float* __restrict__ et_c, float s_tgt, int D, int bs, long long hw, int c, float ratio, float* out) {
  __shared__ float red[kDiffEditThreads];
  const int b = blockIdx.x;
  float* o = out + static_cast<long long>(b) * hw;
  const float dc = static_cast<float>(static_cast<long long>(D) * c);
  float part = 0.f;
  for (long long p = threadIdx.x; p < hw; p += blockDim.x) {
    float acc = 0.f;
    for (int d = 0; d < D; ++d) {
      const long long base = ((static_cast<long long>(d) * bs + b) * hw + p) * c;
      for (int ch = 0; ch < c; ++ch) {
        float es = es_c[base + ch], et = et_c[base + ch];
        if (es_u) es = __fadd_rn(es_u[base + ch], __fmul_rn(s_src, __fsub_rn(es, es_u[base + ch])));
        if (et_u) et = __fadd_rn(et_u[base + ch], __fmul_rn(s_tgt, __fsub_rn(et, et_u[base + ch])));
        acc = __fadd_rn(acc, fabsf(__fsub_rn(et, es)));
      }
    }
    const float dist = __fdiv_rn(acc, dc);
    o[p] = dist;
    part = __fadd_rn(part, dist);
  }
  red[threadIdx.x] = part;
  __syncthreads();
  for (int w = kDiffEditThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] = __fadd_rn(red[threadIdx.x], red[threadIdx.x + w]);
    __syncthreads();
  }
  const float cap = __fmul_rn(ratio, __fdiv_rn(red[0], static_cast<float>(hw)));
  for (long long p = threadIdx.x; p < hw; p += blockDim.x)
    o[p] = (cap > 0.f && __fdiv_rn(fminf(o[p], cap), cap) >= 0.5f) ? 1.f : 0.f;
}

// Prompt-to-Prompt's local blend (lib/model_zoo/prompt_edit.py) after a step, when flags[*step_idx] != 0.  One CTA per target image
// b = 1 .. n-1 of x fp32 NHWC [n, H, W, C]; map fp32 [n, h, w], the word maps of the conditional rows.  For s in {0, b}:
//   pooled_s = 3x3 max-pool (stride 1, pad 1) of map[s];  mx_s = max of pooled_s
//   mask_s(y, x) = mx_s > 0 && pooled_s[floor(y h / H), floor(x w / W)] / mx_s > threshold   (division rounded to nearest)
// then x_b = mask_blend(m, x_b, x_0) with m = mask_b || mask_0 in {0, 1}: a selection, so outside the mask x_b takes x_0's bits.
// x_dup (may be NULL) receives the rows written.  Max is order-independent, so the result is bit-reproducible.
constexpr int kBlendThreads = 256, kBlendMaxMap = 4096;

__global__ void __launch_bounds__(kBlendThreads) local_blend_kernel(float* x, float* x_dup, const float* __restrict__ map,
                                                                    const int* __restrict__ flags, const int* __restrict__ step_idx,
                                                                    int H, int W, int C, int h, int w, float threshold) {
  __shared__ float pooled[2][kBlendMaxMap];
  __shared__ float red[2][kBlendThreads];
  if (!flags[*step_idx]) return;
  const int b = blockIdx.x + 1;
  const int hw = h * w;
  float part[2] = {-INFINITY, -INFINITY};
  for (int i = threadIdx.x; i < hw; i += kBlendThreads) {
    const int y = i / w, xx = i % w;
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const float* m = map + static_cast<long long>(s ? b : 0) * hw;
      float v = -INFINITY;
      for (int dy = -1; dy <= 1; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
          const int yy = y + dy, xw = xx + dx;
          if (yy >= 0 && yy < h && xw >= 0 && xw < w) v = fmaxf(v, m[yy * w + xw]);
        }
      pooled[s][i] = v;
      part[s] = fmaxf(part[s], v);
    }
  }
  red[0][threadIdx.x] = part[0];
  red[1][threadIdx.x] = part[1];
  __syncthreads();
  for (int k = kBlendThreads / 2; k > 0; k >>= 1) {
    if (threadIdx.x < k)
      for (int s = 0; s < 2; ++s) red[s][threadIdx.x] = fmaxf(red[s][threadIdx.x], red[s][threadIdx.x + k]);
    __syncthreads();
  }
  const float mx0 = red[0][0], mxb = red[1][0];
  const long long hwc = static_cast<long long>(H) * W * C;
  const float* x0 = x;
  float* xb = x + b * hwc;
  float* db = x_dup ? x_dup + b * hwc : nullptr;
  for (long long e = threadIdx.x; e < hwc; e += kBlendThreads) {
    const long long pix = e / C;
    const int y = static_cast<int>(pix / W), xx = static_cast<int>(pix % W);
    const int cell = static_cast<int>(static_cast<long long>(y) * h / H) * w + static_cast<int>(static_cast<long long>(xx) * w / W);
    const bool m0 = mx0 > 0.f && __fdiv_rn(pooled[0][cell], mx0) > threshold;
    const bool mb = mxb > 0.f && __fdiv_rn(pooled[1][cell], mxb) > threshold;
    const float v = mask_blend(m0 || mb ? 1.f : 0.f, xb[e], x0[e]);
    xb[e] = v;
    if (db) db[e] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// MultiDiffusion region prompts (lib/model_zoo/regions.py) on a window layout; a panorama's window fusion (lib/model_zoo/
// panorama.py) is the walk with no regions, R = 0.  The canvas is fp32 NHWC [bs, H, W, C]; window g = iy*nx + ix covers rows
// oy[iy] .. oy[iy]+h-1 and columns (ox[ix] + j) mod W, j < w, so a circular layout reads across the W seam and every other layout
// never wraps.  VW = 4 moves whole float4s (C % 4 == 0, the latent's 4 channels); VW = 1 moves one float at a time.
// masks fp32 [R, bs, H, W] on the canvas, region r >= 1 at row r - 1; region 0 is the background, of weight m_0 = max(0, 1 - S),
// S = m_1 + ... + m_R.  A chunk's UNet batch is ub + R + 1 blocks of [k*bs, h, w, C]: ub u blocks (0; 1, region 0's; or R + 1, one
// per region), then the R + 1 c blocks, region r at c block r.  Row j*bs + b of a block is window first + j of image b.
// ---------------------------------------------------------------------------------------------
constexpr unsigned kRegionTag = 0x72676e73u;   // "rgns"
constexpr int kRegionsMax = 8;

// the background entry of region r >= 1, image b at step `step`: floor(w nb / 2^32), w the first word at counter
// (r*bs + b, step, "rgns", 1)
__device__ __forceinline__ int region_pick(unsigned long long key, int r, int b, int bs, int step, int nb) {
  const uint4 v = curand_Philox4x32_10(make_uint4(static_cast<unsigned>(r * bs + b), static_cast<unsigned>(step), kRegionTag, 1u),
                                       make_uint2(static_cast<unsigned>(key), static_cast<unsigned>(key >> 32)));
  return static_cast<int>((static_cast<unsigned long long>(v.x) * static_cast<unsigned>(nb)) >> 32);
}

// canvas x -> the chunk's batch out.  Block 0 of each half, and every block while the step's flag is off (or rows is NULL), is an
// exact copy.  While it is on (row *step_idx of rows {on, a, b, 0}), region r >= 1 reads m x + (1 - m) (a bg + b z): the exact
// selects of mask_blend, k = a*bg + b*z rounded as the inpainting blend's.  z: noise (canvas NHWC) when given, else four normals
// per canvas element quad at counter (quad, step, "rgns", 0); bg: row region_pick of the backgrounds [nb, C].
template <int VW>
__global__ void region_gather_kernel(const float* __restrict__ x, int bs, int H, int W, int C, const int* __restrict__ oy,
                                     const int* __restrict__ ox, int nx, int h, int w, int first, int k, int ub,
                                     const float* __restrict__ masks, const float* __restrict__ rows,
                                     const int* __restrict__ step_idx, const unsigned long long* __restrict__ seed,
                                     const float* __restrict__ bg, int nb, const float* __restrict__ noise, long long total,
                                     float* __restrict__ out) {
  int idx = 0;
  bool on = false;
  float a = 0.f, bz = 0.f;
  if (rows) {
    idx = *step_idx;
    on = rows[4 * idx] != 0.f;
    a = rows[4 * idx + 1];
    bz = rows[4 * idx + 2];
  }
  const unsigned long long key = on ? *seed : 0ull;
  const int cv = C / VW;
  const int kb = k * bs;
  const long long plane = static_cast<long long>(bs) * H * W;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(e % cv) * VW;
    long long p = e / cv;
    const int wx = static_cast<int>(p % w);
    p /= w;
    const int wy = static_cast<int>(p % h);
    const long long row = p / h;
    const int blk = static_cast<int>(row / kb), rb = static_cast<int>(row % kb);
    const int b = rb % bs, g = first + rb / bs;
    const int r = blk < ub ? (ub == 1 ? 0 : blk) : blk - ub;
    int sx = ox[g % nx] + wx;
    if (sx >= W) sx -= W;
    const long long pix = (static_cast<long long>(b) * H + oy[g / nx] + wy) * W + sx;
    const long long src = pix * C + c;
    float v[VW];
    if (VW == 4) *reinterpret_cast<float4*>(v) = __ldg(reinterpret_cast<const float4*>(x + src));
    else v[0] = __ldg(x + src);
    if (on && r > 0) {
      const float m = __ldg(masks + (r - 1) * plane + pix);
      if (m != 1.f) {
        const float* bgr = bg + static_cast<long long>(region_pick(key, r, b, bs, idx, nb)) * C + c;
        float z[4];
        if (noise) {
          if (VW == 4) *reinterpret_cast<float4*>(z) = __ldg(reinterpret_cast<const float4*>(noise + src));
          else z[0] = __ldg(noise + src);
        } else {
          philox_normals(key, static_cast<unsigned>(src >> 2), idx, kRegionTag, z);
          if (VW == 1) {    // the element's lane of its quad, selected without indexing the array by a runtime value
            const int lane = static_cast<int>(src & 3);
            z[0] = lane == 0 ? z[0] : lane == 1 ? z[1] : lane == 2 ? z[2] : z[3];
          }
        }
#pragma unroll
        for (int q = 0; q < VW; ++q) {       // VW == 4: src is a multiple of 4, so lane q is element src + q
          const float kq = __fadd_rn(__fmul_rn(a, __ldg(bgr + q)), __fmul_rn(bz, z[q]));
          v[q] = mask_blend(m, v[q], kq);
        }
      }
    }
    if (VW == 4) *reinterpret_cast<float4*>(out + e * 4) = *reinterpret_cast<float4*>(v);
    else out[e] = v[0];
  }
}

// the gather's draws of step *step_idx: z for canvas elements [0, n), and picks[(r - 1)*bs + b] for r = 1..R
__global__ void region_noise_kernel(const unsigned long long* __restrict__ seed, const int* __restrict__ step_idx, long long n,
                                    int R, int bs, int nb, float* __restrict__ z, int* __restrict__ picks) {
  const unsigned long long key = *seed;
  const int idx = *step_idx;
  const long long quads = (n + 3) / 4;
  const long long total = quads > static_cast<long long>(R) * bs ? quads : static_cast<long long>(R) * bs;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    if (i < quads) {
      float v[4];
      philox_normals(key, static_cast<unsigned>(i), idx, kRegionTag, v);
      for (int q = 0; q < 4; ++q)
        if (4 * i + q < n) z[4 * i + q] = v[q];
    }
    if (i < static_cast<long long>(R) * bs)
      picks[i] = region_pick(key, static_cast<int>(i / bs) + 1, static_cast<int>(i % bs), bs, idx, nb);
  }
}

// The weighted merge of windows [first, first+k): eps [halves*(R+1)*k*bs, h, w, C], block s*(R+1) + r; out [halves*bs, H, W, C].
// The windows covering row y are iy in [cover_y[2y], cover_y[2y+1]); those covering column x are ix in [cover_x[4x], cover_x[4x+1])
// then [cover_x[4x+2], cover_x[4x+3]), in ascending order.  Per element p: S = m_1 + ... + m_R (ascending, rounded; the first mask
// sets S, and S = 0 when R = 0), m_0 = max(0, 1 - S), D = m_0 + S.  Over its covering windows in ascending index, and r = 0..R
// inside each, every term m_r e_{j,r} of nonzero weight is one rounded product: the first sets out, later ones are added; the
// launch holding the last window divides once by n D.  Calls over consecutive ranges therefore make the same operations in the
// same order as one call over all windows: the result does not depend on the chunking.  Some weight is nonzero at every element
// (D >= 1 - 2^-24), so every covering window adds at least one term.
// With no regions (R = 0, masks unused) this is the uniform window average bit for bit: m_0 = max(0, 1 - 0) = 1, each term
// 1 * e_j is e_j exactly for every finite or infinite value, so the first window's eps sets out and each later one is added with
// one rounding; and n D = n * (1 + 0) is n exactly, so the last launch divides once by the count.  An element with one covering
// window therefore gets that window's eps bit for bit.
template <int VW>
__global__ void region_merge_kernel(const float* __restrict__ eps, int bs, int H, int W, int C, const int* __restrict__ oy,
                                    const int* __restrict__ ox, const int* __restrict__ cover_y, const int* __restrict__ cover_x,
                                    int nx, int h, int w, int first, int k, int R, const float* __restrict__ masks, long long total,
                                    float* __restrict__ out) {
  const int cv = C / VW;
  const int last = first + k;
  const long long plane = static_cast<long long>(h) * w * C, mplane = static_cast<long long>(bs) * H * W;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(e % cv) * VW;
    long long p = e / cv;
    const int x = static_cast<int>(p % W);
    p /= W;
    const int y = static_cast<int>(p % H);
    const long long ob = p / H;                               // output row s*bs + b
    const int s = static_cast<int>(ob / bs), b = static_cast<int>(ob % bs);
    const int y0 = cover_y[2 * y], y1 = cover_y[2 * y + 1];
    const int4 cx = *reinterpret_cast<const int4*>(cover_x + 4 * x);
    const int xlo = cx.y > cx.x ? cx.x : cx.z, xhi = cx.w > cx.z ? cx.w - 1 : cx.y - 1;
    const int g_first = y0 * nx + xlo, g_last = (y1 - 1) * nx + xhi;
    if (g_last < first || g_first >= last) continue;          // no covering window in this range
    const float* mp = masks + (static_cast<long long>(b) * H + y) * W + x;
    float S = R ? __ldg(mp) : 0.f;
    for (int r = 2; r <= R; ++r) S = __fadd_rn(S, __ldg(mp + (r - 1) * mplane));
    const float m0 = fmaxf(0.f, __fsub_rn(1.f, S));
    float acc[VW];
    float* o = out + ((ob * H + y) * W + x) * C + c;
    bool started = g_first < first;
    if (started) {
      if (VW == 4) *reinterpret_cast<float4*>(acc) = *reinterpret_cast<const float4*>(o);
      else acc[0] = o[0];
    }
    for (int iy = y0; iy < y1; ++iy) {
      const int wy = y - oy[iy];
      for (int part = 0; part < 2; ++part) {
        const int a0 = part ? cx.z : cx.x, a1 = part ? cx.w : cx.y;
        for (int ix = a0; ix < a1; ++ix) {
          const int g = iy * nx + ix;
          if (g < first || g >= last) continue;
          int wx = x - ox[ix];
          if (wx < 0) wx += W;
          const float* src = eps + ((static_cast<long long>(s) * (R + 1) * k + (g - first)) * bs + b) * plane +
                             (static_cast<long long>(wy) * w + wx) * C + c;
          for (int r = 0; r <= R; ++r, src += k * bs * plane) {
            const float m = r == 0 ? m0 : __ldg(mp + (r - 1) * mplane);
            if (m == 0.f) continue;
            float v[VW];
            if (VW == 4) *reinterpret_cast<float4*>(v) = __ldg(reinterpret_cast<const float4*>(src));
            else v[0] = __ldg(src);
#pragma unroll
            for (int q = 0; q < VW; ++q) acc[q] = started ? __fadd_rn(acc[q], __fmul_rn(m, v[q])) : __fmul_rn(m, v[q]);
            started = true;
          }
        }
      }
    }
    if (g_last < last) {
      const float dn = __fmul_rn(static_cast<float>((y1 - y0) * ((cx.y - cx.x) + (cx.w - cx.z))), __fadd_rn(m0, S));
#pragma unroll
      for (int q = 0; q < VW; ++q) acc[q] = __fdiv_rn(acc[q], dn);
    }
    if (VW == 4) *reinterpret_cast<float4*>(o) = *reinterpret_cast<float4*>(acc);
    else o[0] = acc[0];
  }
}

// Self-attention guidance (lib/model_zoo/sag.py).  sag_degrade_kernel: one CTA per (kSagTile x kSagTile pixels, image b).  The
// tile's x0 with its 4-wide reflected halo sits in shared memory; the 9-tap Gaussian runs along rows into a second buffer, then
// along columns, each sum in tap order.  The mask cell of pixel (y, x) is mass[b, (y hm / H) wm + x wm / W] > 1.
constexpr int kSagTile = 16, kSagHalo = 4, kSagTaps = 2 * kSagHalo + 1, kSagMaxC = 8, kSagMaxMap = 4096;

struct SagTaps {
  float g[kSagTaps];
};

__device__ __forceinline__ int reflect_index(int i, int n) {
  i = i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i);
  return min(max(i, 0), n - 1);        // rows past the reflected range feed no pixel of the image
}

__global__ void __launch_bounds__(kSagTile * kSagTile) sag_degrade_kernel(
    const float* __restrict__ x, const float* __restrict__ e, const float* __restrict__ mass, const float* __restrict__ table,
    const int* __restrict__ step_idx, SagTaps taps, int H, int W, int C, int hm, int wm, float* __restrict__ out) {
  constexpr int S = kSagTile + 2 * kSagHalo;
  __shared__ float sx[S * S * kSagMaxC];
  __shared__ float sh[S * kSagTile * kSagMaxC];
  const int idx = *step_idx;
  const float sa = table[2 * idx], s1 = table[2 * idx + 1];
  const int b = blockIdx.z, y0 = blockIdx.y * kSagTile, x0 = blockIdx.x * kSagTile;
  const long long img = static_cast<long long>(b) * H * W * C;
  for (int i = threadIdx.x; i < S * S * C; i += blockDim.x) {
    const int c = i % C, lx = (i / C) % S, ly = i / (C * S);
    const long long g = img + (static_cast<long long>(reflect_index(y0 + ly - kSagHalo, H)) * W +
                               reflect_index(x0 + lx - kSagHalo, W)) * C + c;
    sx[i] = __fdiv_rn(__fsub_rn(x[g], __fmul_rn(s1, e[g])), sa);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < S * kSagTile * C; i += blockDim.x) {
    const int c = i % C, tx = (i / C) % kSagTile, ly = i / (C * kSagTile);
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < kSagTaps; ++k) acc = fmaf(taps.g[k], sx[(ly * S + tx + k) * C + c], acc);
    sh[i] = acc;
  }
  __syncthreads();
  const int ty = threadIdx.x / kSagTile, tx = threadIdx.x % kSagTile, y = y0 + ty, xx = x0 + tx;
  if (y >= H || xx >= W) return;
  const bool m = mass[static_cast<long long>(b) * hm * wm + (y * hm / H) * wm + xx * wm / W] > 1.f;
  for (int c = 0; c < C; ++c) {
    float v = sx[((ty + kSagHalo) * S + tx + kSagHalo) * C + c];
    if (m) {
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < kSagTaps; ++k) acc = fmaf(taps.g[k], sh[((ty + k) * kSagTile + tx) * C + c], acc);
      v = acc;
    }
    const long long g = img + (static_cast<long long>(y) * W + xx) * C + c;
    out[g] = __fadd_rn(__fmul_rn(sa, v), __fmul_rn(s1, e[g]));
  }
}

// d = s (e_src - e_deg), e_src = e_u when given (CFG), else e_c; added to e_c and e_u in place
__global__ void sag_guide_kernel(float* e_u, float* e_c, const float* __restrict__ e_deg, float s, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float ec = e_c[i];
    if (e_u) {
      const float eu = e_u[i];
      const float d = __fmul_rn(s, __fsub_rn(eu, e_deg[i]));
      e_u[i] = __fadd_rn(eu, d);
      e_c[i] = __fadd_rn(ec, d);
    } else {
      e_c[i] = __fadd_rn(ec, __fmul_rn(s, __fsub_rn(ec, e_deg[i])));
    }
  }
}

__global__ void add_int_kernel(int* p, int delta) { *p += delta; }

// y = c0*x0 + c1*x1 + c2*x2 + c3*x3 (null pointers skipped) — the Adams-Bashforth eps combination of the PLMS
// sampler (north-star addition; absent from the reference)
__global__ void lincomb4_kernel(const float* __restrict__ x0, const float* __restrict__ x1, const float* __restrict__ x2,
                                const float* __restrict__ x3, float c0, float c1, float c2, float c3,
                                float* __restrict__ y, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float v = c0 * x0[i];
    if (x1) v += c1 * x1[i];
    if (x2) v += c2 * x2[i];
    if (x3) v += c3 * x3[i];
    y[i] = v;
  }
}

// y = a*x + b*z  (VD_v2_0.q_sample, vd.py:221-224: sqrt(ac_t)*x0 + sqrt(1-ac_t)*noise)
__global__ void axpby_kernel(const float* __restrict__ x, const float* __restrict__ z, float a, float b,
                             float* __restrict__ y, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    y[i] = __fadd_rn(__fmul_rn(a, x[i]), __fmul_rn(b, z[i]));
}

// ---------------------------------------------------------------------------------------------
// GroupNorm(32) statistics over NHWC bf16, optional two-source channel concat.
// grid (nsplit, B), block 512. Thread t owns channel-vector v = t % V (8 channels) and pixel lane
// t / V; per-thread fp32 sum / sum-of-squares, then shared-memory atomics into the 32 groups.
// partial[b][split][g][2] = {sum, sumsq} over this CTA's pixel range (no global atomics: the
// result is deterministic, which the N-rank == 1-rank bit-reproducibility test relies on).
// ---------------------------------------------------------------------------------------------
constexpr int kGnThreads = 512;

// scratch layout (floats): [2*kGnMaxBatch arrival / departure counters (int), always at the front so that calls with different
// shapes never alias them][B*2*groups {mean, rstd}][B*nsplit*2*groups partial sums]
constexpr int kGnMaxBatch = 1024;
__global__ void __launch_bounds__(kGnThreads) gn_stats_kernel(const __nv_bfloat16* __restrict__ x1, int C1,
                                                              const __nv_bfloat16* __restrict__ x2, int C2,
                                                              int HW, int groups, float eps, float* __restrict__ scratch) {
  const int C = C1 + C2;
  const int V = C / 8;
  const int cpg = C / groups;
  const int b = blockIdx.y, split = blockIdx.x, nsplit = gridDim.x, B = gridDim.y;
  int* counters = reinterpret_cast<int*>(scratch);
  float* stats = scratch + 2 * kGnMaxBatch;
  float* partial = stats + static_cast<size_t>(B) * 2 * groups;
  const int pix_per = (HW + nsplit - 1) / nsplit;
  const int p_begin = split * pix_per;
  const int p_end = min(HW, p_begin + pix_per);
  // deterministic two-level reduction (no float atomics): [pixel lane][channel][sum|sumsq] -> channel -> group
  __shared__ float part[kGnThreads * 16];
  __shared__ int is_last;
  const int lanes = kGnThreads / V;  // pixel lanes (>= 1 because V <= 512)
  const int v = threadIdx.x % V;
  const int pl = threadIdx.x / V;
  if (pl < lanes) {
    float s[8], q[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; }
    const bool first = v * 8 < C1;
    const __nv_bfloat16* src = first ? x1 + static_cast<long long>(b) * HW * C1 + v * 8
                                     : x2 + static_cast<long long>(b) * HW * C2 + (v * 8 - C1);
    const long long Cs = first ? C1 : C2;
    int p = p_begin + pl;
    for (; p + 3 * lanes < p_end; p += 4 * lanes) {   // 4 independent 16-byte loads in flight per thread
      uint4 u[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(src + (p + k * lanes) * Cs));
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t w[4] = {u[k].x, u[k].y, u[k].z, u[k].w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = unpack_bf16x2(w[i]);
          s[2 * i] += f.x; q[2 * i] += f.x * f.x;
          s[2 * i + 1] += f.y; q[2 * i + 1] += f.y * f.y;
        }
      }
    }
    for (; p < p_end; p += lanes) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(src + p * Cs));
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack_bf16x2(w[i]);
        s[2 * i] += f.x; q[2 * i] += f.x * f.x;
        s[2 * i + 1] += f.y; q[2 * i + 1] += f.y * f.y;
      }
    }
    float* dst = part + (static_cast<size_t>(pl) * V + v) * 16;
#pragma unroll
    for (int i = 0; i < 8; ++i) { dst[i] = s[i]; dst[8 + i] = q[i]; }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kGnThreads) {
    float s = 0.f, q = 0.f;
    for (int l = 0; l < lanes; ++l) {
      const float* src = part + (static_cast<size_t>(l) * V + c / 8) * 16 + (c & 7);
      s += src[0]; q += src[8];
    }
    float* own = part + (static_cast<size_t>(c / 8)) * 16 + (c & 7);  // lane-0 slot of this channel (only this thread touches it)
    own[0] = s; own[8] = q;
  }
  __syncthreads();
  if (threadIdx.x < groups) {
    float s = 0.f, q = 0.f;
    for (int c = threadIdx.x * cpg; c < (threadIdx.x + 1) * cpg; ++c) {
      const float* src = part + (static_cast<size_t>(c / 8)) * 16 + (c & 7);
      s += src[0]; q += src[8];
    }
    float* o = partial + (static_cast<long long>(b) * nsplit + split) * 2 * groups + 2 * threadIdx.x;
    o[0] = s; o[1] = q;
  }
  // the last CTA of this batch item to finish folds the partials (fixed order => deterministic) into mean / rstd
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(&counters[b], 1) == nsplit - 1);
  __syncthreads();
  if (is_last) {
    __threadfence();
    if (threadIdx.x < groups) {
      float s = 0.f, q = 0.f;
      const float* pp = partial + static_cast<long long>(b) * nsplit * 2 * groups + 2 * threadIdx.x;
#pragma unroll 4
      for (int i = 0; i < nsplit; ++i) { s += __ldcg(pp + static_cast<long long>(i) * 2 * groups); q += __ldcg(pp + static_cast<long long>(i) * 2 * groups + 1); }
      const float inv_n = 1.0f / (static_cast<float>(HW) * cpg);
      const float mean = s * inv_n;
      const float var = fmaxf(q * inv_n - mean * mean, 0.f);
      stats[(static_cast<long long>(b) * groups + threadIdx.x) * 2] = mean;
      stats[(static_cast<long long>(b) * groups + threadIdx.x) * 2 + 1] = rsqrtf(var + eps);
    }
    if (threadIdx.x == 0) counters[b] = 0;   // ready for the next launch (stream-ordered reuse of the scratch)
  }
}

// y = act((x - mean) * rstd * gamma + beta), written as one concatenated NHWC bf16 tensor.
// grid (nblk, B), block 256; dynamic smem = 2*C floats (per-channel scale/shift).
__global__ void __launch_bounds__(256) gn_apply_kernel(const __nv_bfloat16* __restrict__ x1, int C1,
                                                       const __nv_bfloat16* __restrict__ x2, int C2, int HW,
                                                       int groups, const float* __restrict__ stats,
                                                       const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, int act,
                                                       __nv_bfloat16* __restrict__ y) {
  extern __shared__ float sm[];
  const int C = C1 + C2;
  const int cpg = C / groups;
  float* scale = sm;
  float* shift = sm + C;
  const int b = blockIdx.y;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const float mean = stats[(static_cast<long long>(b) * groups + g) * 2];
    const float rstd = stats[(static_cast<long long>(b) * groups + g) * 2 + 1];
    const float sc = rstd * __ldg(gamma + c);
    scale[c] = sc;
    shift[c] = __ldg(beta + c) - mean * sc;
  }
  __syncthreads();
  const int V = C / 8;
  const long long total = static_cast<long long>(HW) * V;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const __nv_bfloat16* xb1 = x1 + static_cast<long long>(b) * HW * C1;
  const __nv_bfloat16* xb2 = x2 ? x2 + static_cast<long long>(b) * HW * C2 : nullptr;
  __nv_bfloat16* yb = y + static_cast<long long>(b) * HW * C;
  for (long long i0 = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i0 < total; i0 += 4 * stride) {
    uint4 u[4];
    int c0[4];
    long long pp[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {   // issue up to 4 independent 16-byte loads before touching any of them
      const long long i = i0 + k * stride;
      if (i < total) {
        const int v = static_cast<int>(i % V);
        pp[k] = i / V;
        c0[k] = v * 8;
        u[k] = (c0[k] < C1) ? __ldg(reinterpret_cast<const uint4*>(xb1 + pp[k] * C1 + c0[k]))
                            : __ldg(reinterpret_cast<const uint4*>(xb2 + pp[k] * C2 + (c0[k] - C1)));
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (i0 + k * stride < total) {
        const uint32_t w[4] = {u[k].x, u[k].y, u[k].z, u[k].w};
        uint32_t o[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 f = unpack_bf16x2(w[q]);
          float a = f.x * scale[c0[k] + 2 * q] + shift[c0[k] + 2 * q];
          float bb = f.y * scale[c0[k] + 2 * q + 1] + shift[c0[k] + 2 * q + 1];
          if (act == 1) { a = silu_bf16_f(a); bb = silu_bf16_f(bb); }
          o[q] = pack_bf16x2(a, bb);
        }
        *reinterpret_cast<uint4*>(yb + pp[k] * C + c0[k]) = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Single-launch GroupNorm: statistics + apply in ONE kernel.  grid (nsplit, B) with nsplit*B <= the number of CTAs that
// are resident at once (occupancy query on the host), so that every CTA of the grid is resident; each CTA reduces its
// pixel range (deterministic, as gn_stats_kernel), publishes its partial, waits on a per-image arrival counter for
// the other CTAs of the image, folds the partials (fixed order: every CTA computes bit-identical mean / rstd) and
// normalises ITS OWN pixel range.  Saves a launch and the statistics kernel's tail per GroupNorm (61 per UNet call).
//   NV == 0: generic.  The pixel range is read twice (the second time L2-hot), 8 independent 16-byte loads in flight
//            per thread in both passes.
//   NV  > 0: a thread owns at most NV pixels (host: ceil(HW / nsplit) <= NV * lanes).  They are loaded ONCE, up front,
//            and stay in registers across the grid-wide wait: the small-resolution layers (8x8 .. 32x32, 45 of the 61
//            GroupNorms of a UNet call) were pure latency chains -- ~21 us each for 1-5 MB tensors, with the loads of
//            both passes serialised in batches of four.
// gamma / beta are requested before the wait (they do not depend on the statistics), so the only global round trips
// after it are the partial rows.
// ---------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(kGnThreads, 2) gn_fused_kernel(const __nv_bfloat16* __restrict__ x1, int C1,
                                                                 const __nv_bfloat16* __restrict__ x2, int C2, int HW,
                                                                 int groups, float eps, int act,
                                                                 const float* __restrict__ gamma,
                                                                 const float* __restrict__ beta, float* __restrict__ scratch,
                                                                 __nv_bfloat16* __restrict__ y) {
  constexpr int UNR = 8;   // generic path: independent loads in flight per thread
  constexpr int kMaxCPT = 6;   // channels per thread for the scale / shift table: C <= 3072
  const int C = C1 + C2;
  const int V = C / 8;
  const int cpg = C / groups;
  const int b = blockIdx.y, split = blockIdx.x, nsplit = gridDim.x, B = gridDim.y;
  int* arrive = reinterpret_cast<int*>(scratch);
  int* depart = arrive + kGnMaxBatch;
  float* partial = scratch + 2 * kGnMaxBatch + static_cast<size_t>(B) * 2 * groups;
  const int pix_per = (HW + nsplit - 1) / nsplit;
  const int p_begin = split * pix_per;
  const int p_end = min(HW, p_begin + pix_per);
  __shared__ float part[kGnThreads * 16];   // phase 1: reduction scratch; phase 2: per-channel scale | shift
  __shared__ float gmean[32], grstd[32];
  const int lanes = kGnThreads / V;
  const int v = threadIdx.x % V;
  const int pl = threadIdx.x / V;
  const bool active = pl < lanes;
  const bool first = v * 8 < C1;
  const __nv_bfloat16* src = first ? x1 + static_cast<long long>(b) * HW * C1 + v * 8
                                   : x2 + static_cast<long long>(b) * HW * C2 + (v * 8 - C1);
  const long long Cs = first ? C1 : C2;
  auto accumulate = [](const uint4& u, float (&s)[8], float (&q)[8]) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = unpack_bf16x2(w[i]);
      s[2 * i] += f.x; q[2 * i] += f.x * f.x;
      s[2 * i + 1] += f.y; q[2 * i + 1] += f.y * f.y;
    }
  };
  // ---- phase 1: partial sums of this CTA's pixels ----
  uint4 keep[NV > 0 ? NV : 1];
  if (active) {
    float s[8], q[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; }
    if constexpr (NV > 0) {
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        const int p = p_begin + pl + k * lanes;
        keep[k] = (p < p_end) ? __ldg(reinterpret_cast<const uint4*>(src + p * Cs)) : make_uint4(0u, 0u, 0u, 0u);
      }
#pragma unroll
      for (int k = 0; k < NV; ++k) accumulate(keep[k], s, q);   // (pixels past the range contribute zeros)
    } else {
      for (int p = p_begin + pl; p < p_end; p += UNR * lanes) {
        uint4 u[UNR];
#pragma unroll
        for (int k = 0; k < UNR; ++k)
          u[k] = (p + k * lanes < p_end) ? __ldg(reinterpret_cast<const uint4*>(src + (p + k * lanes) * Cs)) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int k = 0; k < UNR; ++k) accumulate(u[k], s, q);
      }
    }
    float* dst = part + (static_cast<size_t>(pl) * V + v) * 16;
#pragma unroll
    for (int i = 0; i < 8; ++i) { dst[i] = s[i]; dst[8 + i] = q[i]; }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kGnThreads) {
    float s = 0.f, q = 0.f;
    for (int l = 0; l < lanes; ++l) {
      const float* ps = part + (static_cast<size_t>(l) * V + c / 8) * 16 + (c & 7);
      s += ps[0]; q += ps[8];
    }
    float* own = part + (static_cast<size_t>(c / 8)) * 16 + (c & 7);
    own[0] = s; own[8] = q;
  }
  __syncthreads();
  if (threadIdx.x < groups) {
    float s = 0.f, q = 0.f;
    for (int c = threadIdx.x * cpg; c < (threadIdx.x + 1) * cpg; ++c) {
      const float* ps = part + (static_cast<size_t>(c / 8)) * 16 + (c & 7);
      s += ps[0]; q += ps[8];
    }
    float* o = partial + (static_cast<long long>(b) * nsplit + split) * 2 * groups + 2 * threadIdx.x;
    o[0] = s; o[1] = q;
  }
  // gamma / beta of the channels this thread will turn into scale / shift: in flight across the wait below
  float gam[kMaxCPT], bet[kMaxCPT];
#pragma unroll
  for (int k = 0; k < kMaxCPT; ++k) {
    const int c = threadIdx.x + k * kGnThreads;
    gam[k] = (c < C) ? __ldg(gamma + c) : 0.f;
    bet[k] = (c < C) ? __ldg(beta + c) : 0.f;
  }
  // ---- publish, then wait for the other CTAs of this image (all CTAs of the grid are resident by construction) ----
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicAdd(&arrive[b], 1);
    int seen;
    do {
      asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(seen) : "l"(arrive + b) : "memory");
      if (seen < nsplit) __nanosleep(32);
    } while (seen < nsplit);
    __threadfence();
  }
  __syncthreads();
  // fold the image's nsplit partial rows (64 floats each: sum | sumsq per group) with the whole CTA: 8 row-lanes x 64
  // columns of coalesced L2 loads, then a fixed-order sum over the lanes -- every CTA of the image computes
  // bit-identical statistics.  (One thread per group walking all rows was ~4 us of serialised L2 latency.)
  {
    float* red = part + 6144;                       // [8][64]; scale | shift below use part[0, 2C), C <= 3072
    const int j = threadIdx.x & 63, sl = threadIdx.x >> 6;
    const float* pp = partial + static_cast<long long>(b) * nsplit * 64 + j;
    float acc = 0.f;
    for (int i = sl; i < nsplit; i += kGnThreads / 64) acc += __ldcg(pp + static_cast<long long>(i) * 64);
    red[sl * 64 + j] = acc;
  }
  __syncthreads();
  if (threadIdx.x < groups) {
    const float* red = part + 6144;
    float s = 0.f, q = 0.f;
#pragma unroll
    for (int l = 0; l < kGnThreads / 64; ++l) { s += red[l * 64 + 2 * threadIdx.x]; q += red[l * 64 + 2 * threadIdx.x + 1]; }
    const float inv_n = 1.0f / (static_cast<float>(HW) * cpg);
    const float mean = s * inv_n;
    const float var = fmaxf(q * inv_n - mean * mean, 0.f);
    gmean[threadIdx.x] = mean;
    grstd[threadIdx.x] = rsqrtf(var + eps);
  }
  __syncthreads();
  if (threadIdx.x == 0) {   // last CTA of the image to have read the partials re-arms both counters for the next launch
    if (atomicAdd(&depart[b], 1) == nsplit - 1) { arrive[b] = 0; depart[b] = 0; }
  }
  float* scale = part;
  float* shift = part + C;
#pragma unroll
  for (int k = 0; k < kMaxCPT; ++k) {
    const int c = threadIdx.x + k * kGnThreads;
    if (c < C) {
      const int g = c / cpg;
      const float sc = grstd[g] * gam[k];
      scale[c] = sc;
      shift[c] = bet[k] - gmean[g] * sc;
    }
  }
  __syncthreads();
  // ---- phase 2: normalise this CTA's pixels ----
  if (active) {
    __nv_bfloat16* dstb = y + static_cast<long long>(b) * HW * C + v * 8;
    const int c0 = v * 8;
    auto apply_store = [&](const uint4& u, int p) {
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
      uint32_t o[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack_bf16x2(w[i]);
        float a = f.x * scale[c0 + 2 * i] + shift[c0 + 2 * i];
        float bb = f.y * scale[c0 + 2 * i + 1] + shift[c0 + 2 * i + 1];
        if (act == 1) { a = silu_bf16_f(a); bb = silu_bf16_f(bb); }
        o[i] = pack_bf16x2(a, bb);
      }
      *reinterpret_cast<uint4*>(dstb + static_cast<long long>(p) * C) = make_uint4(o[0], o[1], o[2], o[3]);
    };
    if constexpr (NV > 0) {
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        const int p = p_begin + pl + k * lanes;
        if (p < p_end) apply_store(keep[k], p);
      }
    } else {
      for (int p = p_begin + pl; p < p_end; p += UNR * lanes) {
        uint4 u[UNR];
#pragma unroll
        for (int k = 0; k < UNR; ++k)
          if (p + k * lanes < p_end) u[k] = __ldg(reinterpret_cast<const uint4*>(src + (p + k * lanes) * Cs));
#pragma unroll
        for (int k = 0; k < UNR; ++k)
          if (p + k * lanes < p_end) apply_store(u[k], p + k * lanes);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// (Round 1 left a thread-block-cluster GroupNorm here — the CTAs of one image as a 16-CTA cluster, pixel ranges kept in 160 KB
// of shared memory.  First GPU run, round 2: 45 us against 26 us for the single-launch kernel above on the 64x64 C = 320 layer,
// slower on every UNet shape.  Removed; the group-bundle kernel below replaces it.)
// ---------------------------------------------------------------------------------------------
VDB_DEVINL float ld_dsmem_f32(uint32_t cluster_addr) {
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(cluster_addr) : "memory");
  return v;
}
VDB_DEVINL void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
VDB_DEVINL void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// Group-bundle GroupNorm (round 2, default wherever it fits): a CTA owns a BUNDLE of G consecutive groups of ONE image
// (G = 1, 2 or 4, the smallest that makes the bundle's channel run a multiple of 16 bytes: 40 / 40 / 120 / 40 / 120 / 80
// channels at C = 320 / 640 / 960 / 1280 / 1920 / 2560) instead of a pixel range of all channels.  A group's statistics
// then never leave the CTA: no grid-wide arrival counter, no global scratch, no residency requirement, and the pixels are
// read ONCE (they stay in registers between the statistics and the normalisation).  Layers whose bundle does not fit the
// registers of one CTA split the pixels over a thread-block cluster of S <= 8 CTAs (grid (bundles, S, B), cluster
// (1, S, 1)); the 2 G partial sums are pushed into every peer's shared memory (st.shared::cluster + a remote mbarrier arrival).
// The single-launch kernel above spent most of its 11-30 us per layer in serialised latency phases (publish, device-wide
// wait, re-read), not in bandwidth.
// Deterministic: fixed-order shuffles / rank-ordered cluster fold (every CTA of a cluster computes identical statistics).
// Per-thread mapping: vec = t % VPB (16-byte channel octet inside the bundle), pixel lane = t / VPB; pixels pl + k * lanes.
// ---------------------------------------------------------------------------------------------
template <int NVMAX, int THREADS>
__global__ void __launch_bounds__(THREADS, (THREADS == 512 && NVMAX <= 6) ? 2 : 1) gn_bundle_kernel(const __nv_bfloat16* __restrict__ x1, int C1,
                                                                           const __nv_bfloat16* __restrict__ x2, int C2, int HW,
                                                                           int groups, int G, float eps, int act,
                                                                           const float* __restrict__ gamma,
                                                                           const float* __restrict__ beta,
                                                                           __nv_bfloat16* __restrict__ y) {
  const int C = C1 + C2;
  const int cpg = C / groups;
  const int BC = G * cpg;                 // channels per bundle (multiple of 8)
  const int VPB = BC / 8;                 // 16-byte vectors per pixel and bundle
  const int lanes = THREADS / VPB;
  const int S = gridDim.y;
  const int b = blockIdx.z, bundle = blockIdx.x, part = blockIdx.y;
  __shared__ float wpart[THREADS / 32][8];          // per-warp partials: sum | sumsq of up to 4 groups
  __shared__ float xpart[8];              // this CTA's partials
  __shared__ float xall[8][8];            // S > 1: every rank's partials, WRITTEN BY THE PEERS (st.shared::cluster)
  __shared__ uint64_t xbar;               // S > 1: counts the 8 S remote-write arrivals
  __shared__ float gstat[8];              // mean[4] | rstd[4]
  if (S > 1) {
    // one-way exchange instead of two cluster barriers (ncu: barrier.cluster.arrive.release + wait were ~30 % of this kernel's
    // stall samples on the 64x64 layers): every CTA pushes its 8 partial sums into each peer's xall[rank] and arrives on the
    // peer's mbarrier; a CTA leaves only after all 8 S arrivals, i.e. after every write into its memory has landed, and its own
    // pushes target CTAs that cannot leave before receiving them.  The only cluster barrier left is split-phase: arrive here,
    // right after the mbarrier is initialised, wait just before the first push (long complete by then).
    if (threadIdx.x == 0) {
      mbar_init(&xbar, 8 * S);
      fence_barrier_init();
    }
    __syncthreads();
    asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
  }
  const int vec = threadIdx.x % VPB, pl = threadIdx.x / VPB;
  const bool active = pl < lanes;
  const int cb = vec * 8;                                 // first channel of this thread inside the bundle
  const int cg = bundle * BC + cb;                        // ... and inside the (concatenated) tensor
  const bool first = cg < C1;
  const __nv_bfloat16* src = first ? x1 + static_cast<long long>(b) * HW * C1 + cg
                                   : x2 + static_cast<long long>(b) * HW * C2 + (cg - C1);
  const long long Cs = first ? C1 : C2;
  const int pix_per = (HW + S - 1) / S;
  const int p_begin = part * pix_per, p_end = min(HW, p_begin + pix_per);
  // THREADS == 1024 (one CTA per SM, 64 registers per thread): the pixels wait in shared memory (cp.async, 16 bytes per
  // request, slot [k][thread]: every thread reads back only what it requested itself) instead of in registers
  constexpr bool kSmem = THREADS > 512;
  extern __shared__ uint4 gn_keep_smem[];
  uint4 keep[kSmem ? 1 : NVMAX];
  float s[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; }
  if (active) {
#pragma unroll
    for (int k = 0; k < NVMAX; ++k) {
      const int p = p_begin + pl + k * lanes;
      if constexpr (kSmem) {
        uint4* slot = gn_keep_smem + k * THREADS + threadIdx.x;
        if (p < p_end) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(slot)), "l"(src + p * Cs) : "memory");
        else *slot = make_uint4(0u, 0u, 0u, 0u);
      } else {
        keep[k] = (p < p_end) ? __ldg(reinterpret_cast<const uint4*>(src + p * Cs)) : make_uint4(0u, 0u, 0u, 0u);
      }
    }
    if constexpr (kSmem) asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
  }
  auto kept = [&](int k) -> uint4 {
    if constexpr (kSmem) return gn_keep_smem[k * THREADS + threadIdx.x]; else return keep[k];
  };
  if (active) {
#pragma unroll
    for (int k = 0; k < NVMAX; ++k) {     // (pixels past the range contribute zeros)
      const uint4 kv = kept(k);
      const uint32_t w[4] = {kv.x, kv.y, kv.z, kv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack_bf16x2(w[i]);
        s[2 * i] += f.x; q[2 * i] += f.x * f.x;
        s[2 * i + 1] += f.y; q[2 * i + 1] += f.y * f.y;
      }
    }
  }
  // this thread's 8 channels belong to at most two groups of the bundle (cpg >= 4): g_lo for channels < nb, g_lo + 1 after
  const int g_lo = cb / cpg;
  const int nb = min(8, (g_lo + 1) * cpg - cb);
  float red[8];                            // sum[4] | sumsq[4]
  {
    float a0 = 0.f, c0 = 0.f, a1 = 0.f, c1 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i < nb) { a0 += s[i]; c0 += q[i]; } else { a1 += s[i]; c1 += q[i]; }
    }
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      red[g] = (g == g_lo) ? a0 : ((g == g_lo + 1) ? a1 : 0.f);
      red[4 + g] = (g == g_lo) ? c0 : ((g == g_lo + 1) ? c1 : 0.f);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) red[j] += __shfl_xor_sync(0xffffffffu, red[j], o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < 8; ++j) wpart[warp][j] = red[j];
  }
  __syncthreads();
  if (threadIdx.x < 8) {
    float a = 0.f;
#pragma unroll
    for (int w = 0; w < THREADS / 32; ++w) a += wpart[w][threadIdx.x];
    xpart[threadIdx.x] = a;
  }
  // gamma / beta of this thread's channel octet: in flight under the barriers below
  float gam[8], bet[8];
  if (active) {
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + cg)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + cg + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + cg)), b1 = __ldg(reinterpret_cast<const float4*>(beta + cg + 4));
    gam[0] = g0.x; gam[1] = g0.y; gam[2] = g0.z; gam[3] = g0.w; gam[4] = g1.x; gam[5] = g1.y; gam[6] = g1.z; gam[7] = g1.w;
    bet[0] = b0.x; bet[1] = b0.y; bet[2] = b0.z; bet[3] = b0.w; bet[4] = b1.x; bet[5] = b1.y; bet[6] = b1.z; bet[7] = b1.w;
  }
  if (S > 1) {
    __syncthreads();                       // xpart complete
    asm volatile("barrier.cluster.wait.aligned;" ::: "memory");   // every peer's mbarrier is initialised
    if (threadIdx.x < 8) {
      const float v = xpart[threadIdx.x];
      const uint32_t slot = smem_u32(&xall[part][threadIdx.x]), bar = smem_u32(&xbar);
      for (int r = 0; r < S; ++r) {
        asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(mapa_u32(slot, static_cast<uint32_t>(r))), "f"(v) : "memory");
        mbar_arrive_cluster(mapa_u32(bar, static_cast<uint32_t>(r)));     // release.cluster: orders this thread's store before it
      }
    }
    if (threadIdx.x < 4) {                 // (the threads that fold the partials wait; the rest meet them at the barrier below)
      uint32_t ok = 0;
      while (!ok) {
        asm volatile(
            "{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P, [%1], %2;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
            : "=r"(ok) : "r"(smem_u32(&xbar)), "r"(0u) : "memory");
      }
    }
  } else {
    __syncthreads();
  }
  if (threadIdx.x < 4) {
    float a = 0.f, c = 0.f;
    if (S > 1) {
      for (int r = 0; r < S; ++r) {        // rank order: identical in every CTA of the cluster
        a += xall[r][threadIdx.x];
        c += xall[r][4 + threadIdx.x];
      }
    } else {
      a = xpart[threadIdx.x]; c = xpart[4 + threadIdx.x];
    }
    const float inv_n = 1.0f / (static_cast<float>(HW) * cpg);
    const float mean = a * inv_n;
    const float var = fmaxf(c * inv_n - mean * mean, 0.f);
    gstat[threadIdx.x] = mean;
    gstat[4 + threadIdx.x] = rsqrtf(var + eps);
  }
  __syncthreads();
  if (active) {
    float sc[8], sh[8];
    const float m0 = gstat[g_lo], r0 = gstat[4 + g_lo], m1 = gstat[min(g_lo + 1, 3)], r1 = gstat[4 + min(g_lo + 1, 3)];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      sc[i] = ((i < nb) ? r0 : r1) * gam[i];
      sh[i] = bet[i] - ((i < nb) ? m0 : m1) * sc[i];
    }
    __nv_bfloat16* dst = y + static_cast<long long>(b) * HW * C + cg;
#pragma unroll
    for (int k = 0; k < NVMAX; ++k) {
      const int p = p_begin + pl + k * lanes;
      if (p < p_end) {
        const uint4 kv = kept(k);
        const uint32_t w[4] = {kv.x, kv.y, kv.z, kv.w};
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = unpack_bf16x2(w[i]);
          float a = f.x * sc[2 * i] + sh[2 * i];
          float c = f.y * sc[2 * i + 1] + sh[2 * i + 1];
          if (act == 1) { a = silu_bf16_f(a); c = silu_bf16_f(c); }
          o[i] = pack_bf16x2(a, c);
        }
        *reinterpret_cast<uint4*>(dst + static_cast<long long>(p) * C) = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// LayerNorm over the last dim of [rows, C] bf16 (one warp per row, two-pass in registers).
// ---------------------------------------------------------------------------------------------
template <int MAXV, int R>  // MAXV: max 16-byte vectors per lane; R: rows processed concurrently per warp (memory-level parallelism)
__global__ void __launch_bounds__(256) layernorm_kernel(const __nv_bfloat16* __restrict__ x, long long rows, int C,
                                                        const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float eps,
                                                        __nv_bfloat16* __restrict__ y) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int V = C / 8;
  for (long long r0 = static_cast<long long>(warp) * R; r0 < rows; r0 += static_cast<long long>(nwarps) * R) {
    uint4 raw[R][MAXV];
#pragma unroll
    for (int j = 0; j < R; ++j)
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        const int v = lane + i * 32;
        if (v < V && r0 + j < rows) raw[j][i] = __ldg(reinterpret_cast<const uint4*>(x + (r0 + j) * C + v * 8));
      }
#pragma unroll
    for (int j = 0; j < R; ++j) {
      if (r0 + j >= rows) break;   // warp-uniform
      float f[MAXV][8];
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        if (lane + i * 32 < V) {
          const uint32_t w[4] = {raw[j][i].x, raw[j][i].y, raw[j][i].z, raw[j][i].w};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float2 t = unpack_bf16x2(w[k]);
            f[i][2 * k] = t.x; f[i][2 * k + 1] = t.y;
            s += t.x + t.y;
          }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float mean = s / C;
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        if (lane + i * 32 < V) {
#pragma unroll
          for (int k = 0; k < 8; ++k) { const float d = f[i][k] - mean; q += d * d; }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      const float rstd = rsqrtf(q / C + eps);
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        const int v = lane + i * 32;
        if (v < V) {
          const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8 + 4));
          const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + v * 8)), b1 = __ldg(reinterpret_cast<const float4*>(beta + v * 8 + 4));
          const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
          const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
          uint32_t o[4];
#pragma unroll
          for (int k = 0; k < 4; ++k)
            o[k] = pack_bf16x2((f[i][2 * k] - mean) * rstd * gg[2 * k] + bb[2 * k],
                               (f[i][2 * k + 1] - mean) * rstd * gg[2 * k + 1] + bb[2 * k + 1]);
          *reinterpret_cast<uint4*>(y + (r0 + j) * C + v * 8) = make_uint4(o[0], o[1], o[2], o[3]);
        }
      }
    }
  }
}

// (A persistent prefetching variant of this kernel was measured slower than the row-group kernel below, which is the default.)
// Row-group LayerNorm (round 2, default when C = 8 * VPL * LPR fits): LPR lanes share a row, each lane owns VPL 16-byte
// vectors (vector l + k * LPR: consecutive lanes read consecutive 16-byte pieces), so a warp covers 32 / LPR rows per
// step with EVERY lane busy — the warp-per-row kernel above leaves 24 of 32 lanes idle on the second vector of a
// C = 320 row (40 vectors) and was measured at 2.3 TB/s in-graph on the 32768 x 320 layers.  Persistent walk with the
// next step's rows requested before the current ones are normalised; gamma / beta live in shared memory.
template <int VPL, int LPR>
__global__ void __launch_bounds__(256, 2) layernorm_rg_kernel(const __nv_bfloat16* __restrict__ x, long long rows, int C,
                                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                                           float eps, __nv_bfloat16* __restrict__ y) {
  constexpr int RPW = 32 / LPR;           // rows per warp and step
  extern __shared__ float ln_gb[];        // gamma[C] | beta[C]
  for (int i = threadIdx.x; i < C; i += blockDim.x) { ln_gb[i] = __ldg(gamma + i); ln_gb[C + i] = __ldg(beta + i); }
  __syncthreads();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int sub = lane / LPR;             // which of the warp's rows
  const int l = lane % LPR;               // position inside the row group
  const long long stride = static_cast<long long>(nwarps) * RPW;
  const float inv_c = 1.0f / static_cast<float>(C);
  auto load_row = [&](long long r, uint4 (&raw)[VPL]) {
    if (r < rows) {
      const uint4* src = reinterpret_cast<const uint4*>(x + r * C) + l;
#pragma unroll
      for (int k = 0; k < VPL; ++k) raw[k] = __ldg(src + k * LPR);
    }
  };
  uint4 cur[VPL], nxt[VPL];
  long long r = static_cast<long long>(warp) * RPW + sub;
  load_row(r, cur);
  for (long long r0 = static_cast<long long>(warp) * RPW; r0 < rows; r0 += stride, r += stride) {
    load_row(r + stride, nxt);            // in flight while the current rows are normalised
    // (the rows are unpacked again in every pass instead of kept as fp32: 40 fewer live registers at VPL = 5)
    float s = 0.f;
    if (r < rows) {
#pragma unroll
      for (int k = 0; k < VPL; ++k) {
        const uint32_t w[4] = {cur[k].x, cur[k].y, cur[k].z, cur[k].w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 t = unpack_bf16x2(w[i]);
          s += t.x + t.y;
        }
      }
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s * inv_c;
    float q = 0.f;
    if (r < rows) {
#pragma unroll
      for (int k = 0; k < VPL; ++k) {
        const uint32_t w[4] = {cur[k].x, cur[k].y, cur[k].z, cur[k].w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 t = unpack_bf16x2(w[i]);
          const float d0 = t.x - mean, d1 = t.y - mean;
          q += d0 * d0 + d1 * d1;
        }
      }
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q * inv_c + eps);
    if (r < rows) {
      uint4* dst = reinterpret_cast<uint4*>(y + r * C) + l;
#pragma unroll
      for (int k = 0; k < VPL; ++k) {
        const int c0 = (l + k * LPR) * 8;
        const float4 g0 = *reinterpret_cast<const float4*>(ln_gb + c0), g1 = *reinterpret_cast<const float4*>(ln_gb + c0 + 4);
        const float4 b0 = *reinterpret_cast<const float4*>(ln_gb + C + c0), b1 = *reinterpret_cast<const float4*>(ln_gb + C + c0 + 4);
        const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        const uint32_t w[4] = {cur[k].x, cur[k].y, cur[k].z, cur[k].w};
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 t = unpack_bf16x2(w[i]);
          o[i] = pack_bf16x2((t.x - mean) * rstd * gg[2 * i] + bb[2 * i], (t.y - mean) * rstd * gg[2 * i + 1] + bb[2 * i + 1]);
        }
        dst[k * LPR] = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
#pragma unroll
    for (int k = 0; k < VPL; ++k) cur[k] = nxt[k];
  }
}

// ---------------------------------------------------------------------------------------------
// CLIP image preprocessing on the device (SURVEY §8f rank 3; opt-in, not yet run on a GPU): the reference converts the
// tensor to PIL on the HOST and lets CLIPProcessor resize it there (clip.py:88-94).  These three kernels reproduce that
// arithmetic exactly — torchvision's ToPILImage (x * 255 truncated to uint8) and Pillow's 8-bit two-pass bicubic resampling
// (int32 fixed-point coefficients with 22 fractional bits, horizontal pass rounded to uint8 before the vertical one), then
// centre crop, / 255 and normalisation — so the image never leaves the GPU.  The coefficient tables are built on the
// host exactly as Pillow's precompute_coeffs / normalize_coeffs_8bpc do (lib/model_zoo/clip.py: pil_bicubic_coeffs).
// ---------------------------------------------------------------------------------------------
__global__ void clip_to_u8_hwc_kernel(const float* __restrict__ x, int n, int H, int W, uint8_t* __restrict__ y) {
  const long long total = static_cast<long long>(n) * H * W * 3;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % 3);
    long long p = i / 3;
    const int w = static_cast<int>(p % W); p /= W;
    const int h = static_cast<int>(p % H);
    const long long b = p / H;
    const float v = fminf(fmaxf(__ldg(x + ((b * 3 + c) * H + h) * W + w), 0.f), 1.f);
    y[i] = static_cast<uint8_t>(__fmul_rn(v, 255.f));      // .byte(): truncation toward zero
  }
}

VDB_DEVINL uint8_t pil_clip8(int acc) {
  const int v = acc >> 22;
  return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// horizontal pass: x [n, H, Win, 3] u8 -> y [n, H, Wout, 3] u8
__global__ void resample_h_u8_kernel(const uint8_t* __restrict__ x, int n, int H, int Win, int Wout,
                                     const int* __restrict__ bounds, const int* __restrict__ kk, int ksize,
                                     uint8_t* __restrict__ y) {
  const long long total = static_cast<long long>(n) * H * Wout * 3;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % 3);
    long long p = i / 3;
    const int xx = static_cast<int>(p % Wout);
    const long long row = p / Wout;                       // b * H + h
    const int xmin = __ldg(bounds + 2 * xx), cnt = __ldg(bounds + 2 * xx + 1);
    const uint8_t* src = x + (row * Win + xmin) * 3 + c;
    const int* k = kk + static_cast<long long>(xx) * ksize;
    int acc = 1 << 21;
    for (int t = 0; t < cnt; ++t) acc += static_cast<int>(src[t * 3]) * __ldg(k + t);
    y[i] = pil_clip8(acc);
  }
}

// vertical pass (ksize == 0: no vertical resize) + centre crop + /255 + normalise: x [n, Hin, W, 3] u8 -> y [n, 3, S, S] fp32
__global__ void resample_v_crop_norm_kernel(const uint8_t* __restrict__ x, int n, int Hin, int W,
                                            const int* __restrict__ bounds, const int* __restrict__ kk, int ksize, int top,
                                            int left, int S, float m0, float m1, float m2, float s0, float s1, float s2,
                                            float* __restrict__ y) {
  const long long total = static_cast<long long>(n) * 3 * S * S;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ox = static_cast<int>(i % S);
    long long p = i / S;
    const int oy = static_cast<int>(p % S); p /= S;
    const int c = static_cast<int>(p % 3);
    const long long b = p / 3;
    const int yy = oy + top, xs = ox + left;
    uint8_t u;
    if (ksize == 0) {
      u = x[((b * Hin + yy) * W + xs) * 3 + c];
    } else {
      const int ymin = __ldg(bounds + 2 * yy), cnt = __ldg(bounds + 2 * yy + 1);
      const int* k = kk + static_cast<long long>(yy) * ksize;
      int acc = 1 << 21;
      for (int t = 0; t < cnt; ++t) acc += static_cast<int>(x[((b * Hin + ymin + t) * W + xs) * 3 + c]) * __ldg(k + t);
      u = pil_clip8(acc);
    }
    const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
    y[i] = __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(u), 255.f), mean), sd);
  }
}

// nearest-neighbour 2x upsample of NHWC bf16           (openaimodel.py:114, autokl_modules.py:54)
__global__ void upsample2x_kernel(const __nv_bfloat16* __restrict__ x, int B, int H, int W, int C,
                                  __nv_bfloat16* __restrict__ y) {
  const int V = C / 8;
  const long long total = static_cast<long long>(B) * 2 * H * 2 * W * V;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % V);
    long long p = i / V;
    const int xo = static_cast<int>(p % (2 * W)); p /= 2 * W;
    const int yo = static_cast<int>(p % (2 * H));
    const int b = static_cast<int>(p / (2 * H));
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(
        x + ((static_cast<long long>(b) * H + (yo >> 1)) * W + (xo >> 1)) * C + v * 8));
    *reinterpret_cast<uint4*>(y + ((static_cast<long long>(b) * 2 * H + yo) * 2 * W + xo) * C + v * 8) = u;
  }
}

// im2col for 3x3/pad-1/stride-1 convs with tiny Cin (latent 4ch, RGB 3ch): fp32 NHWC in,
// bf16 [B*H*W, Kpad] out with column (ky*3+kx)*Cin + c, zero padded to Kpad.
// One thread per (pixel, 16-byte chunk of the row): 32-bit index math, one 16-byte store (one bf16 per thread behind five 64-bit
// divisions was far slower).
__global__ void im2col3x3_small_kernel(const float* __restrict__ x, int B, int H, int W, int Cin, int Kpad,
                                       float in_scale, float in_shift, __nv_bfloat16* __restrict__ y) {
  const int chunks = Kpad >> 3;
  const long long total = static_cast<long long>(B) * H * W * chunks;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int q = static_cast<int>(i % chunks);
    const long long p = i / chunks;
    const int xo = static_cast<int>(p % W);
    const int yo = static_cast<int>((p / W) % H);
    const int b = static_cast<int>(p / (static_cast<long long>(W) * H));
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = q * 8 + e;
      float val = 0.f;
      if (k < 9 * Cin) {
        const int t = k / Cin, c = k - t * Cin;
        const int ty = t / 3, tx = t - ty * 3;
        const int xi = xo + tx - 1, yi = yo + ty - 1;
        if (xi >= 0 && xi < W && yi >= 0 && yi < H)
          val = __ldg(x + ((static_cast<long long>(b) * H + yi) * W + xi) * Cin + c) * in_scale + in_shift;
      }
      v[e] = val;
    }
    *reinterpret_cast<uint4*>(y + p * Kpad + q * 8) =
        make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
  }
}

// fp32 NCHW <-> NHWC permutes for the latent / image boundaries; optional affine + clamp on the way out
__global__ void permute_f32_kernel(const float* __restrict__ x, int B, int C, int HW, int to_nhwc, float mul,
                                   float add, int clamp01, float* __restrict__ y) {
  const long long total = static_cast<long long>(B) * C * HW;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    long long src;
    if (to_nhwc) {  // i indexes NHWC output
      const int c = static_cast<int>(i % C);
      const long long p = (i / C) % HW;
      const long long b = i / (static_cast<long long>(C) * HW);
      src = (b * C + c) * HW + p;
    } else {        // i indexes NCHW output
      const long long p = i % HW;
      const int c = static_cast<int>((i / HW) % C);
      const long long b = i / (static_cast<long long>(C) * HW);
      src = (b * HW + p) * C + c;
    }
    float v = x[src] * mul + add;
    if (clamp01) v = fminf(fmaxf(v, 0.f), 1.f);
    y[i] = v;
  }
}

// y[p, o] = (sum_c W[o, c] * x[p, c] + b[o]) * mul for tiny channel counts (post_quant_conv 4->4,
// quant_conv 8->8: autokl.py:26-27,36,45), fp32 NHWC in/out.
__global__ void pointwise_small_kernel(const float* __restrict__ x, long long npix, int Cin, int Cout,
                                       const float* __restrict__ Wm, const float* __restrict__ bias, float pre_mul,
                                       float* __restrict__ y) {
  for (long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; p < npix;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    float xin[8];
    for (int c = 0; c < Cin; ++c) xin[c] = x[p * Cin + c] * pre_mul;
    for (int o = 0; o < Cout; ++o) {
      float acc = bias ? bias[o] : 0.f;
      for (int c = 0; c < Cin; ++c) acc += Wm[o * Cin + c] * xin[c];
      y[p * Cout + o] = acc;
    }
  }
}

// DiagonalGaussianDistribution.sample (distributions.py:24-37) on NHWC fp32 moments [npix, 2*C]:
// z = (mean + exp(0.5 * clamp(logvar, -30, 20)) * noise) * post_mul ; noise NHWC [npix, C] or null (mode)
__global__ void gaussian_sample_kernel(const float* __restrict__ moments, const float* __restrict__ noise, int C,
                                       long long npix, float post_mul, float* __restrict__ z) {
  const long long total = npix * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / C;
    const int c = static_cast<int>(i % C);
    const float mean = moments[p * 2 * C + c];
    float lv = moments[p * 2 * C + C + c];
    lv = fminf(fmaxf(lv, -30.f), 20.f);
    float v = mean;
    if (noise) v = __fadd_rn(mean, __fmul_rn(expf(0.5f * lv), noise[i]));
    z[i] = v * post_mul;
  }
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    y[i] = __float2bfloat16(x[i]);
}
__global__ void cast_bf16_f32_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ y, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    y[i] = __bfloat162float(x[i]);
}

// ---------------------------------------------------------------------------------------------
// Sinusoidal timestep embedding [cos | sin]              (diffusion_utils.py:131-151)
// t from ts[b] (int64), or ts_table[*step_idx] broadcast to all rows when step_idx != null.
// ---------------------------------------------------------------------------------------------
__global__ void timestep_embedding_kernel(const long long* __restrict__ ts, const int* __restrict__ step_idx,
                                          int B, int dim, float neg_log_period, float* __restrict__ out) {
  const int half = dim / 2;
  const int total = B * half;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int b = i / half, k = i % half;
    const float t = static_cast<float>(step_idx ? ts[*step_idx] : ts[b]);
    // freqs = exp(-ln(max_period) * k / half) in fp32, as torch does (host passes fp32(-ln(max_period)))
    const float fr = expf(__fdiv_rn(__fmul_rn(neg_log_period, static_cast<float>(k)), static_cast<float>(half)));
    const float a = t * fr;
    out[b * dim + k] = cosf(a);
    out[b * dim + half + k] = sinf(a);
    if ((dim & 1) && k == 0) out[b * dim + dim - 1] = 0.f;
  }
}

// ---------------------------------------------------------------------------------------------
// Skinny linear for M <= 16 rows (time-embedding MLP, ResBlock.emb_layers): weight-bandwidth bound.
//   out[m, n] = act_out( sum_k act_in(x[m, k]) * W[n, k] + bias[n] )          fp32 x/out, bf16 W
// One warp per output column; x staged (activated) in shared memory.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) linear_small_kernel(const float* __restrict__ x, int M, int K,
                                                           const __nv_bfloat16* __restrict__ Wt, int N,
                                                           const float* __restrict__ bias, int act_in, int act_out,
                                                           float* __restrict__ out) {
  extern __shared__ float xs[];  // [M, K]
  {
    // stage (activated) x: float4 loads, several in flight per thread (a scalar dependent-load loop cost ~20 us here)
    const int n4 = (M * K) >> 2;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    float4* xs4 = reinterpret_cast<float4*>(xs);
#pragma unroll 4
    for (int i = threadIdx.x; i < n4; i += blockDim.x) {
      float4 v = __ldg(x4 + i);
      if (act_in == 1) { v.x = silu_f(v.x); v.y = silu_f(v.y); v.z = silu_f(v.z); v.w = silu_f(v.w); }
      xs4[i] = v;
    }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nwarps = blockDim.x >> 5;
  constexpr int NC = 4;  // output columns per warp iteration: NC independent weight streams in flight
  for (int n0 = (blockIdx.x * nwarps + warp) * NC; n0 < N; n0 += gridDim.x * nwarps * NC) {
    float acc[NC][16];
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int m = 0; m < 16; ++m) acc[c][m] = 0.f;
    for (int k = lane * 8; k < K; k += 256) {
      uint4 u[NC];
#pragma unroll
      for (int c = 0; c < NC; ++c)
        if (n0 + c < N) u[c] = __ldg(reinterpret_cast<const uint4*>(Wt + static_cast<long long>(n0 + c) * K + k));
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        if (n0 + c < N) {
          const uint32_t w[4] = {u[c].x, u[c].y, u[c].z, u[c].w};
          float wf[8];
#pragma unroll
          for (int q = 0; q < 4; ++q) { const float2 t = unpack_bf16x2(w[q]); wf[2 * q] = t.x; wf[2 * q + 1] = t.y; }
#pragma unroll
          for (int m = 0; m < 16; ++m) {
            if (m < M) {
              const float* xr = xs + m * K + k;
#pragma unroll
              for (int q = 0; q < 8; ++q) acc[c][m] += xr[q] * wf[q];
            }
          }
        }
      }
    }
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      if (n0 + c >= N) break;
#pragma unroll
      for (int m = 0; m < 16; ++m) {
        if (m < M) {
          float v = acc[c][m];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
          if (lane == 0) {
            v += bias ? bias[n0 + c] : 0.f;
            if (act_out == 1) v = silu_f(v);
            out[static_cast<long long>(m) * N + n0 + c] = v;
          }
        }
      }
    }
  }
}

// row softmax over [rows, n] bf16 with scale, fp32 math, bf16 out (VAE AttnBlock, autokl_modules.py:186-188)
__global__ void __launch_bounds__(256) softmax_rows_kernel(const __nv_bfloat16* __restrict__ x, long long rows,
                                                           int n, long long ld, float scale,
                                                           __nv_bfloat16* __restrict__ y) {
  __shared__ float red[32];
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const __nv_bfloat16* xr = x + r * ld;
    float mx = -INFINITY;
    for (int i = threadIdx.x; i < n; i += blockDim.x) mx = fmaxf(mx, __bfloat162float(xr[i]) * scale);
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = red[0];
    for (int w = 1; w < (blockDim.x >> 5); ++w) mx = fmaxf(mx, red[w]);
    __syncthreads();
    float s = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s += __expf(__bfloat162float(xr[i]) * scale - mx);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    s = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) s += red[w];
    __syncthreads();
    const float inv = 1.f / s;
    __nv_bfloat16* yr = y + r * ld;
    for (int i = threadIdx.x; i < n; i += blockDim.x)
      yr[i] = __float2bfloat16(__expf(__bfloat162float(xr[i]) * scale - mx) * inv);
  }
}

// ---------------------------------------------------------------------------------------------
// CLIP front/back ends (HF CLIPModel arithmetic around the transformer blocks; reference call sites clip.py:57-62,
// 95-101).  Token streams are stored [B, Lp, C] with Lp = L rounded up to 8 and zero pad rows.
// ---------------------------------------------------------------------------------------------
// x[b, n, :] = tok_emb[tokens[b, n], :] + pos_emb[n, :]          (CLIPTextEmbeddings)
__global__ void clip_text_embed_kernel(const long long* __restrict__ tokens, const float* __restrict__ tok_emb,
                                       const float* __restrict__ pos_emb, int B, int L, int Lp, int C,
                                       __nv_bfloat16* __restrict__ x) {
  const long long total = static_cast<long long>(B) * Lp * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    const int n = static_cast<int>((i / C) % Lp);
    const int b = static_cast<int>(i / (static_cast<long long>(C) * Lp));
    float v = 0.f;
    if (n < L) v = tok_emb[tokens[b * L + n] * C + c] + pos_emb[static_cast<long long>(n) * C + c];
    x[i] = __float2bfloat16(v);
  }
}

// non-overlapping PxP patches of NCHW fp32 pixels -> bf16 rows [B*G*G, Kpad], column (c*P + py)*P + px (the
// flattening of the patch_embedding conv weight [C_out, 3, P, P]); zero padded to Kpad
__global__ void patchify_kernel(const float* __restrict__ px, int B, int Cin, int HW, int P, int Kpad,
                                __nv_bfloat16* __restrict__ y) {
  const int G = HW / P;
  const long long total = static_cast<long long>(B) * G * G * Kpad;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % Kpad);
    const long long row = i / Kpad;
    float v = 0.f;
    if (k < Cin * P * P) {
      const int c = k / (P * P), py = (k / P) % P, pxx = k % P;
      const int gx = static_cast<int>(row % G), gy = static_cast<int>((row / G) % G);
      const int b = static_cast<int>(row / (G * G));
      v = px[((static_cast<long long>(b) * Cin + c) * HW + gy * P + py) * HW + gx * P + pxx];
    }
    y[i] = __float2bfloat16(v);
  }
}

// x[b, 0] = cls + pos[0]; x[b, 1+j] = patch[b, j] + pos[1+j]; optional per-token scale (masked variant,
// clip.py:117-133); rows >= L zero                                              (CLIPVisionEmbeddings)
__global__ void vit_assemble_kernel(const __nv_bfloat16* __restrict__ patches, const float* __restrict__ cls,
                                    const float* __restrict__ pos, const float* __restrict__ tok_scale, int B, int L,
                                    int Lp, int C, __nv_bfloat16* __restrict__ x) {
  const long long total = static_cast<long long>(B) * Lp * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    const int n = static_cast<int>((i / C) % Lp);
    const int b = static_cast<int>(i / (static_cast<long long>(C) * Lp));
    float v = 0.f;
    if (n < L) {
      v = (n == 0) ? cls[c] : __bfloat162float(patches[(static_cast<long long>(b) * (L - 1) + n - 1) * C + c]);
      v += pos[static_cast<long long>(n) * C + c];
      if (tok_scale) v *= tok_scale[b * L + n];
    }
    x[i] = __float2bfloat16(v);
  }
}

// out[b, n, :] = z[b, n, :] / || z[b, idx[b], :] ||  [* row_scale[b, n]]   (clip.py:60-61, 99-100, 142)
__global__ void __launch_bounds__(256) scale_by_row_norm_kernel(const __nv_bfloat16* __restrict__ z,
                                                                const int* __restrict__ idx,
                                                                const float* __restrict__ row_scale, int L, int Lp,
                                                                int C, float* __restrict__ out) {
  __shared__ float red[8];
  __shared__ float inv;
  const int b = blockIdx.x;
  const int r = idx ? idx[b] : 0;
  const __nv_bfloat16* zr = z + (static_cast<long long>(b) * Lp + r) * C;
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) { const float v = __bfloat162float(zr[c]); s += v * v; }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) t += red[w];
    inv = 1.0f / sqrtf(t);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < L * C; i += blockDim.x) {
    const int n = i / C, c = i % C;
    float v = __bfloat162float(z[(static_cast<long long>(b) * Lp + n) * C + c]) * inv;
    if (row_scale) v *= row_scale[b * L + n];
    out[(static_cast<long long>(b) * L + n) * C + c] = v;
  }
}

// y[r, i] = act(x[r, i] * gamma[i] + beta[i]) on bf16 rows (fp32 parameters): the position-dependent GroupNorm affine of the
// 0-D diffuser's FCBlock (gamma / beta per flattened channel c*sdim + s, openaimodel.py:2100-2112) after the statistics pass
__global__ void affine_act_rows_kernel(const __nv_bfloat16* __restrict__ x, long long rows, int n, const float* __restrict__ gamma,
                                       const float* __restrict__ beta, int act, __nv_bfloat16* __restrict__ y) {
  const long long total = rows * (n / 8);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c0 = static_cast<int>(i % (n / 8)) * 8;
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(x) + i);
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c0)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c0 + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c0)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c0 + 4));
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16x2(w[k]);
      float a = f.x * gg[2 * k] + bb[2 * k], c = f.y * gg[2 * k + 1] + bb[2 * k + 1];
      if (act == 1) { a = silu_bf16_f(a); c = silu_bf16_f(c); }
      o[k] = pack_bf16x2(a, c);
    }
    reinterpret_cast<uint4*>(y)[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// ---- load-time weight repack (fp32 checkpoint layouts -> bf16 kernel layouts) ----
__global__ void pack_conv_weight_kernel(const float* __restrict__ w, int Cout, int Cin, int kh, int kw,
                                        __nv_bfloat16* __restrict__ out, long long ldo, long long col0) {
  const long long total = static_cast<long long>(Cout) * kh * kw * Cin;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % Cin);
    long long r = i / Cin;
    const int t = static_cast<int>(r % (kh * kw));
    const long long n = r / (kh * kw);
    out[n * ldo + col0 + static_cast<long long>(t) * Cin + ci] = __float2bfloat16(__ldg(w + (n * Cin + ci) * (kh * kw) + t));
  }
}
__global__ void pack_geglu_kernel(const float* __restrict__ w, const float* __restrict__ b, int n2, int K,
                                  __nv_bfloat16* __restrict__ w_out, float* __restrict__ b_out) {
  const long long total = 2LL * n2 * K;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % K);
    const int row = static_cast<int>(i / K);            // packed row: tile t = row / 256, r = row % 256
    const int t = row >> 8, r = row & 255;
    const int srow = (r < 128) ? t * 128 + r : n2 + t * 128 + (r - 128);
    w_out[i] = __float2bfloat16(__ldg(w + static_cast<long long>(srow) * K + k));
    if (k == 0 && b) b_out[row] = __ldg(b + srow);
  }
}
__global__ void pad_heads_kernel(const float* __restrict__ w, int H, int d, int dpad, int K, __nv_bfloat16* __restrict__ out) {
  const long long total = static_cast<long long>(H) * dpad * K;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % K);
    const int row = static_cast<int>(i / K);
    const int h = row / dpad, c = row % dpad;
    out[i] = (c < d) ? __float2bfloat16(__ldg(w + (static_cast<long long>(h) * d + c) * K + k)) : __float2bfloat16(0.f);
  }
}

// The last vdb_groupnorm_nhwc / vdb_layernorm launch on this thread (vdb_norm_last_plan): family, two template parameters,
// G, S, nsplit, grid x / y / z.  Families: 1 gn_bundle <NVMAX, THREADS>, 2 gn_fused <NV, 0>, 3 gn_stats_apply (the statistics
// kernel's grid), 4 ln_rg <VPL, LPR>, 5 ln_warp <MAXV, R>.
constexpr int kNormPlanFields = 9;
static thread_local int g_norm_plan[kNormPlanFields] = {0};
static void set_norm_plan(int family, int t0, int t1, int G, int S, int nsplit, dim3 grid) {
  const int plan[kNormPlanFields] = {family, t0, t1, G, S, nsplit, static_cast<int>(grid.x), static_cast<int>(grid.y),
                                     static_cast<int>(grid.z)};
  for (int i = 0; i < kNormPlanFields; ++i) g_norm_plan[i] = plan[i];
}

static int ew_blocks(long long work_items, int threads) {
  long long b = (work_items + threads - 1) / threads;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return static_cast<int>(b);
}

// whether a_floats floats from a and b_floats floats from b share a byte (a NULL pointer shares none)
static bool overlaps(const void* a, long long a_floats, const void* b, long long b_floats) {
  if (!a || !b) return false;
  const uintptr_t a_lo = reinterpret_cast<uintptr_t>(a), a_hi = a_lo + static_cast<uintptr_t>(a_floats) * sizeof(float);
  const uintptr_t b_lo = reinterpret_cast<uintptr_t>(b), b_hi = b_lo + static_cast<uintptr_t>(b_floats) * sizeof(float);
  return a_lo < b_hi && b_lo < a_hi;
}

}  // namespace vdb

using namespace vdb;

extern "C" {

int vdb_ddim_cfg_step(const float* e_uncond, const float* e_cond, const float* x, const float* noise,
                      const float* coef, const int* step_idx, float scale, float temperature, float* x_prev,
                      float* x_prev_dup, float* pred_x0, long long n, void* stream) {
  if (!e_cond || !x || !coef || !x_prev || n <= 0) return set_error(VDB_ERR_INVALID, "ddim_cfg_step: null/empty argument");
  if ((reinterpret_cast<uintptr_t>(e_cond) | reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(x_prev) |
       reinterpret_cast<uintptr_t>(e_uncond) | reinterpret_cast<uintptr_t>(noise) | reinterpret_cast<uintptr_t>(pred_x0) |
       reinterpret_cast<uintptr_t>(x_prev_dup)) & 15)
    return set_error(VDB_ERR_INVALID, "ddim_cfg_step: pointers must be 16-byte aligned");
  const int threads = 256;
  return launch(ddim_cfg_step_kernel, ew_blocks((n + 3) / 4, threads), threads, 0, stream, e_uncond, e_cond, x, noise, coef,
                step_idx, scale, temperature, x_prev, x_prev_dup, pred_x0, n);
}

int vdb_dpmpp_cfg_step(const float* e_uncond, const float* e_cond, const float* x, const float* coef, const int* step_idx,
                       float scale, float* hist, float* x_next, float* x_next_dup, float* pred_x0, long long n, void* stream) {
  if (!e_cond || !x || !coef || !step_idx || !hist || !x_next || n <= 0)
    return set_error(VDB_ERR_INVALID, "dpmpp_cfg_step: null/empty argument");
  if ((reinterpret_cast<uintptr_t>(e_cond) | reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(x_next) |
       reinterpret_cast<uintptr_t>(e_uncond) | reinterpret_cast<uintptr_t>(hist) | reinterpret_cast<uintptr_t>(pred_x0) |
       reinterpret_cast<uintptr_t>(x_next_dup)) & 15)
    return set_error(VDB_ERR_INVALID, "dpmpp_cfg_step: pointers must be 16-byte aligned");
  // the ring is written while x is read and x_next / x_next_dup / pred_x0 are written: it must not share a byte with them
  for (const float* p : {x, static_cast<const float*>(x_next), static_cast<const float*>(x_next_dup),
                         static_cast<const float*>(pred_x0)})
    if (overlaps(hist, 3 * n, p, n)) return set_error(VDB_ERR_INVALID, "dpmpp_cfg_step: hist overlaps x, x_next, x_next_dup or pred_x0");
  const int threads = 256;
  return launch(dpmpp_cfg_step_kernel, ew_blocks((n + 3) / 4, threads), threads, 0, stream, e_uncond, e_cond, x, coef, step_idx,
                scale, hist, x_next, x_next_dup, pred_x0, n);
}

int vdb_dpmpp_sde_cfg_step(const float* e_uncond, const float* e_cond, const float* x, const float* coef, const int* step_idx,
                           float scale, float* hist, float* x_next, float* x_next_dup, float* pred_x0, long long n,
                           const unsigned long long* seed, const float* noise, void* stream) {
  if (!e_cond || !x || !coef || !step_idx || !hist || !x_next || n <= 0)
    return set_error(VDB_ERR_INVALID, "dpmpp_sde_cfg_step: null/empty argument");
  if (!seed && !noise) return set_error(VDB_ERR_INVALID, "dpmpp_sde_cfg_step: null seed and noise (one is needed)");
  if ((reinterpret_cast<uintptr_t>(e_cond) | reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(x_next) |
       reinterpret_cast<uintptr_t>(e_uncond) | reinterpret_cast<uintptr_t>(hist) | reinterpret_cast<uintptr_t>(pred_x0) |
       reinterpret_cast<uintptr_t>(x_next_dup) | reinterpret_cast<uintptr_t>(noise)) & 15)
    return set_error(VDB_ERR_INVALID, "dpmpp_sde_cfg_step: pointers must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(seed) & 7) return set_error(VDB_ERR_INVALID, "dpmpp_sde_cfg_step: seed must be 8-byte aligned");
  for (const float* p : {x, static_cast<const float*>(x_next), static_cast<const float*>(x_next_dup),
                         static_cast<const float*>(pred_x0)})
    if (overlaps(hist, 3 * n, p, n))
      return set_error(VDB_ERR_INVALID, "dpmpp_sde_cfg_step: hist overlaps x, x_next, x_next_dup or pred_x0");
  // the noise is read through the read-only path while the outputs are written: it must not share a byte with them
  if (overlaps(noise, n, hist, 3 * n) || overlaps(noise, n, x_next, n) || overlaps(noise, n, x_next_dup, n) ||
      overlaps(noise, n, pred_x0, n))
    return set_error(VDB_ERR_INVALID, "dpmpp_sde_cfg_step: noise overlaps hist, x_next, x_next_dup or pred_x0");
  const int threads = 256;
  return launch(dpmpp_sde_cfg_step_kernel, ew_blocks((n + 3) / 4, threads), threads, 0, stream, e_uncond, e_cond, x, coef,
                step_idx, scale, hist, x_next, x_next_dup, pred_x0, n, seed, noise);
}

int vdb_inpaint_blend_f32(float* x, float* x_dup, const float* x0, const float* mask, int mask_per_item, const float* table,
                          const int* step_idx, const unsigned long long* seed, const float* noise, int bs, long long hw, int c,
                          void* stream) {
  if (!x || !x0 || !mask || !table || !step_idx || (!seed && !noise) || bs <= 0 || hw <= 0 || c <= 0)
    return set_error(VDB_ERR_INVALID, "inpaint_blend: null/empty argument");
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(x_dup) | reinterpret_cast<uintptr_t>(x0) |
       reinterpret_cast<uintptr_t>(mask) | reinterpret_cast<uintptr_t>(table) | reinterpret_cast<uintptr_t>(noise)) & 15)
    return set_error(VDB_ERR_INVALID, "inpaint_blend: pointers must be 16-byte aligned");
  const long long n = static_cast<long long>(bs) * hw * c;
  // x / x_dup are written while x0, the mask and the noise are read through the read-only path: no byte may be shared
  for (const float* o : {static_cast<const float*>(x), static_cast<const float*>(x_dup)})
    if (overlaps(o, n, x0, n) || overlaps(o, n, mask, (mask_per_item ? bs : 1) * hw) || overlaps(o, n, noise, n))
      return set_error(VDB_ERR_INVALID, "inpaint_blend: x0, mask or noise overlaps x or x_dup");
  const int threads = 256;
  return launch(inpaint_blend_kernel, ew_blocks((n + 3) / 4, threads), threads, 0, stream, x, x_dup, x0, mask, mask_per_item,
                table, step_idx, seed, noise, n, hw, c);
}

int vdb_inpaint_noise_f32(const unsigned long long* seed, const int* step_idx, long long n, float* out, void* stream) {
  if (!seed || !step_idx || !out || n <= 0) return set_error(VDB_ERR_INVALID, "inpaint_noise: null/empty argument");
  return launch(inpaint_noise_kernel, ew_blocks((n + 3) / 4, 256), 256, 0, stream, seed, step_idx, n, out);
}

int vdb_mask_to_latent(const float* mask, int n, int H8, int W8, float* out, void* stream) {
  if (!mask || !out || n <= 0 || H8 <= 0 || W8 <= 0) return set_error(VDB_ERR_INVALID, "mask_to_latent: null/empty argument");
  if (H8 % 8 || W8 % 8) return set_error(VDB_ERR_INVALID, "mask_to_latent: H8 and W8 must be multiples of 8");
  return launch(mask_to_latent_kernel, ew_blocks(static_cast<long long>(n) * (H8 / 8) * (W8 / 8), 256), 256, 0, stream, mask, n,
                H8, W8, out);
}

int vdb_composite_f32(const float* decoded, const float* image, const float* mask, int mask_per_item, int n, int c, long long hw,
                      float* out, void* stream) {
  if (!decoded || !image || !mask || !out || n <= 0 || c <= 0 || hw <= 0)
    return set_error(VDB_ERR_INVALID, "composite: null/empty argument");
  const long long total = static_cast<long long>(n) * c * hw;
  return launch(composite_kernel, ew_blocks(total, 256), 256, 0, stream, decoded, image, mask, mask_per_item, c, hw, total, out);
}

int vdb_latent_store_slot_f32(const float* x, float* ring, int slots, const int* step_idx, int offset, long long n,
                              void* stream) {
  if (!x || !ring || !step_idx || slots <= 0 || n <= 0) return set_error(VDB_ERR_INVALID, "latent_store_slot: null/empty argument");
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(ring)) & 15)
    return set_error(VDB_ERR_INVALID, "latent_store_slot: pointers must be 16-byte aligned");
  if (overlaps(x, n, ring, static_cast<long long>(slots) * n))
    return set_error(VDB_ERR_INVALID, "latent_store_slot: x overlaps the ring");
  return launch(latent_store_slot_kernel, ew_blocks((n + 3) / 4, 256), 256, 0, stream, x, ring, slots, step_idx, offset, n);
}

int vdb_inversion_blend_f32(float* x, float* x_dup, const float* ring, int slots, const float* mask, int mask_per_item,
                            const int* step_idx, int bs, long long hw, int c, void* stream) {
  if (!x || !ring || !mask || !step_idx || slots <= 0 || bs <= 0 || hw <= 0 || c <= 0)
    return set_error(VDB_ERR_INVALID, "inversion_blend: null/empty argument");
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(x_dup) | reinterpret_cast<uintptr_t>(ring) |
       reinterpret_cast<uintptr_t>(mask)) & 15)
    return set_error(VDB_ERR_INVALID, "inversion_blend: pointers must be 16-byte aligned");
  const long long n = static_cast<long long>(bs) * hw * c;
  // x / x_dup are written while the ring and the mask are read through the read-only path: no byte may be shared
  for (const float* o : {static_cast<const float*>(x), static_cast<const float*>(x_dup)})
    if (overlaps(o, n, ring, static_cast<long long>(slots) * n) || overlaps(o, n, mask, (mask_per_item ? bs : 1) * hw))
      return set_error(VDB_ERR_INVALID, "inversion_blend: ring or mask overlaps x or x_dup");
  return launch(inversion_blend_kernel, ew_blocks((n + 3) / 4, 256), 256, 0, stream, x, x_dup, ring, slots, mask, mask_per_item,
                step_idx, n, hw, c);
}

int vdb_local_blend_f32(float* x, float* x_dup, const float* map, const int* flags, const int* step_idx, int n, int H, int W, int C,
                        int h, int w, float threshold, void* stream) {
  if (!x || !map || !flags || !step_idx || n < 2 || H <= 0 || W <= 0 || C <= 0 || h <= 0 || w <= 0)
    return set_error(VDB_ERR_INVALID, "local_blend: null/empty argument (n >= 2: a source and a target)");
  if (static_cast<long long>(h) * w > kBlendMaxMap)
    return set_error(VDB_ERR_INVALID, "local_blend: word maps of at most %d cells, got %d x %d", kBlendMaxMap, h, w);
  if (!(threshold == threshold) || threshold == INFINITY || threshold == -INFINITY)
    return set_error(VDB_ERR_INVALID, "local_blend: threshold must be finite");
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(x_dup) | reinterpret_cast<uintptr_t>(map) |
       reinterpret_cast<uintptr_t>(flags) | reinterpret_cast<uintptr_t>(step_idx)) & 3)
    return set_error(VDB_ERR_INVALID, "local_blend: pointers must be 4-byte aligned");
  const long long nx = static_cast<long long>(n) * H * W * C;
  if (overlaps(x, nx, map, static_cast<long long>(n) * h * w) || (x_dup && (overlaps(x_dup, nx, map, static_cast<long long>(n) * h * w) ||
                                                                         overlaps(x_dup, nx, x, nx))))
    return set_error(VDB_ERR_INVALID, "local_blend: x, x_dup and map must not overlap");
  return launch(local_blend_kernel, n - 1, kBlendThreads, 0, stream, x, x_dup, map, flags, step_idx, H, W, C, h, w, threshold);
}

// the refusals shared by the region gather and merge: sizes, the window range and the tables' alignment
static int window_args(const char* what, const void* x, int bs, int H, int W, int C, const int* oy, const int* ox, int ny, int nx,
                       int h, int w, int first, int k) {
  if (!x || !oy || !ox || bs <= 0 || H <= 0 || W <= 0 || C <= 0 || ny <= 0 || nx <= 0 || h <= 0 || w <= 0 || k <= 0)
    return set_error(VDB_ERR_INVALID, "%s: null/empty argument", what);
  if (h > H || w > W) return set_error(VDB_ERR_INVALID, "%s: window %d x %d larger than the canvas %d x %d", what, h, w, H, W);
  if (first < 0 || static_cast<long long>(first) + k > static_cast<long long>(ny) * nx)
    return set_error(VDB_ERR_INVALID, "%s: windows [%d, %d + %d) outside the layout's %d x %d", what, first, first, k, ny, nx);
  if ((reinterpret_cast<uintptr_t>(oy) | reinterpret_cast<uintptr_t>(ox)) & 3)
    return set_error(VDB_ERR_INVALID, "%s: tables must be 4-byte aligned", what);
  return 0;
}

int vdb_region_gather_f32(const float* x, int bs, int H, int W, int C, const int* oy, const int* ox, int ny, int nx, int h, int w,
                          int first, int k, int R, int u_blocks, const float* masks, const float* rows, const int* step_idx,
                          const unsigned long long* seed, const float* bg, int nb, const float* noise, float* out, void* stream) {
  if (!out) return set_error(VDB_ERR_INVALID, "region_gather: null/empty argument");
  if (int st = window_args("region_gather", x, bs, H, W, C, oy, ox, ny, nx, h, w, first, k)) return st;
  if (R < 0 || R > kRegionsMax) return set_error(VDB_ERR_INVALID, "region_gather: R must be in [0, %d], got %d", kRegionsMax, R);
  if (u_blocks != 0 && u_blocks != 1 && u_blocks != R + 1)
    return set_error(VDB_ERR_INVALID, "region_gather: u_blocks must be 0, 1 or R + 1 = %d, got %d", R + 1, u_blocks);
  if (rows && ((R > 0 && !masks) || !step_idx || !seed || !bg || nb <= 0))
    return set_error(VDB_ERR_INVALID, "region_gather: null/empty argument (rows needs masks, step_idx, seed and nb > 0 backgrounds)");
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(noise)) & 15 ||
      (reinterpret_cast<uintptr_t>(masks) | reinterpret_cast<uintptr_t>(rows) | reinterpret_cast<uintptr_t>(bg) |
       reinterpret_cast<uintptr_t>(step_idx)) & 3 || reinterpret_cast<uintptr_t>(seed) & 7)
    return set_error(VDB_ERR_INVALID, "region_gather: x, out and noise must be 16-byte aligned, masks, rows, bg and step_idx 4-byte, "
                                      "seed 8-byte");
  const long long nin = static_cast<long long>(bs) * H * W * C;
  const long long nout = static_cast<long long>(u_blocks + R + 1) * k * bs * h * w * C;
  // the batch is written while everything else is read through the read-only path: no byte may be shared
  if (overlaps(out, nout, x, nin) || (rows && (overlaps(out, nout, masks, static_cast<long long>(R) * bs * H * W) ||
                                                overlaps(out, nout, noise, nin) || overlaps(out, nout, bg, static_cast<long long>(nb) * C))))
    return set_error(VDB_ERR_INVALID, "region_gather: out overlaps x, masks, noise or bg");
  if ((C & 3) == 0)
    return launch(region_gather_kernel<4>, ew_blocks(nout / 4, 256), 256, 0, stream, x, bs, H, W, C, oy, ox, nx, h, w, first, k,
                  u_blocks, masks, rows, step_idx, seed, bg, nb, noise, nout / 4, out);
  return launch(region_gather_kernel<1>, ew_blocks(nout, 256), 256, 0, stream, x, bs, H, W, C, oy, ox, nx, h, w, first, k, u_blocks,
                masks, rows, step_idx, seed, bg, nb, noise, nout, out);
}

int vdb_region_noise_f32(const unsigned long long* seed, const int* step_idx, long long n, int R, int bs, int nb, float* z, int* picks,
                         void* stream) {
  if (!seed || !step_idx || !z || !picks || n <= 0 || bs <= 0 || nb <= 0)
    return set_error(VDB_ERR_INVALID, "region_noise: null/empty argument");
  if (R < 1 || R > kRegionsMax) return set_error(VDB_ERR_INVALID, "region_noise: R must be in [1, %d], got %d", kRegionsMax, R);
  const long long quads = (n + 3) / 4, total = quads > static_cast<long long>(R) * bs ? quads : static_cast<long long>(R) * bs;
  return launch(region_noise_kernel, ew_blocks(total, 256), 256, 0, stream, seed, step_idx, n, R, bs, nb, z, picks);
}

int vdb_region_merge_f32(const float* eps, int halves, int bs, int H, int W, int C, const int* oy, const int* ox, const int* cover_y,
                         const int* cover_x, int ny, int nx, int h, int w, int first, int k, int R, const float* masks, float* out,
                         void* stream) {
  if (!out || !cover_y || !cover_x || (R > 0 && !masks) || (halves != 1 && halves != 2))
    return set_error(VDB_ERR_INVALID, "region_merge: null/empty argument (halves 1 or 2)");
  if (int st = window_args("region_merge", eps, bs, H, W, C, oy, ox, ny, nx, h, w, first, k)) return st;
  if (R < 0 || R > kRegionsMax) return set_error(VDB_ERR_INVALID, "region_merge: R must be in [0, %d], got %d", kRegionsMax, R);
  if ((reinterpret_cast<uintptr_t>(eps) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(cover_x)) & 15 ||
      (reinterpret_cast<uintptr_t>(cover_y) | reinterpret_cast<uintptr_t>(masks)) & 3)
    return set_error(VDB_ERR_INVALID, "region_merge: eps, out and cover_x must be 16-byte aligned, cover_y and masks 4-byte");
  const long long nout = static_cast<long long>(halves) * bs * H * W * C;
  if (overlaps(out, nout, eps, static_cast<long long>(halves) * (R + 1) * k * bs * h * w * C) ||
      overlaps(out, nout, masks, static_cast<long long>(R) * bs * H * W))
    return set_error(VDB_ERR_INVALID, "region_merge: eps or masks overlaps out");
  if ((C & 3) == 0)
    return launch(region_merge_kernel<4>, ew_blocks(nout / 4, 256), 256, 0, stream, eps, bs, H, W, C, oy, ox, cover_y, cover_x, nx,
                  h, w, first, k, R, masks, nout / 4, out);
  return launch(region_merge_kernel<1>, ew_blocks(nout, 256), 256, 0, stream, eps, bs, H, W, C, oy, ox, cover_y, cover_x, nx, h, w,
                first, k, R, masks, nout, out);
}

int vdb_diffedit_mask_f32(const float* e_src_u, const float* e_src_c, float s_src, const float* e_tgt_u, const float* e_tgt_c,
                          float s_tgt, int D, int bs, long long hw, int c, float ratio, float* out, void* stream) {
  if (!e_src_c || !e_tgt_c || !out || D <= 0 || bs <= 0 || hw <= 0 || c <= 0)
    return set_error(VDB_ERR_INVALID, "diffedit_mask: null/empty argument");
  if (!(ratio > 0.f) || !(ratio < INFINITY)) return set_error(VDB_ERR_INVALID, "diffedit_mask: ratio must be finite and > 0");
  if ((reinterpret_cast<uintptr_t>(e_src_u) | reinterpret_cast<uintptr_t>(e_src_c) | reinterpret_cast<uintptr_t>(e_tgt_u) |
       reinterpret_cast<uintptr_t>(e_tgt_c) | reinterpret_cast<uintptr_t>(out)) & 15)
    return set_error(VDB_ERR_INVALID, "diffedit_mask: pointers must be 16-byte aligned");
  const long long n = static_cast<long long>(D) * bs * hw * c;
  for (const float* e : {e_src_u, e_src_c, e_tgt_u, e_tgt_c})
    if (overlaps(out, static_cast<long long>(bs) * hw, e, n))
      return set_error(VDB_ERR_INVALID, "diffedit_mask: out overlaps an eps input");
  return launch(diffedit_mask_kernel, bs, kDiffEditThreads, 0, stream, e_src_u, e_src_c, s_src, e_tgt_u, e_tgt_c, s_tgt, D, bs,
                hw, c, ratio, out);
}

int vdb_sag_degrade_f32(const float* x, const float* e, const float* mass, const float* table, const int* step_idx, int bs, int H,
                        int W, int C, int hm, int wm, float* out, void* stream) {
  if (!x || !e || !mass || !table || !step_idx || !out || bs <= 0 || H <= 0 || W <= 0 || C <= 0 || hm <= 0 || wm <= 0)
    return set_error(VDB_ERR_INVALID, "sag_degrade: null/empty argument");
  if (H <= kSagHalo || W <= kSagHalo)
    return set_error(VDB_ERR_INVALID, "sag_degrade: reflect padding by %d needs sides >= %d, got %d x %d", kSagHalo, kSagHalo + 1, H, W);
  if (C > kSagMaxC || hm > H || wm > W || hm * wm > kSagMaxMap)
    return set_error(VDB_ERR_UNSUPPORTED, "sag_degrade: need C <= %d and a map of hm <= H, wm <= W, hm * wm <= %d (got C %d, %d x %d)",
                     kSagMaxC, kSagMaxMap, C, hm, wm);
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(e) | reinterpret_cast<uintptr_t>(mass) |
       reinterpret_cast<uintptr_t>(table) | reinterpret_cast<uintptr_t>(step_idx) | reinterpret_cast<uintptr_t>(out)) & 3)
    return set_error(VDB_ERR_INVALID, "sag_degrade: pointers must be 4-byte aligned");
  const long long n = static_cast<long long>(bs) * H * W * C;
  if (overlaps(out, n, x, n) || overlaps(out, n, e, n) || overlaps(out, n, mass, static_cast<long long>(bs) * hm * wm))
    return set_error(VDB_ERR_INVALID, "sag_degrade: out overlaps x, e or mass");
  // the Gaussian of sigma 1: exp(-k^2 / 2) for k = -4 .. 4, normalised to sum 1 in double
  SagTaps taps;
  double g[kSagTaps], sum = 0.0;
  for (int k = 0; k < kSagTaps; ++k) sum += g[k] = exp(-0.5 * (k - kSagHalo) * (k - kSagHalo));
  for (int k = 0; k < kSagTaps; ++k) taps.g[k] = static_cast<float>(g[k] / sum);
  return launch(sag_degrade_kernel, dim3((W + kSagTile - 1) / kSagTile, (H + kSagTile - 1) / kSagTile, bs),
                dim3(kSagTile * kSagTile), 0, stream, x, e, mass, table, step_idx, taps, H, W, C, hm, wm, out);
}

int vdb_sag_guide_f32(float* e_u, float* e_c, const float* e_deg, float s, long long n, void* stream) {
  if (!e_c || !e_deg || n <= 0) return set_error(VDB_ERR_INVALID, "sag_guide: null/empty argument");
  if (!std::isfinite(s)) return set_error(VDB_ERR_INVALID, "sag_guide: scale must be finite");
  if ((reinterpret_cast<uintptr_t>(e_u) | reinterpret_cast<uintptr_t>(e_c) | reinterpret_cast<uintptr_t>(e_deg)) & 3)
    return set_error(VDB_ERR_INVALID, "sag_guide: pointers must be 4-byte aligned");
  if (overlaps(e_c, n, e_deg, n) || overlaps(e_u, n, e_deg, n) || overlaps(e_u, n, e_c, n))
    return set_error(VDB_ERR_INVALID, "sag_guide: e_u, e_c and e_deg must not overlap");
  const int threads = 256;
  return launch(sag_guide_kernel, ew_blocks(n, threads), threads, 0, stream, e_u, e_c, e_deg, s, n);
}

int vdb_axpby_f32(const float* x, const float* z, float a, float b, float* y, long long n, void* stream) {
  if (!x || !z || !y || n <= 0) return set_error(VDB_ERR_INVALID, "axpby: null/empty argument");
  return launch(axpby_kernel, ew_blocks(n, 256), 256, 0, stream, x, z, a, b, y, n);
}

int vdb_lincomb4_f32(const float* x0, const float* x1, const float* x2, const float* x3, float c0, float c1, float c2,
                     float c3, float* y, long long n, void* stream) {
  if (!x0 || !y || n <= 0) return set_error(VDB_ERR_INVALID, "lincomb4: null/empty argument");
  return launch(lincomb4_kernel, ew_blocks(n, 256), 256, 0, stream, x0, x1, x2, x3, c0, c1, c2, c3, y, n);
}

int vdb_add_int(int* p, int delta, void* stream) {
  if (!p) return set_error(VDB_ERR_INVALID, "add_int: null");
  return launch(add_int_kernel, 1, 1, 0, stream, p, delta);
}

// see include/vdb200.h
int vdb_norm_last_plan(int* out, int n) {
  for (int i = 0; out && i < n && i < kNormPlanFields; ++i) out[i] = g_norm_plan[i];
  return kNormPlanFields;
}

// scratch: ZERO-INITIALISED device buffer of vdb_groupnorm_scratch_floats(B, HW) floats (reusable across calls on
// one stream: the kernels leave its counters at zero)
int vdb_groupnorm_nsplit(int B, int HW) {
  int ns = (HW + 127) / 128;
  const int want = std::max(1, (4 * num_sms()) / std::max(B, 1));
  ns = std::min(ns, want);
  ns = std::min(ns, 256);
  return std::max(ns, 1);
}
long long vdb_groupnorm_scratch_floats(int B, int HW) {
  const long long ns = vdb_groupnorm_nsplit(B, HW);
  const long long parts = std::max<long long>(static_cast<long long>(B) * ns, 2 * num_sms());  // single-launch path: <= 2 CTAs / SM
  return 2 * kGnMaxBatch + static_cast<long long>(B) * 64 + parts * 64;
}

int vdb_groupnorm_nhwc(const void* x1, int C1, const void* x2, int C2, int B, int HW, int groups, const float* gamma,
                       const float* beta, float eps, int act, float* scratch, void* y, void* stream) {
  const int C = C1 + (x2 ? C2 : 0);
  if (!x1 || !gamma || !beta || !scratch || !y) return set_error(VDB_ERR_INVALID, "groupnorm: null argument");
  if (B > kGnMaxBatch) return set_error(VDB_ERR_UNSUPPORTED, "groupnorm: batch > %d", kGnMaxBatch);
  if (groups != 32 || (C % groups) || (C1 % 8) || (x2 && (C2 % 8)) || C / 8 > kGnThreads)
    return set_error(VDB_ERR_UNSUPPORTED, "groupnorm: need 32 groups, C %% 32 == 0, C/8 <= 512 (C=%d)", C);
  if (!x2) C2 = 0;
  // group-bundle kernel: see gn_bundle_kernel
  if (groups == 32) {
    const int cpg = C / groups;
    int G = 1;
    while (G <= 4 && ((G * cpg) % 8)) G *= 2;
    const int BC = G * cpg, VPB = BC / 8;
    if (G <= 4 && cpg >= 4 && VPB >= 1 && VPB <= 64) {
      const __nv_bfloat16* x1b = reinterpret_cast<const __nv_bfloat16*>(x1);
      const __nv_bfloat16* x2b = reinterpret_cast<const __nv_bfloat16*>(x2);
      __nv_bfloat16* yb = reinterpret_cast<__nv_bfloat16*>(y);
      auto launch_bundle = [&](auto kernel, int nvmax, int threads, int S, size_t smem = 0) -> int {
        const dim3 grid(groups / G, S, B);
        set_norm_plan(1, nvmax, threads, G, S, 0, grid);
        return launch(dim3(1, S, 1), kernel, grid, dim3(threads), smem, stream, x1b, C1, x2b, C2, HW, groups, G, eps, act, gamma,
                      beta, yb);
      };
      auto nper_t = [&](int threads, int S) { const int ln = threads / VPB; return (((HW + S - 1) / S) + ln - 1) / ln; };
      // big layers (the 64x64 level at B = 8): 1024-thread CTAs, one per SM, the pixels staged in up to 176 KB of shared memory:
      // a 4096-pixel C = 320 layer is ONE wave of 128 CTAs (2-CTA clusters) — with 512-thread register-resident CTAs it needs
      // 8-CTA clusters = 512 CTAs = 1.7 waves of the 296 resident slots (18 us measured) — and the C = 960 / 1920 concat
      // layers that fit neither variant before no longer fall back to the pixel-range kernel
      if (static_cast<long long>(HW) * B >= 16384) {
        for (int S = 1; S <= 8; S *= 2) {
          if (static_cast<long long>(groups / G) * S * B > 4LL * num_sms()) break;   // (at most ~4 waves of one CTA per SM)
          if (nper_t(1024, S) <= 11) {
            constexpr size_t smem = 11 * 1024 * sizeof(uint4);
            static bool configured = false;
            if (!configured) {
              VDB_CUDA_CHECK(cudaFuncSetAttribute(gn_bundle_kernel<11, 1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
              configured = true;
            }
            return launch_bundle(gn_bundle_kernel<11, 1024>, 11, 1024, S, smem);
          }
        }
      }
      const int lanes = 512 / VPB;
      auto nper = [&](int S) { return (((HW + S - 1) / S) + lanes - 1) / lanes; };
      int S = 1;
      while (S < 8 && nper(S) > 6) S *= 2;
      // small grids: more CTAs per image while every thread still keeps >= 2 pixels
      while (S < 8 && static_cast<long long>(groups / G) * S * B < num_sms() && nper(S * 2) >= 2) S *= 2;
      const int n = nper(S);
      if (n <= 2) return launch_bundle(gn_bundle_kernel<2, 512>, 2, 512, S);
      if (n <= 6) return launch_bundle(gn_bundle_kernel<6, 512>, 6, 512, S);
      if (n <= 12) return launch_bundle(gn_bundle_kernel<12, 512>, 12, 512, S);
    }
  }
  // every CTA of the single-launch kernel must be resident: ask the runtime how many fit (registers / shared memory)
  static const int occ0 = [] { int n = 0; cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, gn_fused_kernel<0>, kGnThreads, 0); return n; }();
  static const int occ4 = [] { int n = 0; cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, gn_fused_kernel<4>, kGnThreads, 0); return n; }();
  const int max_resident = std::min(2, std::min(occ0, occ4)) * num_sms();   // (the scratch is sized for 2 CTAs / SM)
  if (max_resident >= B && C <= 3072) {   // (shared-memory plan of the single-launch kernel)
    const int max_ns = max_resident / B;
    const int lanes = kGnThreads / (C / 8);
    const int ns4 = (HW + 4 * lanes - 1) / (4 * lanes);   // splits needed for <= 4 pixels per thread
    const __nv_bfloat16* x1b = reinterpret_cast<const __nv_bfloat16*>(x1);
    const __nv_bfloat16* x2b = reinterpret_cast<const __nv_bfloat16*>(x2);
    __nv_bfloat16* yb = reinterpret_cast<__nv_bfloat16*>(y);
    if (ns4 <= max_ns) {   // register-resident variant for the small layers
      const int ns = std::max(1, std::min(max_ns, std::max(ns4, (HW + 7) / 8)));
      set_norm_plan(2, 4, 0, 0, 0, ns, dim3(ns, B));
      return launch(gn_fused_kernel<4>, dim3(ns, B), dim3(kGnThreads), 0, stream, x1b, C1, x2b, C2, HW, groups, eps, act, gamma,
                    beta, scratch, yb);
    }
    const int ns = std::max(1, std::min(max_ns, (HW + 31) / 32));
    set_norm_plan(2, 0, 0, 0, 0, ns, dim3(ns, B));
    return launch(gn_fused_kernel<0>, dim3(ns, B), dim3(kGnThreads), 0, stream, x1b, C1, x2b, C2, HW, groups, eps, act, gamma, beta,
                  scratch, yb);
  }
  const int nsplit = vdb_groupnorm_nsplit(B, HW);
  set_norm_plan(3, 0, 0, 0, 0, nsplit, dim3(nsplit, B));
  const int rc = launch(gn_stats_kernel, dim3(nsplit, B), dim3(kGnThreads), 0, stream, reinterpret_cast<const __nv_bfloat16*>(x1),
                        C1, reinterpret_cast<const __nv_bfloat16*>(x2), C2, HW, groups, eps, scratch);
  if (rc) return rc;
  const float* stats = scratch + 2 * kGnMaxBatch;
  const long long work = static_cast<long long>(HW) * (C / 8);
  // ~8 vectors per thread: amortises the per-CTA scale/shift prologue
  int nblk = static_cast<int>(std::min<long long>((work + 2047) / 2048, std::max(1, (num_sms() * 8) / std::max(B, 1))));
  return launch(gn_apply_kernel, dim3(nblk, B), dim3(256), 2 * C * sizeof(float), stream, reinterpret_cast<const __nv_bfloat16*>(x1),
                C1, reinterpret_cast<const __nv_bfloat16*>(x2), C2, HW, groups, stats, gamma, beta, act,
                reinterpret_cast<__nv_bfloat16*>(y));
}

int vdb_layernorm(const void* x, long long rows, int C, const float* gamma, const float* beta, float eps, void* y,
                  void* stream) {
  if (!x || !gamma || !beta || !y || rows <= 0) return set_error(VDB_ERR_INVALID, "layernorm: null/empty argument");
  if ((C % 8) || C > 8 * 32 * 8) return set_error(VDB_ERR_UNSUPPORTED, "layernorm: C must be a multiple of 8, <= 2048");
  const int threads = 256;
  const int V = C / 8;
  const int R = V <= 64 ? 4 : (V <= 160 ? 2 : 1);
  const int blocks = static_cast<int>(std::min<long long>((rows + 8 * R - 1) / (8 * R), num_sms() * 8LL));
  const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(x);
  __nv_bfloat16* yp = reinterpret_cast<__nv_bfloat16*>(y);
  // row-group kernel where C = 8 * VPL * LPR has an instantiation, else the warp-per-row kernels
  auto launch_rg = [&](auto kernel, int vpl, int rpw) -> int {
    int occ = 0;
    const size_t smem = 2 * static_cast<size_t>(C) * sizeof(float);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, threads, smem) != cudaSuccess || occ < 1) occ = 1;
    const long long steps = (rows + rpw - 1) / rpw;                         // warp steps
    const int grid = static_cast<int>(std::max<long long>(1, std::min<long long>((steps + 7) / 8, static_cast<long long>(occ) * num_sms())));
    set_norm_plan(4, vpl, 32 / rpw, 0, 0, 0, dim3(grid));
    return launch(kernel, dim3(grid), dim3(threads), smem, stream, xp, rows, C, gamma, beta, eps, yp);
  };
  switch (V) {
    case 40: return launch_rg(layernorm_rg_kernel<5, 8>, 5, 4);      // C 320
    case 80: return launch_rg(layernorm_rg_kernel<5, 16>, 5, 2);     // C 640
    case 160: return launch_rg(layernorm_rg_kernel<5, 32>, 5, 1);    // C 1280
    case 96: return launch_rg(layernorm_rg_kernel<3, 32>, 3, 1);     // C 768  (CLIP text)
    case 128: return launch_rg(layernorm_rg_kernel<4, 32>, 4, 1);    // C 1024 (CLIP vision)
    case 8: return launch_rg(layernorm_rg_kernel<1, 8>, 1, 4);       // C 64   (reduced-width test nets)
    case 16: return launch_rg(layernorm_rg_kernel<2, 8>, 2, 4);      // C 128
    case 32: return launch_rg(layernorm_rg_kernel<4, 8>, 4, 4);      // C 256
    default: break;
  }
  set_norm_plan(5, V <= 64 ? 2 : (V <= 160 ? 5 : 8), R, 0, 0, 0, dim3(blocks));
  if (V <= 64) return launch(layernorm_kernel<2, 4>, dim3(blocks), dim3(threads), 0, stream, xp, rows, C, gamma, beta, eps, yp);
  if (V <= 160) return launch(layernorm_kernel<5, 2>, dim3(blocks), dim3(threads), 0, stream, xp, rows, C, gamma, beta, eps, yp);
  return launch(layernorm_kernel<8, 1>, dim3(blocks), dim3(threads), 0, stream, xp, rows, C, gamma, beta, eps, yp);
}

int vdb_affine_act_rows(const void* x, long long rows, int n, const float* gamma, const float* beta, int act, void* y, void* stream) {
  if (!x || !gamma || !beta || !y || rows <= 0 || n <= 0 || (n % 8)) return set_error(VDB_ERR_INVALID, "affine_act_rows: bad argument (n %% 8 == 0)");
  return launch(affine_act_rows_kernel, ew_blocks(rows * (n / 8), 256), 256, 0, stream, reinterpret_cast<const __nv_bfloat16*>(x),
                rows, n, gamma, beta, act, reinterpret_cast<__nv_bfloat16*>(y));
}

int vdb_pack_conv_weight(const float* w, int Cout, int Cin, int kh, int kw, void* out, long long ldo, long long col0, void* stream) {
  if (!w || !out || Cout <= 0 || Cin <= 0 || kh <= 0 || kw <= 0) return set_error(VDB_ERR_INVALID, "pack_conv_weight: null/empty argument");
  if (ldo < col0 + static_cast<long long>(kh) * kw * Cin) return set_error(VDB_ERR_INVALID, "pack_conv_weight: ldo too small");
  const long long total = static_cast<long long>(Cout) * kh * kw * Cin;
  return launch(pack_conv_weight_kernel, ew_blocks(total, 256), 256, 0, stream, w, Cout, Cin, kh, kw,
                reinterpret_cast<__nv_bfloat16*>(out), ldo, col0);
}

int vdb_pack_geglu(const float* w, const float* b, int n2, int K, void* w_out, float* b_out, void* stream) {
  if (!w || !w_out || n2 <= 0 || K <= 0 || (b && !b_out)) return set_error(VDB_ERR_INVALID, "pack_geglu: null/empty argument");
  if (n2 % 128) return set_error(VDB_ERR_INVALID, "pack_geglu: the GEGLU width must be a multiple of 128");
  return launch(pack_geglu_kernel, ew_blocks(2LL * n2 * K, 256), 256, 0, stream, w, b, n2, K,
                reinterpret_cast<__nv_bfloat16*>(w_out), b_out);
}

int vdb_pad_heads(const float* w, int H, int d, int dpad, int K, void* out, void* stream) {
  if (!w || !out || H <= 0 || d <= 0 || dpad < d || K <= 0) return set_error(VDB_ERR_INVALID, "pad_heads: bad argument");
  return launch(pad_heads_kernel, ew_blocks(static_cast<long long>(H) * dpad * K, 256), 256, 0, stream, w, H, d, dpad, K,
                reinterpret_cast<__nv_bfloat16*>(out));
}

int vdb_upsample2x_nhwc(const void* x, int B, int H, int W, int C, void* y, void* stream) {
  if (!x || !y || (C % 8)) return set_error(VDB_ERR_INVALID, "upsample2x: null argument or C %% 8 != 0");
  const long long total = static_cast<long long>(B) * 4 * H * W * (C / 8);
  return launch(upsample2x_kernel, ew_blocks(total, 256), 256, 0, stream, reinterpret_cast<const __nv_bfloat16*>(x), B, H, W, C,
                reinterpret_cast<__nv_bfloat16*>(y));
}

int vdb_clip_to_u8_hwc(const float* x, int n, int H, int W, void* y, void* stream) {
  if (!x || !y || n <= 0 || H <= 0 || W <= 0) return set_error(VDB_ERR_INVALID, "clip_to_u8_hwc: bad argument");
  return launch(clip_to_u8_hwc_kernel, ew_blocks(static_cast<long long>(n) * H * W * 3, 256), 256, 0, stream, x, n, H, W,
                reinterpret_cast<uint8_t*>(y));
}

int vdb_resample_h_u8(const void* x, int n, int H, int Win, int Wout, const int* bounds, const int* kk, int ksize, void* y,
                      void* stream) {
  if (!x || !y || !bounds || !kk || n <= 0 || H <= 0 || Win <= 0 || Wout <= 0 || ksize <= 0)
    return set_error(VDB_ERR_INVALID, "resample_h_u8: bad argument");
  return launch(resample_h_u8_kernel, ew_blocks(static_cast<long long>(n) * H * Wout * 3, 256), 256, 0, stream,
                reinterpret_cast<const uint8_t*>(x), n, H, Win, Wout, bounds, kk, ksize, reinterpret_cast<uint8_t*>(y));
}

int vdb_resample_v_crop_norm(const void* x, int n, int Hin, int W, const int* bounds, const int* kk, int ksize, int top,
                             int left, int S, const float* mean3, const float* std3, float* y, void* stream) {
  if (!x || !y || !mean3 || !std3 || n <= 0 || Hin <= 0 || W <= 0 || S <= 0 || top < 0 || left < 0 || left + S > W ||
      (ksize > 0 && (!bounds || !kk)) || (ksize == 0 && top + S > Hin))
    return set_error(VDB_ERR_INVALID, "resample_v_crop_norm: bad argument");
  return launch(resample_v_crop_norm_kernel, ew_blocks(static_cast<long long>(n) * 3 * S * S, 256), 256, 0, stream,
                reinterpret_cast<const uint8_t*>(x), n, Hin, W, bounds, kk, ksize, top, left, S, mean3[0], mean3[1], mean3[2],
                std3[0], std3[1], std3[2], y);
}

int vdb_im2col3x3_small(const float* x, int B, int H, int W, int Cin, int Kpad, float in_scale, float in_shift,
                        void* y, void* stream) {
  if (!x || !y || 9 * Cin > Kpad || (Kpad % 8)) return set_error(VDB_ERR_INVALID, "im2col3x3_small: bad argument");
  const long long total = static_cast<long long>(B) * H * W * (Kpad / 8);
  return launch(im2col3x3_small_kernel, ew_blocks(total, 256), 256, 0, stream, x, B, H, W, Cin, Kpad, in_scale, in_shift,
                reinterpret_cast<__nv_bfloat16*>(y));
}

int vdb_permute_f32(const float* x, int B, int C, long long HW, int to_nhwc, float mul, float add, int clamp01,
                    float* y, void* stream) {
  if (!x || !y) return set_error(VDB_ERR_INVALID, "permute_f32: null argument");
  const long long total = static_cast<long long>(B) * C * HW;
  return launch(permute_f32_kernel, ew_blocks(total, 256), 256, 0, stream, x, B, C, static_cast<int>(HW), to_nhwc, mul, add,
                clamp01, y);
}

int vdb_pointwise_small(const float* x, long long npix, int Cin, int Cout, const float* Wm, const float* bias,
                        float pre_mul, float* y, void* stream) {
  if (!x || !Wm || !y || Cin <= 0 || Cin > 8 || Cout <= 0 || Cout > 8)
    return set_error(VDB_ERR_INVALID, "pointwise_small: need 1 <= Cin, Cout <= 8");
  return launch(pointwise_small_kernel, ew_blocks(npix, 256), 256, 0, stream, x, npix, Cin, Cout, Wm, bias, pre_mul, y);
}

int vdb_gaussian_sample(const float* moments, const float* noise, int C, long long npix, float post_mul, float* z,
                        void* stream) {
  if (!moments || !z || C <= 0 || npix <= 0) return set_error(VDB_ERR_INVALID, "gaussian_sample: bad argument");
  return launch(gaussian_sample_kernel, ew_blocks(npix * C, 256), 256, 0, stream, moments, noise, C, npix, post_mul, z);
}

int vdb_cast_f32_bf16(const float* x, void* y, long long n, void* stream) {
  if (!x || !y) return set_error(VDB_ERR_INVALID, "cast: null argument");
  return launch(cast_f32_bf16_kernel, ew_blocks(n, 256), 256, 0, stream, x, reinterpret_cast<__nv_bfloat16*>(y), n);
}
int vdb_cast_bf16_f32(const void* x, float* y, long long n, void* stream) {
  if (!x || !y) return set_error(VDB_ERR_INVALID, "cast: null argument");
  return launch(cast_bf16_f32_kernel, ew_blocks(n, 256), 256, 0, stream, reinterpret_cast<const __nv_bfloat16*>(x), y, n);
}

int vdb_timestep_embedding(const long long* ts, const int* step_idx, int B, int dim, float neg_log_period, float* out,
                           void* stream) {
  if (!ts || !out || B <= 0 || dim <= 1) return set_error(VDB_ERR_INVALID, "timestep_embedding: bad argument");
  return launch(timestep_embedding_kernel, ew_blocks(static_cast<long long>(B) * (dim / 2), 128), 128, 0, stream, ts, step_idx, B,
                dim, neg_log_period, out);
}

int vdb_linear_small(const float* x, int M, int K, const void* Wt, int N, const float* bias, int act_in, int act_out,
                     float* out, void* stream) {
  if (!x || !Wt || !out || M <= 0 || M > 16 || (K % 8)) return set_error(VDB_ERR_INVALID, "linear_small: need 1 <= M <= 16, K %% 8 == 0");
  const size_t smem = static_cast<size_t>(M) * K * sizeof(float);
  if (smem > 200 * 1024) return set_error(VDB_ERR_UNSUPPORTED, "linear_small: M*K too large for shared memory");
  static bool configured = false;
  if (!configured) {
    VDB_CUDA_CHECK(cudaFuncSetAttribute(linear_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured = true;
  }
  const int blocks = std::min((N + 31) / 32, num_sms() * 2);
  return launch(linear_small_kernel, blocks, 256, smem, stream, x, M, K, reinterpret_cast<const __nv_bfloat16*>(Wt), N, bias,
                act_in, act_out, out);
}

int vdb_clip_text_embed(const long long* tokens, const float* tok_emb, const float* pos_emb, int B, int L, int Lp, int C,
                        void* x, void* stream) {
  if (!tokens || !tok_emb || !pos_emb || !x || Lp < L) return set_error(VDB_ERR_INVALID, "clip_text_embed: bad argument");
  return launch(clip_text_embed_kernel, ew_blocks(static_cast<long long>(B) * Lp * C, 256), 256, 0, stream, tokens, tok_emb,
                pos_emb, B, L, Lp, C, reinterpret_cast<__nv_bfloat16*>(x));
}

int vdb_patchify(const float* pixels, int B, int Cin, int HW, int P, int Kpad, void* y, void* stream) {
  if (!pixels || !y || HW % P || Cin * P * P > Kpad || (Kpad % 8)) return set_error(VDB_ERR_INVALID, "patchify: bad argument");
  const int G = HW / P;
  return launch(patchify_kernel, ew_blocks(static_cast<long long>(B) * G * G * Kpad, 256), 256, 0, stream, pixels, B, Cin, HW, P,
                Kpad, reinterpret_cast<__nv_bfloat16*>(y));
}

int vdb_vit_assemble(const void* patches, const float* cls, const float* pos, const float* tok_scale, int B, int L, int Lp,
                     int C, void* x, void* stream) {
  if (!patches || !cls || !pos || !x || Lp < L) return set_error(VDB_ERR_INVALID, "vit_assemble: bad argument");
  return launch(vit_assemble_kernel, ew_blocks(static_cast<long long>(B) * Lp * C, 256), 256, 0, stream,
                reinterpret_cast<const __nv_bfloat16*>(patches), cls, pos, tok_scale, B, L, Lp, C,
                reinterpret_cast<__nv_bfloat16*>(x));
}

int vdb_scale_by_row_norm(const void* z, const int* idx, const float* row_scale, int B, int L, int Lp, int C, float* out,
                          void* stream) {
  if (!z || !out || B <= 0 || Lp < L) return set_error(VDB_ERR_INVALID, "scale_by_row_norm: bad argument");
  return launch(scale_by_row_norm_kernel, B, 256, 0, stream, reinterpret_cast<const __nv_bfloat16*>(z), idx, row_scale, L, Lp, C,
                out);
}

int vdb_softmax_rows(const void* x, long long rows, int n, long long ld, float scale, void* y, void* stream) {
  if (!x || !y || rows <= 0 || n <= 0) return set_error(VDB_ERR_INVALID, "softmax_rows: bad argument");
  const int blocks = static_cast<int>(std::min<long long>(rows, num_sms() * 8LL));
  return launch(softmax_rows_kernel, blocks, 256, 0, stream, reinterpret_cast<const __nv_bfloat16*>(x), rows, n, ld, scale,
                reinterpret_cast<__nv_bfloat16*>(y));
}

}  // extern "C"
