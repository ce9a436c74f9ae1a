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
// ---------------------------------------------------------------------------------------------
__global__ void dpmpp_cfg_step_kernel(const float* __restrict__ e_uncond, const float* __restrict__ e_cond,
                                      const float* x, const float* __restrict__ coef, const int* __restrict__ step_idx,
                                      float scale, float* __restrict__ hist, float* x_next, float* __restrict__ x_next_dup,
                                      float* __restrict__ pred_x0, long long n) {
  const int idx = *step_idx;
  const float* c = coef + 8 * idx;
  const float P = c[0], Q = c[1], A = c[2], B = c[3], C = c[4], D = c[5];
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
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float e = ec[q];
      if (e_uncond) e = __fadd_rn(eu[q], __fmul_rn(scale, __fsub_rn(ec[q], eu[q])));
      const float px0 = __fadd_rn(__fmul_rn(P, xv[q]), __fmul_rn(Q, e));
      float v = __fadd_rn(__fmul_rn(A, xv[q]), __fmul_rn(B, px0));
      if (C != 0.f) v = __fadd_rn(v, __fmul_rn(C, a1[q]));
      if (D != 0.f) v = __fadd_rn(v, __fmul_rn(D, a2[q]));
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

// ---------------------------------------------------------------------------------------------
// Inpainting (lib/model_zoo/inpaint.py): blended latent diffusion.  After every sampler step the kept region (mask 0) is
// overwritten with the original latent re-noised to the step's target point, row *step_idx of the table {a, b}:
//   k  = a*x0 + b*z                       (explicit _rn: an fp32 CPU restatement is bitwise)
//   x' = m == 1 ? x' : m == 0 ? k : m*x' + (1 - m)*k
// z is the explicit noise when given, else the Philox4x32-10 stream below.  The exact selects at m = 0 and m = 1 make a hard
// mask keep x0 bit for bit at the last row {1, 0} and leave the generated region bit for bit as the step wrote it.
// ---------------------------------------------------------------------------------------------
constexpr unsigned kInpaintTag = 0x696e7074u;   // "inpt": the text decoder's stream uses "text" (0x74657874)

// Four standard normals of counter (quad, step, "inpt", 0) under a 64-bit key: two Box-Muller pairs, u = (b + 0.5) 2^-32 in
// fp64 (never 0 or 1), (r cos 2 pi u', r sin 2 pi u') with r = sqrt(-2 ln u), rounded to fp32.
__device__ __forceinline__ void inpaint_normals(unsigned long long key, unsigned quad, int step, float z[4]) {
  const uint4 b = curand_Philox4x32_10(make_uint4(quad, static_cast<unsigned>(step), kInpaintTag, 0u),
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
      xv[q] = m == 1.f ? xv[q] : m == 0.f ? k : __fadd_rn(__fmul_rn(m, xv[q]), __fmul_rn(__fsub_rn(1.f, m), k));
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
  pdl_launch_dependents();
  pdl_wait();
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
  pdl_launch_dependents();
  pdl_wait();
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
// Debug build only (-DVDB_TIMELINE, tools/gn_timeline.py): globaltimer stamps of thread 0 of CTA (0,0) of the single-launch
// GroupNorm: 0 start, 1 statistics loads + accumulation done, 2 partial published, 3 every CTA of the image arrived,
// 4 statistics folded, 5 scale / shift table ready, 6 normalised + stored.
__device__ unsigned long long* g_gn_timeline_dev = nullptr;
#ifdef VDB_TIMELINE
#define VDB_GTL(slot) do { if (g_gn_timeline_dev && threadIdx.x == 0 && blockIdx.x == 0 && blockIdx.y == 0) g_gn_timeline_dev[slot] = gtime(); } while (0)
#else
#define VDB_GTL(slot) do { } while (0)
#endif

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
  pdl_launch_dependents();
  pdl_wait();
  VDB_GTL(0);
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
  VDB_GTL(1);
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
  VDB_GTL(2);
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
  VDB_GTL(3);
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
  VDB_GTL(4);
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
  VDB_GTL(5);
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
  VDB_GTL(6);
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
  pdl_launch_dependents();
  pdl_wait();
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
  pdl_launch_dependents();
  pdl_wait();
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
  pdl_launch_dependents();
  pdl_wait();
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
  ddim_cfg_step_kernel<<<ew_blocks((n + 3) / 4, threads), threads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      e_uncond, e_cond, x, noise, coef, step_idx, scale, temperature, x_prev, x_prev_dup, pred_x0, n);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
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
  const uintptr_t h_lo = reinterpret_cast<uintptr_t>(hist), h_hi = h_lo + 3 * static_cast<uintptr_t>(n) * sizeof(float);
  for (const float* p : {x, static_cast<const float*>(x_next), static_cast<const float*>(x_next_dup),
                         static_cast<const float*>(pred_x0)}) {
    const uintptr_t lo = reinterpret_cast<uintptr_t>(p), hi = lo + static_cast<uintptr_t>(n) * sizeof(float);
    if (p && lo < h_hi && h_lo < hi) return set_error(VDB_ERR_INVALID, "dpmpp_cfg_step: hist overlaps x, x_next, x_next_dup or pred_x0");
  }
  const int threads = 256;
  dpmpp_cfg_step_kernel<<<ew_blocks((n + 3) / 4, threads), threads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      e_uncond, e_cond, x, coef, step_idx, scale, hist, x_next, x_next_dup, pred_x0, n);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
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
  const long long in_len[3] = {n, (mask_per_item ? bs : 1) * hw, n};
  const float* ins[3] = {x0, mask, noise};
  for (const float* o : {static_cast<const float*>(x), static_cast<const float*>(x_dup)}) {
    const uintptr_t o_lo = reinterpret_cast<uintptr_t>(o), o_hi = o_lo + static_cast<uintptr_t>(n) * sizeof(float);
    for (int k = 0; k < 3; ++k) {
      const uintptr_t lo = reinterpret_cast<uintptr_t>(ins[k]), hi = lo + static_cast<uintptr_t>(in_len[k]) * sizeof(float);
      if (o && ins[k] && lo < o_hi && o_lo < hi)
        return set_error(VDB_ERR_INVALID, "inpaint_blend: x0, mask or noise overlaps x or x_dup");
    }
  }
  const int threads = 256;
  inpaint_blend_kernel<<<ew_blocks((n + 3) / 4, threads), threads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, x_dup, x0, mask, mask_per_item, table, step_idx, seed, noise, n, hw, c);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_inpaint_noise_f32(const unsigned long long* seed, const int* step_idx, long long n, float* out, void* stream) {
  if (!seed || !step_idx || !out || n <= 0) return set_error(VDB_ERR_INVALID, "inpaint_noise: null/empty argument");
  inpaint_noise_kernel<<<ew_blocks((n + 3) / 4, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(seed, step_idx, n, out);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_mask_to_latent(const float* mask, int n, int H8, int W8, float* out, void* stream) {
  if (!mask || !out || n <= 0 || H8 <= 0 || W8 <= 0) return set_error(VDB_ERR_INVALID, "mask_to_latent: null/empty argument");
  if (H8 % 8 || W8 % 8) return set_error(VDB_ERR_INVALID, "mask_to_latent: H8 and W8 must be multiples of 8");
  mask_to_latent_kernel<<<ew_blocks(static_cast<long long>(n) * (H8 / 8) * (W8 / 8), 256), 256, 0,
                          reinterpret_cast<cudaStream_t>(stream)>>>(mask, n, H8, W8, out);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_composite_f32(const float* decoded, const float* image, const float* mask, int mask_per_item, int n, int c, long long hw,
                      float* out, void* stream) {
  if (!decoded || !image || !mask || !out || n <= 0 || c <= 0 || hw <= 0)
    return set_error(VDB_ERR_INVALID, "composite: null/empty argument");
  const long long total = static_cast<long long>(n) * c * hw;
  composite_kernel<<<ew_blocks(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(decoded, image, mask, mask_per_item,
                                                                                               c, hw, total, out);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_axpby_f32(const float* x, const float* z, float a, float b, float* y, long long n, void* stream) {
  if (!x || !z || !y || n <= 0) return set_error(VDB_ERR_INVALID, "axpby: null/empty argument");
  axpby_kernel<<<ew_blocks(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, z, a, b, y, n);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_lincomb4_f32(const float* x0, const float* x1, const float* x2, const float* x3, float c0, float c1, float c2,
                     float c3, float* y, long long n, void* stream) {
  if (!x0 || !y || n <= 0) return set_error(VDB_ERR_INVALID, "lincomb4: null/empty argument");
  lincomb4_kernel<<<ew_blocks(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x0, x1, x2, x3, c0, c1, c2, c3, y, n);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_add_int(int* p, int delta, void* stream) {
  if (!p) return set_error(VDB_ERR_INVALID, "add_int: null");
  add_int_kernel<<<1, 1, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, delta);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

// debug aid (stamps exist only in a -DVDB_TIMELINE build): 8 x u64 device buffer receiving the single-launch GroupNorm's phases
void vdb_debug_gn_timeline(void* buf) {
  unsigned long long* p = reinterpret_cast<unsigned long long*>(buf);
  cudaMemcpyToSymbol(vdb::g_gn_timeline_dev, &p, sizeof(p));
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
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
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
      auto launch = [&](auto kernel, int nvmax, int threads, int S, size_t smem = 0) -> int {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(groups / G, S, B); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
        set_norm_plan(1, nvmax, threads, G, S, 0, cfg.gridDim);
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = 1; attr[0].val.clusterDim.y = S; attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        VDB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, x1b, C1, x2b, C2, HW, groups, G, eps, act, gamma, beta, yb));
        count_launch();
        return VDB_OK;
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
            return launch(gn_bundle_kernel<11, 1024>, 11, 1024, S, smem);
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
      if (n <= 2) return launch(gn_bundle_kernel<2, 512>, 2, 512, S);
      if (n <= 6) return launch(gn_bundle_kernel<6, 512>, 6, 512, S);
      if (n <= 12) return launch(gn_bundle_kernel<12, 512>, 12, 512, S);
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
      VDB_CUDA_CHECK(launch_pdl(gn_fused_kernel<4>, dim3(ns, B), dim3(kGnThreads), 0, st, x1b, C1, x2b, C2, HW, groups, eps,
                                act, gamma, beta, scratch, yb));
    } else {
      const int ns = std::max(1, std::min(max_ns, (HW + 31) / 32));
      set_norm_plan(2, 0, 0, 0, 0, ns, dim3(ns, B));
      VDB_CUDA_CHECK(launch_pdl(gn_fused_kernel<0>, dim3(ns, B), dim3(kGnThreads), 0, st, x1b, C1, x2b, C2, HW, groups, eps,
                                act, gamma, beta, scratch, yb));
    }
    count_launch(1);
    return VDB_OK;
  }
  const int nsplit = vdb_groupnorm_nsplit(B, HW);
  set_norm_plan(3, 0, 0, 0, 0, nsplit, dim3(nsplit, B));
  VDB_CUDA_CHECK(launch_pdl(gn_stats_kernel, dim3(nsplit, B), dim3(kGnThreads), 0, st,
                            reinterpret_cast<const __nv_bfloat16*>(x1), C1, reinterpret_cast<const __nv_bfloat16*>(x2), C2,
                            HW, groups, eps, scratch));
  const float* stats = scratch + 2 * kGnMaxBatch;
  const long long work = static_cast<long long>(HW) * (C / 8);
  // ~8 vectors per thread: amortises the per-CTA scale/shift prologue
  int nblk = static_cast<int>(std::min<long long>((work + 2047) / 2048, std::max(1, (num_sms() * 8) / std::max(B, 1))));
  VDB_CUDA_CHECK(launch_pdl(gn_apply_kernel, dim3(nblk, B), dim3(256), 2 * C * sizeof(float), st,
                            reinterpret_cast<const __nv_bfloat16*>(x1), C1, reinterpret_cast<const __nv_bfloat16*>(x2), C2,
                            HW, groups, stats, gamma, beta, act, reinterpret_cast<__nv_bfloat16*>(y)));
  count_launch(2);
  return VDB_OK;
}

int vdb_layernorm(const void* x, long long rows, int C, const float* gamma, const float* beta, float eps, void* y,
                  void* stream) {
  if (!x || !gamma || !beta || !y || rows <= 0) return set_error(VDB_ERR_INVALID, "layernorm: null/empty argument");
  if ((C % 8) || C > 8 * 32 * 8) return set_error(VDB_ERR_UNSUPPORTED, "layernorm: C must be a multiple of 8, <= 2048");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
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
    VDB_CUDA_CHECK(launch_pdl(kernel, dim3(grid), dim3(threads), smem, st, xp, rows, C, gamma, beta, eps, yp));
    count_launch();
    return VDB_OK;
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
  if (V <= 64)
    VDB_CUDA_CHECK(launch_pdl(layernorm_kernel<2, 4>, dim3(blocks), dim3(threads), 0, st, xp, rows, C, gamma, beta, eps, yp));
  else if (V <= 160)
    VDB_CUDA_CHECK(launch_pdl(layernorm_kernel<5, 2>, dim3(blocks), dim3(threads), 0, st, xp, rows, C, gamma, beta, eps, yp));
  else
    VDB_CUDA_CHECK(launch_pdl(layernorm_kernel<8, 1>, dim3(blocks), dim3(threads), 0, st, xp, rows, C, gamma, beta, eps, yp));
  count_launch();
  return VDB_OK;
}

int vdb_affine_act_rows(const void* x, long long rows, int n, const float* gamma, const float* beta, int act, void* y, void* stream) {
  if (!x || !gamma || !beta || !y || rows <= 0 || n <= 0 || (n % 8)) return set_error(VDB_ERR_INVALID, "affine_act_rows: bad argument (n %% 8 == 0)");
  affine_act_rows_kernel<<<ew_blocks(rows * (n / 8), 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), rows, n, gamma, beta, act, reinterpret_cast<__nv_bfloat16*>(y));
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_pack_conv_weight(const float* w, int Cout, int Cin, int kh, int kw, void* out, long long ldo, long long col0, void* stream) {
  if (!w || !out || Cout <= 0 || Cin <= 0 || kh <= 0 || kw <= 0) return set_error(VDB_ERR_INVALID, "pack_conv_weight: null/empty argument");
  if (ldo < col0 + static_cast<long long>(kh) * kw * Cin) return set_error(VDB_ERR_INVALID, "pack_conv_weight: ldo too small");
  const long long total = static_cast<long long>(Cout) * kh * kw * Cin;
  pack_conv_weight_kernel<<<ew_blocks(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      w, Cout, Cin, kh, kw, reinterpret_cast<__nv_bfloat16*>(out), ldo, col0);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_pack_geglu(const float* w, const float* b, int n2, int K, void* w_out, float* b_out, void* stream) {
  if (!w || !w_out || n2 <= 0 || K <= 0 || (b && !b_out)) return set_error(VDB_ERR_INVALID, "pack_geglu: null/empty argument");
  if (n2 % 128) return set_error(VDB_ERR_INVALID, "pack_geglu: the GEGLU width must be a multiple of 128");
  pack_geglu_kernel<<<ew_blocks(2LL * n2 * K, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      w, b, n2, K, reinterpret_cast<__nv_bfloat16*>(w_out), b_out);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_pad_heads(const float* w, int H, int d, int dpad, int K, void* out, void* stream) {
  if (!w || !out || H <= 0 || d <= 0 || dpad < d || K <= 0) return set_error(VDB_ERR_INVALID, "pad_heads: bad argument");
  pad_heads_kernel<<<ew_blocks(static_cast<long long>(H) * dpad * K, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      w, H, d, dpad, K, reinterpret_cast<__nv_bfloat16*>(out));
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_upsample2x_nhwc(const void* x, int B, int H, int W, int C, void* y, void* stream) {
  if (!x || !y || (C % 8)) return set_error(VDB_ERR_INVALID, "upsample2x: null argument or C %% 8 != 0");
  const long long total = static_cast<long long>(B) * 4 * H * W * (C / 8);
  upsample2x_kernel<<<ew_blocks(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), B, H, W, C, reinterpret_cast<__nv_bfloat16*>(y));
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_clip_to_u8_hwc(const float* x, int n, int H, int W, void* y, void* stream) {
  if (!x || !y || n <= 0 || H <= 0 || W <= 0) return set_error(VDB_ERR_INVALID, "clip_to_u8_hwc: bad argument");
  clip_to_u8_hwc_kernel<<<ew_blocks(static_cast<long long>(n) * H * W * 3, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, n, H, W, reinterpret_cast<uint8_t*>(y));
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_resample_h_u8(const void* x, int n, int H, int Win, int Wout, const int* bounds, const int* kk, int ksize, void* y,
                      void* stream) {
  if (!x || !y || !bounds || !kk || n <= 0 || H <= 0 || Win <= 0 || Wout <= 0 || ksize <= 0)
    return set_error(VDB_ERR_INVALID, "resample_h_u8: bad argument");
  resample_h_u8_kernel<<<ew_blocks(static_cast<long long>(n) * H * Wout * 3, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint8_t*>(x), n, H, Win, Wout, bounds, kk, ksize, reinterpret_cast<uint8_t*>(y));
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_resample_v_crop_norm(const void* x, int n, int Hin, int W, const int* bounds, const int* kk, int ksize, int top,
                             int left, int S, const float* mean3, const float* std3, float* y, void* stream) {
  if (!x || !y || !mean3 || !std3 || n <= 0 || Hin <= 0 || W <= 0 || S <= 0 || top < 0 || left < 0 || left + S > W ||
      (ksize > 0 && (!bounds || !kk)) || (ksize == 0 && top + S > Hin))
    return set_error(VDB_ERR_INVALID, "resample_v_crop_norm: bad argument");
  resample_v_crop_norm_kernel<<<ew_blocks(static_cast<long long>(n) * 3 * S * S, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint8_t*>(x), n, Hin, W, bounds, kk, ksize, top, left, S, mean3[0], mean3[1], mean3[2], std3[0],
      std3[1], std3[2], y);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_im2col3x3_small(const float* x, int B, int H, int W, int Cin, int Kpad, float in_scale, float in_shift,
                        void* y, void* stream) {
  if (!x || !y || 9 * Cin > Kpad || (Kpad % 8)) return set_error(VDB_ERR_INVALID, "im2col3x3_small: bad argument");
  const long long total = static_cast<long long>(B) * H * W * (Kpad / 8);
  im2col3x3_small_kernel<<<ew_blocks(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, B, H, W, Cin, Kpad, in_scale, in_shift, reinterpret_cast<__nv_bfloat16*>(y));
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_permute_f32(const float* x, int B, int C, long long HW, int to_nhwc, float mul, float add, int clamp01,
                    float* y, void* stream) {
  if (!x || !y) return set_error(VDB_ERR_INVALID, "permute_f32: null argument");
  const long long total = static_cast<long long>(B) * C * HW;
  permute_f32_kernel<<<ew_blocks(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, B, C, static_cast<int>(HW), to_nhwc, mul, add, clamp01, y);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_pointwise_small(const float* x, long long npix, int Cin, int Cout, const float* Wm, const float* bias,
                        float pre_mul, float* y, void* stream) {
  if (!x || !Wm || !y || Cin <= 0 || Cin > 8 || Cout <= 0 || Cout > 8)
    return set_error(VDB_ERR_INVALID, "pointwise_small: need 1 <= Cin, Cout <= 8");
  pointwise_small_kernel<<<ew_blocks(npix, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, npix, Cin, Cout, Wm,
                                                                                                  bias, pre_mul, y);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_gaussian_sample(const float* moments, const float* noise, int C, long long npix, float post_mul, float* z,
                        void* stream) {
  if (!moments || !z || C <= 0 || npix <= 0) return set_error(VDB_ERR_INVALID, "gaussian_sample: bad argument");
  gaussian_sample_kernel<<<ew_blocks(npix * C, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      moments, noise, C, npix, post_mul, z);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_cast_f32_bf16(const float* x, void* y, long long n, void* stream) {
  if (!x || !y) return set_error(VDB_ERR_INVALID, "cast: null argument");
  cast_f32_bf16_kernel<<<ew_blocks(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, reinterpret_cast<__nv_bfloat16*>(y), n);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}
int vdb_cast_bf16_f32(const void* x, float* y, long long n, void* stream) {
  if (!x || !y) return set_error(VDB_ERR_INVALID, "cast: null argument");
  cast_bf16_f32_kernel<<<ew_blocks(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), y, n);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_timestep_embedding(const long long* ts, const int* step_idx, int B, int dim, float neg_log_period, float* out,
                           void* stream) {
  if (!ts || !out || B <= 0 || dim <= 1) return set_error(VDB_ERR_INVALID, "timestep_embedding: bad argument");
  timestep_embedding_kernel<<<ew_blocks(static_cast<long long>(B) * (dim / 2), 128), 128, 0,
                              reinterpret_cast<cudaStream_t>(stream)>>>(ts, step_idx, B, dim, neg_log_period, out);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
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
  linear_small_kernel<<<blocks, 256, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, M, K, reinterpret_cast<const __nv_bfloat16*>(Wt), N, bias, act_in, act_out, out);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_clip_text_embed(const long long* tokens, const float* tok_emb, const float* pos_emb, int B, int L, int Lp, int C,
                        void* x, void* stream) {
  if (!tokens || !tok_emb || !pos_emb || !x || Lp < L) return set_error(VDB_ERR_INVALID, "clip_text_embed: bad argument");
  clip_text_embed_kernel<<<ew_blocks(static_cast<long long>(B) * Lp * C, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      tokens, tok_emb, pos_emb, B, L, Lp, C, reinterpret_cast<__nv_bfloat16*>(x));
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_patchify(const float* pixels, int B, int Cin, int HW, int P, int Kpad, void* y, void* stream) {
  if (!pixels || !y || HW % P || Cin * P * P > Kpad || (Kpad % 8)) return set_error(VDB_ERR_INVALID, "patchify: bad argument");
  const int G = HW / P;
  patchify_kernel<<<ew_blocks(static_cast<long long>(B) * G * G * Kpad, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      pixels, B, Cin, HW, P, Kpad, reinterpret_cast<__nv_bfloat16*>(y));
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_vit_assemble(const void* patches, const float* cls, const float* pos, const float* tok_scale, int B, int L, int Lp,
                     int C, void* x, void* stream) {
  if (!patches || !cls || !pos || !x || Lp < L) return set_error(VDB_ERR_INVALID, "vit_assemble: bad argument");
  vit_assemble_kernel<<<ew_blocks(static_cast<long long>(B) * Lp * C, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(patches), cls, pos, tok_scale, B, L, Lp, C, reinterpret_cast<__nv_bfloat16*>(x));
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_scale_by_row_norm(const void* z, const int* idx, const float* row_scale, int B, int L, int Lp, int C, float* out,
                          void* stream) {
  if (!z || !out || B <= 0 || Lp < L) return set_error(VDB_ERR_INVALID, "scale_by_row_norm: bad argument");
  scale_by_row_norm_kernel<<<B, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(z), idx, row_scale, L, Lp, C, out);
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

int vdb_softmax_rows(const void* x, long long rows, int n, long long ld, float scale, void* y, void* stream) {
  if (!x || !y || rows <= 0 || n <= 0) return set_error(VDB_ERR_INVALID, "softmax_rows: bad argument");
  const int blocks = static_cast<int>(std::min<long long>(rows, num_sms() * 8LL));
  softmax_rows_kernel<<<blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), rows, n, ld, scale, reinterpret_cast<__nv_bfloat16*>(y));
  VDB_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return VDB_OK;
}

}  // extern "C"
