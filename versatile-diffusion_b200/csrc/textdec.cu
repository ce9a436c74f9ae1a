// vdb200 — the Optimus GPT-2 text decoder, one token step at a time (sm_90a).
//
// The decoder (12 layers, width 768, 12 heads of 64, vocabulary 50260) runs a handful of rows (one per text latent, <= 16)
// through ~247 MB of bf16 weights per token: every kernel here is bound by weight bandwidth or by launch latency, none is
// tensor-core sized.  A token step is
//   embed -> 12 x [ln_1+c_attn, attention over the KV cache, attn.c_proj(+resid), ln_2+c_fc+gelu, mlp.c_proj(+resid)]
//         -> ln_f+lm_head [-> repetition penalty / n-gram bans] -> sampler -> step += 1
// and reads the step index from a device counter, so one captured CUDA graph serves every step.
#include <curand_philox4x32_x.h>

#include "common.cuh"
#include "host_util.h"

namespace vdb {

namespace {

constexpr int kGvWarps = 8;                   // warps per GEMV CTA
constexpr int kGvMaxRows = 16;                // the mma M dimension: rows beyond R are zero in shared memory
constexpr int kGvMaxK = 3072;                 // mlp.c_proj's input width
constexpr int kActGeluTanh = 5;               // VDB_ACT_GELU_TANH
constexpr int kActTanh = 6;                   // VDB_ACT_TANH (the BERT encoder's pooler)
constexpr int kHeadDim = 64;
constexpr int kSampleThreads = 1024;

VDB_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;   // xor butterfly: every lane ends with the same bits (each pairwise sum is formed in both orders)
}

VDB_DEVINL void mma_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

VDB_DEVINL uint4 ldg_stream(const void* p) {   // weights are read once per token: do not keep them in L1
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

VDB_DEVINL uint4 lds_u4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}

// GPT-2's gelu (optimus_gpt2.py:99-100): the tanh approximation, not the erf form of VDB_ACT_GELU
VDB_DEVINL float gelu_tanh(float x) {
  return 0.5f * x * (1.0f + tanhf(0.7978845608028654f * (x + 0.044715f * x * x * x)));
}

// ---------------------------------------------------------------------------------------------------------------------------
// Weight-streaming GEMV:  out[r, n] (=|+=) act( LN?(x)[r, :] . W[n, :] + bias[n] ),  r < R <= 16, W bf16 [N, K] row-major.
//
// Prologue: each CTA normalises (optional LayerNorm, fp32 statistics, two passes) the fp32 rows of x into a bf16 [16, K]
// operand in shared memory; rows >= R are zero.  The row stride is padded to 64 mod 128 bytes so the 16-byte loads of one
// quarter-warp (two rows x four lanes) hit distinct banks.
// Main loop: a warp owns 8 output columns (one m16n8k16 tile, N = 8) and a 1/ks share of K.  Lane (g = lane/4, t = lane%4)
// streams 16 contiguous bytes W[n0+g, kb + 8t .. +8) per 32-wide k chunk, and the A fragment is loaded from the same
// physical k positions: the mma's logical k order is permuted identically on both operands (a dot product does not care),
// so each chunk is one 16-byte global load, two 16-byte shared loads and two mma per lane, with no shuffles.
// Epilogue: ks == 1 straight from the accumulator fragment; ks > 1 sums the ks partials in shared memory in a fixed order.
// Deterministic (no atomics); every weight byte is read once per call.
// ---------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kGvWarps * 32, 2)
textdec_gemv_kernel(const float* __restrict__ x, int R, int K, long long ldx, const float* __restrict__ ln_g,
                    const float* __restrict__ ln_b, float ln_eps, const __nv_bfloat16* __restrict__ W, int N, long long ldw,
                    const float* __restrict__ bias, int act, int accumulate, float* __restrict__ out, long long ldo, int ks,
                    int ldxs) {
  extern __shared__ __align__(16) unsigned char smem[];
  __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(smem);
  float* red = reinterpret_cast<float*>(smem + static_cast<size_t>(kGvMaxRows) * ldxs * 2);   // [warps][16 rows][8 cols]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  for (int r = warp; r < kGvMaxRows; r += kGvWarps) {
    __nv_bfloat16* dst = xs + static_cast<size_t>(r) * ldxs;
    if (r >= R) {
      for (int k = lane; k < K; k += 32) dst[k] = __float2bfloat16(0.0f);
      continue;
    }
    const float* src = x + static_cast<size_t>(r) * ldx;
    if (ln_g) {
      float s = 0.0f;
      for (int k = lane; k < K; k += 32) s += src[k];
      const float mean = warp_sum(s) / K;
      float v = 0.0f;
      for (int k = lane; k < K; k += 32) { const float d = src[k] - mean; v += d * d; }
      const float rstd = rsqrtf(warp_sum(v) / K + ln_eps);
      for (int k = lane; k < K; k += 32) dst[k] = __float2bfloat16((src[k] - mean) * rstd * ln_g[k] + ln_b[k]);
    } else {
      for (int k = lane; k < K; k += 32) dst[k] = __float2bfloat16(src[k]);
    }
  }
  __syncthreads();

  const int g = lane >> 2, t = lane & 3;
  const int slots = kGvWarps / ks, slot = warp / ks, kp = warp % ks;
  const int nchunks = K / 32, per = nchunks / ks, c0 = kp * per;
  const int tiles = (N + 7) / 8;
  const bool hi = R > 8;
  const uint32_t xs_base = static_cast<uint32_t>(__cvta_generic_to_shared(xs));
  const uint32_t a_lo = xs_base + (g * ldxs + t * 8) * 2, a_hi = a_lo + 8 * ldxs * 2;

  for (int base = blockIdx.x * slots; base < tiles; base += gridDim.x * slots) {
    const int tile = base + slot;
    const int n0 = tile * 8;
    const int nrow = min(n0 + g, N - 1);                                 // clamp: the tail tile's spare rows load a valid row
    const __nv_bfloat16* wrow = W + static_cast<size_t>(nrow) * ldw + t * 8;
    float c[4] = {0.f, 0.f, 0.f, 0.f};
    if (tile < tiles) {
      constexpr int U = 8;
      for (int cc = c0; cc < c0 + per; cc += U) {
        uint4 w[U];
#pragma unroll
        for (int u = 0; u < U; ++u)
          if (cc + u < c0 + per) w[u] = ldg_stream(wrow + (cc + u) * 32);
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (cc + u < c0 + per) {
            const uint32_t off = (cc + u) * 64;
            const uint4 xl = lds_u4(a_lo + off);
            const uint4 xh = hi ? lds_u4(a_hi + off) : make_uint4(0u, 0u, 0u, 0u);
            mma_16816(c, xl.x, xh.x, xl.y, xh.y, w[u].x, w[u].y);
            mma_16816(c, xl.z, xh.z, xl.w, xh.w, w[u].z, w[u].w);
          }
        }
      }
    }
    // fragment: c0,c1 = (row g, cols n0 + 2t, +1); c2,c3 = (row g + 8, same cols)
    auto epi = [&](int r, int n, float v) {
      if (r >= R || n >= N) return;
      if (bias) v += bias[n];
      if (act == kActGeluTanh) v = gelu_tanh(v);
      else if (act == kActTanh) v = tanhf(v);
      float* o = out + static_cast<size_t>(r) * ldo + n;
      *o = accumulate ? *o + v : v;
    };
    if (ks == 1) {
      if (tile < tiles) {
        epi(g, n0 + 2 * t, c[0]); epi(g, n0 + 2 * t + 1, c[1]);
        epi(g + 8, n0 + 2 * t, c[2]); epi(g + 8, n0 + 2 * t + 1, c[3]);
      }
    } else {
      float* rw = red + warp * 128;
      rw[g * 8 + 2 * t] = c[0]; rw[g * 8 + 2 * t + 1] = c[1];
      rw[(g + 8) * 8 + 2 * t] = c[2]; rw[(g + 8) * 8 + 2 * t + 1] = c[3];
      __syncthreads();
      for (int i = threadIdx.x; i < slots * 128; i += blockDim.x) {
        const int sl = i >> 7, e = i & 127, tl = base + sl;
        if (tl >= tiles) continue;
        float v = 0.0f;
        for (int p = 0; p < ks; ++p) v += red[(sl * ks + p) * 128 + e];
        epi(e >> 3, tl * 8 + (e & 7), v);
      }
      __syncthreads();
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Single-query attention over the KV cache, one warp per (row, head), d_head 64 (two dims per lane).
// Position 0 is the layer's latent slice (key == value, raw: GPT2Model_XX.forward, optimus_gpt2.py:882-895); positions
// 1 .. s+1 are tokens 0 .. s, s = *step.  This step's k / v (from c_attn) are appended at cache slot s and used from registers.
// fp32 online softmax, scale 1/sqrt(64); the causal mask admits every cached position.
// kIndexed (beam search): cache slot j < s of row r is read from physical row src[r * T + j]; this step's k / v still go to row
// r, slot s.  src is the last parameter, so the kIndexed = false instantiation keeps the parameter layout it had without it.
// ---------------------------------------------------------------------------------------------------------------------------
template <bool kIndexed>
__global__ void textdec_attention_kernel(const float* __restrict__ qkv, long long ldq, const float* __restrict__ mem,
                                         long long ldm, float* __restrict__ kc, float* __restrict__ vc, int R, int H, int T,
                                         const int* __restrict__ step, float scale, float* __restrict__ out, long long ldo,
                                         const int* __restrict__ src) {
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= R * H) return;
  const int s = *step;
  if (s < 0 || s >= T) return;
  const int r = w / H, h = w % H, D = H * kHeadDim, d = 2 * lane;
  const float* row = qkv + static_cast<size_t>(r) * ldq + h * kHeadDim + d;
  const float2 q = make_float2(row[0], row[1]);
  const float2 kn = make_float2(row[D], row[D + 1]);
  const float2 vn = make_float2(row[2 * D], row[2 * D + 1]);
  float* kb = kc + static_cast<size_t>(r * H + h) * T * kHeadDim + d;
  float* vb = vc + static_cast<size_t>(r * H + h) * T * kHeadDim + d;
  kb[static_cast<size_t>(s) * kHeadDim] = kn.x; kb[static_cast<size_t>(s) * kHeadDim + 1] = kn.y;
  vb[static_cast<size_t>(s) * kHeadDim] = vn.x; vb[static_cast<size_t>(s) * kHeadDim + 1] = vn.y;
  const float* lm = mem + static_cast<size_t>(r) * ldm + h * kHeadDim + d;
  const float2 lat = make_float2(lm[0], lm[1]);

  float m = -INFINITY, l = 0.0f;
  float2 acc = make_float2(0.0f, 0.0f);
  for (int j = 0; j <= s + 1; ++j) {
    float2 kj, vj;
    if (j == 0) { kj = lat; vj = lat; }
    else if (j == s + 1) { kj = kn; vj = vn; }
    else if constexpr (kIndexed) {
      const int pr = src[static_cast<size_t>(r) * T + j - 1];
      const size_t o = (static_cast<size_t>(pr * H + h) * T + j - 1) * kHeadDim + d;
      kj = make_float2(kc[o], kc[o + 1]); vj = make_float2(vc[o], vc[o + 1]);
    } else {
      const size_t o = static_cast<size_t>(j - 1) * kHeadDim;
      kj = make_float2(kb[o], kb[o + 1]); vj = make_float2(vb[o], vb[o + 1]);
    }
    const float sc = warp_sum(q.x * kj.x + q.y * kj.y) * scale;
    const float mn = fmaxf(m, sc);
    const float corr = __expf(m - mn), p = __expf(sc - mn);
    l = l * corr + p;
    acc.x = acc.x * corr + p * vj.x;
    acc.y = acc.y * corr + p * vj.y;
    m = mn;
  }
  float* o = out + static_cast<size_t>(r) * ldo + h * kHeadDim + d;
  o[0] = acc.x / l; o[1] = acc.y / l;
}

// h[r, :] = wte[tokens[r, s]] + wpe[s + pos_offset] + emb[r, :]    (GPT2Model_XX.forward: inputs_embeds + position_embeds
// + linear_emb(z), optimus_gpt2.py:941-948, same fp32 order)
__global__ void textdec_embed_kernel(const int* __restrict__ tokens, int ldt, const int* __restrict__ step,
                                     const float* __restrict__ wte, int V, const float* __restrict__ wpe, int P, int pos_offset,
                                     const float* __restrict__ emb, int D, float* __restrict__ h) {
  const int r = blockIdx.x, s = *step;
  int tok = tokens[static_cast<size_t>(r) * ldt + s];
  tok = min(max(tok, 0), V - 1);
  const int pos = min(s + pos_offset, P - 1);
  for (int i = threadIdx.x; i < D; i += blockDim.x)
    h[static_cast<size_t>(r) * D + i] =
        (wte[static_cast<size_t>(tok) * D + i] + wpe[static_cast<size_t>(pos) * D + i]) + emb[static_cast<size_t>(r) * D + i];
}

// ---------------------------------------------------------------------------------------------------------------------------
// top-k / nucleus filter of the sampler (kFilter instantiation).  The row's scaled logits l are staged once in shared memory
// as order-preserving uint32 keys; both cuts are MSD radix selects over them, 8 bits per pass, with 256-bin histograms
// privatised per group of 4 warps.  top-k counts tokens; the nucleus weighs each survivor by its probability as a 64-bit
// fixed-point integer (exp(l - max) / Z scaled by 2^62, Z the survivors' fp64 sum in a fixed order): integer atomics are exact
// and order-free, so graph replays stay bitwise repeatable.
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int kFilterHists = 8;                 // privatised histograms (kSampleThreads / 32 warps share them 4 to 1)
constexpr int kFilterMaxV = 53248;              // staged keys (4 B each) + the histograms fit in the 227 KiB opt-in
constexpr size_t kFilterHistBytes = kFilterHists * 256 * sizeof(unsigned long long);
constexpr double kMassOne = 0x1.0p62;           // fixed-point unit of probability mass

VDB_DEVINL uint32_t order_key(float f) {         // a < b  <=>  order_key(a) < order_key(b)  (non-NaN)
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

VDB_DEVINL float key_value(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

VDB_DEVINL unsigned long long key_mass(uint32_t k, float mx, double scale) {
  return __double2ull_rn(static_cast<double>(expf(key_value(k) - mx)) * scale);
}

struct FilterShared {
  unsigned long long above;
  double red[32];
  int bin, found;
  int ties[32];
};

struct Selected {
  bool found;
  uint32_t key;
  unsigned long long above;
};

// The largest key v among the staged keys >= lo with W(>= v) > T, where W sums 1 per key (kMass false) or key_mass (kMass
// true) over the keys >= lo.  found is false when all of them together weigh <= T; else key = v and above = W(> v).
template <bool kMass>
VDB_DEVINL Selected radix_select(const uint32_t* keys, int V, uint32_t lo, unsigned long long T, float mx, double scale,
                                 unsigned long long* hist, FilterShared& sh) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  unsigned long long* mine = hist + (warp % kFilterHists) * 256;
  uint32_t prefix = 0;
  unsigned long long ab = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < kFilterHists * 256; i += blockDim.x) hist[i] = 0ull;
    __syncthreads();
    const uint32_t hi = shift == 24 ? 0u : 0xffffffffu << (shift + 8);
    for (int i = tid; i < V; i += blockDim.x) {
      const uint32_t k = keys[i];
      if (k >= lo && (k & hi) == prefix) atomicAdd(mine + ((k >> shift) & 255u), kMass ? key_mass(k, mx, scale) : 1ull);
    }
    __syncthreads();
    if (tid < 256) {
      unsigned long long t = hist[tid];
      for (int h = 1; h < kFilterHists; ++h) t += hist[h * 256 + tid];
      hist[tid] = t;
    }
    __syncthreads();
    if (warp == 0) {                               // lane L holds bins 255 - 8L - j, j < 8: the bins in descending order
      unsigned long long own = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) own += hist[255 - 8 * lane - j];
      unsigned long long inc = own;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long n = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += n;
      }
      const unsigned hit = __ballot_sync(0xffffffffu, ab + inc > T);
      if (lane == 0) sh.found = hit != 0u;
      if (hit && lane == __ffs(hit) - 1) {
        unsigned long long c = ab + inc - own;
        int b = 255 - 8 * lane;
        for (int j = 0; j < 8; ++j, --b) {
          if (c + hist[b] > T) break;
          c += hist[b];
        }
        sh.bin = b;
        sh.above = c;
      }
    }
    __syncthreads();
    if (!sh.found) return Selected{false, 0u, 0ull};   // only the first pass can miss: later ones refine a bin that crossed T
    prefix |= static_cast<uint32_t>(sh.bin) << shift;
    ab = sh.above;
  }
  return Selected{true, prefix, ab};
}

// ---------------------------------------------------------------------------------------------------------------------------
// Sampler, one CTA per row: token s+1 ~ softmax(logits / temperature) by inverse CDF of a uniform u in [0, 1).
// Each thread owns a contiguous slice of the vocabulary; exp(x - max) is summed in fp64 per slice, the slice sums are
// scanned across the block in a fixed order, and the thread whose [prefix, next prefix) holds u * total walks its slice.
// u: uniforms[r * ldu + s] when given, else the 53-bit Philox4x32-10 draw at counter (r, s) under key *seed.
// forced (teacher forcing) replaces the draw.  A finished row (done[r] != 0) is left untouched.  After writing token s+1:
// == eos ends the row; otherwise when s+1 == max_len - 2 the row gets eos at s+2 (optimus.py:682-688 overwrites the 30th
// token, so that last draw is skipped).  record (may be NULL) receives this step's raw logits at [s][r][:].
// kFilter: the same pick over the tokens the top-k / nucleus cuts keep (vdb_textdec_sample's top_k / top_p), removed tokens weigh 0.
// The kept set is every key > bound plus the first `cap` keys == bound in vocabulary order.
// ---------------------------------------------------------------------------------------------------------------------------
template <bool kFilter>
__global__ void __launch_bounds__(kSampleThreads, 1)   // one CTA per SM: without the 1, ptxas caps it at 32 registers and spills
textdec_sample_kernel(const float* __restrict__ logits, int R, int V, long long ldl, float temperature,
                      const unsigned long long* __restrict__ seed, const double* __restrict__ uniforms, int ldu,
                      const int* __restrict__ forced, int ldf, int* __restrict__ tokens, int ldt, int* __restrict__ done,
                      int* __restrict__ lengths, const int* __restrict__ step, int eos, int max_len, float* __restrict__ record,
                      int top_k, float top_p) {
  extern __shared__ __align__(16) unsigned char s_filter[];   // kFilter: histograms, then the V staged keys
  __shared__ float s_max[32];
  __shared__ double s_scan[32];
  __shared__ int s_tok, s_last;
  const int r = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int s = *step;
  const float* lr = logits + static_cast<size_t>(r) * ldl;
  if (record) {
    float* dst = record + (static_cast<size_t>(s) * R + r) * V;
    for (int i = tid; i < V; i += blockDim.x) dst[i] = lr[i];
  }
  if (done[r]) return;

  int tok;
  if (forced) {
    tok = forced[static_cast<size_t>(r) * ldf + s + 1];
  } else {
    const int per = (V + blockDim.x - 1) / blockDim.x;
    const int i0 = min(V, tid * per), i1 = min(V, i0 + per);
    unsigned long long* hist = reinterpret_cast<unsigned long long*>(s_filter);
    uint32_t* keys = reinterpret_cast<uint32_t*>(s_filter + kFilterHistBytes);
    float mx = -INFINITY;
    if constexpr (kFilter) {
      for (int i = tid; i < V; i += blockDim.x) {
        const float l = lr[i] / temperature;
        keys[i] = order_key(l);
        mx = fmaxf(mx, l);
      }
    } else {
      for (int i = i0; i < i1; ++i) mx = fmaxf(mx, lr[i] / temperature);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) s_max[warp] = mx;
    if (tid == 0) { s_tok = -1; s_last = -1; }
    __syncthreads();
    mx = s_max[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) mx = fmaxf(mx, s_max[i]);

    uint32_t bound = 0u;
    int cap = INT_MAX, rank0 = 0;
    if constexpr (kFilter) {
      __shared__ FilterShared sh;
      if (top_k > 0 && top_k < V)        // the k-th largest key: W(>= v) > k - 1 counted
        bound = radix_select<false>(keys, V, 0u, static_cast<unsigned long long>(top_k - 1), mx, 0.0, hist, sh).key;
      if (top_p > 0.0f && top_p < 1.0f) {
        double z = 0.0;                  // Z over the top-k survivors: per-thread strided sums, then a fixed tree
        for (int i = tid; i < V; i += blockDim.x)
          if (keys[i] >= bound) z += static_cast<double>(expf(key_value(keys[i]) - mx));
#pragma unroll
        for (int o = 16; o; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
        if (lane == 0) sh.red[warp] = z;
        __syncthreads();
        z = sh.red[0];
        for (int i = 1; i < (int)(blockDim.x >> 5); ++i) z += sh.red[i];
        const double scale = kMassOne / z;
        const unsigned long long P = __double2ull_rn(static_cast<double>(top_p) * kMassOne);
        // boundary b: the largest value whose survivors at or above it weigh > top_p.  Everything above b is kept; the ties
        // at b, taken in vocabulary order, each have exclusive mass above + t q, kept while that is <= top_p.
        const Selected b = radix_select<true>(keys, V, bound, P, mx, scale, hist, sh);
        if (b.found) {
          const unsigned long long q = key_mass(b.key, mx, scale), n = 1ull + (P - b.above) / q;
          bound = b.key;
          cap = n < static_cast<unsigned long long>(INT_MAX) ? static_cast<int>(n) : INT_MAX;
        }
      }
      if (cap != INT_MAX) {              // rank0: the ties at the bound in the slices before this thread's
        int t = 0;
        for (int i = i0; i < i1; ++i) t += keys[i] == bound;
        int inc = t;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int n = __shfl_up_sync(0xffffffffu, inc, o);
          if (lane >= o) inc += n;
        }
        if (lane == 31) sh.ties[warp] = inc;
        __syncthreads();
        int off = 0;
        for (int w = 0; w < warp; ++w) off += sh.ties[w];
        rank0 = off + inc - t;
      }
    }
    // exp(l - max) of token i, or 0 for a token the cuts remove; rank counts the ties at the bound met so far
    auto weight = [&](int i, int& rank) -> float {
      if constexpr (kFilter) {
        const uint32_t k = keys[i];
        if (k < bound || (k == bound && rank++ >= cap)) return 0.0f;
        return expf(key_value(k) - mx);
      } else {
        return expf(lr[i] / temperature - mx);
      }
    };

    double sum = 0.0;
    int last = -1, rank = rank0;
    for (int i = i0; i < i1; ++i) {
      const float e = weight(i, rank);
      sum += static_cast<double>(e);
      if (e > 0.0f) last = i;
    }
    double inc = sum;   // inclusive scan within the warp, then across warps
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double n = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += n;
    }
    if (lane == 31) s_scan[warp] = inc;
    atomicMax(&s_last, last);
    __syncthreads();
    if (warp == 0) {
      double v = lane < (int)(blockDim.x >> 5) ? s_scan[lane] : 0.0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const double n = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += n;
      }
      s_scan[lane] = v;
    }
    __syncthreads();
    const double off = warp ? s_scan[warp - 1] : 0.0;
    const double hi = inc + off;                                          // == the next thread's prefix
    const double lo = __shfl_up_sync(0xffffffffu, inc, 1);
    const double pre = (lane ? lo : 0.0) + off;
    const double total = s_scan[31];

    double u;
    if (uniforms) {
      u = uniforms[static_cast<size_t>(r) * ldu + s];
    } else {
      const unsigned long long k = *seed;
      const uint4 x = curand_Philox4x32_10(make_uint4(static_cast<unsigned>(r), static_cast<unsigned>(s), 0x74657874u, 0u),
                                           make_uint2(static_cast<unsigned>(k), static_cast<unsigned>(k >> 32)));
      u = static_cast<double>((static_cast<unsigned long long>(x.x) << 21) | (x.y >> 11)) * 0x1.0p-53;
    }
    const double target = u * total;
    if (target >= pre && target < hi) {
      double c = pre;
      int pick = last;
      rank = rank0;
      for (int i = i0; i < i1; ++i) {
        c += static_cast<double>(weight(i, rank));       // a removed token adds 0: it can never be the pick
        if (target < c) { pick = i; break; }
      }
      s_tok = pick;
    }
    __syncthreads();
    tok = s_tok >= 0 ? s_tok : s_last;
  }
  if (tid == 0) {
    int* tr = tokens + static_cast<size_t>(r) * ldt;
    tr[s + 1] = tok;
    if (tok == eos) {
      done[r] = 1; lengths[r] = s + 2;
    } else if (s + 1 >= max_len - 2) {
      tr[s + 2] = eos; done[r] = 1; lengths[r] = s + 3;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Beam search step (vdb_textdec_beam_step), two launches.  Row r = latent * K + beam.
// (a) textdec_beam_topk_kernel, one CTA per row: the fp64 log-softmax logp(v) = l_v - lse, l_v = logit_v / temperature,
//     lse = max + log(sum exp(l - max)) (per-thread slice sums, then a fixed tree), and the row's K best tokens: the filter's
//     radix select with top_k = K over the raw logits' keys (dividing by temperature > 0 keeps their order), every key > bound
//     plus the first K - #(> bound) keys == bound in vocabulary order.  Writes the K (token, logp) candidates in vocabulary
//     order.  A finished row only records its logits.
// (b) textdec_beam_select_kernel, one CTA per latent: candidates are (parent b, token v, S_b + logp_b(v)) for each live beam's
//     K tokens and (b, -1, S_b) for each finished beam; rank = the number of candidates that beat it (higher score, then lower
//     parent, then lower token): at most K x K of them, so the O(n^2) count is cheap and exact.  Candidate of rank j becomes
//     beam j: its token and src rows are staged through shared memory from the parent's.
// No floating-point atomics: replays are bitwise repeatable.
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int kBeamMax = 16;
constexpr int kSelectThreads = 256;
constexpr int kStageCols = 64;                    // token / src columns staged per pass of the permutation

__global__ void __launch_bounds__(kSampleThreads, 1)
textdec_beam_topk_kernel(const float* __restrict__ logits, int R, int V, long long ldl, float temperature, int K,
                         const int* __restrict__ done, const int* __restrict__ step, int* __restrict__ cand_tok,
                         double* __restrict__ cand_logp, float* __restrict__ record) {
  extern __shared__ __align__(16) unsigned char s_filter[];   // histograms, then the V staged keys
  __shared__ FilterShared sh;
  __shared__ float s_max[32];
  __shared__ int s_n, s_tok[kBeamMax];
  const int r = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nw = blockDim.x >> 5;
  const int s = *step;
  const float* lr = logits + static_cast<size_t>(r) * ldl;
  if (record) {
    float* dst = record + (static_cast<size_t>(s) * R + r) * V;
    for (int i = tid; i < V; i += blockDim.x) dst[i] = lr[i];
  }
  if (done[r]) return;
  unsigned long long* hist = reinterpret_cast<unsigned long long*>(s_filter);
  uint32_t* keys = reinterpret_cast<uint32_t*>(s_filter + kFilterHistBytes);
  float mx = -INFINITY;
  for (int i = tid; i < V; i += blockDim.x) {
    const float l = lr[i];
    keys[i] = order_key(l == 0.0f ? 0.0f : l);    // -0 and +0 are one value: one key
    mx = fmaxf(mx, l);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) s_max[warp] = mx;
  if (tid == 0) s_n = 0;
  __syncthreads();
  mx = s_max[0];
  for (int i = 1; i < nw; ++i) mx = fmaxf(mx, s_max[i]);

  const double t = static_cast<double>(temperature), m = static_cast<double>(mx) / t;
  const int per = (V + blockDim.x - 1) / blockDim.x;
  const int i0 = min(V, tid * per), i1 = min(V, i0 + per);
  double z = 0.0;
  for (int i = i0; i < i1; ++i) z += exp(static_cast<double>(key_value(keys[i])) / t - m);
#pragma unroll
  for (int o = 16; o; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
  if (lane == 0) sh.red[warp] = z;
  __syncthreads();
  z = sh.red[0];
  for (int i = 1; i < nw; ++i) z += sh.red[i];
  const double lse = m + log(z);

  // the K-th largest key; K <= V, so it always exists
  const Selected b = radix_select<false>(keys, V, 0u, static_cast<unsigned long long>(K - 1), 0.0f, 0.0, hist, sh);
  const uint32_t bound = b.key;
  const int cap = K - static_cast<int>(b.above);
  int nt = 0;                                       // rank0: the ties at the bound in the slices before this thread's
  for (int i = i0; i < i1; ++i) nt += keys[i] == bound;
  int inc = nt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += n;
  }
  if (lane == 31) sh.ties[warp] = inc;
  __syncthreads();
  int rank = inc - nt;
  for (int w = 0; w < warp; ++w) rank += sh.ties[w];
  for (int i = i0; i < i1; ++i) {
    const uint32_t k = keys[i];
    if (k > bound || (k == bound && rank++ < cap)) s_tok[atomicAdd(&s_n, 1)] = i;
  }
  __syncthreads();
  if (tid == 0) {                                   // exactly K picks; put them in vocabulary order
    for (int i = 1; i < K; ++i)
      for (int j = i; j > 0 && s_tok[j - 1] > s_tok[j]; --j) { const int x = s_tok[j]; s_tok[j] = s_tok[j - 1]; s_tok[j - 1] = x; }
  }
  __syncthreads();
  if (tid < K) {
    const int v = s_tok[tid];
    cand_tok[r * K + tid] = v;
    cand_logp[r * K + tid] = static_cast<double>(lr[v]) / t - lse;
  }
}

__global__ void __launch_bounds__(kSelectThreads)
textdec_beam_select_kernel(int R, int K, const int* __restrict__ cand_tok, const double* __restrict__ cand_logp,
                           int* __restrict__ tokens, int ldt, int* __restrict__ src, int lds, double* __restrict__ scores,
                           int* __restrict__ done, int* __restrict__ lengths, const int* __restrict__ step, int eos, int max_len,
                           double* __restrict__ trace) {
  __shared__ double c_score[kBeamMax * kBeamMax];
  __shared__ int c_tok[kBeamMax * kBeamMax];       // -1: a finished beam carried over as itself; -2: no candidate
  __shared__ double b_score[kBeamMax];
  __shared__ int b_done[kBeamMax], b_len[kBeamMax], sel[kBeamMax];
  __shared__ int stage[kBeamMax * kStageCols];
  const int tid = threadIdx.x, row0 = blockIdx.x * K, nc = K * K;
  const int s = *step;
  if (s < 0 || s >= lds || s + 1 >= ldt) return;
  if (tid < K) {
    b_done[tid] = done[row0 + tid]; b_len[tid] = lengths[row0 + tid]; b_score[tid] = scores[row0 + tid];
  }
  __syncthreads();
  for (int i = tid; i < nc; i += blockDim.x) {
    const int p = i / K, j = i % K;
    if (b_done[p]) {
      c_tok[i] = j == 0 ? -1 : -2;
      c_score[i] = b_score[p];
    } else {
      c_tok[i] = cand_tok[(row0 + p) * K + j];
      c_score[i] = b_score[p] + cand_logp[(row0 + p) * K + j];
    }
  }
  __syncthreads();
  for (int i = tid; i < nc; i += blockDim.x) {
    const int t = c_tok[i], p = i / K;
    if (t == -2) continue;
    const double sc = c_score[i];
    int rank = 0;
    for (int c = 0; c < nc; ++c) {
      const int tc = c_tok[c], pc = c / K;
      if (tc == -2) continue;
      rank += c_score[c] > sc || (c_score[c] == sc && (pc < p || (pc == p && tc < t)));
    }
    if (rank < K) sel[rank] = i;
  }
  __syncthreads();
  // beam j <- its parent's tokens 0 .. s+1 and src slots 0 .. s-1; src slot s <- the parent's row (its k / v of this step)
  for (int pass = 0; pass < 2; ++pass) {
    int* base = pass ? src : tokens;
    const int ld = pass ? lds : ldt, ncol = pass ? s : s + 2;
    for (int c0 = 0; c0 < ncol; c0 += kStageCols) {
      const int w = min(kStageCols, ncol - c0);
      for (int i = tid; i < K * w; i += blockDim.x) {
        const int j = i / w, c = c0 + i % w;
        stage[i] = base[static_cast<size_t>(row0 + sel[j] / K) * ld + c];
      }
      __syncthreads();
      for (int i = tid; i < K * w; i += blockDim.x) {
        const int j = i / w, c = c0 + i % w;
        base[static_cast<size_t>(row0 + j) * ld + c] = stage[i];
      }
      __syncthreads();
    }
  }
  if (tid < K) {
    const int i = sel[tid], p = i / K, t = c_tok[i], row = row0 + tid;
    int* tr = tokens + static_cast<size_t>(row) * ldt;
    src[static_cast<size_t>(row) * lds + s] = row0 + p;
    int d = 1, len = b_len[p];
    if (t >= 0) {                                   // a live parent's child
      tr[s + 1] = t;
      if (t == eos) {
        len = s + 2;
      } else if (s + 1 >= max_len - 2) {           // the forced, unscored <eos>
        if (s + 2 < ldt) tr[s + 2] = eos;
        len = s + 3;
      } else {
        d = 0;
      }
    }
    scores[row] = c_score[i]; done[row] = d; lengths[row] = len;
    if (trace) {
      double* tp = trace + (static_cast<size_t>(s) * R + row) * 3;
      tp[0] = p; tp[1] = t; tp[2] = c_score[i];
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Repetition penalty and no-repeat n-gram bans (vdb_textdec_repetition), one CTA per row, editing the row's logits in place
// before the sampler or the beam step reads them.  h = tokens[r, 0 .. s], s = *step.  Thread j takes history position j:
//   penalty pass: the first occurrence of each id in [0, V) scales its logit once (later occurrences of the id skip it);
//   ban pass (after a barrier, so a ban lands on the penalised value): position j <= s - n + 1 whose n - 1 tokens equal the
//   last n - 1 tokens of h sets logit h[j + n - 1] to -inf.  Two positions may ban one id: they write the same value.
// Reads the s + 1 history tokens only and touches at most 2 (s + 1) logits of the row, never the whole vocabulary.
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int kRepThreads = 32;                   // one warp: the history of a decode is at most 32 tokens

__global__ void __launch_bounds__(kRepThreads)
textdec_repetition_kernel(float* __restrict__ logits, int V, long long ldl, const int* __restrict__ tokens, int ldt,
                          const int* __restrict__ done, const int* __restrict__ step, float penalty, int ngram) {
  const int r = blockIdx.x, s = *step;
  if (s < 0 || s + 1 >= ldt || done[r]) return;
  float* lr = logits + static_cast<size_t>(r) * ldl;
  const int* h = tokens + static_cast<size_t>(r) * ldt;
  if (penalty != 1.0f) {
    for (int j = threadIdx.x; j <= s; j += blockDim.x) {
      const int v = h[j];
      if (v < 0 || v >= V) continue;
      bool first = true;
      for (int k = 0; k < j && first; ++k) first = h[k] != v;
      if (first) {
        const float l = lr[v];
        lr[v] = l < 0.0f ? __fmul_rn(l, penalty) : __fdiv_rn(l, penalty);
      }
    }
  }
  __syncthreads();
  if (ngram > 0) {
    const int tail = s - ngram + 2;               // h[tail .. s]: the last n - 1 tokens
    for (int j = threadIdx.x; j <= s - ngram + 1; j += blockDim.x) {
      bool match = true;
      for (int k = 0; k < ngram - 1 && match; ++k) match = h[j + k] == h[tail + k];
      const int v = h[j + ngram - 1];
      if (match && v >= 0 && v < V) lr[v] = -INFINITY;
    }
  }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" {

int vdb_textdec_gemv(const float* x, int R, long long K, long long ldx, const float* ln_gamma, const float* ln_beta,
                     float ln_eps, const void* W, long long N, long long ldw, const float* bias, int act, int accumulate,
                     float* out, long long ldo, void* stream) {
  if (!x || !W || !out) return set_error(VDB_ERR_INVALID, "textdec_gemv: null x / W / out");
  if (R < 1 || R > kGvMaxRows) return set_error(VDB_ERR_INVALID, "textdec_gemv: need 1 <= R <= %d rows, got %d", kGvMaxRows, R);
  if (K < 32 || K > kGvMaxK || K % 32) return set_error(VDB_ERR_INVALID, "textdec_gemv: need K %% 32 == 0 and 32 <= K <= %d, got %lld", kGvMaxK, K);
  if (N < 1 || N > (1LL << 30)) return set_error(VDB_ERR_INVALID, "textdec_gemv: bad N %lld", N);
  if (ldx < K || ldw < K || ldo < N) return set_error(VDB_ERR_INVALID, "textdec_gemv: leading dimensions smaller than the rows");
  if (!aligned16(W) || ldw % 8) return set_error(VDB_ERR_INVALID, "textdec_gemv: W must be 16-byte aligned with ldw %% 8 == 0");
  if (!ln_gamma != !ln_beta) return set_error(VDB_ERR_INVALID, "textdec_gemv: LayerNorm needs both gamma and beta");
  if (act != 0 && act != kActGeluTanh && act != kActTanh)
    return set_error(VDB_ERR_INVALID, "textdec_gemv: act must be VDB_ACT_NONE, VDB_ACT_GELU_TANH or VDB_ACT_TANH");
  if (static_cast<const void*>(x) == static_cast<const void*>(out)) return set_error(VDB_ERR_INVALID, "textdec_gemv: x must not alias out");
  const int k = static_cast<int>(K), n = static_cast<int>(N);
  const int ldxs = k + (k % 64 == 0 ? 32 : 0);   // row stride = 64 mod 128 bytes
  const size_t smem = static_cast<size_t>(kGvMaxRows) * ldxs * 2 + kGvWarps * 128 * sizeof(float);
  static bool configured = false;
  if (!configured) {
    const size_t most = static_cast<size_t>(kGvMaxRows) * (kGvMaxK + 32) * 2 + kGvWarps * 128 * sizeof(float);
    VDB_CUDA_CHECK(cudaFuncSetAttribute(textdec_gemv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(most)));
    configured = true;
  }
  // split K over up to 8 warps until every warp slot of the GPU (2 CTAs x 8 warps per SM) has work
  const int tiles = (n + 7) / 8, want = num_sms() * 2 * kGvWarps, chunks = k / 32;
  int ks = 1;
  while (ks < kGvWarps && static_cast<long long>(tiles) * ks < want && chunks % (ks * 2) == 0) ks *= 2;
  const int slots = kGvWarps / ks;
  const int blocks = std::min((tiles + slots - 1) / slots, num_sms() * 2);
  return launch(textdec_gemv_kernel, blocks, kGvWarps * 32, smem, stream, x, R, k, ldx, ln_gamma, ln_beta, ln_eps,
                reinterpret_cast<const __nv_bfloat16*>(W), n, ldw, bias, act, accumulate, out, ldo, ks, ldxs);
}

int vdb_textdec_attention(const float* qkv, long long ldq, const float* mem, long long ldm, float* kcache, float* vcache,
                          const int* src, int R, int H, int T, const int* step, float scale, float* out, long long ldo, void* stream) {
  if (!qkv || !mem || !kcache || !vcache || !step || !out) return set_error(VDB_ERR_INVALID, "textdec_attention: null pointer");
  if (R < 1 || R > kGvMaxRows || H < 1 || H > 64 || T < 1 || T > 1024)
    return set_error(VDB_ERR_INVALID, "textdec_attention: need 1 <= R <= 16, 1 <= H <= 64, 1 <= T <= 1024");
  const long long D = static_cast<long long>(H) * kHeadDim;
  if (ldq < 3 * D || ldm < D || ldo < D) return set_error(VDB_ERR_INVALID, "textdec_attention: leading dimensions smaller than the rows");
  if ((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(mem) | reinterpret_cast<uintptr_t>(out) |
       reinterpret_cast<uintptr_t>(kcache) | reinterpret_cast<uintptr_t>(vcache) | reinterpret_cast<uintptr_t>(src)) & 3)
    return set_error(VDB_ERR_INVALID, "textdec_attention: buffers must be 4-byte aligned");
  const int warps = R * H;
  return launch(src == nullptr ? textdec_attention_kernel<false> : textdec_attention_kernel<true>, (warps + 3) / 4, 128, 0, stream,
                qkv, ldq, mem, ldm, kcache, vcache, R, H, T, step, scale, out, ldo, src);
}

int vdb_textdec_embed(const int* tokens, int ldt, const int* step, const float* wte, int V, const float* wpe, int P, int pos_offset,
                      const float* emb, int R, int D, float* h, void* stream) {
  if (!tokens || !step || !wte || !wpe || !emb || !h) return set_error(VDB_ERR_INVALID, "textdec_embed: null pointer");
  if (R < 1 || R > kGvMaxRows || D < 1 || V < 1 || P < 1 || ldt < 1 || pos_offset < 0)
    return set_error(VDB_ERR_INVALID, "textdec_embed: need 1 <= R <= 16 and positive sizes");
  return launch(textdec_embed_kernel, R, 256, 0, stream, tokens, ldt, step, wte, V, wpe, P, pos_offset, emb, D, h);
}

int vdb_textdec_sample(const float* logits, int R, int V, long long ldl, float temperature, int top_k, float top_p,
                       const unsigned long long* seed, const double* uniforms, int ldu, const int* forced, int ldf, int* tokens, int ldt,
                       int* done, int* lengths, const int* step, int eos, int max_len, float* record, void* stream) {
  if (top_k < 0) return set_error(VDB_ERR_INVALID, "textdec_sample: top_k must be >= 0, got %d", top_k);
  if (!(top_p >= 0.0f && top_p <= 1.0f))
    return set_error(VDB_ERR_INVALID, "textdec_sample: top_p must be in [0, 1], got %g", static_cast<double>(top_p));
  if (!logits || !tokens || !done || !lengths || !step) return set_error(VDB_ERR_INVALID, "textdec_sample: null pointer");
  if (!forced && !uniforms && !seed) return set_error(VDB_ERR_INVALID, "textdec_sample: need a seed, uniforms or forced tokens");
  if (R < 1 || R > kGvMaxRows || V < 1 || ldl < V) return set_error(VDB_ERR_INVALID, "textdec_sample: need 1 <= R <= 16, ldl >= V >= 1");
  if (!(temperature > 0.0f)) return set_error(VDB_ERR_INVALID, "textdec_sample: temperature must be > 0");
  if (ldt < 2 || max_len < 2 || (uniforms && ldu < 1) || (forced && ldf < 2))
    return set_error(VDB_ERR_INVALID, "textdec_sample: bad token / uniform row strides");
  if ((reinterpret_cast<uintptr_t>(seed) & 7) || (reinterpret_cast<uintptr_t>(uniforms) & 7))
    return set_error(VDB_ERR_INVALID, "textdec_sample: seed / uniforms must be 8-byte aligned");
  // forced tokens replace the draw, so the cuts have nothing to act on
  const bool filter = !forced && ((top_k > 0 && top_k < V) || (top_p > 0.0f && top_p < 1.0f));
  if (!filter)
    return launch(textdec_sample_kernel<false>, R, kSampleThreads, 0, stream, logits, R, V, ldl, temperature, seed, uniforms, ldu,
                  forced, ldf, tokens, ldt, done, lengths, step, eos, max_len, record, 0, 0.0f);
  if (V > kFilterMaxV)
    return set_error(VDB_ERR_INVALID, "textdec_sample: top-k / top-p stage at most %d logits per row, got V = %d", kFilterMaxV, V);
  const size_t smem = kFilterHistBytes + static_cast<size_t>(V) * sizeof(uint32_t);
  static bool configured = false;
  if (!configured) {
    VDB_CUDA_CHECK(cudaFuncSetAttribute(textdec_sample_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(kFilterHistBytes + kFilterMaxV * sizeof(uint32_t))));
    configured = true;
  }
  return launch(textdec_sample_kernel<true>, R, kSampleThreads, smem, stream, logits, R, V, ldl, temperature, seed, uniforms, ldu,
                forced, ldf, tokens, ldt, done, lengths, step, eos, max_len, record, top_k, top_p);
}

int vdb_textdec_beam_step(const float* logits, int R, int V, long long ldl, float temperature, int K, int* tokens, int ldt, int* src,
                          int lds, double* scores, int* done, int* lengths, const int* step, int eos, int max_len, int* cand_tok,
                          double* cand_logp, float* record, double* trace, void* stream) {
  if (!logits || !tokens || !src || !scores || !done || !lengths || !step || !cand_tok || !cand_logp)
    return set_error(VDB_ERR_INVALID, "textdec_beam_step: null pointer");
  if (K < 1 || K > kBeamMax) return set_error(VDB_ERR_INVALID, "textdec_beam_step: need 1 <= K <= %d beams, got %d", kBeamMax, K);
  if (R < 1 || R > kGvMaxRows || R % K)
    return set_error(VDB_ERR_INVALID, "textdec_beam_step: need R = n * K <= %d rows, got R = %d, K = %d", kGvMaxRows, R, K);
  if (V < K || V > kFilterMaxV || ldl < V)
    return set_error(VDB_ERR_INVALID, "textdec_beam_step: need K <= V <= %d (staged keys) and ldl >= V, got V = %d", kFilterMaxV, V);
  if (!(temperature > 0.0f)) return set_error(VDB_ERR_INVALID, "textdec_beam_step: temperature must be > 0");
  if (max_len < 2 || ldt < max_len || lds < 1)
    return set_error(VDB_ERR_INVALID, "textdec_beam_step: need max_len >= 2, ldt >= max_len and lds >= 1");
  if ((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(tokens) | reinterpret_cast<uintptr_t>(src) |
       reinterpret_cast<uintptr_t>(done) | reinterpret_cast<uintptr_t>(lengths) | reinterpret_cast<uintptr_t>(step) |
       reinterpret_cast<uintptr_t>(cand_tok) | reinterpret_cast<uintptr_t>(record)) & 3)
    return set_error(VDB_ERR_INVALID, "textdec_beam_step: fp32 / int32 buffers must be 4-byte aligned");
  if ((reinterpret_cast<uintptr_t>(scores) | reinterpret_cast<uintptr_t>(cand_logp) | reinterpret_cast<uintptr_t>(trace)) & 7)
    return set_error(VDB_ERR_INVALID, "textdec_beam_step: scores / cand_logp / trace must be 8-byte aligned");
  const size_t smem = kFilterHistBytes + static_cast<size_t>(V) * sizeof(uint32_t);
  static bool configured = false;
  if (!configured) {
    VDB_CUDA_CHECK(cudaFuncSetAttribute(textdec_beam_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(kFilterHistBytes + kFilterMaxV * sizeof(uint32_t))));
    configured = true;
  }
  const int rc = launch(textdec_beam_topk_kernel, R, kSampleThreads, smem, stream, logits, R, V, ldl, temperature, K, done, step,
                       cand_tok, cand_logp, record);
  if (rc) return rc;
  return launch(textdec_beam_select_kernel, R / K, kSelectThreads, 0, stream, R, K, cand_tok, cand_logp, tokens, ldt, src, lds,
                scores, done, lengths, step, eos, max_len, trace);
}

int vdb_textdec_repetition(float* logits, int R, int V, long long ldl, const int* tokens, int ldt, const int* done, const int* step,
                           float penalty, int ngram, void* stream) {
  if (!logits || !tokens || !done || !step) return set_error(VDB_ERR_INVALID, "textdec_repetition: null pointer");
  if (R < 1 || R > kGvMaxRows || V < 1 || ldl < V || ldt < 1)
    return set_error(VDB_ERR_INVALID, "textdec_repetition: need 1 <= R <= 16, ldl >= V >= 1 and ldt >= 1, got R = %d, V = %d", R, V);
  if (!(penalty > 0.0f) || !isfinite(penalty))
    return set_error(VDB_ERR_INVALID, "textdec_repetition: penalty must be finite and > 0, got %g", static_cast<double>(penalty));
  if (ngram < 0 || ngram > ldt)
    return set_error(VDB_ERR_INVALID, "textdec_repetition: need 0 <= ngram <= ldt, got ngram = %d, ldt = %d", ngram, ldt);
  if ((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(tokens) | reinterpret_cast<uintptr_t>(done) |
       reinterpret_cast<uintptr_t>(step)) & 3)
    return set_error(VDB_ERR_INVALID, "textdec_repetition: buffers must be 4-byte aligned");
  if (penalty == 1.0f && ngram == 0) return VDB_OK;
  return launch(textdec_repetition_kernel, R, kRepThreads, 0, stream, logits, V, ldl, tokens, ldt, done, step, penalty, ngram);
}

}  // extern "C"

}  // namespace vdb
