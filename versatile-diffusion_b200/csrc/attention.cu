// vdb200 — flash-style scaled-dot-product attention on wgmma (sm_90a).
//
// Replaces the reference's materialised  sim = q k^T * d^-1/2 ; softmax ; attn v  of
// CrossAttention.forward (lib/model_zoo/attention.py:178-192) — self-attention N = M in
// {4096,1024,256,64}, d_head in {40,80,160}; cross-attention M = 77 (text) / 257 (image) /
// n*257 (multi-image) — and the CLIP encoder attention (d_head 64, optional causal mask).
//
// One CTA = one (q-tile of 128 rows, head, batch).
//   warps 0-7 : two consumer warpgroups; warpgroup g owns query rows [64 g, 64 g + 64) of the tile.  Per kv tile:
//               S = Q K_j^T (wgmma, both operands from shared memory, fp32 in registers), online softmax in registers
//               (lazy rescale of O), P -> bf16 register fragments, O += P V_j (wgmma with A from registers).
//   TMA loads (Q once; K and V^T tiles through two independent rings) come from one of two places:
//   * TMA_WARP (d_head 160): a ninth warp issues them; 288 threads, one CTA per SM.
//   * otherwise (d_head <= 80): lane 0 of warp 0 refills the K ring and lane 0 of warp 4 the V^T ring, each for tile
//     j + KV_STAGES - 1 while its warpgroup's S_j product runs.  256 threads fit 128 registers at two CTAs per SM, so one
//     CTA's softmax (bound by MUFU ex2) can run under the other's wgmma; with a ninth warp, two CTAs would put five warps on
//     some SM sub-partitions and cap registers at 96, which serialises the wgmmas.
// Operand layouts (all K-major, 128B swizzle, written by the projection GEMMs):
// Batch b occupies rows [b*q_bs, b*q_bs+Nq) of Q/O, rows [b*kv_bs, +Nk) of K, columns [b*kv_bs, +Nk) of Vt.
//   Q  [B*Nq, ldq]  head h at columns q_col0 + h*DK .. (+DK, zero padded beyond d_head)
//   K  [B*Nk, ldk]  head h at columns k_col0 + h*DK ..
//   Vt [H*DVP, >=B*Nk]  row h*DVP + c = channel c of head h (zero rows beyond d_head), column b*Nk + j
//   O  [B*Nq, ldo]  head h at columns h*dv .. (+dv)   (dense, feeds to_out)
#include "common.cuh"
#include "host_util.h"

namespace vdb {

constexpr int kBQ = 128;   // query rows per CTA
constexpr float kRescaleThreshold = 8.0f;  // in log2 units (P stays <= 2^8)

constexpr int attention_threads(bool tma_warp) { return tma_warp ? 288 : 256; }

struct alignas(64) AttnParams {
  CUtensorMap tmQ;   // 2D (cols, rows) box (64, 128)
  CUtensorMap tmK;   // 2D (cols, rows) box (64, BKV)
  CUtensorMap tmV;   // 2D (kv, H*DVP) box (64, DVP)
  int Nq, Nk;        // per-batch query / key counts
  int q_bs, kv_bs;   // per-batch row stride of Q/out, row (K) / column (Vt) stride of the keys (kv_bs % 8 == 0)
  int q_col0, k_col0;
  int dv;            // valid head channels (<= DVP)
  int causal;
  float scale_log2;  // d^-1/2 * log2(e)
  __nv_bfloat16* out;
  long long ldo;
  const int* kv_len; // [B] valid keys per batch item (VARLEN instantiations only; key j of item b is visible iff j < kv_len[b])
  const int* items;  // INDEXED: [rows][3][B] int32 source items {bq, bk, bv} of output item b, row *step_idx
  const int* step_idx;
  int accumulate;    // INDEXED: out = bf16(float(out) + O)
};

template <int DK, int DVP, int BKV, int KV_STAGES>
constexpr size_t attention_smem_bytes() {
  return (DK / 64) * kBQ * 128 + KV_STAGES * ((DK / 64) * BKV * 128 + (BKV / 64) * DVP * 128) + (1 + 4 * KV_STAGES) * 8 + 1024;
}

// DK = padded q/k head width (64-channel swizzle atoms), DVP = padded v head width (the N of the PV product),
// BKV = keys per tile (the N of the QK^T product), TMA_WARP = a ninth warp issues the loads (see the top of the file).
// VARLEN: batch item b sees only its first min(kv_len[b], Nk) keys (BERT's padding mask); an item with no key writes zero rows.
// INDEXED: output item b takes its Q, K and V from items {bq, bk, bv} of row *step_idx of the table (Prompt-to-Prompt's attention
// injection, lib/model_zoo/prompt_edit.py); bv < 0 skips the item.
template <int DK, int DVP, int BKV, int KV_STAGES, bool TMA_WARP, bool VARLEN = false, bool INDEXED = false>
__global__ void __launch_bounds__(attention_threads(TMA_WARP), TMA_WARP ? 1 : 2)
    attention_kernel(const __grid_constant__ AttnParams p) {
  constexpr int KA = DK / 64;                      // 64-wide K atoms of the QK^T reduction
  constexpr int KVA = BKV / 64;                    // 64-kv atoms per tile (K dimension of the PV product)
  constexpr uint32_t kQBytes = KA * kBQ * 128;     // Q tile
  constexpr uint32_t kKBytes = KA * BKV * 128;     // one K stage
  constexpr uint32_t kVAtom = DVP * 128;           // one 64-kv atom of V^T
  constexpr uint32_t kVBytes = KVA * kVAtom;       // one V stage (BKV kv)
  // K16 steps of QK^T: Q is zero past d_head <= DVP, so the steps past DVP add nothing (d 40: 3 of 4, d 80 in DK 128: 5 of 8).
  // A fixed count issues the steps as one wgmma chain; with a count read at run time each step sat behind its own branch, and
  // the registers ptxas kept around the conditional wgmmas (159 at d 40, 168 at d 80) ruled out two CTAs per SM.
  constexpr int kQKSteps = (DVP < DK ? DVP : DK) / 16;
  static_assert(BKV == 64 || BKV == 128, "kv tile");
  static_assert(kVAtom % 1024 == 0, "V atom must keep 1024B alignment");
  static_assert(DVP % 16 == 0 && DVP <= 256, "invalid wgmma N for PV");

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kQBytes;
  uint8_t* sV = sK + KV_STAGES * kKBytes;
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sV + KV_STAGES * kVBytes);
  uint64_t* k_full = q_full + 1;                  // [KV_STAGES]
  uint64_t* k_empty = k_full + KV_STAGES;         // [KV_STAGES] (count 8: one arrive per consumer warp)
  uint64_t* v_full = k_empty + KV_STAGES;         // [KV_STAGES]
  uint64_t* v_empty = v_full + KV_STAGES;         // [KV_STAGES] (count 8)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kBQ;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  int bq = b, bk = b, bv = b;
  if constexpr (INDEXED) {
    const int* row = p.items + static_cast<long long>(*p.step_idx) * 3 * gridDim.z;
    bq = row[b];
    bk = row[gridDim.z + b];
    bv = row[2 * gridDim.z + b];
    if (bv < 0) return;                            // the whole CTA, before any barrier, load or write
  }

  int nk = 0;                                      // VARLEN: this item's key count
  int ntiles = (p.Nk + BKV - 1) / BKV;
  if (p.causal) ntiles = min(ntiles, (q0 + kBQ + BKV - 1) / BKV);

  if (warp == (TMA_WARP ? 8 : 0) && lane == 0) {
    tma_prefetch_desc(&p.tmQ);
    tma_prefetch_desc(&p.tmK);
    tma_prefetch_desc(&p.tmV);
  }
  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < KV_STAGES; ++s) {
      mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], 8);
      mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();
  if constexpr (VARLEN) {
    nk = max(0, min(p.kv_len[b], p.Nk));
    ntiles = (nk + BKV - 1) / BKV;
  }

  // One thread each: the tile's Q, and K / V^T tile t into its stage once all eight consumer warps released the stage's
  // previous tile (t - KV_STAGES).
  auto load_q = [&] {
    mbar_arrive_expect_tx(q_full, kQBytes);
    for (int a = 0; a < KA; ++a)
      tma_load_2d(sQ + a * kBQ * 128, &p.tmQ, q_full, p.q_col0 + head * DK + a * 64, bq * p.q_bs + q0);
  };
  auto load_k = [&](int t) {
    const int st = t % KV_STAGES;
    mbar_wait(&k_empty[st], ((t / KV_STAGES) & 1) ^ 1);
    mbar_arrive_expect_tx(&k_full[st], kKBytes);
    for (int a = 0; a < KA; ++a)
      tma_load_2d(sK + st * kKBytes + a * BKV * 128, &p.tmK, &k_full[st], p.k_col0 + head * DK + a * 64, bk * p.kv_bs + t * BKV);
  };
  auto load_v = [&](int t) {
    const int st = t % KV_STAGES;
    mbar_wait(&v_empty[st], ((t / KV_STAGES) & 1) ^ 1);
    mbar_arrive_expect_tx(&v_full[st], kVBytes);
    for (int a = 0; a < KVA; ++a)
      tma_load_2d(sV + st * kVBytes + a * kVAtom, &p.tmV, &v_full[st], bv * p.kv_bs + t * BKV + a * 64, head * DVP);
  };

  if constexpr (TMA_WARP) {
    if (warp == 8) {
      if (lane == 0) {
        load_q();
        for (int j = 0; j < ntiles; ++j) {
          load_k(j);
          load_v(j);
        }
      }
      return;
    }
  } else {   // the first KV_STAGES - 1 tiles; iteration j of the loop below loads tile j + KV_STAGES - 1
    if (lane == 0 && warp == 0) {
      load_q();
      for (int t = 0; t < min(KV_STAGES - 1, ntiles); ++t) load_k(t);
    }
    if (lane == 0 && warp == 4)
      for (int t = 0; t < min(KV_STAGES - 1, ntiles); ++t) load_v(t);
    __syncwarp();
  }

  // ------------------------------ consumer warpgroup g ------------------------------
  // Fragment ownership (see wgmma.cuh): this thread holds rows row0 and row0 + 8 of the group's 64, columns 8 jj + 2 c + {0, 1}.
  const int g = warp >> 2;
  const int row0 = g * 64 + (warp & 3) * 16 + (lane >> 2);
  const int c2 = 2 * (lane & 3);
  const int q_idx[2] = {q0 + row0, q0 + row0 + 8};
  float o[DVP / 2];
#pragma unroll
  for (int i = 0; i < DVP / 2; ++i) o[i] = 0.f;
  float m_ref[2] = {-INFINITY, -INFINITY};
  float l_sum[2] = {0.f, 0.f};                   // this thread's share of the row sums
  mbar_wait(q_full, 0);
#pragma unroll 1
  for (int j = 0; j < ntiles; ++j) {
    const int st = j % KV_STAGES;
    const uint32_t ph = (j / KV_STAGES) & 1;
    float s[BKV / 2];
    mbar_wait(&k_full[st], ph);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kQKSteps; ++k) {
      const uint64_t qd = make_desc_sw128(smem_u32(sQ + (k / 4) * kBQ * 128 + g * 64 * 128));
      const uint64_t kd = make_desc_sw128(smem_u32(sK + st * kKBytes + (k / 4) * BKV * 128));
      wgmma_ss<BKV>(s, qd + 2 * (k % 4), kd + 2 * (k % 4), k > 0 ? 1u : 0u);
    }
    wgmma_commit();
    if constexpr (!TMA_WARP) {   // refill the stage of tile j - 1 (K by warpgroup 0, V^T by warpgroup 1) under the S product
      const int t = j + KV_STAGES - 1;
      if ((warp & 3) == 0 && lane == 0 && t < ntiles) {
        if (g == 0)
          load_k(t);
        else
          load_v(t);
      }
      __syncwarp();
    }
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    __syncwarp();
    if (lane == 0) mbar_arrive(&k_empty[st]);

    const int kv0 = j * BKV;
    if (kv0 + BKV > (VARLEN ? nk : p.Nk) || p.causal) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int lim = p.causal ? min(p.Nk, q_idx[i] + 1) : (VARLEN ? nk : p.Nk);   // valid kv indices are < lim
#pragma unroll
        for (int jj = 0; jj < BKV / 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (kv0 + 8 * jj + c2 + e >= lim) s[4 * jj + 2 * i + e] = -INFINITY;
      }
    }
    float m_scaled[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < BKV / 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * i], s[4 * jj + 2 * i + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_ref[i], mx);
      if (j == 0 || m_ref[i] == -INFINITY) {
        m_ref[i] = m_new;
      } else if ((m_new - m_ref[i]) * p.scale_log2 > kRescaleThreshold) {   // lazy rescale: only when P could exceed 2^8
        const float factor = ex2_mufu((m_ref[i] - m_new) * p.scale_log2);
        m_ref[i] = m_new;
        l_sum[i] *= factor;
#pragma unroll
        for (int jj = 0; jj < DVP / 8; ++jj) {
          o[4 * jj + 2 * i] *= factor;
          o[4 * jj + 2 * i + 1] *= factor;
        }
      }
      m_scaled[i] = (m_ref[i] == -INFINITY) ? 0.f : m_ref[i] * p.scale_log2;
    }
    // P = exp2(s * scale - m) as bf16 A fragments of the PV product: k-step kk covers kv columns [16 kk, 16 kk + 16)
    uint32_t pa[BKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        const int i = h & 1;                      // fragment registers alternate rows row0 / row0 + 8
        const int idx = 8 * kk + 4 * (h >> 1) + 2 * i;
        const float e0 = ex2_mufu(fmaf(s[idx], p.scale_log2, -m_scaled[i]));
        const float e1 = ex2_mufu(fmaf(s[idx + 1], p.scale_log2, -m_scaled[i]));
        l_sum[i] += e0 + e1;
        pa[kk][h] = pack_bf16x2(e0, e1);
      }
    }
    mbar_wait(&v_full[st], ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      const uint64_t vd = make_desc_sw128(smem_u32(sV + st * kVBytes + (kk >> 2) * kVAtom));
      wgmma_rs<DVP>(o, pa[kk], vd + 2 * (kk & 3), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&v_empty[st]);
  }

  // epilogue: O / l -> bf16
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float l = l_sum[i];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv_l = (VARLEN && !(l > 0.f)) ? 0.f : 1.f / l;   // VARLEN, no visible key: o == 0, write zeros, not 0 / 0
    if (q_idx[i] >= p.Nq) continue;
    __nv_bfloat16* orow = p.out + (static_cast<long long>(b) * p.q_bs + q_idx[i]) * p.ldo + head * p.dv;
#pragma unroll
    for (int jj = 0; jj < DVP / 8; ++jj) {
      const int col = 8 * jj + c2;
      if (col < p.dv) {   // (dv % 8 == 0: the pair never straddles the end)
        float v0 = o[4 * jj + 2 * i] * inv_l, v1 = o[4 * jj + 2 * i + 1] * inv_l;
        if (INDEXED && p.accumulate) {
          const __nv_bfloat162 prev = *reinterpret_cast<const __nv_bfloat162*>(orow + col);
          v0 += __bfloat162float(prev.x);
          v1 += __bfloat162float(prev.y);
        }
        *reinterpret_cast<uint32_t*>(orow + col) = pack_bf16x2(v0, v1);
      }
    }
  }
}

struct AttnArgs {   // what the C ABI received; the tensor maps depend on the kernel variant's kv tile
  const void *Q, *K, *Vt;
  long long ldq, ldk, ldv;
  int B, H, q_bstride, kv_bstride;
  int Bq, Bkv;       // items in Q and in K / V^T (B unless indexed)
};

template <int DK, int DVP, int BKV, int KV_STAGES, bool TMA_WARP, bool VARLEN = false, bool INDEXED = false>
static int launch_attention(AttnParams& p, const AttnArgs& a, void* stream) {
  constexpr size_t smem = attention_smem_bytes<DK, DVP, BKV, KV_STAGES>();
  // two CTAs per SM need twice the dynamic window plus 1 KB each reserved by the system, within 228 KB
  static_assert(smem <= (TMA_WARP ? 227 * 1024 : 113 * 1024), "attention smem budget");
  auto kernel = attention_kernel<DK, DVP, BKV, KV_STAGES, TMA_WARP, VARLEN, INDEXED>;
  static bool configured = false;
  if (!configured) {
    VDB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    if (!TMA_WARP)   // the second CTA per SM is the point of this form: ask for the whole carveout, not the driver's pick
      VDB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    configured = true;
  }
  int rc = make_tmap_2d(&p.tmQ, a.Q, static_cast<uint64_t>(a.ldq), static_cast<uint64_t>(a.Bq) * a.q_bstride, a.ldq * 2, 64, kBQ);
  if (rc) return rc;
  rc = make_tmap_2d(&p.tmK, a.K, static_cast<uint64_t>(a.ldk), static_cast<uint64_t>(a.Bkv) * a.kv_bstride, a.ldk * 2, 64, BKV);
  if (rc) return rc;
  rc = make_tmap_2d(&p.tmV, a.Vt, static_cast<uint64_t>(a.Bkv) * a.kv_bstride, static_cast<uint64_t>(a.H) * DVP, a.ldv * 2, 64, DVP);
  if (rc) return rc;
  dim3 grid((p.Nq + kBQ - 1) / kBQ, a.H, a.B);
  return launch(kernel, grid, dim3(attention_threads(TMA_WARP)), smem, stream, p);
}

// The instantiation for the head pads (DK, DVP) of p.dv, plain or indexed.  d_head <= 80: two CTAs per SM, each within 128
// registers and half the shared memory (d_head <= 64: 128-key tiles, 3 / 2 stages; d_head 80: 64-key tiles, 3 stages).
// d_head 160 keeps the TMA warp and one CTA per SM: two CTAs' Q and K / V^T stages do not fit; 64-key tiles keep its S + O + P
// within the register budget.
template <bool INDEXED>
static int launch_for_pads(int DK, int DVP, AttnParams& p, const AttnArgs& a, void* stream) {
  if (DK == 64 && DVP == 48) return launch_attention<64, 48, 128, 3, false, false, INDEXED>(p, a, stream);
  if (DK == 64 && DVP == 64) return launch_attention<64, 64, 128, 2, false, false, INDEXED>(p, a, stream);
  if (DK == 128 && DVP == 80) return launch_attention<128, 80, 64, 3, false, false, INDEXED>(p, a, stream);
  if (DK == 192 && DVP == 160) return launch_attention<192, 160, 64, 2, true, false, INDEXED>(p, a, stream);
  return set_error(VDB_ERR_UNSUPPORTED, "attention: no kernel for d_head %d", p.dv);
}

// Prompt-to-Prompt's word maps (lib/model_zoo/prompt_edit.py) from the bf16 operands of a cross-attention call, fp32 math:
//   map[r, p] += sum over h of sum over j < L of w[r, j] softmax_j(scale q[(row0 + r) N + p, head h] . k[(row0 + r) kv_bs + j, head h])
// One CTA per (block of kWmapQ queries, r).  K of one head at a time sits in shared memory; warp g owns queries
// g*kWmapQ/8 .. of the block, lane l keys l, l + 32, l + 64.  The heads are summed in order, the keys by partial sums per lane
// and a fixed xor tree, and every map entry has one writer: the result is bit-reproducible.
constexpr int kWmapThreads = 256, kWmapQ = 16, kWmapMaxL = 80, kWmapMaxD = 160;

__global__ void __launch_bounds__(kWmapThreads) xattn_word_map_kernel(
    const __nv_bfloat16* __restrict__ Q, long long ldq, const __nv_bfloat16* __restrict__ K, long long ldk,
    const float* __restrict__ w, float* __restrict__ map, int row0, int H, int N, int L, int kv_bs, int d, int DK,
    float scale_log2) {
  constexpr int kPerWarp = kWmapQ / (kWmapThreads / 32);
  constexpr int kRowWords = kWmapMaxD / 2 + 1;     // odd row stride in 4-byte words: lanes reading 32 rows hit 32 banks
  __shared__ __nv_bfloat162 sK[kWmapMaxL * kRowWords];
  __shared__ float sq[kWmapThreads / 32][kWmapMaxD];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.y, item = row0 + r;
  const int rw = d / 2 + 1;
  float wj[3];
#pragma unroll
  for (int t = 0; t < 3; ++t) wj[t] = lane + 32 * t < L ? w[static_cast<long long>(r) * L + lane + 32 * t] : 0.f;
  float acc[kPerWarp];
#pragma unroll
  for (int qq = 0; qq < kPerWarp; ++qq) acc[qq] = 0.f;
  for (int h = 0; h < H; ++h) {
    __syncthreads();
    for (int e = threadIdx.x; e < L * (d / 2); e += kWmapThreads) {
      const int j = e / (d / 2), c2 = e % (d / 2);
      sK[j * rw + c2] = *reinterpret_cast<const __nv_bfloat162*>(K + (static_cast<long long>(item) * kv_bs + j) * ldk + h * DK + 2 * c2);
    }
    __syncthreads();
#pragma unroll
    for (int qq = 0; qq < kPerWarp; ++qq) {
      const int p = blockIdx.x * kWmapQ + warp * kPerWarp + qq;
      if (p >= N) break;
      const __nv_bfloat16* qrow = Q + (static_cast<long long>(item) * N + p) * ldq + h * DK;
      for (int c = lane; c < d; c += 32) sq[warp][c] = __bfloat162float(qrow[c]);
      __syncwarp();
      float sc[3];
      float mx = -INFINITY;
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        const int j = lane + 32 * t;
        sc[t] = -INFINITY;
        if (j < L) {
          float dot = 0.f;
          for (int c2 = 0; c2 < d / 2; ++c2) {
            const float2 kv = __bfloat1622float2(sK[j * rw + c2]);
            dot = fmaf(sq[warp][2 * c2], kv.x, dot);
            dot = fmaf(sq[warp][2 * c2 + 1], kv.y, dot);
          }
          sc[t] = dot;
          mx = fmaxf(mx, dot);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float den = 0.f, num = 0.f;
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        const float e = lane + 32 * t < L ? exp2f((sc[t] - mx) * scale_log2) : 0.f;
        den += e;
        num = fmaf(wj[t], e, num);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        den += __shfl_xor_sync(0xffffffffu, den, o);
        num += __shfl_xor_sync(0xffffffffu, num, o);
      }
      acc[qq] += num / den;
      __syncwarp();
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int qq = 0; qq < kPerWarp; ++qq) {
      const int p = blockIdx.x * kWmapQ + warp * kPerWarp + qq;
      if (p < N) map[static_cast<long long>(r) * N + p] += acc[qq];
    }
  }
}

// Self-attention guidance's key mass (lib/model_zoo/sag.py) from the bf16 operands of a self-attention call, fp32 math:
//   mass[r, j] += w * sum over h of sum over p < N of softmax_j(scale q[(row0 + r) N + p, head h] . k[(row0 + r) kv_bs + j, head h])
// A column sum of a row softmax, in two launches.  sattn_row_stats_kernel: one CTA per (kMassQ queries, head, r) walks the keys in
// shared-memory tiles of kMassKT; warp g owns queries g*kMassQ/8 .., lane l keys l, l + 32 of each tile, with a running
// (max, sum) per lane merged by a fixed xor tree -> stats[r, h, p] = {max of the raw dots, sum of exp2((dot - max) scale_log2)}.
// sattn_key_mass_kernel: one CTA per (32 keys, r); lane l owns key l of the block, warp g queries p = g mod 8, all heads in order;
// the eight warps' partial sums are added in warp order and each mass entry has one writer: the result is bit-reproducible.
constexpr int kMassThreads = 256, kMassQ = 32, kMassKT = 64, kMassKeys = 32, kMassMaxD = 160, kMassMaxN = 4096;

__device__ __forceinline__ void merge_stats(float& m, float& l, float mo, float lo, float scale_log2) {
  const float mn = fmaxf(m, mo);
  const float a = m == -INFINITY ? 0.f : l * exp2f((m - mn) * scale_log2);
  const float b = mo == -INFINITY ? 0.f : lo * exp2f((mo - mn) * scale_log2);
  m = mn;
  l = a + b;
}

__global__ void __launch_bounds__(kMassThreads) sattn_row_stats_kernel(
    const __nv_bfloat16* __restrict__ Q, long long ldq, const __nv_bfloat16* __restrict__ K, long long ldk,
    float* __restrict__ stats, int row0, int H, int N, int kv_bs, int d, int DK, float scale_log2) {
  constexpr int kPerWarp = kMassQ / (kMassThreads / 32);
  constexpr int kRowWords = kMassMaxD / 2 + 1;     // odd row stride in 4-byte words: lanes reading 32 rows hit 32 banks
  __shared__ __nv_bfloat162 sK[kMassKT * kRowWords];
  __shared__ float sq[kMassThreads / 32][kPerWarp][kMassMaxD];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y, r = blockIdx.z, item = row0 + r;
  const int rw = d / 2 + 1;
#pragma unroll
  for (int qq = 0; qq < kPerWarp; ++qq) {
    const int p = min(blockIdx.x * kMassQ + warp * kPerWarp + qq, N - 1);
    const __nv_bfloat16* qrow = Q + (static_cast<long long>(item) * N + p) * ldq + h * DK;
    for (int c = lane; c < d; c += 32) sq[warp][qq][c] = __bfloat162float(qrow[c]);
  }
  float m[kPerWarp], l[kPerWarp];
#pragma unroll
  for (int qq = 0; qq < kPerWarp; ++qq) m[qq] = -INFINITY, l[qq] = 0.f;
  for (int j0 = 0; j0 < N; j0 += kMassKT) {
    const int nk = min(kMassKT, N - j0);
    __syncthreads();
    for (int e = threadIdx.x; e < nk * (d / 2); e += kMassThreads) {
      const int j = e / (d / 2), c2 = e % (d / 2);
      sK[j * rw + c2] =
          *reinterpret_cast<const __nv_bfloat162*>(K + (static_cast<long long>(item) * kv_bs + j0 + j) * ldk + h * DK + 2 * c2);
    }
    __syncthreads();
#pragma unroll
    for (int t = 0; t < kMassKT / 32; ++t) {
      const int j = lane + 32 * t;
      if (j >= nk) break;
      float dot[kPerWarp];
#pragma unroll
      for (int qq = 0; qq < kPerWarp; ++qq) dot[qq] = 0.f;
      for (int c2 = 0; c2 < d / 2; ++c2) {
        const float2 kv = __bfloat1622float2(sK[j * rw + c2]);
#pragma unroll
        for (int qq = 0; qq < kPerWarp; ++qq) {
          dot[qq] = fmaf(sq[warp][qq][2 * c2], kv.x, dot[qq]);
          dot[qq] = fmaf(sq[warp][qq][2 * c2 + 1], kv.y, dot[qq]);
        }
      }
#pragma unroll
      for (int qq = 0; qq < kPerWarp; ++qq) merge_stats(m[qq], l[qq], dot[qq], 1.f, scale_log2);
    }
  }
#pragma unroll
  for (int qq = 0; qq < kPerWarp; ++qq) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float mo = __shfl_xor_sync(0xffffffffu, m[qq], o), lo = __shfl_xor_sync(0xffffffffu, l[qq], o);
      merge_stats(m[qq], l[qq], mo, lo, scale_log2);
    }
    const int p = blockIdx.x * kMassQ + warp * kPerWarp + qq;
    if (lane == 0 && p < N) {
      float* s = stats + ((static_cast<long long>(r) * H + h) * N + p) * 2;
      s[0] = m[qq];
      s[1] = l[qq];
    }
  }
}

__global__ void __launch_bounds__(kMassThreads) sattn_key_mass_kernel(
    const __nv_bfloat16* __restrict__ Q, long long ldq, const __nv_bfloat16* __restrict__ K, long long ldk,
    const float* __restrict__ stats, float w, float* __restrict__ mass, int row0, int H, int N, int kv_bs, int d, int DK,
    float scale_log2) {
  constexpr int kWarps = kMassThreads / 32;
  constexpr int kRowWords = kMassMaxD / 2 + 1;
  __shared__ __nv_bfloat162 sK[kMassKeys * kRowWords];
  __shared__ float sq[kWarps][kMassMaxD];
  __shared__ float part[kWarps][kMassKeys];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.y, item = row0 + r;
  const int j0 = blockIdx.x * kMassKeys, nk = min(kMassKeys, N - j0);
  const int rw = d / 2 + 1;
  float acc = 0.f;
  for (int h = 0; h < H; ++h) {
    __syncthreads();
    for (int e = threadIdx.x; e < nk * (d / 2); e += kMassThreads) {
      const int j = e / (d / 2), c2 = e % (d / 2);
      sK[j * rw + c2] =
          *reinterpret_cast<const __nv_bfloat162*>(K + (static_cast<long long>(item) * kv_bs + j0 + j) * ldk + h * DK + 2 * c2);
    }
    __syncthreads();
    const float* st = stats + (static_cast<long long>(r) * H + h) * N * 2;
    for (int p = warp; p < N; p += kWarps) {
      const __nv_bfloat16* qrow = Q + (static_cast<long long>(item) * N + p) * ldq + h * DK;
      for (int c = lane; c < d; c += 32) sq[warp][c] = __bfloat162float(qrow[c]);
      __syncwarp();
      if (lane < nk) {
        float dot = 0.f;
        for (int c2 = 0; c2 < d / 2; ++c2) {
          const float2 kv = __bfloat1622float2(sK[lane * rw + c2]);
          dot = fmaf(sq[warp][2 * c2], kv.x, dot);
          dot = fmaf(sq[warp][2 * c2 + 1], kv.y, dot);
        }
        acc += exp2f((dot - st[2 * p]) * scale_log2) / st[2 * p + 1];
      }
      __syncwarp();
    }
  }
  part[warp][lane] = acc;
  __syncthreads();
  if (warp == 0 && lane < nk) {
    float s = 0.f;
#pragma unroll
    for (int g = 0; g < kWarps; ++g) s += part[g][lane];
    mass[static_cast<long long>(r) * N + j0 + lane] += w * s;
  }
}

}  // namespace vdb

using namespace vdb;

extern "C" {

// Padded head sizes the projection GEMMs must produce for a given d_head (see include/vdb200.h).
int vdb_attention_dk_pad(int d_head) { return d_head <= 64 ? 64 : (d_head <= 128 ? 128 : (d_head <= 192 ? 192 : -1)); }
int vdb_attention_dv_pad(int d_head) {
  if (d_head <= 48) return 48;
  if (d_head <= 64) return 64;
  if (d_head <= 80) return 80;
  if (d_head <= 160) return 160;
  return -1;
}

int vdb_attention_bf16(const void* Q, long long ldq, int q_col0, const void* K, long long ldk, int k_col0,
                       const void* Vt, long long ldv, void* out, long long ldo, int B, int H, int Nq, int Nk,
                       int q_bstride, int kv_bstride, int d_head, float scale, int causal,
                       const int* kv_len, int Bq, int Bkv, const int* items, const int* step_idx, int accumulate,
                       void* stream) {
  // each form's own checks come first.  Any argument of the item table asks for the indexed form, which needs the table.
  if (items || step_idx || Bq || Bkv || accumulate) {
    if (!items || !step_idx || (reinterpret_cast<uintptr_t>(items) & 3) || (reinterpret_cast<uintptr_t>(step_idx) & 3))
      return set_error(VDB_ERR_INVALID, "attention: items and step_idx must be non-null, 4-byte aligned device int32 "
                                        "(Bq, Bkv and accumulate belong to them)");
    if (kv_len) return set_error(VDB_ERR_UNSUPPORTED, "attention: no kernel takes both kv_len and items");
    if (Bq <= 0 || Bkv <= 0) return set_error(VDB_ERR_INVALID, "attention: Bq and Bkv must be > 0 (got %d, %d)", Bq, Bkv);
  } else if (kv_len) {
    if (reinterpret_cast<uintptr_t>(kv_len) & 3)
      return set_error(VDB_ERR_INVALID, "attention: kv_len must be a 4-byte aligned device int32 [B]");
    if (causal) return set_error(VDB_ERR_INVALID, "attention: causal masking together with kv_len is not supported");
    if (vdb_attention_dk_pad(d_head) != 64 || vdb_attention_dv_pad(d_head) != 64)
      return set_error(VDB_ERR_UNSUPPORTED, "attention: with kv_len only d_head 64 (BERT) is instantiated, got %d", d_head);
  }
  if (!Q || !K || !Vt || !out || B <= 0 || H <= 0 || Nq <= 0 || Nk <= 0)
    return set_error(VDB_ERR_INVALID, "attention: null/empty argument");
  const int DK = vdb_attention_dk_pad(d_head), DVP = vdb_attention_dv_pad(d_head);
  if (DK < 0 || DVP < 0) return set_error(VDB_ERR_UNSUPPORTED, "attention: d_head %d not supported (<= 160)", d_head);
  if ((d_head % 8) || (ldo % 8) || (ldq % 8) || (ldk % 8) || (ldv % 8))
    return set_error(VDB_ERR_INVALID, "attention: d_head and leading dims must be multiples of 8");
  if (q_bstride <= 0) q_bstride = Nq;
  if (kv_bstride <= 0) kv_bstride = Nk;
  // TMA needs the innermost box coordinate (the kv column of V^T) on a 16-byte boundary
  if (q_bstride < Nq || kv_bstride < Nk || (kv_bstride % 8))
    return set_error(VDB_ERR_INVALID, "attention: need q_bstride >= Nq, kv_bstride >= Nk and kv_bstride %% 8 == 0 (got %d, %d)",
                     q_bstride, kv_bstride);
  AttnParams p;
  memset(&p, 0, sizeof(p));
  p.Nq = Nq; p.Nk = Nk; p.q_bs = q_bstride; p.kv_bs = kv_bstride; p.q_col0 = q_col0; p.k_col0 = k_col0; p.dv = d_head; p.causal = causal;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.ldo = ldo;
  p.kv_len = kv_len;
  p.items = items;
  p.step_idx = step_idx;
  p.accumulate = accumulate ? 1 : 0;
  const AttnArgs a{Q, K, Vt, ldq, ldk, ldv, B, H, q_bstride, kv_bstride, items ? Bq : B, items ? Bkv : B};
  if (!kv_len && !items) return launch_for_pads<false>(DK, DVP, p, a, stream);
  if (kv_len) return launch_attention<64, 64, 128, 2, false, true>(p, a, stream);
  return launch_for_pads<true>(DK, DVP, p, a, stream);
}

int vdb_xattn_word_map_f32(const void* Q, long long ldq, const void* K, long long ldk, const float* w, float* map, int n, int row0,
                           int H, int N, int L, int kv_bstride, int d_head, float scale, void* stream) {
  if (!Q || !K || !w || !map || n <= 0 || row0 < 0 || H <= 0 || N <= 0 || L <= 0)
    return set_error(VDB_ERR_INVALID, "xattn_word_map: null/empty argument");
  if (L > kWmapMaxL) return set_error(VDB_ERR_UNSUPPORTED, "xattn_word_map: at most %d keys (a text context), got %d", kWmapMaxL, L);
  const int DK = vdb_attention_dk_pad(d_head);
  if (DK < 0 || d_head > kWmapMaxD || d_head % 8)
    return set_error(VDB_ERR_UNSUPPORTED, "xattn_word_map: d_head %d not supported (a multiple of 8, <= %d)", d_head, kWmapMaxD);
  if (kv_bstride <= 0) kv_bstride = L;
  if (kv_bstride < L || ldq < static_cast<long long>(H) * DK || ldk < static_cast<long long>(H) * DK || (ldq & 1) || (ldk & 1))
    return set_error(VDB_ERR_INVALID, "xattn_word_map: need kv_bstride >= L and even ldq, ldk >= H * %d", DK);
  if ((reinterpret_cast<uintptr_t>(Q) | reinterpret_cast<uintptr_t>(K) | reinterpret_cast<uintptr_t>(w) |
       reinterpret_cast<uintptr_t>(map)) & 3)
    return set_error(VDB_ERR_INVALID, "xattn_word_map: pointers must be 4-byte aligned");
  const char *m0 = reinterpret_cast<const char*>(map), *m1 = m0 + static_cast<long long>(n) * N * 4;
  const char *w0 = reinterpret_cast<const char*>(w), *w1 = w0 + static_cast<long long>(n) * L * 4;
  if (m0 < w1 && w0 < m1) return set_error(VDB_ERR_INVALID, "xattn_word_map: map overlaps w");
  dim3 grid((N + kWmapQ - 1) / kWmapQ, n);
  return launch(xattn_word_map_kernel, grid, dim3(kWmapThreads), 0, stream, reinterpret_cast<const __nv_bfloat16*>(Q), ldq,
                reinterpret_cast<const __nv_bfloat16*>(K), ldk, w, map, row0, H, N, L, kv_bstride, d_head, DK,
                scale * 1.4426950408889634f);
}

int vdb_sattn_key_mass_f32(const void* Q, long long ldq, int q_col0, const void* K, long long ldk, int k_col0, float* stats,
                           float w, float* mass, int n, int row0, int H, int N, int kv_bstride, int d_head, float scale,
                           void* stream) {
  if (!Q || !K || !stats || !mass || n <= 0 || row0 < 0 || H <= 0 || N <= 0)
    return set_error(VDB_ERR_INVALID, "sattn_key_mass: null/empty argument");
  if (N > kMassMaxN) return set_error(VDB_ERR_UNSUPPORTED, "sattn_key_mass: at most %d tokens, got %d", kMassMaxN, N);
  const int DK = vdb_attention_dk_pad(d_head);
  if (DK < 0 || d_head <= 0 || d_head > kMassMaxD || d_head % 8)
    return set_error(VDB_ERR_UNSUPPORTED, "sattn_key_mass: d_head %d not supported (a multiple of 8, <= %d)", d_head, kMassMaxD);
  if (kv_bstride <= 0) kv_bstride = N;
  const long long cols = static_cast<long long>(H) * DK;
  if (kv_bstride < N || q_col0 < 0 || k_col0 < 0 || (q_col0 & 1) || (k_col0 & 1) || (ldq & 1) || (ldk & 1) ||
      ldq < q_col0 + cols || ldk < k_col0 + cols)
    return set_error(VDB_ERR_INVALID, "sattn_key_mass: need kv_bstride >= N, even column offsets and even ldq, ldk >= col0 + H * %d",
                     DK);
  if ((reinterpret_cast<uintptr_t>(Q) | reinterpret_cast<uintptr_t>(K) | reinterpret_cast<uintptr_t>(stats) |
       reinterpret_cast<uintptr_t>(mass)) & 3)
    return set_error(VDB_ERR_INVALID, "sattn_key_mass: pointers must be 4-byte aligned");
  const char *m0 = reinterpret_cast<const char*>(mass), *m1 = m0 + static_cast<long long>(n) * N * 4;
  const char *s0 = reinterpret_cast<const char*>(stats), *s1 = s0 + static_cast<long long>(n) * H * N * 2 * 4;
  if (m0 < s1 && s0 < m1) return set_error(VDB_ERR_INVALID, "sattn_key_mass: mass overlaps stats");
  const __nv_bfloat16* q = reinterpret_cast<const __nv_bfloat16*>(Q) + q_col0;
  const __nv_bfloat16* k = reinterpret_cast<const __nv_bfloat16*>(K) + k_col0;
  const float scale_log2 = scale * 1.4426950408889634f;
  int st = launch(sattn_row_stats_kernel, dim3((N + kMassQ - 1) / kMassQ, H, n), dim3(kMassThreads), 0, stream, q, ldq, k, ldk,
                  stats, row0, H, N, kv_bstride, d_head, DK, scale_log2);
  if (st) return st;
  return launch(sattn_key_mass_kernel, dim3((N + kMassKeys - 1) / kMassKeys, n), dim3(kMassThreads), 0, stream, q, ldq, k, ldk,
                static_cast<const float*>(stats), w, mass, row0, H, N, kv_bstride, d_head, DK, scale_log2);
}

}  // extern "C"
