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
};

template <int DK, int DVP, int BKV, int KV_STAGES>
constexpr size_t attention_smem_bytes() {
  return (DK / 64) * kBQ * 128 + KV_STAGES * ((DK / 64) * BKV * 128 + (BKV / 64) * DVP * 128) + (1 + 4 * KV_STAGES) * 8 + 1024;
}

// DK = padded q/k head width (64-channel swizzle atoms), DVP = padded v head width (the N of the PV product),
// BKV = keys per tile (the N of the QK^T product), TMA_WARP = a ninth warp issues the loads (see the top of the file).
// VARLEN: batch item b sees only its first min(kv_len[b], Nk) keys (BERT's padding mask); an item with no key writes zero rows.
template <int DK, int DVP, int BKV, int KV_STAGES, bool TMA_WARP, bool VARLEN = false>
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
  pdl_launch_dependents();
  pdl_wait();
  if constexpr (VARLEN) {   // kv_len may be written by the kernel this launch overlaps: read it only after pdl_wait
    nk = max(0, min(p.kv_len[b], p.Nk));
    ntiles = (nk + BKV - 1) / BKV;
  }

  // One thread each: the tile's Q, and K / V^T tile t into its stage once all eight consumer warps released the stage's
  // previous tile (t - KV_STAGES).
  auto load_q = [&] {
    mbar_arrive_expect_tx(q_full, kQBytes);
    for (int a = 0; a < KA; ++a)
      tma_load_2d(sQ + a * kBQ * 128, &p.tmQ, q_full, p.q_col0 + head * DK + a * 64, b * p.q_bs + q0);
  };
  auto load_k = [&](int t) {
    const int st = t % KV_STAGES;
    mbar_wait(&k_empty[st], ((t / KV_STAGES) & 1) ^ 1);
    mbar_arrive_expect_tx(&k_full[st], kKBytes);
    for (int a = 0; a < KA; ++a)
      tma_load_2d(sK + st * kKBytes + a * BKV * 128, &p.tmK, &k_full[st], p.k_col0 + head * DK + a * 64, b * p.kv_bs + t * BKV);
  };
  auto load_v = [&](int t) {
    const int st = t % KV_STAGES;
    mbar_wait(&v_empty[st], ((t / KV_STAGES) & 1) ^ 1);
    mbar_arrive_expect_tx(&v_full[st], kVBytes);
    for (int a = 0; a < KVA; ++a)
      tma_load_2d(sV + st * kVBytes + a * kVAtom, &p.tmV, &v_full[st], b * p.kv_bs + t * BKV + a * 64, head * DVP);
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
      if (col < p.dv)   // (dv % 8 == 0: the pair never straddles the end)
        *reinterpret_cast<uint32_t*>(orow + col) = pack_bf16x2(o[4 * jj + 2 * i] * inv_l, o[4 * jj + 2 * i + 1] * inv_l);
    }
  }
}

struct AttnArgs {   // what the C ABI received; the tensor maps depend on the kernel variant's kv tile
  const void *Q, *K, *Vt;
  long long ldq, ldk, ldv;
  int B, H, q_bstride, kv_bstride;
};

template <int DK, int DVP, int BKV, int KV_STAGES, bool TMA_WARP, bool VARLEN = false>
static int launch_attention(AttnParams& p, const AttnArgs& a, cudaStream_t stream) {
  constexpr size_t smem = attention_smem_bytes<DK, DVP, BKV, KV_STAGES>();
  // two CTAs per SM need twice the dynamic window plus 1 KB each reserved by the system, within 228 KB
  static_assert(smem <= (TMA_WARP ? 227 * 1024 : 113 * 1024), "attention smem budget");
  auto kernel = attention_kernel<DK, DVP, BKV, KV_STAGES, TMA_WARP, VARLEN>;
  static bool configured = false;
  if (!configured) {
    VDB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    if (!TMA_WARP)   // the second CTA per SM is the point of this form: ask for the whole carveout, not the driver's pick
      VDB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    configured = true;
  }
  int rc = make_tmap_2d(&p.tmQ, a.Q, static_cast<uint64_t>(a.ldq), static_cast<uint64_t>(a.B) * a.q_bstride, a.ldq * 2, 64, kBQ);
  if (rc) return rc;
  rc = make_tmap_2d(&p.tmK, a.K, static_cast<uint64_t>(a.ldk), static_cast<uint64_t>(a.B) * a.kv_bstride, a.ldk * 2, 64, BKV);
  if (rc) return rc;
  rc = make_tmap_2d(&p.tmV, a.Vt, static_cast<uint64_t>(a.B) * a.kv_bstride, static_cast<uint64_t>(a.H) * DVP, a.ldv * 2, 64, DVP);
  if (rc) return rc;
  dim3 grid((p.Nq + kBQ - 1) / kBQ, a.H, a.B);
  VDB_CUDA_CHECK(launch_pdl(kernel, grid, dim3(attention_threads(TMA_WARP)), smem, stream, p));
  count_launch();
  return VDB_OK;
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

// Argument checks and parameter block shared by both entry points; returns VDB_OK or the error status.
static int attention_prepare(const void* Q, long long ldq, int q_col0, const void* K, long long ldk, int k_col0, const void* Vt,
                             long long ldv, void* out, long long ldo, int B, int H, int Nq, int Nk, int q_bstride, int kv_bstride,
                             int d_head, float scale, int causal, AttnParams& p, AttnArgs& a) {
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
  memset(&p, 0, sizeof(p));
  a = AttnArgs{Q, K, Vt, ldq, ldk, ldv, B, H, q_bstride, kv_bstride};
  p.Nq = Nq; p.Nk = Nk; p.q_bs = q_bstride; p.kv_bs = kv_bstride; p.q_col0 = q_col0; p.k_col0 = k_col0; p.dv = d_head; p.causal = causal;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.ldo = ldo;
  return VDB_OK;
}

int vdb_attention_bf16(const void* Q, long long ldq, int q_col0, const void* K, long long ldk, int k_col0,
                       const void* Vt, long long ldv, void* out, long long ldo, int B, int H, int Nq, int Nk,
                       int q_bstride, int kv_bstride, int d_head, float scale, int causal, void* stream) {
  AttnParams p;
  AttnArgs a{};
  const int rc = attention_prepare(Q, ldq, q_col0, K, ldk, k_col0, Vt, ldv, out, ldo, B, H, Nq, Nk, q_bstride, kv_bstride, d_head,
                                   scale, causal, p, a);
  if (rc) return rc;
  const int DK = vdb_attention_dk_pad(d_head), DVP = vdb_attention_dv_pad(d_head);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // d_head <= 80: two CTAs per SM, each within 128 registers and half the shared memory (d_head <= 64: 128-key tiles,
  // 3 / 2 stages; d_head 80: 64-key tiles, 3 stages).  d_head 160 keeps the TMA warp and one CTA per SM: two CTAs' Q and
  // K / V^T stages do not fit; 64-key tiles keep its S + O + P within the register budget.
  if (DK == 64 && DVP == 48) return launch_attention<64, 48, 128, 3, false>(p, a, st);
  if (DK == 64 && DVP == 64) return launch_attention<64, 64, 128, 2, false>(p, a, st);
  if (DK == 128 && DVP == 80) return launch_attention<128, 80, 64, 3, false>(p, a, st);
  if (DK == 192 && DVP == 160) return launch_attention<192, 160, 64, 2, true>(p, a, st);
  return set_error(VDB_ERR_UNSUPPORTED, "attention: no kernel for d_head %d", d_head);
}

int vdb_attention_varlen_bf16(const void* Q, long long ldq, int q_col0, const void* K, long long ldk, int k_col0,
                              const void* Vt, long long ldv, void* out, long long ldo, int B, int H, int Nq, int Nk,
                              int q_bstride, int kv_bstride, int d_head, float scale, int causal, const int* kv_len,
                              void* stream) {
  if (!kv_len || (reinterpret_cast<uintptr_t>(kv_len) & 3))
    return set_error(VDB_ERR_INVALID, "attention_varlen: kv_len must be a non-null, 4-byte aligned device int32 [B]");
  if (causal) return set_error(VDB_ERR_INVALID, "attention_varlen: causal masking together with kv_len is not supported");
  if (vdb_attention_dk_pad(d_head) != 64 || vdb_attention_dv_pad(d_head) != 64)
    return set_error(VDB_ERR_UNSUPPORTED, "attention_varlen: only d_head 64 (BERT) is instantiated, got %d", d_head);
  AttnParams p;
  AttnArgs a{};
  const int rc = attention_prepare(Q, ldq, q_col0, K, ldk, k_col0, Vt, ldv, out, ldo, B, H, Nq, Nk, q_bstride, kv_bstride, d_head,
                                   scale, causal, p, a);
  if (rc) return rc;
  p.kv_len = kv_len;
  return launch_attention<64, 64, 128, 2, false, true>(p, a, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
