// vdb200 — persistent wgmma implicit-GEMM mainloop (sm_90a).
//
// One kernel family serves every GEMM-shaped stage of the Versatile-Diffusion sampling path:
//   * Linear layers and 1x1 convs on NHWC activations (CrossAttention.to_q/k/v/to_out,
//     FeedForward/GEGLU, SpatialTransformer.proj_in/out — reference lib/model_zoo/attention.py:37-64,
//     152-193, 221-266; AutoencoderKL AttnBlock q/k/v/proj_out — autokl_modules.py:150-202),
//   * 3x3 convolutions as implicit GEMM over 9 filter taps (ResBlock in_layers[2]/out_layers[3],
//     Downsample.op, Upsample.conv — openaimodel.py:89-274; VAE ResnetBlock/Downsample/Upsample —
//     autokl_modules.py:42-141), with the 1x1 skip_connection of a channel-changing ResBlock folded
//     in as extra K segments of the same accumulator.
//
// Structure: grid = #SMs (persistent, static round-robin over output tiles), 288 threads:
//   warps 0-7: two consumer warpgroups (wgmma m64 x BN x 16 each, fp32 accumulators in registers), then the epilogue
//              (TMA-store modes: straight from the registers -> bias / LayerNorm / GEGLU / residual -> bf16 TMA stores;
//              other modes: accumulator parked in shared memory -> bias/act/residual -> coalesced bf16 / fp32 stores)
//   warp 8   : TMA producer  (cp.async.bulk.tensor 4D box loads of A, 2D box loads of W)
// smem ring of STAGES x (A 128x64 bf16 | W BNx64 bf16), both 128B-swizzled K-major.
#include "common.cuh"
#include "host_util.h"

namespace vdb {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;  // bf16 elements = 128 B = one swizzle row
constexpr int kMaxA = 6;     // A tensor maps per launch
constexpr int kMaxSeg = 12;  // K segments per launch
// threads = 64 + 32 * EW: warp 0 TMA, warp 1 MMA, EW epilogue warps (8, or 16 for the short-K GEMMs whose tiles
// are bound by the epilogue's instruction latency rather than by the mainloop)
constexpr uint32_t kABytes = kBlockM * kBlockK * 2;

struct ASeg {
  int16_t tmap;  // which A tensor map
  int16_t dw;    // W-coordinate shift of this segment (filter tap / parity lattice)
  int16_t dh;    // H-coordinate shift
  int16_t nkb;   // number of 64-channel k-blocks
  int32_t c0;    // first channel coordinate
};

struct alignas(64) IgemmParams {
  CUtensorMap tmA[kMaxA];  // 4D (C, W, H, B) bf16, box (64, TW, TH, TB), SWIZZLE_128B
  CUtensorMap tmB;         // 2D (Ktot, N) bf16, box (64, BN), SWIZZLE_128B
  CUtensorMap tmO;         // TMA-store epilogues: 4D (N, Wo, Ho, Bo) bf16 output, box (32, bw, bh, bb) = one warp's 16-row x 32-column chunk, SWIZZLE_64B
  ASeg seg[kMaxSeg];
  int nseg;
  int kb_total;      // total k-blocks over all segments
  int ksplit;        // split-K factor (>=1); >1 => fp32 partial output
  int kb_per_split;  // ceil(kb_total / ksplit)
  int TW, TH, TB;    // M tile = TW*TH*TB = 128 output pixels
  int Wo, Ho, Bo;    // output pixel grid (GEMM view: Wo = M, Ho = Bo = 1)
  int tilesW, tilesH, tilesB, tilesN;
  int N;             // valid output columns (GEGLU: packed columns, output has N/2)
  // epilogue
  const float* bias;          // [bias_rows, N] fp32 or null
  long long bias_bstride;     // 0: shared bias row; else stride between per-batch rows
  int rows_per_batch;         // output pixels per batch element (for bias_bstride != 0)
  const __nv_bfloat16* resid; // [M, ldr] bf16 or null (added after activation)
  long long ldr;
  void* out;                  // bf16 or fp32 [M, ldo]
  long long ldo;
  int out_f32;                // 1: fp32 output
  int act;                    // 0 none, 1 silu, 2 gelu(erf), 3 quick_gelu, 4 geglu (packed halves)
  float alpha;                // out = act(alpha * (acc + bias)) + resid
  float* partial;             // split-K: [ksplit, M, N] fp32
  // LayerNorm folded into the GEMM (modes 5 / 6 consume, mode 7 produces; see the epilogue):
  const float* ln_stats;      // [ln_parts][ln_mstat][2] fp32: partial (sum, sum of squares) over column ranges of the normalised rows
  long long ln_mstat;         // rows of the statistics table
  int ln_parts;               // partials per row (what the producer launch reported)
  int ln_on_cols;             // 0: the statistics belong to the OUTPUT ROWS (x is the A operand); 1: to the output COLUMNS (x is B)
  float ln_inv_dim, ln_eps;   // 1 / normalised width, epsilon
  const float* ln_colsum;     // on_cols 0: [N] sum_k W'[n, k];  on_cols 1: [M] (per output row)
  const float* ln_rowbias;    // on_cols 1: [M] beta-term of the output row (null = 0); on_cols 0 the beta term lives in `bias`
  float* stats_out;           // mode 7: [2 * tilesN][M][2] fp32: (sum, sum of squares) over the even (slot 2n) and the odd
                              // (slot 2n + 1) 32-column chunks of N tile n, for every OUTPUT row
  unsigned long long* timeline; // debug: per-tile role timestamps of CTA 0 (null = off)
  unsigned smem_bytes;        // dynamic shared memory of the launch (LN modes check their carve-up against it)
};

enum { ACT_NONE = 0, ACT_SILU = 1, ACT_GELU = 2, ACT_QGELU = 3, ACT_GEGLU = 4 };

#ifdef VDB_TIMELINE   // debug build only (tools/gemm_timeline.py): per-tile role timestamps of CTA 0
#define VDB_TL(slot, it) do { if (p.timeline && blockIdx.x == 0 && (it) < 8) p.timeline[(it) * 16 + (slot)] = gtime(); } while (0)
#define VDB_TLE(slot, it) do { if (warp == 0 && lane == 0) VDB_TL(slot, it); } while (0)
#else
#define VDB_TL(slot, it) do { } while (0)
#define VDB_TLE(slot, it) do { } while (0)
#endif

VDB_DEVINL float apply_act(float v, int act) {
  switch (act) {
    case ACT_SILU: return silu_f(v);
    case ACT_GELU: return gelu_erf_f(v);
    case ACT_QGELU: return quick_gelu_f(v);
    default: return v;
  }
}

// MODE selects the epilogue that is compiled in: 0 = every path (split-K partials, GEGLU, fp32 / ragged / per-row-bias
// tiles), 3 = only the bf16 fast path (act none, alpha 1, N % 32 == 0, one bias row per tile), 4 = only GEGLU, both with the
// tile leaving through shared memory + TMA stores.  Keeping the rarely used paths out of the common instantiations keeps the
// epilogue's instruction footprint small.  Modes 5 / 6 are modes 3 / 4 for a GEMM whose
// input is a LayerNorm: the operand is the RAW activation x and the weights carry gamma (W' = W * gamma), so with the row's mean mu
// and rstd r       LN(x) W^T + b  =  r * (x W'^T  -  mu * s) + c,     s[n] = sum_k W'[n,k],  c[n] = sum_k beta_k W[n,k] + b[n]
// is a rank-1 correction in the epilogue (2 FMAs per element) — the normalised tensor is never written or read.  mu and r come
// from per-32-channel partial sums that the PRODUCER of x wrote from its own epilogue (mode 7 = mode 3 + those sums).  When x is
// the B operand (the transposed V^T projection) the statistics belong to the output columns instead (ln_on_cols).
//
// Roles: warps 0-7 are two consumer warpgroups (warpgroup g computes output rows [64 g, 64 g + 64) of the tile with wgmma, fp32
// accumulators in registers), warp 8 is the TMA producer.
// Modes 3-7 run the epilogue from the registers, in the wgmma fragment layout: warp w owns 16 rows of the tile and walks their
// 32-column chunks, staging each as a 16 x 32 bf16 box (stmatrix) for a TMA store.  The warpgroups do not wait for each other
// after the mainloop, and the producer is gated by the empty barriers alone: it loads the next tile's first STAGES k-blocks while
// the epilogue runs, so the next mainloop starts on a full ring.  tests/test_igemm_protocol_tma_epi.py models this protocol.
// Mode 0 parks the accumulator in shared memory (sacc, [128][BN + 4] fp32, aliasing the operand ring) after the mainloop and
// runs the epilogue on it: each warp reads 32-column chunks of one ROW per thread (acc_ld32), the layout its paths are written
// for.  The producer starts the next tile's loads once every consumer warp is done with sacc (acc_free;
// tests/test_igemm_protocol.py).
template <int BN, int STAGES, int EW, int MODE>
__global__ void __launch_bounds__(32 + 32 * EW, 1) igemm_kernel(const __grid_constant__ IgemmParams p) {
  constexpr bool kTmaEpi = MODE >= 3;                 // TMA-store epilogues
  constexpr bool kGegluEpi = MODE == 4 || MODE == 6;
  constexpr bool kLnIn = MODE == 5 || MODE == 6;
  constexpr bool kStatsOut = MODE == 7;
  constexpr int kNumEpiWarps = EW;
  constexpr int kNumEpiThreads = EW * 32;
  constexpr int kWPQ = EW / 4;           // epilogue warps per 32-row quarter of the tile
  static_assert(EW == 8, "two consumer warpgroups of 64 rows each");
  constexpr uint32_t kBBytes = BN * kBlockK * 2;
  constexpr uint32_t kStageBytes = kABytes + kBBytes;
  constexpr int kAccStride = BN + 4;     // sacc row stride in floats (row-per-thread 16-byte reads are conflict-free)
  constexpr uint32_t kRingBytes = STAGES * kStageBytes;
  constexpr uint32_t kAccBytes = kBlockM * kAccStride * 4;
  constexpr uint32_t kRegion = kRingBytes > kAccBytes ? kRingBytes : kAccBytes;
  static_assert(kBBytes % 1024 == 0, "B stage must keep 1024B alignment");
  static_assert(BN % 32 == 0 && BN >= 32 && BN <= 256, "invalid wgmma N");

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smemA = smem;
  uint8_t* smemB = smem + STAGES * kABytes;
  float* sacc = reinterpret_cast<float*>(smem);                            // [128][kAccStride] fp32 accumulator of the tile
  float* sstage = reinterpret_cast<float*>(smem + kRegion);                // kNumEpiWarps x 4 KB, 1024-byte aligned: [32][32] fp32
                                                                           // transposition tiles, or 2 x 2 KB bf16 TMA-store tiles
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kRegion + EW * 4096);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* acc_free = empty_bar + STAGES;    // [1]
  float* sbias = reinterpret_cast<float*>(acc_free + 2);      // [BN] bias of the current output tile
  float* slnx = sbias + BN;                                   // [BN] LN modes: colsum s (on_cols 0) / column mean (on_cols 1)
  const uint32_t sbias_s = smem_u32(sbias), slnx_s = smem_u32(slnx);   // (shared-space addresses: LDS, not generic LD)
  (void)slnx_s;
  if constexpr (kLnIn) {
    if (reinterpret_cast<uint8_t*>(slnx + BN) > smem_raw + p.smem_bytes) __trap();
  }
  auto epi_bar_sync = [] { asm volatile("bar.sync 1, %0;" ::"n"(EW * 32) : "memory"); };   // the consumer warps only

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == EW && lane == 0) {
    for (int i = 0; i < kMaxA; ++i) tma_prefetch_desc(&p.tmA[i]);
    tma_prefetch_desc(&p.tmB);
    if constexpr (MODE >= 3) tma_prefetch_desc(&p.tmO);
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kNumEpiWarps);
    }
    mbar_init(acc_free, kNumEpiWarps);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();   // everything above overlapped the previous kernel's tail; global inputs are valid from here

  const int tilesM = p.tilesW * p.tilesH * p.tilesB;
  const int unitsM = tilesM;
  const int num_tiles = unitsM * p.tilesN * p.ksplit;
  // Tile walk of this CTA (both roles use the same bounds): tiles c, c + grid, ..., with M as the fast tile index.
  const int t_first = blockIdx.x, t_step = gridDim.x, t_end = num_tiles;

  if (warp == EW) {
    // ------------------------------ TMA producer ------------------------------
    if (lane == 0) {
      uint32_t stage = 0, phase = 0;
      const bool flat = (p.tilesH == 1) && (p.tilesB == 1);
      const int step_m = t_step % unitsM, step_r = t_step / unitsM;
      int unit_m = t_first % unitsM, rest = t_first / unitsM;
      int it = 0;
      for (int t = t_first; t < t_end; t += t_step, ++it) {
        const int m_idx = unit_m;
        int n_idx = rest, ks = 0;
        if (p.ksplit > 1) { n_idx = rest % p.tilesN; ks = rest / p.tilesN; }
        int wt = m_idx, ht = 0, bt = 0;
        if (!flat) {
          wt = m_idx % p.tilesW;
          const int q = m_idx / p.tilesW;
          ht = q % p.tilesH;
          bt = q / p.tilesH;
        }
        unit_m += step_m; rest += step_r;
        if (unit_m >= unitsM) { unit_m -= unitsM; ++rest; }
        const int w0 = wt * p.TW, h0 = ht * p.TH, b0 = bt * p.TB;
        const int n0 = n_idx * BN;
        const int kb_begin = ks * p.kb_per_split;
        const int kb_end = min(p.kb_total, kb_begin + p.kb_per_split);
        int kb = 0;
        // mode 0: the ring holds the previous tile's accumulator until its epilogue ends.  The TMA-store modes keep it in
        // registers, so only the empty barriers gate the ring and the next tile's first STAGES k-blocks load during the epilogue.
        if (!kTmaEpi && it > 0) mbar_wait(acc_free, (it - 1) & 1);
        VDB_TL(0, it);   // producer: starts issuing this tile
        for (int s = 0; s < p.nseg; ++s) {
          const ASeg sg = p.seg[s];
          if (kb + sg.nkb <= kb_begin) { kb += sg.nkb; continue; }
          for (int j = 0; j < sg.nkb; ++j, ++kb) {
            if (kb < kb_begin) continue;
            if (kb >= kb_end) break;
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
            tma_load_4d(smemA + stage * kABytes, &p.tmA[sg.tmap], &full_bar[stage],
                        sg.c0 + j * kBlockK, w0 + sg.dw, h0 + sg.dh, b0);
            tma_load_2d(smemB + stage * kBBytes, &p.tmB, &full_bar[stage], kb * kBlockK, n0);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
          if (kb >= kb_end) break;
        }
      }
    }
  } else {
    // ------------------------------ consumers: wgmma mainloop, then the epilogue ------------------------------
    // Epilogue: warps w and w+4 own the same 32-row quarter of the tile (w & 3) and alternate 32-column chunks.
    // acc_ld32 hands each thread one ROW of 32 columns; the transposing paths write the raw fp32 block to a private
    // XOR-swizzled 4 KB shared-memory tile and read it back transposed, so every global access is 8 rows x 64 contiguous
    // bytes per instruction (4 lanes per row), and bias / activation / residual / bf16 conversion run on 8 fixed columns
    // per lane (bias lives in registers).
    const int quarter = warp & 3;          // 32-row quarter of the tile
    const int half = warp >> 2;            // which of the kWPQ warps of the quarter
    const int r = quarter * 32 + lane;
    const int tr_row = lane >> 2, tr_q = lane & 3;   // transposed role: rows tr_row + 8k, columns tr_q*8 .. +7
    float* stage = sstage + warp * 1024;             // [32 rows][32 fp32], 16-byte chunk j of row i at (j ^ (i & 7))
    const uint32_t sacc_row = smem_u32(sacc) + static_cast<uint32_t>(r * kAccStride * 4);
    auto acc_ld32 = [&](int col, uint32_t (&v)[32]) {   // row r, columns [col, col + 32) of the parked accumulator
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 x = lds_f4(sacc_row + (col + 4 * i) * 4);
        v[4 * i] = __float_as_uint(x.x); v[4 * i + 1] = __float_as_uint(x.y);
        v[4 * i + 2] = __float_as_uint(x.z); v[4 * i + 3] = __float_as_uint(x.w);
      }
    };
    // mainloop of one tile: warpgroup g multiplies its 64 rows of A by the BN x 64 B tile of every k-block, then (modes 0-2)
    // both warpgroups park the accumulator in sacc
    uint32_t ml_stage = 0, ml_phase = 0;
    float acc[BN / 2];
    auto mainloop = [&](int kb_begin, int kb_end) {
      const int g = warp >> 2;
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      uint32_t prev = 0;
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&full_bar[ml_stage], ml_phase);
        wgmma_fence();
        const uint64_t adesc = make_desc_sw128(smem_u32(smemA + ml_stage * kABytes + g * (64 * 128)));
        const uint64_t bdesc = make_desc_sw128(smem_u32(smemB + ml_stage * kBBytes));
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) wgmma_ss<BN>(acc, adesc + 2 * k, bdesc + 2 * k, (kb > kb_begin || k > 0) ? 1u : 0u);
        wgmma_commit();
        if (kb > kb_begin) {            // the previous k-block's MMAs have read their stage: hand it back to the producer
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = ml_stage;
        if (++ml_stage == STAGES) { ml_stage = 0; ml_phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      __syncwarp();
      if (lane == 0 && kb_end > kb_begin) mbar_arrive(&empty_bar[prev]);
      if constexpr (!kTmaEpi) {
        epi_bar_sync();                 // sacc aliases the ring: both warpgroups' MMAs have finished reading it
        float* srow = sacc + (g * 64 + (warp & 3) * 16 + (lane >> 2)) * kAccStride + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          *reinterpret_cast<float2*>(srow + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(srow + 8 * kAccStride + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        epi_bar_sync();
      }
    };
    auto stage_write = [&](const uint32_t (&v)[32]) {
      float* srow = stage + lane * 32;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<uint4*>(srow + ((j ^ (lane & 7)) << 2)) = make_uint4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    };
    auto stage_read = [&](int k, float (&o)[8]) {   // row tr_row + 8k, columns tr_q*8 .. +7
      const int row = k * 8 + tr_row;
      const float* srow = stage + row * 32;
      const float4 x0 = *reinterpret_cast<const float4*>(srow + (((2 * tr_q) ^ (row & 7)) << 2));
      const float4 x1 = *reinterpret_cast<const float4*>(srow + (((2 * tr_q + 1) ^ (row & 7)) << 2));
      o[0] = x0.x; o[1] = x0.y; o[2] = x0.z; o[3] = x0.w; o[4] = x1.x; o[5] = x1.y; o[6] = x1.z; o[7] = x1.w;
    };
    int it = 0;
    int st_buf = 0;                     // TMA-store epilogues: which of this warp's four staging boxes is written next
    (void)st_buf;
    const float* sbias_src = nullptr;   // which bias row/offset currently sits in sbias
    // The per-tile bookkeeping sits on the critical path of epilogue-bound GEMMs (it was ~0.75 us of every ~3.6 us
    // tile): the tile index advances incrementally (no divisions in the GEMM view), row indices are 32-bit, and
    // everything that depends only on the thread is hoisted.
    const int tw = r % p.TW;
    const int th = (r / p.TW) % p.TH;
    const int tb = r / (p.TW * p.TH);
    const bool flat = (p.tilesH == 1) && (p.tilesB == 1);   // GEMM view: M tiles along W only
    const int step_m = t_step % unitsM, step_r = t_step / unitsM;
    int unit_m = t_first % unitsM, rest = t_first / unitsM;
    // TMA-store epilogues: the accumulator stays in the wgmma fragment layout, so warp w owns the 16 tile rows from e_row0 on
    // (warpgroup w / 4, quarter w % 4) and this thread rows e_row0 + lane / 4 and e_row0 + lane / 4 + 8, at columns
    // 8 j + 2 (lane % 4) + {0, 1}
    const int e_row0 = (warp >> 2) * 64 + (warp & 3) * 16;
    int e_tw[2], e_th[2], e_tb[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int er = e_row0 + (lane >> 2) + 8 * h;
      e_tw[h] = er % p.TW; e_th[h] = (er / p.TW) % p.TH; e_tb[h] = er / (p.TW * p.TH);
    }
    // folded LayerNorm, row statistics: partial sums of the warp's rows in the NEXT tile, requested a tile ahead.  Lane l serves
    // row e_row0 + l % 16: lanes 0-15 load partials 0-7, lanes 16-31 partials 8-15 of the same rows (kLnPre each)
    constexpr int kLnPre = 8;
    float2 ln_pre[kLnIn ? kLnPre : 1];
    auto ln_prefetch = [&](int row) {
      if constexpr (kLnIn) {
        const bool ok = row < p.Wo;
        const int i0 = (lane >> 4) * kLnPre;
#pragma unroll
        for (int i = 0; i < kLnPre; ++i)
          ln_pre[i] = (ok && i0 + i < p.ln_parts)
                          ? __ldg(reinterpret_cast<const float2*>(p.ln_stats) + static_cast<long long>(i0 + i) * p.ln_mstat + row)
                          : make_float2(0.f, 0.f);
      }
    };
    if constexpr (kLnIn) {
      if (!p.ln_on_cols && p.ln_parts <= 2 * kLnPre && t_first < t_end) ln_prefetch((t_first % unitsM) * kBlockM + e_row0 + (lane & 15));
    }
    for (int t = t_first; t < t_end; t += t_step, ++it) {
      const int m_idx = unit_m;
      int n_idx = rest, ks = 0;
      if (p.ksplit > 1) { n_idx = rest % p.tilesN; ks = rest / p.tilesN; }
      int wt = m_idx, ht = 0, bt = 0;
      if (!flat) {
        wt = m_idx % p.tilesW;
        const int q = m_idx / p.tilesW;
        ht = q % p.tilesH;
        bt = q / p.tilesH;
      }
      unit_m += step_m; rest += step_r;
      if (unit_m >= unitsM) { unit_m -= unitsM; ++rest; }
      const int w = wt * p.TW + tw, h = ht * p.TH + th, b = bt * p.TB + tb;
      const bool row_ok = (w < p.Wo) && (h < p.Ho) && (b < p.Bo);
      const int gp = (b * p.Ho + h) * p.Wo + w;     // output pixel (row of the GEMM); host guarantees M < 2^31
      const int gp_first = ((bt * p.TB) * p.Ho + ht * p.TH) * p.Wo + wt * p.TW;
      const int n0 = n_idx * BN;

      // per-tile row bookkeeping for the transposed role (independent of the accumulator: done before the wait)
      int gp_k[4];
      bool ok_k[4];
      if constexpr (!kTmaEpi) {
        const unsigned okmask = __ballot_sync(0xffffffffu, row_ok);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int src = k * 8 + tr_row;
          gp_k[k] = __shfl_sync(0xffffffffu, gp, src);
          ok_k[k] = (okmask >> src) & 1u;
        }
      }
      // bias tile -> shared memory (one global read per tile); one row serves the tile unless the bias is per-batch
      // and the tile's first / last rows belong to different batch items
      const int gp_last = ((bt * p.TB + p.TB - 1) * p.Ho + ht * p.TH + p.TH - 1) * p.Wo + wt * p.TW + p.TW - 1;
      const bool bias_uniform = (MODE != 0) ? (p.bias != nullptr)    // host: a tile never straddles two bias rows
                                            : (p.bias && p.ksplit == 1 &&
                                               (p.bias_bstride == 0 || gp_first / p.rows_per_batch == gp_last / p.rows_per_batch));
      if constexpr (kLnIn) {
        // folded-LayerNorm tiles: sbias = c[n] (beta term + bias), slnx = s[n]; or, when the statistics belong to the
        // columns, sbias = rstd[n], slnx = mean[n] computed here from the producer's partial sums (one column per thread)
        const float* key = reinterpret_cast<const float*>(static_cast<uintptr_t>(n0) + 1);
        if (key != sbias_src) {
          epi_bar_sync();
          for (int i = threadIdx.x; i < BN; i += kNumEpiThreads) {
            const int n = n0 + i;
            float a = 0.f, b = 0.f;
            if (n < p.N) {
              if (p.ln_on_cols) {
                float su = 0.f, sq = 0.f;
#pragma unroll 8
                for (int ch = 0; ch < p.ln_parts; ++ch) {
                  const float2 v = __ldg(reinterpret_cast<const float2*>(p.ln_stats) + static_cast<long long>(ch) * p.ln_mstat + n);
                  su += v.x; sq += v.y;
                }
                const float mu = su * p.ln_inv_dim;
                a = mu;
                b = rsqrtf(fmaxf(sq * p.ln_inv_dim - mu * mu, 0.f) + p.ln_eps);
              } else {
                a = __ldg(p.ln_colsum + n);
                b = p.bias ? __ldg(p.bias + n) : 0.f;
              }
            }
            slnx[i] = a;
            sbias[i] = b;
          }
          epi_bar_sync();
          sbias_src = key;
        }
      } else if (bias_uniform) {
        // consecutive tiles of a CTA usually share the N tile (M is the fast tile index): reload only on change,
        // otherwise the ~0.7 us global-load latency + two barriers sit between every two tiles
        const float* brow = p.bias + (p.bias_bstride ? static_cast<long long>(gp_first / p.rows_per_batch) * p.bias_bstride : 0) + n0;
        if (brow != sbias_src) {              // uniform across the epilogue threads
          epi_bar_sync();                     // previous tile's readers are done with sbias
          for (int i = threadIdx.x; i < BN; i += kNumEpiThreads) sbias[i] = (n0 + i < p.N) ? __ldg(brow + i) : 0.f;
          epi_bar_sync();
          sbias_src = brow;
        }
      }
      const float* bias_g = (p.bias && !bias_uniform)
                                ? p.bias + (p.bias_bstride ? static_cast<long long>(gp / p.rows_per_batch) * p.bias_bstride : 0) : nullptr;

      const int f_nchunks = min(BN / 32, (p.N - n0) / 32);
      const bool has_resid = p.resid != nullptr;

      // TMA-store epilogues: output pixels (GEMM rows) of this thread's two accumulator rows
      int e_gp[2];
      bool e_ok[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ew = wt * p.TW + e_tw[h], eh = ht * p.TH + e_th[h], eb = bt * p.TB + e_tb[h];
        e_ok[h] = (ew < p.Wo) && (eh < p.Ho) && (eb < p.Bo);
        e_gp[h] = (eb * p.Ho + eh) * p.Wo + ew;
      }
      // folded LayerNorm: the scalars of this thread's two rows (requested before the accumulator wait)
      float ln_a0[2] = {0.f, 0.f}, ln_a1[2] = {1.f, 1.f};   // on_cols 0: (mean, rstd) of the row;  on_cols 1: (s[m], c[m]) of the output row
      if constexpr (kLnIn) {
        if (p.ln_on_cols) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (e_ok[h]) {
              ln_a0[h] = __ldg(p.ln_colsum + e_gp[h]);
              ln_a1[h] = p.ln_rowbias ? __ldg(p.ln_rowbias + e_gp[h]) : 0.f;
            }
          }
        } else {
          // lane l sums the partials of row e_row0 + l % 16 in the order 0, 1, 2, ... and hands mean and rstd to the two lanes that
          // hold the row (lanes 16-31 compute nothing useful)
          float su = 0.f, sq = 0.f;
          if (p.ln_parts <= 2 * kLnPre) {
            // the partials of THIS tile's rows were requested one tile ago (ln_pre): a tile's own request would sit on the
            // critical path of every epilogue-bound tile (first version: +75 % on the K = 320 GEMMs)
#pragma unroll
            for (int i = 0; i < kLnPre; ++i) { su += ln_pre[i].x; sq += ln_pre[i].y; }
#pragma unroll
            for (int i = 0; i < kLnPre; ++i) {
              su += __shfl_sync(0xffffffffu, ln_pre[i].x, lane | 16);
              sq += __shfl_sync(0xffffffffu, ln_pre[i].y, lane | 16);
            }
          } else {
            const int row = m_idx * kBlockM + e_row0 + (lane & 15);
            if (row < p.Wo) {
#pragma unroll 8
              for (int ch = 0; ch < p.ln_parts; ++ch) {
                const float2 v = __ldg(reinterpret_cast<const float2*>(p.ln_stats) + static_cast<long long>(ch) * p.ln_mstat + row);
                su += v.x; sq += v.y;
              }
            }
          }
          const float mu = su * p.ln_inv_dim;
          const float rs = rsqrtf(fmaxf(sq * p.ln_inv_dim - mu * mu, 0.f) + p.ln_eps);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            ln_a0[h] = __shfl_sync(0xffffffffu, mu, (lane >> 2) + 8 * h);
            ln_a1[h] = __shfl_sync(0xffffffffu, rs, (lane >> 2) + 8 * h);
          }
        }
        // request the next tile's row partials (GEMM view, M-fast order: unit_m already points at the next tile)
        if (!p.ln_on_cols && p.ln_parts <= 2 * kLnPre && t + t_step < t_end) ln_prefetch(unit_m * kBlockM + e_row0 + (lane & 15));
      }
      VDB_TLE(4, it);   // consumers: mainloop starts
      mainloop(ks * p.kb_per_split, min(p.kb_total, ks * p.kb_per_split + p.kb_per_split));
      VDB_TLE(5, it);   // consumers: accumulator parked

      auto geglu_tile = [&] {
        // packed tile: columns [0,BN/2) = value rows, [BN/2,BN) = gate rows of the same outputs
        constexpr int HALF = BN / 2;
        const int nout0 = n_idx * HALF;
        const int Nout = p.N / 2;
#pragma unroll 1
        for (int c = (((HALF / 32) % kWPQ) != 0) ? ((half + it) % kWPQ) : half; c < HALF / 32; c += kWPQ) {
          uint32_t v[32];
          float a[4][8];
          acc_ld32(c * 32, v);
          stage_write(v);
          __syncwarp();
#pragma unroll
          for (int k = 0; k < 4; ++k) stage_read(k, a[k]);
          __syncwarp();
          acc_ld32(HALF + c * 32, v);
          stage_write(v);
          __syncwarp();
          float bv[8], bg[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            bv[i] = p.bias ? sbias[c * 32 + tr_q * 8 + i] : 0.f;
            bg[i] = p.bias ? sbias[HALF + c * 32 + tr_q * 8 + i] : 0.f;
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            float g[8];
            stage_read(k, g);
            if (ok_k[k] && nout0 + c * 32 + tr_q * 8 + 7 < Nout) {
              float o[8];
#pragma unroll
              for (int i = 0; i < 8; ++i) o[i] = (a[k][i] + bv[i]) * gelu_fast_f(g[i] + bg[i]);
              *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + static_cast<long long>(gp_k[k]) * p.ldo + nout0 + c * 32 + tr_q * 8) =
                  make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
            }
          }
          __syncwarp();
        }
      };
      if constexpr (kTmaEpi) {
        // ---- TMA-store epilogues, straight from the wgmma registers (no park, no barrier between the warpgroups).  Each warp
        // walks the 32-column chunks of its 16 rows: per-element fp32 arithmetic on the thread's 2 rows x 8 columns of the chunk,
        // bf16 pack, two stmatrix into one 1 KB staging box of this warp (16 rows of 64 B, SWIZZLE_64B pattern), then lane 0
        // hands the box to the TMA unit (cp.async.bulk.tensor store; out-of-range rows / columns are clipped by the tensor
        // map).  Four boxes per warp rotate: a box is rewritten once the store issued from it three chunks ago has read it.
        // Bias / LayerNorm tables are read from shared memory as 8-byte broadcasts (columns 2 (lane % 4) + {0, 1}).
        const uint32_t stg_s = smem_u32(sstage) + warp * 4096;
        const int ow = wt * p.TW + (e_row0 % p.TW), oh = ht * p.TH + ((e_row0 / p.TW) % p.TH), ob = bt * p.TB + e_row0 / (p.TW * p.TH);
        constexpr int OUTC = kGegluEpi ? BN / 2 : BN;                    // output columns per tile
        const int ochunks = kGegluEpi ? OUTC / 32 : f_nchunks;
        const int ocol0 = n_idx * OUTC;
        const int tq2 = 2 * (lane & 3);                                  // this thread's first column of every 8-column group
        // residual (modes 3 / 7): the thread's 2 bf16 of row h and 8-column group jj of a chunk, one 4-byte load each,
        // requested a chunk ahead
        const bool do_resid = (MODE == 3 || MODE == 7) && has_resid;
        const uint32_t* rrow[2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
          rrow[h] = (do_resid && e_ok[h]) ? reinterpret_cast<const uint32_t*>(p.resid + static_cast<long long>(e_gp[h]) * p.ldr + ocol0 + tq2)
                                          : nullptr;
        auto load_resid = [&](int c, uint32_t (&rr)[2][4]) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) rr[h][jj] = rrow[h] ? __ldg(rrow[h] + (c * 32 + 8 * jj) / 2) : 0u;
        };
        uint32_t rr[2][4];
        if (do_resid) load_resid(0, rr);
        float st_su[2][2] = {{0.f, 0.f}, {0.f, 0.f}}, st_sq[2][2] = {{0.f, 0.f}, {0.f, 0.f}};   // mode 7: [row][chunk parity]
        (void)st_su; (void)st_sq;
        float nrm[2];                                                    // LN rows: -rstd * mean of the row
#pragma unroll
        for (int h = 0; h < 2; ++h) nrm[h] = -ln_a1[h] * ln_a0[h];
        (void)nrm;
#pragma unroll
        for (int c = 0; c < OUTC / 32; ++c) {
          if (c >= ochunks) break;
          float o[4][2][2];                                              // [8-column group][row][column]
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int n = c * 32 + 8 * jj + tq2;                         // tile column of o[jj][.][0]
            const float* va = acc + 4 * (4 * c + jj);                    // {row 0: n, n + 1; row 8: n, n + 1}
            if constexpr (kGegluEpi) {
              const float* vg = acc + 4 * (BN / 16 + 4 * c + jj);        // gate columns OUTC + n
              if constexpr (kLnIn) {   // GEGLU over a folded LayerNorm: r * (acc - mu * s) + c == fma(r, acc, fma(-r mu, s, c))
                const float2 sa = lds_f2(slnx_s + 4 * n), ca = lds_f2(sbias_s + 4 * n);
                const float2 sg = lds_f2(slnx_s + 4 * (OUTC + n)), cg = lds_f2(sbias_s + 4 * (OUTC + n));
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  o[jj][h][0] = fmaf(ln_a1[h], va[2 * h], fmaf(nrm[h], sa.x, ca.x)) * gelu_fast_f(fmaf(ln_a1[h], vg[2 * h], fmaf(nrm[h], sg.x, cg.x)));
                  o[jj][h][1] = fmaf(ln_a1[h], va[2 * h + 1], fmaf(nrm[h], sa.y, ca.y)) * gelu_fast_f(fmaf(ln_a1[h], vg[2 * h + 1], fmaf(nrm[h], sg.y, cg.y)));
                }
              } else {
                const float2 ba = p.bias ? lds_f2(sbias_s + 4 * n) : make_float2(0.f, 0.f);
                const float2 bg = p.bias ? lds_f2(sbias_s + 4 * (OUTC + n)) : make_float2(0.f, 0.f);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  o[jj][h][0] = (va[2 * h] + ba.x) * gelu_fast_f(vg[2 * h] + bg.x);
                  o[jj][h][1] = (va[2 * h + 1] + ba.y) * gelu_fast_f(vg[2 * h + 1] + bg.y);
                }
              }
            } else if constexpr (kLnIn) {
              if (p.ln_on_cols) {      // out = rstd[n] * (acc - mean[n] * s[m]) + c[m]
                const float2 mu = lds_f2(slnx_s + 4 * n), rs = lds_f2(sbias_s + 4 * n);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  o[jj][h][0] = fmaf(rs.x, fmaf(mu.x, -ln_a0[h], va[2 * h]), ln_a1[h]);
                  o[jj][h][1] = fmaf(rs.y, fmaf(mu.y, -ln_a0[h], va[2 * h + 1]), ln_a1[h]);
                }
              } else {                 // out = rstd[m] * (acc - mean[m] * s[n]) + c[n] == fma(r, acc, fma(-r mu, s, c))
                const float2 sx = lds_f2(slnx_s + 4 * n), cx = lds_f2(sbias_s + 4 * n);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  o[jj][h][0] = fmaf(ln_a1[h], va[2 * h], fmaf(nrm[h], sx.x, cx.x));
                  o[jj][h][1] = fmaf(ln_a1[h], va[2 * h + 1], fmaf(nrm[h], sx.y, cx.y));
                }
              }
            } else {                   // modes 3 / 7: acc + bias, then + residual
              const float2 bb = p.bias ? lds_f2(sbias_s + 4 * n) : make_float2(0.f, 0.f);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                o[jj][h][0] = va[2 * h] + bb.x;
                o[jj][h][1] = va[2 * h + 1] + bb.y;
              }
            }
          }
          if (do_resid) {
            uint32_t rn[2][4];
            const bool more = c + 1 < ochunks;
            if (more) load_resid(c + 1, rn);
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const float2 x = unpack_bf16x2(rr[h][jj]);
                o[jj][h][0] += x.x;
                o[jj][h][1] += x.y;
              }
            if (more) {
#pragma unroll
              for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) rr[h][jj] = rn[h][jj];
            }
          }
          if constexpr (kStatsOut) {
            // LayerNorm statistics of the rows this GEMM produces (fp32, before the rounding), split by chunk parity
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  st_su[h][c & 1] += o[jj][h][e];
                  st_sq[h][c & 1] = fmaf(o[jj][h][e], o[jj][h][e], st_sq[h][c & 1]);
                }
          }
          // the box about to be rewritten was handed to the TMA unit three chunks ago: wait until it has been read
          if (lane == 0) bulk_wait_read<3>();
          __syncwarp();
          const uint32_t box = stg_s + st_buf * 1024;
          {
            // stmatrix x4 per 16 columns: matrix i = rows (i & 1) * 8 + 0..7 of 16-byte unit 2 u + i / 2; lane l addresses row
            // l % 8 of matrix l / 8.  SWIZZLE_64B: unit q of box row rr sits at unit q ^ ((rr / 2) % 4)
            const int mi = lane >> 3, brow = (mi & 1) * 8 + (lane & 7);
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int unit = 2 * u + (mi >> 1);
              stmatrix_x4(box + brow * 64 + ((unit ^ ((brow >> 1) & 3)) << 4),
                          pack_bf16x2(o[2 * u][0][0], o[2 * u][0][1]), pack_bf16x2(o[2 * u][1][0], o[2 * u][1][1]),
                          pack_bf16x2(o[2 * u + 1][0][0], o[2 * u + 1][0][1]), pack_bf16x2(o[2 * u + 1][1][0], o[2 * u + 1][1][1]));
            }
          }
          fence_proxy_async_smem();      // every writer: generic-proxy stores -> visible to the TMA (async proxy) read
          __syncwarp();
          if (lane == 0) {
            tma_store_4d(&p.tmO, reinterpret_cast<const uint8_t*>(sstage) + warp * 4096 + st_buf * 1024, ocol0 + c * 32, ow, oh, ob);
            bulk_commit();
          }
          st_buf = (st_buf + 1) & 3;
        }
        if constexpr (kStatsOut) {
          // one (sum, sum of squares) per row, N tile and chunk parity: slot 2 n_idx + parity of [2 tilesN][M][2].  The four lanes
          // of a row reduce over the quad; a parity without chunks writes zeros
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int par = 0; par < 2; ++par) {
              float su = st_su[h][par], sq = st_sq[h][par];
              su += __shfl_xor_sync(0xffffffffu, su, 1); sq += __shfl_xor_sync(0xffffffffu, sq, 1);
              su += __shfl_xor_sync(0xffffffffu, su, 2); sq += __shfl_xor_sync(0xffffffffu, sq, 2);
              if ((lane & 3) == 0 && e_ok[h])
                reinterpret_cast<float2*>(p.stats_out)[static_cast<long long>(n_idx * 2 + par) * (static_cast<long long>(p.Bo) * p.Ho * p.Wo) + e_gp[h]] =
                    make_float2(su, sq);
            }
        }
      } else if (p.ksplit > 1) {
        // fp32 partials, reduced (+bias/act/residual) by splitk_reduce_kernel
        const long long Mtot = static_cast<long long>(p.Bo) * p.Ho * p.Wo;
        float* dst = p.partial + (static_cast<long long>(ks) * Mtot + gp) * p.N + n0;
#pragma unroll 1
        for (int c = half; c < BN / 32; c += kWPQ) {
          if (n0 + c * 32 >= p.N) break;
          uint32_t v[32];
          acc_ld32(c * 32, v);
          if (row_ok) {
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const int n = n0 + c * 32 + j;
              if (n + 3 < p.N) {
                *reinterpret_cast<float4*>(dst + c * 32 + j) =
                    make_float4(__uint_as_float(v[j]), __uint_as_float(v[j + 1]),
                                __uint_as_float(v[j + 2]), __uint_as_float(v[j + 3]));
              } else {
                for (int q = 0; q < 4; ++q)
                  if (n + q < p.N) dst[c * 32 + j + q] = __uint_as_float(v[j + q]);
              }
            }
          }
        }
      } else if (p.act == ACT_GEGLU) {
        geglu_tile();
      } else {
        const int nchunks = min(BN / 32, (p.N - n0 + 31) / 32);
        auto chunk = [&](int c, const uint32_t (&v)[32], const uint4 (&rr)[4], bool fast) {
          const int nb = n0 + c * 32;
          if (fast) {
            stage_write(v);
            __syncwarp();
            if (c == half) VDB_TLE(8, it);
            float bb[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) bb[i] = p.bias ? sbias[c * 32 + tr_q * 8 + i] : 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              float o[8];
              stage_read(k, o);
              if (ok_k[k]) {
#pragma unroll
                for (int i = 0; i < 8; ++i) o[i] += bb[i];
                if (p.alpha != 1.f) {
#pragma unroll
                  for (int i = 0; i < 8; ++i) o[i] *= p.alpha;
                }
                if (p.act != ACT_NONE) {
#pragma unroll
                  for (int i = 0; i < 8; ++i) o[i] = apply_act(o[i], p.act);
                }
                if (p.resid) {
                  const uint32_t w4[4] = {rr[k].x, rr[k].y, rr[k].z, rr[k].w};
#pragma unroll
                  for (int q = 0; q < 4; ++q) {
                    const float2 x = unpack_bf16x2(w4[q]);
                    o[2 * q] += x.x;
                    o[2 * q + 1] += x.y;
                  }
                }
                *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + static_cast<long long>(gp_k[k]) * p.ldo + nb + tr_q * 8) =
                    make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
              }
              if (c == half && k == 0) VDB_TLE(9, it);
            }
            __syncwarp();   // the tile is rewritten by this warp's next chunk
            if (c == half) VDB_TLE(10, it);
          } else if (row_ok) {
            // slow path (fp32 output, partial last chunk, per-row bias): one row per thread
            float f[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] = __uint_as_float(v[j]);
            if (p.bias) {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (nb + j < p.N) f[j] += bias_uniform ? sbias[c * 32 + j] : __ldg(bias_g + nb + j);
            }
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] = apply_act(f[j] * p.alpha, p.act);
            if (p.resid) {
              const __nv_bfloat16* rs = p.resid + static_cast<long long>(gp) * p.ldr + nb;
#pragma unroll
              for (int j = 0; j < 32; ++j) if (nb + j < p.N) f[j] += __bfloat162float(rs[j]);
            }
            if (p.out_f32) {
              float* dst = reinterpret_cast<float*>(p.out) + static_cast<long long>(gp) * p.ldo + nb;
#pragma unroll
              for (int j = 0; j < 32; ++j) if (nb + j < p.N) dst[j] = f[j];
            } else {
              __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.out) + static_cast<long long>(gp) * p.ldo + nb;
#pragma unroll
              for (int j = 0; j < 32; ++j) if (nb + j < p.N) dst[j] = __float2bfloat16(f[j]);
            }
          }
        };
        auto is_fast = [&](int c) { return (n0 + c * 32 + 32 <= p.N) && !p.out_f32 && (bias_uniform || !p.bias); };
        auto load_resid = [&](int c, uint4 (&rr)[4]) {
          if (p.resid && is_fast(c)) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
              if (ok_k[k]) rr[k] = __ldg(reinterpret_cast<const uint4*>(p.resid + static_cast<long long>(gp_k[k]) * p.ldr + n0 + c * 32 + tr_q * 8));
          }
        };
        // this warp's chunks: half, half+2, ... (kept un-pipelined: double-buffering the 32-register accumulator chunk
        // pushed the kernel into spills and was measured slower)
        // chunk count not a multiple of the warps per quarter (BN = 160: five): rotate who takes the extra chunk
        const int first = (((BN / 32) % kWPQ) != 0) ? ((half + it) % kWPQ) : half;
#pragma unroll 1
        for (int c = first; c < nchunks; c += kWPQ) {
          uint4 rr[4];
          load_resid(c, rr);          // residual loads are in flight while the accumulator chunk is fetched
          uint32_t v[32];
          acc_ld32(c * 32, v);
          if (c == first) VDB_TLE(7, it);
          chunk(c, v, rr, is_fast(c));
        }
      }
      if constexpr (!kTmaEpi) {
        fence_proxy_async_smem();      // this warp's sacc reads are ordered before the producer's next TMA writes
        __syncwarp();
        VDB_TLE(6, it);   // epilogue: tile stored (this warp)
        if (lane == 0) mbar_arrive(acc_free);
      }
    }
    if constexpr (MODE >= 3) {
      if (lane == 0) bulk_wait<0>();     // every TMA store of this thread has completed before the CTA may exit
    }
  }
}

// split-K reduction + epilogue: out[m, n] = act(alpha * (sum_s partial[s, m, n] + bias)) + resid
__global__ void splitk_reduce_kernel(const float* __restrict__ partial, int ksplit, long long M, int N,
                                     const float* __restrict__ bias, long long bias_bstride, int rows_per_batch,
                                     const __nv_bfloat16* __restrict__ resid, long long ldr, void* out,
                                     long long ldo, int out_f32, int act, float alpha) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = M * (N / 4);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long m = i / (N / 4);
    const int n = static_cast<int>(i % (N / 4)) * 4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    // (one partial per iteration on purpose: with all ksplit loads of a thread in flight at once — addresses M*N*4 bytes apart —
    // the 8x8-level convs were measured slower per launch)
    for (int s = 0; s < ksplit; ++s) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(partial + (static_cast<long long>(s) * M + m) * N + n));
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    float f[4] = {acc.x, acc.y, acc.z, acc.w};
    if (bias) {
      const float* bp = bias + (bias_bstride ? (m / rows_per_batch) * bias_bstride : 0) + n;
      for (int q = 0; q < 4; ++q) f[q] += __ldg(bp + q);
    }
    for (int q = 0; q < 4; ++q) f[q] *= alpha;
    for (int q = 0; q < 4; ++q) f[q] = apply_act(f[q], act);
    if (resid) {
      for (int q = 0; q < 4; ++q) f[q] += __bfloat162float(resid[m * ldr + n + q]);
    }
    if (out_f32) {
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + m * ldo + n) = make_float4(f[0], f[1], f[2], f[3]);
    } else {
      uint2 o = make_uint2(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]));
      *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + m * ldo + n) = o;
    }
  }
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------
template <int BN, int STAGES, int EW, int MODE>
static int launch_igemm(const IgemmParams& p0, int num_units, cudaStream_t stream) {
  constexpr bool kLn = MODE == 5 || MODE == 6;       // one more [BN] fp32 table (colsum / column mean)
  constexpr size_t ring = STAGES * (kABytes + BN * kBlockK * 2), acc = kBlockM * (BN + 4) * 4;   // (see igemm_kernel)
  constexpr size_t need = (ring > acc ? ring : acc) + (2 * STAGES + 2) * 8 + BN * 4 + (kLn ? BN * 4 : 0) + EW * 4096;
  // + up to 1024 bytes of slack for the 1024-byte alignment of the operand ring (the LN modes at BN 256 may get less: the dynamic
  // window starts 1024-aligned in practice, and the kernel traps if its carve-up would not fit)
  constexpr size_t smem = (need + 1024 <= 227 * 1024) ? need + 1024 : 227 * 1024;
  static_assert(need + 896 <= 227 * 1024, "igemm shared-memory budget");
  constexpr int threads = 32 + 32 * EW;
  IgemmParams p = p0;
  p.smem_bytes = static_cast<unsigned>(smem);
  static bool configured = false;
  if (!configured) {
    VDB_CUDA_CHECK(cudaFuncSetAttribute(igemm_kernel<BN, STAGES, EW, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(smem)));
    configured = true;
  }
  const int grid = std::min(num_units, num_sms());
  VDB_CUDA_CHECK(launch_pdl(igemm_kernel<BN, STAGES, EW, MODE>, dim3(grid), dim3(threads), smem, stream, p));
  count_launch();
  return VDB_OK;
}

static int pick_bn(int N, int act, int forced) {
  if (forced) return forced;
  if (act == ACT_GEGLU) return 256;
  if (N <= 64) return 64;
  if (N % 256 == 0) return 256;
  if (N % 160 == 0) return 160;
  if (N % 128 == 0) return 128;
  if (N <= 128) return 128;
  if (N <= 160) return 160;
  return 256;
}

static unsigned long long* g_timeline = nullptr;

// The last run_igemm decision on this thread (vdb_igemm_last_plan): BN, STAGES, MODE, ksplit, grid, tilesM, tilesN
constexpr int kPlanFields = 7;
static thread_local int g_last_plan[kPlanFields] = {0};

// Mode 0 stores bf16 output rows and loads residual rows as 16-byte vectors, the split-K reduction stores fp32 rows as float4,
// and the TMA-store epilogues need a 16-byte aligned output map, so out / resid must be 16-byte aligned.  Checked before any
// tensor map is built, so that a bad pointer is reported as an argument error.
static int check_epilogue_pointers(const void* out, long long ldo, int out_f32, const void* resid, long long ldr, const char* who) {
  if ((reinterpret_cast<uintptr_t>(out) & 15) || (resid && (reinterpret_cast<uintptr_t>(resid) & 15)))
    return set_error(VDB_ERR_INVALID, "%s: out and resid must be 16-byte aligned", who);
  if (!out_f32 && (ldo % 8)) return set_error(VDB_ERR_INVALID, "%s: ldo must be a multiple of 8 for bf16 out", who);
  if (resid && (ldr % 8)) return set_error(VDB_ERR_INVALID, "%s: ldr must be a multiple of 8", who);
  return VDB_OK;
}

struct IgemmEpilogue {
  const float* bias = nullptr;
  long long bias_bstride = 0;
  int rows_per_batch = 1;
  const void* resid = nullptr;
  long long ldr = 0;
  void* out = nullptr;
  long long ldo = 0;
  int out_f32 = 0;
  int act = 0;
  float alpha = 1.f;
  // folded LayerNorm (see igemm_kernel): consumer side ...
  const float* ln_stats = nullptr;
  long long ln_mstat = 0;
  int ln_parts = 0;
  int ln_dim = 0;
  float ln_eps = 0.f;
  const float* ln_colsum = nullptr;
  int ln_on_cols = 0;
  const float* ln_rowbias = nullptr;
  // ... and producer side
  float* stats_out = nullptr;
  int* stats_parts = nullptr;     // host out: partials per row the launch wrote (2 * N tiles)
  // folded upsample writing straight into the interleaved [B, 2Ho, 2Wo, N] tensor: output parity (py * 2 + px), -1 = compact output
  int out_parity = -1;
};

// Finish IgemmParams (tiling, split-K, B map) and launch.
static int run_igemm(IgemmParams& p, const void* Wt, long long N, long long Ktot, long long ldw,
                     const IgemmEpilogue& e, int bn_forced, int ksplit_forced, void* workspace,
                     size_t ws_bytes, cudaStream_t stream) {
  const bool ln_in = e.ln_stats != nullptr, st_out = e.stats_out != nullptr;
  if (ln_in || st_out) ksplit_forced = 1;               // the statistics ride on the single-pass TMA-store epilogues
  int BN = pick_bn(static_cast<int>(N), e.act, bn_forced);
  // Tile-width model: the persistent grid runs
  // waves = ceil(tiles / #SMs) rounds of one tile per CTA, a tile costs kb * c(BN) cycles of mainloop (operand fill at ~90 B/clk
  // per SM or the MMA itself, whichever is longer) plus ~1500 cycles of pipeline fill / epilogue tail.  The divisibility rule sent
  // e.g. M 2048 x N 1280 x K 1280 (15 launches per step) to BN 256 = 80 tiles on 148 SMs; BN 160 gives 128 shorter tiles.
  if (!bn_forced && e.act != ACT_GEGLU && p.kb_total >= 8) {
    const long long tm = static_cast<long long>(p.tilesW) * p.tilesH * p.tilesB;
    const int cand[4] = {256, 160, 128, 64};
    double best = 1e30;
    for (int c : cand) {
      const long long tiles = tm * ((N + c - 1) / c);      // (a partial last N tile is computed in full)
      // split-K exactly as decided below: small MN grids with a deep K run kb / ks blocks per unit plus a reduction pass
      long long ks = 1;
      if (ksplit_forced > 0) ks = ksplit_forced;
      else if (tiles * 2 <= num_sms() && p.kb_total >= 16 && (N % 4) == 0 && workspace)
        ks = std::max<long long>(1, std::min<long long>(std::min<long long>(num_sms() / tiles, p.kb_total / 8), 16));
      const long long waves = (tiles * ks + num_sms() - 1) / num_sms();
      const double per_kb = std::max(2.0 * c, (16384.0 + 128.0 * c) / 90.0);
      const double kb_unit = static_cast<double>((p.kb_total + ks - 1) / ks);
      const double cost = static_cast<double>(waves) * (kb_unit * per_kb + 1500.0) + (ks > 1 ? 12000.0 : 0.0);
      if (cost < best * 0.97) { best = cost; BN = c; }     // (prefer the wider tile unless the gain is clear)
    }
  }
  if (BN != 64 && BN != 128 && BN != 160 && BN != 256) return set_error(VDB_ERR_INVALID, "igemm: bad BN");
  if (e.act == ACT_GEGLU && (N % BN) != 0) return set_error(VDB_ERR_INVALID, "igemm: GEGLU needs N % 256 == 0");
  p.N = static_cast<int>(N);
  p.tilesN = static_cast<int>((N + BN - 1) / BN);
  p.bias = e.bias; p.bias_bstride = e.bias_bstride; p.rows_per_batch = e.rows_per_batch > 0 ? e.rows_per_batch : 1;
  p.resid = reinterpret_cast<const __nv_bfloat16*>(e.resid); p.ldr = e.ldr;
  p.out = e.out; p.ldo = e.ldo; p.out_f32 = e.out_f32; p.act = e.act; p.alpha = e.alpha;
  const long long M = static_cast<long long>(p.Bo) * p.Ho * p.Wo;
  if (M >= (1LL << 30)) return set_error(VDB_ERR_UNSUPPORTED, "igemm: more than 2^30 output rows");
  const int tilesM = p.tilesW * p.tilesH * p.tilesB;
  const int mn_tiles = tilesM * p.tilesN;
  // split-K heuristic: fill the machine when the MN grid is small and K is deep
  int ksplit = 1;
  if (ksplit_forced > 0) {
    ksplit = ksplit_forced;
  } else if (e.act != ACT_GEGLU && mn_tiles * 2 <= num_sms() && p.kb_total >= 16 && (N % 4) == 0) {
    ksplit = std::min(std::min(num_sms() / mn_tiles, p.kb_total / 8), 16);
    if (ksplit < 1) ksplit = 1;
  }
  if (ksplit > 1) {
    const size_t need = static_cast<size_t>(ksplit) * M * N * sizeof(float);
    // (the reduction stores fp32 rows as float4: an fp32 row stride must keep them 16-byte aligned)
    if (workspace == nullptr || ws_bytes < need || e.act == ACT_GEGLU || (N % 4) || (e.out_f32 && (e.ldo % 4))) ksplit = 1;
  }
  p.ksplit = ksplit;
  p.kb_per_split = (p.kb_total + ksplit - 1) / ksplit;
  // drop empty trailing splits
  p.ksplit = (p.kb_total + p.kb_per_split - 1) / p.kb_per_split;
  p.partial = reinterpret_cast<float*>(workspace);
  p.ln_stats = e.ln_stats; p.ln_mstat = e.ln_mstat; p.ln_parts = e.ln_parts; p.ln_on_cols = e.ln_on_cols;
  if (e.stats_parts) *e.stats_parts = 2 * p.tilesN;
  p.ln_inv_dim = e.ln_dim > 0 ? 1.f / static_cast<float>(e.ln_dim) : 0.f; p.ln_eps = e.ln_eps;
  p.ln_colsum = e.ln_colsum; p.ln_rowbias = e.ln_rowbias; p.stats_out = e.stats_out;
  p.timeline = g_timeline;
  int rc = make_tmap_2d(&p.tmB, Wt, static_cast<uint64_t>(Ktot), static_cast<uint64_t>(N),
                        static_cast<uint64_t>(ldw) * 2, kBlockK, BN);
  if (rc) return rc;
  const int num_tiles = mn_tiles * p.ksplit;
  // epilogue specialisation (see igemm_kernel): 3 = plain bf16 fast path, 4 = GEGLU, 0 = everything else
  int mode = 0;
  // one bias row per tile: shared bias, or per-image rows with tiles that never straddle two images
  const bool one_bias_row = e.bias == nullptr || e.bias_bstride == 0 ||
                            (p.TB == 1 && (static_cast<long long>(p.Ho) * p.Wo == p.rows_per_batch ||
                                           (p.Ho == 1 && p.Bo == 1 && p.rows_per_batch % kBlockM == 0)));
  if (p.ksplit == 1 && !e.out_f32 && one_bias_row) {
    if (e.act == ACT_GEGLU && BN == 256) mode = 4;
    else if (e.act == ACT_NONE && e.alpha == 1.f && (N % 32) == 0) mode = 3;
  }
  // modes 3 / 4 store the output tile through shared memory + cp.async.bulk.tensor: a warp's 16 rows x 32 columns are one box
  // of the output tensor map (the M tile shapes hold at least 16 / (bw * bh) images; check_epilogue_pointers has checked the
  // alignment of out / resid)
  if (mode == 3 || mode == 4) {
    const int bw = std::min(p.TW, 16), bh = std::min(p.TH, 16 / bw), bb = 16 / (bw * bh);
    const long long ncols = (mode == 4) ? N / 2 : N;
    // out_parity >= 0: the same tile, written into every second pixel of every second row of the [B, 2Ho, 2Wo, N] tensor —
    // only the strides and the base of the output tensor map change, the kernel does not know
    const int py = e.out_parity >= 0 ? (e.out_parity >> 1) : 0, px = e.out_parity >= 0 ? (e.out_parity & 1) : 0;
    const uint64_t il = e.out_parity >= 0 ? 2 : 1;
    const void* obase = reinterpret_cast<const __nv_bfloat16*>(e.out) + (static_cast<long long>(py) * (il * p.Wo) + px) * e.ldo;
    rc = make_tmap_4d_sw64(&p.tmO, obase, static_cast<uint64_t>(ncols), static_cast<uint64_t>(p.Wo), static_cast<uint64_t>(p.Ho),
                           static_cast<uint64_t>(p.Bo), il * static_cast<uint64_t>(e.ldo) * 2,
                           il * il * static_cast<uint64_t>(p.Wo) * e.ldo * 2,
                           il * il * static_cast<uint64_t>(p.Ho) * p.Wo * e.ldo * 2, 32, bw, bh, bb);
    if (rc) return rc;
  }
  if (e.out_parity >= 0 && mode != 3)
    return set_error(VDB_ERR_UNSUPPORTED, "igemm: the interleaved-output upsample modes need the TMA-store epilogue (bf16 out, no "
                                          "activation, N %% 32 == 0)");
  if (ln_in || st_out) {
    // folded LayerNorm: only on the TMA-store epilogues (bf16 out, act none / GEGLU, alpha 1, N % 32 == 0)
    if (ln_in && st_out) return set_error(VDB_ERR_UNSUPPORTED, "igemm: a launch either consumes or produces LayerNorm statistics");
    if (mode != 3 && !(mode == 4 && ln_in))
      return set_error(VDB_ERR_UNSUPPORTED, "igemm: LayerNorm statistics need the TMA-store epilogue (bf16 out, no activation or "
                                            "GEGLU, alpha 1, N %% 32 == 0)");
    if (ln_in && e.resid) return set_error(VDB_ERR_UNSUPPORTED, "igemm: a folded-LayerNorm GEMM takes no residual");
    if (ln_in && mode == 4 && e.ln_on_cols) return set_error(VDB_ERR_UNSUPPORTED, "igemm: GEGLU with column statistics");
    mode = st_out ? 7 : mode + 2;
  }
  {
    const int stages = BN == 64 ? 8 : BN == 128 ? 6 : BN == 160 ? 5 : 4;   // (as instantiated below)
    const int plan[kPlanFields] = {BN, stages, mode, p.ksplit, std::min(num_tiles, num_sms()), tilesM, p.tilesN};
    for (int i = 0; i < kPlanFields; ++i) g_last_plan[i] = plan[i];
  }
  if (mode == 7) {
    switch (BN) {
      case 64: rc = launch_igemm<64, 8, 8, 7>(p, num_tiles, stream); break;
      case 128: rc = launch_igemm<128, 6, 8, 7>(p, num_tiles, stream); break;
      case 160: rc = launch_igemm<160, 5, 8, 7>(p, num_tiles, stream); break;
      default: rc = launch_igemm<256, 4, 8, 7>(p, num_tiles, stream); break;
    }
  } else if (mode == 6) {
    rc = launch_igemm<256, 4, 8, 6>(p, num_tiles, stream);
  } else if (mode == 5) {
    switch (BN) {
      case 64: rc = launch_igemm<64, 8, 8, 5>(p, num_tiles, stream); break;
      case 128: rc = launch_igemm<128, 6, 8, 5>(p, num_tiles, stream); break;
      case 160: rc = launch_igemm<160, 5, 8, 5>(p, num_tiles, stream); break;
      default: rc = launch_igemm<256, 4, 8, 5>(p, num_tiles, stream); break;
    }
  } else if (mode == 4) {
    rc = launch_igemm<256, 4, 8, 4>(p, num_tiles, stream);
  } else if (mode == 3) {
    switch (BN) {
      case 64: rc = launch_igemm<64, 8, 8, 3>(p, num_tiles, stream); break;
      case 128: rc = launch_igemm<128, 6, 8, 3>(p, num_tiles, stream); break;
      case 160: rc = launch_igemm<160, 5, 8, 3>(p, num_tiles, stream); break;
      default: rc = launch_igemm<256, 4, 8, 3>(p, num_tiles, stream); break;
    }
  } else {
    switch (BN) {
      case 64: rc = launch_igemm<64, 8, 8, 0>(p, num_tiles, stream); break;
      case 128: rc = launch_igemm<128, 6, 8, 0>(p, num_tiles, stream); break;
      case 160: rc = launch_igemm<160, 5, 8, 0>(p, num_tiles, stream); break;
      default: rc = launch_igemm<256, 4, 8, 0>(p, num_tiles, stream); break;
    }
  }
  if (rc) return rc;
  if (p.ksplit > 1) {
    const long long total = M * (N / 4);
    const int threads = 256;
    const int blocks = static_cast<int>(std::min<long long>((total + threads - 1) / threads, num_sms() * 8LL));
    VDB_CUDA_CHECK(launch_pdl(splitk_reduce_kernel, dim3(blocks), dim3(threads), 0, stream, (const float*)p.partial,
                              p.ksplit, M, static_cast<int>(N), p.bias, p.bias_bstride, p.rows_per_batch, p.resid,
                              p.ldr, p.out, p.ldo, p.out_f32, p.act, p.alpha));
    count_launch();
  }
  return VDB_OK;
}

static int pow2_ceil(int v) { int t = 1; while (t < v) t <<= 1; return t; }

// M tile = 128 output pixels as a (TW, TH, TB) box of the (W, H, B) pixel grid; box extents are
// powers of two so that TW*TH*TB == 128 (rows past the grid are zero-filled by TMA and masked on store).
static void set_tile_shape(IgemmParams& p, int Wo, int Ho, int Bo) {
  p.Wo = Wo; p.Ho = Ho; p.Bo = Bo;
  const int TW = std::min(pow2_ceil(Wo), 128);
  const int TH = std::min(pow2_ceil(Ho), 128 / TW);
  const int TB = 128 / (TW * TH);
  p.TW = TW; p.TH = TH; p.TB = TB;
  p.tilesW = (Wo + TW - 1) / TW;
  p.tilesH = (Ho + TH - 1) / TH;
  p.tilesB = (Bo + TB - 1) / TB;
}

}  // namespace vdb

using namespace vdb;

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

// debug aid (not part of the product ABI): device buffer of 16*8 u64 receiving CTA 0's per-tile role timestamps
void vdb_debug_igemm_timeline(void* buf) { g_timeline = reinterpret_cast<unsigned long long*>(buf); }

// see include/vdb200.h
int vdb_igemm_last_plan(int* out, int n) {
  for (int i = 0; out && i < n && i < kPlanFields; ++i) out[i] = g_last_plan[i];
  return kPlanFields;
}

// out[M,N] = act(alpha * ([A | A2] @ W^T + bias)) + resid     (see include/vdb200.h)
int vdb_gemm_bf16(const void* A, long long M, long long K, long long lda, const void* A2, long long K2,
                  long long lda2, const void* W, long long N, long long ldw, const float* bias,
                  long long bias_bstride, long long rows_per_batch, const void* resid, long long ldr, void* out,
                  long long ldo, int out_f32, int act, float alpha, int bn, int ksplit, void* workspace,
                  size_t ws_bytes, void* stream) {
  if (!A || !W || !out || M <= 0 || N <= 0 || K <= 0) return set_error(VDB_ERR_INVALID, "gemm: null/empty argument");
  if ((K % 8) || (lda % 8) || (ldw % 8)) return set_error(VDB_ERR_INVALID, "gemm: K, lda, ldw must be multiples of 8");
  if (A2 && ((K % kBlockK) || (K2 % 8) || (lda2 % 8)))
    return set_error(VDB_ERR_INVALID, "gemm: two-source A needs K % 64 == 0 and K2, lda2 % 8 == 0");
  if (M > 0x7fffffffLL || N > 0x7fffffffLL) return set_error(VDB_ERR_INVALID, "gemm: dimension too large");
  int rc = check_epilogue_pointers(out, ldo, out_f32, resid, ldr, "gemm");
  if (rc) return rc;
  IgemmParams p;
  memset(&p, 0, sizeof(p));
  // GEMM view of the pixel grid: one row of M "pixels"; the box is always 128 rows (TMA zero-fills past M)
  p.Wo = static_cast<int>(M); p.Ho = 1; p.Bo = 1;
  p.TW = kBlockM; p.TH = 1; p.TB = 1;
  p.tilesW = static_cast<int>((M + kBlockM - 1) / kBlockM); p.tilesH = 1; p.tilesB = 1;
  rc = make_tmap_4d(&p.tmA[0], A, K, M, 1, 1, lda * 2, lda * 2 * M, lda * 2 * M, kBlockK, p.TW, 1, 1);
  if (rc) return rc;
  p.seg[0] = ASeg{0, 0, 0, static_cast<int16_t>((K + kBlockK - 1) / kBlockK), 0};
  p.nseg = 1;
  p.kb_total = p.seg[0].nkb;
  if (A2) {
    rc = make_tmap_4d(&p.tmA[1], A2, K2, M, 1, 1, lda2 * 2, lda2 * 2 * M, lda2 * 2 * M, kBlockK, p.TW, 1, 1);
    if (rc) return rc;
    p.seg[1] = ASeg{1, 0, 0, static_cast<int16_t>((K2 + kBlockK - 1) / kBlockK), 0};
    p.nseg = 2;
    p.kb_total += p.seg[1].nkb;
  }
  for (int i = p.nseg; i < kMaxA; ++i) p.tmA[i] = p.tmA[0];
  IgemmEpilogue e;
  e.bias = bias; e.bias_bstride = bias_bstride; e.rows_per_batch = static_cast<int>(rows_per_batch);
  e.resid = resid; e.ldr = ldr; e.out = out; e.ldo = ldo; e.out_f32 = out_f32; e.act = act; e.alpha = alpha;
  return run_igemm(p, W, N, K + (A2 ? K2 : 0), ldw, e, bn, ksplit, workspace, ws_bytes,
                   reinterpret_cast<cudaStream_t>(stream));
}

// GEMM with a LayerNorm folded in (consumer) or LayerNorm statistics written out (producer); see include/vdb200.h
int vdb_gemm_ln_bf16(const void* A, long long M, long long K, long long lda, const void* W, long long N, long long ldw,
                     const float* bias, const void* resid, long long ldr, void* out, long long ldo, int act,
                     const float* ln_stats, long long ln_rows, int ln_parts, int ln_dim, float ln_eps, const float* ln_colsum,
                     int ln_on_cols, const float* ln_rowbias, float* stats_out, int* stats_parts, int bn, void* stream) {
  if (!A || !W || !out || M <= 0 || N <= 0 || K <= 0) return set_error(VDB_ERR_INVALID, "gemm_ln: null/empty argument");
  if ((K % 8) || (lda % 8) || (ldw % 8)) return set_error(VDB_ERR_INVALID, "gemm_ln: K, lda, ldw must be multiples of 8");
  if (M > 0x7fffffffLL || N > 0x7fffffffLL) return set_error(VDB_ERR_INVALID, "gemm_ln: dimension too large");
  if (!ln_stats && !stats_out) return set_error(VDB_ERR_INVALID, "gemm_ln: neither ln_stats nor stats_out given (use vdb_gemm_bf16)");
  if (ln_stats) {
    if (!ln_colsum || ln_dim <= 0 || ln_dim != K || ln_parts <= 0)
      return set_error(VDB_ERR_INVALID, "gemm_ln: need ln_colsum, ln_parts > 0 and ln_dim == K");
    if (ln_rows < (ln_on_cols ? N : M)) return set_error(VDB_ERR_INVALID, "gemm_ln: statistics table has too few rows");
  }
  if (stats_out && ((N % 32) || !stats_parts)) return set_error(VDB_ERR_INVALID, "gemm_ln: stats_out needs N %% 32 == 0 and stats_parts");
  int rc = check_epilogue_pointers(out, ldo, 0, resid, ldr, "gemm_ln");
  if (rc) return rc;
  IgemmParams p;
  memset(&p, 0, sizeof(p));
  p.Wo = static_cast<int>(M); p.Ho = 1; p.Bo = 1;
  p.TW = kBlockM; p.TH = 1; p.TB = 1;
  p.tilesW = static_cast<int>((M + kBlockM - 1) / kBlockM); p.tilesH = 1; p.tilesB = 1;
  rc = make_tmap_4d(&p.tmA[0], A, K, M, 1, 1, lda * 2, lda * 2 * M, lda * 2 * M, kBlockK, p.TW, 1, 1);
  if (rc) return rc;
  p.seg[0] = ASeg{0, 0, 0, static_cast<int16_t>((K + kBlockK - 1) / kBlockK), 0};
  p.nseg = 1;
  p.kb_total = p.seg[0].nkb;
  for (int i = p.nseg; i < kMaxA; ++i) p.tmA[i] = p.tmA[0];
  IgemmEpilogue e;
  e.bias = bias; e.resid = resid; e.ldr = ldr; e.out = out; e.ldo = ldo; e.act = act;
  e.ln_stats = ln_stats; e.ln_mstat = ln_rows; e.ln_parts = ln_parts; e.ln_dim = ln_dim; e.ln_eps = ln_eps; e.ln_colsum = ln_colsum;
  e.ln_on_cols = ln_on_cols; e.ln_rowbias = ln_rowbias; e.stats_out = stats_out; e.stats_parts = stats_parts;
  return run_igemm(p, W, N, K, ldw, e, bn, 1, nullptr, 0, reinterpret_cast<cudaStream_t>(stream));
}

// 3x3 convolution on NHWC bf16 as implicit GEMM.
//   mode 0: stride 1, pad 1                       (out H x W)
//   mode 1: stride 2, pad 1                       (out H/2 x W/2)      openaimodel.py:150-152
//   mode 2: stride 2, pad (0,1,0,1) then pad 0    (out H/2 x W/2)      autokl_modules.py:72-76
//   mode 3 + 2*py + px: one parity sub-lattice of "nearest 2x upsample, then 3x3 conv pad 1" (openaimodel.py:107-117,
//           autokl_modules.py:54-58) computed on the SOURCE image: output pixel (2y+py, 2x+px) of the upsampled conv only
//           sees the 2x2 source pixels (y + ty - 1 + py, x + tx - 1 + px), ty, tx in {0,1}, so the 9 taps fold into 4 with
//           pre-summed weights (host: fold_upsample_conv3x3).  X = source [B,H,W,C], out = [B,H,W,N] (that parity, dense),
//           Wt = [N, 4*C] with K ordered (ty, tx, c).  2.25x fewer FLOPs than upsampling first; no skip inputs.
// Wt is [N, 9*C + Cs1 + Cs2] bf16 with K ordered (ky, kx, c) then the 1x1-skip columns.
// skip1/skip2: optional raw NHWC tensors at OUTPUT resolution whose 1x1 conv is accumulated too.
int vdb_conv3x3_bf16(const void* X, int B, int H, int Wd, int C, int mode, const void* Wt, int N, long long ldw,
                     const void* skip1, int Cs1, const void* skip2, int Cs2, const float* bias,
                     long long bias_bstride, const void* resid, long long ldr, void* out, long long ldo,
                     int out_f32, int act, int bn, int ksplit, void* workspace, size_t ws_bytes, void* stream) {
  if (!X || !Wt || !out || B <= 0 || H <= 0 || Wd <= 0 || C <= 0 || N <= 0)
    return set_error(VDB_ERR_INVALID, "conv3x3: null/empty argument");
  if ((C % kBlockK) || (ldw % 8)) return set_error(VDB_ERR_INVALID, "conv3x3: C must be a multiple of 64, ldw of 8");
  if ((skip1 && (Cs1 % kBlockK)) || (skip2 && (Cs2 % kBlockK)))
    return set_error(VDB_ERR_INVALID, "conv3x3: skip channels must be multiples of 64");
  if (mode < 0 || mode > 10) return set_error(VDB_ERR_INVALID, "conv3x3: bad mode");
  const int out_parity = mode >= 7 ? mode - 7 : -1;     // modes 7..10 = modes 3..6 writing into the interleaved [B, 2H, 2W, N] tensor
  if (mode >= 7) mode -= 4;
  if (out_parity >= 0 && (resid || out_f32 || ksplit > 1)) return set_error(VDB_ERR_INVALID, "conv3x3: modes 7..10 take no residual, bf16 out, no split-K");
  if (out_parity >= 0) ksplit = 1;
  const bool strided = (mode == 1 || mode == 2), folded = mode >= 3;
  if (strided && ((H & 1) || (Wd & 1))) return set_error(VDB_ERR_UNSUPPORTED, "conv3x3: stride 2 needs even H, W");
  if (folded && (skip1 || skip2)) return set_error(VDB_ERR_INVALID, "conv3x3: the folded-upsample modes take no skip inputs");
  int rc = check_epilogue_pointers(out, ldo, out_f32, resid, ldr, "conv3x3");
  if (rc) return rc;
  IgemmParams p;
  memset(&p, 0, sizeof(p));
  const int Ho = strided ? H / 2 : H, Wo = strided ? Wd / 2 : Wd;
  set_tile_shape(p, Wo, Ho, B);
  const uint64_t eb = 2;
  const int nkb = C / kBlockK;
  int nmaps = 0;
  int ntaps = 9;
  if (mode == 0 || folded) {
    rc = make_tmap_4d(&p.tmA[0], X, C, Wd, H, B, C * eb, (uint64_t)Wd * C * eb, (uint64_t)H * Wd * C * eb, kBlockK,
                      p.TW, p.TH, p.TB);
    if (rc) return rc;
    nmaps = 1;
    if (mode == 0) {
      for (int t = 0; t < 9; ++t)
        p.seg[t] = ASeg{0, static_cast<int16_t>(t % 3 - 1), static_cast<int16_t>(t / 3 - 1), static_cast<int16_t>(nkb), 0};
    } else {
      const int py = (mode - 3) >> 1, px = (mode - 3) & 1;
      ntaps = 4;
      for (int t = 0; t < 4; ++t)      // t = ty * 2 + tx; source pixel (y + ty - 1 + py, x + tx - 1 + px)
        p.seg[t] = ASeg{0, static_cast<int16_t>((t & 1) - 1 + px), static_cast<int16_t>((t >> 1) - 1 + py), static_cast<int16_t>(nkb), 0};
    }
  } else {
    // four parity sub-lattices of the input: X[b, 2*yo+py, 2*xo+px, c]
    for (int py = 0; py < 2; ++py)
      for (int px = 0; px < 2; ++px) {
        const uint8_t* base = reinterpret_cast<const uint8_t*>(X) + (static_cast<uint64_t>(py) * Wd + px) * C * eb;
        rc = make_tmap_4d(&p.tmA[py * 2 + px], base, C, Wo, Ho, B, 2ull * C * eb, 2ull * Wd * C * eb,
                          (uint64_t)H * Wd * C * eb, kBlockK, p.TW, p.TH, p.TB);
        if (rc) return rc;
      }
    nmaps = 4;
    for (int t = 0; t < 9; ++t) {
      const int ky = t / 3, kx = t % 3;
      int py, dy, px, dx;
      if (mode == 1) {  // input row = 2*yo + ky - 1
        py = (ky == 1) ? 0 : 1; dy = (ky == 0) ? -1 : 0;
        px = (kx == 1) ? 0 : 1; dx = (kx == 0) ? -1 : 0;
      } else {          // input row = 2*yo + ky (zero pad on bottom/right only)
        py = (ky == 1) ? 1 : 0; dy = (ky == 2) ? 1 : 0;
        px = (kx == 1) ? 1 : 0; dx = (kx == 2) ? 1 : 0;
      }
      p.seg[t] = ASeg{static_cast<int16_t>(py * 2 + px), static_cast<int16_t>(dx), static_cast<int16_t>(dy),
                      static_cast<int16_t>(nkb), 0};
    }
  }
  p.nseg = ntaps;
  p.kb_total = ntaps * nkb;
  const void* sk[2] = {skip1, skip2};
  const int sc[2] = {Cs1, Cs2};
  for (int i = 0; i < 2; ++i) {
    if (!sk[i]) continue;
    rc = make_tmap_4d(&p.tmA[nmaps], sk[i], sc[i], Wo, Ho, B, sc[i] * eb, (uint64_t)Wo * sc[i] * eb,
                      (uint64_t)Ho * Wo * sc[i] * eb, kBlockK, p.TW, p.TH, p.TB);
    if (rc) return rc;
    p.seg[p.nseg] = ASeg{static_cast<int16_t>(nmaps), 0, 0, static_cast<int16_t>(sc[i] / kBlockK), 0};
    p.kb_total += sc[i] / kBlockK;
    ++p.nseg;
    ++nmaps;
  }
  for (int i = nmaps; i < kMaxA; ++i) p.tmA[i] = p.tmA[0];
  IgemmEpilogue e;
  e.bias = bias; e.bias_bstride = bias_bstride; e.rows_per_batch = Ho * Wo;
  e.resid = resid; e.ldr = ldr; e.out = out; e.ldo = ldo; e.out_f32 = out_f32; e.act = act; e.alpha = 1.f;
  e.out_parity = out_parity;
  return run_igemm(p, Wt, N, static_cast<long long>(p.kb_total) * kBlockK, ldw, e, bn, ksplit, workspace, ws_bytes,
                   reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
