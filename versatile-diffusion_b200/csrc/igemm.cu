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
// Structure: grid = #SMs (persistent, static round-robin over output tiles), 288 threads (384 where the accumulator needs the
// producer's registers, see igemm_realloc):
//   warps 0-7: two consumer warpgroups (BM / 128 wgmma m64 x BN x 16 each per k16 step, fp32 accumulators in registers), then the
//              epilogue straight from the registers: bias / LayerNorm / activation / GEGLU / residual -> bf16 TMA stores, or fp32
//              stores (fp32 output, split-K partials)
//   warp 8   : TMA producer  (cp.async.bulk.tensor 4D box loads of A, 2D box loads of W)
// smem ring of STAGES x (A BMx64 bf16 | W BNx64 bf16), both 128B-swizzled K-major; the tile is BM = 128 or 256 rows high.
#include "common.cuh"
#include "host_util.h"

namespace vdb {

constexpr int kBlockM = 128;  // tile height of every launch the 256-row rule in choose_tile does not take
constexpr int kBlockK = 64;  // bf16 elements = 128 B = one swizzle row
constexpr int kMaxA = 6;     // A tensor maps per launch
constexpr int kMaxSeg = 12;  // K segments per launch
constexpr int kNumEpiWarps = 8;  // the two consumer warpgroups, which run the epilogue too; the producer warp follows them
// A 256-row tile (160 accumulator registers per thread) or a 256-column one (128) does not fit the 168 registers that 288
// threads leave each thread: those instantiations launch a whole producer warpgroup (384 threads, one warp of it works) that
// hands its registers to the consumers (setmaxnreg: 128 x 40 + 256 x 232 = 64512 of the SM's 65536).
__host__ __device__ constexpr bool igemm_realloc(int BM, int BN) { return BM == 256 || BN == 256; }
__host__ __device__ constexpr int igemm_threads(int BM, int BN) { return 32 * kNumEpiWarps + (igemm_realloc(BM, BN) ? 128 : 32); }
// TMA-store staging boxes (1 KB) per epilogue warp: four, or two where four 52 KB stages leave no room for more
__host__ __device__ constexpr int igemm_boxes(int BM) { return BM == 256 ? 2 : 4; }

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
  CUtensorMap tmR;         // modes 3 / 7 with a residual: tmO's geometry over resid / ldr (loaded into the staging boxes)
  ASeg seg[kMaxSeg];
  int nseg;
  int kb_total;      // total k-blocks over all segments
  int ksplit;        // split-K factor (>=1); >1 => fp32 partial output
  int kb_per_split;  // ceil(kb_total / ksplit)
  int TW, TH, TB;    // M tile = TW*TH*TB = BM output pixels
  int Wo, Ho, Bo;    // output pixel grid (GEMM view: Wo = M, Ho = Bo = 1)
  int tilesW, tilesH, tilesB, tilesN;
  int n_fast;        // tile walk: 0 = M tile index fastest, 1 = N tile index fastest (run_igemm decides; see igemm_kernel)
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
  unsigned smem_bytes;        // dynamic shared memory of the launch (LN modes check their carve-up against it)
};

enum { ACT_NONE = 0, ACT_SILU = 1, ACT_GELU = 2, ACT_QGELU = 3, ACT_GEGLU = 4 };

VDB_DEVINL float apply_act(float v, int act) {
  switch (act) {
    case ACT_SILU: return silu_f(v);
    case ACT_GELU: return gelu_erf_f(v);
    case ACT_QGELU: return quick_gelu_f(v);
    default: return v;
  }
}

// v = act(alpha * v) over 8 of the values of a thread's epilogue chunk: one branch on the activation per 8 values, so the code a
// chunk executes stays contiguous (a switch per element spreads it over every activation's code); 8 at a time, not 16, keeps the
// interleaved activations inside the registers the accumulator leaves
VDB_DEVINL void alpha_act8(float* v, float alpha, int act) {
  switch (act) {
    case ACT_SILU:
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = silu_f(__fmul_rn(v[i], alpha));
      break;
    case ACT_GELU:
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = gelu_erf_f(__fmul_rn(v[i], alpha));
      break;
    case ACT_QGELU:
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = quick_gelu_f(__fmul_rn(v[i], alpha));
      break;
    default:
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = __fmul_rn(v[i], alpha);
  }
}

// MODE selects the epilogue that is compiled in: 0 = every path (split-K partials, GEGLU, activation / alpha, fp32 output,
// ragged N, per-row bias), 3 = only plain bf16 (act none, alpha 1, N % 32 == 0, one bias row per tile), 4 = only GEGLU.  Keeping
// the rarely used paths out of the common instantiations keeps the epilogue's instruction footprint small.  Modes 5 / 6 are
// modes 3 / 4 for a GEMM whose
// input is a LayerNorm: the operand is the RAW activation x and the weights carry gamma (W' = W * gamma), so with the row's mean mu
// and rstd r       LN(x) W^T + b  =  r * (x W'^T  -  mu * s) + c,     s[n] = sum_k W'[n,k],  c[n] = sum_k beta_k W[n,k] + b[n]
// is a rank-1 correction in the epilogue (2 FMAs per element) — the normalised tensor is never written or read.  mu and r come
// from per-32-channel partial sums that the PRODUCER of x wrote from its own epilogue (mode 7 = mode 3 + those sums).  When x is
// the B operand (the transposed V^T projection) the statistics belong to the output columns instead (ln_on_cols).
//
// Roles: warps 0-7 are two consumer warpgroups (warpgroup g computes output rows [BM / 2 * g, BM / 2 * (g + 1)) of the tile with
// wgmma, as BM / 128 blocks of 64 rows that share the W descriptor, fp32 accumulators in registers), warp 8 is the TMA producer.
// Every mode runs the epilogue from the registers, in the wgmma fragment layout: warp w owns 16 rows of the tile and walks their
// 32-column chunks, staging each as a 16 x 32 bf16 box (stmatrix) for a TMA store, or storing it to global memory directly when
// the output is fp32.  The warpgroups do not wait for each other after the mainloop, and the producer is gated by the empty
// barriers alone: it loads the next tile's first STAGES k-blocks while the epilogue runs, so the next mainloop starts on a full
// ring.  tests/test_igemm_protocol_tma_epi.py models this protocol.
template <int BM, int BN, int STAGES, int MODE>
__global__ void __launch_bounds__(igemm_threads(BM, BN), 1) igemm_kernel(const __grid_constant__ IgemmParams p) {
  constexpr bool kGegluEpi = MODE == 4 || MODE == 6;
  constexpr bool kLnIn = MODE == 5 || MODE == 6;
  constexpr bool kStatsOut = MODE == 7;
  constexpr int kNumEpiThreads = kNumEpiWarps * 32;
  static_assert(BM == 128 || (BM == 256 && (MODE == 3 || MODE == 7) && BN <= 160), "256-row tiles: modes 3 and 7, 160 accumulator registers");
  constexpr int kMB = BM / 128;          // 64-row blocks per consumer warpgroup
  constexpr int kBoxes = igemm_boxes(BM);
  constexpr uint32_t kStgWarp = kBoxes * 1024;   // staging bytes per epilogue warp
  constexpr uint32_t kABytes = BM * kBlockK * 2;
  constexpr uint32_t kBBytes = BN * kBlockK * 2;
  constexpr uint32_t kStageBytes = kABytes + kBBytes;
  constexpr uint32_t kRingBytes = STAGES * kStageBytes;
  static_assert(kBBytes % 1024 == 0, "B stage must keep 1024B alignment");
  static_assert(BN % 32 == 0 && BN >= 32 && BN <= 256, "invalid wgmma N");

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smemA = smem;
  uint8_t* smemB = smem + STAGES * kABytes;
  uint8_t* sstage = smem + kRingBytes;                        // kNumEpiWarps x kBoxes 1 KB bf16 TMA-store boxes, 1024-byte aligned
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sstage + kNumEpiWarps * kStgWarp);
  uint64_t* empty_bar = full_bar + STAGES;
  float* sbias = reinterpret_cast<float*>(empty_bar + STAGES);  // [BN] bias of the current output tile
  float* slnx = sbias + BN;                                   // [BN] LN modes: colsum s (on_cols 0) / column mean (on_cols 1)
  uint64_t* rbar = reinterpret_cast<uint64_t*>(slnx + (kLnIn ? BN : 0));   // modes 3 / 7: [kNumEpiWarps][kBoxes] residual loads
  const uint32_t sbias_s = smem_u32(sbias), slnx_s = smem_u32(slnx);   // (shared-space addresses: LDS, not generic LD)
  (void)slnx_s;
  if constexpr (kLnIn) {
    if (reinterpret_cast<uint8_t*>(slnx + BN) > smem_raw + p.smem_bytes) __trap();
  }
  auto epi_bar_sync = [] { asm volatile("bar.sync 1, %0;" ::"n"(kNumEpiThreads) : "memory"); };   // the consumer warps only
  // modes 3 / 7 TMA-load the residual of a chunk into the staging box the chunk is stored from (tmR); mode 0 reads it from
  // global memory into registers (its accumulator leaves no registers for the box protocol), and split-K adds it in
  // splitk_reduce_kernel
  constexpr bool kResidTma = MODE == 3 || MODE == 7;
  const bool resid_tma = kResidTma && p.resid != nullptr;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == kNumEpiWarps && lane == 0) {
    for (int i = 0; i < kMaxA; ++i) tma_prefetch_desc(&p.tmA[i]);
    tma_prefetch_desc(&p.tmB);
    if (MODE != 0 || (!p.out_f32 && p.ksplit == 1)) tma_prefetch_desc(&p.tmO);   // (mode 0 builds it for bf16 output only)
    if (resid_tma) tma_prefetch_desc(&p.tmR);
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kNumEpiWarps);
    }
    if constexpr (kResidTma)
      for (int i = 0; i < kNumEpiWarps * kBoxes; ++i) mbar_init(&rbar[i], 1);
    fence_barrier_init();
  }
  __syncthreads();

  const int tilesM = p.tilesW * p.tilesH * p.tilesB;
  const int num_tiles = tilesM * p.tilesN * p.ksplit;
  // Tile walk of this CTA (both roles use the same bounds and the same incremental arithmetic): tiles c, c + grid, ..., tile t =
  // unit_f + units_f * unit_s.  M-fast (n_fast 0): unit_f = M tile, unit_s = N tile + tilesN * k-split.  N-fast (n_fast 1,
  // ksplit 1 only): unit_f = N tile, unit_s = M tile, so a wave reads each band of A rows once, for all its N tiles together.
  const int units_f = p.n_fast ? p.tilesN : tilesM;
  const int step_f = gridDim.x % units_f, step_s = gridDim.x / units_f;
  const int t_first = blockIdx.x, t_step = gridDim.x, t_end = num_tiles;

  if (warp >= kNumEpiWarps) {
    // ------------------------------ TMA producer ------------------------------
    if constexpr (igemm_realloc(BM, BN)) setmaxnreg_dec<40>();     // the whole producer warpgroup; its first warp alone works
    if (warp == kNumEpiWarps && lane == 0) {
      uint32_t stage = 0, phase = 0;
      const bool flat = (p.tilesH == 1) && (p.tilesB == 1);
      int unit_f = t_first % units_f, unit_s = t_first / units_f;
      for (int t = t_first; t < t_end; t += t_step) {
        const int m_idx = p.n_fast ? unit_s : unit_f;
        int n_idx = p.n_fast ? unit_f : unit_s, ks = 0;
        if (p.ksplit > 1) { n_idx = unit_s % p.tilesN; ks = unit_s / p.tilesN; }
        int wt = m_idx, ht = 0, bt = 0;
        if (!flat) {
          wt = m_idx % p.tilesW;
          const int q = m_idx / p.tilesW;
          ht = q % p.tilesH;
          bt = q / p.tilesH;
        }
        unit_f += step_f; unit_s += step_s;
        if (unit_f >= units_f) { unit_f -= units_f; ++unit_s; }
        const int w0 = wt * p.TW, h0 = ht * p.TH, b0 = bt * p.TB;
        const int n0 = n_idx * BN;
        const int kb_begin = ks * p.kb_per_split;
        const int kb_end = min(p.kb_total, kb_begin + p.kb_per_split);
        int kb = 0;
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
    if constexpr (igemm_realloc(BM, BN)) setmaxnreg_inc<232>();
    // mainloop of one tile: warpgroup g multiplies its kMB blocks of 64 rows of A by the BN x 64 B tile of every k-block (block
    // hb sits 8 KB after block hb - 1 in the stage)
    uint32_t ml_stage = 0, ml_phase = 0;
    float acc[kMB][BN / 2];
    auto mainloop = [&](int kb_begin, int kb_end, auto&& after_first_kblock) {
      const int g = warp >> 2;
#pragma unroll
      for (int hb = 0; hb < kMB; ++hb)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[hb][i] = 0.f;
      uint32_t prev = 0;
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&full_bar[ml_stage], ml_phase);
        wgmma_fence();
        uint64_t adesc[kMB];
#pragma unroll
        for (int hb = 0; hb < kMB; ++hb)
          adesc[hb] = make_desc_sw128(smem_u32(smemA + ml_stage * kABytes + (g * kMB + hb) * (64 * 128)));
        const uint64_t bdesc = make_desc_sw128(smem_u32(smemB + ml_stage * kBBytes));
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k)
#pragma unroll
          for (int hb = 0; hb < kMB; ++hb) wgmma_ss<BN>(acc[hb], adesc[hb] + 2 * k, bdesc + 2 * k, (kb > kb_begin || k > 0) ? 1u : 0u);
        wgmma_commit();
        if (kb == kb_begin) after_first_kblock();
        if (kb > kb_begin) {            // the previous k-block's MMAs have read their stage: hand it back to the producer
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = ml_stage;
        if (++ml_stage == STAGES) { ml_stage = 0; ml_phase ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int hb = 0; hb < kMB; ++hb) wgmma_fence_regs(acc[hb]);
      __syncwarp();
      if (lane == 0 && kb_end > kb_begin) mbar_arrive(&empty_bar[prev]);
    };
    int st_buf = 0;                     // which of this warp's kBoxes staging boxes is written next
    uint32_t rphase = 0;                // modes 3 / 7, bit b: parity of the next residual load into box b
    const float* sbias_src = nullptr;   // which bias row/offset currently sits in sbias
    // The per-tile bookkeeping sits on the critical path of epilogue-bound GEMMs: the tile index advances incrementally (no
    // divisions in the GEMM view), row indices are 32-bit, and everything that depends only on the thread is hoisted.
    const bool flat = (p.tilesH == 1) && (p.tilesB == 1);   // GEMM view: M tiles along W only
    int unit_f = t_first % units_f, unit_s = t_first / units_f;
    // the accumulator stays in the wgmma fragment layout, so in each 64-row block hb of its warpgroup warp w
    // owns the 16 tile rows from e_row0 + 64 hb on (warpgroup w / 4, quarter w % 4) and this thread rows + lane / 4 and
    // + lane / 4 + 8 of them, at columns 8 j + 2 (lane % 4) + {0, 1}
    const int e_row0 = (warp >> 2) * (BM / 2) + (warp & 3) * 16;
    int e_tw[kMB][2], e_th[kMB][2], e_tb[kMB][2];
#pragma unroll
    for (int hb = 0; hb < kMB; ++hb)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int er = e_row0 + 64 * hb + (lane >> 2) + 8 * h;
        e_tw[hb][h] = er % p.TW; e_th[hb][h] = (er / p.TW) % p.TH; e_tb[hb][h] = er / (p.TW * p.TH);
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
      if (!p.ln_on_cols && p.ln_parts <= 2 * kLnPre && t_first < t_end) ln_prefetch((p.n_fast ? unit_s : unit_f) * kBlockM + e_row0 + (lane & 15));
    }
    for (int t = t_first; t < t_end; t += t_step) {
      const int m_idx = p.n_fast ? unit_s : unit_f;
      int n_idx = p.n_fast ? unit_f : unit_s, ks = 0;
      if (p.ksplit > 1) { n_idx = unit_s % p.tilesN; ks = unit_s / p.tilesN; }
      int wt = m_idx, ht = 0, bt = 0;
      if (!flat) {
        wt = m_idx % p.tilesW;
        const int q = m_idx / p.tilesW;
        ht = q % p.tilesH;
        bt = q / p.tilesH;
      }
      unit_f += step_f; unit_s += step_s;
      if (unit_f >= units_f) { unit_f -= units_f; ++unit_s; }
      const int gp_first = ((bt * p.TB) * p.Ho + ht * p.TH) * p.Wo + wt * p.TW;
      const int n0 = n_idx * BN;

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
        // consecutive tiles of a CTA often share the N tile (M-fast walks; N-fast ones whose grid is a multiple of tilesN):
        // reload only on change, otherwise the ~0.7 us global-load latency + two barriers sit between every two tiles
        const float* brow = p.bias + (p.bias_bstride ? static_cast<long long>(gp_first / p.rows_per_batch) * p.bias_bstride : 0) + n0;
        if (brow != sbias_src) {              // uniform across the epilogue threads
          epi_bar_sync();                     // previous tile's readers are done with sbias
          for (int i = threadIdx.x; i < BN; i += kNumEpiThreads) sbias[i] = (n0 + i < p.N) ? __ldg(brow + i) : 0.f;
          epi_bar_sync();
          sbias_src = brow;
        }
      }
      // output pixels (GEMM rows) of this thread's two accumulator rows
      int e_gp[kMB][2];
      bool e_ok[kMB][2];
#pragma unroll
      for (int hb = 0; hb < kMB; ++hb)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int ew = wt * p.TW + e_tw[hb][h], eh = ht * p.TH + e_th[hb][h], eb = bt * p.TB + e_tb[hb][h];
          e_ok[hb][h] = (ew < p.Wo) && (eh < p.Ho) && (eb < p.Bo);
          e_gp[hb][h] = (eb * p.Ho + eh) * p.Wo + ew;
        }
      // folded LayerNorm: the scalars of this thread's two rows (requested before the accumulator wait)
      float ln_a0[2] = {0.f, 0.f}, ln_a1[2] = {1.f, 1.f};   // on_cols 0: (mean, rstd) of the row;  on_cols 1: (s[m], c[m]) of the output row
      if constexpr (kLnIn) {
        if (p.ln_on_cols) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (e_ok[0][h]) {
              ln_a0[h] = __ldg(p.ln_colsum + e_gp[0][h]);
              ln_a1[h] = p.ln_rowbias ? __ldg(p.ln_rowbias + e_gp[0][h]) : 0.f;
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
        // request the next tile's row partials (GEMM view: unit_f / unit_s already point at the next tile)
        if (!p.ln_on_cols && p.ln_parts <= 2 * kLnPre && t + t_step < t_end)
          ln_prefetch((p.n_fast ? unit_s : unit_f) * kBlockM + e_row0 + (lane & 15));
      }
      // residual (modes 3 / 7, lane 0): chunk j = ochunks hb + c of this warp's chunks of the tile -> staging box `box`,
      // completing on the box's mbarrier.  Rows and columns past the output are zero-filled.
      auto resid_chunks = [&] { return min(BN / 32, (p.N - n_idx * BN + 31) / 32); };
      auto req_resid = [&](int j, int box) {
        const int och = resid_chunks();
        const int hb = (kMB > 1 && j >= och) ? 1 : 0, c = j - hb * och;
        const int b_row0 = e_row0 + 64 * hb;
        uint64_t* bar = rbar + warp * kBoxes + box;
        mbar_arrive_expect_tx(bar, 1024);
        tma_load_4d(sstage + warp * kStgWarp + box * 1024, &p.tmR, bar, n_idx * BN + c * 32, wt * p.TW + (b_row0 % p.TW),
                    ht * p.TH + ((b_row0 / p.TW) % p.TH), bt * p.TB + b_row0 / (p.TW * p.TH));
      };
      // the tile's first kBoxes boxes are requested under its mainloop, once the first k-block's products are issued, and once
      // the stores of the previous tile have read them
      mainloop(ks * p.kb_per_split, min(p.kb_total, ks * p.kb_per_split + p.kb_per_split), [&] {
        if constexpr (kResidTma) {
          if (resid_tma && lane == 0) {
            bulk_wait_read<0>();
            const int n = min(kBoxes, kMB * resid_chunks());
            for (int j = 0; j < n; ++j) req_resid(j, (st_buf + j) & (kBoxes - 1));
          }
          __syncwarp();
        }
      });

      // ---- the epilogue, straight from the wgmma registers (no barrier between the warpgroups).  Each warp walks the 32-column
      // chunks of its 16 rows: per-element fp32 arithmetic on the thread's 2 rows x 8 columns of the chunk, bf16 pack, two
      // stmatrix into one 1 KB staging box of this warp (16 rows of 64 B, SWIZZLE_64B pattern), then lane 0 hands the box to the
      // TMA unit (cp.async.bulk.tensor store; out-of-range rows / columns are clipped by the tensor map).  The kBoxes boxes of a
      // warp rotate: a box is rewritten once the store issued from it kBoxes - 1 chunks ago has read it.  fp32 output and split-K
      // partials (mode 0) skip the boxes: each thread stores its column pairs to global memory.  Bias / LayerNorm tables are read
      // from shared memory as 8-byte broadcasts (columns 2 (lane % 4) + {0, 1}).  A 256-row tile runs this once per 64-row block
      // of the warpgroup.
      const uint32_t stg_s = smem_u32(sstage) + warp * kStgWarp;
      // what modes 3-7 fix at compile time, mode 0 reads from the launch
      const bool split = MODE == 0 && p.ksplit > 1;                      // raw fp32 partials, reduced by splitk_reduce_kernel
      const bool f32_out = MODE == 0 && (split || p.out_f32);
      const bool geglu = kGegluEpi || (MODE == 0 && p.act == ACT_GEGLU);
      constexpr int kChunks = kGegluEpi ? BN / 64 : BN / 32;            // 32-column output chunks per tile
      const int outc = geglu ? BN / 2 : BN;                             // output columns per tile
      const int ocol0 = n_idx * outc;
      const int nvalid = (geglu ? p.N / 2 : p.N) - ocol0;               // output columns of this tile inside the output
      const int ochunks = geglu ? BN / 64 : min(BN / 32, (nvalid + 31) / 32);
      const int tq2 = 2 * (lane & 3);                                    // this thread's first column of every 8-column group
      // residual, mode 0: the thread's 2 bf16 of row h and 8-column group jj of a chunk, one 4-byte load each (one 2-byte load
      // for a pair that ends at N, none past it), requested a chunk ahead
      const bool do_resid = MODE == 0 && !split && !geglu && p.resid != nullptr;
      // stmatrix / ldmatrix x4 per 16 columns u of a box: matrix i = rows (i & 1) * 8 + 0..7 of 16-byte unit 2 u + i / 2; lane l
      // addresses row l % 8 of matrix l / 8.  SWIZZLE_64B: unit q of box row rr sits at unit q ^ ((rr / 2) % 4)
      const int x4_row = ((lane >> 3) & 1) * 8 + (lane & 7);
      auto x4_addr = [&](uint32_t box, int u) { return box + x4_row * 64 + (((2 * u + (lane >> 4)) ^ ((x4_row >> 1) & 3)) << 4); };
      const bool row_bias = MODE == 0 && p.bias && !bias_uniform && !split;   // a tile that one bias row does not cover
#pragma unroll
      for (int hb = 0; hb < kMB; ++hb) {
        const int b_row0 = e_row0 + 64 * hb;
        const int ow = wt * p.TW + (b_row0 % p.TW), oh = ht * p.TH + ((b_row0 / p.TW) % p.TH), ob = bt * p.TB + b_row0 / (p.TW * p.TH);
        const uint32_t* rrow[2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
          rrow[h] = (do_resid && e_ok[hb][h]) ? reinterpret_cast<const uint32_t*>(p.resid + static_cast<long long>(e_gp[hb][h]) * p.ldr + ocol0 + tq2)
                                              : nullptr;
        // row_bias: the bias row of the thread's row h (computed where it is used: kept live, it costs registers the whole epilogue)
        auto rbias = [&](int h) { return p.bias + static_cast<long long>(e_gp[hb][h] / p.rows_per_batch) * p.bias_bstride + n0; };
        auto load_resid = [&](int c, uint32_t (&rr)[2][4]) {
          if (MODE != 0 || c * 32 + 32 <= nvalid) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) rr[h][jj] = rrow[h] ? __ldg(rrow[h] + (c * 32 + 8 * jj) / 2) : 0u;
          } else {                       // the last chunk of a ragged N
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const uint32_t* q = rrow[h] + (c * 32 + 8 * jj) / 2;
                const int left = nvalid - (c * 32 + 8 * jj + tq2);     // columns of the pair inside the output
                rr[h][jj] = !rrow[h] || left <= 0 ? 0u : left >= 2 ? __ldg(q) : __ldg(reinterpret_cast<const unsigned short*>(q));
              }
          }
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
        for (int c = 0; c < kChunks; ++c) {
          if (c >= ochunks) break;
          float o[4][2][2];                                              // [8-column group][row][column]
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int n = c * 32 + 8 * jj + tq2;                         // tile column of o[jj][.][0]
            const float* va = acc[hb] + 4 * (4 * c + jj);                // {row 0: n, n + 1; row 8: n, n + 1}
            if (split) {
#pragma unroll
              for (int h = 0; h < 2; ++h) { o[jj][h][0] = va[2 * h]; o[jj][h][1] = va[2 * h + 1]; }
            } else if (geglu && c < BN / 64) {   // (c: mode 0 unrolls BN / 32 chunks, GEGLU has BN / 64)
              const float* vg = acc[hb] + 4 * (BN / 16 + 4 * c + jj);    // gate columns outc + n
              if constexpr (kLnIn) {   // GEGLU over a folded LayerNorm: r * (acc - mu * s) + c == fma(r, acc, fma(-r mu, s, c))
                const float2 sa = lds_f2(slnx_s + 4 * n), ca = lds_f2(sbias_s + 4 * n);
                const float2 sg = lds_f2(slnx_s + 4 * (outc + n)), cg = lds_f2(sbias_s + 4 * (outc + n));
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  o[jj][h][0] = fmaf(ln_a1[h], va[2 * h], fmaf(nrm[h], sa.x, ca.x)) * gelu_fast_f(fmaf(ln_a1[h], vg[2 * h], fmaf(nrm[h], sg.x, cg.x)));
                  o[jj][h][1] = fmaf(ln_a1[h], va[2 * h + 1], fmaf(nrm[h], sa.y, ca.y)) * gelu_fast_f(fmaf(ln_a1[h], vg[2 * h + 1], fmaf(nrm[h], sg.y, cg.y)));
                }
              } else {
                const float2 bas = bias_uniform ? lds_f2(sbias_s + 4 * n) : make_float2(0.f, 0.f);
                const float2 bgs = bias_uniform ? lds_f2(sbias_s + 4 * (outc + n)) : make_float2(0.f, 0.f);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  float2 ba = bas, bg = bgs;
                  if (MODE == 0 && row_bias && e_ok[hb][h]) {
                    const float* b = rbias(h);
                    ba = make_float2(__ldg(b + n), __ldg(b + n + 1));
                    bg = make_float2(__ldg(b + outc + n), __ldg(b + outc + n + 1));
                  }
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
            } else {                   // modes 0 / 3 / 7: acc + bias, then (mode 0) * alpha and the activation, then + residual
              // (_rn: every step rounds on its own, as the kernel always has; no FMA contraction across them)
              const float2 bb = bias_uniform ? lds_f2(sbias_s + 4 * n) : make_float2(0.f, 0.f);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                o[jj][h][0] = __fadd_rn(va[2 * h], bb.x);
                o[jj][h][1] = __fadd_rn(va[2 * h + 1], bb.y);
              }
            }
          }
          if (MODE == 0 && !split && !geglu) {
            if (row_bias) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                if (!e_ok[hb][h]) continue;
                const float* b = rbias(h);
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                  const int n = c * 32 + 8 * jj + tq2;
                  const float* va = acc[hb] + 4 * (4 * c + jj) + 2 * h;
                  o[jj][h][0] = __fadd_rn(va[0], n < nvalid ? __ldg(b + n) : 0.f);
                  o[jj][h][1] = __fadd_rn(va[1], n + 1 < nvalid ? __ldg(b + n + 1) : 0.f);
                }
              }
            }
            alpha_act8(&o[0][0][0], p.alpha, p.act);
            alpha_act8(&o[2][0][0], p.alpha, p.act);
          }
          if (resid_tma) {
            // the residual box of this chunk, read at the addresses the stmatrix below writes: it arrives in the fragment layout
            mbar_wait(&rbar[warp * kBoxes + st_buf], (rphase >> st_buf) & 1u);
            rphase ^= 1u << st_buf;
            uint32_t rb[2][4];
#pragma unroll
            for (int u = 0; u < 2; ++u) ldmatrix_x4(x4_addr(stg_s + st_buf * 1024, u), rb[0][2 * u], rb[1][2 * u], rb[0][2 * u + 1], rb[1][2 * u + 1]);
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const float2 x = unpack_bf16x2(rb[h][jj]);
                o[jj][h][0] = __fadd_rn(o[jj][h][0], x.x);
                o[jj][h][1] = __fadd_rn(o[jj][h][1], x.y);
              }
          } else if (do_resid) {
            uint32_t rn[2][4];
            const bool more = c + 1 < ochunks;
            if (more) load_resid(c + 1, rn);
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const float2 x = unpack_bf16x2(rr[h][jj]);
                o[jj][h][0] = __fadd_rn(o[jj][h][0], x.x);
                o[jj][h][1] = __fadd_rn(o[jj][h][1], x.y);
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
          if (f32_out) {
            // fp32 columns pairs straight to global memory: float2 where the row stride keeps the pair 8-byte aligned (out is
            // 16-byte aligned, the partials' row stride N is a multiple of 4), single floats otherwise and at the end of a row
            float* const base = split ? p.partial + static_cast<long long>(ks) * p.Bo * p.Ho * p.Wo * p.N : reinterpret_cast<float*>(p.out);
            const long long ld = split ? p.N : p.ldo;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              if (!e_ok[hb][h]) continue;
              float* const row = base + static_cast<long long>(e_gp[hb][h]) * ld + ocol0 + c * 32 + tq2;
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const int left = nvalid - (c * 32 + 8 * jj + tq2);
                if (left >= 2 && !(ld & 1)) {
                  *reinterpret_cast<float2*>(row + 8 * jj) = make_float2(o[jj][h][0], o[jj][h][1]);
                } else {
                  if (left >= 1) row[8 * jj] = o[jj][h][0];
                  if (left >= 2) row[8 * jj + 1] = o[jj][h][1];
                }
              }
            }
            continue;
          }
          if (resid_tma) {
            // this box was refilled only once its previous store had read it.  The box of the previous chunk j - 1 takes the
            // residual of chunk j - 1 + kBoxes, once the store of chunk j - 1 has read it
            const int j = hb * ochunks + c;
            if (lane == 0 && j >= 1 && j - 1 + kBoxes < kMB * ochunks) {
              bulk_wait_read<0>();
              req_resid(j - 1 + kBoxes, (st_buf + kBoxes - 1) & (kBoxes - 1));
            }
          } else if (lane == 0) {
            bulk_wait_read<kBoxes - 1>();  // the box about to be rewritten was handed to the TMA unit kBoxes - 1 chunks ago
          }
          __syncwarp();
          const uint32_t box = stg_s + st_buf * 1024;
#pragma unroll
          for (int u = 0; u < 2; ++u)
            stmatrix_x4(x4_addr(box, u), pack_bf16x2(o[2 * u][0][0], o[2 * u][0][1]), pack_bf16x2(o[2 * u][1][0], o[2 * u][1][1]),
                        pack_bf16x2(o[2 * u + 1][0][0], o[2 * u + 1][0][1]), pack_bf16x2(o[2 * u + 1][1][0], o[2 * u + 1][1][1]));
          fence_proxy_async_smem();      // every writer: generic-proxy stores -> visible to the TMA (async proxy) read
          __syncwarp();
          if (lane == 0) {
            tma_store_4d(&p.tmO, sstage + warp * kStgWarp + st_buf * 1024, ocol0 + c * 32, ow, oh, ob);
            bulk_commit();
          }
          st_buf = (st_buf + 1) & (kBoxes - 1);
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
              if ((lane & 3) == 0 && e_ok[hb][h])
                reinterpret_cast<float2*>(p.stats_out)[static_cast<long long>(n_idx * 2 + par) * (static_cast<long long>(p.Bo) * p.Ho * p.Wo) + e_gp[hb][h]] =
                    make_float2(su, sq);
            }
        }
      }
    }
    if (lane == 0) bulk_wait<0>();     // every TMA store of this thread has completed before the CTA may exit
  }
}

// split-K reduction + epilogue: out[m, n] = act(alpha * (sum_s partial[s, m, n] + bias)) + resid
__global__ void splitk_reduce_kernel(const float* __restrict__ partial, int ksplit, long long M, int N,
                                     const float* __restrict__ bias, long long bias_bstride, int rows_per_batch,
                                     const __nv_bfloat16* __restrict__ resid, long long ldr, void* out,
                                     long long ldo, int out_f32, int act, float alpha) {
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
template <int BM, int BN, int STAGES, int MODE>
static int launch_igemm(const IgemmParams& p0, int num_units, void* stream) {
  constexpr bool kLn = MODE == 5 || MODE == 6;       // one more [BN] fp32 table (colsum / column mean)
  constexpr bool kResid = MODE == 3 || MODE == 7;     // one residual mbarrier per staging box
  constexpr size_t need = STAGES * (BM + BN) * kBlockK * 2 + 2 * STAGES * 8 + BN * 4 + (kLn ? BN * 4 : 0) +
                          kNumEpiWarps * igemm_boxes(BM) * (1024 + (kResid ? 8 : 0));   // (see igemm_kernel)
  // + up to 1024 bytes of slack for the 1024-byte alignment of the operand ring (the LN modes at BN 256 may get less: the dynamic
  // window starts 1024-aligned in practice, and the kernel traps if its carve-up would not fit)
  constexpr size_t smem = (need + 1024 <= 227 * 1024) ? need + 1024 : 227 * 1024;
  static_assert(need + 896 <= 227 * 1024, "igemm shared-memory budget");
  constexpr int threads = igemm_threads(BM, BN);
  IgemmParams p = p0;
  p.smem_bytes = static_cast<unsigned>(smem);
  static bool configured = false;
  if (!configured) {
    VDB_CUDA_CHECK(cudaFuncSetAttribute(igemm_kernel<BM, BN, STAGES, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(smem)));
    configured = true;
  }
  const int grid = std::min(num_units, num_sms());
  return launch(igemm_kernel<BM, BN, STAGES, MODE>, dim3(grid), dim3(threads), smem, stream, p);
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

// The last run_igemm decision on this thread (vdb_igemm_last_plan): BN, STAGES, MODE, ksplit, grid, tilesM, tilesN; and its tile
// height (vdb_igemm_last_bm)
constexpr int kPlanFields = 7;
static thread_local int g_last_plan[kPlanFields] = {0};
static thread_local int g_last_bm = 0;
static thread_local int g_last_n_fast = 0;     // and its tile walk (vdb_igemm_last_n_fast)

// bf16 output leaves through a TMA output map (16-byte aligned base and row stride), the split-K reduction stores fp32 rows as
// float4 and the fp32 epilogue column pairs as float2, so out / resid must be 16-byte aligned.  Checked before any tensor map is
// built, so that a bad pointer is reported as an argument error.
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

static int pow2_ceil(int v) { int t = 1; while (t < v) t <<= 1; return t; }

// M tile = BM output pixels as a (TW, TH, TB) box of the (W, H, B) pixel grid; box extents are
// powers of two so that TW*TH*TB == BM (rows past the grid are zero-filled by TMA and masked on store).
// GEMM view (one row of M "pixels"): the box is always BM rows.
static void set_tile_shape(IgemmParams& p, int BM, int Wo, int Ho, int Bo, bool gemm_view) {
  p.Wo = Wo; p.Ho = Ho; p.Bo = Bo;
  const int TW = gemm_view ? BM : std::min(pow2_ceil(Wo), BM);
  const int TH = std::min(pow2_ceil(Ho), BM / TW);
  const int TB = BM / (TW * TH);
  p.TW = TW; p.TH = TH; p.TB = TB;
  p.tilesW = (Wo + TW - 1) / TW;
  p.tilesH = (Ho + TH - 1) / TH;
  p.tilesB = (Bo + TB - 1) / TB;
}

// one bias row per tile: shared bias, or per-image rows with tiles that never straddle two images
static bool one_bias_row(const IgemmParams& p, int BM, const IgemmEpilogue& e) {
  const int rpb = e.rows_per_batch > 0 ? e.rows_per_batch : 1;
  return e.bias == nullptr || e.bias_bstride == 0 ||
         (p.TB == 1 && (static_cast<long long>(p.Ho) * p.Wo == rpb || (p.Ho == 1 && p.Bo == 1 && rpb % BM == 0)));
}

// `bn` argument of the entry points: a forced tile width, optionally with this flag for the 256-row tile (VDB_IGEMM_BM256)
constexpr int kForceBM256 = 0x1000;

// The (BM, BN) tile of a launch, from the shape alone unless the caller forces it.
//
// Model: the persistent grid runs waves = ceil(tiles / #SMs) rounds of one tile per CTA.  A k-block of a BM x BN tile costs the
// longer of its wgmma time, 4 BN clocks per 128 rows (4096 dense bf16 FLOP per clock per SM), and its operand fill, (BM + BN) x
// 128 bytes from L2 at kFillBytesPerClk per SM; a tile adds kTileClocks per 128 rows of pipeline fill and epilogue tail, a
// split-K launch kSplitKClocks for its reduction pass.
// kFillBytesPerClk = 42 is fitted to the 3x3 conv B 8, 64x64, 320 -> 320 timed alone at BN 64 / 128 / 160
// (tools/igemm_tile_sweep.py) on an H100 80GB HBM3 at 700 W, taking 1.83 GHz: 590, 888 and 809 clocks per k-block.  So every
// 128-row tile is fill-bound, (16384 + 128 BN) / 42 clocks per k-block against 4 BN of wgmma, and the 256 x 160 tile is the
// first that is not: 1280 clocks of wgmma over 1268 of fill, for twice the rows of a 128 x 160 k-block that takes 878.
// kTileClocks and kSplitKClocks were tuned against a fill term of 90 B/clk (1500 and 12000 clocks) on the 16x16 and 8x8 levels,
// which have not been re-measured: they keep that ratio to the fill term, so no 128-row choice moves.
//
// A 256-row tile needs the plain TMA-store epilogue or its statistics-writing variant (modes 3 / 7 of igemm_kernel) and is
// taken only where its tiles make one wave that covers at least 7/8 of the SMs (the 32x32 level of the UNet at batch 8: 128
// tiles).  Fewer tiles (the 16x16 and 8x8 levels) would leave SMs idle for the whole launch.  More than one wave (the 64x64
// level: 256 tiles) doubles the rows of A the CTAs of a wave hold in L2 between them: measured on the same card, its 3x3
// convs from 640 and 960 channels ran 12 % and 44 % slower on 256 rows and the level as a whole lost.
struct Tile { int BM, BN; };
constexpr double kFillBytesPerClk = 42.0, kTileClocks = 1500.0 * 90.0 / kFillBytesPerClk, kSplitKClocks = 12000.0 * 90.0 / kFillBytesPerClk;

static Tile choose_tile(int Wo, int Ho, int Bo, bool gemm_view, long long N, int kb_total, const IgemmEpilogue& e, int bn_arg,
                        int ksplit_forced, const void* workspace) {
  const int bn_forced = bn_arg & ~kForceBM256;
  if (bn_arg & kForceBM256) return Tile{256, bn_forced};
  Tile best_tile{kBlockM, pick_bn(static_cast<int>(N), e.act, bn_forced)};
  if (bn_forced || e.act == ACT_GEGLU || kb_total < 8) return best_tile;
  const bool stats = e.ln_stats != nullptr || e.stats_out != nullptr;
  if (stats) ksplit_forced = 1;                          // the statistics ride on the single-pass TMA-store epilogues
  IgemmParams s128, s256;
  set_tile_shape(s128, 128, Wo, Ho, Bo, gemm_view);
  set_tile_shape(s256, 256, Wo, Ho, Bo, gemm_view);
  const bool can256 = !e.ln_stats && !e.out_f32 && e.act == ACT_NONE && e.alpha == 1.f && (N % 32) == 0 && ksplit_forced <= 1 &&
                      one_bias_row(s256, 256, e);
  const Tile cand[5] = {{256, 160}, {128, 256}, {128, 160}, {128, 128}, {128, 64}};
  double best = 1e30;
  for (const Tile& c : cand) {
    const IgemmParams& sh = c.BM == 256 ? s256 : s128;
    const long long tiles = static_cast<long long>(sh.tilesW) * sh.tilesH * sh.tilesB * ((N + c.BN - 1) / c.BN);   // (a partial
                                                                                         // last N tile is computed in full)
    if (c.BM == 256 && (!can256 || tiles * 8 < num_sms() * 7LL || tiles > num_sms())) continue;
    // split-K exactly as run_igemm decides it: small MN grids with a deep K run kb / ks blocks per unit plus a reduction pass
    long long ks = 1;
    if (ksplit_forced > 0) ks = ksplit_forced;
    else if (tiles * 2 <= num_sms() && kb_total >= 16 && (N % 4) == 0 && workspace)
      ks = std::max<long long>(1, std::min<long long>(std::min<long long>(num_sms() / tiles, kb_total / 8), 16));
    const long long waves = (tiles * ks + num_sms() - 1) / num_sms();
    const double rows = c.BM / 128.0;
    const double per_kb = std::max(4.0 * c.BN * rows, (c.BM + c.BN) * 128.0 / kFillBytesPerClk);
    const double kb_unit = static_cast<double>((kb_total + ks - 1) / ks);
    const double cost = static_cast<double>(waves) * (kb_unit * per_kb + kTileClocks * rows) + (ks > 1 ? kSplitKClocks : 0.0);
    if (cost < best * 0.97) { best = cost; best_tile = c; }     // (prefer the larger tile unless the gain is clear)
  }
  return best_tile;
}

// Finish IgemmParams (split-K, B map, epilogue) and launch; p holds the M tiling of `tile` (set_tile_shape).
static int run_igemm(IgemmParams& p, const void* Wt, long long N, long long Ktot, long long ldw,
                     const IgemmEpilogue& e, Tile tile, int ksplit_forced, void* workspace,
                     size_t ws_bytes, void* stream) {
  const bool ln_in = e.ln_stats != nullptr, st_out = e.stats_out != nullptr;
  if (ln_in || st_out) ksplit_forced = 1;               // the statistics ride on the single-pass TMA-store epilogues
  const int BM = tile.BM, BN = tile.BN;
  if (BN != 64 && BN != 128 && BN != 160 && BN != 256) return set_error(VDB_ERR_INVALID, "igemm: bad BN");
  if (BM == 256 && BN != 160) return set_error(VDB_ERR_INVALID, "igemm: the 256-row tile is 160 columns wide");
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
  int rc = make_tmap_2d(&p.tmB, Wt, static_cast<uint64_t>(Ktot), static_cast<uint64_t>(N),
                        static_cast<uint64_t>(ldw) * 2, kBlockK, BN);
  if (rc) return rc;
  const int num_tiles = mn_tiles * p.ksplit;
  // Tile walk.  M-fast, the CTAs of a wave share a few N tiles and read a band of A rows per N tile; when A is the larger
  // operand that band has usually left the L2 before the next N tile of the same rows comes round (ff-down at 64x64: 84 MB of A,
  // two N tiles two waves apart), so A is read from HBM once per N tile.  N-fast, a wave takes every N tile of its rows together
  // and A is read once; W, the smaller operand, is the one re-read.  A's bytes: output pixels times the channels of every A map
  // (the pixels of a stride-2 conv's four parity maps add up to the input's).
  {
    long long a_chan = 0;
    for (int m = 0; m < kMaxA; ++m) {
      int c = 0;
      for (int s = 0; s < p.nseg; ++s)
        if (p.seg[s].tmap == m) c = std::max(c, p.seg[s].c0 + p.seg[s].nkb * kBlockK);
      a_chan += c;
    }
    p.n_fast = p.ksplit == 1 && p.tilesN > 1 && M * a_chan > N * Ktot;
  }
  // epilogue specialisation (see igemm_kernel): 3 = plain bf16 fast path, 4 = GEGLU, 0 = everything else
  int mode = 0;
  if (p.ksplit == 1 && !e.out_f32 && one_bias_row(p, BM, e)) {
    if (e.act == ACT_GEGLU && BN == 256) mode = 4;
    else if (e.act == ACT_NONE && e.alpha == 1.f && (N % 32) == 0) mode = 3;
  }
  // bf16 output leaves through shared memory + cp.async.bulk.tensor: a warp's 16 rows x 32 columns are one box of the output
  // tensor map, which clips the rows and columns past the output (the M tile shapes hold at least 16 / (bw * bh) images;
  // check_epilogue_pointers has checked the alignment of out / resid).  fp32 output and split-K partials are stored directly.
  if (!e.out_f32 && p.ksplit == 1) {
    const int bw = std::min(p.TW, 16), bh = std::min(p.TH, 16 / bw), bb = 16 / (bw * bh);
    const long long ncols = (e.act == ACT_GEGLU) ? N / 2 : N;
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
  if (e.resid && (mode == 3 || mode == 7)) {
    // the residual enters through the staging boxes: the output map's geometry over resid / ldr (the interleaved-output upsample
    // modes take no residual)
    const int bw = std::min(p.TW, 16), bh = std::min(p.TH, 16 / bw), bb = 16 / (bw * bh);
    rc = make_tmap_4d_sw64(&p.tmR, e.resid, static_cast<uint64_t>(N), static_cast<uint64_t>(p.Wo), static_cast<uint64_t>(p.Ho),
                           static_cast<uint64_t>(p.Bo), static_cast<uint64_t>(e.ldr) * 2, static_cast<uint64_t>(p.Wo) * e.ldr * 2,
                           static_cast<uint64_t>(p.Ho) * p.Wo * e.ldr * 2, 32, bw, bh, bb);
    if (rc) return rc;
  }
  if (BM == 256 && mode != 3 && mode != 7)
    return set_error(VDB_ERR_UNSUPPORTED, "igemm: the 256-row tile needs the plain TMA-store epilogue (bf16 out, no activation, alpha 1, "
                                          "N %% 32 == 0, one bias row per tile, no split-K, no LayerNorm input)");
  {
    const int stages = BN == 64 ? 8 : BN == 128 ? 6 : (BN == 160 && BM == 128) ? 5 : 4;   // (as instantiated below)
    const int plan[kPlanFields] = {BN, stages, mode, p.ksplit, std::min(num_tiles, num_sms()), tilesM, p.tilesN};
    for (int i = 0; i < kPlanFields; ++i) g_last_plan[i] = plan[i];
    g_last_bm = BM;
    g_last_n_fast = p.n_fast;
  }
  if (BM == 256) {
    rc = mode == 7 ? launch_igemm<256, 160, 4, 7>(p, num_tiles, stream) : launch_igemm<256, 160, 4, 3>(p, num_tiles, stream);
  } else if (mode == 7) {
    switch (BN) {
      case 64: rc = launch_igemm<128, 64, 8, 7>(p, num_tiles, stream); break;
      case 128: rc = launch_igemm<128, 128, 6, 7>(p, num_tiles, stream); break;
      case 160: rc = launch_igemm<128, 160, 5, 7>(p, num_tiles, stream); break;
      default: rc = launch_igemm<128, 256, 4, 7>(p, num_tiles, stream); break;
    }
  } else if (mode == 6) {
    rc = launch_igemm<128, 256, 4, 6>(p, num_tiles, stream);
  } else if (mode == 5) {
    switch (BN) {
      case 64: rc = launch_igemm<128, 64, 8, 5>(p, num_tiles, stream); break;
      case 128: rc = launch_igemm<128, 128, 6, 5>(p, num_tiles, stream); break;
      case 160: rc = launch_igemm<128, 160, 5, 5>(p, num_tiles, stream); break;
      default: rc = launch_igemm<128, 256, 4, 5>(p, num_tiles, stream); break;
    }
  } else if (mode == 4) {
    rc = launch_igemm<128, 256, 4, 4>(p, num_tiles, stream);
  } else if (mode == 3) {
    switch (BN) {
      case 64: rc = launch_igemm<128, 64, 8, 3>(p, num_tiles, stream); break;
      case 128: rc = launch_igemm<128, 128, 6, 3>(p, num_tiles, stream); break;
      case 160: rc = launch_igemm<128, 160, 5, 3>(p, num_tiles, stream); break;
      default: rc = launch_igemm<128, 256, 4, 3>(p, num_tiles, stream); break;
    }
  } else {
    switch (BN) {
      case 64: rc = launch_igemm<128, 64, 8, 0>(p, num_tiles, stream); break;
      case 128: rc = launch_igemm<128, 128, 6, 0>(p, num_tiles, stream); break;
      case 160: rc = launch_igemm<128, 160, 5, 0>(p, num_tiles, stream); break;
      default: rc = launch_igemm<128, 256, 4, 0>(p, num_tiles, stream); break;
    }
  }
  if (rc || p.ksplit == 1) return rc;
  const long long total = M * (N / 4);
  const int threads = 256;
  const int blocks = static_cast<int>(std::min<long long>((total + threads - 1) / threads, num_sms() * 8LL));
  return launch(splitk_reduce_kernel, dim3(blocks), dim3(threads), 0, stream, p.partial, p.ksplit, M, static_cast<int>(N), p.bias,
                p.bias_bstride, p.rows_per_batch, p.resid, p.ldr, p.out, p.ldo, p.out_f32, p.act, p.alpha);
}

}  // namespace vdb

using namespace vdb;

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

// see include/vdb200.h
int vdb_igemm_last_plan(int* out, int n) {
  for (int i = 0; out && i < n && i < kPlanFields; ++i) out[i] = g_last_plan[i];
  return kPlanFields;
}

// see include/vdb200.h
int vdb_igemm_last_bm(void) { return g_last_bm; }

// see include/vdb200.h
int vdb_igemm_last_n_fast(void) { return g_last_n_fast; }

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
  IgemmEpilogue e;
  e.bias = bias; e.bias_bstride = bias_bstride; e.rows_per_batch = static_cast<int>(rows_per_batch);
  e.resid = resid; e.ldr = ldr; e.out = out; e.ldo = ldo; e.out_f32 = out_f32; e.act = act; e.alpha = alpha;
  IgemmParams p;
  memset(&p, 0, sizeof(p));
  p.seg[0] = ASeg{0, 0, 0, static_cast<int16_t>((K + kBlockK - 1) / kBlockK), 0};
  p.nseg = 1;
  p.kb_total = p.seg[0].nkb + (A2 ? static_cast<int>((K2 + kBlockK - 1) / kBlockK) : 0);
  // GEMM view of the pixel grid: one row of M "pixels"; the box is always BM rows (TMA zero-fills past M)
  const Tile tile = choose_tile(static_cast<int>(M), 1, 1, true, N, p.kb_total, e, bn, ksplit, workspace);
  set_tile_shape(p, tile.BM, static_cast<int>(M), 1, 1, true);
  rc = make_tmap_4d(&p.tmA[0], A, K, M, 1, 1, lda * 2, lda * 2 * M, lda * 2 * M, kBlockK, p.TW, 1, 1);
  if (rc) return rc;
  if (A2) {
    rc = make_tmap_4d(&p.tmA[1], A2, K2, M, 1, 1, lda2 * 2, lda2 * 2 * M, lda2 * 2 * M, kBlockK, p.TW, 1, 1);
    if (rc) return rc;
    p.seg[1] = ASeg{1, 0, 0, static_cast<int16_t>((K2 + kBlockK - 1) / kBlockK), 0};
    p.nseg = 2;
  }
  for (int i = p.nseg; i < kMaxA; ++i) p.tmA[i] = p.tmA[0];
  return run_igemm(p, W, N, K + (A2 ? K2 : 0), ldw, e, tile, ksplit, workspace, ws_bytes, stream);
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
  IgemmEpilogue e;
  e.bias = bias; e.resid = resid; e.ldr = ldr; e.out = out; e.ldo = ldo; e.act = act;
  e.ln_stats = ln_stats; e.ln_mstat = ln_rows; e.ln_parts = ln_parts; e.ln_dim = ln_dim; e.ln_eps = ln_eps; e.ln_colsum = ln_colsum;
  e.ln_on_cols = ln_on_cols; e.ln_rowbias = ln_rowbias; e.stats_out = stats_out; e.stats_parts = stats_parts;
  IgemmParams p;
  memset(&p, 0, sizeof(p));
  p.seg[0] = ASeg{0, 0, 0, static_cast<int16_t>((K + kBlockK - 1) / kBlockK), 0};
  p.nseg = 1;
  p.kb_total = p.seg[0].nkb;
  const Tile tile = choose_tile(static_cast<int>(M), 1, 1, true, N, p.kb_total, e, bn, 1, nullptr);
  set_tile_shape(p, tile.BM, static_cast<int>(M), 1, 1, true);
  rc = make_tmap_4d(&p.tmA[0], A, K, M, 1, 1, lda * 2, lda * 2 * M, lda * 2 * M, kBlockK, p.TW, 1, 1);
  if (rc) return rc;
  for (int i = p.nseg; i < kMaxA; ++i) p.tmA[i] = p.tmA[0];
  return run_igemm(p, W, N, K, ldw, e, tile, 1, nullptr, 0, stream);
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
  const uint64_t eb = 2;
  const int nkb = C / kBlockK;
  IgemmEpilogue e;
  e.bias = bias; e.bias_bstride = bias_bstride; e.rows_per_batch = Ho * Wo;
  e.resid = resid; e.ldr = ldr; e.out = out; e.ldo = ldo; e.out_f32 = out_f32; e.act = act; e.alpha = 1.f;
  e.out_parity = out_parity;
  const Tile tile = choose_tile(Wo, Ho, B, false, N, (folded ? 4 : 9) * nkb + (skip1 ? Cs1 / kBlockK : 0) + (skip2 ? Cs2 / kBlockK : 0),
                                e, bn, ksplit, workspace);
  set_tile_shape(p, tile.BM, Wo, Ho, B, false);
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
  return run_igemm(p, Wt, N, static_cast<long long>(p.kb_total) * kBlockK, ldw, e, tile, ksplit, workspace, ws_bytes, stream);
}

}  // extern "C"
