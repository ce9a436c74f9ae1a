// vdb200 — semantic/style disentanglement: the rank adjustment of the image context (sm_90a).
//
// One item x [m, n] (m = 256 or 257 CLIP image tokens, n = 768 features) goes through
//   X = x - rowmean(x);  randomized PCA of X with q = 20 and niter subspace iterations (torch.pca_lowrank, center=False,
//   which works on A = X^T because m < n);  S scaled by a factor vector f;  x_new = U diag(S f) V^T + mean [+ X - U diag(S) V^T];
//   x_new *= std(x) / std(x_new).
//
// The 100 iterations are a chain of 201 dependent (n x m)(m x q) products and thin QRs: latency-bound, so the whole game is to
// keep X on chip.  One thread-block cluster of 8 CTAs (the portable maximum) holds one item: CTA r owns a block of ceil(m/8)
// rows of X in shared memory (33 x 768 x 4 B = 99 KB for m = 257), loaded once.  16-CTA clusters would halve the FMA work per
// SM but need the non-portable cluster attribute.  The FMA work is not what limits a call: each iteration also runs four
// serial q x q fp64 factorizations and six cluster barriers.
//
// In the orientation of x (Qn: n x q, Qm: m x q, both orthonormal):
//   Qn = qr(X^T R);  niter times { Qm = qr(X Qn);  Qn = qr(X^T Qm) };  C = X Qn  (= B^T of torch's B = Q^T A).
// X^T Qm is a sum over rows, i.e. over CTAs: each CTA writes its partial [n, q] product, reduces its 96-row slice of it from
// the 8 peers through distributed shared memory, orthonormalises the slices, and all-gathers them into a full Qn.  X Qn is
// local to each CTA's rows.  Every QR is CholeskyQR2: the q x q Gram matrix in fp64 (summed over the cluster in rank order),
// Cholesky and the triangular inverse in fp64 in every CTA, applied to the local rows in fp64; twice.
//
// The final SVD B = Ub S Vb^T needs only the eigen-decomposition of B B^T = C^T C (q x q, fp64 cyclic Jacobi in every CTA):
// U diag(S f) V^T = C (Ub diag(f) Ub^T) Qn^T, so with W = Ub diag(f) Ub^T
//   keep_remainder:  x_new = x + C (W - I) Qn^T        else:  x_new = mean + C W Qn^T.
// The signs of the QR columns and of the eigenvectors cancel in W and in C Qn^T.  Deterministic: fixed-order reductions only.
#include "common.cuh"
#include "host_util.h"

namespace vdb {

namespace {

constexpr int kN = 768;                  // features (the CLIP width)
constexpr int kQ = 20;                   // rank of the approximation
constexpr int kQQ = kQ * kQ;
constexpr int kCluster = 8;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kJ = kN / kThreads;        // feature columns per thread in the X^T Qm product and the reconstruction
constexpr int kSlice = kN / kCluster;    // rows of Qn each CTA reduces and orthonormalises
constexpr int kMaxRows = 320;            // m <= 320: 40 rows per CTA
constexpr int kJacobiSweeps = 16;
static_assert(kN % kThreads == 0 && kN % kCluster == 0 && kQ % 4 == 0, "layout");

struct Smem {
  float* x;        // [rows_cap][kN]    this CTA's rows of X (centred), later x_new
  float* pq;       // [kN][kQ]          partial X^T Qm, then the gathered Qn
  float* ys;       // [kSlice][kQ]      this CTA's slice of X^T Qm / Qn
  float* qm;       // [rows_cap][kQ]    local rows of R / Qm / C / C W
  float* mean;     // [rows_cap]
  float* w;        // [kQQ]             W (or W - I), fp32
  double* gpart;   // [2][kQQ]          this CTA's Gram partial (double-buffered: read by the peers)
  double* g;       // [kQQ]             summed Gram / Jacobi matrix
  double* l;       // [kQQ]             Cholesky factor / Jacobi eigenvectors
  double* linv;    // [kQQ]             L^-1 / the (c, s) pairs of a Jacobi round
  double* stat;    // [2]               this CTA's (sum, sum of squares), read by the peers
  double* red;     // [kWarps][2]
  int* perm;       // [kQ]              eigenvalue order, descending
};

VDB_DEVINL float4 ld_dsmem_f4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
VDB_DEVINL double ld_dsmem_f64(uint32_t addr) {
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(addr) : "memory");
  return v;
}

// Sum of (a, b) over the CTA in a fixed order; the result is valid in thread 0.
VDB_DEVINL void block_sum2(Smem& s, double& a, double& b) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { s.red[2 * warp] = a; s.red[2 * warp + 1] = b; }
  __syncthreads();
  if (threadIdx.x == 0) {
    a = 0.0; b = 0.0;
    for (int w = 0; w < kWarps; ++w) { a += s.red[2 * w]; b += s.red[2 * w + 1]; }
  }
}

// Unbiased standard deviation over the cluster's item from each CTA's (sum, sum of squares) in thread 0.
// Ends with every thread of every CTA holding the same value.
VDB_DEVINL double cluster_std(Smem& s, double sum, double sq, double count) {
  if (threadIdx.x == 0) { s.stat[0] = sum; s.stat[1] = sq; }
  cluster_sync_all();
  double ts = 0.0, tq = 0.0;
  for (int r = 0; r < kCluster; ++r) {
    const uint32_t a = mapa_u32(smem_u32(s.stat), static_cast<uint32_t>(r));
    ts += ld_dsmem_f64(a);
    tq += ld_dsmem_f64(a + 8);
  }
  const double var = (tq - ts * ts / count) / (count - 1.0);
  return sqrt(fmax(var, 0.0));
}

// G = sum over the cluster of Y^T Y (Y: this CTA's nrows x kQ rows), fp64, identical in every CTA.  One cluster barrier;
// the partial buffer alternates so a peer still reading the previous one is never overwritten.
VDB_DEVINL void cluster_gram(Smem& s, const float* y, int nrows, int& par) {
  double* gp = s.gpart + par * kQQ;
  for (int e = threadIdx.x; e < kQQ; e += kThreads) {
    const int a = e / kQ, b = e % kQ;
    double acc = 0.0;
    for (int i = 0; i < nrows; ++i) acc = fma(static_cast<double>(y[i * kQ + a]), static_cast<double>(y[i * kQ + b]), acc);
    gp[e] = acc;
  }
  cluster_sync_all();
  for (int e = threadIdx.x; e < kQQ; e += kThreads) {
    double acc = 0.0;
    for (int r = 0; r < kCluster; ++r) acc += ld_dsmem_f64(mapa_u32(smem_u32(gp + e), static_cast<uint32_t>(r)));
    s.g[e] = acc;
  }
  par ^= 1;
  __syncthreads();
}

// One CholeskyQR pass over the cluster's distributed rows: Y <- Y L^-T with G = L L^T.
VDB_DEVINL void cholqr_pass(Smem& s, float* y, int nrows, int& par) {
  cluster_gram(s, y, nrows, par);
  const int lane = threadIdx.x & 31;
  if (threadIdx.x < 32) {
    double* g = s.g;
    double* l = s.l;
    for (int k = 0; k < kQ; ++k) {             // right-looking Cholesky on the lower triangle of g
      if (lane == k) l[k * kQ + k] = sqrt(fmax(g[k * kQ + k], 1e-300));
      __syncwarp();
      if (lane > k && lane < kQ) l[lane * kQ + k] = g[lane * kQ + k] / l[k * kQ + k];
      __syncwarp();
      if (lane > k && lane < kQ)
        for (int j = k + 1; j <= lane; ++j) g[lane * kQ + j] -= l[lane * kQ + k] * l[j * kQ + k];
      __syncwarp();
    }
    if (lane < kQ) {                            // column `lane` of L^-1 by forward substitution
      const int c = lane;
      s.linv[c * kQ + c] = 1.0 / l[c * kQ + c];
      for (int i = c + 1; i < kQ; ++i) {
        double acc = 0.0;
        for (int k = c; k < i; ++k) acc = fma(l[i * kQ + k], s.linv[k * kQ + c], acc);
        s.linv[i * kQ + c] = -acc / l[i * kQ + i];
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nrows; i += kThreads) {   // y_new[c] = sum_{p <= c} Linv[c][p] y[p]
    double v[kQ];
#pragma unroll
    for (int c = 0; c < kQ; ++c) v[c] = y[i * kQ + c];
#pragma unroll
    for (int c = 0; c < kQ; ++c) {
      double acc = 0.0;
#pragma unroll
      for (int p = 0; p <= c; ++p) acc = fma(s.linv[c * kQ + p], v[p], acc);
      y[i * kQ + c] = static_cast<float>(acc);
    }
  }
  __syncthreads();
}

VDB_DEVINL void cholqr2(Smem& s, float* y, int nrows, int& par) {
  cholqr_pass(s, y, nrows, par);
  cholqr_pass(s, y, nrows, par);
}

// pq[j][:] = sum_i X[i][j] qm[i][:] over this CTA's rows (a partial of X^T Qm).
VDB_DEVINL void xt_q(Smem& s, int nr) {
  const int t = threadIdx.x;
  float acc[kJ][kQ];
#pragma unroll
  for (int k = 0; k < kJ; ++k)
#pragma unroll
    for (int c = 0; c < kQ; ++c) acc[k][c] = 0.f;
  const uint32_t qm = smem_u32(s.qm);
  for (int i = 0; i < nr; ++i) {
    float q[kQ];
#pragma unroll
    for (int c = 0; c < kQ; c += 4) {
      const float4 v = lds_f4(qm + (i * kQ + c) * 4);
      q[c] = v.x; q[c + 1] = v.y; q[c + 2] = v.z; q[c + 3] = v.w;
    }
#pragma unroll
    for (int k = 0; k < kJ; ++k) {
      const float xv = s.x[i * kN + t + k * kThreads];
#pragma unroll
      for (int c = 0; c < kQ; ++c) acc[k][c] = fmaf(xv, q[c], acc[k][c]);
    }
  }
#pragma unroll
  for (int k = 0; k < kJ; ++k) {
    float4* dst = reinterpret_cast<float4*>(s.pq + (t + k * kThreads) * kQ);
#pragma unroll
    for (int c = 0; c < kQ; c += 4) dst[c / 4] = make_float4(acc[k][c], acc[k][c + 1], acc[k][c + 2], acc[k][c + 3]);
  }
}

// qm[i][:] = X[i][:] . Qn for this CTA's rows.  Warp w owns rows w, w + 8, ... (RW of them; rows past nr repeat row 0 and
// are discarded), lane l the features l + 32 k; the 32 lane partials are summed with a butterfly.
template <int RW>
VDB_DEVINL void x_q(Smem& s, int nr) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc[RW][kQ];
  int row[RW];
#pragma unroll
  for (int r = 0; r < RW; ++r) {
    row[r] = warp + r * kWarps < nr ? warp + r * kWarps : 0;
#pragma unroll
    for (int c = 0; c < kQ; ++c) acc[r][c] = 0.f;
  }
  const uint32_t pq = smem_u32(s.pq);
#pragma unroll 2
  for (int j = lane; j < kN; j += 32) {
    float q[kQ];
#pragma unroll
    for (int c = 0; c < kQ; c += 4) {
      const float4 v = lds_f4(pq + (j * kQ + c) * 4);
      q[c] = v.x; q[c + 1] = v.y; q[c + 2] = v.z; q[c + 3] = v.w;
    }
#pragma unroll
    for (int r = 0; r < RW; ++r) {
      const float xv = s.x[row[r] * kN + j];
#pragma unroll
      for (int c = 0; c < kQ; ++c) acc[r][c] = fmaf(xv, q[c], acc[r][c]);
    }
  }
#pragma unroll
  for (int r = 0; r < RW; ++r)
#pragma unroll
    for (int c = 0; c < kQ; ++c)
#pragma unroll
      for (int o = 16; o; o >>= 1) acc[r][c] += __shfl_xor_sync(0xffffffffu, acc[r][c], o);
#pragma unroll
  for (int r = 0; r < RW; ++r)
    if (warp + r * kWarps < nr && lane < kQ) {
      float v = acc[r][0];
#pragma unroll
      for (int c = 1; c < kQ; ++c) v = lane == c ? acc[r][c] : v;
      s.qm[(warp + r * kWarps) * kQ + lane] = v;
    }
}

// Eigen-decomposition of the symmetric s.g (q x q, fp64) by cyclic Jacobi in round-robin order (10 disjoint rotations per
// round, 19 rounds per sweep); eigenvalues on the diagonal of s.g, eigenvectors in the columns of s.l.
VDB_DEVINL void jacobi_eig(Smem& s) {
  const int t = threadIdx.x;
  double* a = s.g;
  double* v = s.l;
  for (int e = t; e < kQQ; e += kThreads) v[e] = (e / kQ == e % kQ) ? 1.0 : 0.0;
  __syncthreads();
  for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
    int rotated = 0;
    for (int round = 0; round < kQ - 1; ++round) {
      // pair k of this round: (round, 19) for k = 0, else ((round + k) % 19, (round - k) % 19)
      auto pair = [&](int k, int& p, int& q) {
        int u = k == 0 ? round : (round + k) % (kQ - 1);
        int w = k == 0 ? kQ - 1 : (round - k + (kQ - 1)) % (kQ - 1);
        p = min(u, w); q = max(u, w);
      };
      if (t < kQ / 2) {
        int p, q;
        pair(t, p, q);
        const double apq = a[p * kQ + q], app = a[p * kQ + p], aqq = a[q * kQ + q];
        double c = 1.0, sn = 0.0;
        if (fabs(apq) > 1e-15 * sqrt(fabs(app * aqq)) && apq != 0.0) {
          rotated = 1;
          const double th = (aqq - app) / (2.0 * apq);
          const double tt = fabs(th) > 1e150 ? 0.5 / th : copysign(1.0, th) / (fabs(th) + sqrt(th * th + 1.0));
          c = 1.0 / sqrt(tt * tt + 1.0);
          sn = tt * c;
        }
        s.linv[2 * t] = c;                      // (c, s) of this round's rotations
        s.linv[2 * t + 1] = sn;
      }
      __syncthreads();
      if (t < kQ / 2 * kQ) {                    // columns: A <- A P, V <- V P
        const int k = t / kQ, i = t % kQ;
        int p, q;
        pair(k, p, q);
        const double c = s.linv[2 * k], sn = s.linv[2 * k + 1];
        const double aip = a[i * kQ + p], aiq = a[i * kQ + q];
        a[i * kQ + p] = c * aip - sn * aiq;
        a[i * kQ + q] = sn * aip + c * aiq;
        const double vip = v[i * kQ + p], viq = v[i * kQ + q];
        v[i * kQ + p] = c * vip - sn * viq;
        v[i * kQ + q] = sn * vip + c * viq;
      }
      __syncthreads();
      if (t < kQ / 2 * kQ) {                    // rows: A <- P^T A
        const int k = t / kQ, i = t % kQ;
        int p, q;
        pair(k, p, q);
        const double c = s.linv[2 * k], sn = s.linv[2 * k + 1];
        const double api = a[p * kQ + i], aqi = a[q * kQ + i];
        a[p * kQ + i] = c * api - sn * aqi;
        a[q * kQ + i] = sn * api + c * aqi;
      }
      __syncthreads();
    }
    if (!__syncthreads_or(rotated)) break;
  }
}

template <int RW>
__global__ void __launch_bounds__(kThreads, 1)
rank_adjust_kernel(const float* __restrict__ xg, int m, const float* __restrict__ R, int niter,
                   const float* __restrict__ factors, int keep_remainder, float* __restrict__ out, float* __restrict__ s_out,
                   float* __restrict__ u_out, float* __restrict__ v_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int rows_cap = (m + kCluster - 1) / kCluster;
  const int rank = static_cast<int>(cluster_ctarank());
  const int row0 = rank * rows_cap;
  const int nr = max(0, min(m, row0 + rows_cap) - row0);
  const int item = blockIdx.y;
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;

  Smem s;
  {
    unsigned char* p = smem_raw;
    s.gpart = reinterpret_cast<double*>(p); p += 2 * kQQ * 8;
    s.g = reinterpret_cast<double*>(p); p += kQQ * 8;
    s.l = reinterpret_cast<double*>(p); p += kQQ * 8;
    s.linv = reinterpret_cast<double*>(p); p += kQQ * 8;
    s.stat = reinterpret_cast<double*>(p); p += 2 * 8;
    s.red = reinterpret_cast<double*>(p); p += 2 * kWarps * 8;
    s.pq = reinterpret_cast<float*>(p); p += kN * kQ * 4;
    s.ys = reinterpret_cast<float*>(p); p += kSlice * kQ * 4;
    s.w = reinterpret_cast<float*>(p); p += kQQ * 4;
    s.perm = reinterpret_cast<int*>(p); p += kQ * 4;
    s.qm = reinterpret_cast<float*>(p); p += rows_cap * kQ * 4;
    s.mean = reinterpret_cast<float*>(p); p += ((rows_cap + 3) / 4) * 16;
    s.x = reinterpret_cast<float*>(p);
  }
  pdl_wait();

  // ---- load this CTA's rows, centre them, and the statistics of x ----
  const float* xi = xg + (static_cast<long long>(item) * m + row0) * kN;
  for (int e = t; e < nr * kN / 4; e += kThreads)
    reinterpret_cast<float4*>(s.x)[e] = __ldg(reinterpret_cast<const float4*>(xi) + e);
  for (int e = t; e < nr * kQ; e += kThreads) s.qm[e] = R[row0 * kQ + e];
  __syncthreads();
  double sum = 0.0, sq = 0.0;
  for (int i = warp; i < nr; i += kWarps) {
    double rs = 0.0;
    for (int j = lane; j < kN; j += 32) {
      const double v = s.x[i * kN + j];
      rs += v;
      sq = fma(v, v, sq);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, o);
    sum += rs;
    const float mu = static_cast<float>(rs / kN);
    for (int j = lane; j < kN; j += 32) s.x[i * kN + j] -= mu;
    if (lane == 0) s.mean[i] = mu;
  }
  sum = lane == 0 ? sum : 0.0;   // every lane of a warp holds the same row sums
  block_sum2(s, sum, sq);
  const double count = static_cast<double>(m) * kN;
  const double std_save = cluster_std(s, sum, sq, count);

  // ---- subspace iteration ----
  int par = 0;
  for (int it = 0;; ++it) {
    xt_q(s, nr);                                         // partial X^T Qm (Qm = R on the first pass)
    cluster_sync_all();
    for (int e = t; e < kSlice * kQ / 4; e += kThreads) { // reduce this CTA's slice from the peers, in rank order
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      const uint32_t src = smem_u32(s.pq + rank * kSlice * kQ) + e * 16;
      for (int r = 0; r < kCluster; ++r) {
        const float4 v = ld_dsmem_f4(mapa_u32(src, static_cast<uint32_t>(r)));
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
      reinterpret_cast<float4*>(s.ys)[e] = acc;
    }
    __syncthreads();
    cholqr2(s, s.ys, kSlice, par);                       // Qn slice
    cluster_sync_all();
    for (int e = t; e < kN * kQ / 4; e += kThreads) {    // all-gather Qn
      const int r = e / (kSlice * kQ / 4), off = e % (kSlice * kQ / 4);
      reinterpret_cast<float4*>(s.pq)[e] = ld_dsmem_f4(mapa_u32(smem_u32(s.ys) + off * 16, static_cast<uint32_t>(r)));
    }
    __syncthreads();
    x_q<RW>(s, nr);                                      // X Qn (the final one is C = B^T)
    __syncthreads();
    if (it == niter) break;
    cholqr2(s, s.qm, nr, par);                           // Qm
  }

  // ---- S and W = Ub diag(f) Ub^T from the eigen-decomposition of C^T C ----
  cluster_gram(s, s.qm, nr, par);
  jacobi_eig(s);
  if (t == 0) {                                          // order the eigenvalues descending (ties keep index order)
    int* perm = s.perm;
    for (int k = 0; k < kQ; ++k) perm[k] = k;
    for (int k = 0; k < kQ; ++k)
      for (int j = k + 1; j < kQ; ++j)
        if (s.g[perm[j] * kQ + perm[j]] > s.g[perm[k] * kQ + perm[k]]) { const int tmp = perm[k]; perm[k] = perm[j]; perm[j] = tmp; }
  }
  __syncthreads();
  const int* perm = s.perm;
  if (rank == 0 && s_out != nullptr && t < kQ)
    s_out[item * kQ + t] = static_cast<float>(sqrt(fmax(s.g[perm[t] * kQ + perm[t]], 0.0)));
  if (v_out != nullptr)                                  // V = Qn Ub: this CTA's slice of rows
    for (int e = t; e < kSlice * kQ; e += kThreads) {
      const int j = rank * kSlice + e / kQ, k = e % kQ;
      double acc = 0.0;
      for (int c = 0; c < kQ; ++c) acc = fma(static_cast<double>(s.pq[j * kQ + c]), s.l[c * kQ + perm[k]], acc);
      v_out[(static_cast<long long>(item) * kN + j) * kQ + k] = static_cast<float>(acc);
    }
  if (u_out != nullptr)                                  // U = Vb = C Ub diag(1 / S): this CTA's rows
    for (int e = t; e < nr * kQ; e += kThreads) {
      const int i = e / kQ, k = e % kQ;
      double acc = 0.0;
      for (int c = 0; c < kQ; ++c) acc = fma(static_cast<double>(s.qm[i * kQ + c]), s.l[c * kQ + perm[k]], acc);
      u_out[(static_cast<long long>(item) * m + row0 + i) * kQ + k] = static_cast<float>(acc / sqrt(s.g[perm[k] * kQ + perm[k]]));
    }
  for (int e = t; e < kQQ; e += kThreads) {
    const int a = e / kQ, b = e % kQ;
    double acc = 0.0;
    for (int k = 0; k < kQ; ++k) acc = fma(s.l[a * kQ + perm[k]] * static_cast<double>(factors[k]), s.l[b * kQ + perm[k]], acc);
    if (keep_remainder && a == b) acc -= 1.0;
    s.w[e] = static_cast<float>(acc);
  }
  __syncthreads();
  for (int i = t; i < nr; i += kThreads) {               // qm <- C W
    float v[kQ];
#pragma unroll
    for (int c = 0; c < kQ; ++c) v[c] = s.qm[i * kQ + c];
#pragma unroll
    for (int c = 0; c < kQ; ++c) {
      float acc = 0.f;
#pragma unroll
      for (int p = 0; p < kQ; ++p) acc = fmaf(v[p], s.w[p * kQ + c], acc);
      s.qm[i * kQ + c] = acc;
    }
  }
  __syncthreads();

  // ---- reconstruct x_new in place and its statistics ----
  sum = 0.0; sq = 0.0;
  {
    float qn[kJ][kQ];
#pragma unroll
    for (int k = 0; k < kJ; ++k)
#pragma unroll
      for (int c = 0; c < kQ; ++c) qn[k][c] = s.pq[(t + k * kThreads) * kQ + c];
    const uint32_t zq = smem_u32(s.qm);
    for (int i = 0; i < nr; ++i) {
      float z[kQ];
#pragma unroll
      for (int c = 0; c < kQ; c += 4) {
        const float4 v = lds_f4(zq + (i * kQ + c) * 4);
        z[c] = v.x; z[c + 1] = v.y; z[c + 2] = v.z; z[c + 3] = v.w;
      }
      const float mu = s.mean[i];
#pragma unroll
      for (int k = 0; k < kJ; ++k) {
        float d = 0.f;
#pragma unroll
        for (int c = 0; c < kQ; ++c) d = fmaf(z[c], qn[k][c], d);
        float& xv = s.x[i * kN + t + k * kThreads];
        const float nv = keep_remainder ? (xv + mu) + d : d + mu;
        xv = nv;
        sum += nv;
        sq = fma(static_cast<double>(nv), static_cast<double>(nv), sq);
      }
    }
  }
  block_sum2(s, sum, sq);
  const double std_new = cluster_std(s, sum, sq, count);
  const float inv_new = static_cast<float>(std_new), save = static_cast<float>(std_save);
  float* oi = out + (static_cast<long long>(item) * m + row0) * kN;
  for (int e = t; e < nr * kN; e += kThreads) oi[e] = s.x[e] / inv_new * save;
  cluster_sync_all();   // no CTA may exit while a peer can still read its shared memory
}

size_t rank_adjust_smem(int m) {
  const int rows_cap = (m + kCluster - 1) / kCluster;
  return 5 * kQQ * 8 + 2 * 8 + 2 * kWarps * 8 + kN * kQ * 4 + kSlice * kQ * 4 + kQQ * 4 + kQ * 4 + rows_cap * kQ * 4 +
         ((rows_cap + 3) / 4) * 16 + static_cast<size_t>(rows_cap) * kN * 4;
}

}  // namespace

}  // namespace vdb

using namespace vdb;

extern "C" int vdb_rank_adjust_f32(const float* x, int n_items, int m, int n, const float* R, int q, int niter,
                                   const float* factors, int keep_remainder, float* out, float* s_out, float* u_out,
                                   float* v_out, void* stream) {
  if (!x || !R || !factors || !out) return set_error(VDB_ERR_INVALID, "rank_adjust: null pointer (x, R, factors and out are required)");
  if (n_items < 1) return set_error(VDB_ERR_INVALID, "rank_adjust: n_items = %d < 1", n_items);
  if (niter < 0) return set_error(VDB_ERR_INVALID, "rank_adjust: niter = %d < 0", niter);
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15)
    return set_error(VDB_ERR_INVALID, "rank_adjust: x and out must be 16-byte aligned");
  if (n != kN || q != kQ || m < 2 * kQ || m > kMaxRows || n_items > 65535)
    return set_error(VDB_ERR_UNSUPPORTED,
                     "rank_adjust: (m, n, q) = (%d, %d, %d), n_items = %d: supported are n = %d, q = %d, %d <= m <= %d, "
                     "n_items <= 65535", m, n, q, n_items, kN, kQ, 2 * kQ, kMaxRows);
  const int rows_cap = (m + kCluster - 1) / kCluster;
  const int rw = (rows_cap + kWarps - 1) / kWarps;
  const size_t smem = rank_adjust_smem(m);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  static bool configured = false;
  if (!configured) {
    for (auto kernel : {rank_adjust_kernel<4>, rank_adjust_kernel<5>})
      VDB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          static_cast<int>(rank_adjust_smem(kMaxRows))));
    configured = true;
  }
  auto launch = [&](auto kernel) -> int {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(kCluster, n_items); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = kCluster; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    VDB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, x, m, R, niter, factors, keep_remainder, out, s_out, u_out, v_out));
    count_launch();
    return VDB_OK;
  };
  return rw <= 4 ? launch(rank_adjust_kernel<4>) : launch(rank_adjust_kernel<5>);
}
