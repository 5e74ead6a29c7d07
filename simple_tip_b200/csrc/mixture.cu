// mixture.cu — the N-sized passes of a full-covariance Gaussian-mixture EM fit (sklearn GaussianMixture,
// covariance_type="full"), in float64 on the fp64 tensor cores of sm_90a (mma.sync m16n8k16 .f64 = DMMA).
//
// The fit chains a covariance, its Cholesky factor and the factor's inverse, which amplifies any error by the
// covariance's condition number, so every pass here is float64; float32 rows are widened exactly on load.
// Every reduction has a fixed order (tile partials, then row chunks / blocks in ascending order) and nothing is
// summed with atomics: the same input on the same device gives the same bits.  The work decomposition depends on
// the shape only (not on the card's SM count).
//
//   gmm_quad_kernel     q[k, i] = |(x_i - mu_k) . L_k|^2 (L_k upper triangular): 64 x 64 output tiles of Y on DMMA,
//                       the zero blocks of the triangle skipped, squared and row-summed in the epilogue (Y is never
//                       stored); one CTA walks all column blocks of its 64 rows in ascending order.  Its store
//                       variant (kLower) is LSA's training-row whitening (x[:, cols] - mu) . W, W lower triangular,
//                       written as fp32
//   gmm_resp_kernel     log w_k - (D log 2pi + q) / 2 + log det L_k, log-sum-exp over k, resp = exp(. - lse), block
//                       partials of sum(lse) (merged by gmm_mean_kernel in ascending block order)
//   gmm_moments_kernel  per row chunk: sum_i r_ik and sum_i r_ik x_i (merged by gmm_moments_finish_kernel, which
//                       also adds sklearn's 10 eps to nk and divides)
//   gmm_scatter_kernel  S_k = sum_i r_ik (x_i - mu_k)(x_i - mu_k)^T over the lower-triangle 64 x 64 tiles on DMMA,
//                       split over row chunks when there are too few tiles to fill the card; mirrored on output
#include <algorithm>
#include "common.cuh"

namespace tip {

constexpr int kGmBM = 64, kGmBN = 64, kGmBK = 32;
constexpr int kGmLd = kGmBN + 4;            // shared leading dimension (doubles): conflict-free fragment reads
constexpr int kGmThreads = 128;             // 4 warps, 2 x 2 over the 64 x 64 tile, 32 x 32 each
constexpr int kGmMaxK = 64;
constexpr int kGmTargetCtas = 264;          // 2 CTAs per SM of a 132-SM H100 SXM: the chunk heuristics aim here
constexpr int64_t kGmScatterBudget = 256ll << 20;   // bytes of scatter chunk partials
constexpr int64_t kGmMomentBudget = 64ll << 20;     // bytes of moment chunk partials
constexpr int kGmRespThreads = 256;

struct GmTile {
  double a[kGmBK][kGmLd];   // A operand, k-major: a[kk][m]
  double b[kGmBK][kGmLd];   // B operand, k-major: b[kk][n]
};

// D[16x8] += A[16x16] . B[16x8], float64 (sm_90 DMMA.16x8x16).  Fragments (g = lane / 4, t = lane % 4):
// a[i] = A[g + 8 (i & 1)][t + 4 (i >> 1)], b[i] = B[t + 4 i][g], c = {D[g][2t], D[g][2t+1], D[g+8][2t], D[g+8][2t+1]}.
__device__ __forceinline__ void dmma16816(double c[4], const double a[8], const double b[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// the warp's 32 x 32 share of one kGmBK-deep step of the 64 x 64 tile
__device__ __forceinline__ void gm_tile_step(const GmTile& s, double acc[2][4][4], int wm, int wn, int g, int t) {
#pragma unroll
  for (int kk = 0; kk < kGmBK; kk += 16) {
    double a[2][8];
#pragma unroll
    for (int mt = 0; mt < 2; mt++)
#pragma unroll
      for (int i = 0; i < 8; i++) a[mt][i] = s.a[kk + t + 4 * (i >> 1)][wm * 32 + mt * 16 + g + 8 * (i & 1)];
#pragma unroll
    for (int nt = 0; nt < 4; nt++) {
      double b[4];
#pragma unroll
      for (int i = 0; i < 4; i++) b[i] = s.b[kk + t + 4 * i][wn * 32 + nt * 8 + g];
#pragma unroll
      for (int mt = 0; mt < 2; mt++) dmma16816(acc[mt][nt], a[mt], b);
    }
  }
}

__device__ __forceinline__ void gm_zero(double acc[2][4][4]) {
#pragma unroll
  for (int mt = 0; mt < 2; mt++)
#pragma unroll
    for (int nt = 0; nt < 4; nt++)
#pragma unroll
      for (int i = 0; i < 4; i++) acc[mt][nt][i] = 0.0;
}

// ---- E-step quadratic forms / LSA's training-row whitening -----------------------------------------------------
// grid (row tiles, K).  Y = (X - mu_k) . L_k tile by tile.
// kLower == false (E-step): L_k is upper triangular, so column block j0 needs the rows l < j0 + 64 of L only, and
//   inside the diagonal block the entries below the diagonal are read as 0.  Epilogue: per (row, column block) the
//   64 squares summed in double (thread: its 8 columns in order; quad: xor butterfly; the two column halves: left +
//   right), accumulated over the column blocks in ascending order.
// kLower == true (LSA whitening, scipy 1.4.1's points . cholesky(inv_cov)): L is lower triangular, so column block
//   j0 needs the rows l >= j0 only (the mirror skip), and inside the diagonal block the entries above the diagonal are
//   read as 0.  X's columns are read through the column list cols (NULL: 0..d-1) of rows of ld entries, and Y is
//   stored as fp32, rounded once from the float64 accumulator.
template <typename T, bool kLower>
__global__ void __launch_bounds__(kGmThreads) gmm_quad_kernel(const T* __restrict__ x, int64_t n, int d,
                                                              const double* __restrict__ mu,
                                                              const double* __restrict__ chol,
                                                              double* __restrict__ q, int64_t ld,
                                                              const int32_t* __restrict__ cols,
                                                              float* __restrict__ y) {
  __shared__ GmTile s;
  __shared__ double s_half[2][kGmBM];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const int wm = warp >> 1, wn = warp & 1;
  const int64_t i0 = (int64_t)blockIdx.x * kGmBM;
  const int k = blockIdx.y;
  const double* muk = mu + (int64_t)k * d;
  const double* L = chol + (int64_t)k * d * d;
  if (!kLower) ld = d;
  double total = 0.0;   // thread tid < 64: row i0 + tid
  double acc[2][4][4];
  for (int j0 = 0; j0 < d; j0 += kGmBN) {
    gm_zero(acc);
    const int lbeg = kLower ? j0 : 0, lend = kLower ? d : min(d, j0 + kGmBN);
    for (int l0 = lbeg; l0 < lend; l0 += kGmBK) {
      __syncthreads();
      for (int e = tid; e < kGmBM * kGmBK; e += kGmThreads) {   // centred rows, widened to double
        const int r = e / kGmBK, l = e % kGmBK;
        const int64_t i = i0 + r;
        double v = 0.0;
        if (i < n && l0 + l < d) {
          const int64_t src = (kLower && cols) ? (int64_t)cols[l0 + l] : (int64_t)(l0 + l);
          v = (double)x[i * ld + src] - muk[l0 + l];
        }
        s.a[l][r] = v;
      }
      for (int e = tid; e < kGmBK * kGmBN; e += kGmThreads) {
        const int l = e / kGmBN, j = e % kGmBN;
        const int gl = l0 + l, gj = j0 + j;
        const bool inside = kLower ? (gl < d && gj < d && gl >= gj) : (gj < d && gl <= gj);
        s.b[l][j] = inside ? L[(int64_t)gl * d + gj] : 0.0;
      }
      __syncthreads();
      gm_tile_step(s, acc, wm, wn, g, t);
    }
    if constexpr (kLower) {
      // staged through the operand tiles (64 x 64 floats fit in one of them), then stored row by row
      float* stage = reinterpret_cast<float*>(&s.a[0][0]);
      __syncthreads();
#pragma unroll
      for (int mt = 0; mt < 2; mt++)
#pragma unroll
        for (int nt = 0; nt < 4; nt++)
#pragma unroll
          for (int h = 0; h < 4; h++)
            stage[(wm * 32 + mt * 16 + g + 8 * (h >> 1)) * kGmBN + wn * 32 + nt * 8 + 2 * t + (h & 1)] =
                __double2float_rn(acc[mt][nt][h]);
      __syncthreads();
      for (int e = tid; e < kGmBM * kGmBN; e += kGmThreads) {
        const int r = e / kGmBN, j = e % kGmBN;
        if (i0 + r < n && j0 + j < d) y[(i0 + r) * d + j0 + j] = stage[e];
      }
    } else {
#pragma unroll
      for (int mt = 0; mt < 2; mt++) {
        double r0 = 0.0, r1 = 0.0;
#pragma unroll
        for (int nt = 0; nt < 4; nt++) {
          r0 = fma(acc[mt][nt][0], acc[mt][nt][0], r0);
          r0 = fma(acc[mt][nt][1], acc[mt][nt][1], r0);
          r1 = fma(acc[mt][nt][2], acc[mt][nt][2], r1);
          r1 = fma(acc[mt][nt][3], acc[mt][nt][3], r1);
        }
        r0 += __shfl_xor_sync(0xffffffffu, r0, 1);
        r0 += __shfl_xor_sync(0xffffffffu, r0, 2);
        r1 += __shfl_xor_sync(0xffffffffu, r1, 1);
        r1 += __shfl_xor_sync(0xffffffffu, r1, 2);
        if (t == 0) {
          s_half[wn][wm * 32 + mt * 16 + g] = r0;
          s_half[wn][wm * 32 + mt * 16 + g + 8] = r1;
        }
      }
      __syncthreads();
      if (tid < kGmBM) total += s_half[0][tid] + s_half[1][tid];
    }
  }
  if (!kLower && tid < kGmBM && i0 + tid < n) q[(int64_t)k * n + i0 + tid] = total;
}

// ---- responsibilities, log-sum-exp, lower bound ---------------------------------------------------------------
__device__ __forceinline__ double gm_logp(const double* __restrict__ q, int64_t n, int64_t i, int k, double dlog2pi,
                                          const double* __restrict__ log_w, const double* __restrict__ log_det) {
  // sklearn: (-.5 * (D log 2pi + q) + log_det) + log_w
  return (-0.5 * (dlog2pi + q[(int64_t)k * n + i]) + log_det[k]) + log_w[k];
}

__global__ void __launch_bounds__(kGmRespThreads) gmm_resp_kernel(const double* __restrict__ q, int64_t n, int kc,
                                                                  double dlog2pi, const double* __restrict__ log_w,
                                                                  const double* __restrict__ log_det,
                                                                  double* __restrict__ resp, double* __restrict__ lse,
                                                                  int64_t* __restrict__ labels,
                                                                  double* __restrict__ part) {
  __shared__ double red[kGmRespThreads];
  const int64_t i = (int64_t)blockIdx.x * kGmRespThreads + threadIdx.x;
  double v = 0.0;
  if (i < n) {
    // scipy logsumexp: a_max, sum of exp(a - a_max) in component order, log(s) + a_max
    double mx = gm_logp(q, n, i, 0, dlog2pi, log_w, log_det);
    int arg = 0;
    for (int k = 1; k < kc; k++) {
      const double a = gm_logp(q, n, i, k, dlog2pi, log_w, log_det);
      if (a > mx) { mx = a; arg = k; }
    }
    const double m0 = isfinite(mx) ? mx : 0.0;
    double s = 0.0;
    for (int k = 0; k < kc; k++) s += exp(gm_logp(q, n, i, k, dlog2pi, log_w, log_det) - m0);
    v = log(s) + m0;
    if (lse) lse[i] = v;
    if (labels) labels[i] = arg;
    if (resp)
      for (int k = 0; k < kc; k++) resp[(int64_t)k * n + i] = exp(gm_logp(q, n, i, k, dlog2pi, log_w, log_det) - v);
  }
  if (!part) return;
  red[threadIdx.x] = v;
  __syncthreads();
  for (int w = kGmRespThreads / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = red[0];
}

// one thread: the block partials in ascending order, / n
__global__ void gmm_mean_kernel(const double* __restrict__ part, int nb, int64_t n, double* __restrict__ out) {
  double s = 0.0;
  for (int b = 0; b < nb; b++) s += part[b];
  *out = s / (double)n;
}

// ---- M-step moments -------------------------------------------------------------------------------------------
// grid (feature blocks of 128, row chunks): thread = one feature, rows of the chunk in order, per component
template <typename T>
__global__ void __launch_bounds__(kGmThreads) gmm_moments_kernel(const T* __restrict__ x, int64_t n, int d,
                                                                 const double* __restrict__ resp, int kc,
                                                                 int64_t rows_per_chunk,
                                                                 double* __restrict__ part_sum,
                                                                 double* __restrict__ part_nk) {
  const int c = blockIdx.y;
  const int64_t r0 = (int64_t)c * rows_per_chunk, r1 = min(n, r0 + rows_per_chunk);
  const int a = blockIdx.x * kGmThreads + threadIdx.x;
  if (a < d)
    for (int k = 0; k < kc; k++) {
      const double* r = resp + (int64_t)k * n;
      double acc = 0.0;
      for (int64_t i = r0; i < r1; i++) acc = fma(r[i], (double)x[i * d + a], acc);
      part_sum[((int64_t)c * kc + k) * d + a] = acc;
    }
  if (blockIdx.x == 0)
    for (int k = threadIdx.x; k < kc; k += kGmThreads) {
      const double* r = resp + (int64_t)k * n;
      double acc = 0.0;
      for (int64_t i = r0; i < r1; i++) acc += r[i];
      part_nk[(int64_t)c * kc + k] = acc;
    }
}

// chunk partials in ascending chunk order; nk = sum + 10 eps (sklearn _estimate_gaussian_parameters), means = sums / nk
__global__ void gmm_moments_finish_kernel(const double* __restrict__ part_sum, const double* __restrict__ part_nk,
                                          int chunks, int kc, int d, double* __restrict__ nk_out,
                                          double* __restrict__ sums_out, double* __restrict__ means_out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)kc * d) return;
  const int k = (int)(e / d), a = (int)(e % d);
  double nk = 0.0;
  for (int c = 0; c < chunks; c++) nk += part_nk[(int64_t)c * kc + k];
  nk += 10.0 * 2.220446049250313e-16;
  double s = 0.0;
  for (int c = 0; c < chunks; c++) s += part_sum[((int64_t)c * kc + k) * d + a];
  if (a == 0 && nk_out) nk_out[k] = nk;
  if (sums_out) sums_out[e] = s;
  if (means_out) means_out[e] = __ddiv_rn(s, nk);
}

// ---- weighted scatter matrices (SYRK over lower-triangle tiles) ------------------------------------------------
__device__ __forceinline__ void gm_tri_tile(int p, int* ti, int* tj) {
  int i = (int)((sqrt(8.0 * p + 1.0) - 1.0) * 0.5);
  while ((int64_t)(i + 1) * (i + 2) / 2 <= p) i++;
  while ((int64_t)i * (i + 1) / 2 > p) i--;
  *ti = i;
  *tj = p - i * (i + 1) / 2;
}

// out[k][a][b] and its mirror for a >= b: S (nk == nullptr) or S / nk + reg_covar on the diagonal
__device__ __forceinline__ void gm_store_cov(double* __restrict__ out, int d, int k, int a, int b, double v,
                                             const double* __restrict__ nk, double reg) {
  if (a >= d || b > a) return;
  if (nk) {
    v = __ddiv_rn(v, nk[k]);
    if (a == b) v = __dadd_rn(v, reg);
  }
  double* o = out + (int64_t)k * d * d;
  o[(int64_t)a * d + b] = v;
  o[(int64_t)b * d + a] = v;
}

// grid (lower tiles, chunks, K).  A[a][i] = r_ik (x_ia - mu_ka), B[i][b] = x_ib - mu_kb, reduced over the rows of
// the chunk.  chunks == 1: stored (finished) straight into out; else the tile partial goes to part[k][c][tile].
template <typename T>
__global__ void __launch_bounds__(kGmThreads) gmm_scatter_kernel(const T* __restrict__ x, int64_t n, int d,
                                                                 const double* __restrict__ resp,
                                                                 const double* __restrict__ mu,
                                                                 int64_t rows_per_chunk, double* __restrict__ part,
                                                                 double* __restrict__ out,
                                                                 const double* __restrict__ nk, double reg) {
  __shared__ GmTile s;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const int wm = warp >> 1, wn = warp & 1;
  const int p = blockIdx.x, c = blockIdx.y, k = blockIdx.z, tiles = gridDim.x, chunks = gridDim.y;
  int ti, tj;
  gm_tri_tile(p, &ti, &tj);
  const int a0 = ti * kGmBM, b0 = tj * kGmBN;
  const int64_t r0 = (int64_t)c * rows_per_chunk, r1 = min(n, r0 + rows_per_chunk);
  const double* muk = mu + (int64_t)k * d;
  const double* rk = resp + (int64_t)k * n;
  double acc[2][4][4];
  gm_zero(acc);
  for (int64_t i0 = r0; i0 < r1; i0 += kGmBK) {
    __syncthreads();
    for (int e = tid; e < kGmBK * kGmBM; e += kGmThreads) {
      const int ii = e / kGmBM, m = e % kGmBM;
      const int64_t i = i0 + ii;
      double va = 0.0, vb = 0.0;
      if (i < r1) {
        const double ri = rk[i];
        if (a0 + m < d) va = ri * ((double)x[i * d + a0 + m] - muk[a0 + m]);
        if (b0 + m < d) vb = (double)x[i * d + b0 + m] - muk[b0 + m];
      }
      s.a[ii][m] = va;
      s.b[ii][m] = vb;
    }
    __syncthreads();
    gm_tile_step(s, acc, wm, wn, g, t);
  }
#pragma unroll
  for (int mt = 0; mt < 2; mt++)
#pragma unroll
    for (int nt = 0; nt < 4; nt++)
#pragma unroll
      for (int h = 0; h < 4; h++) {
        const int rr = wm * 32 + mt * 16 + g + 8 * (h >> 1), cc = wn * 32 + nt * 8 + 2 * t + (h & 1);
        if (chunks == 1)
          gm_store_cov(out, d, k, a0 + rr, b0 + cc, acc[mt][nt][h], nk, reg);
        else
          part[(((int64_t)k * chunks + c) * tiles + p) * (kGmBM * kGmBN) + rr * kGmBN + cc] = acc[mt][nt][h];
      }
}

// the chunk partials of every lower tile in ascending chunk order, then stored like the single-chunk case
__global__ void gmm_scatter_merge_kernel(const double* __restrict__ part, int tiles, int chunks, int kc, int d,
                                         double* __restrict__ out, const double* __restrict__ nk, double reg) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t per = (int64_t)tiles * kGmBM * kGmBN;
  if (e >= per * kc) return;
  const int k = (int)(e / per);
  const int64_t w = e % per;
  const int p = (int)(w / (kGmBM * kGmBN)), rr = (int)(w % (kGmBM * kGmBN)) / kGmBN, cc = (int)(w % kGmBN);
  int ti, tj;
  gm_tri_tile(p, &ti, &tj);
  double v = 0.0;
  for (int c = 0; c < chunks; c++) v += part[(((int64_t)k * chunks + c) * tiles + p) * (kGmBM * kGmBN) + rr * kGmBN + cc];
  gm_store_cov(out, d, k, ti * kGmBM + rr, tj * kGmBN + cc, v, nk, reg);
}

// ---- host side -------------------------------------------------------------------------------------------------
static int gm_check(int64_t n, int64_t d, int32_t k) {
  TIP_REQUIRE(k >= 1 && k <= kGmMaxK, "k must be in [1, 64]");
  TIP_REQUIRE(n >= 1 && n < (1LL << 31) && d >= 1 && d <= 65536, "shape");
  TIP_REQUIRE((n + kGmBM - 1) / kGmBM < (1LL << 31), "shape");
  return TIP_OK;
}

static int64_t gm_tiles(int64_t d) {
  const int64_t t = (d + kGmBM - 1) / kGmBM;
  return t * (t + 1) / 2;
}

// scatter row chunks: enough CTAs to fill the card, at least 256 rows each, shrunk until the partials fit the budget
static int gm_scatter_chunks(int64_t n, int64_t d, int32_t k, int32_t requested) {
  const int64_t per_chunk = (int64_t)k * gm_tiles(d) * kGmBM * kGmBN * 8;
  int64_t c = requested > 0 ? requested : (kGmTargetCtas + (int64_t)k * gm_tiles(d) - 1) / ((int64_t)k * gm_tiles(d));
  c = std::min<int64_t>(c, std::max<int64_t>(1, n / 256));
  c = std::min<int64_t>(c, 65535);
  while (c > 1 && c * per_chunk > kGmScatterBudget) c--;
  return (int)std::max<int64_t>(1, c);
}

static int gm_moment_chunks(int64_t n, int64_t d, int32_t k) {
  const int64_t fb = (d + kGmThreads - 1) / kGmThreads;
  int64_t c = (kGmTargetCtas + fb - 1) / fb;
  c = std::min<int64_t>(c, std::max<int64_t>(1, n / 64));
  while (c > 1 && c * k * (d + 1) * 8 > kGmMomentBudget) c--;
  return (int)std::max<int64_t>(1, c);
}

static int64_t gm_align(int64_t b) { return (b + 255) & ~(int64_t)255; }

static int64_t gm_work_bytes(int64_t n, int64_t d, int32_t k, int32_t scatter_chunks) {
  const int sc = gm_scatter_chunks(n, d, k, scatter_chunks);
  const int64_t scatter = sc > 1 ? (int64_t)sc * k * gm_tiles(d) * kGmBM * kGmBN * 8 : 0;
  const int mc = gm_moment_chunks(n, d, k);
  const int64_t moments = gm_align((int64_t)mc * k * d * 8) + gm_align((int64_t)mc * k * 8);
  const int64_t resp = gm_align((n + kGmRespThreads - 1) / kGmRespThreads * 8);
  return std::max(std::max(scatter, moments), resp) + 256;
}

}  // namespace tip

using namespace tip;

extern "C" int32_t tip_gmm_scatter_chunks(int64_t n, int64_t d, int32_t k, int32_t requested) {
  if (gm_check(n, d, k) != TIP_OK || requested < 0) return -1;
  return gm_scatter_chunks(n, d, k, requested);
}

extern "C" int64_t tip_gmm_work_bytes(int64_t n, int64_t d, int32_t k, int32_t scatter_chunks) {
  if (gm_check(n, d, k) != TIP_OK || scatter_chunks < 0) return -1;
  return gm_work_bytes(n, d, k, scatter_chunks);
}

extern "C" int tip_gmm_quad(const void* x, int dtype, int64_t n, int64_t d, const double* means,
                            const double* prec_chol, int32_t k, double* q, void* stream) {
  TIP_REQUIRE(dtype == TIP_F32 || dtype == TIP_F64, "dtype must be TIP_F32 or TIP_F64");
  int rc = gm_check(n, d, k);
  if (rc != TIP_OK) return rc;
  TIP_REQUIRE(x && means && prec_chol && q, "null pointer");
  const dim3 grid((unsigned)((n + kGmBM - 1) / kGmBM), (unsigned)k);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == TIP_F32)
    gmm_quad_kernel<float, false><<<grid, kGmThreads, 0, st>>>((const float*)x, n, (int)d, means, prec_chol, q, d,
                                                               nullptr, nullptr);
  else
    gmm_quad_kernel<double, false><<<grid, kGmThreads, 0, st>>>((const double*)x, n, (int)d, means, prec_chol, q, d,
                                                                nullptr, nullptr);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_whiten_dmma(const void* x, int dtype, int64_t m, int64_t d_in, const int32_t* cols, int64_t d_out,
                               const double* mu, const double* w_lower, float* out, void* stream) {
  TIP_REQUIRE(dtype == TIP_F32 || dtype == TIP_F64, "dtype must be TIP_F32 or TIP_F64");
  int rc = gm_check(m, d_out, 1);
  if (rc != TIP_OK) return rc;
  TIP_REQUIRE(d_in >= d_out && (cols || d_in == d_out), "shape");
  TIP_REQUIRE(x && mu && w_lower && out, "null pointer");
  const dim3 grid((unsigned)((m + kGmBM - 1) / kGmBM), 1u);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == TIP_F32)
    gmm_quad_kernel<float, true><<<grid, kGmThreads, 0, st>>>((const float*)x, m, (int)d_out, mu, w_lower, nullptr,
                                                              d_in, cols, out);
  else
    gmm_quad_kernel<double, true><<<grid, kGmThreads, 0, st>>>((const double*)x, m, (int)d_out, mu, w_lower, nullptr,
                                                               d_in, cols, out);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_gmm_resp(const double* q, int64_t n, int64_t d, int32_t k, const double* log_weights,
                            const double* log_det, double* resp, double* lse, int64_t* labels, double* lower_bound,
                            void* work, void* stream) {
  int rc = gm_check(n, d, k);
  if (rc != TIP_OK) return rc;
  TIP_REQUIRE(q && log_weights && log_det, "null pointer");
  TIP_REQUIRE(!lower_bound || work, "lower_bound needs work");
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = (int)((n + kGmRespThreads - 1) / kGmRespThreads);
  double* part = lower_bound ? (double*)work : nullptr;
  const double dlog2pi = (double)d * 1.8378770664093453;   // n_features * np.log(2 * np.pi)
  gmm_resp_kernel<<<nb, kGmRespThreads, 0, st>>>(q, n, k, dlog2pi, log_weights, log_det, resp, lse, labels, part);
  TIP_LAUNCH_CHECK();
  if (lower_bound) {
    gmm_mean_kernel<<<1, 1, 0, st>>>(part, nb, n, lower_bound);
    TIP_LAUNCH_CHECK();
  }
  return TIP_OK;
}

extern "C" int tip_gmm_moments(const void* x, int dtype, int64_t n, int64_t d, const double* resp, int32_t k,
                               double* nk, double* sums, double* means, void* work, void* stream) {
  TIP_REQUIRE(dtype == TIP_F32 || dtype == TIP_F64, "dtype must be TIP_F32 or TIP_F64");
  int rc = gm_check(n, d, k);
  if (rc != TIP_OK) return rc;
  TIP_REQUIRE(x && resp && work && (nk || sums || means), "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int chunks = gm_moment_chunks(n, d, k);
  const int64_t rows = (n + chunks - 1) / chunks;
  double* part_sum = (double*)work;
  double* part_nk = (double*)((char*)work + gm_align((int64_t)chunks * k * d * 8));
  const dim3 grid((unsigned)((d + kGmThreads - 1) / kGmThreads), (unsigned)chunks);
  if (dtype == TIP_F32)
    gmm_moments_kernel<float><<<grid, kGmThreads, 0, st>>>((const float*)x, n, (int)d, resp, k, rows, part_sum, part_nk);
  else
    gmm_moments_kernel<double><<<grid, kGmThreads, 0, st>>>((const double*)x, n, (int)d, resp, k, rows, part_sum,
                                                            part_nk);
  TIP_LAUNCH_CHECK();
  const int64_t total = (int64_t)k * d;
  gmm_moments_finish_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(part_sum, part_nk, chunks, k, (int)d, nk,
                                                                             sums, means);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_gmm_scatter(const void* x, int dtype, int64_t n, int64_t d, const double* resp,
                               const double* means, int32_t k, const double* nk, double reg_covar,
                               int32_t scatter_chunks, double* out, void* work, void* stream) {
  TIP_REQUIRE(dtype == TIP_F32 || dtype == TIP_F64, "dtype must be TIP_F32 or TIP_F64");
  int rc = gm_check(n, d, k);
  if (rc != TIP_OK) return rc;
  TIP_REQUIRE(scatter_chunks >= 0 && reg_covar >= 0.0, "scatter_chunks / reg_covar");
  TIP_REQUIRE(x && resp && means && out, "null pointer");
  const int chunks = gm_scatter_chunks(n, d, k, scatter_chunks);
  TIP_REQUIRE(chunks == 1 || work, "null pointer (work)");
  const int64_t tiles = gm_tiles(d);
  TIP_REQUIRE(tiles < (1LL << 31), "shape");
  const int64_t rows = (n + chunks - 1) / chunks;
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)tiles, (unsigned)chunks, (unsigned)k);
  double* part = (double*)work;
  if (dtype == TIP_F32)
    gmm_scatter_kernel<float><<<grid, kGmThreads, 0, st>>>((const float*)x, n, (int)d, resp, means, rows, part, out, nk,
                                                           reg_covar);
  else
    gmm_scatter_kernel<double><<<grid, kGmThreads, 0, st>>>((const double*)x, n, (int)d, resp, means, rows, part, out,
                                                            nk, reg_covar);
  TIP_LAUNCH_CHECK();
  if (chunks > 1) {
    const int64_t total = (int64_t)k * tiles * kGmBM * kGmBN;
    gmm_scatter_merge_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(part, (int)tiles, chunks, k, (int)d, out,
                                                                             nk, reg_covar);
    TIP_LAUNCH_CHECK();
  }
  return TIP_OK;
}
