// kmeans.cu — device k-means (sklearn KMeans, algorithm="lloyd") and the last step of the silhouette score
// (sklearn.metrics.silhouette_samples), sm_90a.
//
// tip_kmeans_fit runs every one of the n_init runs of a fit inside ONE persistent cooperative kernel: greedy
// k-means++ seeding, then Lloyd iterations with a grid.sync between phases, so a fit makes no host round trip
// per iteration.  One pass over the rows per phase serves all runs.  Every reduction has a fixed order (block
// partials in row order, then ascending block index) and nothing is summed with atomics, so the same input,
// seed and device give the same bits.
#include <cooperative_groups.h>

#include <algorithm>
#include "common.cuh"

namespace cg = cooperative_groups;

namespace tip {

constexpr int kKmThreads = 256;
constexpr int kKmWarps = kKmThreads / 32;
constexpr int kKmMaxK = 64;
constexpr int kKmMaxTrials = 6;                 // 2 + int(ln 64)
constexpr int kKmAccDoubles = 4096;             // 32 KB of per-block centre-sum accumulators (+ 8 KB static: < 48 KB)
constexpr int64_t kKmPartBudget = 256ll << 20;  // bytes of per-block centre sums, all blocks together

enum { KM_ACTIVE = 0, KM_STRICT = 1, KM_TOL = 2, KM_MAXITER = 3 };

// ---- counter-based RNG: splitmix64 (km_mix, common.cuh) over the key (seed, k, run, step, trial) -------------
__device__ __forceinline__ double km_uniform(uint64_t seed, int k, int run, int step, int trial) {
  uint64_t h = km_mix(seed);
  h = km_mix(h ^ (uint64_t)k);
  h = km_mix(h ^ (uint64_t)run);
  h = km_mix(h ^ (uint64_t)step);
  h = km_mix(h ^ (uint64_t)trial);
  return (double)(h >> 11) * 0x1.0p-53;   // [0, 1)
}

__host__ __device__ __forceinline__ int64_t min64(int64_t a, int64_t b) { return a < b ? a : b; }

// sum_j (x_j - c_j)^2 in T over one warp (lane-strided partials, xor butterfly: every lane gets the same bits)
template <typename T>
__device__ __forceinline__ T warp_sqdist(const T* __restrict__ x, const T* __restrict__ c, int d, int lane) {
  T s = 0;
  for (int j = lane; j < d; j += 32) {
    const T t = x[j] - c[j];
    s = fma(t, t, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

// nearest of k centres (ties: lowest index), squared distance in T
template <typename T>
__device__ __forceinline__ int warp_nearest(const T* __restrict__ x, const T* __restrict__ cen, int k, int d, int lane,
                                            T* best_d) {
  int best = 0;
  T bd = warp_sqdist(x, cen, d, lane);
  for (int c = 1; c < k; c++) {
    const T v = warp_sqdist(x, cen + (int64_t)c * d, d, lane);
    if (v < bd) { bd = v; best = c; }
  }
  *best_d = bd;
  return best;
}

struct KmArgs {
  const void* x;
  int64_t n;
  int d, k, runs, trials, max_iter, dc;   // dc: dimensions per pass of the block's centre-sum accumulators
  double tol;                             // absolute: mean(var(X, axis=0)) * tol
  uint64_t seed;
  void* cen;                              // runs x k x d (T): the centres, also the output
  int32_t* n_iter;                        // runs
  // workspace (tip_kmeans_work_bytes)
  double *closest, *dtrial, *bpart, *bpot, *psum, *sums, *dist;
  int32_t *cand, *pcnt, *cnt, *labels, *bchanged, *status;
};

// fixed-order block reductions (every thread gets the result)
__device__ __forceinline__ double block_sum(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = kKmThreads / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}
// largest v, ties to the lowest index
__device__ __forceinline__ int64_t block_argmax(double v, int64_t i, double* red, int64_t* redi) {
  red[threadIdx.x] = v;
  redi[threadIdx.x] = i;
  __syncthreads();
  for (int s = kKmThreads / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) {
      const double v2 = red[threadIdx.x + s];
      const int64_t i2 = redi[threadIdx.x + s];
      if (v2 > red[threadIdx.x] || (v2 == red[threadIdx.x] && i2 < redi[threadIdx.x])) {
        red[threadIdx.x] = v2;
        redi[threadIdx.x] = i2;
      }
    }
    __syncthreads();
  }
  const int64_t r = redi[0];
  __syncthreads();
  return r;
}

template <typename T>
__global__ void __launch_bounds__(kKmThreads, 1) kmeans_fit_kernel(const KmArgs a) {
  cg::grid_group grid = cg::this_grid();
  extern __shared__ double s_acc[];
  __shared__ double s_red[kKmThreads];
  __shared__ int64_t s_redi[kKmThreads];
  __shared__ double s_pot[kKmMaxTrials * 64];
  __shared__ int s_best[64];
  __shared__ int s_changed[64];
  __shared__ int64_t s_taken[kKmMaxK];
  __shared__ int s_empty[kKmMaxK];

  const T* X = (const T*)a.x;
  T* C = (T*)a.cen;
  const int64_t n = a.n;
  const int D = a.d, K = a.k, R = a.runs, TR = a.trials, G = gridDim.x, b = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int per = ((int)n + G - 1) / G;   // n < 2^31
  const int64_t lo = min64(n, (int64_t)b * per), hi = min64(n, lo + per);

  for (int64_t i = lo + tid; i < hi; i += kKmThreads)
    for (int r = 0; r < R; r++) a.labels[(int64_t)r * n + i] = -1;
  if (b == 0 && tid < R) {
    a.status[tid] = KM_ACTIVE;
    a.n_iter[tid] = 0;
    a.cand[tid * TR] = (int32_t)min64(n - 1, (int64_t)(km_uniform(a.seed, K, tid, 0, 0) * (double)n));
  }

  // ================= greedy k-means++ (sklearn _kmeans_plusplus) =================
  for (int step = 0; step < K; step++) {
    const int nt = step == 0 ? 1 : TR;
    grid.sync();
    // D^2 of every row of the slice to every candidate, floored by the current closest distance
    for (int64_t i = lo + warp; i < hi; i += kKmWarps) {
      const T* xi = X + i * D;
      for (int r = 0; r < R; r++)
        for (int t = 0; t < nt; t++) {
          double v = (double)warp_sqdist(xi, X + (int64_t)a.cand[r * TR + t] * D, D, lane);
          if (step > 0) v = fmin(v, a.closest[(int64_t)r * n + i]);
          if (lane == 0) a.dtrial[((int64_t)r * TR + t) * n + i] = v;
        }
    }
    __syncthreads();
    for (int j = tid; j < R * nt; j += kKmThreads) {
      const int r = j / nt, t = j % nt;
      const double* dt = a.dtrial + ((int64_t)r * TR + t) * n;
      double s = 0.0;
      for (int64_t i = lo; i < hi; i++) s += dt[i];
      a.bpart[((int64_t)b * R + r) * TR + t] = s;
    }
    grid.sync();
    // the candidate with the lowest potential (ties: lowest trial), identically in every block
    for (int j = tid; j < R * nt; j += kKmThreads) {
      const int r = j / nt, t = j % nt;
      double s = 0.0;
      for (int bb = 0; bb < G; bb++) s += a.bpart[((int64_t)bb * R + r) * TR + t];
      s_pot[r * TR + t] = s;
    }
    __syncthreads();
    if (tid < R) {
      int best = 0;
      for (int t = 1; t < nt; t++)
        if (s_pot[tid * TR + t] < s_pot[tid * TR + best]) best = t;
      s_best[tid] = best;
      a.bpot[(int64_t)b * R + tid] = a.bpart[((int64_t)b * R + tid) * TR + best];
    }
    __syncthreads();
    for (int r = 0; r < R; r++) {
      const double* src = a.dtrial + ((int64_t)r * TR + s_best[r]) * n;
      for (int64_t i = lo + tid; i < hi; i += kKmThreads) a.closest[(int64_t)r * n + i] = src[i];
    }
    if (b == 0)
      for (int r = 0; r < R; r++) {
        const T* src = X + (int64_t)a.cand[r * TR + s_best[r]] * D;
        for (int j = tid; j < D; j += kKmThreads) C[((int64_t)r * K + step) * D + j] = src[j];
      }
    if (step + 1 == K) break;
    grid.sync();
    // draw the next candidates: first row whose running sum of D^2 reaches u * potential (np.searchsorted on
    // the cumulative sum; block partials first, then the rows of the block in order)
    if (b == 0)
      for (int j = tid; j < R * TR; j += kKmThreads) {
        const int r = j / TR, t = j % TR;
        const double target = km_uniform(a.seed, K, r, step + 1, t) * s_pot[r * TR + s_best[r]];
        double cum = 0.0;
        int blk = -1, last = -1;
        for (int bb = 0; bb < G; bb++) {
          const double p = a.bpot[(int64_t)bb * R + r];
          if (p > 0.0) last = bb;
          if (p > 0.0 && cum + p >= target) { blk = bb; break; }
          cum += p;
        }
        if (blk < 0) { blk = last < 0 ? 0 : last; cum = 0.0; for (int bb = 0; bb < blk; bb++) cum += a.bpot[(int64_t)bb * R + r]; }
        const int64_t b_lo = min64(n, (int64_t)blk * per), b_hi = min64(n, b_lo + per);
        const double* cl = a.closest + (int64_t)r * n;
        int64_t pick = -1, last_pos = b_lo;
        for (int64_t i = b_lo; i < b_hi; i++) {
          if (cl[i] > 0.0) last_pos = i;
          cum += cl[i];
          if (cum >= target && cl[i] > 0.0) { pick = i; break; }
        }
        a.cand[j] = (int32_t)(pick < 0 ? last_pos : pick);
      }
  }

  // ================= Lloyd iterations =================
  const int dc = a.dc;
  for (int it = 0; it < a.max_iter; it++) {
    grid.sync();
    bool any = false;
    for (int r = 0; r < R; r++) any |= a.status[r] == KM_ACTIVE;
    if (!any) break;
    if (tid < R) s_changed[tid] = 0;
    __syncthreads();
    // (A) assignment of the slice's rows for every active run
    for (int64_t i = lo + warp; i < hi; i += kKmWarps) {
      const T* xi = X + i * D;
      for (int r = 0; r < R; r++) {
        if (a.status[r] != KM_ACTIVE) continue;
        T bd;
        const int lab = warp_nearest(xi, C + (int64_t)r * K * D, K, D, lane, &bd);
        if (lane == 0) {
          int32_t* l = a.labels + (int64_t)r * n + i;
          if (*l != lab) s_changed[r] = 1;
          *l = lab;
          a.dist[(int64_t)r * n + i] = (double)bd;
        }
      }
    }
    __syncthreads();
    // per-block centre sums in double, rows in order; every thread owns its own accumulator columns
    for (int r = 0; r < R; r++) {
      if (a.status[r] != KM_ACTIVE) continue;
      const int32_t* lab = a.labels + (int64_t)r * n;
      for (int d0 = 0; d0 < D; d0 += dc) {
        const int w = min(dc, D - d0);
        for (int j = tid; j < K * dc; j += kKmThreads) s_acc[j] = 0.0;
        __syncthreads();
        for (int64_t i = lo; i < hi; i++) {
          const int c = lab[i];
          for (int j = tid; j < w; j += kKmThreads) s_acc[c * dc + j] += (double)X[i * D + d0 + j];
        }
        __syncthreads();
        double* dst = a.psum + (((int64_t)b * R + r) * K) * D + d0;
        for (int j = tid; j < K * w; j += kKmThreads) dst[(int64_t)(j / w) * D + j % w] = s_acc[(j / w) * dc + j % w];
        __syncthreads();
      }
      for (int c = tid; c < K; c += kKmThreads) {
        int cnt = 0;
        for (int64_t i = lo; i < hi; i++) cnt += lab[i] == c;
        a.pcnt[((int64_t)b * R + r) * K + c] = cnt;
      }
      if (tid == 0) a.bchanged[(int64_t)b * R + r] = s_changed[r];
    }
    grid.sync();
    // (B) merge the block partials in ascending block order
    {
      const int total = R * K * D, stride = G * kKmThreads;   // runs * k * d < 2^31
      for (int e = b * kKmThreads + tid; e < total; e += stride) {
        const int r = e / (K * D);
        if (a.status[r] != KM_ACTIVE) continue;
        double s = 0.0;
        for (int bb = 0; bb < G; bb++) s += a.psum[(int64_t)bb * total + e];
        a.sums[e] = s;
      }
      for (int e = b * kKmThreads + tid; e < R * K; e += stride) {
        if (a.status[e / K] != KM_ACTIVE) continue;
        int s = 0;
        for (int bb = 0; bb < G; bb++) s += a.pcnt[(int64_t)bb * R * K + e];
        a.cnt[e] = s;
      }
    }
    grid.sync();
    // (C) one block per run: relocate empty clusters, new centres, convergence test
    for (int r = b; r < R; r += G) {
      if (a.status[r] != KM_ACTIVE) continue;
      int ch = 0;
      for (int bb = tid; bb < G; bb += kKmThreads) ch |= a.bchanged[(int64_t)bb * R + r];
      ch = __syncthreads_or(ch);
      int32_t* cnt = a.cnt + (int64_t)r * K;
      double* sums = a.sums + (int64_t)r * K * D;
      // sklearn _relocate_empty_clusters: the set of empty clusters is fixed before any row moves (a donor emptied
      // here stays empty until the next assignment), and nothing moves when every row sits on its centre
      int n_empty = 0;
      for (int c = 0; c < K; c++) {
        if (cnt[c] != 0) continue;   // block-uniform (written before the last grid.sync)
        if (tid == 0) s_empty[n_empty] = c;
        n_empty++;
      }
      __syncthreads();
      if (n_empty > 0) {
        double mx = 0.0;
        for (int64_t i = tid; i < n; i += kKmThreads) mx = fmax(mx, a.dist[(int64_t)r * n + i]);
        if (!__syncthreads_or(mx > 0.0)) n_empty = 0;
      }
      for (int q = 0; q < n_empty; q++) {
        const int c = s_empty[q];
        // the row farthest from its centre (descending over the empty clusters, ties: lowest row) moves to c
        double bv = -1.0;
        int64_t bi = n;
        for (int64_t i = tid; i < n; i += kKmThreads) {
          bool taken = false;
          for (int j = 0; j < q; j++) taken |= s_taken[j] == i;
          const double v = a.dist[(int64_t)r * n + i];
          if (!taken && v > bv) { bv = v; bi = i; }
        }
        const int64_t far = block_argmax(bv, bi, s_red, s_redi);
        const int donor = a.labels[(int64_t)r * n + far];
        for (int j = tid; j < D; j += kKmThreads) {
          const double xv = (double)X[far * D + j];
          sums[(int64_t)donor * D + j] -= xv;
          sums[(int64_t)c * D + j] = xv;
        }
        __syncthreads();
        if (tid == 0) { cnt[donor] -= 1; cnt[c] = 1; s_taken[q] = far; }
        __syncthreads();
      }
      double shift = 0.0;
      T* cen = C + (int64_t)r * K * D;
#pragma unroll 1
      for (int e = tid; e < K * D; e += kKmThreads) {
        const int c = e / D;
        const T old = cen[e];
        // sums / count: reciprocal + one residual correction (the division's slow-path call would spill)
        const double cn = (double)cnt[c], rc = __drcp_rn(cn), q0 = sums[e] * rc;
        const T nv = cnt[c] > 0 ? (T)fma(fma(-cn, q0, sums[e]), rc, q0) : old;
        const double df = (double)nv - (double)old;
        shift += df * df;
        cen[e] = nv;
      }
      shift = block_sum(shift, s_red);
      if (tid == 0) {
        a.n_iter[r] = it + 1;
        if (!ch) a.status[r] = KM_STRICT;
        else if (shift <= a.tol) a.status[r] = KM_TOL;
        else if (it + 1 == a.max_iter) a.status[r] = KM_MAXITER;
      }
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(kKmThreads) kmeans_predict_kernel(const T* __restrict__ x, int64_t n, int d,
                                                                    const T* __restrict__ cen, int k, int runs,
                                                                    int32_t* __restrict__ labels,
                                                                    double* __restrict__ sqdist) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * kKmWarps;
  for (int64_t i = (int64_t)blockIdx.x * kKmWarps + (threadIdx.x >> 5); i < n; i += warps) {
    for (int r = 0; r < runs; r++) {
      T bd;
      const int lab = warp_nearest(x + i * d, cen + (int64_t)r * k * d, k, d, lane, &bd);
      if (lane == 0) {
        labels[(int64_t)r * n + i] = lab;
        if (sqdist) sqdist[(int64_t)r * n + i] = (double)bd;
      }
    }
  }
}

// one block per run: inertia[r] = sum_i sqdist[r][i] in a fixed order
__global__ void __launch_bounds__(kKmThreads) kmeans_inertia_kernel(const double* __restrict__ sqdist, int64_t n,
                                                                    double* __restrict__ inertia) {
  __shared__ double red[kKmThreads];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += kKmThreads) s += sqdist[(int64_t)blockIdx.x * n + i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) inertia[blockIdx.x] = s;
}

// ---- silhouette: per-row merge of the tip_sil_dsum partials ---------------------------------------------------
// Row i (label-sorted) of cluster L: per-cluster distance sums over its slots in ascending slot order (double);
// a = sum_L / (n_L - 1), b = min over the other clusters of sum_c / n_c, s = (b - a) / max(a, b); s = 0 for a
// singleton cluster and for a = b = 0 (sklearn's nan_to_num).
__global__ void __launch_bounds__(256) sil_finish_kernel(const float* __restrict__ part, int64_t n, int slots,
                                                         const int32_t* __restrict__ slot_cluster,
                                                         const int32_t* __restrict__ lab,
                                                         const int32_t* __restrict__ counts,
                                                         const int32_t* __restrict__ out_idx,
                                                         double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int own = lab[i];
  double a = 0.0, b = __longlong_as_double(0x7ff0000000000000LL), acc = 0.0;
  int cur = slots > 0 ? slot_cluster[0] : -1;
  for (int s = 0; s <= slots; s++) {
    const int c = s < slots ? slot_cluster[s] : -1;
    if (c != cur) {
      if (cur == own) a = counts[cur] > 1 ? acc / (double)(counts[cur] - 1) : 0.0;
      else if (counts[cur] > 0) b = fmin(b, acc / (double)counts[cur]);
      acc = 0.0;
      cur = c;
    }
    if (s < slots) acc += (double)part[(int64_t)s * n + i];
  }
  double v = 0.0;
  const double mx = fmax(a, b);
  if (counts[own] > 1 && mx > 0.0 && b < __longlong_as_double(0x7ff0000000000000LL)) v = (b - a) / mx;
  out[out_idx ? out_idx[i] : i] = v;
}

// ---- host side -------------------------------------------------------------------------------------------------
static int km_trials(int k) { return 2 + (int)std::log((double)k); }

static int km_dc(int d, int k) { return std::min(d, kKmAccDoubles / k); }

template <typename T>
static int km_grid(int64_t n, int d, int k, int runs, int* grid) {
  int per_sm = 0;
  const size_t smem = (size_t)k * km_dc(d, k) * sizeof(double);
  TIP_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kmeans_fit_kernel<T>, kKmThreads, smem));
  TIP_REQUIRE(per_sm >= 1, "cooperative kernel does not fit");
  int64_t g = (int64_t)sm_count() * std::min(per_sm, 2);
  g = std::min<int64_t>(g, (n + 7) / 8);
  g = std::min<int64_t>(g, std::max<int64_t>(1, kKmPartBudget / ((int64_t)runs * k * d * 8)));
  *grid = (int)std::max<int64_t>(1, g);
  return TIP_OK;
}

struct KmLayout {
  int64_t off[13];
  int64_t bytes;
};
static KmLayout km_layout(int64_t n, int d, int k, int runs, int grid) {
  const int tr = km_trials(k);
  const int64_t rn = (int64_t)runs * n, rkd = (int64_t)runs * k * d;
  const int64_t sizes[13] = {rn * 8,                              // closest
                             rn * tr * 8,                         // dtrial
                             (int64_t)grid * runs * tr * 8,       // bpart
                             (int64_t)grid * runs * 8,            // bpot
                             (int64_t)grid * rkd * 8,             // psum
                             rkd * 8,                             // sums
                             rn * 8,                              // dist
                             (int64_t)runs * tr * 4,              // cand
                             (int64_t)grid * runs * k * 4,        // pcnt
                             (int64_t)runs * k * 4,               // cnt
                             rn * 4,                              // labels
                             (int64_t)grid * runs * 4,            // bchanged
                             (int64_t)runs * 4};                  // status
  KmLayout l;
  int64_t o = 0;
  for (int i = 0; i < 13; i++) {
    l.off[i] = o;
    o += (sizes[i] + 255) & ~(int64_t)255;
  }
  l.bytes = o;
  return l;
}

static int km_check(int dtype, int64_t n, int64_t d, int32_t k, int32_t runs) {
  TIP_REQUIRE(dtype == TIP_F32 || dtype == TIP_F64, "dtype must be TIP_F32 or TIP_F64");
  TIP_REQUIRE(k >= 1 && k <= kKmMaxK, "k must be in [1, 64]");
  TIP_REQUIRE(runs >= 1 && runs <= 64, "runs must be in [1, 64]");
  TIP_REQUIRE(n >= k && n < (1LL << 31) && d >= 1 && (int64_t)runs * k * d < (1LL << 31), "shape");
  return TIP_OK;
}

}  // namespace tip

using namespace tip;

extern "C" int64_t tip_kmeans_work_bytes(int64_t n, int64_t d, int32_t k, int32_t runs, int dtype) {
  if (km_check(dtype, n, d, k, runs) != TIP_OK) return -1;
  int grid = 0;
  const int rc = dtype == TIP_F32 ? km_grid<float>(n, (int)d, k, runs, &grid) : km_grid<double>(n, (int)d, k, runs, &grid);
  if (rc != TIP_OK) return -1;
  return km_layout(n, (int)d, k, runs, grid).bytes;
}

extern "C" int tip_kmeans_fit(const void* x, int dtype, int64_t n, int64_t d, int32_t k, int32_t runs, int32_t max_iter,
                              double tol, uint64_t seed, void* work, void* centers, int32_t* n_iter, void* stream) {
  int rc = km_check(dtype, n, d, k, runs);
  if (rc != TIP_OK) return rc;
  TIP_REQUIRE(x && work && centers && n_iter, "null pointer");
  TIP_REQUIRE(max_iter >= 0 && tol >= 0.0, "max_iter / tol");   // max_iter 0: the k-means++ seeds alone
  int grid = 0;
  rc = dtype == TIP_F32 ? km_grid<float>(n, (int)d, k, runs, &grid) : km_grid<double>(n, (int)d, k, runs, &grid);
  if (rc != TIP_OK) return rc;
  const KmLayout l = km_layout(n, (int)d, k, runs, grid);
  char* w = (char*)work;
  KmArgs a{};
  a.x = x; a.n = n; a.d = (int)d; a.k = k; a.runs = runs; a.trials = km_trials(k); a.max_iter = max_iter;
  a.dc = km_dc((int)d, k); a.tol = tol; a.seed = seed; a.cen = centers; a.n_iter = n_iter;
  a.closest = (double*)(w + l.off[0]); a.dtrial = (double*)(w + l.off[1]); a.bpart = (double*)(w + l.off[2]);
  a.bpot = (double*)(w + l.off[3]); a.psum = (double*)(w + l.off[4]); a.sums = (double*)(w + l.off[5]);
  a.dist = (double*)(w + l.off[6]); a.cand = (int32_t*)(w + l.off[7]); a.pcnt = (int32_t*)(w + l.off[8]);
  a.cnt = (int32_t*)(w + l.off[9]); a.labels = (int32_t*)(w + l.off[10]); a.bchanged = (int32_t*)(w + l.off[11]);
  a.status = (int32_t*)(w + l.off[12]);
  const size_t smem = (size_t)k * a.dc * sizeof(double);
  void* args[] = {(void*)&a};
  const void* fn = dtype == TIP_F32 ? (const void*)kmeans_fit_kernel<float> : (const void*)kmeans_fit_kernel<double>;
  TIP_CHECK_CUDA(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(kKmThreads), args, smem, (cudaStream_t)stream));
  tip::count_launch();
  return TIP_OK;
}

extern "C" int tip_kmeans_predict(const void* x, int dtype, int64_t n, int64_t d, const void* centers, int32_t k,
                                  int32_t runs, int32_t* labels, double* sqdist, double* inertia, void* stream) {
  TIP_REQUIRE(dtype == TIP_F32 || dtype == TIP_F64, "dtype must be TIP_F32 or TIP_F64");
  TIP_REQUIRE(k >= 1 && k <= kKmMaxK && runs >= 1 && n >= 0 && d >= 1 && d < (1LL << 31), "shape");
  TIP_REQUIRE(x && centers && labels, "null pointer");
  TIP_REQUIRE(!inertia || sqdist, "inertia needs sqdist");
  if (n == 0) return TIP_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = (int)std::min<int64_t>((n + kKmWarps - 1) / kKmWarps, (int64_t)sm_count() * 8);
  if (dtype == TIP_F32)
    kmeans_predict_kernel<float><<<grid, kKmThreads, 0, st>>>((const float*)x, n, (int)d, (const float*)centers, k, runs,
                                                              labels, sqdist);
  else
    kmeans_predict_kernel<double><<<grid, kKmThreads, 0, st>>>((const double*)x, n, (int)d, (const double*)centers, k,
                                                               runs, labels, sqdist);
  TIP_LAUNCH_CHECK();
  if (inertia) {
    kmeans_inertia_kernel<<<runs, kKmThreads, 0, st>>>(sqdist, n, inertia);
    TIP_LAUNCH_CHECK();
  }
  return TIP_OK;
}

extern "C" int tip_sil_finish(const float* part_sum, int64_t n, int32_t slots, const int32_t* slot_cluster,
                              const int32_t* labels_sorted, const int32_t* counts, const int32_t* out_idx, double* out,
                              void* stream) {
  TIP_REQUIRE(part_sum && slot_cluster && labels_sorted && counts && out, "null pointer");
  TIP_REQUIRE(n >= 0 && slots >= 1, "shape");
  if (n == 0) return TIP_OK;
  sil_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(part_sum, n, slots, slot_cluster,
                                                                                  labels_sorted, counts, out_idx, out);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}
