// common.cuh — shared helpers for libb200tip.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/b200tip.h"

namespace tip {

// ---- error plumbing ---------------------------------------------------------------------
void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define TIP_CHECK_CUDA(expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      tip::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return TIP_ERR_CUDA;                                                                \
    }                                                                                     \
  } while (0)

#define TIP_REQUIRE(cond, msg)                                                            \
  do {                                                                                    \
    if (!(cond)) {                                                                        \
      tip::set_error("%s:%d invalid argument: %s (%s)", __FILE__, __LINE__, msg, #cond);  \
      return TIP_ERR_INVALID;                                                             \
    }                                                                                     \
  } while (0)

#define TIP_LAUNCH_CHECK()                                                                \
  do {                                                                                    \
    tip::count_launch();                                                                  \
    TIP_CHECK_CUDA(cudaGetLastError());                                                   \
  } while (0)

int sm_count();

// ---- counter-based RNG: one splitmix64 step; a key (seed, k1, k2, ...) is hashed as mix(...mix(mix(seed) ^ k1) ^ k2...)
__host__ __device__ __forceinline__ uint64_t km_mix(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// ---- IEEE arithmetic without FMA contraction (NumPy never fuses) --------------------------
template <typename T> struct Rn;
template <> struct Rn<float> {
  static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float sqrt(float a) { return __fsqrt_rn(a); }
  static __device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
  static __device__ __forceinline__ float inf() { return __int_as_float(0x7f800000); }
};
template <> struct Rn<double> {
  static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double sqrt(double a) { return __dsqrt_rn(a); }
  static __device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }
  static __device__ __forceinline__ double inf() { return __longlong_as_double(0x7ff0000000000000LL); }
};

// ---- NumPy's pairwise summation of a per-element term -------------------------------------------
// numpy/_core/src/umath/loops_utils.h: a block of at most kPairwiseLeaf elements is a leaf (n < 8 sequential from 0;
// else eight stride-8 accumulators, combined ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the tail sequentially); a
// larger block is split at pairwise_split(n) and its halves' sums are added.  Every sum below takes the element's
// term as term(i) -> T: (x-y)^2 for the DSA re-rank, x^2 for DeepGini, q*log2(q) for the entropy, the covariance's
// values and squared deviations.  All adds are IEEE roundings without contraction (Rn<T>), as NumPy's.
constexpr int kPairwiseLeaf = 128;

__host__ __device__ constexpr int pairwise_split(int n) { return n / 2 - (n / 2) % 8; }

// one leaf [off, off + n) by one thread
template <typename T, typename F>
__device__ __forceinline__ T np_leaf_sum(const F& term, int off, int n) {
  using R = Rn<T>;
  if (n < 8) {
    T res = (T)0;
    for (int i = 0; i < n; i++) res = R::add(res, term(off + i));
    return res;
  }
  T r0 = term(off + 0), r1 = term(off + 1), r2 = term(off + 2), r3 = term(off + 3);
  T r4 = term(off + 4), r5 = term(off + 5), r6 = term(off + 6), r7 = term(off + 7);
  int i = 8;
  const int lim = n - (n % 8);
  for (; i < lim; i += 8) {
    r0 = R::add(r0, term(off + i + 0)); r1 = R::add(r1, term(off + i + 1));
    r2 = R::add(r2, term(off + i + 2)); r3 = R::add(r3, term(off + i + 3));
    r4 = R::add(r4, term(off + i + 4)); r5 = R::add(r5, term(off + i + 5));
    r6 = R::add(r6, term(off + i + 6)); r7 = R::add(r7, term(off + i + 7));
  }
  T res = R::add(R::add(R::add(r0, r1), R::add(r2, r3)), R::add(R::add(r4, r5), R::add(r6, r7)));
  for (; i < n; i++) res = R::add(res, term(off + i));
  return res;
}

// One leaf by a group of 8 consecutive lanes.  Lane `sub` (0..7) owns NumPy's stride-8 accumulator r[sub]; the tree
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) is three xor-shuffles (IEEE addition is commutative, so every lane of the
// group ends with the same bits).  gmask names the 8 lanes of the calling group, so the four groups of a warp may
// diverge.  A leaf has at most 128 elements = 16 steps of the lane's accumulator: leaf_load_g8 issues all its terms
// up front (one memory round trip; this code sits at the end of a chain of dependent loads, latency is all that
// matters), leaf_reduce_g8 adds them in NumPy's order.  For n < 8 the tail registers hold elements 0..n-1 and the
// tree adds only zeros, so the tail is summed sequentially from +0 as NumPy does.
template <typename T>
struct LeafRegs {
  T t[16];
  T tail[7];
};

template <typename T, typename F>
__device__ __forceinline__ void leaf_load_g8(LeafRegs<T>& r, const F& term, int off, int n, int sub) {
  const int lim = n - (n % 8);
#pragma unroll
  for (int u = 0; u < 16; u++) r.t[u] = 8 * u + sub < lim ? term(off + 8 * u + sub) : (T)0;
#pragma unroll
  for (int u = 0; u < 7; u++) r.tail[u] = lim + u < n ? term(off + lim + u) : (T)0;
}

template <typename T>
__device__ __forceinline__ T leaf_reduce_g8(const LeafRegs<T>& r, int n, unsigned gmask) {
  using R = Rn<T>;
  const int lim = n - (n % 8);
  T acc = r.t[0];
#pragma unroll
  for (int u = 1; u < 16; u++)
    if (8 * u < lim) acc = R::add(acc, r.t[u]);          // uniform: lim is a multiple of 8
  acc = R::add(acc, __shfl_xor_sync(gmask, acc, 1));
  acc = R::add(acc, __shfl_xor_sync(gmask, acc, 2));
  acc = R::add(acc, __shfl_xor_sync(gmask, acc, 4));
#pragma unroll
  for (int u = 0; u < 7; u++)
    if (lim + u < n) acc = R::add(acc, r.tail[u]);
  return acc;
}

// The one-call form.  Below 8 elements every lane sums the leaf itself: with lim >= 8 known on the other path, ptxas
// adds the terms as they arrive and the wide row-statistic kernels keep their register budget (ENTROPY float: 55;
// 64 when this form is only reduce(load())).
template <typename T, typename F>
__device__ __forceinline__ T np_leaf_sum_g8(const F& term, int off, int n, int sub, unsigned gmask) {
  if (n < 8) return np_leaf_sum<T>(term, off, n);
  LeafRegs<T> r;
  leaf_load_g8<T>(r, term, off, n, sub);
  return leaf_reduce_g8<T>(r, n, gmask);
}

// NumPy's recursion over n elements with an explicit stack (depth <= 32 for n < 2^31); leaf(off, len) -> T sums one
// leaf, by np_leaf_sum or np_leaf_sum_g8
template <typename T, typename L>
__device__ T np_pairwise(const L& leaf, int n) {
  if (n <= kPairwiseLeaf) return leaf(0, n);
  int off[32], len[32];
  unsigned char phase[32];
  T vals[32];
  int sp = 1, vp = 0;
  off[0] = 0; len[0] = n; phase[0] = 0;
  while (sp > 0) {
    const int top = sp - 1;
    const int o = off[top], l = len[top];
    if (l <= kPairwiseLeaf) {
      vals[vp++] = leaf(o, l);
      sp--;
      continue;
    }
    const int n2 = pairwise_split(l);
    if (phase[top] == 0) {
      phase[top] = 1;
      off[sp] = o; len[sp] = n2; phase[sp] = 0; sp++;
    } else if (phase[top] == 1) {
      phase[top] = 2;
      off[sp] = o + n2; len[sp] = l - n2; phase[sp] = 0; sp++;
    } else {
      const T rgt = vals[--vp];
      const T lft = vals[--vp];
      vals[vp++] = Rn<T>::add(lft, rgt);
      sp--;
    }
  }
  return vals[0];
}

// NumPy's pairwise sum of term(0 .. n-1) by one thread
template <typename T, typename F>
__device__ T np_sum(const F& term, int n) {
  return np_pairwise<T>([&](int o, int l) { return np_leaf_sum<T>(term, o, l); }, n);
}

// ---- the same recursion as a precomputed leaf program -------------------------------------------
// The recursion visits its leaves left to right and combines the partial sums as a binary tree in post-order.  For
// a given width n that schedule is fixed, so the host flattens it once (sum_prog_for) into one word per leaf:
// offset/8 (20 bits) | len-1 (7 bits) | number of tree merges to perform after this leaf (5 bits).  Widths up to
// kSumProgMaxN fit: their walks hold at most 17 partial sums and merge at most 16 times after one leaf.
constexpr int64_t kSumProgMaxN = 1LL << 23;

struct SumLeaf {
  int off, len, merges;
};

__device__ __forceinline__ SumLeaf sum_leaf(uint32_t w) {
  return {(int)(w & 0xFFFFFu) * 8, (int)((w >> 20) & 127u) + 1, (int)(w >> 27)};
}

// The program for width n (1 <= n <= kSumProgMaxN) in device memory, cached per (device, n); defined in simple.cu.
// Allocates on first use, so the first call for a width must not be under stream capture.
int sum_prog_for(int64_t n, const uint32_t** prog, int* n_leaves);

// A program walk by a group of 8 lanes, with the value stack held in REGISTERS (static indexing: a push / merge
// shifts the whole stack) instead of the recursion's dynamically indexed arrays, which live in local memory
// (measured: the re-rank of 10 000 queries at D = 2048 took 0.85-1.0 ms with the recursion).  The next leaf's terms
// are loaded while the current one is reduced.
constexpr int kSumStack = 24;

template <typename T, typename F>
__device__ __forceinline__ T np_sum_prog_g8(const F& term, const uint32_t* __restrict__ prog, int n_leaves, int sub,
                                            unsigned gmask) {
  T st[kSumStack];
#pragma unroll
  for (int i = 0; i < kSumStack; i++) st[i] = (T)0;
  LeafRegs<T> cur, nxt;
  SumLeaf lf = sum_leaf(prog[0]);
  leaf_load_g8<T>(cur, term, lf.off, lf.len, sub);
  for (int li = 0; li < n_leaves; li++) {
    SumLeaf ln{0, 0, 0};
    if (li + 1 < n_leaves) {
      ln = sum_leaf(prog[li + 1]);
      leaf_load_g8<T>(nxt, term, ln.off, ln.len, sub);
    }
    const T v = leaf_reduce_g8<T>(cur, lf.len, gmask);
#pragma unroll
    for (int i = kSumStack - 1; i > 0; i--) st[i] = st[i - 1];     // push
    st[0] = v;
    for (int m = 0; m < lf.merges; m++) {                           // post-order merges: left + right
      st[0] = Rn<T>::add(st[1], st[0]);
#pragma unroll
      for (int i = 1; i < kSumStack - 1; i++) st[i] = st[i + 1];
    }
    cur = nxt;
    lf = ln;
  }
  return st[0];
}

__device__ __forceinline__ float warp_min(float v) {
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ int warp_sum(int v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Seed of a query's running minimum in tip_nn_filter's "approximate squared distance" space from an upper
// bound `ub` on the exact distance to SOME row of the range it is about to scan (DESIGN.md §4): that row's
// accumulator value s satisfies s <= (d + e)^2 + g with e the summed input-rounding norms and g the accumulation
// slack, so every threshold derived from the seed is at least as wide as the one the scan would reach on its
// own — the candidate set still contains NumPy's argmin, it just stops collecting far-away rows from tile one.
struct SeedParams {
  const float* ub;     // per train row (by position), +inf = no bound; nullptr = no seeding
  float t_rmax, t_err, gamma;
};

__device__ __forceinline__ uint32_t seed_row_min_bits(float ub, float nx, float q_err, const SeedParams& sp) {
  if (!(ub < __int_as_float(0x7f800000))) return 0x7f800000u;
  const float r = sqrtf(nx) + sp.t_rmax;
  const float e = (q_err + sp.t_err + 1.2e-7f * r) * 1.00001f;
  const float g = sp.gamma * r * r;
  const float d = ub * 1.000004f + e;
  const float s = (d * d + g) * 1.000002f;
  return s < __int_as_float(0x7f800000) ? __float_as_uint(s) : 0x7f800000u;
}

// One query row -> packed bf16 operand of tip_nn_filter (one segment) + reset filter state, by a full
// warp: the arithmetic of pair_prep_kernel (query role): centre in fp32, round to bf16, |h|^2 and
// the dropped part's norm accumulated in double.  src == nullptr packs a zero row.
template <typename T>
__device__ __forceinline__ void warp_pack_query(const T* __restrict__ src, int d, const float* __restrict__ center,
                                                __nv_bfloat16* __restrict__ out, int64_t pitch, float* sqnorm,
                                                float* rounderr, uint32_t* row_min, int32_t* cand_cnt, int lane,
                                                float seed_ub = 3.4e38f, const SeedParams* sp = nullptr) {
  const int d16 = (d + 15) & ~15;
  double acc = 0.0, err = 0.0;
  for (int c = lane; c < d16; c += 32) {
    float v = 0.f;
    if (c < d) {
      const T xv = src ? src[c] : (T)0;
      const float ctr = center ? center[c] : 0.f;
      v = sizeof(T) == 8 ? (float)((double)xv - (double)ctr) : __fsub_rn((float)xv, ctr);
    }
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    const float hf = __bfloat162float(h);
    const float res = __fsub_rn(v, hf);
    acc += (double)hf * (double)hf;
    err += (double)res * (double)res;
    out[c] = h;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    acc += __shfl_xor_sync(0xffffffffu, acc, o);
    err += __shfl_xor_sync(0xffffffffu, err, o);
  }
  for (int c = d16 + lane; c < pitch; c += 32) out[c] = __float2bfloat16_rn(c - d16 < 3 ? 1.f : 0.f);
  if (lane == 0) {
    const float nx = (float)acc;
    const float qe = (float)sqrt(err) * 1.000001f;
    *sqnorm = nx;
    if (rounderr) *rounderr = qe;
    // the seed needs the measured rounding norm; without it (a-priori window) no seeding
    *row_min = (sp && sp->ub && rounderr) ? seed_row_min_bits(seed_ub, nx, qe, *sp) : 0x7f800000u;
    *cand_cnt = 0;
  }
}

}  // namespace tip
