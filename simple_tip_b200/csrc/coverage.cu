// coverage.cu — the coverage criteria next to KMNC and their fit step (SURVEY.md §8 f2), plus the
// Coverage-Additional Method over dense boolean profiles as a bitset (§8 f1).
//
//   tip_cover_threshold  NAC  a > t                       neuron_coverage.py:52-62
//                        SNAC a >= max + s*std            neuron_coverage.py:135-148
//                        NBC  a <= min - s*std | a >= max + s*std   neuron_coverage.py:97-132
//                        (boundaries are computed by the caller with the reference's NumPy expressions;
//                        the kernel compares in NumPy's promoted dtype, so profiles are bit-identical)
//   tip_tknc             top-k neurons of one layer per sample                    neuron_coverage.py:151-173
//   tip_stats_update     streaming min / max / Welford (mean, M2) per neuron over batches of samples:
//                        the fit of KMNC / NBC / SNAC (aggregate_statistics.py:37-67, welford==0.2.5
//                        `add`: count += 1; delta = x - m; m += delta / count; s += delta * (x - m),
//                        applied sample by sample in the activation dtype — reproduced bit for bit)
//   tip_cam_bits         cam() of prioritizers.py:16-45 on bit-packed profiles, one persistent
//                        cooperative kernel for all greedy rounds
//   tip_cam_bits_stack   the same kernel's STACK instance for the profiles of a stack of models: one greedy loop
//                        per model, all under one grid barrier per round
//
// All three profile kernels write the reference's dense boolean profile (one byte per entry, what the
// classes return) and/or the same profile bit-packed for tip_cam_bits.  Packed layout (a fixed
// permutation of the profile entries, which CAM is invariant to): neurons are taken in groups of 128;
// word 4*g + i of a row holds, in bit `l`, the entry of neuron 128*g + 4*l + i.  NBC has two such planes
// (lower-boundary entries, then upper-boundary entries).
#include <cooperative_groups.h>

#include <algorithm>
#include "common.cuh"

namespace cg = cooperative_groups;

namespace tip {

template <typename TA, typename TS> struct Cmp { using type = double; };
template <> struct Cmp<float, float> { using type = float; };

__host__ __device__ inline int64_t packed_words(int64_t d) { return 4 * ((d + 127) / 128); }

// ---- NAC / SNAC / NBC -------------------------------------------------------------------------------
// A block owns 1024 consecutive neurons (4 per thread, boundaries in registers) and walks down a group of
// samples; per sample a thread loads its 4 activations (one 128-bit load when aligned), compares, stores 4
// (NAC/SNAC) or 8 (NBC) profile bytes, contributes to the packed words by ballot, and the warp adds its
// count to the sample's score with one atomic.
template <typename TA, typename TS, int MODE>
__global__ void __launch_bounds__(256) cover_threshold_kernel(const TA* __restrict__ act, int64_t n, int64_t d,
                                                              const TS* __restrict__ lo, const TS* __restrict__ hi,
                                                              double thr, unsigned char* __restrict__ profile,
                                                              uint32_t* __restrict__ bits, int32_t* __restrict__ score,
                                                              int rows_per_block) {
  using C = typename Cmp<TA, TS>::type;
  const int lane = threadIdx.x & 31;
  const int64_t c0 = (int64_t)blockIdx.x * 1024 + threadIdx.x * 4;
  const int64_t words = packed_words(d);
  const bool vec = (d % 4 == 0) && sizeof(TA) == 4 && ((uintptr_t)act % 16 == 0);
  C blo[4], bhi[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const bool in = c0 + j < d;
    blo[j] = (MODE == TIP_COVER_NBC && in) ? (C)lo[c0 + j] : (C)0;
    bhi[j] = MODE == TIP_COVER_NAC ? (C)thr : (in ? (C)hi[c0 + j] : (C)0);
  }
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
  const int64_t r1 = r0 + rows_per_block < n ? r0 + rows_per_block : n;
  for (int64_t r = r0; r < r1; r++) {
    C a[4];
    if (vec && c0 + 3 < d) {
      const float4 v = *reinterpret_cast<const float4*>(act + r * d + c0);
      a[0] = (C)v.x; a[1] = (C)v.y; a[2] = (C)v.z; a[3] = (C)v.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; j++) a[j] = c0 + j < d ? (C)act[r * d + c0 + j] : (C)0;
    }
    bool up[4], dn[4];
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const bool in = c0 + j < d;
      up[j] = in && (MODE == TIP_COVER_NAC ? a[j] > bhi[j] : a[j] >= bhi[j]);
      dn[j] = MODE == TIP_COVER_NBC && in && a[j] <= blo[j];
      cnt += (int)up[j] + (int)dn[j];
    }
    if (profile) {
      if (MODE == TIP_COVER_NBC) {
        unsigned char* p = profile + (r * d + c0) * 2;
        if (c0 + 3 < d && ((uintptr_t)p % 8 == 0)) {
          uint2 w;
          w.x = (uint32_t)dn[0] | ((uint32_t)up[0] << 8) | ((uint32_t)dn[1] << 16) | ((uint32_t)up[1] << 24);
          w.y = (uint32_t)dn[2] | ((uint32_t)up[2] << 8) | ((uint32_t)dn[3] << 16) | ((uint32_t)up[3] << 24);
          *reinterpret_cast<uint2*>(p) = w;
        } else {
#pragma unroll
          for (int j = 0; j < 4; j++)
            if (c0 + j < d) { p[2 * j] = dn[j]; p[2 * j + 1] = up[j]; }
        }
      } else {
        unsigned char* p = profile + r * d + c0;
        if (c0 + 3 < d && ((uintptr_t)p % 4 == 0)) {
          *reinterpret_cast<uint32_t*>(p) = (uint32_t)up[0] | ((uint32_t)up[1] << 8) | ((uint32_t)up[2] << 16) | ((uint32_t)up[3] << 24);
        } else {
#pragma unroll
          for (int j = 0; j < 4; j++)
            if (c0 + j < d) p[j] = up[j];
        }
      }
    }
    if (bits) {
      const int64_t g = c0 / 128;                  // this warp's group of 128 neurons
      uint32_t* row = bits + r * (MODE == TIP_COVER_NBC ? 2 * words : words);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const uint32_t bu = __ballot_sync(0xffffffffu, up[j]);
        if (MODE == TIP_COVER_NBC) {
          const uint32_t bd = __ballot_sync(0xffffffffu, dn[j]);
          if (lane == 0 && c0 < d) { row[4 * g + j] = bd; row[words + 4 * g + j] = bu; }
        } else if (lane == 0 && c0 < d) {
          row[4 * g + j] = bu;
        }
      }
    }
    cnt = warp_sum(cnt);
    if (lane == 0 && cnt) atomicAdd(score + r, cnt);
  }
}

// ---- TKNC -------------------------------------------------------------------------------------------
// One block per sample: k rounds of "largest remaining value" over the layer held in registers/shared
// memory; k >= d_layer marks the whole layer without any round.  Ties at equal values go to the HIGHER index (where a stable ascending argsort puts them last);
// NumPy's own argsort is not stable, so for tied values the reference's choice is implementation-defined
// (its test accepts either, tests/test_coverage_metrics.py:157-162).
template <typename T>
__global__ void __launch_bounds__(256) tknc_kernel(const T* __restrict__ act, int64_t n, int64_t d_layer, int k,
                                                   unsigned char* __restrict__ profile, int64_t row_stride,
                                                   int64_t col_off, uint32_t* __restrict__ bits, int64_t bit_words) {
  extern __shared__ unsigned char s_raw[];
  unsigned char* taken = s_raw;                   // d_layer flags
  __shared__ double s_val[8];
  __shared__ long long s_idx[8];
  const int64_t r = blockIdx.x;
  const T* x = act + r * d_layer;
  const bool all = k >= d_layer;                  // the whole layer: no rounds
  for (int64_t i = threadIdx.x; i < d_layer; i += 256) taken[i] = all;
  __syncthreads();
  const int kk = all ? 0 : k;
  for (int round = 0; round < kk; round++) {
    double bv = -INFINITY;
    long long bi = -1;
    for (int64_t i = threadIdx.x; i < d_layer; i += 256) {
      if (taken[i]) continue;
      const double v = (double)x[i];
      // NaN sorts last in np.argsort: treat as larger than everything
      const bool better = bi < 0 || (v != v ? true : (bv == bv && (v > bv || (v == bv && i > bi))));
      if (better) { bv = v; bi = i; }
    }
    auto take = [](double v, long long i, double v2, long long i2) {
      if (i2 < 0) return false;
      if (i < 0) return true;
      const bool n1 = v != v, n2 = v2 != v2;
      if (n1 != n2) return n2;
      if (n1) return i2 > i;
      return v2 > v || (v2 == v && i2 > i);
    };
    for (int o = 16; o > 0; o >>= 1) {
      const double v2 = __shfl_xor_sync(0xffffffffu, bv, o);
      const long long i2 = __shfl_xor_sync(0xffffffffu, bi, o);
      if (take(bv, bi, v2, i2)) { bv = v2; bi = i2; }
    }
    if ((threadIdx.x & 31) == 0) { s_val[threadIdx.x >> 5] = bv; s_idx[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < 8; w++)
        if (take(bv, bi, s_val[w], s_idx[w])) { bv = s_val[w]; bi = s_idx[w]; }
      if (bi >= 0) taken[bi] = 1;
    }
    __syncthreads();
  }
  for (int64_t i = threadIdx.x; i < d_layer; i += 256) {
    if (profile) profile[r * row_stride + col_off + i] = taken[i];
    if (bits && taken[i]) {
      const int64_t c = col_off + i;
      atomicOr(bits + r * bit_words + 4 * (c / 128) + (c % 4), 1u << ((c % 128) / 4));
    }
  }
}

// ---- streaming statistics -----------------------------------------------------------------------------
// One thread per neuron walks down the batch in order (welford's add_all is a sequential loop over the
// samples; mean and M2 live in the activation dtype, count is an integer); loads of the next samples are
// issued ahead of the dependent arithmetic.  IEEE ops, no FMA contraction.
template <typename T>
__global__ void __launch_bounds__(128) stats_update_kernel(const T* __restrict__ act, int64_t n, int64_t d,
                                                           int64_t count0, T* __restrict__ mean, T* __restrict__ m2,
                                                           T* __restrict__ mn, T* __restrict__ mx) {
  using R = Rn<T>;
  const int64_t c = (int64_t)blockIdx.x * 128 + threadIdx.x;
  if (c >= d) return;
  T m = mean[c], s = m2[c], lo = mn[c], hi = mx[c];
  int64_t cnt = count0;
  constexpr int U = 8;
  int64_t r = 0;
  for (; r + U <= n; r += U) {
    T x[U];
#pragma unroll
    for (int u = 0; u < U; u++) x[u] = act[(r + u) * d + c];
#pragma unroll
    for (int u = 0; u < U; u++) {
      cnt += 1;
      const T delta = R::sub(x[u], m);
      m = R::add(m, R::div(delta, (T)cnt));
      s = R::add(s, R::mul(delta, R::sub(x[u], m)));
      lo = x[u] < lo ? x[u] : lo;      // np.minimum propagates NaN; NaN activations are unsupported input
      hi = x[u] > hi ? x[u] : hi;
    }
  }
  for (; r < n; r++) {
    const T xv = act[r * d + c];
    cnt += 1;
    const T delta = R::sub(xv, m);
    m = R::add(m, R::div(delta, (T)cnt));
    s = R::add(s, R::mul(delta, R::sub(xv, m)));
    lo = xv < lo ? xv : lo;
    hi = xv > hi ? xv : hi;
  }
  mean[c] = m; m2[c] = s; mn[c] = lo; mx[c] = hi;
}

// ---- CAM over bit-packed profiles: one persistent cooperative kernel ---------------------------------------
// Per round: (A) every block finds the best (gain, lowest index) of its own slice of samples and publishes
// it; grid.sync; (B) every block reduces the published candidates to the same pick, derives the newly
// covered words new = profile[pick] & ~covered (kept as a compact list of non-zero words in shared memory)
// — block 0 records the pick and writes covered | new into the other half of the double-buffered covered
// set; (C) every block subtracts popcount(profile[n] & new) from the gains of its slice.  A block only ever
// reads gains it wrote itself, so one grid.sync per round suffices (candidates and covered are
// double-buffered by round parity).
//
// STACK: the profiles of a stack of models, one greedy loop per model under the same grid.sync.  The grid is cut
// into gridDim.x / bpm groups of bpm consecutive blocks; group g runs (A)/(B)/(C) on model g's profile, gains,
// covered set, order and state, and its first block takes block 0's part.  After the barrier each block reduces
// its own group's candidates to that model's pick and also checks whether any group still has a positive best;
// when none has, every block leaves.  A pick depends only on the model's gains (first index of the largest), never
// on the block partition, so slice g equals the single-model kernel on model g.  bpm is a parameter of the stack
// instance only (the pack Bpm is empty for STACK = false), so each instance keeps its own parameter layout.
constexpr int kCamThreads = 256;
constexpr int kCamMaxList = 4096;     // non-zero words of `new` kept in shared memory (32 KB as int2)

template <bool STACK, class... Bpm>
__global__ void __launch_bounds__(kCamThreads) cam_bits_kernel(const uint32_t* __restrict__ prof, int n, int words,
                                                               Bpm... bpm_arg, int32_t* __restrict__ gain,
                                                               uint32_t* __restrict__ covered2,
                                                               int2* __restrict__ cand2, int32_t* __restrict__ order,
                                                               int32_t* __restrict__ state, int max_rounds) {
  static_assert(sizeof...(Bpm) == (STACK ? 1 : 0), "bpm (blocks per model) is the stack instance's parameter");
  cg::grid_group grid = cg::this_grid();
  __shared__ int2 s_list[kCamMaxList];
  __shared__ int s_gain[kCamThreads / 32], s_idx[kCamThreads / 32];
  __shared__ int s_n, s_pick, s_best;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nb = gridDim.x;
  int bpm = nb, g = 0, gb = blockIdx.x;            // one model: one group of all blocks
  if constexpr (STACK) {
    bpm = (bpm_arg + ...);
    g = blockIdx.x / bpm;
    gb = blockIdx.x - g * bpm;
  }
  const int g0 = g * bpm;
  const int per = (n + bpm - 1) / bpm;
  const int lo = gb * per, hi = min(n, lo + per);
  if constexpr (STACK) {
    prof += (size_t)g * n * words;
    gain += (size_t)g * n;
    covered2 += (size_t)g * 2 * words;
    order += (size_t)g * n;
    state += 4 * g;
  }
  // the thread that records the group's picks and state; the single-model instance tests it at each store, as
  // hoisting the test would change that instance's code
  const bool first_thread = gb == 0 && threadIdx.x == 0;
  auto lead = [&] { return STACK ? first_thread : gb == 0 && threadIdx.x == 0; };
  auto better = [](int a, int i, int a2, int i2) { return a2 > a || (a2 == a && i2 < i); };
  int picks = state[0];
  bool done = false;
  if constexpr (STACK) done = state[1] != 0;      // a finished group still joins every grid.sync, see below
  else if (state[1]) return;
  for (int round = 0; round < max_rounds; round++) {
    const int par = round & 1;
    // (A) best of the own slice; a finished group publishes (-1, -)
    int bg = -1, bi = 0x7fffffff;
    for (int i = lo + threadIdx.x, end = done ? lo : hi; i < end; i += kCamThreads) {
      const int gi = gain[i];
      if (gi > bg) { bg = gi; bi = i; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const int g2 = __shfl_xor_sync(0xffffffffu, bg, o), i2 = __shfl_xor_sync(0xffffffffu, bi, o);
      if (better(bg, bi, g2, i2)) { bg = g2; bi = i2; }
    }
    if (lane == 0) { s_gain[warp] = bg; s_idx[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kCamThreads / 32; w++)
        if (better(bg, bi, s_gain[w], s_idx[w])) { bg = s_gain[w]; bi = s_idx[w]; }
      cand2[par * nb + blockIdx.x] = make_int2(bg, bi);
    }
    // STACK: a finished group keeps taking part in every grid.sync: the barrier counts every block of the grid, so a
    // block that returned while others still loop would hang it.  Blocks leave only all together, below.
    grid.sync();
    // (B) the own model's pick, identically in every block of the group, and whether any group goes on
    bg = -1; bi = 0x7fffffff;
    int live = 0;
    for (int b = threadIdx.x; b < nb; b += kCamThreads) {
      const int2 c = cand2[par * nb + b];
      live |= c.x > 0;
      if ((!STACK || (b >= g0 && b < g0 + bpm)) && better(bg, bi, c.x, c.y)) { bg = c.x; bi = c.y; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const int g2 = __shfl_xor_sync(0xffffffffu, bg, o), i2 = __shfl_xor_sync(0xffffffffu, bi, o);
      if (better(bg, bi, g2, i2)) { bg = g2; bi = i2; }
    }
    if (lane == 0) { s_gain[warp] = bg; s_idx[warp] = bi; }
    bool any_live = true;
    if constexpr (STACK) any_live = __syncthreads_or(live);
    else __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kCamThreads / 32; w++)
        if (better(bg, bi, s_gain[w], s_idx[w])) { bg = s_gain[w]; bi = s_idx[w]; }
      s_best = bg; s_pick = bi; s_n = 0;
    }
    __syncthreads();
    if (!done && s_best <= 0) {                      // nothing new can be covered (prioritizers.py:30-31)
      done = true;
      if (lead()) { state[1] = 1; state[0] = picks; }
      if constexpr (!STACK) return;
    }
    if (!any_live) return;
    if (done) continue;
    const int pick = s_pick;
    const uint32_t* cov = covered2 + (size_t)par * words;
    uint32_t* cov_next = covered2 + (size_t)(par ^ 1) * words;
    const uint32_t* prow = prof + (size_t)pick * words;
    for (int w = threadIdx.x; w < words; w += kCamThreads) {
      const uint32_t c = cov[w];
      const uint32_t fresh = prow[w] & ~c;
      if (gb == 0) cov_next[w] = c | fresh;
      if (fresh) {
        const int pos = atomicAdd(&s_n, 1);
        if (pos < kCamMaxList) s_list[pos] = make_int2(w, (int)fresh);
      }
    }
    __syncthreads();
    if (lead()) order[picks] = pick;
    picks++;
    const int nn = s_n;
    // (C) gains of the own slice
    for (int i = lo + warp; i < hi; i += kCamThreads / 32) {
      if (gain[i] == 0) continue;                   // warp-uniform
      const uint32_t* row = prof + (size_t)i * words;
      int cnt = 0;
      if (nn <= kCamMaxList) {
        for (int e = lane; e < nn; e += 32) cnt += __popc(row[s_list[e].x] & (uint32_t)s_list[e].y);
      } else {                                      // very dense pick: walk all words
        for (int w = lane; w < words; w += 32) cnt += __popc(row[w] & prow[w] & ~cov[w]);
      }
      cnt = warp_sum(cnt);
      if (lane == 0 && cnt) gain[i] -= cnt;
    }
    __syncthreads();
  }
  if (lead()) state[0] = picks;
}

__global__ void __launch_bounds__(256) popcount_rows_kernel(const uint32_t* __restrict__ prof, int n, int words,
                                                            int32_t* __restrict__ gain) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= n) return;
  int cnt = 0;
  for (int w = lane; w < words; w += 32) cnt += __popc(prof[(size_t)row * words + w]);
  cnt = warp_sum(cnt);
  if (lane == 0) gain[row] = cnt;
}

// byte profile [n, f] -> packed words (plain order: bit b of word w = entry 32*w + b); used for profiles
// that arrive as dense boolean arrays (the reference's `cam(scores, profiles)` signature)
__global__ void __launch_bounds__(256) pack_bool_kernel(const unsigned char* __restrict__ prof, int64_t n, int64_t f,
                                                        int64_t words, uint32_t* __restrict__ bits) {
  const int lane = threadIdx.x & 31;
  const int64_t wid = ((int64_t)blockIdx.x * 256 + threadIdx.x) >> 5;
  if (wid >= n * words) return;
  const int64_t r = wid / words, w = wid - r * words;
  const int64_t e = w * 32 + lane;
  const uint32_t b = __ballot_sync(0xffffffffu, e < f && prof[r * f + e] != 0);
  if (lane == 0) bits[wid] = b;
}

}  // namespace tip

using namespace tip;

extern "C" int64_t tip_cover_packed_words(int64_t d) { return d < 1 ? -1 : packed_words(d); }

extern "C" int tip_cover_threshold(const void* act, int act_dtype, int64_t n, int64_t d, const void* lo, const void* hi,
                                   int stat_dtype, double threshold, int mode, void* profile_u8, uint32_t* bits,
                                   int32_t* score, void* stream) {
  TIP_REQUIRE(act && score, "null pointer");
  TIP_REQUIRE(mode == TIP_COVER_NAC || mode == TIP_COVER_SNAC || mode == TIP_COVER_NBC, "mode");
  TIP_REQUIRE(mode == TIP_COVER_NAC || hi != nullptr, "upper boundaries");
  TIP_REQUIRE(mode != TIP_COVER_NBC || lo != nullptr, "lower boundaries");
  TIP_REQUIRE(n >= 0 && d >= 1, "shape");
  TIP_REQUIRE((act_dtype == TIP_F32 || act_dtype == TIP_F64) && (stat_dtype == TIP_F32 || stat_dtype == TIP_F64), "dtype");
  if (n == 0) return TIP_OK;
  cudaStream_t st = (cudaStream_t)stream;
  TIP_CHECK_CUDA(cudaMemsetAsync(score, 0, (size_t)n * sizeof(int32_t), st));
  const int gx = (int)((d + 1023) / 1024);
  // enough blocks to fill the chip a few times over, whole rows per block
  int64_t gy = std::max<int64_t>(1, std::min<int64_t>(n, (int64_t)sm_count() * 8 / gx));
  const int rows = (int)((n + gy - 1) / gy);
  gy = (n + rows - 1) / rows;
  TIP_REQUIRE(gy <= 65535, "too many row groups");
  dim3 grid((unsigned)gx, (unsigned)gy);
#define TIP_COVER(TA, TS, M)                                                                                       \
  cover_threshold_kernel<TA, TS, M><<<grid, 256, 0, st>>>((const TA*)act, n, d, (const TS*)lo, (const TS*)hi, threshold, \
                                                         (unsigned char*)profile_u8, bits, score, rows)
#define TIP_COVER_M(TA, TS)                                                   \
  do {                                                                        \
    if (mode == TIP_COVER_NAC) TIP_COVER(TA, TS, TIP_COVER_NAC);              \
    else if (mode == TIP_COVER_SNAC) TIP_COVER(TA, TS, TIP_COVER_SNAC);       \
    else TIP_COVER(TA, TS, TIP_COVER_NBC);                                    \
  } while (0)
  if (act_dtype == TIP_F32 && stat_dtype == TIP_F32) TIP_COVER_M(float, float);
  else if (act_dtype == TIP_F32) TIP_COVER_M(float, double);
  else if (stat_dtype == TIP_F32) TIP_COVER_M(double, float);
  else TIP_COVER_M(double, double);
#undef TIP_COVER_M
#undef TIP_COVER
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_tknc(const void* act, int dtype, int64_t n, int64_t d_layer, int32_t k, void* profile_u8,
                        int64_t row_stride, int64_t col_off, uint32_t* bits, int64_t bit_words, void* stream) {
  TIP_REQUIRE(act && (profile_u8 || bits), "null pointer");
  TIP_REQUIRE(n >= 0 && d_layer >= 1 && k >= 0 && n < (1LL << 31), "shape");
  TIP_REQUIRE(d_layer <= 200 * 1024, "layer too wide for the shared-memory flags (max 204800 neurons)");
  TIP_REQUIRE(dtype == TIP_F32 || dtype == TIP_F64, "dtype");
  if (n == 0) return TIP_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = (size_t)d_layer;
  if (dtype == TIP_F32) {
    if (smem > 48 * 1024) TIP_CHECK_CUDA(cudaFuncSetAttribute(tknc_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    tknc_kernel<float><<<(unsigned)n, 256, smem, st>>>((const float*)act, n, d_layer, k, (unsigned char*)profile_u8,
                                                      row_stride, col_off, bits, bit_words);
  } else {
    if (smem > 48 * 1024) TIP_CHECK_CUDA(cudaFuncSetAttribute(tknc_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    tknc_kernel<double><<<(unsigned)n, 256, smem, st>>>((const double*)act, n, d_layer, k, (unsigned char*)profile_u8,
                                                       row_stride, col_off, bits, bit_words);
  }
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_stats_update(const void* act, int dtype, int64_t n, int64_t d, int64_t count_before, void* mean,
                                void* m2, void* mins, void* maxs, void* stream) {
  TIP_REQUIRE(act && mean && m2 && mins && maxs, "null pointer");
  TIP_REQUIRE(n >= 0 && d >= 1 && count_before >= 0, "shape");
  TIP_REQUIRE(dtype == TIP_F32 || dtype == TIP_F64, "dtype");
  if (n == 0) return TIP_OK;
  const unsigned blocks = (unsigned)((d + 127) / 128);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == TIP_F32)
    stats_update_kernel<float><<<blocks, 128, 0, st>>>((const float*)act, n, d, count_before, (float*)mean, (float*)m2,
                                                      (float*)mins, (float*)maxs);
  else
    stats_update_kernel<double><<<blocks, 128, 0, st>>>((const double*)act, n, d, count_before, (double*)mean,
                                                       (double*)m2, (double*)mins, (double*)maxs);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_pack_bool(const void* profile_u8, int64_t n, int64_t f, uint32_t* bits, void* stream) {
  TIP_REQUIRE(profile_u8 && bits, "null pointer");
  TIP_REQUIRE(n >= 0 && f >= 1, "shape");
  if (n == 0) return TIP_OK;
  const int64_t words = (f + 31) / 32;
  const int64_t warps = n * words;
  pack_bool_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const unsigned char*)profile_u8,
                                                                                         n, f, words, bits);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

// Both CAM entry points: `models` profiles [n, words] back to back, each with its own gains, covered set, order and
// state.  A co-resident grid holds cap blocks; a chunk of c models gets bpm = max(1, min(cap / c, ceil(n / 64)))
// blocks per model.  For one model (tip_cam_bits) that is one group of max(1, min(SMs x min(per_sm, 2), ceil(n / 64),
// TIP_CAM_MAX_BLOCKS)) blocks: at most two per SM and at least 64 samples per block.  Models beyond one co-resident
// grid run in consecutive chunks, each model keeping its own state across them.
template <bool STACK>
static int cam_bits_launch(const uint32_t* bits, int64_t models, int64_t n, int64_t words, int32_t* gain,
                           uint32_t* covered2, int32_t* cand_scratch, int32_t* order, int32_t* state, int32_t max_rounds,
                           int32_t init_gain, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (init_gain) {
    popcount_rows_kernel<<<(unsigned)((models * n + 7) / 8), 256, 0, st>>>(bits, (int)(models * n), (int)words, gain);
    TIP_LAUNCH_CHECK();
  }
  if (max_rounds == 0) return TIP_OK;
  const void* kernel = STACK ? (const void*)cam_bits_kernel<true, int> : (const void*)cam_bits_kernel<false>;
  int per_sm = 0;
  TIP_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kCamThreads, 0));
  TIP_REQUIRE(per_sm >= 1, "cooperative kernel does not fit");
  const int cap = (int)std::min<int64_t>((int64_t)sm_count() * std::min(per_sm, 2), TIP_CAM_MAX_BLOCKS);
  for (int64_t m0 = 0; m0 < models; m0 += cap) {
    const int chunk = (int)std::min<int64_t>(cap, models - m0);
    int bpm = (int)std::max<int64_t>(1, std::min<int64_t>(cap / chunk, (n + 63) / 64));
    const uint32_t* b = bits + (size_t)m0 * n * words;
    int32_t* g = gain + (size_t)m0 * n;
    uint32_t* cov = covered2 + (size_t)m0 * 2 * words;
    int32_t* ord = order + (size_t)m0 * n;
    int32_t* sta = state + (size_t)m0 * 4;
    int2* cand = (int2*)cand_scratch;
    int ni = (int)n, wi = (int)words, mr = max_rounds;
    void* args[] = {(void*)&b, (void*)&ni, (void*)&wi, (void*)&bpm, (void*)&g, (void*)&cov, (void*)&cand,
                    (void*)&ord, (void*)&sta, (void*)&mr};
    void* args_one[] = {(void*)&b, (void*)&ni, (void*)&wi, (void*)&g, (void*)&cov, (void*)&cand, (void*)&ord,
                        (void*)&sta, (void*)&mr};   // cam_bits_kernel<false> takes no bpm
    TIP_CHECK_CUDA(cudaLaunchCooperativeKernel(kernel, dim3(chunk * bpm), dim3(kCamThreads), STACK ? args : args_one,
                                               0, st));
    tip::count_launch();
  }
  return TIP_OK;
}

extern "C" int tip_cam_bits(const uint32_t* bits, int64_t n, int64_t words, int32_t* gain, uint32_t* covered2,
                            int32_t* cand_scratch, int32_t* order, int32_t* state, int32_t max_rounds, int32_t init_gain,
                            void* stream) {
  TIP_REQUIRE(bits && gain && covered2 && cand_scratch && order && state, "null pointer");
  TIP_REQUIRE(n >= 1 && n < (1LL << 31) && words >= 1 && words < (1LL << 31) && max_rounds >= 0, "shape");
  return cam_bits_launch<false>(bits, 1, n, words, gain, covered2, cand_scratch, order, state, max_rounds, init_gain,
                                stream);
}

extern "C" int tip_cam_bits_stack(const uint32_t* bits, int64_t models, int64_t n, int64_t words, int32_t* gain,
                                  uint32_t* covered2, int32_t* cand_scratch, int32_t* order, int32_t* state,
                                  int32_t max_rounds, int32_t init_gain, void* stream) {
  TIP_REQUIRE(bits && gain && covered2 && cand_scratch && order && state, "null pointer");
  TIP_REQUIRE(models >= 1 && models < (1LL << 31) && n >= 1 && n < (1LL << 31) && models * n < (1LL << 31) &&
              words >= 1 && words < (1LL << 31) && max_rounds >= 0, "shape");
  return cam_bits_launch<true>(bits, models, n, words, gain, covered2, cand_scratch, order, state, max_rounds,
                               init_gain, stream);
}
