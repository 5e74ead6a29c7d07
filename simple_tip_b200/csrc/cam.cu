// cam.cu — Coverage-Additional Method (prioritizers.py:16-59) over COMPACT coverage profiles.
//
// The reference's `cam(scores, profiles)` walks a dense boolean profile N x (D*k); for k-multisection
// coverage that profile is one-hot per neuron (neuron_coverage.py:82-94), i.e. fully described by the
// bucket ids tip_kmnc emits (N x D, -1 = no section), and at k = 1000 the dense form is 41 GB.  Here the
// greedy loop runs on the bucket ids: per round
//   pick    = first index of the largest remaining gain            (np.argmax, prioritizers.py:26)
//   collect = the cells (d, bucket[pick, d]) not covered before     (:27, :40-41), marked in a D*k bitset
//   update  = gain[n] -= #newly covered cells sample n shares       (:38-39)
// until the best gain is 0 (:30-31).  The order of the picks is written to `order`; the tail of the
// reference's generator (the not-yet-yielded samples by np.argsort(-scores), :47-59) stays on the host
// so that NumPy's own (unstable) sort decides ties exactly as in the reference.
#include <algorithm>
#include "common.cuh"

namespace tip {

// state[0] = picks so far, state[1] = done flag, state[2] = cells newly covered by the last pick,
// state[3] = last pick
__global__ void __launch_bounds__(1024) cam_pick_kernel(const int32_t* __restrict__ gain, int n,
                                                        int32_t* __restrict__ order, int32_t* __restrict__ state) {
  __shared__ int s_gain[32];
  __shared__ int s_idx[32];
  if (state[1]) return;
  int bg = -1, bi = 0x7fffffff;
  for (int i = threadIdx.x; i < n; i += 1024) {
    const int g = gain[i];
    if (g > bg) { bg = g; bi = i; }          // ascending i inside a thread: strict > keeps the first index
  }
  auto better = [](int g, int i, int g2, int i2) { return g2 > g || (g2 == g && i2 < i); };
  for (int o = 16; o > 0; o >>= 1) {
    const int g2 = __shfl_xor_sync(0xffffffffu, bg, o), i2 = __shfl_xor_sync(0xffffffffu, bi, o);
    if (better(bg, bi, g2, i2)) { bg = g2; bi = i2; }
  }
  if ((threadIdx.x & 31) == 0) { s_gain[threadIdx.x >> 5] = bg; s_idx[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x < 32) {
    bg = s_gain[threadIdx.x]; bi = s_idx[threadIdx.x];
    for (int o = 16; o > 0; o >>= 1) {
      const int g2 = __shfl_xor_sync(0xffffffffu, bg, o), i2 = __shfl_xor_sync(0xffffffffu, bi, o);
      if (better(bg, bi, g2, i2)) { bg = g2; bi = i2; }
    }
    if (threadIdx.x == 0) {
      if (bg <= 0) {
        state[1] = 1;                        // nothing new can be covered (prioritizers.py:30-31)
      } else {
        order[state[0]] = bi;
        state[0] = state[0] + 1;
        state[3] = bi;
        state[2] = 0;
      }
    }
  }
}

template <typename TB>
__global__ void __launch_bounds__(256) cam_collect_kernel(const TB* __restrict__ bucket, int d, int k,
                                                          uint32_t* __restrict__ covered,
                                                          int2* __restrict__ newlist, int32_t* __restrict__ state) {
  if (state[1]) return;
  const int col = blockIdx.x * 256 + threadIdx.x;
  if (col >= d) return;
  const int pick = state[3];
  const int c = (int)bucket[(int64_t)pick * d + col];
  if (c < 0 || c >= k) return;
  const int64_t bit = (int64_t)col * k + c;
  const uint32_t mask = 1u << (bit & 31);
  const uint32_t old = atomicOr(covered + (bit >> 5), mask);
  if (!(old & mask)) newlist[atomicAdd(state + 2, 1)] = make_int2(col, c);
}

template <typename TB>
__global__ void __launch_bounds__(256) cam_update_kernel(const TB* __restrict__ bucket, int n, int d,
                                                         const int2* __restrict__ newlist,
                                                         int32_t* __restrict__ gain, const int32_t* __restrict__ state) {
  if (state[1]) return;
  const int nn = state[2];
  if (nn == 0) return;
  const int lane = threadIdx.x & 31;
  for (int row = blockIdx.x * 8 + (threadIdx.x >> 5); row < n; row += gridDim.x * 8) {
    if (gain[row] == 0) continue;            // warp-uniform: nothing left to lose
    const TB* b = bucket + (int64_t)row * d;
    int cnt = 0;
    for (int i = lane; i < nn; i += 32) {
      const int2 e = newlist[i];
      cnt += ((int)b[e.x] == e.y);
    }
    cnt = warp_sum(cnt);
    if (lane == 0 && cnt) gain[row] -= cnt;
  }
}

template <typename TB>
static int launch_cam(const void* bucket, int64_t n, int64_t d, int32_t k, int32_t* gain, uint32_t* covered,
                      int32_t* newlist, int32_t* order, int32_t* state, int32_t rounds, cudaStream_t st) {
  const int grid_u = (int)std::max<int64_t>(1, std::min<int64_t>((n + 7) / 8, (int64_t)sm_count() * 8));
  const int grid_c = (int)((d + 255) / 256);
  for (int r = 0; r < rounds; r++) {
    cam_pick_kernel<<<1, 1024, 0, st>>>(gain, (int)n, order, state);
    cam_collect_kernel<TB><<<grid_c, 256, 0, st>>>((const TB*)bucket, (int)d, k, covered, (int2*)newlist, state);
    cam_update_kernel<TB><<<grid_u, 256, 0, st>>>((const TB*)bucket, (int)n, (int)d, (const int2*)newlist, gain,
                                                  state);
  }
  tip::count_launch(3 * rounds);
  TIP_CHECK_CUDA(cudaGetLastError());
  return TIP_OK;
}

// ---- Surprise-coverage CAM (handler_surprise.py:101-115 over prioritizers.py:16-45) -------------------------
// SurpriseCoverageMapper's profile is profile[i, b] = t[b] <= v[i] < t[b+1].  For NaN-free, non-decreasing t the
// buckets are disjoint, so every row holds at most one True: a sample's gain is 1 while its bucket is uncovered
// and 0 after, np.argmax takes the lowest such index, and covering a bucket zeroes every other sample in it.  The
// greedy picks are therefore the first sample of every non-empty bucket, in ascending sample order.  One pass
// finds each bucket's first sample (sc_first_kernel); one block sorts those (sc_rank_kernel).
constexpr int kScThreads = 256;
constexpr uint32_t kScNone = 0xffffffffu;      // bucket without a sample; larger than every index

template <typename T>
__global__ void __launch_bounds__(kScThreads) sc_first_kernel(const T* __restrict__ v, int n,
                                                              const double* __restrict__ t, int sections,
                                                              uint32_t* __restrict__ first) {
  extern __shared__ double s_t[];                        // t[0..sections], then the block's first[0..sections)
  uint32_t* s_first = reinterpret_cast<uint32_t*>(s_t + sections + 1);
  for (int j = threadIdx.x; j <= sections; j += kScThreads) s_t[j] = t[j];
  for (int j = threadIdx.x; j < sections; j += kScThreads) s_first[j] = kScNone;
  __syncthreads();
  for (int i = blockIdx.x * kScThreads + threadIdx.x; i < n; i += gridDim.x * kScThreads) {
    const double x = (double)v[i];                       // float32 -> float64 is exact: NumPy's promotion
    int lo = 0, hi = sections + 1;                       // lo = number of thresholds <= x (NaN: 0)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (s_t[mid] <= x) lo = mid + 1; else hi = mid;
    }
    const int b = lo - 1;
    if (b >= 0 && b < sections && s_t[b] <= x && x < s_t[b + 1] && (uint32_t)i < s_first[b])
      atomicMin(s_first + b, (uint32_t)i);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < sections; j += kScThreads)
    if (s_first[j] != kScNone) atomicMin(first + j, s_first[j]);
}

// order[rank] = first[b] for every non-empty bucket, rank = number of smaller entries (the entries are distinct
// sample indices); count = number of non-empty buckets.
__global__ void __launch_bounds__(1024) sc_rank_kernel(const uint32_t* __restrict__ first, int sections,
                                                       int32_t* __restrict__ order, int32_t* __restrict__ count) {
  __shared__ uint32_t s_f[TIP_SC_CAM_MAX_SECTIONS];
  __shared__ int s_count;
  if (threadIdx.x == 0) s_count = 0;
  for (int j = threadIdx.x; j < sections; j += 1024) s_f[j] = first[j];
  __syncthreads();
  int mine = 0;
  for (int j = threadIdx.x; j < sections; j += 1024) {
    const uint32_t f = s_f[j];
    if (f == kScNone) continue;
    int rank = 0;
    for (int k = 0; k < sections; k++) rank += s_f[k] < f;
    order[rank] = (int32_t)f;
    mine++;
  }
  mine = warp_sum(mine);
  if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&s_count, mine);
  __syncthreads();
  if (threadIdx.x == 0) *count = s_count;
}

template <typename T>
static int launch_sc_first(const void* values, int64_t n, const double* t, int sections, uint32_t* first,
                           cudaStream_t st) {
  const size_t smem = (size_t)(sections + 1) * sizeof(double) + (size_t)sections * sizeof(uint32_t);
  if (smem > 48 * 1024)
    TIP_CHECK_CUDA(cudaFuncSetAttribute(sc_first_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n + 8 * kScThreads - 1) / (8 * kScThreads),
                                                                (int64_t)sm_count() * 4));
  sc_first_kernel<T><<<grid, kScThreads, smem, st>>>((const T*)values, (int)n, t, sections, first);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

}  // namespace tip

using namespace tip;

extern "C" int tip_cam_buckets(const void* bucket, int bucket_dtype, int64_t n, int64_t d, int32_t sections,
                               int32_t* gain, uint32_t* covered, int32_t* newlist, int32_t* order, int32_t* state,
                               int32_t rounds, void* stream) {
  TIP_REQUIRE(bucket && gain && covered && newlist && order && state, "null pointer");
  TIP_REQUIRE(bucket_dtype == TIP_I16 || bucket_dtype == TIP_I32, "bucket dtype");
  TIP_REQUIRE(n >= 1 && n < (1LL << 31) && d >= 1 && d < (1LL << 31) && sections >= 1 && rounds >= 0, "shape");
  if (rounds == 0) return TIP_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (bucket_dtype == TIP_I16)
    return launch_cam<int16_t>(bucket, n, d, sections, gain, covered, newlist, order, state, rounds, st);
  return launch_cam<int32_t>(bucket, n, d, sections, gain, covered, newlist, order, state, rounds, st);
}

extern "C" int tip_sc_cam(const void* values, int dtype, int64_t n, const double* thresholds, int32_t sections,
                          uint32_t* first, int32_t* order, int32_t* count, void* stream) {
  TIP_REQUIRE((values || n == 0) && thresholds && first && order && count, "null pointer");
  TIP_REQUIRE(n >= 0 && n < (1LL << 31), "shape");
  TIP_REQUIRE(sections >= 1 && sections <= TIP_SC_CAM_MAX_SECTIONS, "sections must be in [1, TIP_SC_CAM_MAX_SECTIONS]");
  TIP_REQUIRE(dtype == TIP_F32 || dtype == TIP_F64, "dtype must be TIP_F32 or TIP_F64");
  cudaStream_t st = (cudaStream_t)stream;
  TIP_CHECK_CUDA(cudaMemsetAsync(first, 0xff, (size_t)sections * sizeof(uint32_t), st));
  if (n > 0) {
    const int rc = dtype == TIP_F32 ? launch_sc_first<float>(values, n, thresholds, sections, first, st)
                                    : launch_sc_first<double>(values, n, thresholds, sections, first, st);
    if (rc != TIP_OK) return rc;
  }
  sc_rank_kernel<<<1, 1024, 0, st>>>(first, sections, order, count);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}
