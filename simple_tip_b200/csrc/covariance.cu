// covariance.cu — the N-sized pass of sklearn's EmpiricalCovariance.fit that the Gaussian-mixture kernels do not
// already cover: the column means.  (The scatter is tip_gmm_scatter with one component and unit weights.)
//
// sklearn's `location_ = X.mean(0)` is NumPy's add.reduce over axis 0 in the input dtype, then one division by n.
// On a C-contiguous [n, d] matrix with d >= 2 that reduce is a sequential sum over the rows, starting from 0; with
// d == 1 the reduced axis is the contiguous one and NumPy sums it pairwise (numpy/_core/src/umath/loops_utils.h:
// blocks of <= 128 with eight stride-8 accumulators, larger blocks split at n/2 - (n/2)%8).  `np.cov(X.T)` centres
// on its own float64 mean, which follows the same two rules in float64.  Both are reproduced here bit for bit:
//
//   cov_location_kernel     d >= 2: one thread per column walks the rows in order (8 loads in flight), one
//                           input-dtype chain and one float64 chain, IEEE adds without contraction
//   cov_location_1d_kernel  d == 1: one thread, NumPy's pairwise sum in both dtypes
//
// The division is done in double and rounded once to the input dtype, which is the correctly rounded quotient for
// float32 as well (NumPy divides float32 by an intp in double and casts back).  Non-finite inputs set flags bits
// (1: NaN, 2: +-inf) so that the fit can raise sklearn's error instead of returning NaN.
//
// tip_col_var (LSA's column selection, np.var(x, axis=0)) runs the same kernels with a second pass over the rows:
// NumPy 2.3's _methods._var subtracts the input-dtype mean above (arr - arrmean, in x's dtype), squares with
// multiply(x, x) as a rounding of its own (no FMA), reduces that with the same add.reduce (sequential for d >= 2,
// pairwise for d == 1) and divides by the intp count the same way.
#include "common.cuh"

namespace tip {

constexpr int kCovThreads = 32;      // one warp per CTA: d = 1600 gives 50 CTAs, latency-bound chains spread out
constexpr int kCovUnroll = 8;

__device__ __forceinline__ int cov_flag(double v) {
  return isnan(v) ? 1 : (isinf(v) ? 2 : 0);
}

template <typename T>
__device__ __forceinline__ T cov_div(T s, int64_t n) {
  return (T)__ddiv_rn((double)s, (double)n);
}

template <typename T>
__global__ void __launch_bounds__(kCovThreads) cov_location_kernel(const T* __restrict__ x, int64_t n, int64_t d,
                                                                   T* __restrict__ loc, double* __restrict__ mean,
                                                                   T* __restrict__ var, int32_t* __restrict__ flags) {
  using R = Rn<T>;
  const int64_t c = (int64_t)blockIdx.x * kCovThreads + threadIdx.x;
  if (c >= d) return;
  T s = (T)0;
  double s64 = 0.0;
  int flag = 0;
  int64_t r = 0;
  for (; r + kCovUnroll <= n; r += kCovUnroll) {
    T v[kCovUnroll];
#pragma unroll
    for (int u = 0; u < kCovUnroll; u++) v[u] = x[(r + u) * d + c];
#pragma unroll
    for (int u = 0; u < kCovUnroll; u++) {
      s = R::add(s, v[u]);
      s64 = __dadd_rn(s64, (double)v[u]);
      flag |= cov_flag((double)v[u]);
    }
  }
  for (; r < n; r++) {
    const T v = x[r * d + c];
    s = R::add(s, v);
    s64 = __dadd_rn(s64, (double)v);
    flag |= cov_flag((double)v);
  }
  const T m = cov_div<T>(s, n);
  if (loc) loc[c] = m;
  mean[c] = __ddiv_rn(s64, (double)n);
  if (flag) atomicOr(flags, flag);      // an integer flag: the result does not depend on the order
  if (!var) return;
  // np.var's second pass: arr - arrmean, then multiply(x, x) as its own rounding, summed in row order
  T s2 = (T)0;
  for (r = 0; r + kCovUnroll <= n; r += kCovUnroll) {
    T v[kCovUnroll];
#pragma unroll
    for (int u = 0; u < kCovUnroll; u++) v[u] = x[(r + u) * d + c];
#pragma unroll
    for (int u = 0; u < kCovUnroll; u++) {
      const T e = R::sub(v[u], m);
      s2 = R::add(s2, R::mul(e, e));
    }
  }
  for (; r < n; r++) {
    const T e = R::sub(x[r * d + c], m);
    s2 = R::add(s2, R::mul(e, e));
  }
  var[c] = cov_div<T>(s2, n);
}

template <typename T>
__global__ void cov_location_1d_kernel(const T* __restrict__ x, int64_t n, T* __restrict__ loc,
                                       double* __restrict__ mean, T* __restrict__ var, int32_t* __restrict__ flags) {
  int flag = 0;
  for (int64_t i = 0; i < n; i++) flag |= cov_flag((double)x[i]);
  // the reduce adds the pairwise sum to the identity 0 (this also turns a -0 sum into +0, as NumPy does)
  const T m = cov_div<T>(Rn<T>::add((T)0, np_sum<T>([&](int i) { return x[i]; }, (int)n)), n);
  if (loc) loc[0] = m;
  mean[0] = __ddiv_rn(__dadd_rn(0.0, np_sum<double>([&](int i) { return (double)x[i]; }, (int)n)), (double)n);
  *flags = flag;
  if (var) {
    const auto sq = [&](int i) {
      const T e = Rn<T>::sub(x[i], m);
      return Rn<T>::mul(e, e);
    };
    var[0] = cov_div<T>(Rn<T>::add((T)0, np_sum<T>(sq, (int)n)), n);
  }
}

static int cov_moments(const void* x, int dtype, int64_t n, int64_t d, void* location, double* mean, void* var,
                       int32_t* flags, void* stream) {
  TIP_REQUIRE(dtype == TIP_F32 || dtype == TIP_F64, "dtype must be TIP_F32 or TIP_F64");
  TIP_REQUIRE(n >= 1 && n < (1LL << 31) && d >= 1 && d <= 65536, "shape");
  TIP_REQUIRE(x && mean && flags, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (d == 1) {
    if (dtype == TIP_F32)
      cov_location_1d_kernel<float><<<1, 1, 0, st>>>((const float*)x, n, (float*)location, mean, (float*)var, flags);
    else
      cov_location_1d_kernel<double><<<1, 1, 0, st>>>((const double*)x, n, (double*)location, mean, (double*)var,
                                                      flags);
    TIP_LAUNCH_CHECK();
    return TIP_OK;
  }
  TIP_CHECK_CUDA(cudaMemsetAsync(flags, 0, sizeof(int32_t), st));
  const unsigned grid = (unsigned)((d + kCovThreads - 1) / kCovThreads);
  if (dtype == TIP_F32)
    cov_location_kernel<float><<<grid, kCovThreads, 0, st>>>((const float*)x, n, d, (float*)location, mean,
                                                             (float*)var, flags);
  else
    cov_location_kernel<double><<<grid, kCovThreads, 0, st>>>((const double*)x, n, d, (double*)location, mean,
                                                              (double*)var, flags);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

}  // namespace tip

using namespace tip;

extern "C" int tip_cov_location(const void* x, int dtype, int64_t n, int64_t d, void* location, double* mean,
                                int32_t* flags, void* stream) {
  TIP_REQUIRE(location, "null pointer");
  return cov_moments(x, dtype, n, d, location, mean, nullptr, flags, stream);
}

extern "C" int tip_col_var(const void* x, int dtype, int64_t n, int64_t d, void* var, double* mean, int32_t* flags,
                           void* stream) {
  TIP_REQUIRE(var, "null pointer");
  return cov_moments(x, dtype, n, d, nullptr, mean, var, flags, stream);
}
