// train.cu — the kernels of one training step of the case studies' models (case_study_*.py `model.fit`): Keras'
// Adam update over every parameter of a model in one launch, the fused softmax cross-entropy head (per segment of
// rows, one segment per model of a stack), and the gather of a step's batch for every model of a stack.
// Convolutions, GEMMs, pooling, normalisation and attention stay with cuDNN / cuBLAS through torch.
//
// tip_keras_adam: one flat index space over all tensors of the table.  A tensor whose param, grad, m and v share
// their address modulo 16 is walked as a scalar head up to the 16-byte boundary, float4 units, and a scalar tail;
// any other tensor element by element.  Every block derives that layout from the table itself (<= 256 tensors, one
// per thread, prefix-summed in shared memory), so the grid size never changes the result and each element is
// written by exactly one thread.  The step counter lives in device memory: every block reads t at its start, and
// the last block to finish (an arrival counter next to t) stores t + 1 and clears the counter, so a captured graph
// can be replayed step after step.
//
// tip_softmax_xent / tip_softmax_xent_seg: one block of 32 warps per segment of rows (a single segment for
// tip_softmax_xent), warp w takes the segment's rows w, w + 32, ...; per row the max, the sums and the argmaxes are
// fixed xor-shuffle trees, the per-row losses are summed in double in row order per warp and the 32 warp sums in a
// fixed tree, so a segment's result depends on nothing but its own rows.
//
// tip_stack_gather: one thread per output element of a stacked batch; row j of model m is pool row
// rows[m][perm[m][start + j]], written model-major [M, b, R] or channel-interleaved [b, P, M, C] (R = P * C).
#include "common.cuh"

namespace tip {

constexpr int kAdamThreads = 256;
constexpr int kAdamMaxTensors = kAdamThreads;
constexpr int kXentWarps = 32;

struct AdamLayout {
  int64_t head, vecs, units;     // scalar head, float4 units, all units of the tensor
};

__device__ __forceinline__ AdamLayout adam_layout(const tip_adam_tensor& t) {
  AdamLayout l;
  const uintptr_t a = reinterpret_cast<uintptr_t>(t.param) & 15;
  const bool same = ((reinterpret_cast<uintptr_t>(t.grad) & 15) == a) && ((reinterpret_cast<uintptr_t>(t.m) & 15) == a) &&
                    ((reinterpret_cast<uintptr_t>(t.v) & 15) == a);
  if (!same) {
    l.head = t.numel;
    l.vecs = 0;
  } else {
    l.head = min((int64_t)(((16 - a) & 15) >> 2), t.numel);
    l.vecs = (t.numel - l.head) >> 2;
  }
  l.units = l.head + l.vecs + (t.numel - l.head - 4 * l.vecs);
  return l;
}

struct AdamCoef {
  float b1, b2, one_m_b1, one_m_b2, lr_t, eps;
};

// m <- b1 m + (1 - b1) g;  v <- b2 v + (1 - b2) g^2;  p <- p - (lr_t m) / (sqrt(v) + eps), each operation rounded once
__device__ __forceinline__ void adam_elem(float& p, float g, float& m, float& v, const AdamCoef& c) {
  m = __fadd_rn(__fmul_rn(c.b1, m), __fmul_rn(c.one_m_b1, g));
  v = __fadd_rn(__fmul_rn(c.b2, v), __fmul_rn(c.one_m_b2, __fmul_rn(g, g)));
  p = __fsub_rn(p, __fdiv_rn(__fmul_rn(c.lr_t, m), __fadd_rn(__fsqrt_rn(v), c.eps)));
}

__global__ void __launch_bounds__(kAdamThreads) keras_adam_kernel(const tip_adam_tensor* __restrict__ table, int n,
                                                                  int32_t* __restrict__ state, float lr, float beta1,
                                                                  float beta2, float epsilon) {
  __shared__ tip_adam_tensor tens[kAdamMaxTensors];
  __shared__ int64_t head[kAdamMaxTensors], vecs[kAdamMaxTensors], off[kAdamMaxTensors + 1];
  __shared__ AdamCoef coef;
  const int tid = threadIdx.x;
  int64_t units = 0;
  if (tid < n) {
    tens[tid] = table[tid];
    const AdamLayout l = adam_layout(tens[tid]);
    head[tid] = l.head;
    vecs[tid] = l.vecs;
    units = l.units;
  }
  off[tid + 1] = units;
  if (tid == 0) {
    off[0] = 0;
    // step t = state[0] + 1; beta^t in float64, rounded once to float32
    const int t = state[0] + 1;
    const float b1p = (float)pow((double)beta1, (double)t), b2p = (float)pow((double)beta2, (double)t);
    coef.b1 = beta1;
    coef.b2 = beta2;
    coef.one_m_b1 = __fsub_rn(1.f, beta1);
    coef.one_m_b2 = __fsub_rn(1.f, beta2);
    coef.lr_t = __fmul_rn(lr, __fdiv_rn(__fsqrt_rn(__fsub_rn(1.f, b2p)), __fsub_rn(1.f, b1p)));
    coef.eps = epsilon;
  }
  __syncthreads();
  for (int s = 1; s < kAdamThreads; s <<= 1) {       // inclusive scan of off[1..256]
    const int64_t add = tid >= s ? off[tid + 1 - s] : 0;
    __syncthreads();
    off[tid + 1] += add;
    __syncthreads();
  }
  const int64_t total = off[n];
  const AdamCoef c = coef;
  for (int64_t u = (int64_t)blockIdx.x * kAdamThreads + tid; u < total; u += (int64_t)gridDim.x * kAdamThreads) {
    int lo = 0, hi = n - 1;                            // the tensor k with off[k] <= u < off[k + 1]
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (off[mid] <= u) lo = mid;
      else hi = mid - 1;
    }
    const tip_adam_tensor& t = tens[lo];
    const int64_t r = u - off[lo], h = head[lo], nv = vecs[lo];
    if (r >= h && r < h + nv) {
      const int64_t e = h + 4 * (r - h);
      float4 p = *reinterpret_cast<const float4*>(t.param + e);
      const float4 g = __ldg(reinterpret_cast<const float4*>(t.grad + e));
      float4 m = *reinterpret_cast<const float4*>(t.m + e);
      float4 v = *reinterpret_cast<const float4*>(t.v + e);
      adam_elem(p.x, g.x, m.x, v.x, c);
      adam_elem(p.y, g.y, m.y, v.y, c);
      adam_elem(p.z, g.z, m.z, v.z, c);
      adam_elem(p.w, g.w, m.w, v.w, c);
      *reinterpret_cast<float4*>(t.param + e) = p;
      *reinterpret_cast<float4*>(t.m + e) = m;
      *reinterpret_cast<float4*>(t.v + e) = v;
    } else {
      const int64_t e = r < h ? r : r + 3 * nv;
      float p = t.param[e], m = t.m[e], v = t.v[e];
      adam_elem(p, __ldg(t.grad + e), m, v, c);
      t.param[e] = p;
      t.m[e] = m;
      t.v[e] = v;
    }
  }
  // the last block to arrive advances the step counter: every block has read it by then
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    if (atomicAdd(&state[1], 1) == (int)gridDim.x - 1) {
      state[0] += 1;
      state[1] = 0;
      __threadfence();
    }
  }
}

__device__ __forceinline__ float warp_max(float v) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum_f(float v) {
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// first index of the maximum (NaN-free input): the smallest lane holding the warp's max
__device__ __forceinline__ int warp_first_argmax(float v, bool live) {
  const float mx = warp_max(live ? v : -__int_as_float(0x7f800000));
  const unsigned hit = __ballot_sync(0xffffffffu, live && v == mx);
  return hit ? __ffs(hit) - 1 : 0;
}

// block s: the segment of rows [s * rows, (s + 1) * rows), its loss into loss[s] and its count into correct[s]
__global__ void __launch_bounds__(kXentWarps * 32) softmax_xent_kernel(const float* __restrict__ z,
                                                                       const float* __restrict__ y, int64_t rows,
                                                                       int classes, float* __restrict__ loss,
                                                                       float* __restrict__ dz,
                                                                       int32_t* __restrict__ correct) {
  const int64_t seg = blockIdx.x, first = seg * rows * classes;
  z += first;
  y += first;
  if (dz) dz += first;
  __shared__ double part[kXentWarps];
  __shared__ int hits[kXentWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool live = lane < classes;
  const float b = (float)rows;
  double acc = 0.0;
  int n_hit = 0;
  for (int64_t r = warp; r < rows; r += kXentWarps) {
    const float zc = live ? z[r * classes + lane] : 0.f, yc = live ? y[r * classes + lane] : 0.f;
    const float mx = warp_max(live ? zc : -__int_as_float(0x7f800000));
    const float e = live ? expf(__fsub_rn(zc, mx)) : 0.f;
    const float s = warp_sum_f(e);
    // lanes with y != 0 also need the sum of the others' terms, o = s - e without the cancellation:
    // p - 1 = -o / s, and -log p = log1p(o) where z is the max (e = 1)
    float o = 0.f;
    unsigned todo = __ballot_sync(0xffffffffu, live && yc != 0.f);
    while (todo) {
      const int k = __ffs(todo) - 1;
      todo &= todo - 1;
      const float ok = warp_sum_f(lane == k ? 0.f : e);
      if (lane == k) o = ok;
    }
    float row_loss = 0.f;
    if (live && yc != 0.f) {
      const float nlp = zc == mx ? log1pf(o) : __fadd_rn(__fsub_rn(mx, zc), logf(s));
      row_loss = __fmul_rn(yc, nlp);
    }
    row_loss = warp_sum_f(row_loss);
    acc += (double)row_loss;
    if (dz && live) {
      const float g = yc == 1.f ? -__fdiv_rn(o, s) : __fsub_rn(__fdiv_rn(e, s), yc);
      dz[r * classes + lane] = __fdiv_rn(g, b);
    }
    const int az = warp_first_argmax(zc, live), ay = warp_first_argmax(yc, live);
    n_hit += az == ay;
  }
  if (lane == 0) {
    part[warp] = acc;
    hits[warp] = n_hit;
  }
  __syncthreads();
  if (warp == 0) {
    double a = part[lane];
    int h = hits[lane];
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o);
      h += __shfl_xor_sync(0xffffffffu, h, o);
    }
    if (lane == 0) {
      loss[seg] = (float)(a / (double)rows);
      correct[seg] = h;
    }
  }
}


// out[m][j][r] (model-major) or out[j][p][m][c] (channel-interleaved, r = p * C + c) = pool[rows[m][perm[m][start + j]]][r]
template <typename Src, typename Dst>
__global__ void __launch_bounds__(256) stack_gather_kernel(const Src* __restrict__ pool, int64_t row_elems,
                                                           const int64_t* __restrict__ rows, int64_t n_rows,
                                                           const int64_t* __restrict__ perm, int64_t n_perm,
                                                           int64_t start, int64_t b, int64_t models,
                                                           int64_t channels, bool interleaved,
                                                           Dst* __restrict__ out) {
  const int64_t total = models * b * row_elems;
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += (int64_t)gridDim.x * blockDim.x) {
    int64_t m, j, r;
    if (interleaved) {
      const int64_t c = o % channels, q = o / channels;
      m = q % models;
      const int64_t jp = q / models, pixels = row_elems / channels;
      j = jp / pixels;
      r = (jp % pixels) * channels + c;
    } else {
      r = o % row_elems;
      const int64_t q = o / row_elems;
      j = q % b;
      m = q / b;
    }
    const int64_t row = rows[m * n_rows + perm[m * n_perm + start + j]];
    out[o] = (Dst)pool[row * row_elems + r];
  }
}

}  // namespace tip

extern "C" int tip_keras_adam(const tip_adam_tensor* table, int32_t n_tensors, int64_t total_numel, int32_t* state,
                              float lr, float beta1, float beta2, float epsilon, void* stream) {
  using namespace tip;
  TIP_REQUIRE(n_tensors >= 1 && n_tensors <= kAdamMaxTensors, "1..256 tensors per table");
  TIP_REQUIRE(total_numel >= 0, "negative element count");
  TIP_REQUIRE(table && state, "null pointer");
  const int64_t blocks_needed = (total_numel / 4 + 4 * n_tensors + kAdamThreads - 1) / kAdamThreads;
  const int grid = (int)max((int64_t)1, min(blocks_needed, (int64_t)sm_count() * 8));
  keras_adam_kernel<<<grid, kAdamThreads, 0, (cudaStream_t)stream>>>(table, n_tensors, state, lr, beta1, beta2,
                                                                      epsilon);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_softmax_xent_seg(const float* z, const float* y, int64_t segments, int64_t rows_per_segment,
                                    int32_t classes, float* loss, float* dz, int32_t* correct, void* stream) {
  using namespace tip;
  TIP_REQUIRE(segments >= 1 && segments <= INT32_MAX, "1..2^31-1 segments");
  TIP_REQUIRE(rows_per_segment >= 1, "at least one row per segment");
  TIP_REQUIRE(classes >= 1 && classes <= 32, "1..32 classes");
  TIP_REQUIRE(z && y && loss && correct, "null pointer");
  softmax_xent_kernel<<<(unsigned)segments, kXentWarps * 32, 0, (cudaStream_t)stream>>>(z, y, rows_per_segment, classes,
                                                                                      loss, dz, correct);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_softmax_xent(const float* z, const float* y, int64_t rows, int32_t classes, float* loss, float* dz,
                                int32_t* correct, void* stream) {
  return tip_softmax_xent_seg(z, y, 1, rows, classes, loss, dz, correct, stream);
}

extern "C" int tip_stack_gather(const void* pool, int32_t dtype, int64_t row_elems,
                                const int64_t* rows, int64_t n_rows, const int64_t* perm, int64_t n_perm,
                                int64_t start, int64_t b, int64_t models, int64_t channels, void* out, void* stream) {
  using namespace tip;
  TIP_REQUIRE(dtype == TIP_F32 || dtype == TIP_F64 || dtype == TIP_I32, "float32, float64 or int32 pool");
  TIP_REQUIRE(row_elems >= 1 && models >= 1 && b >= 1, "empty rows or batch");
  TIP_REQUIRE(n_perm >= 1 && n_perm <= n_rows, "perm indexes the first n_perm of each model's n_rows rows");
  TIP_REQUIRE(start >= 0 && start + b <= n_perm, "batch [start, start + b) within the permutation");
  TIP_REQUIRE(channels >= 0 && (channels == 0 || row_elems % channels == 0), "row_elems is pixels x channels");
  TIP_REQUIRE(pool && rows && perm && out, "null pointer");
  const bool interleaved = channels > 0;
  const int64_t total = models * b * row_elems;
  const int grid = (int)max((int64_t)1, min((total + 255) / 256, (int64_t)sm_count() * 16));
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == TIP_F32)
    stack_gather_kernel<float, float><<<grid, 256, 0, s>>>((const float*)pool, row_elems, rows, n_rows, perm, n_perm,
                                                            start, b, models, channels, interleaved, (float*)out);
  else if (dtype == TIP_F64)
    stack_gather_kernel<double, float><<<grid, 256, 0, s>>>((const double*)pool, row_elems, rows, n_rows, perm, n_perm,
                                                             start, b, models, channels, interleaved, (float*)out);
  else
    stack_gather_kernel<int32_t, int32_t><<<grid, 256, 0, s>>>((const int32_t*)pool, row_elems, rows, n_rows, perm,
                                                                n_perm, start, b, models, channels, interleaved,
                                                                (int32_t*)out);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}
