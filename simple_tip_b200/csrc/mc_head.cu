// mc_head.cu — MC-dropout samples of a model's dropout head (handler_model.py get_pred_and_uncertainty) from the
// trunk activations the point pass already produced: the dropout masks, the dense layers and the last layer's
// softmax of every (row, sample) pair, in one launch.  The masked [rows * samples, in] operand never exists: each
// thread draws its masks in registers while it walks the input units.  The arithmetic is include/b200tip.h's.
//
// One thread owns SPT (row, sample) pairs and their layer-0 accumulators [SPT][WP] (WP = layer 0's width padded to
// a multiple of 4); a block owns kMcThreads * SPT consecutive pairs of the flattened (row, sample) space, so a
// block's pairs span at most kMcTileRows rows.  Layer 0 is walked in stages of kMcChunk input units: the stage's
// kernel rows [kMcChunk][WP] and h columns [rows][kMcChunk] go to shared memory, zero-padded to an even unit count
// (a padded term adds +0 to an accumulator that is never -0, so it changes no bits), and every thread then walks the
// stage two units at a time — one splitmix64 step per pair of units and sample — reading the kernel rows as
// broadcast float4s.  All products and sums are __fmul_rn / __fadd_rn on the FP32 pipe, in ascending unit order.
//
// Heads with more than one layer (TW > 0: SPT = 1, WP = TW) keep layer 0's activations in registers x[TW] and run
// the later layers (widths <= TW <= 64) from shared memory, fully unrolled, with the same masks and order.
//
// tip_mc_head_stack runs M heads of one shape (a StackedSequential's) in one launch: blockIdx.y picks the model, whose
// h, kernels, biases, output and seed the block uses; the pair space, the tiling and the key are tip_mc_head's, so
// model m's slice is bit for bit tip_mc_head's launch on model m.  tip_mc_head is the body with model 0.
#include <math.h>

#include <type_traits>

#include "common.cuh"

namespace tip {

constexpr int kMcThreads = 256;
constexpr int kMcMaxLayers = 4;
constexpr int kMcMaxWidth = 64;
constexpr int kMcMaxIn = 8192;
constexpr int kMcChunk = 32;        // layer-0 input units per shared-memory stage
constexpr int kMcTileRows = 64;     // h rows a block's pairs may span
constexpr int kMcHStride = kMcChunk + 1;

struct McLayer {
  const float* kernel;
  const float* bias;
  uint64_t thresh;      // dropped iff u < thresh
  float scale;
  int in, out, act;
  int woff;             // later layers: offset of [in rounded up to even][TW] weights + [TW] bias in shared memory
};

struct McArgs {
  const float* h;
  int64_t rows, ld, row0, sample0, samples, pairs_per_block;
  uint64_t seed;
  float* out;
  int n_layers, mode;
  McLayer L[kMcMaxLayers];
};

constexpr int kMcStackChunk = 256;  // models per tip_mc_head_stack launch: their seeds ride in the kernel parameters

struct McStackArgs : McArgs {      // kernels [M][in][out], biases [M][out], out [M][rows][samples][C]
  int64_t ldm;                      // h: model m's row i at h + m * ldm + i * ld
  int64_t model0;                   // the launch's first model
  uint64_t seeds[kMcStackChunk];    // seeds[blockIdx.y] = model model0 + blockIdx.y's
};

__device__ __forceinline__ uint64_t mc_key(uint64_t seed, int layer, int64_t row, int64_t sample) {
  uint64_t h = km_mix(seed);
  h = km_mix(h ^ (uint64_t)layer);
  h = km_mix(h ^ (uint64_t)row);
  return km_mix(h ^ (uint64_t)sample);
}

__device__ __forceinline__ float mc_keep(float x, uint32_t u, uint64_t thresh, float scale) {
  return (uint64_t)u < thresh ? 0.f : __fmul_rn(x, scale);
}

__device__ __forceinline__ float mc_act(float z, int act) { return act == TIP_MC_RELU ? (z < 0.f ? 0.f : z) : z; }

// writes the last layer's C values of one pair from its pre-activations z (bias added; overwritten)
template <int N>
__device__ __forceinline__ void mc_store(float (&z)[N], int C, int act, int mode, float* __restrict__ dst) {
  if (mode == TIP_MC_PREACT || act != TIP_MC_SOFTMAX) {
#pragma unroll
    for (int c = 0; c < N; c++)
      if (c < C) dst[c] = mode == TIP_MC_PREACT ? z[c] : mc_act(z[c], act);
    return;
  }
  float m = z[0];
#pragma unroll
  for (int c = 1; c < N; c++)
    if (c < C) m = fmaxf(m, z[c]);
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < N; c++)
    if (c < C) {
      z[c] = expf(__fsub_rn(z[c], m));
      s = __fadd_rn(s, z[c]);
    }
#pragma unroll
  for (int c = 0; c < N; c++)
    if (c < C) dst[c] = __fdiv_rn(z[c], s);
}

// p + off for a stack's model; tip_mc_head's kernel (STACK = false) addresses a's pointers as they are
template <bool STACK, class T>
__device__ __forceinline__ T* mc_at(T* p, int64_t off) {
  if constexpr (STACK) return p + off;
  else return p;
}

// STACK = false: tip_mc_head's kernel on McArgs.  STACK = true: tip_mc_head_stack's on McStackArgs, block
// (blockIdx.x, blockIdx.y) = tip_mc_head's block blockIdx.x on model model0 + blockIdx.y.
template <int WP, int SPT, int TW, bool STACK = false>
__global__ void __launch_bounds__(kMcThreads, 1)
    mc_head_kernel(const __grid_constant__ std::conditional_t<STACK, McStackArgs, McArgs> p) {
  const McArgs& a = p;
  int64_t m = 0, ldm = 0;
  const uint64_t* seedp = &a.seed;
  if constexpr (STACK) {
    m = p.model0 + blockIdx.y;
    ldm = p.ldm;
    seedp = &p.seeds[blockIdx.y];
  }
  const uint64_t& seed = *seedp;
  extern __shared__ __align__(16) float smem[];
  float* sK = smem;                                  // [kMcChunk][WP]
  float* sH = sK + kMcChunk * WP;                    // [kMcTileRows][kMcHStride]
  float* sT = sH + kMcTileRows * kMcHStride;         // later layers (TW > 0)
  const int tid = threadIdx.x;
  const int64_t S = a.samples, total = a.rows * S;
  const int64_t q0 = (int64_t)blockIdx.x * a.pairs_per_block;
  const int64_t q1 = min(q0 + a.pairs_per_block, total);
  const int64_t r_lo = q0 / S;
  const int n_rows = (int)((q1 - 1) / S - r_lo + 1);
  const McLayer& L0 = a.L[0];

  if constexpr (TW > 0) {
    for (int l = 1; l < a.n_layers; l++) {
      const McLayer& L = a.L[l];
      const int in2 = (L.in + 1) & ~1;
      float* w = sT + L.woff;
      for (int i = tid; i < (in2 + 1) * TW; i += kMcThreads) {
        const int j = i / TW, c = i - j * TW;
        float v = 0.f;
        if (c < L.out)
          v = j < L.in ? mc_at<STACK>(L.kernel, m * L.in * L.out)[(int64_t)j * L.out + c]
                       : (j == in2 ? mc_at<STACK>(L.bias, m * L.out)[c] : 0.f);
        w[i] = v;
      }
    }
  }

  int rl[SPT];
  uint64_t key[SPT];
#pragma unroll
  for (int k = 0; k < SPT; k++) {
    const int64_t q = min(q0 + tid + (int64_t)k * kMcThreads, q1 - 1);
    const int64_t r = q / S;
    rl[k] = (int)(r - r_lo) * kMcHStride;
    key[k] = mc_key(seed, 0, a.row0 + r, a.sample0 + (q - r * S));
  }
  float acc[SPT][WP];
#pragma unroll
  for (int k = 0; k < SPT; k++)
#pragma unroll
    for (int c = 0; c < WP; c++) acc[k][c] = 0.f;

  const int D = L0.in, W0 = L0.out;
  const uint64_t t0 = L0.thresh;
  const float scale0 = L0.scale;
  for (int d0 = 0; d0 < D; d0 += kMcChunk) {
    const int dn = min(kMcChunk, D - d0);
    __syncthreads();
    for (int i = tid; i < kMcChunk * WP; i += kMcThreads) {
      const int j = i / WP, c = i - j * WP;
      sK[i] = (j < dn && c < W0) ? __ldg(mc_at<STACK>(L0.kernel, m * D * W0) + (int64_t)(d0 + j) * W0 + c) : 0.f;
    }
    for (int i = tid; i < n_rows * kMcChunk; i += kMcThreads) {
      const int r = i / kMcChunk, j = i - r * kMcChunk;
      sH[r * kMcHStride + j] = j < dn ? __ldg(mc_at<STACK>(a.h, m * ldm) + (r_lo + r) * a.ld + d0 + j) : 0.f;
    }
    __syncthreads();
    const int dn2 = (dn + 1) & ~1;
#pragma unroll 1
    for (int j = 0; j < dn2; j += 2) {
      float v0[SPT], v1[SPT];
#pragma unroll
      for (int k = 0; k < SPT; k++) {
        const float x0 = sH[rl[k] + j], x1 = sH[rl[k] + j + 1];
        const uint64_t w = t0 ? km_mix(key[k] ^ (uint64_t)((d0 + j) >> 1)) : ~0ull;
        v0[k] = mc_keep(x0, (uint32_t)w, t0, scale0);
        v1[k] = mc_keep(x1, (uint32_t)(w >> 32), t0, scale0);
      }
#pragma unroll
      for (int c = 0; c < WP; c += 4) {
        const float4 k0 = *reinterpret_cast<const float4*>(sK + j * WP + c);
        const float4 k1 = *reinterpret_cast<const float4*>(sK + (j + 1) * WP + c);
#pragma unroll
        for (int k = 0; k < SPT; k++) {
          acc[k][c + 0] = __fadd_rn(__fadd_rn(acc[k][c + 0], __fmul_rn(v0[k], k0.x)), __fmul_rn(v1[k], k1.x));
          acc[k][c + 1] = __fadd_rn(__fadd_rn(acc[k][c + 1], __fmul_rn(v0[k], k0.y)), __fmul_rn(v1[k], k1.y));
          acc[k][c + 2] = __fadd_rn(__fadd_rn(acc[k][c + 2], __fmul_rn(v0[k], k0.z)), __fmul_rn(v1[k], k1.z));
          acc[k][c + 3] = __fadd_rn(__fadd_rn(acc[k][c + 3], __fmul_rn(v0[k], k0.w)), __fmul_rn(v1[k], k1.w));
        }
      }
    }
  }

#pragma unroll
  for (int k = 0; k < SPT; k++) {
    const int64_t q = q0 + tid + (int64_t)k * kMcThreads;
    if (q >= q1) break;
    float z[WP];
#pragma unroll
    for (int c = 0; c < WP; c++) z[c] = c < W0 ? __fadd_rn(acc[k][c], __ldg(mc_at<STACK>(L0.bias, m * W0) + c)) : 0.f;
    if constexpr (TW == 0) {
      mc_store(z, W0, L0.act, a.mode, mc_at<STACK>(a.out, m * total * W0) + q * W0);
    } else {
      const int64_t r = q / S, s = q - r * S;
      float x[TW];
#pragma unroll
      for (int c = 0; c < TW; c++) x[c] = c < W0 ? mc_act(z[c], L0.act) : 0.f;
      for (int l = 1; l < a.n_layers; l++) {
        const McLayer& L = a.L[l];
        const float* w = sT + L.woff;
        const uint64_t kl = mc_key(seed, l, a.row0 + r, a.sample0 + s);
        float y[TW];
#pragma unroll
        for (int c = 0; c < TW; c++) y[c] = 0.f;
#pragma unroll
        for (int j = 0; j < TW; j += 2) {
          if (j < L.in) {
            const uint64_t u = L.thresh ? km_mix(kl ^ (uint64_t)(j >> 1)) : ~0ull;
            const float x0 = mc_keep(x[j], (uint32_t)u, L.thresh, L.scale);
            const float x1 = mc_keep(x[j + 1], (uint32_t)(u >> 32), L.thresh, L.scale);
#pragma unroll
            for (int c = 0; c < TW; c += 4) {
              const float4 k0 = *reinterpret_cast<const float4*>(w + j * TW + c);
              const float4 k1 = *reinterpret_cast<const float4*>(w + (j + 1) * TW + c);
              y[c + 0] = __fadd_rn(__fadd_rn(y[c + 0], __fmul_rn(x0, k0.x)), __fmul_rn(x1, k1.x));
              y[c + 1] = __fadd_rn(__fadd_rn(y[c + 1], __fmul_rn(x0, k0.y)), __fmul_rn(x1, k1.y));
              y[c + 2] = __fadd_rn(__fadd_rn(y[c + 2], __fmul_rn(x0, k0.z)), __fmul_rn(x1, k1.z));
              y[c + 3] = __fadd_rn(__fadd_rn(y[c + 3], __fmul_rn(x0, k0.w)), __fmul_rn(x1, k1.w));
            }
          }
        }
        const float* bias = w + ((L.in + 1) & ~1) * TW;
#pragma unroll
        for (int c = 0; c < TW; c++) y[c] = c < L.out ? __fadd_rn(y[c], bias[c]) : 0.f;
        if (l + 1 == a.n_layers) {
          mc_store(y, L.out, L.act, a.mode, mc_at<STACK>(a.out, m * total * L.out) + q * L.out);
        } else {
#pragma unroll
          for (int c = 0; c < TW; c++) x[c] = c < L.out ? mc_act(y[c], L.act) : 0.f;
        }
      }
    }
  }
}

// models == 0: tip_mc_head's launch of a; else models heads in launches of kMcStackChunk models, s's McArgs = a
template <int WP, int SPT, int TW>
int mc_launch(McArgs& a, McStackArgs* s, int64_t models, const uint64_t* seeds, cudaStream_t stream) {
  a.pairs_per_block = min((int64_t)kMcThreads * SPT, (int64_t)(kMcTileRows - 1) * a.samples);
  const int64_t total = a.rows * a.samples;
  const int64_t grid = (total + a.pairs_per_block - 1) / a.pairs_per_block;
  TIP_REQUIRE(grid <= INT32_MAX, "rows x samples too large for one launch");
  int tail = 0;
  for (int l = 1; l < a.n_layers; l++) {
    a.L[l].woff = tail;
    tail += (((a.L[l].in + 1) & ~1) + 1) * TW;
  }
  const size_t bytes = sizeof(float) * ((size_t)kMcChunk * WP + (size_t)kMcTileRows * kMcHStride + tail);
  if (models == 0) {
    auto kern = mc_head_kernel<WP, SPT, TW>;
    if (bytes > 48 * 1024) TIP_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    kern<<<(unsigned)grid, kMcThreads, bytes, stream>>>(a);
    TIP_LAUNCH_CHECK();
    return TIP_OK;
  }
  auto kern = mc_head_kernel<WP, SPT, TW, true>;
  if (bytes > 48 * 1024) TIP_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  static_cast<McArgs&>(*s) = a;
  for (int64_t m0 = 0; m0 < models; m0 += kMcStackChunk) {
    const int n = (int)min((int64_t)kMcStackChunk, models - m0);
    s->model0 = m0;
    for (int k = 0; k < n; k++) s->seeds[k] = seeds[m0 + k];
    kern<<<dim3((unsigned)grid, (unsigned)n), kMcThreads, bytes, stream>>>(*s);
    TIP_LAUNCH_CHECK();
  }
  return TIP_OK;
}

// the layer table's checks and McArgs (everything but h, ld and out) of tip_mc_head and tip_mc_head_stack
int mc_args(int64_t rows, int64_t row0, int64_t sample0, int64_t samples, const tip_mc_layer* layers,
            int32_t n_layers, int32_t mode, McArgs& a, int& widest) {
  TIP_REQUIRE(layers && n_layers >= 1 && n_layers <= kMcMaxLayers, "1..4 layers");
  TIP_REQUIRE(mode == TIP_MC_OUTPUT || mode == TIP_MC_PREACT, "mode is TIP_MC_OUTPUT or TIP_MC_PREACT");
  TIP_REQUIRE(rows >= 0 && samples >= 1 && row0 >= 0 && sample0 >= 0, "rows >= 0, samples >= 1, row0, sample0 >= 0");
  memset(&a, 0, sizeof(a));
  widest = 0;
  for (int l = 0; l < n_layers; l++) {
    const tip_mc_layer& L = layers[l];
    TIP_REQUIRE(L.kernel && L.bias, "null kernel or bias");
    TIP_REQUIRE(L.p >= 0.0 && L.p <= 1.0, "dropout rate in [0, 1]");
    TIP_REQUIRE(L.out >= 1 && L.out <= kMcMaxWidth, "1..64 units per layer");
    TIP_REQUIRE(l == 0 ? (L.in >= 1 && L.in <= kMcMaxIn) : L.in == layers[l - 1].out,
                "layer 0 takes 1..8192 inputs, every later layer the previous layer's units");
    TIP_REQUIRE(L.activation == TIP_MC_LINEAR || L.activation == TIP_MC_RELU ||
                    (L.activation == TIP_MC_SOFTMAX && l == n_layers - 1),
                "linear, relu, or softmax on the last layer");
    McLayer& d = a.L[l];
    d.kernel = L.kernel;
    d.bias = L.bias;
    d.thresh = (uint64_t)rint(L.p * 4294967296.0);
    d.scale = L.p >= 1.0 ? 0.f : (float)(1.0 / (double)(float)(1.0 - L.p));
    d.in = L.in;
    d.out = L.out;
    d.act = L.activation;
    if (L.out > widest) widest = L.out;
  }
  a.rows = rows;
  a.row0 = row0;
  a.sample0 = sample0;
  a.samples = samples;
  a.n_layers = n_layers;
  a.mode = mode;
  return TIP_OK;
}

int mc_dispatch(McArgs& a, int widest, McStackArgs* s, int64_t models, const uint64_t* seeds, cudaStream_t st) {
  if (a.n_layers > 1) {
    if (widest <= 8) return mc_launch<8, 1, 8>(a, s, models, seeds, st);
    if (widest <= 16) return mc_launch<16, 1, 16>(a, s, models, seeds, st);
    if (widest <= 32) return mc_launch<32, 1, 32>(a, s, models, seeds, st);
    return mc_launch<64, 1, 64>(a, s, models, seeds, st);
  }
  if (widest <= 4) return mc_launch<4, 8, 0>(a, s, models, seeds, st);
  if (widest <= 8) return mc_launch<8, 8, 0>(a, s, models, seeds, st);
  if (widest <= 12) return mc_launch<12, 4, 0>(a, s, models, seeds, st);
  if (widest <= 16) return mc_launch<16, 4, 0>(a, s, models, seeds, st);
  if (widest <= 32) return mc_launch<32, 2, 0>(a, s, models, seeds, st);
  return mc_launch<64, 1, 0>(a, s, models, seeds, st);
}

}  // namespace tip

extern "C" int tip_mc_head(const float* h, int64_t rows, int64_t ld, int64_t row0, int64_t sample0, int64_t samples,
                           const tip_mc_layer* layers, int32_t n_layers, uint64_t seed, int32_t mode, float* out,
                           void* stream) {
  using namespace tip;
  McArgs a;
  int widest = 0;
  const int rc = mc_args(rows, row0, sample0, samples, layers, n_layers, mode, a, widest);
  if (rc != TIP_OK) return rc;
  TIP_REQUIRE(out && (h || rows == 0), "null pointer");
  TIP_REQUIRE(ld >= layers[0].in, "row stride below the input width");
  if (rows == 0) return TIP_OK;
  a.h = h;
  a.ld = ld;
  a.seed = seed;
  a.out = out;
  return mc_dispatch(a, widest, nullptr, 0, nullptr, (cudaStream_t)stream);
}

extern "C" int tip_mc_head_stack(const float* h, int64_t models, int64_t rows, int64_t ld, int64_t ldm, int64_t row0,
                                 int64_t sample0, int64_t samples, const tip_mc_layer* layers, int32_t n_layers,
                                 const uint64_t* seeds, int32_t mode, float* out, void* stream) {
  using namespace tip;
  McArgs a;
  int widest = 0;
  const int rc = mc_args(rows, row0, sample0, samples, layers, n_layers, mode, a, widest);
  if (rc != TIP_OK) return rc;
  TIP_REQUIRE(models >= 0 && ldm >= 0, "models >= 0, ldm >= 0");
  TIP_REQUIRE(seeds || models == 0, "null seeds");
  TIP_REQUIRE(out && (h || rows == 0 || models == 0), "null pointer");
  TIP_REQUIRE(ld >= layers[0].in, "row stride below the input width");
  if (rows == 0 || models == 0) return TIP_OK;
  a.h = h;
  a.ld = ld;
  a.out = out;
  McStackArgs s;
  memset(&s, 0, sizeof(s));
  s.ldm = ldm;
  return mc_dispatch(a, widest, &s, models, seeds, (cudaStream_t)stream);
}
