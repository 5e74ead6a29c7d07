// shard.cu — exchange steps of the N_train-sharded search (SURVEY.md §8e, north_star: "the N_train
// axis shards across the 8 GPUs of one box with a single all-reduce of per-shard min distances /
// partial KDE sums over NVLink").
//
// The dependency that forces an exchange is surprise.py:615-631: stage 2's queries are the GLOBAL
// stage-1 winners, so every rank needs (min distance, first-occurrence index) over all shards before
// it can start stage 2, and the global stage-2 minimum before dist_a / dist_b.  Both messages are one
// 16-byte record per test input.  They travel over NVLink as plain peer stores:
//
//   tip_comm_push_*     every rank writes its m records straight into the receive slots of all peers
//                       (symmetric cudaMalloc buffers opened through CUDA IPC), then raises one flag
//                       per peer (fence.sys + last-block-done pattern);
//   consumer kernels    (tip_shard_winner_queries, tip_comm_min, tip_comm_lse) spin on the local
//                       flags, reduce the `world` records of every query from LOCAL memory and go
//                       straight on with the next compute step of the pipeline — the all-reduce is
//                       fused into the prologue of its consumer; no NCCL launch, no extra pass over
//                       the records, and the whole sharded call stays one CUDA graph.
//
// Records are ordered as unsigned (hi, lo) pairs: a non-negative IEEE distance orders like its bit
// pattern, the original train index breaks exact ties towards the first occurrence (np.argmin).
// Receive slots are double-buffered by the parity of the exchange's sequence number, so a fast rank's
// next push can never overwrite records a slow rank is still reading (it cannot get two exchanges
// ahead: every consumer waits for all peers' flags of the current exchange).
//
// The same consumers also run without a tip_comm (records already reduced by NCCL / gloo through
// torch.distributed): that is the fallback when peer access is unavailable, and what the CPU
// protocol test mirrors.
#include <vector>

#include "common.cuh"

struct tip_comm {
  int rank, world;
  int64_t cap;          // records per rank and slot
  int64_t bytes;
  unsigned char* local;
  unsigned char* peer[TIP_COMM_MAX_WORLD];   // peer[rank] == local
  bool opened[TIP_COMM_MAX_WORLD];
};

namespace tip {

constexpr int kHdrBytes = 1024;        // flags[world] at 0, seq at 256, done counter at 260
// "No row of that range on this shard" is a quiet NaN's pattern, above +inf's: a real distance can be +inf
// (squared differences that overflow), and unsigned order still puts it ahead of "none" (engine.dist_keys).
constexpr uint64_t kNoneHi64 = 0x7ff8000000000000ull;
constexpr uint64_t kNoneHi32 = 0x7fc00000ull;
constexpr uint64_t kInfHi64 = 0x7ff0000000000000ull;
constexpr uint64_t kInfHi32 = 0x7f800000ull;
constexpr uint64_t kNoneLo = 0x7fffffffull;

struct CommDev {
  int rank, world;
  int64_t cap;
  unsigned char* local;
  unsigned char* peer[TIP_COMM_MAX_WORLD];
};

static CommDev comm_dev(const tip_comm* c) {
  CommDev d{};
  d.rank = c->rank; d.world = c->world; d.cap = c->cap; d.local = c->local;
  for (int p = 0; p < c->world; p++) d.peer[p] = c->peer[p];
  return d;
}

__host__ __device__ inline int64_t comm_bytes(int world, int64_t cap) {
  return kHdrBytes + 2 * (int64_t)world * cap * 16;
}

__device__ __forceinline__ ulonglong2* rec_slot(unsigned char* base, const CommDev& c, uint32_t seq, int from) {
  return reinterpret_cast<ulonglong2*>(base + kHdrBytes) + ((int64_t)(seq & 1u) * c.world + from) * c.cap;
}

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ ulonglong2 ld_cg_u128(const ulonglong2* p) {
  ulonglong2 v;
  asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ long long globaltimer_ns() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Blocks until every peer has raised its flag for the current exchange (the one this rank's last
// push started); returns its sequence number.  Bounded: a peer that never arrives traps the kernel
// after 20 s instead of hanging the GPU.
__device__ __forceinline__ uint32_t comm_wait(const CommDev& c) {
  __shared__ uint32_t s_seq;
  const uint32_t* flags = reinterpret_cast<const uint32_t*>(c.local);
  if (threadIdx.x < (unsigned)c.world) {
    const uint32_t seq = *reinterpret_cast<const volatile uint32_t*>(c.local + 256);
    const long long t0 = globaltimer_ns();
    while ((int32_t)(ld_acquire_sys(flags + threadIdx.x) - seq) < 0) {
      if (globaltimer_ns() - t0 > 20000000000LL) __trap();
    }
    if (threadIdx.x == 0) s_seq = seq;
  }
  __syncthreads();
  return s_seq;
}

// ---- producers -----------------------------------------------------------------------------------
enum { PUSH_NN = 0, PUSH_LSE = 1 };

template <typename T>
__device__ __forceinline__ uint64_t dist_bits(T v);
template <>
__device__ __forceinline__ uint64_t dist_bits<float>(float v) {
  return v != v ? kNoneHi32 : (uint64_t)__float_as_uint(v);    // NaN = "no row of that range on this shard"
}
template <>
__device__ __forceinline__ uint64_t dist_bits<double>(double v) {
  return v != v ? kNoneHi64 : (uint64_t)__double_as_longlong(v);
}

template <typename T, int KIND>
__global__ void __launch_bounds__(256) comm_push_kernel(const CommDev c, const T* __restrict__ a,
                                                        const int32_t* __restrict__ gid,
                                                        const float* __restrict__ b, int64_t m) {
  uint32_t* seq_p = reinterpret_cast<uint32_t*>(c.local + 256);
  uint32_t* done_p = reinterpret_cast<uint32_t*>(c.local + 260);
  const uint32_t seq = *reinterpret_cast<volatile uint32_t*>(seq_p) + 1u;   // stable until the last block is through
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < m; i += (int64_t)gridDim.x * 256) {
    ulonglong2 rec;
    if (KIND == PUSH_NN) {
      rec.x = dist_bits<T>(a[i]);
      const int g = gid ? gid[i] : 0;
      rec.y = g < 0 ? kNoneLo : (uint64_t)(uint32_t)g;
    } else {
      rec.x = (uint64_t)__float_as_uint((float)a[i]);    // running maximum
      rec.y = (uint64_t)__float_as_uint(b[i]);           // sum of exp(. - maximum)
    }
    for (int p = 0; p < c.world; p++) rec_slot(c.peer[p], c, seq, c.rank)[i] = rec;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    if (atomicAdd(done_p, 1u) == gridDim.x - 1) {
      __threadfence_system();
      *done_p = 0;
      *reinterpret_cast<volatile uint32_t*>(seq_p) = seq;
      __threadfence_system();
      for (int p = 0; p < c.world; p++) st_release_sys(reinterpret_cast<uint32_t*>(c.peer[p]) + c.rank, seq);
    }
  }
}

// ---- consumers -----------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T bits_dist(uint64_t hi);
template <>
__device__ __forceinline__ float bits_dist<float>(uint64_t hi) {
  return hi > kInfHi32 ? __int_as_float(0x7fc00000) : __uint_as_float((uint32_t)hi);
}
template <>
__device__ __forceinline__ double bits_dist<double>(uint64_t hi) {
  return hi > kInfHi64 ? (double)NAN : __longlong_as_double((long long)hi);
}

__device__ __forceinline__ ulonglong2 reduce_min_records(const CommDev& c, uint32_t seq, int64_t i) {
  ulonglong2 best = ld_cg_u128(rec_slot(c.local, c, seq, 0) + i);
  for (int p = 1; p < c.world; p++) {
    const ulonglong2 r = ld_cg_u128(rec_slot(c.local, c, seq, p) + i);
    if (r.x < best.x || (r.x == best.x && r.y < best.y)) best = r;
  }
  return best;
}

// Global stage-1 winners -> stage-2 queries (surprise.py:627-629: the queries of the other-class
// search are the winning TRAIN rows).  One warp per test input: reduce the per-shard records (or
// take the already reduced gdist/ggid), fetch the winner's trace from the replicated training
// set by original index and emit it in the trace dtype (the re-rank's query) and as the packed
// bf16 operand + reset filter state of the next tip_nn_filter call.
template <typename T, bool COMM>
__global__ void __launch_bounds__(256) winner_queries_kernel(const CommDev c, const T* __restrict__ gdist,
                                                             const int32_t* __restrict__ ggid, int64_t m, int d,
                                                             const T* __restrict__ train_full, int64_t n_full,
                                                             const float* __restrict__ center,
                                                             T* __restrict__ out_dist, int32_t* __restrict__ out_gid,
                                                             T* __restrict__ out_rows,
                                                             __nv_bfloat16* __restrict__ next_pack, int64_t pitch,
                                                             float* __restrict__ next_sqnorm,
                                                             float* __restrict__ next_rounderr,
                                                             uint32_t* __restrict__ next_row_min,
                                                             int32_t* __restrict__ next_cand_cnt) {
  uint32_t seq = 0;
  if (COMM) seq = comm_wait(c);
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= m) return;
  T dist;
  int gid;
  if (COMM) {
    const ulonglong2 best = reduce_min_records(c, seq, row);
    dist = bits_dist<T>(best.x);
    gid = best.y >= kNoneLo ? -1 : (int)best.y;
  } else {
    dist = gdist[row];
    gid = ggid[row];
  }
  // only "no row" (the NaN sentinel) or an index outside the training set drops the winner; +inf is a distance
  if (gid < 0 || gid >= n_full || dist != dist) { gid = -1; dist = (T)NAN; }
  if (lane == 0) {
    out_dist[row] = dist;
    out_gid[row] = gid;
  }
  const T* src = gid >= 0 ? train_full + (int64_t)gid * d : nullptr;
  T* dst = out_rows + row * (int64_t)d;
  for (int i = lane; i < d; i += 32) dst[i] = src ? src[i] : (T)0;
  warp_pack_query<T>(src, d, center, next_pack + row * pitch, pitch, next_sqnorm + row,
                     next_rounderr ? next_rounderr + row : nullptr, next_row_min + row, next_cand_cnt + row, lane);
}

template <typename T>
__global__ void __launch_bounds__(256) comm_min_kernel(const CommDev c, int64_t m, T* __restrict__ out) {
  const uint32_t seq = comm_wait(c);
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < m; i += (int64_t)gridDim.x * 256)
    out[i] = bits_dist<T>(reduce_min_records(c, seq, i).x);
}

// Partial KDE sums (max_r, sum_r) of every shard merged in rank order, identically on every rank:
// M = max_r max_r; S = sum_r sum_r * exp(max_r - M) in double.
__global__ void __launch_bounds__(256) comm_lse_kernel(const CommDev c, int64_t m, float* __restrict__ out_max,
                                                       double* __restrict__ out_sum) {
  const uint32_t seq = comm_wait(c);
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < m; i += (int64_t)gridDim.x * 256) {
    float mx = -INFINITY;
    for (int p = 0; p < c.world; p++)
      mx = fmaxf(mx, __uint_as_float((uint32_t)ld_cg_u128(rec_slot(c.local, c, seq, p) + i).x));
    double s = 0.0;
    for (int p = 0; p < c.world; p++) {
      const ulonglong2 r = ld_cg_u128(rec_slot(c.local, c, seq, p) + i);
      const float pm = __uint_as_float((uint32_t)r.x), ps = __uint_as_float((uint32_t)r.y);
      if (pm > -INFINITY) s += (double)ps * exp((double)pm - (double)mx);
    }
    out_max[i] = mx;
    out_sum[i] = s;
  }
}

static int grid_for(int64_t m) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((m + 255) / 256, 2 * (int64_t)sm_count()));
}

}  // namespace tip

using namespace tip;

extern "C" int64_t tip_comm_bytes(int32_t world, int64_t cap_records) {
  if (world < 1 || world > TIP_COMM_MAX_WORLD || cap_records < 1) return -1;
  return comm_bytes(world, cap_records);
}

extern "C" int tip_comm_alloc(int32_t world, int64_t cap_records, void** local_buf, void* ipc_handle) {
  TIP_REQUIRE(local_buf && ipc_handle, "null pointer");
  TIP_REQUIRE(world >= 1 && world <= TIP_COMM_MAX_WORLD && cap_records >= 1, "world / cap_records");
  static_assert(sizeof(cudaIpcMemHandle_t) == TIP_COMM_HANDLE_BYTES, "ipc handle size");
  const int64_t bytes = comm_bytes(world, cap_records);
  void* p = nullptr;
  TIP_CHECK_CUDA(cudaMalloc(&p, (size_t)bytes));
  TIP_CHECK_CUDA(cudaMemset(p, 0, (size_t)bytes));
  TIP_CHECK_CUDA(cudaDeviceSynchronize());
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    cudaFree(p);
    set_error("cudaIpcGetMemHandle -> %s", cudaGetErrorString(e));
    return TIP_ERR_CUDA;
  }
  memcpy(ipc_handle, &h, sizeof(h));
  *local_buf = p;
  return TIP_OK;
}

extern "C" int tip_comm_free_local(void* local_buf) {
  if (local_buf) TIP_CHECK_CUDA(cudaFree(local_buf));
  return TIP_OK;
}

extern "C" int tip_comm_open(int32_t rank, int32_t world, void* local_buf, const void* all_handles,
                             int64_t cap_records, tip_comm** out) {
  TIP_REQUIRE(local_buf && all_handles && out, "null pointer");
  TIP_REQUIRE(world >= 1 && world <= TIP_COMM_MAX_WORLD && rank >= 0 && rank < world && cap_records >= 1, "rank / world");
  tip_comm* c = new tip_comm();
  c->rank = rank; c->world = world; c->cap = cap_records; c->bytes = comm_bytes(world, cap_records);
  c->local = (unsigned char*)local_buf;
  for (int p = 0; p < world; p++) {
    c->opened[p] = false;
    if (p == rank) { c->peer[p] = c->local; continue; }
    cudaIpcMemHandle_t h;
    memcpy(&h, (const unsigned char*)all_handles + (size_t)p * TIP_COMM_HANDLE_BYTES, sizeof(h));
    void* ptr = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      set_error("cudaIpcOpenMemHandle(peer %d) -> %s", p, cudaGetErrorString(e));
      for (int q = 0; q < p; q++)
        if (c->opened[q]) cudaIpcCloseMemHandle(c->peer[q]);
      delete c;
      cudaGetLastError();
      return TIP_ERR_CUDA;
    }
    c->peer[p] = (unsigned char*)ptr;
    c->opened[p] = true;
  }
  *out = c;
  return TIP_OK;
}

extern "C" int tip_comm_close(tip_comm* c) {
  if (!c) return TIP_OK;
  for (int p = 0; p < c->world; p++)
    if (c->opened[p]) cudaIpcCloseMemHandle(c->peer[p]);
  delete c;
  return TIP_OK;
}

extern "C" int tip_comm_push_nn(tip_comm* c, const void* dist, int dtype, const int32_t* gid, int64_t m, void* stream) {
  TIP_REQUIRE(c && dist, "null pointer");
  TIP_REQUIRE(m >= 1 && m <= c->cap, "more records than the communicator was sized for");
  cudaStream_t st = (cudaStream_t)stream;
  const CommDev cd = comm_dev(c);
  if (dtype == TIP_F32)
    comm_push_kernel<float, PUSH_NN><<<grid_for(m), 256, 0, st>>>(cd, (const float*)dist, gid, nullptr, m);
  else if (dtype == TIP_F64)
    comm_push_kernel<double, PUSH_NN><<<grid_for(m), 256, 0, st>>>(cd, (const double*)dist, gid, nullptr, m);
  else
    TIP_REQUIRE(false, "dtype must be TIP_F32 or TIP_F64");
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_comm_push_lse(tip_comm* c, const float* part_max, const float* part_sum, int64_t m, void* stream) {
  TIP_REQUIRE(c && part_max && part_sum, "null pointer");
  TIP_REQUIRE(m >= 1 && m <= c->cap, "more records than the communicator was sized for");
  comm_push_kernel<float, PUSH_LSE><<<grid_for(m), 256, 0, (cudaStream_t)stream>>>(comm_dev(c), part_max, nullptr,
                                                                                 part_sum, m);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_comm_min(tip_comm* c, int dtype, int64_t m, void* out_dist, void* stream) {
  TIP_REQUIRE(c && out_dist, "null pointer");
  TIP_REQUIRE(m >= 1 && m <= c->cap, "more records than the communicator was sized for");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == TIP_F32) comm_min_kernel<float><<<grid_for(m), 256, 0, st>>>(comm_dev(c), m, (float*)out_dist);
  else if (dtype == TIP_F64) comm_min_kernel<double><<<grid_for(m), 256, 0, st>>>(comm_dev(c), m, (double*)out_dist);
  else TIP_REQUIRE(false, "dtype must be TIP_F32 or TIP_F64");
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_comm_lse(tip_comm* c, int64_t m, float* out_max, double* out_sum, void* stream) {
  TIP_REQUIRE(c && out_max && out_sum, "null pointer");
  TIP_REQUIRE(m >= 1 && m <= c->cap, "more records than the communicator was sized for");
  comm_lse_kernel<<<grid_for(m), 256, 0, (cudaStream_t)stream>>>(comm_dev(c), m, out_max, out_sum);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_shard_winner_queries(tip_comm* c, const void* gdist, const int32_t* ggid, int dtype, int64_t m,
                                        int64_t d, const void* train_full, int64_t n_full, const float* center,
                                        void* out_dist, int32_t* out_gid, void* out_rows, void* next_pack,
                                        float* next_sqnorm, float* next_rounderr, uint32_t* next_row_min_bits,
                                        int32_t* next_cand_cnt, void* stream) {
  TIP_REQUIRE(train_full && out_dist && out_gid && out_rows && next_pack && next_sqnorm && next_row_min_bits &&
                  next_cand_cnt, "null pointer");
  TIP_REQUIRE(c != nullptr || (gdist != nullptr && ggid != nullptr), "either a communicator or reduced (dist, index) arrays");
  TIP_REQUIRE(m >= 0 && d >= 1 && d < (1LL << 31) && n_full >= 1 && n_full < (1LL << 31), "shape");
  TIP_REQUIRE(c == nullptr || m <= c->cap, "more records than the communicator was sized for");
  if (m == 0) return TIP_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t pitch = tip_pair_pitch(d, 1);
  const unsigned blocks = (unsigned)((m + 7) / 8);
  const CommDev cd = c ? comm_dev(c) : CommDev{};
#define TIP_WQ(T, COMM)                                                                                           \
  winner_queries_kernel<T, COMM><<<blocks, 256, 0, st>>>(cd, (const T*)gdist, ggid, m, (int)d, (const T*)train_full, \
                                                         n_full, center, (T*)out_dist, out_gid, (T*)out_rows,     \
                                                         (__nv_bfloat16*)next_pack, pitch, next_sqnorm,           \
                                                         next_rounderr, next_row_min_bits, next_cand_cnt)
  if (dtype == TIP_F32) { if (c) TIP_WQ(float, true); else TIP_WQ(float, false); }
  else if (dtype == TIP_F64) { if (c) TIP_WQ(double, true); else TIP_WQ(double, false); }
  else TIP_REQUIRE(false, "dtype must be TIP_F32 or TIP_F64");
#undef TIP_WQ
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}
