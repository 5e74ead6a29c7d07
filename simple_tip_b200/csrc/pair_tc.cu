// pair_tc.cu — the tensor-core pass over (query, train) activation-trace pairs (sm_90a).
//
// One persistent, warp-specialised kernel computes, for 128 query rows x 128 train rows at a
// time, the fp32 accumulator
//        acc[i][j] = norm_coef*|y_j|^2 + scale*<x_i, y_j>
// (both terms come out of the same wgmma K-loop: the packed operands carry a 16-wide tail
// block with a 3-way bf16 split of the norm on the train side and ones on the query side, see
// tip_pair_prep) and reduces it on the fly — no N_test x N_train intermediate ever leaves the SM:
//   MODE_NN   per-row running minimum + candidate emission (DSA, surprise.py:638-647)
//   MODE_LSE  per-row online log-sum-exp (LSA / Gaussian KDE, scipy 1.4.1 gaussian_kernel_estimate)
//   MODE_DSUM per-row sum of Euclidean distances over the item's span (silhouette score, sklearn
//             silhouette_samples); the query's own column contributes 0
//   MODE_DUMP raw accumulator tile (bring-up / validation)
//
// Roles: warpgroup 0 = TMA producer and work-item hand-out (one lane of warp 0) and, in the resident MODE_NN kernel,
// three drain warps; warpgroups 1.. = consumers.  Consumer warpgroup g owns query rows [64 g, 64 g + 64) of the tile:
// it issues m64n128k16 wgmma for them, keeps the accumulator in registers and reduces it there.  In the wgmma
// accumulator layout the four lanes of a quad hold one row between them (8 of every 32 consecutive columns each), so
// the per-row reductions finish with two quad shuffles.  The consumer warpgroups drift out of phase, so one's MMAs
// overlap another's reduction.  The resident MODE_NN kernel has three consumer warpgroups on 192-row query tiles
// (512 threads; warpgroup 0 hands registers to the consumers with setmaxnreg): while one reduces, the other two
// keep the tensor core busy, and each train tile fetched from L2 feeds 1.5x the MMAs.  Handing the tensor core from
// one warpgroup to the next (each issues a tile's MMAs only after the previous one has issued its own) was measured
// slower: alone, one warpgroup's nine m64n128k16 run at about half the tensor core's rate, so the three warpgroups'
// MMAs take longer one after another than together (DESIGN.md §8).  At d = 128 its consumers hold most of the query
// tile's K steps in registers (wgmma with a register A operand), so their MMAs read mostly the train tile from shared
// memory.  A consumer warpgroup whose rows all lie past the item's query rows issues no MMAs.  Every other
// instantiation has two consumer warpgroups on 128-row tiles (384 threads).
// Pipeline: kStages-deep shared-memory ring (full/empty mbarriers, TMA -> wgmma).  Streaming variant:
// one commit group per K chunk, each waited for and its stage released before the next chunk.
// Resident-query variant (RESA, short packed rows): the query tile's K chunks are loaded once per run
// of consecutive work items on the same query tile, the ring carries train chunks only, and a tile's
// MMAs form one commit group whose stages are released after its wait.
// MODE_NN events, resident variant: per row and tile the consumers reduce all four 32-column chunks in one pass,
// move the running minimum and threshold once, to the tile's minimum, and write one record per chunk inside that
// end-of-tile threshold into the tile's mailbox (two, by tile parity, with full/empty mbarriers); the drain warps
// own the per-row candidate staging (compaction, direct emission when full, the flush at the end of an item).  With no data-dependent staging or divergent shuffles in
// the consumers' tile loop, ptxas keeps the wgmma asynchronous: a tile's HGMMAs issue back to back.
// Streaming variant: the quad's first lane stages its events itself; there ptxas still serialises the
// wgmma (C7520), which costs little next to the per-chunk waits, and moving the staging to the drain
// warps made the C5 slice slower (DESIGN.md §8).
#include <cuda.h>
#include <cudaTypedefs.h>

#include <algorithm>
#include <cstdlib>
#include "common.cuh"

namespace tip {

constexpr int BM = 128;  // query rows per tile, except in the resident MODE_NN kernel (Layout::kRows)
constexpr int BN = 128;
constexpr int BK = 64;  // bf16 elements per smem row = one 128-byte swizzle atom
constexpr int kStages = 6;
constexpr int kABytes = BM * BK * 2;
constexpr int kBBytes = BN * BK * 2;
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kRingBytes = kStages * kStageBytes;
constexpr int kResAChunks = 5;               // resident-query variant: query tiles of up to 5 x 64 K elements
constexpr int kCandSlots = 8;   // per-query staging slots for candidates (MODE_NN)
constexpr int kEvSlots = BN / 32;   // MODE_NN events per row and tile: one per 32-column chunk
constexpr int kDrainWarps = 3;      // warps 1..3 of warpgroup 0
// MODE_NN event mailbox, one per tile parity: the consumers record a tile's events, the drain warps stage them
struct EvRecord { int col; uint32_t mask; float mn, thr; };   // chunk start, column mask, chunk minimum, row thr
struct EvRow { float thr; int ev; };                          // row thr after the tile, bit c = event in chunk c
template <int ROWS>
struct EvBuf {
  EvRecord rec[ROWS * kEvSlots];
  EvRow row[ROWS];
  int q_row0, flags, pad[2];
};
enum { kEvLast = 1, kEvStop = 2 };   // EvBuf::flags: last tile of the item (flush), no more tiles
constexpr int kBarBytes = 256;
constexpr int kSmemMax = 232448;   // 227 KB per block on sm_90
// tip_nn_filter keeps the query tile resident for packed rows of at most this many K16 steps (d <= 128)
constexpr int kRsMaxK16 = 9;

enum { MODE_NN = 0, MODE_LSE = 1, MODE_DUMP = 2, MODE_DSUM = 3 };

// Per-instantiation shape of pair_kernel.  Shared memory: [kFront: streaming ring, or resident query tile + train
// ring] [barriers + hand-out slots] [candidate staging] [two event mailboxes].
template <int MODE, bool RESA>
struct Layout {
  static constexpr int kWgs = MODE == MODE_NN && RESA ? 3 : 2;   // consumer warpgroups
  static constexpr int kRows = 64 * kWgs;                         // query rows per tile
  static constexpr int kConsumerWarps = 4 * kWgs;
  static constexpr int kThreads = 128 + 32 * kConsumerWarps;
  static constexpr int kABytes = kRows * BK * 2;                  // one resident K chunk of the query tile
  static constexpr int kResAChunks = kWgs == 3 ? (kRsMaxK16 + 3) / 4 : tip::kResAChunks;
  static constexpr int kFront = kWgs == 3 ? kResAChunks * kABytes + kStages * kBBytes : kRingBytes;
  static constexpr int kCandBytes = kCandSlots * kRows * 12;      // value, chunk start, 32-bit column mask
  static constexpr int kSmemBytes = kFront + 1024 /*align slack*/ + kBarBytes + kCandBytes + 2 * (int)sizeof(EvBuf<kRows>);
  static_assert(!RESA || kResAChunks * kABytes + kStages * kBBytes <= kFront, "resident-query layout does not fit");
  static_assert(kSmemBytes <= kSmemMax, "pair kernel does not fit");
};

struct PairArgs {
  const tip_work_item* items;
  int n_items;
  // items [0, n_static) are scheduled statically (CTA b runs b, b + G, ...), items [n_static, n_items)
  // form a pool that CTAs drain through the atomic counter once they run dry
  int n_static;
  int* sched_counter;
  // optional (tip_nn_filter_live): query rows at and past q_live_end[q_row0] hold no query; an item's rows end there,
  // and an item without rows is skipped by the producer (no query-tile load, no ring stage)
  const int32_t* q_live_end;
  int k16;  // number of K=16 MMA steps per tile (packed width / 16)
  int64_t m;
  // MODE_NN
  const int32_t* q_class;     // with class_off: per-query excluded train range (items flagged 1)
  const int32_t* class_off;
  const float* q_sqnorm;
  float rmax, eps2, gamma;  // error-window constants (DESIGN.md §4)
  const float* q_err;       // measured input-rounding norms |x~ - bf16(x~)| per query (or nullptr: a-priori bound)
  float t_err;              // max over the train rows of the same
  uint32_t* row_min_bits;
  int32_t* cand_idx;
  int32_t* cand_cnt;
  int cap;
  // MODE_LSE (MODE_DSUM: part_sum only)
  float* part_max;
  float* part_sum;
  // MODE_DUMP
  float* dump;
  // bring-up: per-tile clock64 stamps of block 0 (16 slots per tile), or nullptr
  long long* timeline;
  int timeline_tiles;
  // bring-up: per-CTA {globaltimer at start, at end, tiles, items}, or nullptr
  long long* cta_clock;
};

// ---- PTX wrappers --------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a protocol bug must surface as a trapped kernel, never as a hung GPU.  BOUNDED = false: the consumers
// of the resident MODE_NN kernel, because ptxas ignores setmaxnreg's larger register budget in a region that can trap
// (and an exit there, with wgmma in flight, serialises the wgmma).  A consumer warp stuck in such a wait never hands
// the drain warps its last mailbox, so their bounded wait traps instead.
template <bool BOUNDED = true>
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, uint32_t max_spins = 200000000u) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (BOUNDED && ++spins > max_spins) __trap();
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// K-major, 128-byte-swizzled operand tile as written by TMA: rows of 128 B, 8-row groups 1024 B apart
// (wgmma matrix descriptor: start>>4 | LBO=1 (unused for swizzled K-major) <<16 | SBO=1024>>4 <<32 | SWIZZLE_128B=1<<62).
// One K=16 slice is +32 bytes inside the swizzle row = +2 in the start field.
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr) {
  return (uint64_t)((addr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Operand fence: the compiler may not move any access to the accumulator registers across this point, so
// reads happen after the wait that retires the MMAs and never while an MMA that writes them is in flight.
__device__ __forceinline__ void acc_fence(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; i++) asm volatile("" : "+f"(d[i])::"memory");
}

#define TIP_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                    "+f"(d[i + 6]), "+f"(d[i + 7])
#define TIP_WGMMA_REGS                                                                                           \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, " \
  "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "   \
  "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, both operands K-major in shared memory; accumulate = 0 overwrites D
template <bool F16>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if (F16) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " TIP_WGMMA_REGS ", %64, %65, p, 1, 1, 0, 0;\n\t}"
        : TIP_ACC8(0), TIP_ACC8(8), TIP_ACC8(16), TIP_ACC8(24), TIP_ACC8(32), TIP_ACC8(40), TIP_ACC8(48), TIP_ACC8(56)
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " TIP_WGMMA_REGS ", %64, %65, p, 1, 1, 0, 0;\n\t}"
        : TIP_ACC8(0), TIP_ACC8(8), TIP_ACC8(16), TIP_ACC8(24), TIP_ACC8(32), TIP_ACC8(40), TIP_ACC8(48), TIP_ACC8(56)
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
  }
}
// The same with A from registers: the m64 x k16 bf16 fragment of this thread in the layout ldmatrix.x4 gives
__device__ __forceinline__ void wgmma_m64n128k16_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc,
                                                    uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " TIP_WGMMA_REGS ", {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      : TIP_ACC8(0), TIP_ACC8(8), TIP_ACC8(16), TIP_ACC8(24), TIP_ACC8(32), TIP_ACC8(40), TIP_ACC8(48), TIP_ACC8(56)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
#undef TIP_ACC8
#undef TIP_WGMMA_REGS

// Acceptance threshold (accumulator space) for a query whose smallest approximate squared
// distance so far is s: every train row whose exact NumPy distance could still be the minimum
// has acc <= thr.  r = |x_b| + max|y_b|, e2 = 2*eps'*r, g = gamma*r^2 (DESIGN.md §4).
__device__ __forceinline__ float nn_threshold(float s, float nx, float e2, float g) {
  float root;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(root) : "f"(s + g));   // <= 2 ulp; covered by the slack below
  float r = root + e2;
  r *= 1.00004f;
  float thr = fmaf(r, r, g) - nx;
  return thr + fabsf(thr) * 1e-6f + 1e-30f;
}

struct EpiState {
  bool valid_row;
  int64_t row;
  int col1;
  int ex_lo, ex_hi;                    // train rows this query must ignore (its own class), or empty
  float nx, e2, g, best, thr, s_ref;   // MODE_NN (identical in the four lanes of the row's quad)
  int n_staged;                        // MODE_NN streaming variant, kept by the quad's first lane only
  float run_max, run_sum;              // MODE_LSE
  double dsum;                         // MODE_DSUM
};
// MODE_NN per-row candidate staging: slot k of local row r at [k * ROWS + r] (ROWS: the tile's query rows)
struct EpiShared {
  float* cand_val;
  int* cand_col;
  uint32_t* cand_mask;
};

// Stage chunk `col` (minimum mn, column mask) of a row with n staged chunks.  Full slots are first compacted against
// thr (the row's current threshold); if they all stay live, the chunk goes straight to the row's list.
template <int ROWS>
__device__ __forceinline__ void stage_chunk(const PairArgs& args, const EpiShared& sh, int r, int& n, int64_t row,
                                            int col, uint32_t mask, float mn, float thr) {
  if (n == kCandSlots) {
    int keep = 0;
    for (int k = 0; k < kCandSlots; k++) {
      const float sv = sh.cand_val[k * ROWS + r];
      if (sv <= thr) {
        sh.cand_val[keep * ROWS + r] = sv;
        sh.cand_col[keep * ROWS + r] = sh.cand_col[k * ROWS + r];
        sh.cand_mask[keep * ROWS + r] = sh.cand_mask[k * ROWS + r];
        keep++;
      }
    }
    n = keep;
  }
  if (n < kCandSlots) {
    sh.cand_val[n * ROWS + r] = mn;
    sh.cand_col[n * ROWS + r] = col;
    sh.cand_mask[n * ROWS + r] = mask;
    n++;
  } else {
    const int pos = atomicAdd(args.cand_cnt + row, 1);
    if (pos < args.cap) {
      args.cand_idx[(row * args.cap + pos) * 2] = col;
      args.cand_idx[(row * args.cap + pos) * 2 + 1] = (int)mask;
    }
  }
}
// End of an item: emit the staged chunks of a row that survive its final threshold.
template <int ROWS>
__device__ __forceinline__ void flush_row(const PairArgs& args, const EpiShared& sh, int r, int n, int64_t row,
                                          float thr) {
  for (int q = 0; q < n; q++) {
    if (sh.cand_val[q * ROWS + r] <= thr) {
      const int pos = atomicAdd(args.cand_cnt + row, 1);
      if (pos < args.cap) {
        args.cand_idx[(row * args.cap + pos) * 2] = sh.cand_col[q * ROWS + r];
        args.cand_idx[(row * args.cap + pos) * 2 + 1] = (int)sh.cand_mask[q * ROWS + r];
      }
    }
  }
}

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Reduce the 32 accumulator columns [cbase, cbase + 32) of one query row.  The row's quad holds them:
// lane `sub` (0..3) has v[2 jj + e] = column cbase + 8 jj + 2 sub + e.  Every lane of the warp calls
// this (the quad shuffles need the whole warp); the running state comes out the same in the four lanes
// of a quad.  MODE_NN here is the streaming variant only (its MMAs are waited for chunk by chunk anyway): the quad's
// first lane stages an event (a chunk inside the row's window) itself (etid = the row's staging column).  The resident
// variant reduces a whole tile per row in one pass in pair_kernel's epilogue.
template <int MODE, bool EXCL>
__device__ __forceinline__ void epi_chunk(const PairArgs& args, EpiState& st, const EpiShared& sh, float (&v)[8],
                                          int cbase, int sub, bool partial, int etid) {
  const float kInf = __int_as_float(0x7f800000);
  if (MODE == MODE_NN) {
    if (partial || (EXCL && cbase < st.ex_hi && cbase + 32 > st.ex_lo)) {
      // rare: the chunk runs past the span, or overlaps the train rows this query must ignore
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const int col = cbase + 8 * (k >> 1) + 2 * sub + (k & 1);
        if (col >= st.col1 || (EXCL && col >= st.ex_lo && col < st.ex_hi)) v[k] = kInf;
      }
    }
    float mn = fminf(fminf(fminf(v[0], v[1]), fminf(v[2], v[3])), fminf(fminf(v[4], v[5]), fminf(v[6], v[7])));
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, 1));
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, 2));
    // event: this chunk holds a value inside the acceptance window of this query (quad-uniform)
    if (st.valid_row && mn <= st.thr && mn < kInf) {
      if (mn < st.best) {
        st.best = mn;
        st.s_ref = fminf(st.s_ref, fmaxf(st.best + st.nx, 0.f));
        st.thr = nn_threshold(st.s_ref, st.nx, st.e2, st.g);
      }
      const unsigned qmask = 0xFu << ((threadIdx.x & 31) & 28);   // the lanes of this quad
      uint32_t mask = 0;
#pragma unroll
      for (int k = 0; k < 8; k++) mask |= (v[k] <= st.thr) ? (1u << (8 * (k >> 1) + 2 * sub + (k & 1))) : 0u;
      mask |= __shfl_xor_sync(qmask, mask, 1);
      mask |= __shfl_xor_sync(qmask, mask, 2);
      if (sub == 0) stage_chunk<BM>(args, sh, etid, st.n_staged, st.row, cbase, mask, mn, st.thr);
    }
  } else if (MODE == MODE_LSE) {
    constexpr float kL2e = 1.4426950408889634f;
    float mx = -kInf;
    if (partial) {
#pragma unroll
      for (int k = 0; k < 8; k++) {
        if (cbase + 8 * (k >> 1) + 2 * sub + (k & 1) >= st.col1) v[k] = -kInf;
        mx = fmaxf(mx, v[k]);
      }
    } else {
#pragma unroll
      for (int k = 0; k < 8; k += 2) mx = fmaxf(mx, fmaxf(v[k], v[k + 1]));
    }
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    if (mx > st.run_max) {
      st.run_sum *= fast_exp2((st.run_max - mx) * kL2e);  // run_max = -inf -> factor 0
      st.run_max = mx;
    }
    float s = 0.f;
    if (st.run_max > -kInf) {
      const float off = -st.run_max * kL2e;
      const float s0 = fast_exp2(fmaf(v[0], kL2e, off)) + fast_exp2(fmaf(v[4], kL2e, off));
      const float s1 = fast_exp2(fmaf(v[1], kL2e, off)) + fast_exp2(fmaf(v[5], kL2e, off));
      const float s2 = fast_exp2(fmaf(v[2], kL2e, off)) + fast_exp2(fmaf(v[6], kL2e, off));
      const float s3 = fast_exp2(fmaf(v[3], kL2e, off)) + fast_exp2(fmaf(v[7], kL2e, off));
      s = (s0 + s1) + (s2 + s3);
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);     // IEEE addition is commutative: the four lanes agree
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    st.run_sum += s;
  } else if (MODE == MODE_DSUM) {
    // acc = |y|^2 - 2<x, y>: + |x|^2, clamp, sqrt.  Columns past the span and the query's own column add 0.
    float dd[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
      float r;
      asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(fmaxf(v[k] + st.nx, 0.f)));
      dd[k] = r;
    }
    if (partial || (EXCL && cbase < st.ex_hi && cbase + 32 > st.ex_lo)) {
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const int c = cbase + 8 * (k >> 1) + 2 * sub + (k & 1);
        if (c >= st.col1 || (EXCL && c >= st.ex_lo && c < st.ex_hi)) dd[k] = 0.f;
      }
    }
    float s = ((dd[0] + dd[4]) + (dd[1] + dd[5])) + ((dd[2] + dd[6]) + (dd[3] + dd[7]));
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    st.dsum += (double)s;
  }
}

template <int MODE, bool EXCL, bool RESA, bool F16>
__global__ void __launch_bounds__(Layout<MODE, RESA>::kThreads, 1)
pair_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const PairArgs args) {
  using L = Layout<MODE, RESA>;
  constexpr int kConsumerWarps = L::kConsumerWarps;
  // 512 threads leave 128 registers each; warpgroup 0 (producer lane, drain warps) runs on 56 and hands the rest to
  // the consumers: 128 x 56 + 384 x 152 = 64 K
  constexpr bool kSplitRegs = L::kWgs == 3;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - raw);
  // streaming: stage s = A tile | B tile at base + s * kStageBytes.  RESA: the query tile's chunks at base, the train
  // ring behind them.
  const uint32_t b_ring = base + (RESA ? L::kResAChunks * L::kABytes : 0);
  const uint32_t bar0 = base + L::kFront;
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (kStages + s); };
  const uint32_t a_full = bar0 + 8u * (2 * kStages), a_empty = bar0 + 8u * (2 * kStages + 1);
  auto sched_full = [&](int s) { return bar0 + 8u * (2 * kStages + 2 + s); };
  auto sched_empty = [&](int s) { return bar0 + 8u * (2 * kStages + 4 + s); };
  auto ev_full = [&](int b) { return bar0 + 8u * (2 * kStages + 6 + b); };
  auto ev_empty = [&](int b) { return bar0 + 8u * (2 * kStages + 8 + b); };
  volatile int* sched_ring = reinterpret_cast<volatile int*>(smem + L::kFront + 8 * (2 * kStages + 10));
  static_assert(8 * (2 * kStages + 10) + 8 <= kBarBytes, "barrier block");
  EpiShared sh;   // MODE_NN candidate staging: drain warps (resident variant) / consumers (streaming variant)
  sh.cand_val = reinterpret_cast<float*>(smem + L::kFront + kBarBytes);
  sh.cand_col = reinterpret_cast<int*>(sh.cand_val + kCandSlots * L::kRows);
  sh.cand_mask = reinterpret_cast<uint32_t*>(sh.cand_col + kCandSlots * L::kRows);
  EvBuf<L::kRows>* evbuf = reinterpret_cast<EvBuf<L::kRows>*>(smem + L::kFront + kBarBytes + L::kCandBytes);

  // warp index through a shuffle: provably warp-uniform, so the compiler keeps the consumers' wgmma asynchronous
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  int tl_tile = 0;
#define TL(slot)                                                                              \
  do {                                                                                        \
    if (args.timeline && blockIdx.x == 0 && tl_tile < args.timeline_tiles)                    \
      args.timeline[(int64_t)tl_tile * 16 + (slot)] = clock64();                              \
  } while (0)
  auto global_ns = [] { long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; };

  if (threadIdx.x == 0) {
    if (args.cta_clock) args.cta_clock[blockIdx.x * 4] = global_ns();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < kStages; s++) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kConsumerWarps); }
    mbar_init(a_full, 1);
    mbar_init(a_empty, kConsumerWarps);
    for (int s = 0; s < 2; s++) { mbar_init(sched_full(s), 1); mbar_init(sched_empty(s), kConsumerWarps); }
    for (int b = 0; b < 2; b++) { mbar_init(ev_full(b), kConsumerWarps); mbar_init(ev_empty(b), kDrainWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int k16 = args.k16;
  const int nchunks = (k16 + 3) >> 2;

  if (warp < 4) {
    if (kSplitRegs) asm volatile("setmaxnreg.dec.sync.aligned.u32 56;" ::: "memory");
    if (warp == 0) {
      // ================= TMA producer + item hand-out =================
      if (lane == 0) {
        int stage = 0;
        uint32_t phase = 0, a_phase = 0;
        int a_row0 = -1;    // query tile in shared memory (RESA): consecutive items of the same tile reuse it
        long long n_tiles_done = 0, n_items_done = 0;
        int w_static = blockIdx.x;
        for (int k = 0;; k++) {
          int w, ntiles = 0;
          tip_work_item it;
          for (;;) {   // the next item with work: padding entries and items without live rows never reach the ring
            if (w_static < args.n_static) { w = w_static; w_static += gridDim.x; }
            else if (args.sched_counter) {
              w = args.n_static + atomicAdd(args.sched_counter, 1);
              if (w >= args.n_items) w = -1;
            } else w = -1;
            if (w < 0) break;
            it = args.items[w];
            ntiles = (it.col1 - it.col0 + BN - 1) / BN;
            if (ntiles > 0 && (!args.q_live_end || args.q_live_end[it.q_row0] > it.q_row0)) break;
          }
          const int slot = k & 1;
          mbar_wait(sched_empty(slot), ((uint32_t)(k >> 1) & 1u) ^ 1u);
          sched_ring[slot] = w;
          mbar_arrive(sched_full(slot));
          if (w < 0) break;
          n_tiles_done += ntiles; n_items_done++;
          if (RESA && it.q_row0 != a_row0) {
            // the consumers arrive once they start an item of another query tile, when every MMA on this one has
            // retired (first load: passes at once)
            mbar_wait(a_empty, a_phase ^ 1u);
            mbar_expect_tx(a_full, (uint32_t)nchunks * L::kABytes);
            for (int c = 0; c < nchunks; c++)
              tma_load_2d(base + (uint32_t)c * L::kABytes, &tmA, a_full, c * BK, it.q_row0);
            a_phase ^= 1u;
            a_row0 = it.q_row0;
          }
          for (int t = 0; t < ntiles; t++) {
            TL(8);
            for (int c = 0; c < nchunks; c++) {
              mbar_wait(empty_bar(stage), phase ^ 1u);
              if (RESA) {
                mbar_expect_tx(full_bar(stage), kBBytes);
                tma_load_2d(b_ring + (uint32_t)stage * kBBytes, &tmB, full_bar(stage), c * BK, it.col0 + t * BN);
              } else {
                mbar_expect_tx(full_bar(stage), kStageBytes);
                const uint32_t a_dst = base + stage * kStageBytes;
                tma_load_2d(a_dst, &tmA, full_bar(stage), c * BK, it.q_row0);
                tma_load_2d(a_dst + kABytes, &tmB, full_bar(stage), c * BK, it.col0 + t * BN);
              }
              if (++stage == kStages) { stage = 0; phase ^= 1u; }
            }
            TL(10);
            tl_tile++;
          }
        }
        if (args.cta_clock) {
          args.cta_clock[blockIdx.x * 4 + 2] = n_tiles_done;
          unsigned smid;
          asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
          args.cta_clock[blockIdx.x * 4 + 3] = n_items_done | ((long long)smid << 32);
        }
      }
      __syncwarp();
    } else {
      // ================= MODE_NN drain (resident variant): stage the consumers' events =================
      // Thread dt owns local rows dt and dt + 96 of the 192-row tile: their staging slots and counts.  Per row, events arrive in column
      // order.  An event is staged unless it is dead against the tighter of the record's thr and the row's thr after
      // its tile; with the slots full they are compacted against that threshold, and a chunk that still finds them
      // full of live chunks goes straight to the row's list.  The last tile of an item flushes the slots that
      // survive the row's final thr (read by the consumers after the item, from the shared running minimum).
      if (MODE == MODE_NN && RESA) {
        static_assert(!(MODE == MODE_NN && RESA) || L::kRows == 2 * 32 * kDrainWarps, "two rows per drain thread");
        const int dt = threadIdx.x - 32;
        int n_staged[2] = {0, 0};
        for (int qt = 0;; qt++) {
          const int b = qt & 1;
          mbar_wait(ev_full(b), (uint32_t)(qt >> 1) & 1u);
          const EvBuf<L::kRows>& e = evbuf[b];
          const int flags = e.flags;
          if (flags & kEvStop) break;
          const bool stamp = args.timeline && blockIdx.x == 0 && dt == 0 && qt < args.timeline_tiles;
          if (stamp) args.timeline[(int64_t)qt * 16 + 11] = clock64();
#pragma unroll
          for (int j = 0; j < 2; j++) {
            const int r = dt + 32 * kDrainWarps * j;
            const EvRow er = e.row[r];
            const int64_t row = (int64_t)e.q_row0 + r;
            for (int c = 0; c < kEvSlots; c++) {
              if (!((er.ev >> c) & 1)) continue;
              const EvRecord rc = e.rec[r * kEvSlots + c];
              const float thr = fminf(rc.thr, er.thr);
              if (rc.mn <= thr) stage_chunk<L::kRows>(args, sh, r, n_staged[j], row, rc.col, rc.mask, rc.mn, thr);
            }
            if (flags & kEvLast) {
              flush_row<L::kRows>(args, sh, r, n_staged[j], row, er.thr);
              n_staged[j] = 0;
            }
          }
          if (stamp) args.timeline[(int64_t)qt * 16 + 12] = clock64();
          __syncwarp();
          if (lane == 0) mbar_arrive(ev_empty(b));
        }
      }
    }
  } else {
    // ================= consumers: wgmma + register epilogue =================
    if (kSplitRegs) asm volatile("setmaxnreg.inc.sync.aligned.u32 152;" ::: "memory");
    const int cw = warp - 4;                    // consumer warp 0 .. kConsumerWarps - 1
    const int g = cw >> 2;                        // consumer warpgroup: query rows [64 g, 64 g + 64)
    const int sub = lane & 3;
    const int lead = lane & 28;                   // the quad's first lane
    // accumulator register i holds row 16 (warp % 4) + lane / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (lane % 4) + i % 2
    const int row_h0 = g * 64 + (cw & 3) * 16 + (lane >> 2);
    const float kInf = __int_as_float(0x7f800000);
    float acc[64];
    int stage = 0, rel_stage = 0;  // next stage to consume / to release
    uint32_t phase = 0, a_phase = 0;
    int a_row0 = -1;
    bool first_item = true;
    // Resident MODE_NN with 9 K16 steps (d = 128): each warp loads its rows of the query tile into registers once per
    // query tile, so most MMAs read only the train tile from shared memory.  With both operands there, an m64n128k16
    // reads 6 KB, and three warpgroups at the tensor rate would read ~94 of shared memory's 128 bytes per clock.  Only
    // the first kRegK steps fit in the consumers' 152 registers without spills; the last two come from shared memory.
    constexpr bool kRegA = MODE == MODE_NN && RESA && !F16;
    const bool reg_a = kRegA && k16 == kRsMaxK16;
    constexpr int kRegK = 7;
    uint32_t afr[kRegK][4];
    int tl_tile0 = 0;           // timeline index of the item's first tile
    int qt = 0;                 // MODE_NN: tiles handed to the drain so far (mailbox qt & 1)
    for (int k = 0;; k++) {
      const int slot = k & 1;
      mbar_wait<!kSplitRegs>(sched_full(slot), (uint32_t)(k >> 1) & 1u);
      const int w = sched_ring[slot];
      __syncwarp();
      if (lane == 0) mbar_arrive(sched_empty(slot));
      if (w < 0) {
        if (MODE == MODE_NN && RESA) {   // release the drain warps
          mbar_wait<!kSplitRegs>(ev_empty(qt & 1), ((uint32_t)(qt >> 1) & 1u) ^ 1u);
          if (cw == 0 && lane == 0) evbuf[qt & 1].flags = kEvStop;
          __syncwarp();
          if (lane == 0) mbar_arrive(ev_full(qt & 1));
        }
        break;
      }
      tip_work_item it = args.items[w];
      const int ntiles = (it.col1 - it.col0 + BN - 1) / BN;
      if (args.q_live_end) it.q_rows = min(it.q_rows, args.q_live_end[it.q_row0] - it.q_row0);
      // a warpgroup whose 64 rows all lie past the item's query rows issues no MMAs; with no valid row its epilogue
      // only hands empty mailbox entries to the drain, and it keeps its place in the ring and query-tile protocols
      const bool idle = L::kWgs == 3 && __shfl_sync(0xffffffffu, (int)(64 * g >= it.q_rows), 0);
      EpiState st[2];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int row_local = row_h0 + 8 * h;
        EpiState& s = st[h];
        s.valid_row = row_local < it.q_rows;
        s.row = (int64_t)it.q_row0 + row_local;
        s.nx = 0.f; s.e2 = 0.f; s.g = 0.f; s.best = kInf; s.thr = kInf; s.s_ref = kInf; s.n_staged = 0;
        s.run_max = -kInf; s.run_sum = 0.f; s.dsum = 0.0;
        s.col1 = it.col1;
        s.ex_lo = 0; s.ex_hi = 0;
        if (MODE == MODE_DSUM && s.valid_row) {
          s.nx = args.q_sqnorm[s.row];
          if (EXCL) { s.ex_lo = (int)s.row; s.ex_hi = (int)s.row + 1; }   // queries and columns: one matrix
        }
        uint32_t ref_bits = 0x7f800000u;
        if (MODE == MODE_NN && s.valid_row) {
          if (EXCL && (it.reserved & 1) && args.q_class) {
            const int cls = args.q_class[s.row];
            s.ex_lo = args.class_off[cls];
            s.ex_hi = args.class_off[cls + 1];
          }
          s.nx = args.q_sqnorm[s.row];
          const float r = sqrtf(s.nx) + args.rmax;
          s.e2 = args.q_err ? 2.f * (args.q_err[s.row] + args.t_err + 1.2e-7f * r) * 1.00001f : args.eps2 * r;
          s.g = args.gamma * r * r;
          if (sub == 0) ref_bits = ld_volatile_u32(args.row_min_bits + s.row);
        }
        if (MODE == MODE_NN) {
          // one read per quad, so that the four lanes of the row start from the same bound
          ref_bits = __shfl_sync(0xffffffffu, ref_bits, lead);
          s.s_ref = __uint_as_float(ref_bits);
          if (s.valid_row) s.thr = nn_threshold(s.s_ref, s.nx, s.e2, s.g);
        }
      }
      if (RESA && it.q_row0 != a_row0) {
        // another query tile: every MMA on the previous one has retired (the tile loop drains), hand its buffer back
        if (a_row0 >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(a_empty);
        }
        mbar_wait<!kSplitRegs>(a_full, a_phase);
        if (reg_a) {
          // ldmatrix.x4: lane l addresses row l % 16 of the warp's 16 rows, 8 K elements (16 bytes) at (l / 16) * 8;
          // 16-byte unit j of a 128-byte row r sits at unit j ^ (r % 8) (SWIZZLE_128B)
          const int r = g * 64 + (cw & 3) * 16 + (lane & 15);
#pragma unroll
          for (int s = 0; s < kRegK; s++) {
            const int j = (s & 3) * 2 + (lane >> 4);
            const uint32_t addr = base + (uint32_t)(s >> 2) * L::kABytes + (uint32_t)r * 128 + (uint32_t)((j ^ (r & 7)) << 4);
            asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                         : "=r"(afr[s][0]), "=r"(afr[s][1]), "=r"(afr[s][2]), "=r"(afr[s][3]) : "r"(addr) : "memory");
          }
        }
        a_phase ^= 1u;
        a_row0 = it.q_row0;
      }
      const bool dump_item = MODE == MODE_DUMP && first_item && blockIdx.x == 0;
      first_item = false;

#define TLT(t, slot)                                                                                      \
  do {                                                                                                    \
    if (cw == 0 && lane == 0 && args.timeline && blockIdx.x == 0 && tl_tile0 + (t) < args.timeline_tiles) \
      args.timeline[(int64_t)(tl_tile0 + (t)) * 16 + (slot)] = clock64();                                 \
  } while (0)

      // Resident query tile: issue the MMAs of tile t into `a`, one commit group for the whole tile.
      auto issue_tile = [&](float (&a)[64], int t) {
        TLT(t, 0);
        acc_fence(a);
        if (idle) {   // the tile's stages are released with everybody else's
          for (int c = 0; c < nchunks; c++) {
            mbar_wait<!kSplitRegs>(full_bar(stage), phase);
            if (++stage == kStages) { stage = 0; phase ^= 1u; }
          }
          return;
        }
        if (kRegA && reg_a) {
#pragma unroll
          for (int c = 0; c < (kRsMaxK16 + 3) / 4; c++) {
            mbar_wait<!kSplitRegs>(full_bar(stage), phase);
            const uint64_t bdesc = smem_desc(b_ring + (uint32_t)stage * kBBytes);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4 && 4 * c + kk < kRsMaxK16; kk++) {
              if (4 * c + kk < kRegK)
                wgmma_m64n128k16_rs(a, afr[4 * c + kk], bdesc + 2u * kk, (c | kk) ? 1u : 0u);
              else
                wgmma_m64n128k16<F16>(a, smem_desc(base + (uint32_t)c * L::kABytes + (uint32_t)g * 64 * 128) + 2u * kk,
                                      bdesc + 2u * kk, 1u);
            }
            if (++stage == kStages) { stage = 0; phase ^= 1u; }
          }
        } else {
          for (int c = 0; c < nchunks; c++) {
            mbar_wait<!kSplitRegs>(full_bar(stage), phase);
            const uint32_t a_addr = base + (uint32_t)c * L::kABytes + (uint32_t)g * 64 * 128;
            const uint32_t b_addr = b_ring + (uint32_t)stage * kBBytes;
            const uint64_t adesc = smem_desc(a_addr), bdesc = smem_desc(b_addr);
            const int nm = min(4, k16 - 4 * c);
            wgmma_fence();
            wgmma_m64n128k16<F16>(a, adesc, bdesc, c > 0 ? 1u : 0u);
            for (int kk = 1; kk < nm; kk++) wgmma_m64n128k16<F16>(a, adesc + 2u * kk, bdesc + 2u * kk, 1u);
            if (++stage == kStages) { stage = 0; phase ^= 1u; }
          }
        }
        wgmma_commit();
        acc_fence(a);
      };
      // Tile t in `a` has retired (the caller waited): release its stages.
      auto retire_tile = [&](float (&a)[64], int t) {
        acc_fence(a);
        __syncwarp();
        for (int c = 0; c < nchunks; c++) {
          if (lane == 0) mbar_arrive(empty_bar(rel_stage));
          if (++rel_stage == kStages) rel_stage = 0;
        }
        TLT(t, 1);
      };
      // The shared running minimum of the rows, read before the wait on the MMAs and used after the epilogue.
      auto load_seen = [&](uint32_t (&sb)[2]) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
          sb[h] = 0x7f800000u;
          if (MODE == MODE_NN && st[h].valid_row && sub == 0) sb[h] = ld_volatile_u32(args.row_min_bits + st[h].row);
        }
      };
      auto epilogue = [&](float (&a)[64], int t, const uint32_t (&sb)[2]) {
        const int col_base = it.col0 + t * BN;
        const bool partial = col_base + BN > it.col1;
        const bool last = t == ntiles - 1;
        EvBuf<L::kRows>* eb = evbuf + (qt & 1);
        int ev[2] = {0, 0};
        // a free mailbox (convergent: the drain released it two tiles ago)
        if (MODE == MODE_NN) mbar_wait<!kSplitRegs>(ev_empty(qt & 1), ((uint32_t)(qt >> 1) & 1u) ^ 1u);
        TLT(t, 2);
        if (MODE == MODE_DUMP) {
          if (dump_item && t < 2) {     // the first 128 rows x 256 columns of the first item
#pragma unroll
            for (int i = 0; i < 64; i++) {
              const int col = t * BN + 8 * (i >> 2) + 2 * sub + (i & 1);
              args.dump[(int64_t)(row_h0 + 8 * ((i >> 1) & 1)) * 256 + col] = a[i];
            }
          }
        } else if (MODE == MODE_NN) {
          // One pass per row and tile.  Value k (0..7) of chunk c of row h sits in a[16 c + 4 (k / 2) + 2 h + k % 2],
          // column col_base + 32 c + 8 (k / 2) + 2 sub + k % 2.  cm: this lane's minimum of each chunk, per row.
          auto ai = [](int h, int c, int k) { return 16 * c + 4 * (k >> 1) + 2 * h + (k & 1); };
          float cm[2][kEvSlots];
#pragma unroll
          for (int h = 0; h < 2; h++)
#pragma unroll
            for (int c = 0; c < kEvSlots; c++)
              cm[h][c] = fminf(fminf(fminf(a[ai(h, c, 0)], a[ai(h, c, 1)]), fminf(a[ai(h, c, 2)], a[ai(h, c, 3)])),
                               fminf(fminf(a[ai(h, c, 4)], a[ai(h, c, 5)]), fminf(a[ai(h, c, 6)], a[ai(h, c, 7)])));
          // thr is the same in the four lanes of a quad, so the quad's minimum lies inside the window exactly when
          // some lane's own minimum does: a tile without any such value changes no state and skips the pass.
          // Masking (partial tile, excluded class) only raises values, so the unmasked minimum decides safely.
          bool in[2];
#pragma unroll
          for (int h = 0; h < 2; h++)
            in[h] = st[h].valid_row && fminf(fminf(cm[h][0], cm[h][1]), fminf(cm[h][2], cm[h][3])) <= st[h].thr;
          const bool any = __any_sync(0xffffffffu, in[0] || in[1]);
          // timeline slot 3: bit cw = consumer warp cw took the pass on this tile
          if (any && lane == 0 && args.timeline && blockIdx.x == 0 && tl_tile0 + t < args.timeline_tiles)
            atomicOr(reinterpret_cast<unsigned long long*>(args.timeline) + (int64_t)(tl_tile0 + t) * 16 + 3,
                     1ull << cw);
          if (any) {
            // rare: the tile runs past the span, or some row of the warp must ignore train rows inside it.  One
            // warp-uniform test per tile, so a full tile without excluded rows pays no per-chunk branch.
            bool masked = partial;
            if (EXCL)
              masked = __any_sync(0xffffffffu, partial || (col_base < st[0].ex_hi && col_base + BN > st[0].ex_lo) ||
                                                    (col_base < st[1].ex_hi && col_base + BN > st[1].ex_lo));
            if (masked) {
#pragma unroll
              for (int h = 0; h < 2; h++)
#pragma unroll
                for (int c = 0; c < kEvSlots; c++) {
                  const int cbase = col_base + 32 * c;
                  if (partial || (EXCL && cbase < st[h].ex_hi && cbase + 32 > st[h].ex_lo)) {
                    // The accumulator is free to overwrite: the next tile's first MMA does not accumulate.
                    float mn = kInf;
#pragma unroll
                    for (int k = 0; k < 8; k++) {
                      const int col = cbase + 8 * (k >> 1) + 2 * sub + (k & 1);
                      if (col >= st[h].col1 || (EXCL && col >= st[h].ex_lo && col < st[h].ex_hi)) a[ai(h, c, k)] = kInf;
                      mn = fminf(mn, a[ai(h, c, k)]);
                    }
                    cm[h][c] = mn;
                  }
                }
            }
            // the quad's minima of all eight chunks, one batch of independent whole-warp shuffles
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
              for (int c = 0; c < kEvSlots; c++) cm[h][c] = fminf(cm[h][c], __shfl_xor_sync(0xffffffffu, cm[h][c], 1));
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
              for (int c = 0; c < kEvSlots; c++) cm[h][c] = fminf(cm[h][c], __shfl_xor_sync(0xffffffffu, cm[h][c], 2));
            // the row's running minimum and threshold move once per tile, to the tile's minimum (the same state a
            // chunk-by-chunk update reaches: that minimum is inside every threshold it would pass through)
#pragma unroll
            for (int h = 0; h < 2; h++) {
              EpiState& s = st[h];
              const float mn = fminf(fminf(cm[h][0], cm[h][1]), fminf(cm[h][2], cm[h][3]));
              if (s.valid_row && mn <= s.thr && mn < s.best) {
                s.best = mn;
                s.s_ref = fminf(s.s_ref, fmaxf(s.best + s.nx, 0.f));
                s.thr = nn_threshold(s.s_ref, s.nx, s.e2, s.g);
              }
            }
            // events: the chunks inside the row's threshold after the tile (the one the drain applies), each with
            // the exact mask of its columns inside it, so the re-rank touches only rows inside the window.  A row has
            // about one event chunk in a tile with an event, so the mask of (row half h, chunk c) is built only when
            // some row of the warp has an event there: the branch is warp-uniform, because shuffles inside a
            // divergent branch make ptxas serialise the wgmma.
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
              for (int c = 0; c < kEvSlots; c++) {
                const bool event = st[h].valid_row && cm[h][c] <= st[h].thr && cm[h][c] < kInf;
                if (__any_sync(0xffffffffu, event)) {
                  uint32_t mk = 0;
#pragma unroll
                  for (int k = 0; k < 8; k++)
                    mk |= (a[ai(h, c, k)] <= st[h].thr) ? (1u << (8 * (k >> 1) + 2 * sub + (k & 1))) : 0u;
                  mk |= __shfl_xor_sync(0xffffffffu, mk, 1);
                  mk |= __shfl_xor_sync(0xffffffffu, mk, 2);
                  if (event) {
                    ev[h] |= 1 << c;
                    if (sub == 0) eb->rec[(row_h0 + 8 * h) * kEvSlots + c] = EvRecord{col_base + 32 * c, mk, cm[h][c], st[h].thr};
                  }
                }
              }
          }
        } else {
#pragma unroll
          for (int c = 0; c < BN / 32; c++) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
              float v[8];
#pragma unroll
              for (int jj = 0; jj < 4; jj++) {
                v[2 * jj] = a[4 * (4 * c + jj) + 2 * h];
                v[2 * jj + 1] = a[4 * (4 * c + jj) + 2 * h + 1];
              }
              epi_chunk<MODE, EXCL>(args, st[h], sh, v, col_base + 32 * c, sub, partial, row_h0 + 8 * h);
            }
          }
        }
        if (MODE == MODE_NN) {
#pragma unroll
          for (int h = 0; h < 2; h++) {
            EpiState& s = st[h];
            const float seen = __uint_as_float(__shfl_sync(0xffffffffu, sb[h], lead));
            if (!s.valid_row) continue;
            // share the running minimum across everybody scanning other columns for the same query
            const float mine = fmaxf(s.best + s.nx, 0.f);
            if (sub == 0 && mine < seen) atomicMin(args.row_min_bits + s.row, __float_as_uint(mine));
            if (seen < s.s_ref) {
              s.s_ref = seen;
              s.thr = nn_threshold(s.s_ref, s.nx, s.e2, s.g);
            }
            if (last && sub == 0) {
              // other CTAs have been scanning other columns of this query meanwhile: the drain flushes only the
              // chunks that survive the best bound known by now (the quad's other lanes are done with this row)
              const float now = __uint_as_float(ld_volatile_u32(args.row_min_bits + s.row));
              if (now < s.s_ref) {
                s.s_ref = now;
                s.thr = nn_threshold(s.s_ref, s.nx, s.e2, s.g);
              }
            }
          }
          // hand the tile's events to the drain: per row its thr after the tile and the chunks with an event
#pragma unroll
          for (int h = 0; h < 2; h++)
            if (sub == 0) eb->row[row_h0 + 8 * h] = EvRow{st[h].thr, ev[h]};
          if (cw == 0 && lane == 0) { eb->q_row0 = it.q_row0; eb->flags = last ? kEvLast : 0; }
          __syncwarp();
          if (lane == 0) mbar_arrive(ev_full(qt & 1));
          qt++;
        }
        TLT(t, 7);
      };

      if (RESA) {
        for (int t = 0; t < ntiles; t++) {
          uint32_t sb[2];
          issue_tile(acc, t);
          load_seen(sb);
          wgmma_wait_all();
          retire_tile(acc, t);
          epilogue(acc, t, sb);
        }
      } else {
        // streaming (wide rows, many chunks per tile): the MMA loop dominates; each chunk is retired before the next
        for (int t = 0; t < ntiles; t++) {
          TLT(t, 0);
          for (int c = 0; c < nchunks; c++) {
            mbar_wait<!kSplitRegs>(full_bar(stage), phase);
            const uint32_t a_addr = base + stage * kStageBytes + (uint32_t)g * 64 * 128;
            const uint32_t b_addr = base + stage * kStageBytes + kABytes;
            const uint64_t adesc = smem_desc(a_addr), bdesc = smem_desc(b_addr);
            const int nm = min(4, k16 - 4 * c);
            wgmma_fence();
            wgmma_m64n128k16<F16>(acc, adesc, bdesc, c > 0 ? 1u : 0u);
            for (int kk = 1; kk < nm; kk++) wgmma_m64n128k16<F16>(acc, adesc + 2u * kk, bdesc + 2u * kk, 1u);
            wgmma_commit();
            wgmma_wait_all();
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(stage));
            if (++stage == kStages) { stage = 0; phase ^= 1u; }
          }
          TLT(t, 1);
          const int col_base = it.col0 + t * BN;
          const bool partial = col_base + BN > it.col1;
          float seen[2];
#pragma unroll
          for (int h = 0; h < 2; h++) {
            uint32_t b = 0x7f800000u;
            if (MODE == MODE_NN && st[h].valid_row && sub == 0) b = ld_volatile_u32(args.row_min_bits + st[h].row);
            if (MODE == MODE_NN) b = __shfl_sync(0xffffffffu, b, lead);
            seen[h] = __uint_as_float(b);
          }
          if (MODE == MODE_DUMP) {
            if (dump_item && t < 2) {     // the first 128 rows x 256 columns of the first item
#pragma unroll
              for (int i = 0; i < 64; i++) {
                const int col = t * BN + 8 * (i >> 2) + 2 * sub + (i & 1);
                args.dump[(int64_t)(row_h0 + 8 * ((i >> 1) & 1)) * 256 + col] = acc[i];
              }
            }
          } else {
#pragma unroll
            for (int c = 0; c < BN / 32; c++) {
#pragma unroll
              for (int h = 0; h < 2; h++) {
                float v[8];
#pragma unroll
                for (int jj = 0; jj < 4; jj++) {
                  v[2 * jj] = acc[4 * (4 * c + jj) + 2 * h];
                  v[2 * jj + 1] = acc[4 * (4 * c + jj) + 2 * h + 1];
                }
                epi_chunk<MODE, EXCL>(args, st[h], sh, v, col_base + 32 * c, sub, partial, row_h0 + 8 * h);
              }
            }
          }
          if (MODE == MODE_NN) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
              EpiState& s = st[h];
              if (!s.valid_row) continue;
              // share the running minimum across everybody scanning other columns for the same query
              const float mine = fmaxf(s.best + s.nx, 0.f);
              if (sub == 0 && mine < seen[h]) atomicMin(args.row_min_bits + s.row, __float_as_uint(mine));
              if (seen[h] < s.s_ref) {
                s.s_ref = seen[h];
                s.thr = nn_threshold(s.s_ref, s.nx, s.e2, s.g);
              }
            }
          }
          TLT(t, 7);
        }
      }
      tl_tile0 += ntiles;
#undef TLT

#pragma unroll
      for (int h = 0; h < 2; h++) {
        EpiState& s = st[h];
        if (!s.valid_row || sub != 0) continue;
        if (MODE == MODE_NN && !RESA) {
          // other CTAs have been scanning other columns of this query meanwhile: only flush the groups that
          // survive the best bound known by now
          const float seen = __uint_as_float(ld_volatile_u32(args.row_min_bits + s.row));
          if (seen < s.s_ref) {
            s.s_ref = seen;
            s.thr = nn_threshold(s.s_ref, s.nx, s.e2, s.g);
          }
          flush_row<BM>(args, sh, row_h0 + 8 * h, s.n_staged, s.row, s.thr);
        } else if (MODE == MODE_LSE) {
          args.part_max[(int64_t)it.slot * args.m + s.row] = s.run_max;
          args.part_sum[(int64_t)it.slot * args.m + s.row] = s.run_sum;
        } else if (MODE == MODE_DSUM) {
          args.part_sum[(int64_t)it.slot * args.m + s.row] = (float)s.dsum;
        }
      }
      __syncwarp();
    }
  }
#undef TL

  __syncthreads();
  if (args.cta_clock && threadIdx.x == 0) args.cta_clock[blockIdx.x * 4 + 1] = global_ns();
  if (args.sched_counter && threadIdx.x == 0) {
    // every CTA has drawn its last pool index by now: the last one out re-arms the counters
    if (atomicAdd(args.sched_counter + 1, 1) == (int)gridDim.x - 1) {
      args.sched_counter[0] = 0;
      args.sched_counter[1] = 0;
    }
  }
}

// ---- host side -----------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (PFN_cuTensorMapEncodeTiled_v12000)p;
  }
  return fn;
}

static int make_map(CUtensorMap* map, const void* basep, int64_t rows, int64_t pitch, int box_rows) {
  auto fn = get_encode();
  if (!fn) { set_error("cuTensorMapEncodeTiled not available from the driver"); return TIP_ERR_CUDA; }
  cuuint64_t gdim[2] = {(cuuint64_t)pitch, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)pitch * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(basep), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return TIP_ERR_CUDA; }
  return TIP_OK;
}

static int check_device() {
  static int ok = -1;
  if (ok < 0) {
    int dev = 0, major = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) {
      set_error("no CUDA device");
      return TIP_ERR_CUDA;
    }
    ok = (major == 9) ? 1 : 0;
  }
  if (!ok) { set_error("libb200tip tensor-core kernels need an sm_90 device"); return TIP_ERR_UNSUPPORTED; }
  return TIP_OK;
}

// resa: the query tile stays resident in shared memory for each work item (needs <= Layout::kResAChunks K chunks)
template <int MODE, bool EXCL = false, bool F16 = false>
static int launch_pair(const void* q_pack, int64_t m, const void* t_pack, int64_t n, int64_t pitch, PairArgs args,
                       bool resa, cudaStream_t st) {
  using LS = Layout<MODE, false>;
  using LR = Layout<MODE, true>;
  int rc = check_device();
  if (rc != TIP_OK) return rc;
  TIP_REQUIRE(((uintptr_t)q_pack & 127) == 0 && ((uintptr_t)t_pack & 127) == 0, "packed operands must be 128-byte aligned");
  TIP_REQUIRE(pitch % 64 == 0 && args.k16 >= 1 && args.k16 * 16 <= pitch, "pitch");
  TIP_REQUIRE(m >= 1 && n >= 1 && m < (1LL << 31) && n < (1LL << 31), "shape");
  TIP_REQUIRE(!resa || (args.k16 + 3) / 4 <= LR::kResAChunks, "packed width too large for the resident-query kernel");
  CUtensorMap ma, mb;
  rc = make_map(&ma, q_pack, m, pitch, resa ? LR::kRows : LS::kRows);
  if (rc != TIP_OK) return rc;
  rc = make_map(&mb, t_pack, n, pitch, BN);
  if (rc != TIP_OK) return rc;
  static bool attr_set = false;   // one flag per template instantiation
  if (!attr_set) {
    TIP_CHECK_CUDA(cudaFuncSetAttribute(pair_kernel<MODE, EXCL, false, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, LS::kSmemBytes));
    TIP_CHECK_CUDA(cudaFuncSetAttribute(pair_kernel<MODE, EXCL, true, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, LR::kSmemBytes));
    attr_set = true;
  }
  const int grid = std::min(args.n_items, sm_count());
  if (resa)
    pair_kernel<MODE, EXCL, true, F16><<<grid, LR::kThreads, LR::kSmemBytes, st>>>(ma, mb, args);
  else
    pair_kernel<MODE, EXCL, false, F16><<<grid, LS::kThreads, LS::kSmemBytes, st>>>(ma, mb, args);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

static int k16_of(int64_t d, int segments) {
  const int64_t d16 = (d + 15) & ~(int64_t)15;
  return (int)((segments * d16 + 16) / 16);
}

}  // namespace tip

using namespace tip;

static long long* g_timeline = nullptr;
static int g_timeline_tiles = 0;
static long long* g_cta_clock = nullptr;
extern "C" int tip_debug_timeline(long long* buf, int32_t tiles) {
  g_timeline = buf;
  g_timeline_tiles = tiles;
  return TIP_OK;
}
extern "C" int tip_debug_cta_clock(long long* buf) {
  g_cta_clock = buf;
  return TIP_OK;
}

extern "C" int tip_nn_filter_live(const void* q_pack, const float* q_sqnorm, int64_t m, const void* t_pack, int64_t n,
                                  int64_t d, int64_t pitch, const tip_work_item* items, int32_t n_items,
                                  const int32_t* q_class, const int32_t* class_off, float t_rmax,
                                  const float* q_rounderr, float t_errmax, uint32_t* row_min_bits, int32_t* cand_idx,
                                  int32_t* cand_cnt, int32_t cap, int32_t n_static, int32_t* sched_counter,
                                  const int32_t* q_live_end, void* stream) {
  TIP_REQUIRE(q_pack && q_sqnorm && t_pack && items && row_min_bits && cand_idx && cand_cnt, "null pointer");
  TIP_REQUIRE(cap >= 1 && n_items >= 0, "cap / n_items");
  TIP_REQUIRE(pitch == tip_pair_pitch(d, 1), "pitch does not match tip_pair_pitch(d, 1)");
  if (n_items == 0) return TIP_OK;
  PairArgs a{};
  a.items = items; a.n_items = n_items; a.k16 = k16_of(d, 1); a.m = m;
  TIP_REQUIRE(n_static >= 0 && n_static <= n_items, "n_static");
  TIP_REQUIRE(sched_counter != nullptr || n_static == n_items, "a pool of dynamic items needs sched_counter");
  a.n_static = n_static; a.sched_counter = n_static < n_items ? sched_counter : nullptr;
  a.q_sqnorm = q_sqnorm; a.rmax = t_rmax;
  a.q_err = q_rounderr; a.t_err = t_errmax;
  TIP_REQUIRE(!q_rounderr || t_errmax >= 0.f, "t_errmax");
  a.q_class = q_class; a.class_off = class_off;
  // eps' = (2^-9 + 2^-23)/(1 - that): bf16 rounding of the centred traces (triangle inequality);
  // gamma: fp32 accumulation over K products + norm rounding, assuming nothing better than
  // truncating adds inside the tensor core.
  a.eps2 = 2.0f * 1.96e-3f;
  a.gamma = (float)(a.k16 * 16 + 16) * 1.1920929e-7f;
  a.row_min_bits = row_min_bits; a.cand_idx = cand_idx; a.cand_cnt = cand_cnt; a.cap = cap;
  a.timeline = g_timeline; a.timeline_tiles = g_timeline_tiles;
  a.cta_clock = g_cta_clock;
  a.q_live_end = q_live_end;
  const bool excl = q_class != nullptr && class_off != nullptr;   // per-query own-class masking compiled in only then
  const bool resa = a.k16 <= kRsMaxK16;
  return excl ? launch_pair<MODE_NN, true>(q_pack, m, t_pack, n, pitch, a, resa, (cudaStream_t)stream)
              : launch_pair<MODE_NN, false>(q_pack, m, t_pack, n, pitch, a, resa, (cudaStream_t)stream);
}

extern "C" int tip_nn_filter(const void* q_pack, const float* q_sqnorm, int64_t m, const void* t_pack, int64_t n,
                             int64_t d, int64_t pitch, const tip_work_item* items, int32_t n_items,
                             const int32_t* q_class, const int32_t* class_off, float t_rmax,
                             const float* q_rounderr, float t_errmax, uint32_t* row_min_bits, int32_t* cand_idx,
                             int32_t* cand_cnt, int32_t cap, int32_t n_static, int32_t* sched_counter,
                             void* stream) {
  return tip_nn_filter_live(q_pack, q_sqnorm, m, t_pack, n, d, pitch, items, n_items, q_class, class_off, t_rmax,
                            q_rounderr, t_errmax, row_min_bits, cand_idx, cand_cnt, cap, n_static, sched_counter,
                            nullptr, stream);
}

extern "C" int tip_nn_filter_tile(int64_t d, int32_t* q_rows, int32_t* t_rows) {
  TIP_REQUIRE(d >= 1 && q_rows && t_rows, "arguments");
  *q_rows = tip_nn_filter_kind(d) == 1 ? Layout<MODE_NN, true>::kRows : Layout<MODE_NN, false>::kRows;
  *t_rows = BN;
  return TIP_OK;
}

extern "C" int tip_nn_filter_kind(int64_t d) {
  if (d < 1) return -1;
  return k16_of(d, 1) <= kRsMaxK16 ? 1 : 0;
}

extern "C" int tip_kde_tile_rows(void) { return BM; }
extern "C" int tip_kde_slot_parts(void) { return 1; }

extern "C" int tip_kde_lse(const void* q_pack, int64_t m, const void* t_pack, int64_t n, int64_t d, int64_t pitch,
                           const tip_work_item* items, int32_t n_items, float* part_max, float* part_sum,
                           void* stream) {
  TIP_REQUIRE(q_pack && t_pack && items && part_max && part_sum, "null pointer");
  TIP_REQUIRE(pitch == tip_pair_pitch(d, 3), "pitch does not match tip_pair_pitch(d, 3)");
  if (n_items == 0) return TIP_OK;
  PairArgs a{};
  a.items = items; a.n_items = n_items; a.n_static = n_items; a.k16 = k16_of(d, 3); a.m = m;
  a.part_max = part_max; a.part_sum = part_sum;
  const bool resa = (a.k16 + 3) / 4 <= kResAChunks;
  return launch_pair<MODE_LSE>(q_pack, m, t_pack, n, pitch, a, resa, (cudaStream_t)stream);
}

extern "C" int tip_kde_lse_f16(const void* q_pack, int64_t m, const void* t_pack, int64_t n, int64_t d, int64_t pitch,
                               const tip_work_item* items, int32_t n_items, float* part_max, float* part_sum,
                               void* stream) {
  TIP_REQUIRE(q_pack && t_pack && items && part_max && part_sum, "null pointer");
  TIP_REQUIRE(pitch == tip_pair_pitch(d, 1), "pitch does not match tip_pair_pitch(d, 1)");
  if (n_items == 0) return TIP_OK;
  PairArgs a{};
  a.items = items; a.n_items = n_items; a.n_static = n_items; a.k16 = k16_of(d, 1); a.m = m;
  a.part_max = part_max; a.part_sum = part_sum;
  const bool resa = (a.k16 + 3) / 4 <= kResAChunks;
  return launch_pair<MODE_LSE, false, true>(q_pack, m, t_pack, n, pitch, a, resa, (cudaStream_t)stream);
}

extern "C" int tip_sil_dsum(const void* q_pack, const void* t_pack, const float* sqnorm, int64_t n, int64_t d,
                            int64_t pitch, const tip_work_item* items, int32_t n_items, float* part_sum, void* stream) {
  TIP_REQUIRE(q_pack && t_pack && sqnorm && items && part_sum, "null pointer");
  TIP_REQUIRE(pitch == tip_pair_pitch(d, 3), "pitch does not match tip_pair_pitch(d, 3)");
  if (n_items == 0) return TIP_OK;
  PairArgs a{};
  a.items = items; a.n_items = n_items; a.n_static = n_items; a.k16 = k16_of(d, 3); a.m = n;
  a.q_sqnorm = sqnorm; a.part_sum = part_sum;
  const bool resa = (a.k16 + 3) / 4 <= kResAChunks;
  return launch_pair<MODE_DSUM, true>(q_pack, n, t_pack, n, pitch, a, resa, (cudaStream_t)stream);
}

extern "C" int tip_pair_probe(const void* q_pack, int64_t m, const void* t_pack, int64_t n, int64_t d, int segments,
                              int64_t pitch, int variant, float* out, void* stream) {
  TIP_REQUIRE(q_pack && t_pack && out, "null pointer");
  TIP_REQUIRE(pitch == tip_pair_pitch(d, segments), "pitch does not match tip_pair_pitch");
  TIP_REQUIRE(variant >= 0 && variant <= 2, "variant: 0 auto, 1 streaming, 2 resident");
  static tip_work_item* d_item = nullptr;
  if (!d_item) TIP_CHECK_CUDA(cudaMalloc(&d_item, sizeof(tip_work_item)));
  const int k16 = k16_of(d, segments);
  const bool resa = variant == 2 || (variant == 0 && k16 <= kRsMaxK16);
  tip_work_item h{0, (int32_t)std::min<int64_t>(m, BM), 0, (int32_t)std::min<int64_t>(n, 256), 0, 0};
  TIP_CHECK_CUDA(cudaMemcpyAsync(d_item, &h, sizeof(h), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  PairArgs a{};
  a.items = d_item; a.n_items = 1; a.n_static = 1; a.k16 = k16; a.m = m; a.dump = out;
  return launch_pair<MODE_DUMP>(q_pack, m, t_pack, n, pitch, a, resa, (cudaStream_t)stream);
}
