// levenshtein.cu — all-pairs unit-cost Levenshtein distances (insert, delete, substitute) of two word blocks, the
// quadratic step of the reference's TextCorruptor._calculate_distances (src/core/text_corruptor.py:282-309), which
// makes one polyleven.levenshtein call per ordered pair of dictionary words.
//
// Words arrive as dense int32 code-point ids (one id per Unicode code point, as Python's str counts them),
// concatenated, with int32 offsets.  out[i * nb + j] (uint8, int64 indexing) = distance(a_i, b_j); every word is at
// most 255 code points (checked by the caller and here), so every distance fits.
//
// Algorithm: Myers' bit-parallel edit distance in Hyyro's formulation.  A block is kCols column words ("patterns",
// one per thread) x kRows row words ("texts").  Each thread keeps its pattern's match masks in shared memory,
// Peq[c][thread] = bit k set iff pattern[k] == c, for the kAlpha smallest ids (the caller numbers code points by
// descending frequency, so these are the common ones); the table is private to its thread's column, so building
// it needs no barrier.  The block then walks its row words in order: the text is the same for every thread, so
// the character loop has one trip count for the whole warp and the text loads are broadcasts.  Per text character
// the vertical deltas (Pv, Mv) advance with ~17 integer operations and the score at the pattern's last row moves
// by the horizontal delta there.  Exact for every input:
//   - a character with id >= kAlpha gets its mask by comparing the pattern's code points directly;
//   - a pattern longer than 64 code points runs the blocked variant (up to four 64-bit blocks, the horizontal
//     delta carried from block to block), with its masks built by direct comparison; such words are rare;
//   - an empty pattern gives the text's length, an empty text the pattern's length.
//
// symmetric != 0 (a and b are the same block): the distance is symmetric, so only tiles on or above the diagonal
// run, each pair j >= i is computed once, and the block writes out[i][j] directly and out[j][i] through a staged
// transpose (32 rows at a time), so both writes are coalesced.
#include "common.cuh"

namespace tip {

constexpr int kLevCols = 128;        // pattern words per block, one per thread
constexpr int kLevRows = 128;        // text words per block (square tiles: the diagonal is tile-aligned)
constexpr int kLevChunk = 32;        // text rows staged per transposed write
constexpr int kLevAlpha = 64;        // ids with a shared-memory mask row
constexpr int kLevStagePitch = kLevCols + 4;   // 33 words: the transposed reads hit 32 distinct banks
constexpr int kLevMaxLen = 255;
constexpr size_t kLevSmem = sizeof(uint64_t) * kLevAlpha * kLevCols + kLevChunk * kLevStagePitch;

// One step of the bit-parallel recurrence for a 64-row block: hin / return value = the horizontal delta entering
// at the block's top / leaving at row `high` (-1, 0, +1).
__device__ __forceinline__ int lev_step(uint64_t& pv, uint64_t& mv, uint64_t eq, int hin, uint64_t high) {
  const uint64_t xv = eq | mv;
  if (hin < 0) eq |= 1ull;
  const uint64_t xh = (((eq & pv) + pv) ^ pv) | eq;
  uint64_t ph = mv | ~(xh | pv);
  uint64_t mh = pv & xh;
  const int hout = (ph & high) ? 1 : ((mh & high) ? -1 : 0);
  ph <<= 1;
  mh <<= 1;
  if (hin < 0) mh |= 1ull;
  else if (hin > 0) ph |= 1ull;
  pv = mh | ~(xv | ph);
  mv = ph & xv;
  return hout;
}

__device__ __forceinline__ uint64_t lev_match(const int32_t* __restrict__ p, int k0, int k1, int32_t c) {
  uint64_t eq = 0;
  for (int k = k0; k < k1; k++) eq |= (uint64_t)(__ldg(p + k) == c) << (k - k0);
  return eq;
}

// Patterns of 65..255 code points: the blocked recurrence, masks by direct comparison.
__device__ __noinline__ int lev_long(const int32_t* __restrict__ p, int m, const int32_t* __restrict__ t, int n) {
  uint64_t pv[4] = {~0ull, ~0ull, ~0ull, ~0ull}, mv[4] = {0, 0, 0, 0};
  const int blocks = (m + 63) >> 6;
  const uint64_t last = 1ull << ((m - 1) & 63);
  int score = m;
  for (int x = 0; x < n; x++) {
    const int32_t c = __ldg(t + x);
    int h = 1;                                         // row 0 of the DP grows by one per text character
#pragma unroll
    for (int b = 0; b < 4; b++) {
      if (b < blocks) {
        const uint64_t eq = lev_match(p, b * 64, min(m, b * 64 + 64), c);
        h = lev_step(pv[b], mv[b], eq, h, b == blocks - 1 ? last : (1ull << 63));
      }
    }
    score += h;
  }
  return score;
}

__global__ void __launch_bounds__(kLevCols) lev_kernel(const int32_t* __restrict__ a_ids, const int32_t* __restrict__ a_off,
                                                       int64_t na, const int32_t* __restrict__ b_ids,
                                                       const int32_t* __restrict__ b_off, int64_t nb, int symmetric,
                                                       uint8_t* __restrict__ out) {
  const int64_t i_base = (int64_t)blockIdx.y * kLevRows, j_base = (int64_t)blockIdx.x * kLevCols;
  if (symmetric && j_base + kLevCols <= i_base) return;           // strictly below the diagonal: mirrored
  extern __shared__ __align__(16) unsigned char lev_smem[];
  uint64_t(*peq)[kLevCols] = reinterpret_cast<uint64_t(*)[kLevCols]>(lev_smem);
  uint8_t* stage = lev_smem + sizeof(uint64_t) * kLevAlpha * kLevCols;

  const int tid = threadIdx.x;
  const int64_t j = j_base + tid;
  const bool live = j < nb;
  const int32_t* p = b_ids;
  int m = 0;
  if (live) {
    p = b_ids + b_off[j];
    m = b_off[j + 1] - b_off[j];
  }
  const bool fast = m <= 64;
  if (fast) {
#pragma unroll 8
    for (int c = 0; c < kLevAlpha; c++) peq[c][tid] = 0;
    for (int k = 0; k < m; k++) {
      const int32_t c = __ldg(p + k);
      if (c < kLevAlpha) peq[c][tid] |= 1ull << k;
    }
  }
  const uint64_t last = m > 0 ? 1ull << ((m - 1) & 63) : 0;

  const int64_t i_end = min(na, i_base + kLevRows);
  for (int64_t i0 = i_base; i0 < i_end; i0 += kLevChunk) {
    const int rows = (int)min((int64_t)kLevChunk, i_end - i0);
    for (int r = 0; r < rows; r++) {
      const int64_t i = i0 + r;
      const int32_t* t = a_ids + __ldg(a_off + i);
      const int n = __ldg(a_off + i + 1) - __ldg(a_off + i);
      if (!live || (symmetric && j < i)) continue;
      int d;
      if (m == 0) {
        d = n;
      } else if (fast) {
        uint64_t pv = ~0ull, mv = 0;
        d = m;
#pragma unroll 4
        for (int x = 0; x < n; x++) {
          const int32_t c = __ldg(t + x);
          const uint64_t eq = c < kLevAlpha ? peq[c][tid] : lev_match(p, 0, m, c);
          d += lev_step(pv, mv, eq, 1, last);
        }
      } else {
        d = lev_long(p, m, t, n);
      }
      out[i * nb + j] = (uint8_t)d;
      stage[r * kLevStagePitch + tid] = (uint8_t)d;
    }
    if (symmetric) {
      // out[j][i] for the pairs j > i of this chunk: lane = row offset, so each warp writes 32 bytes of one row
      __syncthreads();
      for (int k = tid; k < kLevCols * kLevChunk; k += kLevCols) {
        const int jl = k / kLevChunk, r = k % kLevChunk;
        const int64_t jj = j_base + jl, ii = i0 + r;
        if (r < rows && jj < nb && jj > ii) out[jj * nb + ii] = stage[r * kLevStagePitch + jl];
      }
      __syncthreads();
    }
  }
}

}  // namespace tip

extern "C" int tip_levenshtein(const int32_t* a_ids, const int32_t* a_off, int64_t na, const int32_t* b_ids,
                               const int32_t* b_off, int64_t nb, int32_t max_len, int symmetric, uint8_t* out,
                               void* stream) {
  using namespace tip;
  TIP_REQUIRE(na >= 0 && nb >= 0, "negative block size");
  TIP_REQUIRE(max_len >= 0 && max_len <= kLevMaxLen, "words are limited to 255 code points");
  TIP_REQUIRE(!symmetric || (na == nb && a_ids == b_ids && a_off == b_off), "symmetric needs a == b");
  if (na == 0 || nb == 0) return TIP_OK;
  TIP_REQUIRE(a_ids && a_off && b_ids && b_off && out, "null pointer");
  const int64_t row_tiles = (na + kLevRows - 1) / kLevRows, col_tiles = (nb + kLevCols - 1) / kLevCols;
  TIP_REQUIRE(row_tiles <= 65535 && col_tiles <= 0x7fffffffLL, "block too large");
  TIP_CHECK_CUDA(cudaFuncSetAttribute(lev_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLevSmem));
  lev_kernel<<<dim3((unsigned)col_tiles, (unsigned)row_tiles), kLevCols, kLevSmem, (cudaStream_t)stream>>>(
      a_ids, a_off, na, b_ids, b_off, nb, symmetric, out);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}
