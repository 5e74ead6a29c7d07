// tokenizer.cu — Keras' word tokenizer (keras_preprocessing 1.1.2: text_to_word_sequence, Tokenizer.fit_on_texts /
// texts_to_sequences, pad_sequences) over UTF-8 bytes, the inputs of the IMDB case study
// (case_study_imdb.py:321-336: Tokenizer(num_words=2000), pad_sequences(maxlen=100)).
//
// Texts arrive as one byte buffer (UTF-8, "surrogatepass") with int64 offsets.  Every separator (the filters and
// the split character) is one ASCII byte, and no multi-byte UTF-8 sequence contains an ASCII byte, so Keras'
// lower -> translate(filters -> split) -> split(split) -> drop empties is a byte test against a 128-bit mask.
// The host lowers non-ASCII texts with str.lower(); the count pass lowers ASCII A-Z in place, which is
// str.lower() for ASCII text and changes nothing after a host lower().
//
// Stages (entry points at the end):
//   count   one warp per text, 32 bytes per step: ballots of non-separator bytes give the word starts, popcounts
//           the number of words; an exclusive scan over the texts gives each text's first word ordinal.  The
//           ordinal (text-major, position-minor) is Keras' iteration order.
//   emit    the same walk writes each word's byte offset, length and text; then one thread per word hashes it.
//   table   open addressing with linear probing.  A slot's key is the ordinal of a representative occurrence
//           (vocabulary entry i < nv, or nv + word ordinal); its bytes are in global memory before the kernel
//           runs, so a probing thread compares hash, length and bytes with it at once: no spin-waits, and a
//           hash collision never merges two words.
//   fit     every occurrence finds or claims its slot, adds one to its count and min-reduces its first
//           occurrence; a second set keyed by (slot, text) counts each word once per text (word_docs).
//   lookup  every occurrence probes the vocabulary table; its id is dropped when unknown or >= num_words (Keras
//           with oov_token=None).  One warp per text then writes the kept ids (ragged, at a scan of the kept
//           counts) and the padded row (pre / post padding and truncation, any int32 fill value).
#include "common.cuh"

namespace tip {

constexpr int kTokThreads = 256;
constexpr int kTokWarps = kTokThreads / 32;      // texts per block in the per-text kernels
constexpr int kTokScanThreads = 1024;
constexpr unsigned long long kTokEmpty = ~0ull;

__device__ __forceinline__ bool tok_is_sep(uint32_t b, uint64_t lo, uint64_t hi) {
  return b < 64 ? ((lo >> b) & 1ull) != 0 : (b < 128 ? ((hi >> (b - 64)) & 1ull) != 0 : false);
}

__device__ __forceinline__ uint64_t tok_mix(uint64_t h) {      // murmur3's 64-bit finaliser
  h ^= h >> 33;
  h *= 0xff51afd7ed558ccdull;
  h ^= h >> 33;
  h *= 0xc4ceb9fe1a85ec53ull;
  h ^= h >> 33;
  return h;
}

// FNV-1a over the bytes, finalised; bits < 64 keeps only the low bits (the collision seam of the tests)
__device__ __forceinline__ uint64_t tok_hash(const uint8_t* __restrict__ p, int32_t len, int bits) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (int32_t k = 0; k < len; k++) h = (h ^ p[k]) * 0x100000001b3ull;
  h = tok_mix(h ^ (uint64_t)len);
  return bits >= 64 ? h : h & ((1ull << bits) - 1);
}

__device__ __forceinline__ int64_t tok_slot(uint64_t h, int64_t cap) { return (int64_t)(tok_mix(h + 0x9e3779b97f4a7c15ull) & (uint64_t)(cap - 1)); }

__device__ __forceinline__ unsigned long long tok_load(const unsigned long long* p) {
  return *reinterpret_cast<const volatile unsigned long long*>(p);
}

__device__ __forceinline__ bool tok_bytes_equal(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, int32_t len) {
  for (int32_t k = 0; k < len; k++)
    if (a[k] != b[k]) return false;
  return true;
}

// Words of the call and the vocabulary, addressed by one key space: key < nv is vocabulary entry key, else word
// ordinal key - nv.
struct TokWords {
  const uint8_t* text;
  const int64_t* start;
  const int32_t* len;
  const uint64_t* hash;
};

struct TokVocab {
  const uint8_t* arena;
  const int64_t* start;
  const int32_t* len;
  const uint64_t* hash;
  int64_t n;
};

__device__ __forceinline__ bool tok_key_matches(unsigned long long key, uint64_t h, int32_t len, const uint8_t* p,
                                                const TokWords& w, const TokVocab& v) {
  const uint8_t* q;
  if ((int64_t)key < v.n) {
    if (v.hash[key] != h || v.len[key] != len) return false;
    q = v.arena + v.start[key];
  } else {
    const int64_t o = (int64_t)key - v.n;
    if (w.hash[o] != h || w.len[o] != len) return false;
    q = w.text + w.start[o];
  }
  return tok_bytes_equal(p, q, len);
}

// One warp per text.  kEmit false: lowercase ASCII in place (lower != 0), word_off[t] = number of words.
// kEmit true: word_off[t] = the text's first word ordinal; writes each word's start, length and text.
template <bool kEmit>
__global__ void __launch_bounds__(kTokThreads) tok_walk_kernel(uint8_t* __restrict__ text, const int64_t* __restrict__ text_off,
                                                               int64_t n_texts, uint64_t sep_lo, uint64_t sep_hi, int lower,
                                                               int64_t* __restrict__ word_off, int64_t* __restrict__ w_start,
                                                               int32_t* __restrict__ w_len, int32_t* __restrict__ w_text) {
  const int lane = threadIdx.x & 31;
  const int64_t t = (int64_t)blockIdx.x * kTokWarps + (threadIdx.x >> 5);
  if (t >= n_texts) return;                         // warp-uniform
  const int64_t s0 = text_off[t], s1 = text_off[t + 1];
  const uint32_t below = (1u << lane) - 1u;
  const int64_t base = kEmit ? word_off[t] : 0;
  int64_t n_start = 0, n_end = 0;
  int64_t open = s0;                                // start of the word still open after the last step
  uint32_t carry = 0;                               // the byte before this step is a word byte
  for (int64_t c = s0; c < s1; c += 32) {
    const int64_t i = c + lane;
    bool word = false;
    if (i < s1) {
      uint32_t b = text[i];
      if (!kEmit && lower && b - 'A' < 26u) {
        b += 32;
        text[i] = (uint8_t)b;
      }
      word = !tok_is_sep(b, sep_lo, sep_hi);
    }
    const uint32_t m = __ballot_sync(0xffffffffu, word);
    const uint32_t prev = (m << 1) | carry;
    const uint32_t starts = m & ~prev, ends = ~m & prev;   // an end is the first byte after a word
    if (kEmit) {
      if ((starts >> lane) & 1u) {
        const int64_t w = base + n_start + __popc(starts & below);
        w_start[w] = i;
        w_text[w] = (int32_t)t;
      }
      if ((ends >> lane) & 1u) {
        const uint32_t sb = starts & below;
        const int64_t st = sb ? c + (31 - __clz(sb)) : open;
        w_len[base + n_end + __popc(ends & below)] = (int32_t)(i - st);
      }
      if (starts) open = c + (31 - __clz(starts));
      n_end += __popc(ends);
    }
    n_start += __popc(starts);
    carry = m >> 31;
  }
  if (kEmit) {
    if (carry && lane == 0) w_len[base + n_end] = (int32_t)(s1 - open);   // the text ends inside a word
  } else if (lane == 0) {
    word_off[t] = n_start;
  }
}

// In-place exclusive scan of data[0, n) by one block; data[n] = the total.
__global__ void __launch_bounds__(kTokScanThreads) tok_scan_kernel(int64_t* __restrict__ data, int64_t n) {
  __shared__ int64_t warp_sum[32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  int64_t carry = 0;
  for (int64_t c = 0; c < n; c += kTokScanThreads) {
    const int64_t i = c + tid;
    const int64_t v = i < n ? data[i] : 0;
    int64_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_sum[wid] = x;
    __syncthreads();
    if (wid == 0) {
      int64_t s = warp_sum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int64_t y = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += y;
      }
      warp_sum[lane] = s;
    }
    __syncthreads();
    if (i < n) data[i] = carry + (wid ? warp_sum[wid - 1] : 0) + x - v;
    carry += warp_sum[31];
    __syncthreads();
  }
  if (tid == 0) data[n] = carry;
}

__global__ void __launch_bounds__(kTokThreads) tok_hash_kernel(const uint8_t* __restrict__ text, const int64_t* __restrict__ start,
                                                               const int32_t* __restrict__ len, int64_t n, int bits,
                                                               uint64_t* __restrict__ hash) {
  const int64_t w = (int64_t)blockIdx.x * kTokThreads + threadIdx.x;
  if (w < n) hash[w] = tok_hash(text + start[w], len[w], bits);
}

// Vocabulary entry i (distinct by construction) -> its slot, key i; first[slot] = i when first != nullptr.
__global__ void __launch_bounds__(kTokThreads) tok_vocab_insert_kernel(const uint64_t* __restrict__ v_hash, int64_t nv,
                                                                       unsigned long long* __restrict__ keys,
                                                                       unsigned long long* __restrict__ first, int64_t cap) {
  const int64_t i = (int64_t)blockIdx.x * kTokThreads + threadIdx.x;
  if (i >= nv) return;
  int64_t slot = tok_slot(v_hash[i], cap);
  while (atomicCAS(&keys[slot], kTokEmpty, (unsigned long long)i) != kTokEmpty) slot = (slot + 1) & (cap - 1);
  if (first) first[slot] = (unsigned long long)i;
}

__global__ void __launch_bounds__(kTokThreads) tok_fit_kernel(TokWords w, const int32_t* __restrict__ w_text, int64_t n_words,
                                                              TokVocab v, unsigned long long* __restrict__ keys,
                                                              unsigned long long* __restrict__ first,
                                                              unsigned long long* __restrict__ count,
                                                              unsigned long long* __restrict__ docs, int64_t cap,
                                                              unsigned long long* __restrict__ doc_keys, int64_t doc_cap) {
  const int64_t o = (int64_t)blockIdx.x * kTokThreads + threadIdx.x;
  if (o >= n_words) return;
  const uint64_t h = w.hash[o];
  const int32_t len = w.len[o];
  const uint8_t* p = w.text + w.start[o];
  const unsigned long long me = (unsigned long long)(v.n + o);
  int64_t slot = tok_slot(h, cap);
  for (;;) {
    unsigned long long k = tok_load(&keys[slot]);
    if (k == kTokEmpty) {
      k = atomicCAS(&keys[slot], kTokEmpty, me);
      if (k == kTokEmpty) break;                    // claimed: this occurrence represents the word
    }
    if (tok_key_matches(k, h, len, p, w, v)) break;
    slot = (slot + 1) & (cap - 1);
  }
  atomicAdd(&count[slot], 1ull);
  if (tok_load(&first[slot]) > me) atomicMin(&first[slot], me);
  // word_docs: the first thread to insert (slot, text) counts the text
  const unsigned long long dk = ((unsigned long long)slot << 32) | (uint32_t)w_text[o];
  int64_t ds = (int64_t)(tok_mix(dk) & (uint64_t)(doc_cap - 1));
  for (;;) {
    unsigned long long k = tok_load(&doc_keys[ds]);
    if (k == kTokEmpty) {
      k = atomicCAS(&doc_keys[ds], kTokEmpty, dk);
      if (k == kTokEmpty) {
        atomicAdd(&docs[slot], 1ull);
        break;
      }
    }
    if (k == dk) break;
    ds = (ds + 1) & (doc_cap - 1);
  }
}

// Every slot this call counted -> one row of out [5][out_cap]: first occurrence key, count, docs, and for a new
// word (first >= nv) the byte offset and length of its first occurrence (else -1, 0).
__global__ void __launch_bounds__(kTokThreads) tok_collect_kernel(const unsigned long long* __restrict__ keys,
                                                                  const unsigned long long* __restrict__ first,
                                                                  const unsigned long long* __restrict__ count,
                                                                  const unsigned long long* __restrict__ docs, int64_t cap,
                                                                  int64_t nv, const int64_t* __restrict__ w_start,
                                                                  const int32_t* __restrict__ w_len, int64_t* __restrict__ out,
                                                                  int64_t out_cap, unsigned long long* __restrict__ n_out) {
  const int64_t s = (int64_t)blockIdx.x * kTokThreads + threadIdx.x;
  if (s >= cap || keys[s] == kTokEmpty || count[s] == 0) return;
  const int64_t r = (int64_t)atomicAdd(n_out, 1ull);
  const int64_t f = (int64_t)first[s];
  out[r] = f;
  out[out_cap + r] = (int64_t)count[s];
  out[2 * out_cap + r] = (int64_t)docs[s];
  out[3 * out_cap + r] = f >= nv ? w_start[f - nv] : -1;
  out[4 * out_cap + r] = f >= nv ? w_len[f - nv] : 0;
}

__global__ void __launch_bounds__(kTokThreads) tok_lookup_kernel(TokWords w, int64_t n_words, TokVocab v,
                                                                 const int32_t* __restrict__ v_index,
                                                                 const unsigned long long* __restrict__ keys, int64_t cap,
                                                                 int64_t num_words, int32_t* __restrict__ w_id) {
  const int64_t o = (int64_t)blockIdx.x * kTokThreads + threadIdx.x;
  if (o >= n_words) return;
  int32_t id = -1;
  if (v.n > 0) {
    const uint64_t h = w.hash[o];
    const int32_t len = w.len[o];
    const uint8_t* p = w.text + w.start[o];
    for (int64_t slot = tok_slot(h, cap);; slot = (slot + 1) & (cap - 1)) {
      const unsigned long long k = keys[slot];
      if (k == kTokEmpty) break;                    // unknown word
      if (tok_key_matches(k, h, len, p, w, v)) {
        const int32_t idx = v_index[k];
        if (!(num_words && idx >= num_words)) id = idx;
        break;
      }
    }
  }
  w_id[o] = id;
}

// One warp per text: kept[t] = number of ids >= 0 among its words (into kept_off, scanned afterwards).
__global__ void __launch_bounds__(kTokThreads) tok_kept_kernel(const int32_t* __restrict__ w_id, const int64_t* __restrict__ word_off,
                                                               int64_t n_texts, int64_t* __restrict__ kept_off) {
  const int lane = threadIdx.x & 31;
  const int64_t t = (int64_t)blockIdx.x * kTokWarps + (threadIdx.x >> 5);
  if (t >= n_texts) return;
  int64_t kept = 0;
  for (int64_t o = word_off[t] + lane; o < word_off[t + 1]; o += 32) kept += w_id[o] >= 0;
  for (int s = 16; s > 0; s >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, s);
  if (lane == 0) kept_off[t] = kept;
}

// One warp per text: the kept ids in order into ragged[kept_off[t] ..) and, when padded != nullptr, the row
// padded[t][0, maxlen) as pad_sequences writes it.
__global__ void __launch_bounds__(kTokThreads) tok_write_kernel(const int32_t* __restrict__ w_id, const int64_t* __restrict__ word_off,
                                                                const int64_t* __restrict__ kept_off, int64_t n_texts,
                                                                int32_t* __restrict__ ragged, int32_t* __restrict__ padded,
                                                                int64_t maxlen, int pre_padding, int pre_truncating,
                                                                int32_t value) {
  const int lane = threadIdx.x & 31;
  const int64_t t = (int64_t)blockIdx.x * kTokWarps + (threadIdx.x >> 5);
  if (t >= n_texts) return;
  const uint32_t below = (1u << lane) - 1u;
  const int64_t kept = kept_off[t + 1] - kept_off[t];
  const int64_t keep = min(kept, maxlen);
  const int64_t skip = pre_truncating ? kept - keep : 0;      // kept ids cut off at the front
  const int64_t col0 = pre_padding ? maxlen - keep : 0;       // column of the first id written
  int32_t* row = padded ? padded + t * maxlen : nullptr;
  if (row)
    for (int64_t c = lane; c < maxlen; c += 32)
      if (c < col0 || c >= col0 + keep) row[c] = value;
  int32_t* out = ragged ? ragged + kept_off[t] : nullptr;
  int64_t r = 0;
  const int64_t o1 = word_off[t + 1];
  for (int64_t o0 = word_off[t]; o0 < o1; o0 += 32) {
    const int64_t o = o0 + lane;
    const int32_t id = o < o1 ? w_id[o] : -1;
    const uint32_t m = __ballot_sync(0xffffffffu, id >= 0);
    if (id >= 0) {
      const int64_t k = r + __popc(m & below);
      if (out) out[k] = id;
      if (row && k >= skip && k < skip + keep) row[col0 + k - skip] = id;
    }
    r += __popc(m);
  }
}

inline unsigned tok_blocks(int64_t n, int per_block) { return (unsigned)((n + per_block - 1) / per_block); }

inline bool tok_pow2(int64_t x) { return x > 0 && (x & (x - 1)) == 0; }

}  // namespace tip

using namespace tip;

extern "C" int tip_tok_count(uint8_t* text, const int64_t* text_off, int64_t n_texts, uint64_t sep_lo, uint64_t sep_hi,
                             int lower, int64_t* word_off, void* stream) {
  TIP_REQUIRE(n_texts >= 0, "negative text count");
  if (n_texts == 0) return TIP_OK;
  TIP_REQUIRE(text_off && word_off, "null pointer");
  TIP_REQUIRE(tok_blocks(n_texts, kTokWarps) <= 0x7fffffffu, "too many texts");
  cudaStream_t st = (cudaStream_t)stream;
  tok_walk_kernel<false><<<tok_blocks(n_texts, kTokWarps), kTokThreads, 0, st>>>(text, text_off, n_texts, sep_lo, sep_hi, lower,
                                                                               word_off, nullptr, nullptr, nullptr);
  TIP_LAUNCH_CHECK();
  tok_scan_kernel<<<1, kTokScanThreads, 0, st>>>(word_off, n_texts);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_tok_emit(const uint8_t* text, const int64_t* text_off, int64_t n_texts, uint64_t sep_lo, uint64_t sep_hi,
                            const int64_t* word_off, int64_t n_words, int32_t hash_bits, int64_t* w_start, int32_t* w_len,
                            int32_t* w_text, uint64_t* w_hash, void* stream) {
  TIP_REQUIRE(n_texts >= 0 && n_words >= 0, "negative size");
  TIP_REQUIRE(hash_bits >= 1 && hash_bits <= 64, "hash_bits must be in [1, 64]");
  TIP_REQUIRE(n_texts < (1LL << 31), "text ids are int32");
  if (n_texts == 0 || n_words == 0) return TIP_OK;
  TIP_REQUIRE(text && text_off && word_off && w_start && w_len && w_text && w_hash, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  tok_walk_kernel<true><<<tok_blocks(n_texts, kTokWarps), kTokThreads, 0, st>>>(
      const_cast<uint8_t*>(text), text_off, n_texts, sep_lo, sep_hi, 0, const_cast<int64_t*>(word_off), w_start, w_len, w_text);
  TIP_LAUNCH_CHECK();
  tok_hash_kernel<<<tok_blocks(n_words, kTokThreads), kTokThreads, 0, st>>>(text, w_start, w_len, n_words, hash_bits, w_hash);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_tok_vocab_table(const uint8_t* arena, const int64_t* v_start, const int32_t* v_len, int64_t nv,
                                   int32_t hash_bits, uint64_t* v_hash, uint64_t* keys, uint64_t* first, int64_t cap,
                                   void* stream) {
  TIP_REQUIRE(nv >= 0 && tok_pow2(cap) && cap >= 2 * nv && cap <= (1LL << 31), "cap must be a power of two >= 2 nv, <= 2^31");
  TIP_REQUIRE(hash_bits >= 1 && hash_bits <= 64, "hash_bits must be in [1, 64]");
  TIP_REQUIRE(keys, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  TIP_CHECK_CUDA(cudaMemsetAsync(keys, 0xff, sizeof(uint64_t) * cap, st));
  if (first) TIP_CHECK_CUDA(cudaMemsetAsync(first, 0xff, sizeof(uint64_t) * cap, st));
  if (nv == 0) return TIP_OK;
  TIP_REQUIRE(arena && v_start && v_len && v_hash, "null pointer");
  tok_hash_kernel<<<tok_blocks(nv, kTokThreads), kTokThreads, 0, st>>>(arena, v_start, v_len, nv, hash_bits, v_hash);
  TIP_LAUNCH_CHECK();
  tok_vocab_insert_kernel<<<tok_blocks(nv, kTokThreads), kTokThreads, 0, st>>>(
      v_hash, nv, reinterpret_cast<unsigned long long*>(keys), reinterpret_cast<unsigned long long*>(first), cap);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_tok_fit(const uint8_t* text, const int64_t* w_start, const int32_t* w_len, const int32_t* w_text,
                           const uint64_t* w_hash, int64_t n_words, const uint8_t* arena, const int64_t* v_start,
                           const int32_t* v_len, const uint64_t* v_hash, int64_t nv, uint64_t* keys, uint64_t* first,
                           uint64_t* count, uint64_t* docs, int64_t cap, uint64_t* doc_keys, int64_t doc_cap, int64_t* out,
                           int64_t out_cap, uint64_t* n_out, void* stream) {
  TIP_REQUIRE(n_words >= 0 && nv >= 0, "negative size");
  TIP_REQUIRE(tok_pow2(cap) && cap >= 2 * (nv + n_words) && cap <= (1LL << 31), "cap must be a power of two >= 2 (nv + n_words), <= 2^31");
  TIP_REQUIRE(tok_pow2(doc_cap) && doc_cap >= 2 * n_words, "doc_cap must be a power of two >= 2 n_words");
  TIP_REQUIRE(out_cap >= nv + n_words, "out_cap < nv + n_words");
  TIP_REQUIRE(keys && first && count && docs && doc_keys && out && n_out, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  TIP_CHECK_CUDA(cudaMemsetAsync(n_out, 0, sizeof(uint64_t), st));
  if (n_words == 0) return TIP_OK;
  TIP_REQUIRE(text && w_start && w_len && w_text && w_hash, "null pointer");
  TIP_REQUIRE(nv == 0 || (arena && v_start && v_len && v_hash), "null pointer");
  TIP_CHECK_CUDA(cudaMemsetAsync(count, 0, sizeof(uint64_t) * cap, st));
  TIP_CHECK_CUDA(cudaMemsetAsync(docs, 0, sizeof(uint64_t) * cap, st));
  TIP_CHECK_CUDA(cudaMemsetAsync(doc_keys, 0xff, sizeof(uint64_t) * doc_cap, st));
  const TokWords w{text, w_start, w_len, w_hash};
  const TokVocab v{arena, v_start, v_len, v_hash, nv};
  auto* k = reinterpret_cast<unsigned long long*>(keys);
  auto* f = reinterpret_cast<unsigned long long*>(first);
  auto* c = reinterpret_cast<unsigned long long*>(count);
  auto* d = reinterpret_cast<unsigned long long*>(docs);
  tok_fit_kernel<<<tok_blocks(n_words, kTokThreads), kTokThreads, 0, st>>>(
      w, w_text, n_words, v, k, f, c, d, cap, reinterpret_cast<unsigned long long*>(doc_keys), doc_cap);
  TIP_LAUNCH_CHECK();
  tok_collect_kernel<<<tok_blocks(cap, kTokThreads), kTokThreads, 0, st>>>(
      k, f, c, d, cap, nv, w_start, w_len, out, out_cap, reinterpret_cast<unsigned long long*>(n_out));
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_tok_lookup(const uint8_t* text, const int64_t* w_start, const int32_t* w_len, const uint64_t* w_hash,
                              int64_t n_words, const uint8_t* arena, const int64_t* v_start, const int32_t* v_len,
                              const uint64_t* v_hash, const int32_t* v_index, int64_t nv, const uint64_t* keys, int64_t cap,
                              int64_t num_words, const int64_t* word_off, int64_t n_texts, int32_t* w_id, int64_t* kept_off,
                              int32_t* ragged, int32_t* padded, int64_t maxlen, int pre_padding, int pre_truncating,
                              int32_t value, void* stream) {
  TIP_REQUIRE(n_words >= 0 && nv >= 0 && n_texts >= 0 && num_words >= 0, "negative size");
  TIP_REQUIRE(!padded || maxlen >= 1, "padded rows need maxlen >= 1");
  TIP_REQUIRE(nv == 0 || (tok_pow2(cap) && cap >= 2 * nv), "cap must be a power of two >= 2 nv");
  if (n_texts == 0) return TIP_OK;
  TIP_REQUIRE(word_off && kept_off && (n_words == 0 || w_id), "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (n_words > 0) {
    TIP_REQUIRE(text && w_start && w_len && w_hash, "null pointer");
    TIP_REQUIRE(nv == 0 || (arena && v_start && v_len && v_hash && v_index && keys), "null pointer");
    const TokWords w{text, w_start, w_len, w_hash};
    const TokVocab v{arena, v_start, v_len, v_hash, nv};
    tok_lookup_kernel<<<tok_blocks(n_words, kTokThreads), kTokThreads, 0, st>>>(
        w, n_words, v, v_index, reinterpret_cast<const unsigned long long*>(keys), cap, num_words, w_id);
    TIP_LAUNCH_CHECK();
  }
  tok_kept_kernel<<<tok_blocks(n_texts, kTokWarps), kTokThreads, 0, st>>>(w_id, word_off, n_texts, kept_off);
  TIP_LAUNCH_CHECK();
  tok_scan_kernel<<<1, kTokScanThreads, 0, st>>>(kept_off, n_texts);
  TIP_LAUNCH_CHECK();
  tok_write_kernel<<<tok_blocks(n_texts, kTokWarps), kTokThreads, 0, st>>>(w_id, word_off, kept_off, n_texts, ragged, padded,
                                                                         maxlen, pre_padding, pre_truncating, value);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}
