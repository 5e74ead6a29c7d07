// corrupt.cu — TextCorruptor.corrupt (IMDB-C) over UTF-8 bytes, string for string what the host port writes
// (simple_tip_b200/core/text_corruptor.py; the arithmetic is restated in include/b200tip.h, tip_corrupt_*).
//
// Texts arrive as one byte buffer (strict UTF-8) with int64 offsets.  Stages (entry points at the end):
//   census  one thread per byte: the distinct non-ASCII code points, as bits of a 0x110000-bit map.  The host
//           classifies those few with Python's own re (\w, \s) and uploads a class table, so the split below equals
//           re.findall(r"\w+|[^\w\s]+", text) by construction.
//   count   one thread per text: its number of tokens (maximal runs of word, or of other, code points).
//   texts   one thread per text: each token's offset, byte and code-point length; the sentence MD5 (" "-joined
//           tokens), the corruption-type draws and Generator.shuffle of the word indexes, all sequential per text.
//   words   one thread per word occurrence: its word MD5s, table lookups (hash + byte compare, so a collision never
//           changes a result) and the autocorrect draw; the result is a reference to bytes plus an optional typo.
//   layout  one thread per text: each word's output position within its text and the text's output length.
//   write   one thread per word: its output bytes and the separating space.
#include "common.cuh"

namespace tip {

constexpr int kCtThreads = 256;
constexpr int kCtSpace = 0;                                       // class table: 0 whitespace, 1 word, 2 other
constexpr int kCtChosen = 4;                                      // w_flags bit: the shuffle picked the word
enum CtSrc : uint8_t { kSrcText = 0, kSrcCommon = 1, kSrcBags = 2, kSrcThesaurus = 3 };

// ---- MD5 (RFC 1321), streamed byte by byte ------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t ct_rotl(uint32_t x, int c) { return (x << c) | (x >> (32 - c)); }

__host__ __device__ inline void md5_block(uint32_t st[4], const uint8_t* blk) {
  const uint32_t K[64] = {
      0xd76aa478, 0xe8c7b756, 0x242070db, 0xc1bdceee, 0xf57c0faf, 0x4787c62a, 0xa8304613, 0xfd469501,
      0x698098d8, 0x8b44f7af, 0xffff5bb1, 0x895cd7be, 0x6b901122, 0xfd987193, 0xa679438e, 0x49b40821,
      0xf61e2562, 0xc040b340, 0x265e5a51, 0xe9b6c7aa, 0xd62f105d, 0x02441453, 0xd8a1e681, 0xe7d3fbc8,
      0x21e1cde6, 0xc33707d6, 0xf4d50d87, 0x455a14ed, 0xa9e3e905, 0xfcefa3f8, 0x676f02d9, 0x8d2a4c8a,
      0xfffa3942, 0x8771f681, 0x6d9d6122, 0xfde5380c, 0xa4beea44, 0x4bdecfa9, 0xf6bb4b60, 0xbebfbc70,
      0x289b7ec6, 0xeaa127fa, 0xd4ef3085, 0x04881d05, 0xd9d4d039, 0xe6db99e5, 0x1fa27cf8, 0xc4ac5665,
      0xf4292244, 0x432aff97, 0xab9423a7, 0xfc93a039, 0x655b59c3, 0x8f0ccc92, 0xffeff47d, 0x85845dd1,
      0x6fa87e4f, 0xfe2ce6e0, 0xa3014314, 0x4e0811a1, 0xf7537e82, 0xbd3af235, 0x2ad7d2bb, 0xeb86d391};
  const int S[16] = {7, 12, 17, 22, 5, 9, 14, 20, 4, 11, 16, 23, 6, 10, 15, 21};
  uint32_t m[16];
#pragma unroll
  for (int i = 0; i < 16; i++)
    m[i] = (uint32_t)blk[4 * i] | ((uint32_t)blk[4 * i + 1] << 8) | ((uint32_t)blk[4 * i + 2] << 16) |
           ((uint32_t)blk[4 * i + 3] << 24);
  uint32_t a = st[0], b = st[1], c = st[2], d = st[3];
#pragma unroll
  for (int i = 0; i < 64; i++) {
    uint32_t f;
    int g;
    if (i < 16) { f = (b & c) | (~b & d); g = i; }
    else if (i < 32) { f = (d & b) | (~d & c); g = (5 * i + 1) & 15; }
    else if (i < 48) { f = b ^ c ^ d; g = (3 * i + 5) & 15; }
    else { f = c ^ (b | ~d); g = (7 * i) & 15; }
    const uint32_t t = d;
    d = c;
    c = b;
    b = b + ct_rotl(a + f + K[i] + m[g], S[(i >> 4) * 4 + (i & 3)]);
    a = t;
  }
  st[0] += a; st[1] += b; st[2] += c; st[3] += d;
}

struct Md5 {
  uint32_t st[4];
  uint8_t buf[64];
  uint32_t nbuf;
  uint64_t total;
  __host__ __device__ Md5() : st{0x67452301u, 0xefcdab89u, 0x98badcfeu, 0x10325476u}, nbuf(0), total(0) {}
  __host__ __device__ void put(uint8_t x) {
    buf[nbuf++] = x;
    total++;
    if (nbuf == 64) {
      md5_block(st, buf);
      nbuf = 0;
    }
  }
  __host__ __device__ void put(const uint8_t* p, int64_t n) {
    for (int64_t k = 0; k < n; k++) put(p[k]);
  }
  __host__ __device__ void put_decimal(int64_t v) {           // str(v), v >= 0
    char d[20];
    int n = 0;
    do { d[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    while (n) put((uint8_t)d[--n]);
  }
  // int(md5.hexdigest(), 16) % 10**6: the digest read as a big-endian 128-bit integer
  __host__ __device__ int64_t mod_1e6() {
    const uint64_t bits = total * 8;
    put(0x80);
    while (nbuf != 56) put(0);
    for (int k = 0; k < 8; k++) put((uint8_t)(bits >> (8 * k)));
    uint64_t r = 0;
    for (int w = 0; w < 4; w++)
      for (int k = 0; k < 4; k++) r = (r * 256 + ((st[w] >> (8 * k)) & 0xff)) % 1000000;
    return (int64_t)r;
  }
};

// ---- NumPy's default_rng(seed): SeedSequence -> PCG64 (XSL-RR 128/64) ------------------------------------------
typedef unsigned __int128 u128;

struct Pcg64 {
  u128 state, inc;
  uint32_t buffered;
  bool has_buffered;

  __host__ __device__ __forceinline__ void step() {
    const u128 mult = ((u128)0x2360ED051FC65DA4ull << 64) | 0x4385DF649FCCF645ull;
    state = state * mult + inc;
  }
  // SeedSequence(seed).generate_state(4, uint64), then pcg64_set_seed(state = w0:w1, seq = w2:w3)
  __host__ __device__ explicit Pcg64(uint64_t seed) : buffered(0), has_buffered(false) {
    const uint32_t ent[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
    const int n_ent = (seed >> 32) ? 2 : 1;
    uint32_t hc = 0x43b0d7e5u;
    auto hashmix = [&](uint32_t v) {
      v ^= hc;
      hc *= 0x931e8875u;
      v *= hc;
      return v ^ (v >> 16);
    };
    auto mix = [](uint32_t x, uint32_t y) {
      uint32_t r = 0xca01f9ddu * x - 0x4973f715u * y;
      return r ^ (r >> 16);
    };
    uint32_t pool[4];
    for (int i = 0; i < 4; i++) pool[i] = hashmix(i < n_ent ? ent[i] : 0u);
    for (int s = 0; s < 4; s++)
      for (int d = 0; d < 4; d++)
        if (s != d) pool[d] = mix(pool[d], hashmix(pool[s]));
    uint32_t hb = 0x8b51f9ddu, w32[8];
    for (int i = 0; i < 8; i++) {
      uint32_t v = pool[i & 3] ^ hb;
      hb *= 0x58f38dedu;
      v *= hb;
      w32[i] = v ^ (v >> 16);
    }
    uint64_t w[4];
    for (int i = 0; i < 4; i++) w[i] = (uint64_t)w32[2 * i] | ((uint64_t)w32[2 * i + 1] << 32);
    const u128 initstate = ((u128)w[0] << 64) | w[1], initseq = ((u128)w[2] << 64) | w[3];
    inc = (initseq << 1) | 1;
    state = 0;
    step();
    state += initstate;
    step();
  }
  __host__ __device__ __forceinline__ uint64_t next64() {
    step();
    const uint64_t x = (uint64_t)(state >> 64) ^ (uint64_t)state;
    const unsigned rot = (unsigned)(state >> 122);
    return (x >> rot) | (x << ((64 - rot) & 63));
  }
  __host__ __device__ __forceinline__ uint32_t next32() {       // low half first, then the high half
    if (has_buffered) {
      has_buffered = false;
      return buffered;
    }
    const uint64_t v = next64();
    buffered = (uint32_t)(v >> 32);
    has_buffered = true;
    return (uint32_t)v;
  }
  __host__ __device__ __forceinline__ double random() { return (double)(next64() >> 11) * (1.0 / 9007199254740992.0); }
  // random_interval(max): masked rejection on buffered uint32 draws (uint64 draws above 2^32 - 1)
  __host__ __device__ uint64_t interval(uint64_t mx) {
    if (mx == 0) return 0;
    uint64_t mask = mx;
    mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16; mask |= mask >> 32;
    uint64_t v;
    if (mx <= 0xffffffffull) {
      while ((v = (next32() & mask)) > mx) {}
    } else {
      while ((v = (next64() & mask)) > mx) {}
    }
    return v;
  }
};

// cdf.searchsorted(u, side="right") of a sorted cdf: the entries <= u (a NaN entry never is, as NumPy sorts NaN last)
__host__ __device__ __forceinline__ int ct_search_right(const double* cdf, int n, double u) {
  int k = 0;
  for (int i = 0; i < n; i++) k += cdf[i] <= u;
  return k;
}

// ---- UTF-8 --------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int ct_cp_len(uint8_t b) { return b < 0x80 ? 1 : b < 0xE0 ? 2 : b < 0xF0 ? 3 : 4; }

__device__ __forceinline__ uint32_t ct_decode(const uint8_t* p, int len) {
  if (len == 1) return p[0];
  uint32_t cp = p[0] & (0x7f >> len);
  for (int k = 1; k < len; k++) cp = (cp << 6) | (p[k] & 0x3f);
  return cp;
}

// ---- word tables ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t ct_mix(uint64_t h) {        // murmur3's 64-bit finaliser
  h ^= h >> 33;
  h *= 0xff51afd7ed558ccdull;
  h ^= h >> 33;
  h *= 0xc4ceb9fe1a85ec53ull;
  h ^= h >> 33;
  return h;
}

__device__ __forceinline__ uint64_t ct_hash(const uint8_t* p, int32_t len) {   // FNV-1a, finalised
  uint64_t h = 0xcbf29ce484222325ull;
  for (int32_t k = 0; k < len; k++) h = (h ^ p[k]) * 0x100000001b3ull;
  return ct_mix(h ^ (uint64_t)len);
}

__device__ __forceinline__ bool ct_equal(const uint8_t* a, const uint8_t* b, int32_t len) {
  for (int32_t k = 0; k < len; k++)
    if (a[k] != b[k]) return false;
  return true;
}

// key index of the bytes p[0, len) in table t, -1 when absent
__device__ int64_t ct_find(const tip_corrupt_table& t, const uint8_t* p, int32_t len) {
  if (t.n == 0) return -1;
  const uint64_t h = ct_hash(p, len);
  for (int64_t s = (int64_t)(ct_mix(h) & (uint64_t)(t.cap - 1));; s = (s + 1) & (t.cap - 1)) {
    const int32_t k = t.slots[s];
    if (k < 0) return -1;
    if (t.key_hash[k] == h && t.key_len[k] == len && ct_equal(t.arena + t.key_off[k], p, len)) return k;
  }
}

__global__ void __launch_bounds__(kCtThreads) ct_table_kernel(tip_corrupt_table t) {
  const int64_t i = (int64_t)blockIdx.x * kCtThreads + threadIdx.x;
  if (i >= t.n) return;
  const uint64_t h = ct_hash(t.arena + t.key_off[i], t.key_len[i]);
  t.key_hash[i] = h;
  int64_t s = (int64_t)(ct_mix(h) & (uint64_t)(t.cap - 1));
  while (atomicCAS(&t.slots[s], -1, (int32_t)i) != -1) s = (s + 1) & (t.cap - 1);
}

// ---- census, split --------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kCtThreads) ct_census_kernel(const uint8_t* __restrict__ text, int64_t n,
                                                               uint32_t* __restrict__ bitmap) {
  for (int64_t i = (int64_t)blockIdx.x * kCtThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kCtThreads) {
    const uint8_t b = text[i];
    if (b < 0xC0) continue;                       // ASCII (classified by the host anyway) or a continuation byte
    const uint32_t cp = ct_decode(text + i, ct_cp_len(b));
    const uint32_t bit = 1u << (cp & 31);
    if (!(bitmap[cp >> 5] & bit)) atomicOr(&bitmap[cp >> 5], bit);
  }
}

struct CtWords {
  int64_t* start;
  int32_t* len;
  int32_t* cps;
  int32_t* text;
};

// Walks text t's code points; kEmit false: returns the number of tokens; true: writes them from word `w`.
template <bool kEmit>
__device__ int64_t ct_split(const uint8_t* __restrict__ text, int64_t s0, int64_t s1, const uint8_t* __restrict__ cls,
                            int64_t w, int32_t t, CtWords out) {
  int64_t n = 0, st = 0;
  int32_t cps = 0;
  int prev = kCtSpace;
  for (int64_t i = s0; i < s1;) {
    const int l = ct_cp_len(text[i]);
    const int c = cls[ct_decode(text + i, l)];
    if (c != prev) {
      if (kEmit && prev != kCtSpace) {
        out.len[w + n - 1] = (int32_t)(i - st);
        out.cps[w + n - 1] = cps;
      }
      if (c != kCtSpace) {
        if (kEmit) {
          out.start[w + n] = i;
          out.text[w + n] = t;
        }
        st = i;
        cps = 0;
        n++;
      }
      prev = c;
    }
    cps += c != kCtSpace;
    i += l;
  }
  if (kEmit && prev != kCtSpace) {
    out.len[w + n - 1] = (int32_t)(s1 - st);
    out.cps[w + n - 1] = cps;
  }
  return n;
}

__global__ void __launch_bounds__(kCtThreads) ct_count_kernel(const uint8_t* __restrict__ text,
                                                              const int64_t* __restrict__ text_off, int64_t n_texts,
                                                              const uint8_t* __restrict__ cls, int64_t* __restrict__ n_words) {
  const int64_t t = (int64_t)blockIdx.x * kCtThreads + threadIdx.x;
  if (t < n_texts) n_words[t] = ct_split<false>(text, text_off[t], text_off[t + 1], cls, 0, 0, CtWords{});
}

struct CtTypeCdf {
  double c[4];
};

__global__ void __launch_bounds__(kCtThreads) ct_texts_kernel(const uint8_t* __restrict__ text,
                                                              const int64_t* __restrict__ text_off, int64_t n_texts,
                                                              const uint8_t* __restrict__ cls,
                                                              const int64_t* __restrict__ word_off, int64_t seed,
                                                              double severity, CtTypeCdf cdf, CtWords w,
                                                              int64_t* __restrict__ w_seed, uint8_t* __restrict__ w_flags,
                                                              int32_t* __restrict__ perm) {
  const int64_t t = (int64_t)blockIdx.x * kCtThreads + threadIdx.x;
  if (t >= n_texts) return;
  const int64_t base = word_off[t];
  const int64_t n = ct_split<true>(text, text_off[t], text_off[t + 1], cls, base, (int32_t)t, w);
  Md5 md5;                                                 // md5(" ".join(words))
  for (int64_t k = 0; k < n; k++) {
    if (k) md5.put(' ');
    md5.put(text + w.start[base + k], w.len[base + k]);
  }
  const int64_t sentence_seed = md5.mod_1e6() + seed;
  Pcg64 types((uint64_t)sentence_seed);
  for (int64_t k = 0; k < n; k++) {
    w_flags[base + k] = (uint8_t)ct_search_right(cdf.c, 4, types.random());
    w_seed[base + k] = sentence_seed + k;
    perm[base + k] = (int32_t)k;
  }
  Pcg64 shuf((uint64_t)sentence_seed);                     // Generator.shuffle(np.arange(n))
  for (int64_t i = n - 1; i >= 1; i--) {
    const int64_t j = (int64_t)shuf.interval((uint64_t)i);
    const int32_t x = perm[base + i];
    perm[base + i] = perm[base + j];
    perm[base + j] = x;
  }
  const int64_t m = (int64_t)rint((double)n * severity);   // Python's round: half to even
  for (int64_t k = 0; k < m; k++) w_flags[base + perm[base + k]] |= kCtChosen;
}

// ---- per word -------------------------------------------------------------------------------------------------------
struct CtTables {
  tip_corrupt_table common, bags, thesaurus;
};

__device__ __forceinline__ int64_t ct_word_hash(const uint8_t* p, int32_t len, int64_t seed, bool synonym) {
  Md5 m;                                                   // md5(f"{w} {seed}") or md5(f"{w} {seed} _corrupt_synonym")
  m.put(p, len);
  m.put(' ');
  m.put_decimal(seed);
  if (synonym) {
    const char* s = " _corrupt_synonym";
    for (int k = 0; s[k]; k++) m.put((uint8_t)s[k]);
  }
  return m.mod_1e6();
}

__global__ void __launch_bounds__(kCtThreads) ct_words_kernel(const uint8_t* __restrict__ text, CtWords w,
                                                              const int64_t* __restrict__ w_seed,
                                                              const uint8_t* __restrict__ w_flags, int64_t n_words,
                                                              CtTables tb, uint8_t* __restrict__ o_src,
                                                              int64_t* __restrict__ o_off, int32_t* __restrict__ o_len,
                                                              int64_t* __restrict__ o_typo,
                                                              unsigned long long* __restrict__ error_word) {
  const int64_t i = (int64_t)blockIdx.x * kCtThreads + threadIdx.x;
  if (i >= n_words) return;
  const int64_t off = w.start[i];
  const int32_t len = w.len[i], cps = w.cps[i];
  const uint8_t flags = w_flags[i];
  uint8_t src = kSrcText;
  int64_t res_off = off, typo = -1;
  int32_t res_len = len;
  if ((flags & kCtChosen) && cps >= 2) {
    const uint8_t* p = text + off;
    const int64_t seed = w_seed[i];
    int type = flags & 3;                                  // 0 typo, 1 synonym, 2 autocomplete, 3 autocorrect
    if (type == 2) {                                       // the start bags of 5, 4, 3 code points, without the word
      int32_t plen[6] = {0, 0, 0, 0, 0, 0};
      for (int c = 0, b = 0; c < 5 && c < cps; c++) {
        b += ct_cp_len(p[b]);
        plen[c + 1] = b;
      }
      int64_t h = -1;
      for (int nc = cps < 5 ? cps : 5; nc >= 3 && type == 2; nc--) {
        const int64_t k = ct_find(tb.bags, p, plen[nc]);
        if (k < 0) continue;
        const int64_t v0 = tb.bags.val_begin[k], v1 = tb.bags.val_begin[k + 1];
        auto is_word = [&](int64_t v) { return tb.bags.val_len[v] == len && ct_equal(tb.bags.arena + tb.bags.val_off[v], p, len); };
        int64_t m = 0;
        for (int64_t v = v0; v < v1; v++) m += !is_word(v);
        if (m == 0) continue;
        if (h < 0) h = ct_word_hash(p, len, seed, false);
        int64_t r = h % m;
        for (int64_t v = v0; v < v1; v++) {
          if (is_word(v)) continue;
          if (r-- == 0) {
            src = kSrcBags;
            res_off = tb.bags.val_off[v];
            res_len = tb.bags.val_len[v];
            break;
          }
        }
        type = -1;
      }
      if (type == 2) type = 3;                             // no bag left: autocorrect
    }
    if (type == 3) {                                       // one of the nearest common words, by a per-word generator
      const int64_t k = ct_find(tb.common, p, len);
      if (k >= 0) {
        const int64_t v0 = tb.common.val_begin[k], v1 = tb.common.val_begin[k + 1];
        if (v0 == v1) {
          atomicMin(error_word, (unsigned long long)i);   // Generator.choice of no candidates raises on the host
        } else {
          Pcg64 rng((uint64_t)seed);
          int64_t v = v0 + ct_search_right(tb.common.val_cdf + v0, (int)(v1 - v0), rng.random());
          if (v >= v1) v = v1 - 1;                         // unreachable: the cdf ends at 1.0 and random() < 1
          src = kSrcCommon;
          res_off = tb.common.val_off[v];
          res_len = tb.common.val_len[v];
        }
      }
    }
    if (type == 1) {                                       // a synonym by hash, else a typo
      const int64_t k = ct_find(tb.thesaurus, p, len);
      const int64_t v0 = k < 0 ? 0 : tb.thesaurus.val_begin[k], v1 = k < 0 ? 0 : tb.thesaurus.val_begin[k + 1];
      if (v1 > v0) {
        const int64_t v = v0 + ct_word_hash(p, len, seed, true) % (v1 - v0);
        src = kSrcThesaurus;
        res_off = tb.thesaurus.val_off[v];
        res_len = tb.thesaurus.val_len[v];
      } else {
        type = 0;
      }
    }
    if (type == 0) {                                       // code point seed % len -> a lower-case letter
      const int64_t kc = seed % cps;
      int32_t b = 0;
      for (int64_t c = 0; c < kc; c++) b += ct_cp_len(p[b]);
      const int l = ct_cp_len(p[b]);
      const uint32_t cp = ct_decode(p + b, l);
      const bool lower = cp >= 'a' && cp <= 'z';
      int32_t r = (int32_t)(ct_word_hash(p, len, seed, false) % (lower ? 25 : 26));
      const uint32_t letter = 'a' + r + (lower && 'a' + (uint32_t)r >= cp ? 1 : 0);
      typo = ((int64_t)b << 16) | ((int64_t)l << 8) | letter;
    }
  }
  o_src[i] = src;
  o_off[i] = res_off;
  o_len[i] = res_len;
  o_typo[i] = typo;
}

__device__ __forceinline__ int64_t ct_out_len(int32_t len, int64_t typo) {
  return typo < 0 ? len : len - ((typo >> 8) & 0xff) + 1;
}

__global__ void __launch_bounds__(kCtThreads) ct_layout_kernel(const int64_t* __restrict__ word_off, int64_t n_texts,
                                                               const int32_t* __restrict__ o_len,
                                                               const int64_t* __restrict__ o_typo,
                                                               int64_t* __restrict__ o_pos, int64_t* __restrict__ text_len) {
  const int64_t t = (int64_t)blockIdx.x * kCtThreads + threadIdx.x;
  if (t >= n_texts) return;
  int64_t pos = 0;
  for (int64_t i = word_off[t]; i < word_off[t + 1]; i++) {
    if (i > word_off[t]) pos++;                            // the separating space
    o_pos[i] = pos;
    pos += ct_out_len(o_len[i], o_typo[i]);
  }
  text_len[t] = pos;
}

__global__ void __launch_bounds__(kCtThreads) ct_write_kernel(const uint8_t* __restrict__ text, const int32_t* __restrict__ w_text,
                                                              const int64_t* __restrict__ word_off, int64_t n_words,
                                                              CtTables tb, const uint8_t* __restrict__ o_src,
                                                              const int64_t* __restrict__ o_off,
                                                              const int32_t* __restrict__ o_len,
                                                              const int64_t* __restrict__ o_typo,
                                                              const int64_t* __restrict__ o_pos,
                                                              const int64_t* __restrict__ out_off, uint8_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * kCtThreads + threadIdx.x;
  if (i >= n_words) return;
  const int32_t t = w_text[i];
  const uint8_t s = o_src[i];
  const uint8_t* p = (s == kSrcText ? text : s == kSrcCommon ? tb.common.arena : s == kSrcBags ? tb.bags.arena
                                                                                               : tb.thesaurus.arena) + o_off[i];
  const int32_t len = o_len[i];
  const int64_t typo = o_typo[i];
  uint8_t* d = out + out_off[t] + o_pos[i];
  int64_t n;
  if (typo < 0) {
    for (int32_t k = 0; k < len; k++) d[k] = p[k];
    n = len;
  } else {
    const int32_t b = (int32_t)(typo >> 16), l = (int32_t)((typo >> 8) & 0xff);
    for (int32_t k = 0; k < b; k++) d[k] = p[k];
    d[b] = (uint8_t)(typo & 0xff);
    for (int32_t k = b + l; k < len; k++) d[k - l + 1] = p[k];
    n = len - l + 1;
  }
  if (i + 1 < word_off[t + 1]) d[n] = ' ';
}

inline unsigned ct_blocks(int64_t n) { return (unsigned)((n + kCtThreads - 1) / kCtThreads); }

inline bool ct_table_ok(const tip_corrupt_table* t) {
  if (!t || t->n < 0) return false;
  if (t->n == 0) return true;
  return t->arena && t->key_off && t->key_len && t->key_hash && t->val_begin && t->val_off && t->val_len && t->slots &&
         t->cap >= 2 * t->n && (t->cap & (t->cap - 1)) == 0 && t->n < (1LL << 31);
}

}  // namespace tip

using namespace tip;

extern "C" int tip_corrupt_table_build(const tip_corrupt_table* table, void* stream) {
  TIP_REQUIRE(ct_table_ok(table), "table: n >= 0, n < 2^31, cap a power of two >= 2 n, non-null arrays");
  if (table->n == 0) return TIP_OK;
  cudaStream_t st = (cudaStream_t)stream;
  TIP_CHECK_CUDA(cudaMemsetAsync(table->slots, 0xff, sizeof(int32_t) * table->cap, st));
  TIP_REQUIRE(ct_blocks(table->n) <= 0x7fffffffu, "too many keys");
  ct_table_kernel<<<ct_blocks(table->n), kCtThreads, 0, st>>>(*table);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_corrupt_census(const uint8_t* text, int64_t n_bytes, uint32_t* bitmap, void* stream) {
  TIP_REQUIRE(n_bytes >= 0, "negative size");
  TIP_REQUIRE(bitmap, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  TIP_CHECK_CUDA(cudaMemsetAsync(bitmap, 0, sizeof(uint32_t) * TIP_CORRUPT_CP_WORDS, st));
  if (n_bytes == 0) return TIP_OK;
  TIP_REQUIRE(text, "null pointer");
  const int64_t blocks = ct_blocks(n_bytes) < 8 * 1024 ? ct_blocks(n_bytes) : 8 * 1024;
  ct_census_kernel<<<(unsigned)blocks, kCtThreads, 0, st>>>(text, n_bytes, bitmap);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_corrupt_count(const uint8_t* text, const int64_t* text_off, int64_t n_texts, const uint8_t* cls,
                                 int64_t* n_words, void* stream) {
  TIP_REQUIRE(n_texts >= 0 && n_texts < (1LL << 31), "n_texts must be in [0, 2^31)");
  if (n_texts == 0) return TIP_OK;
  TIP_REQUIRE(text && text_off && cls && n_words, "null pointer");
  ct_count_kernel<<<ct_blocks(n_texts), kCtThreads, 0, (cudaStream_t)stream>>>(text, text_off, n_texts, cls, n_words);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_corrupt_texts(const uint8_t* text, const int64_t* text_off, int64_t n_texts, const uint8_t* cls,
                                 const int64_t* word_off, int64_t seed, double severity, const double* type_cdf,
                                 int64_t* w_start, int32_t* w_len, int32_t* w_cps, int32_t* w_text, int64_t* w_seed,
                                 uint8_t* w_flags, int32_t* perm, void* stream) {
  TIP_REQUIRE(n_texts >= 0 && n_texts < (1LL << 31), "n_texts must be in [0, 2^31)");
  TIP_REQUIRE(seed >= 0, "seed must be >= 0");
  TIP_REQUIRE(severity >= 0.0 && severity <= 1.0, "severity must be in [0, 1]");
  TIP_REQUIRE(type_cdf, "null pointer");
  if (n_texts == 0) return TIP_OK;
  TIP_REQUIRE(text && text_off && cls && word_off && w_start && w_len && w_cps && w_text && w_seed && w_flags && perm,
              "null pointer");
  CtTypeCdf cdf;
  for (int k = 0; k < 4; k++) cdf.c[k] = type_cdf[k];
  ct_texts_kernel<<<ct_blocks(n_texts), kCtThreads, 0, (cudaStream_t)stream>>>(
      text, text_off, n_texts, cls, word_off, seed, severity, cdf, CtWords{w_start, w_len, w_cps, w_text}, w_seed,
      w_flags, perm);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_corrupt_words(const uint8_t* text, const int64_t* w_start, const int32_t* w_len, const int32_t* w_cps,
                                 const int64_t* w_seed, const uint8_t* w_flags, int64_t n_words,
                                 const tip_corrupt_table* common, const tip_corrupt_table* bags,
                                 const tip_corrupt_table* thesaurus, uint8_t* o_src, int64_t* o_off, int32_t* o_len,
                                 int64_t* o_typo, int64_t* error_word, void* stream) {
  TIP_REQUIRE(n_words >= 0, "negative size");
  TIP_REQUIRE(ct_table_ok(common) && ct_table_ok(bags) && ct_table_ok(thesaurus), "invalid table");
  TIP_REQUIRE(common->n == 0 || common->val_cdf, "the common-word table needs val_cdf");
  TIP_REQUIRE(error_word, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  TIP_CHECK_CUDA(cudaMemsetAsync(error_word, 0x7f, sizeof(int64_t), st));
  if (n_words == 0) return TIP_OK;
  TIP_REQUIRE(text && w_start && w_len && w_cps && w_seed && w_flags && o_src && o_off && o_len && o_typo, "null pointer");
  TIP_REQUIRE(ct_blocks(n_words) <= 0x7fffffffu, "too many words");
  ct_words_kernel<<<ct_blocks(n_words), kCtThreads, 0, st>>>(
      text, CtWords{const_cast<int64_t*>(w_start), const_cast<int32_t*>(w_len), const_cast<int32_t*>(w_cps), nullptr},
      w_seed, w_flags, n_words, CtTables{*common, *bags, *thesaurus}, o_src, o_off, o_len, o_typo,
      reinterpret_cast<unsigned long long*>(error_word));
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_corrupt_layout(const int64_t* word_off, int64_t n_texts, const int32_t* o_len, const int64_t* o_typo,
                                  int64_t* o_pos, int64_t* text_len, void* stream) {
  TIP_REQUIRE(n_texts >= 0 && n_texts < (1LL << 31), "n_texts must be in [0, 2^31)");
  if (n_texts == 0) return TIP_OK;
  TIP_REQUIRE(word_off && text_len, "null pointer");
  ct_layout_kernel<<<ct_blocks(n_texts), kCtThreads, 0, (cudaStream_t)stream>>>(word_off, n_texts, o_len, o_typo, o_pos,
                                                                               text_len);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}

extern "C" int tip_corrupt_write(const uint8_t* text, const int32_t* w_text, const int64_t* word_off, int64_t n_words,
                                 const tip_corrupt_table* common, const tip_corrupt_table* bags,
                                 const tip_corrupt_table* thesaurus, const uint8_t* o_src, const int64_t* o_off,
                                 const int32_t* o_len, const int64_t* o_typo, const int64_t* o_pos,
                                 const int64_t* out_off, uint8_t* out, void* stream) {
  TIP_REQUIRE(n_words >= 0, "negative size");
  TIP_REQUIRE(ct_table_ok(common) && ct_table_ok(bags) && ct_table_ok(thesaurus), "invalid table");
  if (n_words == 0) return TIP_OK;
  TIP_REQUIRE(text && w_text && word_off && o_src && o_off && o_len && o_typo && o_pos && out_off && out, "null pointer");
  TIP_REQUIRE(ct_blocks(n_words) <= 0x7fffffffu, "too many words");
  ct_write_kernel<<<ct_blocks(n_words), kCtThreads, 0, (cudaStream_t)stream>>>(
      text, w_text, word_off, n_words, CtTables{*common, *bags, *thesaurus}, o_src, o_off, o_len, o_typo, o_pos, out_off,
      out);
  TIP_LAUNCH_CHECK();
  return TIP_OK;
}
