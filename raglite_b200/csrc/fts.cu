// Text analysis of DuckDB's fts index on the GPU: the tokenizer, the english stop list and Snowball's porter stemmer of
// raglite_b200/_fts.py (Analyzer.analyze), bit for bit.
//
// Tokenizer.  lower(strip_accents(text)) can be taken one code point at a time: each code point is a letter a-z, is
// dropped (combining marks and what decomposes into marks only), or is a separator; the caller's class table says which.
// On the stream with the dropped code points removed, a letter is swallowed by the `\\.` alternative exactly when the run
// of backslashes right before it has odd length.  That is a three-state automaton over the code points (SEP: not after a
// kept letter nor an odd backslash run; WORD: after a kept letter; ODD: after an odd run of backslashes), run in parallel
// as a scan of its transition functions: a function of the three states packs into 6 bits, composition is associative.
// fts_tile_fold folds each 4096-byte tile, fts_tile_carry scans the tiles in order, fts_mark replays each thread's bytes
// from its exact entry state.  A byte that is not a lead byte changes nothing (it belongs to its lead's code point).
//
// Stemmer.  One thread per word.  Every step of porter only deletes a suffix of the word and appends a short
// replacement, so a stem is (the first `keep` letters of the word, then at most 8 appended letters packed in a uint64).
// R1, R2, the first vowel and the y -> Y marks come from one pass over the whole word; the marks of its last 32 letters
// are kept, which covers every position the steps read (the steps delete at most 20 letters before step 5a, whose
// short-syllable test reads 4 more).
#include "common.cuh"

namespace rl {
namespace {

constexpr int kFtsThreads = 256;
constexpr int kBytesPerThread = 16;
constexpr int64_t kTileBytes = (int64_t)kFtsThreads * kBytesPerThread;
constexpr int kMaxCodePoint = 0x10FFFF;
constexpr uint8_t kClassDrop = 0xFF;   // class table: 0 separator, 1..26 the letters a..z, 0xFF dropped

__host__ __device__ __forceinline__ int64_t align256(int64_t b) { return (b + 255) / 256 * 256; }
__host__ __device__ __forceinline__ int64_t n_tiles(int64_t n_bytes) { return (n_bytes + kTileBytes - 1) / kTileBytes; }

// ---- the tokenizer automaton ------------------------------------------------------------------------------------------
enum : uint32_t { kSep = 0, kWord = 1, kOdd = 2 };
// f(s) in bits 2s .. 2s+1
constexpr uint32_t kIdentity = 0u | (1u << 2) | (2u << 4);
constexpr uint32_t kOnLetter = kWord | (kWord << 2) | (kSep << 4);        // ODD swallows the letter
constexpr uint32_t kOnBackslash = kOdd | (kOdd << 2) | (kSep << 4);       // a second backslash closes the pair
constexpr uint32_t kOnSep = 0u;

__device__ __forceinline__ uint32_t apply(uint32_t f, uint32_t s) { return (f >> (2 * s)) & 3u; }
// f, then g
__device__ __forceinline__ uint32_t then(uint32_t f, uint32_t g) {
  return apply(g, apply(f, 0)) | (apply(g, apply(f, 1)) << 2) | (apply(g, apply(f, 2)) << 4);
}

struct Sym {
  uint32_t f;       // transition
  uint8_t letter;   // 'a'..'z' when f == kOnLetter
};

// The code point led by byte i (the caller's bytes are UTF-8; anything else is read without leaving the buffer).
__device__ __forceinline__ Sym classify(const uint8_t* __restrict__ text, int64_t n, int64_t i, uint8_t b0,
                                        const uint8_t* __restrict__ cls) {
  if ((b0 & 0xC0) == 0x80) return {kIdentity, 0};
  uint32_t cp;
  int extra;
  if (b0 < 0x80) {
    cp = b0, extra = 0;
  } else if (b0 < 0xE0) {
    cp = b0 & 0x1F, extra = 1;
  } else if (b0 < 0xF0) {
    cp = b0 & 0x0F, extra = 2;
  } else {
    cp = b0 & 0x07, extra = 3;
  }
  for (int k = 1; k <= extra; ++k) cp = (cp << 6) | (i + k < n ? (text[i + k] & 0x3F) : 0);
  if (cp == '\\') return {kOnBackslash, 0};
  const uint8_t c = cp <= (uint32_t)kMaxCodePoint ? __ldg(cls + cp) : 0;
  if (c == kClassDrop) return {kIdentity, 0};
  if (c >= 1 && c <= 26) return {kOnLetter, (uint8_t)('a' + c - 1)};
  return {kOnSep, 0};
}

// Exclusive scan of the threads' functions in thread order; *total = the block's fold.
__device__ uint32_t block_exclusive(uint32_t f, uint32_t* total) {
  __shared__ uint32_t warp_fold[kFtsThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = f;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t up = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc = then(up, inc);
  }
  if (lane == 31) warp_fold[warp] = inc;
  __syncthreads();
  uint32_t before = kIdentity, all = kIdentity;
  for (int w = 0; w < kFtsThreads / 32; ++w) {
    if (w == warp) before = all;
    all = then(all, warp_fold[w]);
  }
  __syncthreads();
  const uint32_t exc_in_warp = __shfl_up_sync(0xffffffffu, inc, 1);
  *total = all;
  return lane == 0 ? before : then(before, exc_in_warp);
}

__device__ __forceinline__ void load_bytes(const uint8_t* __restrict__ text, int64_t n, int64_t i0, uint8_t (&b)[16]) {
  if (i0 + kBytesPerThread <= n && ((uintptr_t)(text + i0) & 15) == 0) {
    const uint4 v = *(const uint4*)(text + i0);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 16; ++k) b[k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
  } else {
#pragma unroll
    for (int k = 0; k < 16; ++k) b[k] = i0 + k < n ? text[i0 + k] : 0x80;   // past the end: changes nothing
  }
}

__device__ __forceinline__ uint32_t thread_fold(const uint8_t* __restrict__ text, int64_t n, int64_t i0,
                                                const uint8_t (&b)[16], const uint8_t* __restrict__ cls) {
  uint32_t f = kIdentity;
#pragma unroll
  for (int k = 0; k < 16; ++k) f = then(f, classify(text, n, i0 + k, b[k], cls).f);
  return f;
}

__global__ void __launch_bounds__(kFtsThreads) fts_tile_fold(const uint8_t* __restrict__ text, int64_t n,
                                                             const uint8_t* __restrict__ cls, uint8_t* __restrict__ fold) {
  const int64_t i0 = blockIdx.x * kTileBytes + (int64_t)threadIdx.x * kBytesPerThread;
  uint8_t b[16];
  load_bytes(text, n, i0, b);
  uint32_t total;
  block_exclusive(thread_fold(text, n, i0, b, cls), &total);
  if (threadIdx.x == 0) fold[blockIdx.x] = (uint8_t)total;
}

// One block: the entry state of every tile, the text starting in SEP.
__global__ void __launch_bounds__(kFtsThreads) fts_tile_carry(const uint8_t* __restrict__ fold, int64_t tiles,
                                                              uint8_t* __restrict__ entry) {
  uint32_t s = kSep;
  for (int64_t t0 = 0; t0 < tiles; t0 += kFtsThreads) {
    const int64_t t = t0 + threadIdx.x;
    uint32_t total;
    const uint32_t before = block_exclusive(t < tiles ? fold[t] : kIdentity, &total);
    if (t < tiles) entry[t] = (uint8_t)apply(before, s);
    s = apply(total, s);
  }
}

// mark[i] = the letter of a kept letter ('a'..'z'; 'A'..'Z' when it starts a word), 0 for every other byte.
__global__ void __launch_bounds__(kFtsThreads) fts_mark(const uint8_t* __restrict__ text, int64_t n,
                                                        const uint8_t* __restrict__ cls, const uint8_t* __restrict__ entry,
                                                        uint8_t* __restrict__ mark) {
  const int64_t i0 = blockIdx.x * kTileBytes + (int64_t)threadIdx.x * kBytesPerThread;
  uint8_t b[16];
  load_bytes(text, n, i0, b);
  uint32_t total;
  const uint32_t before = block_exclusive(thread_fold(text, n, i0, b, cls), &total);
  uint32_t s = apply(before, entry[blockIdx.x]);
  uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const Sym y = classify(text, n, i0 + k, b[k], cls);
    if (y.f == kOnLetter && s != kOdd) w[k >> 2] |= (uint32_t)(s == kSep ? y.letter - 32 : y.letter) << (8 * (k & 3));
    s = apply(y.f, s);
  }
  if (i0 + kBytesPerThread <= n && ((uintptr_t)(mark + i0) & 15) == 0) {
    *(uint4*)(mark + i0) = make_uint4(w[0], w[1], w[2], w[3]);
  } else {
    for (int k = 0; k < 16 && i0 + k < n; ++k) mark[i0 + k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
  }
}

// ---- stop list and stemmer --------------------------------------------------------------------------------------------
struct Stem {   // the current string: word[0 .. keep) then the `na` letters of app, low byte first
  const uint8_t* word;
  int n;
  uint32_t ymask;   // bit k: letter n - 1 - k is marked Y (k < 32)
  int keep, na;
  uint64_t app;

  __device__ __forceinline__ int len() const { return keep + na; }
  __device__ __forceinline__ uint8_t at(int i) const {
    if (i >= keep) return (uint8_t)(app >> (8 * (i - keep)));
    const int k = n - 1 - i;
    return (k < 32 && ((ymask >> k) & 1u)) ? 'Y' : word[i];
  }
  __device__ __forceinline__ void del(int d) {
    if (d <= na) {
      na -= d;
      app &= na ? (~0ull >> (64 - 8 * na)) : 0ull;
    } else {
      keep -= d - na;
      na = 0;
      app = 0;
    }
  }
  __device__ __forceinline__ void add(const char* s) {
    for (; *s; ++s) app |= (uint64_t)(uint8_t)*s << (8 * na++);
  }
  __device__ __forceinline__ bool ends(const char* s, int m) const {
    const int L = len();
    if (m > L) return false;
    for (int j = 0; j < m; ++j)
      if (at(L - m + j) != (uint8_t)s[j]) return false;
    return true;
  }
};

__device__ __forceinline__ bool is_v(uint8_t c) {   // 'aeiouy' (a marked 'Y' is not a vowel)
  return c == 'a' || c == 'e' || c == 'i' || c == 'o' || c == 'u' || c == 'y';
}
__device__ __forceinline__ bool shortv(const Stem& s, int L) {   // non-v_WXY v non-v at the end of the first L letters
  if (L < 3) return false;
  const uint8_t c = s.at(L - 1);
  return !(is_v(c) || c == 'w' || c == 'x' || c == 'Y') && is_v(s.at(L - 2)) && !is_v(s.at(L - 3));
}

struct Rule {
  const char* suf;
  int len;
  const char* rep;
};
__device__ const Rule kStep2[] = {
    {"tional", 6, "tion"}, {"enci", 4, "ence"}, {"anci", 4, "ance"},  {"abli", 4, "able"},  {"entli", 5, "ent"},
    {"eli", 3, "e"},       {"izer", 4, "ize"},  {"ization", 7, "ize"}, {"ational", 7, "ate"}, {"ation", 5, "ate"},
    {"ator", 4, "ate"},    {"alli", 4, "al"},   {"alism", 5, "al"},    {"aliti", 5, "al"},    {"fulness", 7, "ful"},
    {"ousli", 5, "ous"},   {"ousness", 7, "ous"}, {"iveness", 7, "ive"}, {"iviti", 5, "ive"}, {"biliti", 6, "ble"}};
__device__ const Rule kStep3[] = {{"alize", 5, "al"}, {"icate", 5, "ic"}, {"iciti", 5, "ic"}, {"ical", 4, "ic"},
                                  {"ative", 5, ""},   {"ful", 3, ""},     {"ness", 4, ""}};
__device__ const Rule kStep4[] = {{"al", 2, ""},   {"ance", 4, ""}, {"ence", 4, ""}, {"er", 2, ""},  {"ic", 2, ""},
                                  {"able", 4, ""}, {"ible", 4, ""}, {"ant", 3, ""},  {"ement", 5, ""}, {"ment", 4, ""},
                                  {"ent", 3, ""},  {"ou", 2, ""},   {"ism", 3, ""},  {"ate", 3, ""},  {"iti", 3, ""},
                                  {"ous", 3, ""},  {"ive", 3, ""},  {"ize", 3, ""},  {"ion", 3, ""}};

template <int N>
__device__ __forceinline__ int longest(const Stem& s, const Rule (&rules)[N]) {
  int best = -1;
  for (int r = 0; r < N; ++r)
    if ((best < 0 || rules[r].len > rules[best].len) && s.ends(rules[r].suf, rules[r].len)) best = r;
  return best;
}

__device__ void porter(Stem& s) {
  // marks, first vowel, R1 and R2 in one pass (region_after: gopast v, gopast non-v)
  const int n = s.n;
  bool prev_v = false;
  int fv = n, p1 = n, p2 = n, phase = 0;   // phase 0/1: v, then non-v for p1; 2/3 the same for p2; 4 done
  uint32_t ymask = 0;
  for (int i = 0; i < n; ++i) {
    const uint8_t c = s.word[i];
    const bool y = c == 'y' && (i == 0 || prev_v);
    const bool v = !y && is_v(c);
    if (y && n - 1 - i < 32) ymask |= 1u << (n - 1 - i);
    if (v && fv == n) fv = i;
    if (phase == 0 || phase == 2) {
      if (v) ++phase;
    } else if (phase == 1 || phase == 3) {
      if (!v) {
        if (phase == 1) p1 = i + 1;
        else p2 = i + 1;
        ++phase;
      }
    }
    prev_v = v;
  }
  s.ymask = ymask;
  // Step 1a
  if (s.ends("sses", 4) || s.ends("ies", 3)) s.del(2);
  else if (s.ends("s", 1) && !s.ends("ss", 2)) s.del(1);
  // Step 1b (until here only deletions: the string is a prefix of the word, so "a vowel before k" is fv < k)
  if (s.ends("eed", 3)) {
    if (s.len() - 3 >= p1) s.del(1);
  } else {
    const int m = s.ends("ed", 2) ? 2 : s.ends("ing", 3) ? 3 : 0;
    if (m && fv < s.len() - m) {
      s.del(m);
      const int L = s.len();
      const uint8_t last = L ? s.at(L - 1) : 0;
      if (s.ends("at", 2) || s.ends("bl", 2) || s.ends("iz", 2)) {
        s.add("e");
      } else if (L >= 2 && last == s.at(L - 2) &&
                 (last == 'b' || last == 'd' || last == 'f' || last == 'g' || last == 'm' || last == 'n' ||
                  last == 'p' || last == 'r' || last == 't')) {
        s.del(1);
      } else if (L == p1 && shortv(s, L)) {
        s.add("e");
      }
    }
  }
  // Step 1c (a string ending in y holds no appended letter: a prefix of the word again)
  {
    const int L = s.len();
    if (L >= 1 && (s.at(L - 1) == 'y' || s.at(L - 1) == 'Y') && fv < L - 1) {
      s.del(1);
      s.add("i");
    }
  }
  // Steps 2 and 3: the longest listed suffix, replaced when it lies in R1
  int r = longest(s, kStep2);
  if (r >= 0 && s.len() - kStep2[r].len >= p1) {
    s.del(kStep2[r].len);
    s.add(kStep2[r].rep);
  }
  r = longest(s, kStep3);
  if (r >= 0 && s.len() - kStep3[r].len >= p1) {
    s.del(kStep3[r].len);
    s.add(kStep3[r].rep);
  }
  // Step 4: the longest listed suffix, deleted when it lies in R2 ('ion' only after 's' or 't')
  r = longest(s, kStep4);
  if (r >= 0 && s.len() - kStep4[r].len >= p2) {
    const int b = s.len() - kStep4[r].len;
    if (r != 18 || (b >= 1 && (s.at(b - 1) == 's' || s.at(b - 1) == 't'))) s.del(kStep4[r].len);
  }
  // Step 5a / 5b
  {
    const int L = s.len();
    if (s.ends("e", 1) && (L - 1 >= p2 || (L - 1 >= p1 && !shortv(s, L - 1)))) s.del(1);
  }
  if (s.ends("ll", 2) && s.len() - 1 >= p2) s.del(1);
}

// Letters packed big-endian, so that (hi, lo) compares as the zero-padded strings do.
__device__ __forceinline__ bool is_stop(const uint8_t* w, int n, const uint64_t* __restrict__ stop, int n_stop) {
  if (n > 16) return false;
  uint64_t hi = 0, lo = 0;
  for (int i = 0; i < 16; ++i) {
    const uint64_t c = i < n ? w[i] : 0;
    if (i < 8) hi = hi << 8 | c;
    else lo = lo << 8 | c;
  }
  int a = 0, b = n_stop;
  while (a < b) {
    const int m = (a + b) >> 1;
    const uint64_t h = stop[2 * m], l = stop[2 * m + 1];
    if (h < hi || (h == hi && l < lo)) a = m + 1;
    else b = m;
  }
  return a < n_stop && stop[2 * a] == hi && stop[2 * a + 1] == lo;
}

__device__ __forceinline__ uint64_t mix64(uint64_t x) {   // splitmix64's finaliser
  x ^= x >> 30;
  x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27;
  x *= 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

struct StemView {   // stem w of the stem arrays
  const uint8_t* letters;
  const int64_t* word_off;
  const int32_t* keep;
  const uint64_t* tail;
  __device__ __forceinline__ int len(int64_t w) const { return keep[w] + ((71 - __clzll(tail[w])) >> 3); }
  __device__ __forceinline__ uint8_t at(int64_t w, int i) const {
    const int k = keep[w];
    return i < k ? letters[word_off[w] + i] : (uint8_t)(tail[w] >> (8 * (i - k)));
  }
};

__global__ void fts_stem(const uint8_t* __restrict__ letters, const int64_t* __restrict__ word_off, int64_t n_words,
                         const uint64_t* __restrict__ stop, int n_stop, uint64_t hash_mask, int32_t* __restrict__ keep,
                         uint64_t* __restrict__ tail, int64_t* __restrict__ hash) {
  for (int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; w < n_words; w += (int64_t)gridDim.x * blockDim.x) {
    const uint8_t* word = letters + word_off[w];
    const int n = (int)(word_off[w + 1] - word_off[w]);
    if (is_stop(word, n, stop, n_stop)) {
      keep[w] = -1;
      tail[w] = 0;
      hash[w] = 0;
      continue;
    }
    Stem s{word, n, 0u, n, 0, 0ull};
    porter(s);
    uint64_t h = 0xcbf29ce484222325ull;   // FNV-1a over the stem's letters, then mixed
    const int L = s.len();
    for (int i = 0; i < L; ++i) h = (h ^ (i < s.keep ? word[i] : (uint8_t)(s.app >> (8 * (i - s.keep))))) * 0x100000001b3ull;
    keep[w] = s.keep;
    tail[w] = s.app;
    hash[w] = (int64_t)(mix64(h ^ (uint64_t)L) & hash_mask);
  }
}

__global__ void fts_verify(StemView v, const int64_t* __restrict__ word_a, const int64_t* __restrict__ word_b,
                           int64_t n, uint8_t* __restrict__ differ) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t a = word_a[t], b = word_b[t];
    const int L = v.len(a);
    bool d = L != v.len(b);
    for (int i = 0; i < L && !d; ++i) d = v.at(a, i) != v.at(b, i);
    differ[t] = d;
  }
}

__global__ void fts_stem_bytes(StemView v, const int64_t* __restrict__ words, int64_t n,
                               const int64_t* __restrict__ out_off, uint8_t* __restrict__ out) {
  for (int64_t u = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; u < n; u += (int64_t)gridDim.x * blockDim.x) {
    const int64_t w = words[u], o = out_off[u];
    const int L = (int)(out_off[u + 1] - o);
    for (int i = 0; i < L; ++i) out[o + i] = v.at(w, i);
  }
}

__global__ void fts_term_keys(const int64_t* __restrict__ tok_stem, const int64_t* __restrict__ owner, int64_t n,
                              const int32_t* __restrict__ stem_term, int64_t chunk_base, int64_t* __restrict__ key) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x)
    key[t] = ((int64_t)stem_term[tok_stem[t]] << 32) | (chunk_base + owner[t]);
}

int grid_for(int64_t n, int threads) {
  const int64_t b = (n + threads - 1) / threads;
  return (int)(b < 65536 ? (b > 0 ? b : 1) : 65536);
}

}  // namespace
}  // namespace rl

using namespace rl;

extern "C" size_t rl_fts_workspace_bytes(int64_t n_bytes) {
  if (n_bytes < 0) return 0;
  return (size_t)(2 * align256(n_tiles(n_bytes)));
}

extern "C" int rl_fts_mark(const uint8_t* text, int64_t n_bytes, const uint8_t* class_table, uint8_t* mark,
                           void* workspace, size_t workspace_bytes, void* stream) {
  RL_REQUIRE(n_bytes >= 0, RL_EINVAL, "rl_fts_mark: n_bytes >= 0");
  if (n_bytes == 0) return RL_OK;
  RL_REQUIRE(text && class_table && mark && workspace, RL_EINVAL, "rl_fts_mark: null pointer");
  RL_REQUIRE(workspace_bytes >= rl_fts_workspace_bytes(n_bytes), RL_ENOSPACE, "rl_fts_mark: workspace too small");
  const int64_t tiles = n_tiles(n_bytes);
  RL_REQUIRE(tiles <= 0x7fffffff, RL_EINVAL, "rl_fts_mark: n_bytes too large");
  uint8_t* fold = (uint8_t*)workspace;
  uint8_t* entry = fold + align256(tiles);
  cudaStream_t st = (cudaStream_t)stream;
  fts_tile_fold<<<(unsigned)tiles, kFtsThreads, 0, st>>>(text, n_bytes, class_table, fold);
  fts_tile_carry<<<1, kFtsThreads, 0, st>>>(fold, tiles, entry);
  fts_mark<<<(unsigned)tiles, kFtsThreads, 0, st>>>(text, n_bytes, class_table, entry, mark);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_fts_stem(const uint8_t* letters, const int64_t* word_off, int64_t n_words, const uint64_t* stop,
                           int n_stop, int hash_bits, int32_t* keep, uint64_t* tail, int64_t* hash, void* stream) {
  RL_REQUIRE(n_words >= 0 && n_stop >= 0 && hash_bits >= 1 && hash_bits <= 64, RL_EINVAL,
             "rl_fts_stem: n_words, n_stop >= 0 and 1 <= hash_bits <= 64");
  if (n_words == 0) return RL_OK;
  RL_REQUIRE(letters && word_off && keep && tail && hash && (stop || n_stop == 0), RL_EINVAL,
             "rl_fts_stem: null pointer");
  const uint64_t mask = hash_bits == 64 ? ~0ull : (1ull << hash_bits) - 1;
  fts_stem<<<grid_for(n_words, 128), 128, 0, (cudaStream_t)stream>>>(letters, word_off, n_words, stop, n_stop, mask,
                                                                     keep, tail, hash);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_fts_verify(const uint8_t* letters, const int64_t* word_off, const int32_t* keep, const uint64_t* tail,
                             const int64_t* word_a, const int64_t* word_b, int64_t n, uint8_t* differ, void* stream) {
  RL_REQUIRE(n >= 0, RL_EINVAL, "rl_fts_verify: n >= 0");
  if (n == 0) return RL_OK;
  RL_REQUIRE(letters && word_off && keep && tail && word_a && word_b && differ, RL_EINVAL, "rl_fts_verify: null pointer");
  fts_verify<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(StemView{letters, word_off, keep, tail}, word_a, word_b,
                                                                 n, differ);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_fts_stem_bytes(const uint8_t* letters, const int64_t* word_off, const int32_t* keep,
                                 const uint64_t* tail, const int64_t* words, int64_t n, const int64_t* out_off,
                                 uint8_t* out, void* stream) {
  RL_REQUIRE(n >= 0, RL_EINVAL, "rl_fts_stem_bytes: n >= 0");
  if (n == 0) return RL_OK;
  RL_REQUIRE(letters && word_off && keep && tail && words && out_off && out, RL_EINVAL,
             "rl_fts_stem_bytes: null pointer");
  fts_stem_bytes<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(StemView{letters, word_off, keep, tail}, words, n,
                                                                     out_off, out);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_fts_term_keys(const int64_t* tok_stem, const int64_t* owner, int64_t n, const int32_t* stem_term,
                                int64_t chunk_base, int64_t* key, void* stream) {
  RL_REQUIRE(n >= 0 && chunk_base >= 0, RL_EINVAL, "rl_fts_term_keys: n, chunk_base >= 0");
  if (n == 0) return RL_OK;
  RL_REQUIRE(tok_stem && owner && stem_term && key, RL_EINVAL, "rl_fts_term_keys: null pointer");
  fts_term_keys<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(tok_stem, owner, n, stem_term, chunk_base, key);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}
