// Tensor-core scan (RL_ALGO_TCGEN05) for sm_90a: warpgroup MMA (wgmma) with register accumulators.
//
// Replaces the per-row distance expression DuckDB evaluates for vector_search (reference
// _search.py:69-79, _typing.py:123-134) with a coarse tensor-core pass whose survivors are
// re-scored exactly in float64 by the finalize kernel (select_finalize.cu).
//
// One persistent CTA per SM (per SM and query group when B > N) walks its tiles of 128 corpus rows:
//   * 8 loader warps stream the fp32 rows from HBM with coalesced 128-bit loads, scale them (cosine:
//     1/|e|, dot/l2: a global power of two), round to fp16 and store them into a 128B-swizzled
//     K-major shared-memory tile (the wgmma A operand); an fp16-stored corpus comes in through a
//     TMA tensor map instead, with the swizzle applied by the copy engine,
//   * lane 0 of the first loader warp bulk-copies (cp.async.bulk) the matching 64-wide K slice of the
//     pre-swizzled fp16 query image (the wgmma B operand, N = 256 queries for an fp32 corpus with B > 128 and
//     d > 960, else 128) into the same stage,
//   * two consumer warpgroups, 64 corpus rows each, issue wgmma.m64n128k16 (fp32 accumulate in
//     registers; N = 256: two per k step) slice by slice, then turn their accumulators into keys and either dump them (sample
//     tiles) or compare them with the per-query threshold; the few survivors are staged in shared
//     memory together with a histogram of their keys, flushed in bulk (one global atomic per touched
//     query / bin), and the global histogram is read back to tighten the thresholds while the scan is
//     running (online refinement).
// Shared-memory stages are handed over with full / empty mbarriers, so the loaders fill the next stages
// while the consumers run their MMAs and epilogue.
#include <cuda.h>
#include <cuda_fp16.h>

#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "hopper_ptx.cuh"
#include "scan_wgmma.cuh"

namespace rl {

namespace {

using namespace tc;

constexpr int kTileM = 128;           // corpus rows per tile (two warpgroups of M = 64)
constexpr int kSliceK = 64;           // fp16 elements per K slice = one 128-byte swizzle row
// Queries per group = wgmma N, the template parameter NQ: 256 or 128 (query_group_width()).
constexpr int kNumConsumerWarps = 8;  // warps 0..7: warpgroup 0 takes rows 0..63 of a tile, warpgroup 1 rows 64..127
constexpr int kNumConsumers = kNumConsumerWarps * 32;
constexpr int kFirstLoaderWarp = 8;  // its lane 0 also brings the query slices (and, fp16 storage, the corpus tiles)
constexpr int kNumLoaderWarps = 8;
// 512 threads: registers are allocated per four warps, so a 17th warp would cost a whole warpgroup's worth
// and hold every thread to 96 registers.
constexpr int kThreads = (kFirstLoaderWarp + kNumLoaderWarps) * 32;
// NQ = 256: the 128 accumulators of a consumer thread do not fit the 128 registers every thread starts with, so the
// loader warpgroups give registers back (setmaxnreg) and the consumer warpgroups take them: 2 x 72 + 2 x 184 = 4 x 128.
constexpr int kLoaderRegs = 72;
constexpr int kConsumerRegs = 184;
static_assert(kLoaderRegs + kConsumerRegs == 2 * 65536 / kThreads, "the register split must use exactly the CTA's registers");
constexpr int kMaxStages = 8;
constexpr int kABytes = kTileM * 128;  // 16 KB per stage
constexpr uint32_t kSmemBudget = 227 * 1024;
// L2 prefetch distance of the fp32 loaders in K-slice items (32 KB per SM each).  NQ = 256 prefetches nothing: measured
// on an H100 80GB HBM3 at 400 W (c4shard, B = 256), distances of 2, 4, 6, 8 and 12 items made the scan 5, 10, 33, 52
// and 79 % slower than none.
template <int NQ>
__host__ __device__ constexpr int prefetch_items() { return NQ == 128 ? 6 : 0; }
constexpr int kListCap = 1024;         // staged hit records (12 KB)
constexpr int kFlushFirst = 192;       // first flush early: it feeds the histogram that tightens the thresholds
constexpr int kFlushAt = 512;          // later flushes: once this many hits are waiting (or at the end)
constexpr int kRefreshEvery = 16;      // tiles between threshold refreshes from the global histogram
constexpr int kMaxBatchPerLaunch = 1024;   // query groups sharing one launch: 8 of 128 or 4 of 256

// Query-group width (the qimg layout and the launch both follow it).  256 removes the duplicated fp32 -> fp16
// conversion of B > 128: one CTA per lane converts each tile once for 256 queries.  It needs an fp32 corpus (fp16 rows
// come in through TMA, unconverted) and long tiles: with 4 stages instead of 6, a tile of fewer than 16 K slices
// cannot hide the 256-column epilogue.  Measured on an H100 80GB HBM3 at 400 W: 1.26x / 1.35x faster at d = 1024 (c4shard,
// c3), 1.3x slower at d = 384 (c2), 1.5x slower with fp16 storage at d = 1024.
inline int query_group_width(const rl_scan_params* p) {
  const int n_ks = (p->d + kSliceK - 1) / kSliceK;
  return (p->B > 128 && p->e_dtype != 1 && n_ks >= 16) ? 256 : 128;
}

struct TcArgs {
  ScanArgs a;
  const __half* qimg;     // [groups][n_ks][NQ][64] fp16, rows pre-swizzled
  const float* q_scale;   // [B] key = acc * q_scale[b] (+ bias)
  const float* row_stats; // [4] max norm, max |element|, min norm, flags
  int nq;                 // padded #queries of a full group (multiple of 16; NQ when par_groups > 1)
  int nq_last;            // padded #queries of the last group
  int par_groups;         // CTA c serves query group c % par_groups of the tiles of lane c / par_groups
  int n_ks;               // K slices
  int stages;
};

// Narrows `a` to its queries q0, q0 + 1, ...; the caller sets B.
__host__ __device__ __forceinline__ void slice_queries(ScanArgs& a, int q0) {
  a.thr += q0; a.cand_cnt += q0; a.eps += q0; a.hist_inv_w += q0; a.q_inv_norm += q0;
  if (a.cnt_all != nullptr) a.cnt_all += q0;
  a.dump += (size_t)q0 * a.n_sample_rows;
  a.cand += (size_t)q0 * a.cap;
  a.ghist += (size_t)q0 * kHistBins;
}

// Global power-of-two row scale for the dot / l2 metrics (keeps |x| <= 1 in fp16).
__device__ __forceinline__ float pow2_scale(float max_abs) {
  return max_abs > 0.f ? exp2f(-ceilf(log2f(max_abs))) : 1.f;
}

// Cosine on a corpus whose rows all have norm >= 0.5 and moderate magnitudes (the normal case:
// embeddings are stored normalised): rows go to fp16 unscaled and the epilogue applies 1/|e|.
// Each role evaluates this for itself: a value computed at kernel scope and kept live into the roles would cost
// registers the NQ = 256 loaders do not have.
template <int METRIC, bool EF16>
__device__ __forceinline__ bool cos_noscale_of(const float* row_stats) {
  return METRIC == RL_METRIC_COSINE &&
         (EF16 || (row_stats[2] > 0.f && row_stats[2] <= 2.f && row_stats[1] <= 1024.f &&
                   row_stats[3] == 0.f));   // (the host only allows fp16 storage when this holds)
}

// A tile of this CTA: its first corpus row and its row count (kTileM, fewer in the shard's last block).
struct TileGeom {
  int64_t row0;
  int rows;
};

// The tiles of a CTA: its lane walks the launch's blocks ord = first, first + stride, ... (count of them).
// Tile counts and block indices stay below 2^24 (n_rows < 2^31), so they are computed in 32 bits: a 64-bit
// division is a subroutine call whose registers the loaders cannot spare at NQ = 256.
struct CtaTiles {
  uint32_t first, stride;
  int64_t count;
  __device__ __forceinline__ CtaTiles(uint32_t n_tiles, uint32_t P)
      : first(blockIdx.x / P), stride(gridDim.x / P), count(first < n_tiles ? (n_tiles - first + stride - 1) / stride : 0) {}
  __device__ __forceinline__ uint32_t ord(int64_t tile) const { return first + (uint32_t)tile * stride; }
  __device__ __forceinline__ TileGeom geom(const ScanArgs& a, int64_t tile) const {
    const uint32_t o = ord(tile), S = (uint32_t)a.S;
    const int64_t blk = a.dump_mode ? o * S : (S <= 1u ? o : o + o / (S - 1u) + 1u);   // mode_block_index() in 32 bits
    const int64_t rem = a.n_rows - blk * kTileM;
    return {blk * kTileM, rem < kTileM ? (int)rem : kTileM};
  }
};

struct SmemLayout {
  uint64_t* full;             // [kMaxStages]
  uint64_t* empty;            // [kMaxStages]
  float* thr;                 // [NQ]
  float* cs;                  // [NQ]
  float* thr0;                // [NQ] threshold from the sample (histogram origin)
  float* inv_w;               // [NQ] 1 / bin width (bin width = 4 eps)
  uint32_t* hist;             // [NQ * kHistBins / 2] staged histogram, two 16-bit counters per word
  int* cnt;                   // [NQ] hits per query staged since the last flush
  int* basev;                 // [NQ] global slot base per query for the current flush
  int* list_n;                // [4] number of staged records
  uint32_t* list;             // [kListCap][3] {col | rank << 16, key bits, row}
  unsigned char* stage_base;  // stages * stage_bytes<NQ>(), after the above (tail_bytes<NQ>())
};

// A stage: the corpus slice of a tile (A) and room for the query slice of a FULL group (B, NQ rows of 128 bytes).
// The wgmma always reads all NQ rows of B; a group of nq < NQ queries only copies nq rows, so rows nq..NQ-1
// hold whatever an earlier slice left there.  They only feed accumulator columns >= nq, which the epilogue never reads,
// and they lie inside the stage, so the MMA never reads another stage or the barriers.
template <int NQ>
__host__ __device__ constexpr uint32_t stage_bytes() { return kABytes + NQ * 128u; }
template <int NQ>
__host__ __device__ constexpr uint32_t tail_bytes() {
  return 2 * kMaxStages * 8 + NQ * (6u * 4u + (uint32_t)kHistBins * 2u) + 16 + kListCap * 12;
}

// (first loader thread, fp32 storage) the query half of a stage: one arrive with the byte count, one bulk copy of
// K slice ks of the group's queries (qbytes bytes each)
template <int NQ>
__device__ __forceinline__ void put_query(const SmemLayout& s, int stage, const unsigned char* qsrc, uint32_t qbytes, int ks) {
  mbar_arrive_expect_tx(&s.full[stage], qbytes);
  bulk_g2s(s.stage_base + (size_t)stage * stage_bytes<NQ>() + kABytes, qsrc + (size_t)ks * qbytes, qbytes, &s.full[stage]);
}

// fp32 loaders: loader thread lt holds float4 column c4 = lt % 16 of rows r0 + 16 i (r0 = lt / 16, i = 0..7) of a K
// slice.  Those rows all have r & 7 == r0 & 7, so they share one 128B-swizzled offset in the stage, i * 2 KB apart.
__device__ __forceinline__ uint32_t swizzled_offset(int r0, int c4) {
  return (uint32_t)r0 * 128u + ((((uint32_t)c4 >> 1) ^ ((uint32_t)r0 & 7u)) << 4) + (((uint32_t)c4 & 1u) << 3);
}
__device__ __forceinline__ float4 scaled(float4 v, float s) { return make_float4(v.x * s, v.y * s, v.z * s, v.w * s); }
// Rounds the thread's eight float4 to fp16 and stores them at dst = stage + swizzled_offset(r0, c4).
__device__ __forceinline__ void store_f16_rows(unsigned char* dst, const float4 (&v)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const __half2 h01 = __floats2half2_rn(v[i].x, v[i].y);
    const __half2 h23 = __floats2half2_rn(v[i].z, v[i].w);
    uint2 packed;
    packed.x = *reinterpret_cast<const uint32_t*>(&h01);
    packed.y = *reinterpret_cast<const uint32_t*>(&h23);
    *reinterpret_cast<uint2*>(dst + i * 16 * 128) = packed;
  }
}

// fp32 loader cursors: `ptr` at float column col of row `row` of this CTA's tile `tile` and the tile's row count, or
// rows = 0 past its last tile.  The prefetch cursor (pf: only the first CTA of a lane pulls a tile from HBM) also
// prefetches the tile's cosine row scales.
__device__ __forceinline__ void ld_cursor_at(const ScanArgs& a, const CtaTiles& tiles, int64_t tile, int row, int col,
                                             int& rows, const unsigned char*& ptr) {
  rows = 0;
  if (tile < tiles.count) {
    const TileGeom g = tiles.geom(a, tile);
    rows = g.rows;
    ptr = reinterpret_cast<const unsigned char*>(a.E + (size_t)(g.row0 + row) * a.ld + col);
  }
}
template <int METRIC>
__device__ __forceinline__ void pf_cursor_at(const ScanArgs& a, const CtaTiles& tiles, int64_t tile, bool lead, int lt,
                                             int& rows, const unsigned char*& ptr) {
  rows = 0;
  if (lead && tile < tiles.count) {
    const TileGeom g = tiles.geom(a, tile);
    rows = g.rows;
    ptr = reinterpret_cast<const unsigned char*>(a.E + (size_t)(g.row0 + (lt >> 1)) * a.ld + (lt & 1) * 32);
    if (METRIC == RL_METRIC_COSINE && lt < 4 && lt * 32 < rows) prefetch_l2(a.inv_norm + g.row0 + lt * 32);
  }
}

// ===== fp16 storage through the tensor map: one thread issues, per K slice, the TMA copy of the corpus tile (the
// engine writes the 128B-swizzled layout itself) and the bulk copy of the query slice; the other loader warps idle.
// `lead`: this CTA is the first of its lane, the one that prefetches the tiles into L2.
template <int NQ>
__device__ __forceinline__ void tma_producer(const SmemLayout& s, const TcArgs& t, const ScanArgs& a, const CtaTiles& tiles,
                                             const CUtensorMap& tmE, const unsigned char* qsrc, uint32_t qbytes, bool lead) {
  if constexpr (NQ == 256) setmaxnreg_dec<kLoaderRegs>();
  if (threadIdx.x != kFirstLoaderWarp * 32) return;
  constexpr uint32_t sbytes = stage_bytes<NQ>();
  const int64_t total_items = tiles.count * t.n_ks;
  int ks = 0, stage = 0;
  uint32_t phase = 0;
  // row0 of the current tile and of the next one, whose slices are prefetched into L2 one tile (n_ks slices =
  // 128 KB per SM at d = 1024) ahead
  int64_t tile = 0;
  auto tile_row0 = [&](int64_t v) -> int { return v < tiles.count ? (int)tiles.geom(a, v).row0 : -1; };
  int row0 = tile_row0(0), row0_next = tile_row0(1);
  for (int64_t item = 0; item < total_items; ++item) {
    mbar_wait(&s.empty[stage], phase ^ 1u);
    mbar_arrive_expect_tx(&s.full[stage], qbytes + (uint32_t)kABytes);
    tma_load_2d(s.stage_base + (size_t)stage * sbytes, &tmE, ks * kSliceK, row0, &s.full[stage]);
    bulk_g2s(s.stage_base + (size_t)stage * sbytes + kABytes, qsrc + (size_t)ks * qbytes, qbytes, &s.full[stage]);
    if (row0_next >= 0 && lead) tma_prefetch_2d(&tmE, ks * kSliceK, row0_next);
    if (++ks == t.n_ks) { ks = 0; ++tile; row0 = row0_next; row0_next = tile_row0(tile + 1); }
    if (++stage == t.stages) { stage = 0; phase ^= 1u; }
  }
}

// ===== corpus loaders, fp32 storage, fast path (d % 128 == 0, no per-row scale) =====
// Same data movement as the generic loader below -- HBM fp32 -> registers -> cvt.rn.f16x2 -> 128B-swizzled smem
// tile; NQ = 128: two K-slice items (64 KB per SM) in flight and an L2 prefetch ahead, NQ = 256: one item and no
// prefetch -- with the bookkeeping cut down: an iteration handles the PAIR of items (ks, ks + 1): one cursor step, row
// pointers with a 32-bit pitch shared by both items through a +256 B immediate, smem / barrier addresses kept
// incrementally.
template <int METRIC, int NQ>
__device__ __forceinline__ void fp32_fast_producer(const SmemLayout& s, const TcArgs& t, const ScanArgs& a,
                                                   const CtaTiles& tiles, const unsigned char* qsrc, uint32_t qbytes,
                                                   bool lead) {
  if constexpr (NQ == 256) setmaxnreg_dec<kLoaderRegs>();
  constexpr uint32_t sbytes = stage_bytes<NQ>();
  constexpr int kPfPairs = prefetch_items<NQ>() / 2;   // L2 prefetch distance in pairs of items
  const int lane = threadIdx.x & 31;
  const bool q_thread = threadIdx.x == kFirstLoaderWarp * 32;
  const int lt = threadIdx.x - kFirstLoaderWarp * 32;  // 0..255
  const int c4 = lt & 15;                              // float4 column within the 64-wide K slice
  const int r0 = lt >> 4;                              // rows r0 + 16 i, i = 0..7
  const float gscale = (METRIC == RL_METRIC_COSINE) ? 1.f : pow2_scale(t.row_stats[1]);
  const bool mul = gscale != 1.f;
  uint32_t n_ks = (uint32_t)t.n_ks, n_stages = (uint32_t)t.stages;
  uint32_t pitch16 = (uint32_t)(a.ld * 16 * (int64_t)sizeof(float));   // bytes between this thread's consecutive rows
  uint32_t sw_off = swizzled_offset(r0, c4);
  // opaque moves: keep these in registers instead of re-deriving them from %tid / the parameter bank per item
  asm volatile("" : "+r"(n_ks), "+r"(n_stages), "+r"(pitch16), "+r"(sw_off));
  // (32 bits: an item is 32 KB of a corpus that fits in device memory)
  const uint32_t total_items = (uint32_t)tiles.count * n_ks;

  struct Cursor { int64_t tile; uint32_t ks; int rows; const unsigned char* ptr; };
  // Load cursor: this thread's row r0 / column c4 of the NEXT pair of items to load.
  Cursor ld{0, 0u, 0, nullptr};
  auto ld_set_tile = [&]() { ld_cursor_at(a, tiles, ld.tile, r0, c4 * 4, ld.rows, ld.ptr); };
  // Prefetch cursor (L2 only, kPfPairs > 0): thread lt covers row lt / 2, 128-byte half lt % 2 of a 256-byte slice.
  Cursor pf{0, 0u, 0, nullptr};
  auto pf_set_tile = [&]() { pf_cursor_at<METRIC>(a, tiles, pf.tile, lead, lt, pf.rows, pf.ptr); };
  auto pf_pair = [&]() {
    if ((lt >> 1) < pf.rows) { prefetch_l2(pf.ptr); prefetch_l2(pf.ptr + 256); }
    pf.ptr += 512;
    pf.ks += 2;
    if (pf.ks == n_ks) { pf.ks = 0; ++pf.tile; pf_set_tile(); }
  };
  float4 ringA[8], ringB[8];
  auto issue = [&](float4 (&buf)[8], int rows, const unsigned char* src) {   // src: row r0 of the item
    if (rows == kTileM) {   // full tile: no per-row predicates
#pragma unroll
      for (int i = 0; i < 8; ++i) buf[i] = ldg_stream(reinterpret_cast<const float*>(src + (size_t)((uint32_t)i * pitch16)));
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (r0 + 16 * i < rows) buf[i] = ldg_stream(reinterpret_cast<const float*>(src + (size_t)((uint32_t)i * pitch16)));
        else buf[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  };
  uint32_t stage = 0, phase = 0, st_ks = 0;
  unsigned char* a_dst = s.stage_base + sw_off;
  auto store = [&](float4 (&buf)[8]) {   // (buf is refilled right after)
    mbar_wait(&s.empty[stage], phase ^ 1u);
    if (q_thread) put_query<NQ>(s, (int)stage, qsrc, qbytes, (int)st_ks);
    if (++st_ks == n_ks) st_ks = 0;
    if (mul) {
#pragma unroll
      for (int i = 0; i < 8; ++i) buf[i] = scaled(buf[i], gscale);
    }
    store_f16_rows(a_dst, buf);
    // (no proxy fence here, see the generic loader: the consumers fence after acquiring the barrier)
    __syncwarp();
    if (lane == 0) mbar_arrive(&s.full[stage]);
    a_dst += sbytes;
    if (++stage == n_stages) { stage = 0; phase ^= 1u; a_dst = s.stage_base + sw_off; }
  };

  ld_set_tile();
  if constexpr (kPfPairs > 0) {
    pf_set_tile();
    for (int i = 0; i < kPfPairs + 1; ++i) pf_pair();   // the load cursor starts one pair ahead of the stores
  }
  if constexpr (NQ == 128) {
    issue(ringA, ld.rows, ld.ptr);
    issue(ringB, ld.rows, ld.ptr + 256);
    for (uint32_t item = 0; item < total_items; item += 2) {
      // advance the load cursor to the next pair (possibly the first pair of the next tile)
      ld.ptr += 512;
      ld.ks += 2;
      if (ld.ks == n_ks) { ld.ks = 0; ++ld.tile; ld_set_tile(); }
      const int rows = ld.rows;
      const unsigned char* src = ld.ptr;
      store(ringA);
      issue(ringA, rows, src);
      store(ringB);
      issue(ringB, rows, src + 256);
      if constexpr (kPfPairs > 0) pf_pair();
    }
  } else {
    // kLoaderRegs registers hold one item (32 KB per SM in flight)
    issue(ringA, ld.rows, ld.ptr);
    for (uint32_t item = 0; item < total_items; item += 2) {
      const int rows = ld.rows;             // the pair being stored
      const unsigned char* src = ld.ptr;
      ld.ptr += 512;
      ld.ks += 2;
      if (ld.ks == n_ks) { ld.ks = 0; ++ld.tile; ld_set_tile(); }
      store(ringA);
      issue(ringA, rows, src + 256);
      store(ringA);
      issue(ringA, ld.rows, ld.ptr);
      if constexpr (kPfPairs > 0) pf_pair();
    }
  }
}

// ===== corpus loaders: HBM fp32 -> registers -> fp16 -> swizzled smem (wgmma A operand) =====
template <int METRIC, int NQ>
__device__ __forceinline__ void fp32_generic_producer(const SmemLayout& s, const TcArgs& t, const ScanArgs& a,
                                                      const CtaTiles& tiles, const unsigned char* qsrc, uint32_t qbytes,
                                                      bool lead) {
  if constexpr (NQ == 256) setmaxnreg_dec<kLoaderRegs>();
  const int lane = threadIdx.x & 31;
  const bool q_thread = threadIdx.x == kFirstLoaderWarp * 32;
  const int lt = threadIdx.x - kFirstLoaderWarp * 32;  // 0..255
  const int c4 = lt & 15;                              // float4 column within the 64-wide K slice
  const int r0 = lt >> 4;                              // rows r0 + 16 i, i = 0..7
  const float gscale = (METRIC == RL_METRIC_COSINE) ? 1.f : pow2_scale(t.row_stats[1]);
  // Rows are converted without a multiply when no scaling is needed (normalised corpora: the
  // cosine 1/|e| then moves to the epilogue; dot/l2: the global scale is 1).
  const bool noscale = (METRIC == RL_METRIC_COSINE) ? cos_noscale_of<METRIC, false>(t.row_stats) : (gscale == 1.f);
  const uint32_t total_items = (uint32_t)tiles.count * (uint32_t)t.n_ks;   // (32 bits, as in the fast path)
  constexpr int kInFlight = NQ == 128 ? 2 : 1;   // items held in registers (NQ = 256: kLoaderRegs has room for one)
  float4 ring[kInFlight][8];
  float rs[8];

  // Incremental cursors (no integer divisions or multiplies on the hot path).  `ld_*` runs kInFlight items
  // ahead of `st_*`; `pf_*` runs prefetch_items<NQ>() ahead of `ld_*` and only touches L2.
  const size_t pitch16_bytes = (size_t)a.ld * 16 * sizeof(float);   // between this thread's consecutive rows
  const size_t slice_bytes = kSliceK * sizeof(float);
  int64_t ld_tile = 0;
  int ld_ks = 0, ld_rows = 0;
  const unsigned char* ld_ptr = nullptr;                 // row r0 of the tile, column c4*4 + ld_ks*64
  auto ld_set_tile = [&]() { ld_cursor_at(a, tiles, ld_tile, r0, c4 * 4, ld_rows, ld_ptr); };
  // One 128-byte line per thread and item: thread lt covers row lt/2, half lt%2 of the 256-byte slice.
  int64_t pf_tile = 0;
  int pf_ks = 0, pf_rows = 0;
  const unsigned char* pf_ptr = nullptr;
  auto pf_set_tile = [&]() { pf_cursor_at<METRIC>(a, tiles, pf_tile, lead, lt, pf_rows, pf_ptr); };
  auto prefetch_item = [&]() {
    if ((lt >> 1) < pf_rows && pf_ks * kSliceK + (lt & 1) * 32 < a.d) prefetch_l2(pf_ptr);
    pf_ptr += slice_bytes;
    if (++pf_ks == t.n_ks) {
      pf_ks = 0;
      ++pf_tile;
      pf_set_tile();
    }
  };
  auto issue_item = [&](float4 (&buf)[8]) {
    const bool col_ok = ld_ks * kSliceK + c4 * 4 < a.d;
    const int rows_left = ld_rows - r0;   // (one register for the eight row predicates below)
    const unsigned char* p = ld_ptr;
    if (col_ok && ld_rows == kTileM) {   // full tile: no per-row predicates
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        buf[i] = ldg_stream(reinterpret_cast<const float*>(p));
        p += pitch16_bytes;
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (col_ok && 16 * i < rows_left) buf[i] = ldg_stream(reinterpret_cast<const float*>(p));
        else buf[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        p += pitch16_bytes;
      }
    }
    ld_ptr += slice_bytes;
    if (++ld_ks == t.n_ks) {
      ld_ks = 0;
      ++ld_tile;
      ld_set_tile();
    }
    if constexpr (prefetch_items<NQ>() > 0) prefetch_item();
  };

  int64_t st_tile = 0;
  int st_ks = 0, stage = 0;
  uint32_t phase = 0;
  // Row scales of a tile are (re)loaded right after the last item of the previous tile has been
  // converted; their latency overlaps the arrive, the next loads and the next barrier wait.
  auto fetch_scales = [&](int64_t tile) {
#pragma unroll
    for (int i = 0; i < 8; ++i) rs[i] = (METRIC == RL_METRIC_COSINE) ? 0.f : gscale;
    if (METRIC == RL_METRIC_COSINE && !noscale && tile < tiles.count) {
      const TileGeom g = tiles.geom(a, tile);
      const int rows_left = g.rows - r0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (16 * i < rows_left) rs[i] = __ldg(a.inv_norm + g.row0 + r0 + 16 * i);
      }
    }
  };
  const uint32_t sw_off = swizzled_offset(r0, c4);
  // Convert + store one item, then refill its register slots with the loads of the item kInFlight
  // ahead: kInFlight stage-loads (32 KB per SM each) stay in flight.
  auto process = [&](float4 (&buf)[8]) {
    mbar_wait(&s.empty[stage], phase ^ 1u);
    if (q_thread) put_query<NQ>(s, stage, qsrc, qbytes, st_ks);
    unsigned char* A = s.stage_base + (size_t)stage * stage_bytes<NQ>() + sw_off;
    if (!noscale) {
#pragma unroll
      for (int i = 0; i < 8; ++i) buf[i] = scaled(buf[i], rs[i]);
    }
    store_f16_rows(A, buf);
    // No proxy fence here: a fence in a thread with global loads in flight stalls until they land and
    // collapses the loaders' memory-level parallelism.  The stores are released by the mbarrier arrive;
    // the consumers acquire the barrier and execute fence.proxy.async before they issue wgmma.
    __syncwarp();
    if (lane == 0) mbar_arrive(&s.full[stage]);
    issue_item(buf);
    if (++stage == t.stages) { stage = 0; phase ^= 1u; }
    if (++st_ks == t.n_ks) { st_ks = 0; ++st_tile; fetch_scales(st_tile); }
  };

  fetch_scales(0);
  ld_set_tile();
  pf_set_tile();
  for (int i = 0; i < prefetch_items<NQ>(); ++i) prefetch_item();
  for (int i = 0; i < kInFlight; ++i) issue_item(ring[i]);
  for (uint32_t item = 0; item < total_items; item += kInFlight) {
    process(ring[0]);
    if constexpr (kInFlight == 2) {
      if (item + 1 < total_items) process(ring[1]);
    }
  }
}

// ===== consumer warpgroups (warps 0..7): wgmma over the K slices, then the epilogue from registers =====

// One tile's MMAs: one stage per K slice; a stage is released once the wgmma of the next slice is in flight.
template <int NQ>
__device__ __forceinline__ void mma_tile(const SmemLayout& s, const TcArgs& t, float (&acc)[NQ / 2], int& stage,
                                         uint32_t& phase) {
  const int wg = threadIdx.x >> 7;   // rows wg * 64 .. wg * 64 + 63 of the tile
  const int lane = threadIdx.x & 31;
  int prev = -1;
  for (int ks = 0; ks < t.n_ks; ++ks) {
    mbar_wait(&s.full[stage], phase);
    fence_proxy_async();   // generic-proxy smem stores of the loaders -> async-proxy (wgmma) reads
    const uint32_t st_addr = smem_u32(s.stage_base + (size_t)stage * stage_bytes<NQ>());
    wgmma_fence();
    wgmma_slice(acc, make_kmajor_sw128_desc(st_addr + (uint32_t)wg * (64u * 128u)), make_kmajor_sw128_desc(st_addr + kABytes),
                ks > 0);
    wgmma_commit();
    if (prev >= 0) {
      wgmma_wait<1>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&s.empty[prev]);
    }
    prev = stage;
    if (++stage == t.stages) { stage = 0; phase ^= 1u; }
  }
  wgmma_wait<0>();
  __syncwarp();
  if (lane == 0) mbar_arrive(&s.empty[prev]);
}

// The per-row terms of a key: l2 adds the row's -|e|^2, cosine on unscaled rows multiplies by its 1/|e|.
struct RowTerms {
  float bias, scale;
};
template <int METRIC>
__device__ __forceinline__ RowTerms row_terms(const ScanArgs& a, bool cos_noscale, bool keyed, int64_t row) {
  return {(METRIC == RL_METRIC_L2 && keyed) ? -a.sq_norm[row] : 0.f,
          (METRIC == RL_METRIC_COSINE && cos_noscale && keyed) ? __ldg(a.inv_norm + row) : 1.f};
}
template <int METRIC>
__device__ __forceinline__ float key_of(float acc, float cs, RowTerms r) {
  return METRIC != RL_METRIC_COSINE ? fmaf(acc, cs, r.bias) : acc * r.scale;
}

// Accumulators -> keys: dumped (sample tiles) or compared with the per-query thresholds, the hits staged in shared
// memory.  Rows r_lo and r_lo + 8 of the tile, columns 8 c8 + c_lane + {0, 1} of the accumulator.
template <int METRIC, int NQ>
__device__ __forceinline__ void epilogue(const SmemLayout& s, const ScanArgs& a, const CtaTiles& tiles, int64_t tile,
                                         const float (&acc)[NQ / 2], int nq, bool cos_noscale) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r_lo = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);
  const int c_lane = 2 * (lane & 3);
  const TileGeom g = tiles.geom(a, tile);
  int r_in[2];
  int64_t row[2];
  bool valid[2], masked_alive[2];
  RowTerms terms[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    r_in[h] = r_lo + 8 * h;
    row[h] = g.row0 + r_in[h];
    valid[h] = row[h] < a.n_rows;
    // rows the metadata filter masks out but that exist (not tombstoned): counted against the threshold when the
    // caller asks for the rank-then-filter bound (rl_maxsim_unfiltered_bound)
    masked_alive[h] = false;
    if (valid[h] && a.row_allowed != nullptr) {
      valid[h] = a.row_allowed[row[h]] != 0;
      if (!valid[h] && a.cnt_all != nullptr) masked_alive[h] = a.row_alive == nullptr || a.row_alive[row[h]] != 0;
    }
    terms[h] = row_terms<METRIC>(a, cos_noscale, valid[h], row[h]);
  }
  if (a.dump_mode) {
    const int64_t ord = tiles.ord(tile);
#pragma unroll
    for (int c8 = 0; c8 < NQ / 8; ++c8) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int h = e >> 1, col = 8 * c8 + c_lane + (e & 1);
        if (col < a.B) {
          const float key = key_of<METRIC>(acc[4 * c8 + e], s.cs[col], terms[h]);
          a.dump[(size_t)col * a.n_sample_rows + ord * kTileM + r_in[h]] = valid[h] ? key : kNegInf;
        }
      }
    }
    return;
  }
#pragma unroll
  for (int c8 = 0; c8 < NQ / 8; ++c8) {
    if (8 * c8 >= nq) break;
    const int c = 8 * c8 + c_lane;
    const float2 th = *reinterpret_cast<const float2*>(s.thr + c);
    const float2 sc = METRIC != RL_METRIC_COSINE ? *reinterpret_cast<const float2*>(s.cs + c) : make_float2(0.f, 0.f);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int h = e >> 1, col = c + (e & 1);
      const float key = key_of<METRIC>(acc[4 * c8 + e], (e & 1) ? sc.y : sc.x, terms[h]);
      if (key >= ((e & 1) ? th.y : th.x)) {   // rare: a few hits per tile
        if (valid[h]) {
          // Stage the hit in shared memory (one returning atomic for the slot; the histogram update
          // does not wait); per-query ranks and global slots are handed out in bulk at the flush.
          const int pos = atomicAdd(&s.list_n[0], 1);
          const int hb = col * kHistBins + hist_bin(key, s.thr0[col], s.inv_w[col]);
          atomicAdd(&s.hist[hb >> 1], 1u << ((hb & 1) * 16));
          if (pos < kListCap) {
            s.list[pos * 3 + 0] = (uint32_t)col;
            s.list[pos * 3 + 1] = __float_as_uint(key);
            s.list[pos * 3 + 2] = (uint32_t)row[h];
          } else {
            emit_candidate(a, col, key, (int32_t)row[h]);
          }
        }
      }
    }
  }
  if (masked_alive[0] || masked_alive[1]) {
    // Rows the filter masks out but that exist are counted against the threshold with their own key (the loop
    // above keys them without the row's -|e|^2 or 1/|e|); only RL_FLAG_COUNT_UNFILTERED on a filtered scan gets here.
    RowTerms mterms[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) mterms[h] = row_terms<METRIC>(a, cos_noscale, masked_alive[h], row[h]);
#pragma unroll
    for (int c8 = 0; c8 < NQ / 8; ++c8) {
      if (8 * c8 >= nq) break;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int h = e >> 1, col = 8 * c8 + c_lane + (e & 1);
        const float key = key_of<METRIC>(acc[4 * c8 + e], s.cs[col], mterms[h]);
        if (masked_alive[h] && key >= s.thr[col]) atomicAdd(a.cnt_all + col, 1);
      }
    }
  }
}

// The n staged hits go out in bulk: one global atomic per query that was hit since the previous flush (the base of
// its slots), plus the staged histogram.
template <int NQ>
__device__ __forceinline__ void flush_staged(const SmemLayout& s, const ScanArgs& a, int n) {
  const int et = threadIdx.x;   // 0..255
  for (int e = et; e < n; e += kNumConsumers) {   // rank of every staged hit within its query
    const int col = (int)s.list[e * 3 + 0];
    s.list[e * 3 + 0] = (uint32_t)col | ((uint32_t)atomicAdd(&s.cnt[col], 1) << 16);
  }
  named_bar_sync(1, kNumConsumers);
  for (int col = et; col < NQ; col += kNumConsumers) {
    const int c = s.cnt[col];
    if (c > 0) {
      s.basev[col] = atomicAdd(a.cand_cnt + col, c);
      s.cnt[col] = 0;
    }
  }
  for (int w = et; w < NQ * kHistBins / 2; w += kNumConsumers) {
    const uint32_t h = s.hist[w];
    if (h != 0u) {
      if (h & 0xFFFFu) atomicAdd(a.ghist + 2 * w, (int)(h & 0xFFFFu));
      if (h >> 16) atomicAdd(a.ghist + 2 * w + 1, (int)(h >> 16));
      s.hist[w] = 0u;
    }
  }
  named_bar_sync(1, kNumConsumers);
  if (et == 0) s.list_n[0] = 0;
  for (int e = et; e < n; e += kNumConsumers) {
    const uint32_t w0 = s.list[e * 3 + 0];
    const int col = (int)(w0 & 0xFFFFu);
    const int slot = s.basev[col] + (int)(w0 >> 16);
    if (slot < a.cap)
      a.cand[(size_t)col * a.cap + slot] = Cand{__uint_as_float(s.list[e * 3 + 1]), (int32_t)s.list[e * 3 + 2]};
  }
}

// Threshold refresh: the highest bin edge with >= sel_count candidates at or above it (all CTAs' hits so far)
// bounds the sel_count-th best key from below; emit from 2 eps under it.
__device__ __forceinline__ void refresh_thresholds(const SmemLayout& s, const ScanArgs& a) {
  for (int col = threadIdx.x; col < a.B; col += kNumConsumers) {
    const int4* gh = reinterpret_cast<const int4*>(a.ghist + (size_t)col * kHistBins);
    int cnts[kHistBins];
#pragma unroll
    for (int q4 = 0; q4 < kHistBins / 4; ++q4) {
      const int4 v4 = __ldcg(gh + q4);
      cnts[4 * q4] = v4.x; cnts[4 * q4 + 1] = v4.y; cnts[4 * q4 + 2] = v4.z; cnts[4 * q4 + 3] = v4.w;
    }
    int cum = 0, best = -1;
#pragma unroll
    for (int bb = kHistBins - 1; bb >= 1; --bb) {
      cum += cnts[bb];
      if (best < 0 && cum >= a.sel_count) best = bb;
    }
    if (best >= 1 && s.inv_w[col] > 0.f) {
      // edge = thr0 + best * w; new emission threshold = edge - 2 eps.  hist_bin rounds (key - thr0) * inv_w, so
      // a key a few ulps under the rounded edge can still fall in bin `best`: any key it counts there is at
      // least thr0 + g (1 - 2u) with g = best / inv_w, u = 2^-24, and the rounded edge exceeds thr0 + g by at most
      // u (g + |edge|).  Lowering the edge by 8u (g + |edge|) covers both and this subtraction's own rounding.
      const float g = (float)best / s.inv_w[col];
      const float e0 = s.thr0[col] + g;
      const float edge = e0 - (g + fabsf(e0)) * 0x1p-21f;
      const float nt = edge - 2.f * a.eps[col];
      if (nt > s.thr[col]) s.thr[col] = nt;
    }
  }
}

template <int METRIC, bool EF16, int NQ>
__device__ __forceinline__ void consumer(const SmemLayout& s, const TcArgs& t, const ScanArgs& a, const CtaTiles& tiles,
                                         int nq) {
  if constexpr (NQ == 256) setmaxnreg_inc<kConsumerRegs>();
  bool flushed_once = false;
  int stage = 0;
  uint32_t phase = 0;
  float acc[NQ / 2];
  const bool cos_noscale = cos_noscale_of<METRIC, EF16>(t.row_stats);
  for (int64_t tile = 0; tile < tiles.count; ++tile) {
    mma_tile<NQ>(s, t, acc, stage, phase);
    epilogue<METRIC, NQ>(s, a, tiles, tile, acc, nq, cos_noscale);
    if (a.dump_mode) continue;
    // Staged hits are flushed when enough have accumulated (or after the last tile).  The two barriers bracket the
    // read of the counter so that all consumer threads decide alike.
    named_bar_sync(1, kNumConsumers);
    const int n_all = s.list_n[0];
    named_bar_sync(1, kNumConsumers);
    const bool last = tile + 1 == tiles.count;
    const bool do_flush = n_all >= (flushed_once ? kFlushAt : kFlushFirst) || (last && n_all > 0);
    if (do_flush) {
      flushed_once = true;
      flush_staged<NQ>(s, a, min(n_all, kListCap));
    }
    const bool periodic = (tile % kRefreshEvery) == kRefreshEvery - 1;
    if ((do_flush || periodic) && !last) refresh_thresholds(s, a);
    if (do_flush || periodic) named_bar_sync(1, kNumConsumers);
  }
}

// EF16: the corpus is stored as fp16 (lossless for RAGLite data, whose embeddings are fp16-rounded,
// reference _embed.py:140): the tensor map brings the rows into the swizzled tile without conversion, half the HBM bytes.
template <int METRIC, bool EF16, int NQ>
__global__ void __launch_bounds__(kThreads, 1) scan_wgmma_kernel(const __grid_constant__ CUtensorMap tmE, const TcArgs t) {
  extern __shared__ unsigned char smem_dyn[];
  // Group-parallel mode (B > NQ): the CTAs of a "lane" -- par_groups consecutive CTAs -- walk the SAME corpus tiles
  // at the same time, one NQ-query group each.  The first of them pulls a tile in from HBM (and, NQ = 128, prefetches
  // it into L2), the others find it in L2 microseconds later, so HBM sees the corpus once.
  const int P = t.par_groups > 1 ? t.par_groups : 1;
  const int pg = P > 1 ? (int)(blockIdx.x % (unsigned)P) : 0;
  ScanArgs a = t.a;
  const float* q_scale_g = t.q_scale;
  const __half* qimg_g = t.qimg;
  if (P > 1) {
    const int q0p = pg * NQ;
    a.B = min(NQ, t.a.B - q0p);
    slice_queries(a, q0p);
    q_scale_g += q0p;
    qimg_g += (size_t)pg * t.n_ks * NQ * kSliceK;
  }
  const unsigned char* qsrc = reinterpret_cast<const unsigned char*>(qimg_g);
  const int nq = (pg == P - 1) ? t.nq_last : t.nq;   // padded width of the group this CTA serves
  const uint32_t qbytes = (uint32_t)nq * 128u;       // one K slice of the group's queries
  // The tail (barriers, per-query arrays, staged list) comes first, at fixed offsets: its addresses are constants,
  // not registers the roles have to carry.  The stages follow, 1024-byte aligned for the 128B-swizzled tiles.
  SmemLayout s;
  s.full = reinterpret_cast<uint64_t*>(smem_dyn);
  s.empty = s.full + kMaxStages;
  s.thr = reinterpret_cast<float*>(s.empty + kMaxStages);
  s.cs = s.thr + NQ;
  s.thr0 = s.cs + NQ;
  s.inv_w = s.thr0 + NQ;
  s.hist = reinterpret_cast<uint32_t*>(s.inv_w + NQ);
  s.cnt = reinterpret_cast<int*>(s.hist + NQ * kHistBins / 2);
  s.basev = s.cnt + NQ;
  s.list_n = s.basev + NQ;
  s.list = reinterpret_cast<uint32_t*>(s.list_n + 4);
  unsigned char* tail_end = smem_dyn + tail_bytes<NQ>();
  s.stage_base = tail_end + ((1024u - (smem_u32(tail_end) & 1023u)) & 1023u);

  const CtaTiles tiles((uint32_t)a.n_mode_blocks, (uint32_t)P);

  if (threadIdx.x == 0) {
    for (int i = 0; i < t.stages; ++i) {
      // loader warps (none when the tensor map brings the rows: fp16 storage) + the query copy (expect_tx)
      mbar_init(&s.full[i], (EF16 ? 0 : kNumLoaderWarps) + 1);
      mbar_init(&s.empty[i], kNumConsumerWarps);
    }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < NQ; i += blockDim.x) {
    s.thr[i] = (i < a.B && !a.dump_mode) ? a.thr[i] : __int_as_float(0x7f800000);  // +inf: never emit
    s.cs[i] = (i < a.B) ? q_scale_g[i] : 0.f;
    s.cnt[i] = 0;
    s.thr0[i] = s.thr[i];
    s.inv_w[i] = (i < a.B && !a.dump_mode) ? a.hist_inv_w[i] : 0.f;
  }
  for (int i = threadIdx.x; i < NQ * kHistBins / 2; i += blockDim.x) s.hist[i] = 0u;
  if (threadIdx.x == 0) { s.list_n[0] = 0; s.list_n[1] = 0; }
  __syncthreads();

  // NQ = 256: each role sets its register budget first thing (whole warpgroups: warps 0..7 consume, warps 8..15
  // load), so that the compiler allocates the role's code within that budget.
  if (threadIdx.x >= kFirstLoaderWarp * 32) {
    if constexpr (EF16) {
      tma_producer<NQ>(s, t, a, tiles, tmE, qsrc, qbytes, pg == 0);
    } else {
      // fp32 loader fast path (uniform): whole K slices in pairs, no per-row scale in the loader
      const bool fast_f32 = a.d % kSliceK == 0 && (t.n_ks & 1) == 0 && a.ld * 64 < (int64_t(1) << 32) &&
                            (METRIC != RL_METRIC_COSINE || cos_noscale_of<METRIC, false>(t.row_stats));
      if (fast_f32) fp32_fast_producer<METRIC, NQ>(s, t, a, tiles, qsrc, qbytes, pg == 0);
      else fp32_generic_producer<METRIC, NQ>(s, t, a, tiles, qsrc, qbytes, pg == 0);
    }
  } else {
    consumer<METRIC, EF16, NQ>(s, t, a, tiles, nq);
  }
}

// Query image: fp16, scaled, laid out exactly as the swizzled smem stage rows.
__global__ void __launch_bounds__(128) query_image_kernel(const float* __restrict__ Q, int B, int d, int metric,
                                                          const float* __restrict__ q_inv_norm,
                                                          const float* __restrict__ row_stats, float* __restrict__ q_scale,
                                                          __half* __restrict__ qimg, int n_ks, int rows_scaled, int gw) {
  __shared__ float red[4];
  const int b = blockIdx.x;
  const int group = b / gw, n = b % gw;   // gw: query-group width (the scan's NQ)
  const int nq = min(gw, (B - group * gw + 15) / 16 * 16);
  const float* q = Q + (size_t)b * d;
  float scale;
  if (metric == RL_METRIC_COSINE) {
    scale = q_inv_norm[b];
    if (threadIdx.x == 0) q_scale[b] = 1.f;
  } else {
    float m = 0.f;
    for (int c = threadIdx.x; c < d; c += blockDim.x) m = fmaxf(m, fabsf(q[c]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
    scale = pow2_scale(m);
    // the loaders of an fp32 corpus multiply the rows by a global power of two (dot / l2); fp16-stored rows stay as they are
    const float rs_e = rows_scaled ? pow2_scale(row_stats[1]) : 1.f;
    if (threadIdx.x == 0) q_scale[b] = (metric == RL_METRIC_L2 ? 2.f : 1.f) / (scale * rs_e);
  }
  __half* img = qimg + (size_t)group * n_ks * gw * kSliceK;  // groups are laid out with the full gw-row pitch
  for (int c = threadIdx.x; c < n_ks * kSliceK; c += blockDim.x) {
    const int ks = c / kSliceK, e = c % kSliceK;
    const float v = c < d ? q[c] * scale : 0.f;
    const int chunk = e >> 3, within = e & 7;
    const size_t off = ((size_t)ks * nq + n) * kSliceK + (size_t)(((chunk ^ (n & 7)) << 3) + within);
    img[off] = __float2half_rn(v);
  }
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda link dependency).
typedef CUresult (*ScanEncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
ScanEncodeTiledFn scan_encode_tiled_fn() {
  static ScanEncodeTiledFn fn = []() -> ScanEncodeTiledFn {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<ScanEncodeTiledFn>(p);
  }();
  return fn;
}
// Tensor map over the fp16-stored corpus E[n_rows, ld] (d valid columns): box = 64 halves (one 128-byte swizzle row)
// x 128 rows = exactly one A stage; rows past n_rows and columns past d read as zero.
bool make_corpus_tensor_map(CUtensorMap* tm, const void* E, int64_t n_rows, int64_t ld, int d) {
  ScanEncodeTiledFn enc = scan_encode_tiled_fn();
  if (enc == nullptr || (reinterpret_cast<uintptr_t>(E) & 15) != 0 || (ld * 2) % 16 != 0 || n_rows >= (int64_t(1) << 31)) return false;
  const cuuint64_t gdim[2] = {(cuuint64_t)d, (cuuint64_t)n_rows};
  const cuuint64_t gstr[1] = {(cuuint64_t)ld * sizeof(__half)};
  const cuuint32_t box[2] = {(cuuint32_t)kSliceK, (cuuint32_t)kTileM};
  const cuuint32_t estr[2] = {1, 1};
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(E), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace

bool wgmma_scan_supported(const rl_scan_params* p) {
  if (p == nullptr || p->n_rows <= 0 || p->B <= 0) return false;
  if (p->e_dtype == 1 && (p->d % 8 != 0 || p->ld % 8 != 0)) return false;
  if (p->d % 4 != 0 || p->ld % 4 != 0) return false;
  if ((reinterpret_cast<uintptr_t>(p->E) & 15) != 0) return false;
  if ((p->d + kSliceK - 1) / kSliceK > 1024) return false;
  return true;
}

size_t wgmma_qimg_bytes(const rl_scan_params* p) {
  const int n_ks = (p->d + kSliceK - 1) / kSliceK;
  const int gw = query_group_width(p);
  const int groups = (p->B + gw - 1) / gw;
  return (size_t)groups * n_ks * gw * kSliceK * sizeof(__half);
}

int wgmma_prepare_queries(const rl_scan_params* p, const float* q_inv_norm, float* q_scale, void* qimg, cudaStream_t stream) {
  const int n_ks = (p->d + kSliceK - 1) / kSliceK;
  RL_CUDA_CHECK(cudaMemsetAsync(qimg, 0, wgmma_qimg_bytes(p), stream));
  query_image_kernel<<<p->B, 128, 0, stream>>>(p->Q, p->B, p->d, p->metric, q_inv_norm, p->row_stats, q_scale,
                                                 reinterpret_cast<__half*>(qimg), n_ks, p->e_dtype == 1 ? 0 : 1,
                                                 query_group_width(p));
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

namespace {

template <bool EF16, int NQ>
auto scan_kernel_for(int metric) {
  return metric == RL_METRIC_COSINE ? scan_wgmma_kernel<RL_METRIC_COSINE, EF16, NQ>
         : metric == RL_METRIC_DOT  ? scan_wgmma_kernel<RL_METRIC_DOT, EF16, NQ>
                                    : scan_wgmma_kernel<RL_METRIC_L2, EF16, NQ>;
}

template <int NQ>
int launch_scan_groups(const ScanArgs& a_in, const rl_scan_params* p, const float* q_scale, const void* qimg, int sm_count,
                       const CUtensorMap& tmE, cudaStream_t stream) {
  auto kernel = scan_kernel_for<false, NQ>(p->metric);
  if (p->e_dtype == 1) {
    if constexpr (NQ == 128) kernel = scan_kernel_for<true, NQ>(p->metric);   // (fp16 storage always runs groups of 128)
    else RL_REQUIRE(false, RL_EUNSUPPORTED, "tensor-core scan: fp16 storage runs query groups of 128");
  }
  const uint32_t avail = kSmemBudget - 1024 - tail_bytes<NQ>();
  int stages = (int)(avail / stage_bytes<NQ>());
  if (stages > kMaxStages) stages = kMaxStages;
  RL_REQUIRE(stages >= 2, RL_EUNSUPPORTED, "tensor-core scan: not enough shared memory for 2 stages");
  const size_t smem = (size_t)stages * stage_bytes<NQ>() + tail_bytes<NQ>() + 1024;
  RL_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int n_ks = (p->d + kSliceK - 1) / kSliceK;
  const int groups = (a_in.B + NQ - 1) / NQ;
  // Up to kMaxBatchPerLaunch / NQ groups of NQ queries share one launch, one group per CTA, so that HBM sees the
  // corpus once per launch; every group needs a CTA of its own in each lane.
  int max_groups = sm_count / 2;
  if (max_groups > kMaxBatchPerLaunch / NQ) max_groups = kMaxBatchPerLaunch / NQ;
  if (max_groups < 1) max_groups = 1;
  for (int g0 = 0; g0 < groups; g0 += max_groups) {
    TcArgs t;
    const int q0 = g0 * NQ;
    const int ng = groups - g0 < max_groups ? groups - g0 : max_groups;
    const int nb = a_in.B - q0 < ng * NQ ? a_in.B - q0 : ng * NQ;
    t.a = a_in;
    t.a.B = nb;
    slice_queries(t.a, q0);
    t.qimg = reinterpret_cast<const __half*>(qimg) + (size_t)g0 * n_ks * NQ * kSliceK;
    t.q_scale = q_scale + q0;
    t.row_stats = p->row_stats;
    t.par_groups = ng;
    const int last_b = nb - (ng - 1) * NQ;                 // queries of the last group
    t.nq_last = (last_b + 15) / 16 * 16;
    t.nq = ng > 1 ? NQ : t.nq_last;                        // a full group (the only group when ng == 1)
    t.n_ks = n_ks;
    t.stages = stages;
    const int lanes = sm_count / ng;
    const unsigned grid = (unsigned)((a_in.n_mode_blocks < lanes ? a_in.n_mode_blocks : lanes) * ng);
    kernel<<<grid, kThreads, smem, stream>>>(tmE, t);
    RL_CUDA_CHECK(cudaGetLastError());
  }
  return RL_OK;
}

}  // namespace

int launch_scan_wgmma(const ScanArgs& a_in, const rl_scan_params* p, const float* q_scale, const void* qimg, int sm_count,
                      cudaStream_t stream) {
  if (a_in.n_mode_blocks == 0 || a_in.B == 0) return RL_OK;
  RL_REQUIRE(p->row_stats != nullptr, RL_EINVAL, "tensor-core scan needs row_stats");
  // fp16 storage: the corpus tiles go HBM -> shared memory through a tensor map (TMA writes the swizzled tile,
  // no loader warps, no registers in between).  wgmma_scan_supported() and make_layout() already guarantee the
  // alignment, pitch and row count the tensor map needs.
  CUtensorMap tmE;
  memset(&tmE, 0, sizeof(tmE));
  RL_REQUIRE(p->e_dtype != 1 || make_corpus_tensor_map(&tmE, p->E, p->n_rows, p->ld, p->d), RL_EUNSUPPORTED,
             "fp16 storage: no TMA tensor map for the corpus (cuTensorMapEncodeTiled unavailable or failed)");
  // the group width must match the query image wgmma_prepare_queries() built
  if (query_group_width(p) == 256) return launch_scan_groups<256>(a_in, p, q_scale, qimg, sm_count, tmE, stream);
  return launch_scan_groups<128>(a_in, p, q_scale, qimg, sm_count, tmE, stream);
}

}  // namespace rl
