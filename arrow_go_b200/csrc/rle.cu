// rle.cu — Parquet page decode on the device: the RLE/bit-packed hybrid stream (definition / repetition levels and
// dictionary indices) and the two value decoders a flat fixed-width column chunk needs.
//   RleDecoder.Next / GetBatch            parquet/internal/utils/rle.go:123-169,203-239
//   LevelDecoder.SetData/SetDataV2/Decode  parquet/internal/encoding/levels.go:188-297
//   dictDecoder.SetData/decode/decodeSpaced parquet/internal/encoding/decoder.go:125-160 over
//                                          TypedRleDecoder.GetBatchWithDict[Spaced] (utils/typed_rle_dict.go:143-236)
//   PlainDecoder.DecodeSpaced              parquet/internal/encoding/plain_encoding_types.go:98 -> spacedExpand (decoder.go:209)
//
// A call decodes a batch of pages (ag_pq_page descriptors, one device buffer of page payloads) in three launches:
//   1. pq_tile_count_kernel (spaced only): valid bits per 1024-slot tile of every page.
//   2. pq_runs_kernel, one block per page: scans the page's tile counts into dense-rank bases, then streams the page
//      bytes through shared memory in 16 KB windows while thread 0 walks the run headers (the chain is sequential; the
//      parallelism comes from the pages).  Each run becomes an 8-byte descriptor {first dense value | literal flag,
//      repeated value or payload byte offset}; the page records its run count, decoded count and an error code.
//      Windows start at the next header, so the bytes of long literal runs between two windows are never loaded.
//   3. pq_expand_kernel, one block per 1024-slot tile of output: finds its page and run by binary search, broadcasts
//      repeated values, unpacks literal values with aligned 32-bit loads + funnel shift, gathers dictionary values
//      (the dictionary stays in L2) with the bounds check fused, and maps slots to dense ranks with a ballot scan of
//      the validity bits (null slots get 0, like FillZero).
// Roofline.  Single pass: encoded bytes read once + values written once (+ 1 bit of validity per slot).  This design
// reads the encoded bytes up to twice (pass 2 only touches the headers' windows and the payload it expands) and
// writes 8 B per run descriptor, so its own bound is (2 x encoded + written) bytes of HBM traffic; the dictionary
// gather is served from L2.
//
// DELTA_BINARY_PACKED INT32 / INT64 (deltaBitPackDecoder, parquet/internal/encoding/delta_bit_packing.go:72-316) reuses
// the tile counts, the window and the tile layout: delta_walk_kernel (one block per page) parses the header and walks
// the block chain into one 16-byte descriptor per miniblock the page needs; delta_values_kernel sums each tile's
// deltas, delta_scan_kernel scans the sums per page, and delta_values_kernel unpacks again, block-scans and writes.
// Every value is the first value plus a prefix sum of the deltas, modulo the physical width.
#include <string.h>

#include <vector>

#include "host_stage.cuh"

namespace ag {

namespace {

constexpr int kRleThreads = 256;
constexpr int kTile = 1024;                 // output slots per expansion block (4 per thread)
constexpr int kWinVec = 1024;               // 16-byte vectors per shared-memory window (16 KB)
constexpr int kWinBytes = kWinVec * 16;
constexpr uint32_t kLiteralFlag = 0x80000000u;

enum PqKind { kLevels = 0, kDict = 1, kPlain = 2, kDelta = 3 };

// per-page error codes (reported through the status and message of the call)
enum PqErr : int {
  kErrNone = 0,
  kErrTruncLiteral = 1,    // literal run payload ends before the values the page asks for
  kErrZeroRun = 2,         // run header with a count of 0
  kErrVarint = 3,          // run header varint runs past the stream, past 5 bytes, or over int32 counts
  kErrTruncRepeated = 4,   // repeated run value cut off by the end of the stream
  kErrBitWidth = 5,        // dictionary page bit width > 32
  kErrLevelsShort = 6,     // v1 level page shorter than its 4-byte length
  kErrLevelsLength = 7,    // v1 level length negative or past the page
  kErrPlainShort = 8,      // PLAIN page holds fewer values than its valid slots
};

struct PageState {          // written by pq_runs_kernel, read by pq_expand_kernel and the host
  int64_t stream;           // absolute byte offset of the hybrid stream / PLAIN values in d_data
  int64_t stream_len;
  int64_t need;             // dense values the page's slots ask for
  int64_t produced;         // dense values decoded
  int64_t slots;            // output slots written (dense: == produced)
  int32_t nruns;
  int32_t bw;
  int32_t err;
  int32_t pad;
};

struct PqPlan {             // device views of the per-call plan (uploaded in one copy)
  const ag_pq_page* pages;
  const int64_t* run_base;  // [n_pages + 1]: first descriptor slot of every page
  const int64_t* tile_base; // [n_pages + 1]: first output tile of every page
  int64_t n_pages;
  int64_t n_tiles;
};

struct PqArgs {
  PqPlan plan;
  const uint8_t* data;
  const uint8_t* valid;     // NULL = every slot valid
  PageState* st;
  uint2* runs;
  int64_t* tile_cnt;        // spaced only: valid bits per tile, then (after pass 2) the tile's first dense rank
  int2* tile_info;          // per tile: {page, run holding the tile's first dense rank}, written by pass 2
  int64_t* d_decoded;       // may be NULL
  unsigned long long* bad;  // dictionary: lowest output slot holding an out-of-range index
  int kind;
  int fixed_bw;             // levels: bits.Len(max_level)
  int v1;                   // levels: 4-byte length prefix
  int width;                // dictionary / PLAIN value width in bytes
  int64_t dict_len;
  const void* dict;
  void* out;
};

__device__ __forceinline__ int64_t find_page(const int64_t* base, int64_t n_pages, int64_t tile) {
  // last page p with base[p] <= tile (pages with no tiles share their base with the next page)
  int64_t lo = 0, hi = n_pages - 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (base[mid] <= tile) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// valid bits per tile of every page: one warp per tile, 32 windows of 32 bits
__global__ void __launch_bounds__(kRleThreads)
pq_tile_count_kernel(PqArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (kRleThreads / 32);
  for (int64_t t = ((int64_t)blockIdx.x * kRleThreads + threadIdx.x) >> 5; t < a.plan.n_tiles; t += warps) {
    const int64_t p = find_page(a.plan.tile_base, a.plan.n_pages, t);
    const ag_pq_page pg = a.plan.pages[p];
    const int64_t s0 = (t - a.plan.tile_base[p]) * kTile + lane * 32;
    const int64_t nb = pg.num_values - s0;
    int c = 0;
    if (nb > 0) {
      const int64_t bit = pg.out + s0;
      uint32_t w = bitmap_load32(a.valid, bit, bit >> 3, (bit + (nb < 32 ? nb : 32) + 7) >> 3);
      if (nb < 32) w &= (1u << nb) - 1u;
      c = __popc(w);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) a.tile_cnt[t] = c;
  }
}

// inclusive block scan of one value per thread (int ranks, or unsigned sums that wrap at their width)
template <typename V>
__device__ __forceinline__ V block_incl_scan(V v, V* warp_tot, V* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  V x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const V y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_tot[wid] = x;
  __syncthreads();
  V off = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kRleThreads / 32; ++w) {
    const V t = warp_tot[w];
    off += (w < wid) ? t : (V)0;
    tot += t;
  }
  __syncthreads();
  *total = tot;
  return off + x;
}

__device__ __forceinline__ int block_excl_scan(int v, int* warp_tot, int* total) {
  return block_incl_scan(v, warp_tot, total) - v;
}

// spaced: turns the valid counts of a page's tiles [t0, t1) into each tile's first dense rank (one block per page);
// returns the page's valid count
__device__ __forceinline__ int64_t scan_tile_ranks(int64_t* tile_cnt, int64_t t0, int64_t t1, int* warp_tot) {
  const int tid = threadIdx.x;
  int64_t run = 0;
  for (int64_t t = t0; t < t1; t += kRleThreads) {
    const int c = (t + tid < t1) ? (int)tile_cnt[t + tid] : 0;
    int tot;
    const int ex = block_excl_scan(c, warp_tot, &tot);
    if (t + tid < t1) tile_cnt[t + tid] = run + ex;   // now the tile's first dense rank
    run += tot;
  }
  return run;
}

// spaced: the page slot of the page's `rank`-th valid value (rank < the page's valid count); tile_cnt holds first ranks
__device__ int64_t slot_of_rank(const uint8_t* valid, int64_t bit0, const int64_t* tile_cnt, int64_t t0, int64_t t1, int64_t rank) {
  int64_t t = t0;
  while (t + 1 < t1 && tile_cnt[t + 1] <= rank) ++t;
  int64_t r = tile_cnt[t];
  int64_t s = (t - t0) * kTile;
  for (;; ++s) {                                                 // the rank-th valid slot lies in tile t
    if (bit_is_set(valid, bit0 + s)) { if (r == rank) break; ++r; }
  }
  return s;
}

// one block per page: stream geometry, spaced rank bases, run table
__global__ void __launch_bounds__(kRleThreads)
pq_runs_kernel(PqArgs a) {
  __shared__ uint4 win[kWinVec];
  __shared__ int warp_tot[kRleThreads / 32];
  __shared__ int64_t s_pos, s_produced;
  __shared__ int s_done, s_nruns, s_err, s_bw;
  __shared__ int64_t s_stream, s_len;
  const int64_t p = blockIdx.x;
  const ag_pq_page pg = a.plan.pages[p];
  const int tid = threadIdx.x;
  if (p == 0 && tid == 0 && a.bad) *a.bad = (unsigned long long)AG_NO_ERROR_POS;

  // ---- need: dense values of the page (spaced: its valid bits, and every tile's first dense rank) ----
  const int64_t need = a.valid ? scan_tile_ranks(a.tile_cnt, a.plan.tile_base[p], a.plan.tile_base[p + 1], warp_tot) : pg.num_values;

  {
    const int64_t t0 = a.plan.tile_base[p], t1 = a.plan.tile_base[p + 1];
    for (int64_t t = t0 + tid; t < t1; t += kRleThreads) a.tile_info[t] = make_int2((int)p, 0);
  }

  // ---- stream geometry ----
  if (tid == 0) {
    int err = kErrNone, bw = a.fixed_bw;
    int64_t stream = pg.data, len = pg.len;
    if (a.kind == kLevels && a.v1) {
      if (len < 4) {
        err = kErrLevelsShort; len = 0;
      } else {
        const uint8_t* b = a.data + pg.data;
        const int32_t nb = (int32_t)((uint32_t)b[0] | ((uint32_t)b[1] << 8) | ((uint32_t)b[2] << 16) | ((uint32_t)b[3] << 24));
        if (nb < 0 || (int64_t)nb > len - 4) { err = kErrLevelsLength; len = 0; }
        else { stream += 4; len = nb; }
      }
    } else if (a.kind == kDict) {
      if (len == 0) {
        bw = 0;                                          // no data: bit width 0 (decoder.go:127-131)
      } else {
        bw = a.data[pg.data];
        stream += 1; len -= 1;
        if (bw > 32) { err = kErrBitWidth; len = 0; }
      }
    }
    s_stream = stream; s_len = len; s_bw = bw; s_err = err;
    s_pos = 0; s_produced = 0; s_nruns = 0;
    s_done = (err != kErrNone || a.kind == kPlain) ? 1 : 0;
    if (a.kind == kPlain) {
      const int64_t have = len / a.width;
      if (need > have) { s_err = kErrPlainShort; s_produced = 0; }
      else s_produced = need;
    }
  }
  __syncthreads();

  // ---- run headers, window by window ----
  const int64_t stream = s_stream, len = s_len;
  const int bw = s_bw;
  const int nbytes_rep = (bw + 7) >> 3;
  uint2* runs = a.runs + (a.runs ? a.plan.run_base[p] : 0);
  const int64_t cap = a.runs ? a.plan.run_base[p + 1] - a.plan.run_base[p] : 0;
  const uint8_t* sb = reinterpret_cast<const uint8_t*>(win);
  const int64_t tile0 = a.plan.tile_base[p], ntiles = a.plan.tile_base[p + 1] - tile0;
  auto tile_rank = [&](int64_t j) -> int64_t { return j >= ntiles ? INT64_MAX : a.valid ? a.tile_cnt[tile0 + j] : j * kTile; };
  int64_t next_tile = 0, next_rank = tile_rank(0);   // thread 0: first tile whose first dense rank no run covered yet
  // thread 0, after emitting run `r` that covers dense values [.., end): it holds the first rank of these tiles
  auto cover = [&](int r, int64_t end) {
    while (next_rank < end) { a.tile_info[tile0 + next_tile].y = r; next_rank = tile_rank(++next_tile); }
  };
  while (true) {
    __syncthreads();
    if (s_done) break;
    // window [a0, a0 + 16 KB) over absolute addresses, a0 = 16-byte aligned start of the next header; only vectors
    // that hold at least one byte of the stream are loaded (an aligned vector never straddles a mapping boundary)
    const uintptr_t sbeg = reinterpret_cast<uintptr_t>(a.data) + stream;
    const uintptr_t send = sbeg + len;
    const uintptr_t a0 = (sbeg + s_pos) & ~(uintptr_t)15;
#pragma unroll 4
    for (int v = tid; v < kWinVec; v += kRleThreads) {
      const uintptr_t ad = a0 + (uintptr_t)v * 16;
      if (ad < send && ad + 16 > sbeg) win[v] = __ldcs(reinterpret_cast<const uint4*>(ad));
    }
    __syncthreads();
    if (tid == 0) {
      int64_t pos = s_pos, produced = s_produced;
      int nruns = s_nruns, err = kErrNone, done = 0;
      const int64_t wend = (int64_t)(a0 + kWinBytes - sbeg);   // stream offset where the window ends
      while (true) {
        if (produced >= need || pos >= len) { done = 1; break; }
        if (pos + 16 > wend && wend < len) break;               // header may straddle the window: reload at pos
        // varint indicator (binary.ReadUvarint), at most 5 bytes for 32-bit counts
        uint64_t ind = 0;
        int k = 0;
        bool more = true;
        while (more) {
          if (pos + k >= len || k == 5) { err = kErrVarint; break; }
          const unsigned c = sb[(sbeg + pos + k) - a0];
          ind |= (uint64_t)(c & 0x7f) << (7 * k);
          more = (c & 0x80) != 0;
          ++k;
        }
        if (err) break;
        const int64_t body = pos + k;
        const uint64_t count = ind >> 1;
        if (count == 0) { err = kErrZeroRun; break; }
        if (nruns >= cap) { err = kErrVarint; break; }          // unreachable: every run takes >= 1 byte and 1 value
        if (ind & 1) {
          if (count > 0x7fffffffull / 8) { err = kErrVarint; break; }
          const int64_t cnt = (int64_t)count * 8;
          const int64_t take = cnt < need - produced ? cnt : need - produced;
          const int64_t avail = (len - body) * 8;
          if (take * bw > avail) {
            // truncated payload: whole 32-value groups that are present (bit_reader_test.go:513-566)
            int64_t got = bw ? avail / (32 * (int64_t)bw) * 32 : take;
            if (got > take) got = take;
            if (got > 0) { runs[nruns++] = make_uint2((uint32_t)produced | kLiteralFlag, (uint32_t)(body)); produced += got; cover(nruns - 1, produced); }
            err = kErrTruncLiteral;
            break;
          }
          runs[nruns++] = make_uint2((uint32_t)produced | kLiteralFlag, (uint32_t)body);
          produced += take;
          cover(nruns - 1, produced);
          pos = body + (int64_t)count * bw;                     // 8 values x bw bits = bw bytes per group
        } else {
          if (count > 0x7fffffffull) { err = kErrVarint; break; }
          if (body + nbytes_rep > len) { err = kErrTruncRepeated; break; }
          uint32_t v = 0;
          for (int j = 0; j < nbytes_rep; ++j) v |= (uint32_t)sb[(sbeg + body + j) - a0] << (8 * j);
          runs[nruns++] = make_uint2((uint32_t)produced, v);
          const int64_t take = (int64_t)count < need - produced ? (int64_t)count : need - produced;
          produced += take;
          cover(nruns - 1, produced);
          pos = body + nbytes_rep;
        }
      }
      s_pos = pos; s_produced = produced; s_nruns = nruns;
      if (err) { s_err = err; done = 1; }
      s_done = done;
    }
  }

  // ---- slots decoded: every slot up to the first valid slot whose value the stream did not deliver ----
  if (tid == 0) {
    cover(s_nruns > 0 ? s_nruns - 1 : 0, INT64_MAX);         // tiles past the last decoded value
    const int64_t produced = s_produced;
    int64_t slots = produced;
    if (s_err == kErrPlainShort) {
      slots = 0;                                               // DecodeSpaced delivers nothing then
    } else if (a.valid) {
      slots = produced < need ? slot_of_rank(a.valid, pg.out, a.tile_cnt, a.plan.tile_base[p], a.plan.tile_base[p + 1], produced)
                              : pg.num_values;
    }
    PageState ps;
    ps.stream = stream; ps.stream_len = len; ps.need = need; ps.produced = produced; ps.slots = slots;
    ps.nruns = s_nruns; ps.bw = bw; ps.err = s_err; ps.pad = 0;
    a.st[p] = ps;
    if (a.d_decoded) a.d_decoded[p] = slots;
  }
}

__device__ __forceinline__ uint32_t unpack_at(const uint8_t* payload, int64_t k, int bw) {
  if (bw == 0) return 0u;                                        // no payload bytes to touch
  const uintptr_t ad = reinterpret_cast<uintptr_t>(payload);
  const uint32_t* base = reinterpret_cast<const uint32_t*>(ad & ~(uintptr_t)3);
  const uint64_t bit = (uint64_t)(ad & 3) * 8 + (uint64_t)k * (unsigned)bw;
  const int64_t w = (int64_t)(bit >> 5);
  const int sh = (int)(bit & 31);
  const uint32_t lo = __ldg(base + w);
  const uint32_t hi = (sh + bw > 32) ? __ldg(base + w + 1) : 0u;   // only when the value reaches into that word
  const uint32_t mask = bw >= 32 ? 0xffffffffu : ((1u << bw) - 1u);
  return __funnelshift_r(lo, hi, sh) & mask;
}

template <typename T>
__device__ __forceinline__ T load_unaligned(const uint8_t* p) {
  if ((reinterpret_cast<uintptr_t>(p) & (sizeof(T) - 1)) == 0) return __ldg(reinterpret_cast<const T*>(p));
  T v = 0;
#pragma unroll
  for (int j = 0; j < (int)sizeof(T); ++j) v |= (T)__ldg(p + j) << (8 * j);
  return v;
}

// one block per tile of 1024 output slots of one page
template <int KIND, typename T, bool SPACED>
__global__ void __launch_bounds__(kRleThreads)
pq_expand_kernel(PqArgs a) {
  __shared__ int warp_tot[kRleThreads / 32];
  const int64_t tile = blockIdx.x;
  const int2 ti = a.tile_info[tile];
  const int64_t p = ti.x;
  const ag_pq_page pg = a.plan.pages[p];
  const PageState ps = a.st[p];
  const int64_t s0 = (tile - a.plan.tile_base[p]) * kTile;
  const int64_t limit = ps.slots;
  if (s0 >= limit) return;                                      // block-uniform
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const uint2* runs = a.runs + (KIND == kPlain ? 0 : a.plan.run_base[p]);
  const uint8_t* stream = a.data + ps.stream;
  T* out = reinterpret_cast<T*>(a.out) + pg.out;

  const int64_t r0 = SPACED ? a.tile_cnt[tile] : s0;   // the tile's first dense rank
  // runs holding this tile's first rank and the next tile's first rank bracket every rank the tile needs
  const int64_t rlo = ti.y;
  int64_t rhi = tile + 1 < a.plan.tile_base[p + 1] ? a.tile_info[tile + 1].y : ps.nruns - 1;
  if (rhi < rlo) rhi = rlo;

  int64_t rank_base = r0;
#pragma unroll
  for (int q = 0; q < kTile / kRleThreads; ++q) {
    const int64_t s = s0 + q * kRleThreads + tid;
    const bool in = s < limit;
    bool v = in;
    int64_t rank = s;
    if (SPACED) {
      v = in && bit_is_set(a.valid, pg.out + s);
      const unsigned m = __ballot_sync(0xffffffffu, v);
      if (lane == 0) warp_tot[wid] = __popc(m);
      __syncthreads();
      int off = 0, tot = 0;
#pragma unroll
      for (int w = 0; w < kRleThreads / 32; ++w) { const int t = warp_tot[w]; off += (w < wid) ? t : 0; tot += t; }
      __syncthreads();
      rank = rank_base + off + __popc(m & ((1u << lane) - 1u));
      rank_base += tot;
    }
    if (!in) continue;
    if (!v) { out[s] = (T)0; continue; }
    uint32_t idx;
    if (KIND == kPlain) {
      out[s] = load_unaligned<T>(stream + rank * (int64_t)sizeof(T));
      continue;
    } else {
      int64_t lo = rlo, hi = rhi;
      while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if ((int64_t)(runs[mid].x & ~kLiteralFlag) <= rank) lo = mid; else hi = mid - 1;
      }
      const uint2 r = runs[lo];
      idx = (r.x & kLiteralFlag) ? unpack_at(stream + r.y, rank - (int64_t)(r.x & ~kLiteralFlag), ps.bw) : r.y;
    }
    if (KIND == kLevels) {
      out[s] = (T)idx;
    } else {
      if ((int64_t)idx < a.dict_len) {
        out[s] = __ldg(reinterpret_cast<const T*>(a.dict) + idx);
      } else {
        out[s] = (T)0;
        atomicMin(a.bad, (unsigned long long)(pg.out + s));
      }
    }
  }
}

// ---------------------------------------------------------------- DELTA_BINARY_PACKED ----
// per-page error codes of the delta decoder; delta_err_text gives the reference's message for each
enum DeltaErr : int {
  kDErrNone = 0,
  kDErrEof = 1,            // header or min-delta varint missing, truncated or over 64 bits
  kDErrZeroBlock = 2,
  kDErrBlockSize = 3,      // arg0 = block size
  kDErrZeroMini = 4,
  kDErrTooManyMini = 5,    // arg0 = miniblocks per block
  kDErrMiniDivide = 6,     // arg0 = miniblocks per block, arg1 = block size
  kDErrVpm = 7,            // arg0 = values per miniblock
  kDErrCount = 8,          // arg0 = total values, arg1 = num_values
  kDErrFirst32 = 9,        // arg0 = first value
  kDErrMinDelta32 = 10,    // arg0 = min delta
  kDErrWidthBytes = 11,    // a touched block's miniblock widths cut off
  kDErrWidth = 12,         // arg0 = miniblock width, arg1 = decoder width
  kDErrPayload = 13,       // a touched miniblock's payload cut off
  kDErrShort = 14,         // spaced: fewer values than valid slots
};

struct __align__(16) DeltaMini {   // one touched miniblock
  uint32_t off;                    // payload byte offset within the page
  uint32_t bw;
  unsigned long long min_delta;
};

struct DeltaPage {          // written by delta_walk_kernel, read by the value passes and the host
  unsigned long long first;
  int64_t produced;         // dense values delivered, the first value included
  int64_t slots;            // output slots written
  unsigned long long arg0, arg1;   // what the error message names
  uint32_t vpm;
  int32_t err;
};

struct DeltaArgs {
  const ag_pq_page* pages;
  const int64_t* mb_base;   // [n_pages + 1]: first miniblock descriptor of every page
  const int64_t* tile_base; // [n_pages + 1]: first output tile of every page
  int64_t n_pages;
  const uint8_t* data;
  const uint8_t* valid;     // NULL = every slot valid
  DeltaPage* st;
  DeltaMini* mb;
  int64_t* tile_cnt;        // spaced only: valid bits per tile, then the tile's first dense rank
  unsigned long long* tile_sum;   // per tile: sum of its deltas, then (after delta_scan_kernel) of the page's deltas before it
  int64_t* d_decoded;       // may be NULL
  int width;                // 4 (INT32) or 8 (INT64)
  void* out;
};

// binary.ReadUvarint: at most 10 bytes, the 10th at most 1
template <typename B>
__device__ __forceinline__ bool read_uvarint(B byte_at, int64_t& pos, int64_t len, unsigned long long* v) {
  unsigned long long x = 0;
  for (int i = 0; i < 10; ++i) {
    if (pos >= len) return false;
    const uint32_t c = byte_at(pos++);
    if (c < 0x80) {
      if (i == 9 && c > 1) return false;
      *v = x | (unsigned long long)c << (7 * i);
      return true;
    }
    x |= (unsigned long long)(c & 0x7f) << (7 * i);
  }
  return false;
}

__device__ __forceinline__ long long unzigzag(unsigned long long u) { return (long long)(u >> 1) ^ -(long long)(u & 1); }

// One block per page: parses the header (SetData) and walks the block chain (initBlock / unpackNextMini) up to the
// last miniblock holding a delta the page needs, writing one descriptor per such miniblock.  The page streams through
// shared memory as in pq_runs_kernel; a header that reaches past the window is read from global memory.  After this
// pass every descriptor's payload lies inside its page.
__global__ void __launch_bounds__(kRleThreads)
delta_walk_kernel(DeltaArgs a) {
  __shared__ uint4 win[kWinVec];
  __shared__ int warp_tot[kRleThreads / 32];
  struct Walk {
    unsigned long long vpm, nmini, arg0, arg1;
    int64_t pos, nmb, want_mb;
    int err, done;
  };
  __shared__ Walk w;                                             // thread 0's walk state between windows
  __shared__ unsigned long long s_first;
  __shared__ int64_t s_total, s_cap;
  const int64_t p = blockIdx.x;
  const ag_pq_page pg = a.pages[p];
  const int tid = threadIdx.x;
  const int64_t t0 = a.tile_base[p], t1 = a.tile_base[p + 1];
  const int64_t need = a.valid ? scan_tile_ranks(a.tile_cnt, t0, t1, warp_tot) : pg.num_values;
  const uint8_t* page = a.data + pg.data;
  const int64_t len = pg.len;

  if (tid == 0) {
    auto gbyte = [&](int64_t i) -> uint32_t { return __ldg(page + i); };
    int err = kDErrNone;
    unsigned long long arg0 = 0, arg1 = 0, first = 0, vpm = 0, nmini = 0, block = 0, tot = 0, fz = 0;
    int64_t pos = 0;
    if (!read_uvarint(gbyte, pos, len, &block)) err = kDErrEof;
    else if (block == 0) err = kDErrZeroBlock;
    else if (block > 0xffffffffull || block % 128) { err = kDErrBlockSize; arg0 = block; }
    else if (!read_uvarint(gbyte, pos, len, &nmini)) err = kDErrEof;
    else if (nmini == 0) err = kDErrZeroMini;
    else if (nmini > 0xffffffffull) { err = kDErrTooManyMini; arg0 = nmini; }
    else if (block % nmini) { err = kDErrMiniDivide; arg0 = nmini; arg1 = block; }
    else if ((vpm = block / nmini) % 32) { err = kDErrVpm; arg0 = vpm; }
    else if (!read_uvarint(gbyte, pos, len, &tot)) err = kDErrEof;
    else if (tot > 0xffffffffull || tot > (unsigned long long)pg.num_values) { err = kDErrCount; arg0 = tot; arg1 = pg.num_values; }
    else if (!read_uvarint(gbyte, pos, len, &fz)) err = kDErrEof;
    else {
      first = (unsigned long long)unzigzag(fz);
      if (a.width == 4 && (long long)first != (long long)(int32_t)first) { err = kDErrFirst32; arg0 = first; }
    }
    const int64_t total = err ? 0 : (int64_t)tot;
    const int64_t cap = need < total ? need : total;            // values delivered when the chain is sound
    w.vpm = vpm; w.nmini = nmini; w.arg0 = arg0; w.arg1 = arg1; w.pos = pos; w.nmb = 0;
    w.want_mb = cap > 1 ? (int64_t)(((unsigned long long)cap - 2) / vpm + 1) : 0;   // miniblocks holding deltas 1..cap-1
    w.err = err;
    w.done = err != kDErrNone || w.want_mb == 0;
    s_first = first; s_total = total; s_cap = cap;
  }

  const uint8_t* sb = reinterpret_cast<const uint8_t*>(win);
  while (true) {
    __syncthreads();
    if (w.done) break;
    // window [a0, a0 + 16 KB) over absolute addresses, a0 = 16-byte aligned start of the next block header
    const uintptr_t sbeg = reinterpret_cast<uintptr_t>(page);
    const uintptr_t send = sbeg + len;
    const uintptr_t a0 = (sbeg + w.pos) & ~(uintptr_t)15;
#pragma unroll 4
    for (int v = tid; v < kWinVec; v += kRleThreads) {
      const uintptr_t ad = a0 + (uintptr_t)v * 16;
      if (ad < send && ad + 16 > sbeg) win[v] = __ldcs(reinterpret_cast<const uint4*>(ad));
    }
    __syncthreads();
    if (tid == 0) {
      const int64_t wlo = (int64_t)(a0 - sbeg), wend = wlo + kWinBytes;   // page offsets the window covers
      auto byte_at = [&](int64_t i) -> uint32_t { return i < wend ? sb[i - wlo] : __ldg(page + i); };
      const uint32_t maxw = 8u * (uint32_t)a.width;
      const unsigned long long vpm = w.vpm, nmini = w.nmini;
      const int64_t want_mb = w.want_mb;
      DeltaMini* mb = a.mb + a.mb_base[p];
      int64_t pos = w.pos, nmb = w.nmb;
      int err = kDErrNone, done = 0;
      while (true) {
        if (nmb >= want_mb) { done = 1; break; }
        if (pos >= wend) break;                                  // past the window: reload at pos
        unsigned long long mz;
        if (!read_uvarint(byte_at, pos, len, &mz)) { err = kDErrEof; break; }
        const long long md = unzigzag(mz);
        if (a.width == 4 && md != (long long)(int32_t)md) { err = kDErrMinDelta32; w.arg0 = (unsigned long long)md; break; }
        if ((unsigned long long)(len - pos) < nmini) { err = kDErrWidthBytes; break; }
        const int64_t wpos = pos;
        pos += (int64_t)nmini;
        for (int64_t j = 0; nmb < want_mb; ++j) {               // nmb < want_mb implies j < nmini
          const uint32_t bw = byte_at(wpos + j);
          if (bw > maxw) { err = kDErrWidth; w.arg0 = bw; w.arg1 = maxw; break; }
          const int64_t nbytes = (int64_t)(vpm / 8 * bw);        // vpm is a multiple of 32
          if (nbytes > len - pos) { err = kDErrPayload; break; }
          mb[nmb++] = DeltaMini{(uint32_t)pos, bw, (unsigned long long)md};
          pos += nbytes;
          if (j + 1 == (int64_t)nmini) break;
        }
        if (err) break;
      }
      w.pos = pos; w.nmb = nmb; w.err = err;
      w.done = done || err != kDErrNone;
    }
  }

  if (tid == 0) {
    // a chain error delivers the first value and every miniblock before the failing one
    int err = w.err;
    const int64_t cap = s_cap;
    int64_t produced = err == kDErrNone ? cap : cap > 0 ? (int64_t)(1 + (unsigned long long)w.nmb * w.vpm) : 0;
    if (err == kDErrNone && a.valid && s_total < need) { err = kDErrShort; produced = 0; }
    int64_t slots = produced;
    if (err == kDErrShort) slots = 0;                            // DecodeSpaced delivers nothing then
    else if (a.valid) slots = produced < need ? slot_of_rank(a.valid, pg.out, a.tile_cnt, t0, t1, produced) : pg.num_values;
    DeltaPage ps;
    ps.first = s_first; ps.produced = produced; ps.slots = slots; ps.arg0 = w.arg0; ps.arg1 = w.arg1;
    ps.vpm = (uint32_t)w.vpm; ps.err = err;
    a.st[p] = ps;
    if (a.d_decoded) a.d_decoded[p] = slots;
  }
}

// the value of bit width bw (0..64) at index k of a bit-packed payload; loads only the (at most 3) aligned words that
// hold its bits
__device__ __forceinline__ unsigned long long unpack64_at(const uint8_t* payload, uint32_t k, int bw) {
  if (bw == 0) return 0ull;
  const uintptr_t ad = reinterpret_cast<uintptr_t>(payload);
  const uint32_t* base = reinterpret_cast<const uint32_t*>(ad & ~(uintptr_t)3);
  const uint64_t bit = (uint64_t)(ad & 3) * 8 + (uint64_t)k * (unsigned)bw;
  const int64_t w = (int64_t)(bit >> 5);
  const int sh = (int)(bit & 31);
  const uint32_t w0 = __ldg(base + w);
  const uint32_t w1 = (sh + bw > 32) ? __ldg(base + w + 1) : 0u;
  const uint32_t w2 = (sh + bw > 64) ? __ldg(base + w + 2) : 0u;
  const unsigned long long v = (unsigned long long)__funnelshift_r(w0, w1, sh) | ((unsigned long long)__funnelshift_r(w1, w2, sh) << 32);
  return bw >= 64 ? v : v & ((1ull << bw) - 1ull);
}

// delta number `r` (r >= 1: value[r] = value[r-1] + delta) of a page, wrapped to T
template <typename T>
__device__ __forceinline__ T delta_at(const uint8_t* page, const DeltaMini* mb, uint32_t vpm, int64_t r) {
  const uint32_t k = (uint32_t)(r - 1), m = k / vpm, i = k - m * vpm;
  const DeltaMini d = mb[m];
  if constexpr (sizeof(T) == 4) return unpack_at(page + d.off, i, (int)d.bw) + (uint32_t)d.min_delta;
  else return (T)unpack64_at(page + d.off, i, (int)d.bw) + (T)d.min_delta;
}

// One block per tile of 1024 output slots.  WRITE = false: the sum of the tile's deltas into tile_sum.  WRITE = true:
// a block scan of the deltas, plus the first value and the deltas of the page's earlier tiles; null slots get 0.
// Slots map to dense ranks as in pq_expand_kernel.  T is the physical width, so every sum wraps like the reference's
// int64 accumulate-then-truncate.
template <typename T, bool SPACED, bool WRITE>
__global__ void __launch_bounds__(kRleThreads)
delta_values_kernel(DeltaArgs a) {
  __shared__ int warp_cnt[kRleThreads / 32];
  __shared__ T warp_sum[kRleThreads / 32];
  const int64_t tile = blockIdx.x;
  const int64_t p = find_page(a.tile_base, a.n_pages, tile);
  const ag_pq_page pg = a.pages[p];
  const DeltaPage ps = a.st[p];
  const int64_t s0 = (tile - a.tile_base[p]) * kTile;
  const int tid = threadIdx.x, lane = tid & 31;
  if (s0 >= ps.slots) {                                          // block-uniform
    if (!WRITE && tid == 0) a.tile_sum[tile] = 0;
    return;
  }
  const uint8_t* page = a.data + pg.data;
  const DeltaMini* mb = a.mb + a.mb_base[p];
  T* out = reinterpret_cast<T*>(a.out) + pg.out;
  int64_t rank_base = SPACED ? a.tile_cnt[tile] : s0;
  T carry = WRITE ? (T)ps.first + (T)a.tile_sum[tile] : (T)0;   // value before the tile's first delta
  T acc = 0;
#pragma unroll
  for (int q = 0; q < kTile / kRleThreads; ++q) {
    const int64_t s = s0 + q * kRleThreads + tid;
    const bool in = s < ps.slots;
    bool v = in;
    int64_t rank = s;
    if (SPACED) {
      v = in && bit_is_set(a.valid, pg.out + s);
      const unsigned m = __ballot_sync(0xffffffffu, v);
      if (lane == 0) warp_cnt[tid >> 5] = __popc(m);
      __syncthreads();
      int off = 0, tot = 0;
#pragma unroll
      for (int w = 0; w < kRleThreads / 32; ++w) { const int t = warp_cnt[w]; off += (w < (tid >> 5)) ? t : 0; tot += t; }
      __syncthreads();
      rank = rank_base + off + __popc(m & ((1u << lane) - 1u));
      rank_base += tot;
    }
    const T d = (v && rank >= 1) ? delta_at<T>(page, mb, ps.vpm, rank) : (T)0;
    if (!WRITE) { acc += d; continue; }
    T tot;
    const T incl = block_incl_scan(d, warp_sum, &tot);
    if (in) out[s] = v ? (T)(carry + incl) : (T)0;
    carry += tot;
  }
  if (!WRITE) {
    T tot;
    block_incl_scan(acc, warp_sum, &tot);
    if (tid == 0) a.tile_sum[tile] = tot;
  }
}

// one block per page: tile sums -> the sum of the page's deltas before each tile
__global__ void __launch_bounds__(kRleThreads)
delta_scan_kernel(DeltaArgs a) {
  __shared__ unsigned long long warp_sum[kRleThreads / 32];
  const int64_t p = blockIdx.x, t0 = a.tile_base[p], t1 = a.tile_base[p + 1];
  unsigned long long run = 0;
  for (int64_t t = t0; t < t1; t += kRleThreads) {
    const int64_t i = t + threadIdx.x;
    const unsigned long long v = i < t1 ? a.tile_sum[i] : 0ull;
    unsigned long long tot;
    const unsigned long long incl = block_incl_scan(v, warp_sum, &tot);
    if (i < t1) a.tile_sum[i] = run + incl - v;
    run += tot;
  }
}

template <typename T, bool SPACED>
ag_status launch_delta_values(const DeltaArgs& a, int64_t n_tiles, cudaStream_t st) {
  delta_values_kernel<T, SPACED, false><<<(unsigned)n_tiles, kRleThreads, 0, st>>>(a);
  AG_TRY(check_launch("delta_values_kernel"));
  delta_scan_kernel<<<(unsigned)a.n_pages, kRleThreads, 0, st>>>(a);
  AG_TRY(check_launch("delta_scan_kernel"));
  delta_values_kernel<T, SPACED, true><<<(unsigned)n_tiles, kRleThreads, 0, st>>>(a);
  return check_launch("delta_values_kernel");
}

void delta_err_text(const DeltaPage& s, char* buf, size_t n) {
  const unsigned long long x = s.arg0, y = s.arg1;
  switch (s.err) {
    case kDErrEof: snprintf(buf, n, "parquet: eof exception"); break;
    case kDErrZeroBlock: snprintf(buf, n, "parquet: cannot have zero values per block"); break;
    case kDErrBlockSize: snprintf(buf, n, "parquet: values per block must be a multiple of 128, got %llu", x); break;
    case kDErrZeroMini: snprintf(buf, n, "parquet: cannot have zero miniblock per block"); break;
    case kDErrTooManyMini: snprintf(buf, n, "parquet: too many miniblocks per block: %llu", x); break;
    case kDErrMiniDivide: snprintf(buf, n, "parquet: miniblocks per block must divide the block size, got %llu miniblocks for %llu values", x, y); break;
    case kDErrVpm: snprintf(buf, n, "parquet: values per miniblock must be a nonzero multiple of 32, got %llu", x); break;
    case kDErrCount: snprintf(buf, n, "parquet: invalid delta value count %llu for %llu buffered values", x, y); break;
    case kDErrFirst32: snprintf(buf, n, "parquet: initial delta value %lld exceeds INT32 range", (long long)x); break;
    case kDErrMinDelta32: snprintf(buf, n, "parquet: minimum delta %lld exceeds INT32 range", (long long)x); break;
    case kDErrWidthBytes: snprintf(buf, n, "failed to read byte"); break;
    case kDErrWidth: snprintf(buf, n, "parquet: delta bit width %llu exceeds decoder width %llu", x, y); break;
    case kDErrPayload: snprintf(buf, n, "unexpected EOF"); break;
    case kDErrShort: snprintf(buf, n, "parquet: number of values / definition levels read did not match"); break;
    default: snprintf(buf, n, "unknown error"); break;
  }
}

const char* err_text(int e) {
  switch (e) {
    case kErrTruncLiteral: return "literal run truncated (unexpected EOF in a bit-packed run)";
    case kErrZeroRun: return "run header with a count of 0";
    case kErrVarint: return "run header varint overruns the stream or the 32-bit run count";
    case kErrTruncRepeated: return "repeated run value truncated";
    case kErrBitWidth: return "invalid or corrupted bit width (dictionary indices take 0..32 bits)";
    case kErrLevelsShort: return "parquet: received invalid levels (corrupt data page?)";
    case kErrLevelsLength: return "parquet: received invalid number of bytes (corrupt data page?)";
    case kErrPlainShort: return "parquet: eof exception decode plain (fewer values than valid slots)";
    default: return "unknown error";
  }
}

template <int KIND, typename T, bool SPACED>
ag_status launch_expand(const PqArgs& a, cudaStream_t st) {
  if (a.plan.n_tiles == 0) return AG_OK;
  pq_expand_kernel<KIND, T, SPACED><<<(unsigned)a.plan.n_tiles, kRleThreads, 0, st>>>(a);
  return check_launch("pq_expand_kernel");
}

}  // namespace

// Decodes a batch of pages.  `pages` is host memory; everything else is device memory on `st`.  Synchronises `st`
// once to read the per-page error codes back.  h_decoded (host, may be NULL) receives the per-page decoded counts.
ag_status parquet_pages_dev(int kind, int fixed_bw, int v1, int width, const void* dict, int64_t dict_len, const uint8_t* data,
                            const ag_pq_page* pages, int64_t n_pages, const uint8_t* valid, void* out, int64_t* d_decoded,
                            int64_t* h_decoded, int64_t* d_bad_pos, cudaStream_t st) {
  const char* fn = kind == kLevels ? "levels_decode" : kind == kDict ? "dict_decode" : "plain_decode_spaced";
  if (n_pages < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative page count", fn);
  if (n_pages == 0) return AG_OK;
  if (!pages) AG_FAIL(AG_ERR_INVALID, "%s: NULL page table", fn);
  // plan: pages | run_base[n+1] | tile_base[n+1]
  const size_t pb = (size_t)n_pages * sizeof(ag_pq_page);
  const size_t plan_bytes = pb + 2 * (size_t)(n_pages + 1) * 8;
  std::vector<uint8_t> h(plan_bytes);
  memcpy(h.data(), pages, pb);
  int64_t* run_base = reinterpret_cast<int64_t*>(h.data() + pb);
  int64_t* tile_base = run_base + n_pages + 1;
  run_base[0] = tile_base[0] = 0;
  bool any_data = false;
  for (int64_t i = 0; i < n_pages; ++i) {
    const ag_pq_page& g = pages[i];
    if (g.data < 0 || g.len < 0 || g.num_values < 0 || g.out < 0 || g.num_values > 0x7fffffffLL || g.len > 0xffffffffLL)
      AG_FAIL(AG_ERR_INVALID, "%s: page %lld: negative field, more than 2^31-1 values or more than 2^32-1 bytes", fn, (long long)i);
    any_data |= g.len > 0;
    const int64_t cap = kind == kPlain ? 0 : (g.num_values < g.len ? g.num_values : g.len);
    run_base[i + 1] = run_base[i] + cap;
    tile_base[i + 1] = tile_base[i] + (g.num_values + kTile - 1) / kTile;
  }
  const int64_t n_runs = run_base[n_pages], n_tiles = tile_base[n_pages];
  if (n_tiles > 0 && !out) AG_FAIL(AG_ERR_INVALID, "%s: NULL output", fn);
  if (any_data && !data) AG_FAIL(AG_ERR_INVALID, "%s: NULL page data", fn);
  if (kind == kDict && dict_len > 0 && !dict) AG_FAIL(AG_ERR_INVALID, "%s: NULL dictionary", fn);
  if (kind == kDict && dict && (reinterpret_cast<uintptr_t>(dict) & (width - 1))) AG_FAIL(AG_ERR_INVALID, "%s: dictionary not aligned to its value width", fn);
  if (out && (reinterpret_cast<uintptr_t>(out) & ((kind == kLevels ? 2 : width) - 1))) AG_FAIL(AG_ERR_INVALID, "%s: output not aligned to its element width", fn);

  const size_t st_bytes = (size_t)n_pages * sizeof(PageState);
  const size_t tc_bytes = valid ? (size_t)n_tiles * 8 : 0;
  const size_t off_st = (plan_bytes + 255) & ~(size_t)255;
  const size_t off_tc = (off_st + st_bytes + 255) & ~(size_t)255;
  const size_t off_ti = (off_tc + tc_bytes + 255) & ~(size_t)255;
  const size_t off_bad = (off_ti + (size_t)n_tiles * 8 + 255) & ~(size_t)255;
  const size_t off_runs = off_bad + 256;
  const size_t total = off_runs + (size_t)n_runs * 8;
  // this call synchronises `st` anyway, so its device scratch may live in a Temps
  Temps t(st);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, total));
  AG_TRY(h2d(d, h.data(), plan_bytes, st));
  PqArgs a;
  a.plan.pages = reinterpret_cast<const ag_pq_page*>(d);
  a.plan.run_base = reinterpret_cast<const int64_t*>(d + pb);
  a.plan.tile_base = a.plan.run_base + n_pages + 1;
  a.plan.n_pages = n_pages;
  a.plan.n_tiles = n_tiles;
  a.data = data;
  a.valid = valid;
  a.st = reinterpret_cast<PageState*>(d + off_st);
  a.tile_cnt = valid ? reinterpret_cast<int64_t*>(d + off_tc) : nullptr;
  a.tile_info = reinterpret_cast<int2*>(d + off_ti);
  a.bad = reinterpret_cast<unsigned long long*>(d_bad_pos ? (void*)d_bad_pos : (void*)(d + off_bad));
  a.runs = n_runs ? reinterpret_cast<uint2*>(d + off_runs) : nullptr;
  a.d_decoded = d_decoded;
  a.kind = kind; a.fixed_bw = fixed_bw; a.v1 = v1; a.width = width;
  a.dict_len = dict_len; a.dict = dict; a.out = out;
  if (valid && n_tiles) {
    pq_tile_count_kernel<<<grid_for(n_tiles, kRleThreads / 32, 8), kRleThreads, 0, st>>>(a);
    AG_TRY(check_launch("pq_tile_count_kernel"));
  }
  pq_runs_kernel<<<(unsigned)n_pages, kRleThreads, 0, st>>>(a);
  AG_TRY(check_launch("pq_runs_kernel"));
  ag_status rc;
  if (kind == kLevels) rc = launch_expand<kLevels, int16_t, false>(a, st);
  else if (kind == kDict && width == 4) rc = valid ? launch_expand<kDict, uint32_t, true>(a, st) : launch_expand<kDict, uint32_t, false>(a, st);
  else if (kind == kDict) rc = valid ? launch_expand<kDict, unsigned long long, true>(a, st) : launch_expand<kDict, unsigned long long, false>(a, st);
  else if (width == 4) rc = valid ? launch_expand<kPlain, uint32_t, true>(a, st) : launch_expand<kPlain, uint32_t, false>(a, st);
  else rc = valid ? launch_expand<kPlain, unsigned long long, true>(a, st) : launch_expand<kPlain, unsigned long long, false>(a, st);
  AG_TRY(rc);
  std::vector<PageState> hs((size_t)n_pages);
  int64_t bad = AG_NO_ERROR_POS;
  AG_TRY(d2h(hs.data(), a.st, st_bytes, st));
  if (kind == kDict) AG_TRY(d2h(&bad, a.bad, 8, st));
  AG_TRY(sync(st));
  if (h_decoded)
    for (int64_t i = 0; i < n_pages; ++i) h_decoded[i] = hs[i].slots;
  for (int64_t i = 0; i < n_pages; ++i)
    if (hs[i].err != kErrNone)
      AG_FAIL(AG_ERR_INVALID, "%s: page %lld: %s (%lld values decoded)", fn, (long long)i, err_text(hs[i].err), (long long)hs[i].slots);
  if (bad != AG_NO_ERROR_POS) AG_FAIL(AG_ERR_INVALID, "%s: invalid index values found for dictionary converter (output slot %lld)", fn, (long long)bad);
  return AG_OK;
}

// DELTA_BINARY_PACKED pages, same contract as parquet_pages_dev.  Launches: tile counts (spaced), the block walk, the
// tile sums, the per-page scan of the tile sums, and the unpack-scan-write pass.
static ag_status delta_pages_dev(int width, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages, const uint8_t* valid, void* out,
                                 int64_t* d_decoded, int64_t* h_decoded, cudaStream_t st) {
  const char* fn = "delta_decode";
  if (n_pages < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative page count", fn);
  if (n_pages == 0) return AG_OK;
  if (!pages) AG_FAIL(AG_ERR_INVALID, "%s: NULL page table", fn);
  // plan: pages | mb_base[n+1] | tile_base[n+1]
  const size_t pb = (size_t)n_pages * sizeof(ag_pq_page);
  const size_t plan_bytes = pb + 2 * (size_t)(n_pages + 1) * 8;
  std::vector<uint8_t> h(plan_bytes);
  memcpy(h.data(), pages, pb);
  int64_t* mb_base = reinterpret_cast<int64_t*>(h.data() + pb);
  int64_t* tile_base = mb_base + n_pages + 1;
  mb_base[0] = tile_base[0] = 0;
  bool any_data = false;
  for (int64_t i = 0; i < n_pages; ++i) {
    const ag_pq_page& g = pages[i];
    if (g.data < 0 || g.len < 0 || g.num_values < 0 || g.out < 0 || g.num_values > 0x7fffffffLL || g.len > 0xffffffffLL)
      AG_FAIL(AG_ERR_INVALID, "%s: page %lld: negative field, more than 2^31-1 values or more than 2^32-1 bytes", fn, (long long)i);
    any_data |= g.len > 0;
    mb_base[i + 1] = mb_base[i] + (g.num_values + 31) / 32;   // a miniblock holds >= 32 deltas
    tile_base[i + 1] = tile_base[i] + (g.num_values + kTile - 1) / kTile;
  }
  const int64_t n_mb = mb_base[n_pages], n_tiles = tile_base[n_pages];
  if (n_tiles > 0 && !out) AG_FAIL(AG_ERR_INVALID, "%s: NULL output", fn);
  if (any_data && !data) AG_FAIL(AG_ERR_INVALID, "%s: NULL page data", fn);
  if (out && (reinterpret_cast<uintptr_t>(out) & (width - 1))) AG_FAIL(AG_ERR_INVALID, "%s: output not aligned to its element width", fn);

  const size_t st_bytes = (size_t)n_pages * sizeof(DeltaPage);
  const size_t off_st = (plan_bytes + 255) & ~(size_t)255;
  const size_t off_tc = (off_st + st_bytes + 255) & ~(size_t)255;
  const size_t off_ts = (off_tc + (valid ? (size_t)n_tiles * 8 : 0) + 255) & ~(size_t)255;
  const size_t off_mb = (off_ts + (size_t)n_tiles * 8 + 255) & ~(size_t)255;
  const size_t total = off_mb + (size_t)n_mb * sizeof(DeltaMini);
  // this call synchronises `st` anyway, so its device scratch may live in a Temps
  Temps t(st);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, total));
  AG_TRY(h2d(d, h.data(), plan_bytes, st));
  DeltaArgs a;
  a.pages = reinterpret_cast<const ag_pq_page*>(d);
  a.mb_base = reinterpret_cast<const int64_t*>(d + pb);
  a.tile_base = a.mb_base + n_pages + 1;
  a.n_pages = n_pages;
  a.data = data;
  a.valid = valid;
  a.st = reinterpret_cast<DeltaPage*>(d + off_st);
  a.mb = reinterpret_cast<DeltaMini*>(d + off_mb);
  a.tile_cnt = valid ? reinterpret_cast<int64_t*>(d + off_tc) : nullptr;
  a.tile_sum = reinterpret_cast<unsigned long long*>(d + off_ts);
  a.d_decoded = d_decoded;
  a.width = width;
  a.out = out;
  if (valid && n_tiles) {
    PqArgs c{};                                                  // the tile counts of the other decoders
    c.plan.pages = a.pages; c.plan.tile_base = a.tile_base; c.plan.n_pages = n_pages; c.plan.n_tiles = n_tiles;
    c.valid = valid; c.tile_cnt = a.tile_cnt;
    pq_tile_count_kernel<<<grid_for(n_tiles, kRleThreads / 32, 8), kRleThreads, 0, st>>>(c);
    AG_TRY(check_launch("pq_tile_count_kernel"));
  }
  delta_walk_kernel<<<(unsigned)n_pages, kRleThreads, 0, st>>>(a);
  AG_TRY(check_launch("delta_walk_kernel"));
  if (n_tiles) {
    AG_TRY(visit_width(8 * width, [&](auto tag) -> ag_status {
      using T = typename decltype(tag)::type;
      if constexpr (sizeof(T) >= 4) return valid ? launch_delta_values<T, true>(a, n_tiles, st) : launch_delta_values<T, false>(a, n_tiles, st);
      else AG_FAIL(AG_ERR_INVALID, "%s: value_width must be 4 or 8", fn);
    }, [&] { AG_FAIL(AG_ERR_INVALID, "%s: value_width must be 4 or 8", fn); }));
  }
  std::vector<DeltaPage> hs((size_t)n_pages);
  AG_TRY(d2h(hs.data(), a.st, st_bytes, st));
  AG_TRY(sync(st));
  if (h_decoded)
    for (int64_t i = 0; i < n_pages; ++i) h_decoded[i] = hs[i].slots;
  for (int64_t i = 0; i < n_pages; ++i)
    if (hs[i].err != kDErrNone) {
      char msg[160];
      delta_err_text(hs[i], msg, sizeof msg);
      AG_FAIL(AG_ERR_INVALID, "%s: page %lld: %s (%lld values decoded)", fn, (long long)i, msg, (long long)hs[i].slots);
    }
  return AG_OK;
}

static int bit_len(int v) { int n = 0; while (v) { ++n; v >>= 1; } return n; }

static ag_status levels_args(int max_level, int encoding, int* bw) {
  if (encoding == AG_PQ_LEVELS_BIT_PACKED) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "levels_decode: deprecated BIT_PACKED levels are not implemented");
  if (encoding != AG_PQ_LEVELS_V1_RLE && encoding != AG_PQ_LEVELS_V2_RLE) AG_FAIL(AG_ERR_INVALID, "levels_decode: unknown level encoding %d", encoding);
  if (max_level < 0 || max_level > 0xffff) AG_FAIL(AG_ERR_INVALID, "levels_decode: max_level must be 0..65535 (bit width 0..16)");
  *bw = bit_len(max_level);
  return AG_OK;
}

// host flavours: stage the page bytes, validity and dictionary, decode, copy back only the slots each page wrote
static ag_status pages_host(int kind, int fixed_bw, int v1, int width, const void* dict, int64_t dict_len, const uint8_t* data,
                            const ag_pq_page* pages, int64_t n_pages, const uint8_t* valid, void* out, int64_t* decoded, int64_t* bad_pos) {
  if (bad_pos) *bad_pos = AG_NO_ERROR_POS;
  if (n_pages < 0) AG_FAIL(AG_ERR_INVALID, "negative page count");
  if (n_pages == 0) return AG_OK;
  if (!pages) AG_FAIL(AG_ERR_INVALID, "NULL page table");
  int64_t data_end = 0, slot_end = 0;
  for (int64_t i = 0; i < n_pages; ++i) {
    if (pages[i].data < 0 || pages[i].len < 0 || pages[i].num_values < 0 || pages[i].out < 0) AG_FAIL(AG_ERR_INVALID, "page %lld: negative field", (long long)i);
    if (pages[i].data + pages[i].len > data_end) data_end = pages[i].data + pages[i].len;
    if (pages[i].out + pages[i].num_values > slot_end) slot_end = pages[i].out + pages[i].num_values;
  }
  if (data_end > 0 && !data) AG_FAIL(AG_ERR_INVALID, "NULL page data");
  if (slot_end > 0 && !out) AG_FAIL(AG_ERR_INVALID, "NULL output");
  if (kind == kDict && dict_len > 0 && !dict) AG_FAIL(AG_ERR_INVALID, "NULL dictionary");
  const int esz = kind == kLevels ? 2 : width;
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  const size_t vbytes = valid ? (size_t)((slot_end + 7) >> 3) : 0;
  const size_t dbytes = kind == kDict ? (size_t)dict_len * width : 0;
  const size_t o_valid = ((size_t)data_end + 255) & ~(size_t)255;
  const size_t o_dict = (o_valid + vbytes + 255) & ~(size_t)255;
  const size_t o_out = (o_dict + dbytes + 255) & ~(size_t)255;
  const size_t o_bad = (o_out + (size_t)slot_end * esz + 255) & ~(size_t)255;
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, o_bad));
  AG_TRY(h2d(d, data, (size_t)data_end, cs));
  AG_TRY(h2d(d + o_valid, valid, vbytes, cs));
  AG_TRY(h2d(d + o_dict, dict, dbytes, cs));
  std::vector<int64_t> dec((size_t)n_pages, 0);   // stays 0 when the call fails before decoding
  const ag_status rc = kind == kDelta
      ? delta_pages_dev(width, d, pages, n_pages, vbytes ? d + o_valid : nullptr, d + o_out, nullptr, dec.data(), cs)
      : parquet_pages_dev(kind, fixed_bw, v1, width, dbytes ? d + o_dict : nullptr, dict_len, d, pages, n_pages,
                          vbytes ? d + o_valid : nullptr, d + o_out, nullptr, dec.data(), reinterpret_cast<int64_t*>(d + o_bad), cs);
  // a decode error still delivers the values decoded before it
  if (rc != AG_OK && rc != AG_ERR_INVALID) return rc;
  if (decoded) memcpy(decoded, dec.data(), (size_t)n_pages * 8);
  for (int64_t i = 0; i < n_pages; ++i) {
    const size_t off = (size_t)pages[i].out * esz;
    AG_TRY(d2h((uint8_t*)out + off, d + o_out + off, (size_t)dec[i] * esz, cs));
  }
  if (kind == kDict && bad_pos) AG_TRY(d2h(bad_pos, d + o_bad, 8, cs));
  const ag_status rs = sync(cs);
  return rc != AG_OK ? rc : rs;
}

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_parquet_levels_decode_dev(int max_level, int encoding, const uint8_t* d_data, const ag_pq_page* pages, int64_t n_pages,
                                       int16_t* d_out, int64_t* d_decoded, ag_stream_t s) {
  AG_TRY(ensure_init());
  int bw;
  AG_TRY(levels_args(max_level, encoding, &bw));
  return parquet_pages_dev(kLevels, bw, encoding == AG_PQ_LEVELS_V1_RLE, 2, nullptr, 0, d_data, pages, n_pages, nullptr, d_out, d_decoded,
                           nullptr, nullptr, resolve_stream(s));
}

ag_status ag_parquet_levels_decode(int max_level, int encoding, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages,
                                   int16_t* out, int64_t* decoded) {
  AG_TRY(ensure_init());
  int bw;
  AG_TRY(levels_args(max_level, encoding, &bw));
  return pages_host(kLevels, bw, encoding == AG_PQ_LEVELS_V1_RLE, 2, nullptr, 0, data, pages, n_pages, nullptr, out, decoded, nullptr);
}

ag_status ag_parquet_dict_decode_dev(int value_width, const void* d_dict, int64_t dict_len, const uint8_t* d_data, const ag_pq_page* pages,
                                     int64_t n_pages, const uint8_t* d_valid, void* d_out, int64_t* d_decoded, int64_t* d_bad_pos, ag_stream_t s) {
  AG_TRY(ensure_init());
  if (value_width != 4 && value_width != 8) AG_FAIL(AG_ERR_INVALID, "dict_decode: value_width must be 4 or 8");
  if (dict_len < 0) AG_FAIL(AG_ERR_INVALID, "dict_decode: negative dictionary length");
  return parquet_pages_dev(kDict, 0, 0, value_width, d_dict, dict_len, d_data, pages, n_pages, d_valid, d_out, d_decoded, nullptr, d_bad_pos,
                           resolve_stream(s));
}

ag_status ag_parquet_dict_decode(int value_width, const void* dict, int64_t dict_len, const uint8_t* data, const ag_pq_page* pages,
                                 int64_t n_pages, const uint8_t* valid, void* out, int64_t* decoded, int64_t* bad_pos) {
  AG_TRY(ensure_init());
  if (bad_pos) *bad_pos = AG_NO_ERROR_POS;
  if (value_width != 4 && value_width != 8) AG_FAIL(AG_ERR_INVALID, "dict_decode: value_width must be 4 or 8");
  if (dict_len < 0) AG_FAIL(AG_ERR_INVALID, "dict_decode: negative dictionary length");
  return pages_host(kDict, 0, 0, value_width, dict, dict_len, data, pages, n_pages, valid, out, decoded, bad_pos);
}

ag_status ag_parquet_plain_decode_spaced_dev(int value_width, const uint8_t* d_data, const ag_pq_page* pages, int64_t n_pages,
                                             const uint8_t* d_valid, void* d_out, ag_stream_t s) {
  AG_TRY(ensure_init());
  if (value_width != 4 && value_width != 8) AG_FAIL(AG_ERR_INVALID, "plain_decode_spaced: value_width must be 4 or 8");
  return parquet_pages_dev(kPlain, 0, 0, value_width, nullptr, 0, d_data, pages, n_pages, d_valid, d_out, nullptr, nullptr, nullptr,
                           resolve_stream(s));
}

ag_status ag_parquet_plain_decode_spaced(int value_width, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages,
                                         const uint8_t* valid, void* out) {
  AG_TRY(ensure_init());
  if (value_width != 4 && value_width != 8) AG_FAIL(AG_ERR_INVALID, "plain_decode_spaced: value_width must be 4 or 8");
  return pages_host(kPlain, 0, 0, value_width, nullptr, 0, data, pages, n_pages, valid, out, nullptr, nullptr);
}

ag_status ag_parquet_delta_decode_dev(int value_width, const uint8_t* d_data, const ag_pq_page* pages, int64_t n_pages,
                                      const uint8_t* d_valid, void* d_out, int64_t* d_decoded, ag_stream_t s) {
  AG_TRY(ensure_init());
  if (value_width != 4 && value_width != 8) AG_FAIL(AG_ERR_INVALID, "delta_decode: value_width must be 4 (INT32) or 8 (INT64)");
  return delta_pages_dev(value_width, d_data, pages, n_pages, d_valid, d_out, d_decoded, nullptr, resolve_stream(s));
}

ag_status ag_parquet_delta_decode(int value_width, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages,
                                  const uint8_t* valid, void* out, int64_t* decoded) {
  AG_TRY(ensure_init());
  if (value_width != 4 && value_width != 8) AG_FAIL(AG_ERR_INVALID, "delta_decode: value_width must be 4 (INT32) or 8 (INT64)");
  return pages_host(kDelta, 0, 0, value_width, nullptr, 0, data, pages, n_pages, valid, out, decoded, nullptr);
}

}  // extern "C"
