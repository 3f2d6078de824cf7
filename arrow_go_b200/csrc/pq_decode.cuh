// pq_decode.cuh — the Parquet page-decode building blocks shared by fixed.cu, rle.cu and byte_array.cu.  Internal, not
// part of the ABI.  The device passes: tile counts, the RLE/bit-packed run walk and expansion, and the
// DELTA_BINARY_PACKED block walk, tile sums and scan (rle.cu's header describes those).  The tile helpers every page
// kernel shares: segment_excl_scan (one block's scan of per-tile values), spaced_rank (a spaced slot's dense rank),
// tile_last_run and find_run (the run holding a rank).  The host side every page driver shares: the checked page plan
// and its upload, the tile-count launch, the read-back of the per-page states, and the host flavour's staging.
//
// A call decodes a batch of pages (ag_pq_page descriptors, one device buffer of page payloads) in three launches:
//   1. pq_tile_count_kernel (spaced only): valid bits per 1024-slot tile of every page.
//   2. pq_runs_kernel, one block per page: scans the page's tile counts into dense-rank bases, then streams the page
//      bytes through the shared-memory window of pq_window.cuh while thread 0 walks the run headers (the chain is
//      sequential; the parallelism comes from the pages).  Each run becomes an 8-byte descriptor {first dense value | literal flag,
//      repeated value or payload byte offset}; the page records its run count, decoded count and an error code.
//      Windows start at the next header, so the bytes of long literal runs between two windows are never loaded.
//   3. pq_expand_kernel, one block per 1024-slot tile of output: finds its page and run by binary search, broadcasts
//      repeated values, unpacks literal values with aligned 32-bit loads + funnel shift, gathers dictionary values
//      (the dictionary stays in L2) with the bounds check fused, and maps slots to dense ranks with spaced_rank (null
//      slots get 0, like FillZero).
// Roofline.  Single pass: encoded bytes read once + values written once (+ 1 bit of validity per slot).  This design
// reads the encoded bytes up to twice (pass 2 only touches the headers' windows and the payload it expands) and
// writes 8 B per run descriptor, so its own bound is (2 x encoded + written) bytes of HBM traffic; the dictionary
// gather is served from L2.
#pragma once

#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "host_stage.cuh"
#include "pq_window.cuh"

namespace ag {

namespace {

constexpr int kRleThreads = kPqThreads;
constexpr int kTile = 1024;                 // output slots per expansion block (4 per thread)
constexpr uint32_t kLiteralFlag = 0x80000000u;

// kIndex: dictionary indices themselves (int32; an index >= dict_len becomes -1 and lowers *bad), for dictionaries the
// expansion cannot gather from, such as byte arrays.  fixed.cu adds an expansion kind and three pass-1 kinds:
//   kRank      (expansion only) the dense rank of every valid slot (int32), for values of any width gathered later
//   kBss       pass 1: BYTE_STREAM_SPLIT page geometry, stride = len / width, checked as SetData does; expansion (4- and
//              8-byte values): each slot's value assembled in a register from its byte in every stream
//   kBoolPlain (pass 1 only) bit-packed PLAIN booleans: need <= 8 * len
//   kBoolRle   (pass 1 only) RLE booleans: a 4-byte length prefix on every page, then runs of bit width 1
enum PqKind { kLevels = 0, kDict = 1, kPlain = 2, kDelta = 3, kIndex = 4, kRank = 5, kBss = 6, kBoolPlain = 7, kBoolRle = 8 };

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
  // fixed.cu's kinds; each but kErrBoolEof delivers nothing of the page
  kErrBssSize = 9,         // BYTE_STREAM_SPLIT: more bytes than num_values values
  kErrBssAlign = 10,       // BYTE_STREAM_SPLIT: bytes not a multiple of the width
  kErrBssEof = 11,         // BYTE_STREAM_SPLIT: the values to read take more than 2^31-1 bytes
  kErrBssShort = 12,       // BYTE_STREAM_SPLIT spaced: fewer values than valid slots
  kErrBoolShort = 13,      // PLAIN booleans: fewer bits than values
  kErrBoolLength = 14,     // RLE booleans: page shorter than its 4-byte length
  kErrBoolBytes = 15,      // RLE booleans: length past the page (PageState.pad holds it)
  kErrBoolEof = 16,        // RLE booleans: the stream ends before the values the page needs
};

__host__ __device__ __forceinline__ bool err_delivers_nothing(int e) { return e == kErrPlainShort || (e >= kErrBssSize && e <= kErrBoolBytes); }

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

// One block turns v[t0, t1) into its exclusive prefix sums in place, kRleThreads values per step, and returns the
// total.  S is the block scan's element type (warp_tot holds kRleThreads / 32 of them); the running sum keeps V's width.
template <typename S, typename V>
__device__ __forceinline__ V segment_excl_scan(V* v, int64_t t0, int64_t t1, S* warp_tot) {
  V run = 0;
  for (int64_t t = t0; t < t1; t += kRleThreads) {
    const int64_t i = t + threadIdx.x;
    const S x = i < t1 ? (S)v[i] : (S)0;
    S tot;
    const S ex = block_excl_scan(x, warp_tot, &tot);
    if (i < t1) v[i] = run + ex;
    run += tot;
  }
  return run;
}

// spaced: turns the valid counts of a page's tiles [t0, t1) into each tile's first dense rank (one block per page);
// returns the page's valid count
__device__ __forceinline__ int64_t scan_tile_ranks(int64_t* tile_cnt, int64_t t0, int64_t t1, int* warp_tot) {
  return segment_excl_scan(tile_cnt, t0, t1, warp_tot);
}

// spaced: one slot per thread of a step of kRleThreads slots, at bit `bit` of the validity bitmap.  Sets v to its
// validity (false when !in) and returns its dense rank, by a ballot scan of the step's validity bits from rank_base,
// which then advances past the step.  Holds two block barriers: every thread of the block calls it.
__device__ __forceinline__ int64_t spaced_rank(bool in, const uint8_t* valid, int64_t bit, int* warp_tot, int64_t& rank_base, bool& v) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  v = in && bit_is_set(valid, bit);
  const unsigned m = __ballot_sync(0xffffffffu, v);
  if (lane == 0) warp_tot[wid] = __popc(m);
  __syncthreads();
  int off = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kRleThreads / 32; ++w) { const int t = warp_tot[w]; off += (w < wid) ? t : 0; tot += t; }
  __syncthreads();
  const int64_t rank = rank_base + off + __popc(m & ((1u << lane) - 1u));
  rank_base += tot;
  return rank;
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

// output slots a page's first `produced` dense values fill: none when its error delivers nothing (DecodeSpaced), else
// every slot up to the first valid slot whose value was not delivered; the page's tiles are [t0, t1)
__device__ __forceinline__ int64_t slots_written(const uint8_t* valid, const ag_pq_page& pg, const int64_t* tile_cnt, int64_t t0, int64_t t1,
                                                 int64_t need, int64_t produced, bool nothing) {
  if (nothing) return 0;
  if (!valid) return produced;
  return produced < need ? slot_of_rank(valid, pg.out, tile_cnt, t0, t1, produced) : pg.num_values;
}

// one block per page: stream geometry, spaced rank bases, run table
__global__ void __launch_bounds__(kRleThreads)
pq_runs_kernel(PqArgs a) {
  __shared__ uint4 win[kWinVec];
  __shared__ int warp_tot[kRleThreads / 32];
  __shared__ int64_t s_pos, s_produced;
  __shared__ int s_done, s_nruns, s_err, s_bw;
  __shared__ int64_t s_stream, s_len;
  __shared__ uint32_t s_arg;
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
    s_arg = 0;
    if (a.kind == kLevels && a.v1) {
      if (len < 4) {
        err = kErrLevelsShort; len = 0;
      } else {
        const uint8_t* b = a.data + pg.data;
        const int32_t nb = (int32_t)((uint32_t)b[0] | ((uint32_t)b[1] << 8) | ((uint32_t)b[2] << 16) | ((uint32_t)b[3] << 24));
        if (nb < 0 || (int64_t)nb > len - 4) { err = kErrLevelsLength; len = 0; }
        else { stream += 4; len = nb; }
      }
    } else if (a.kind == kDict || a.kind == kIndex) {
      if (len == 0) {
        bw = 0;                                          // no data: bit width 0 (decoder.go:127-131)
      } else {
        bw = a.data[pg.data];
        stream += 1; len -= 1;
        if (bw > 32) { err = kErrBitWidth; len = 0; }
      }
    } else if (a.kind == kBoolRle) {                     // RleBooleanDecoder.SetData (boolean_decoder.go:321-341)
      if (len < 4) {
        err = kErrBoolLength;
      } else {
        const uint8_t* b = a.data + pg.data;
        const uint32_t nb = (uint32_t)b[0] | ((uint32_t)b[1] << 8) | ((uint32_t)b[2] << 16) | ((uint32_t)b[3] << 24);
        if ((int64_t)nb > len - 4) { err = kErrBoolBytes; s_arg = nb; }
        else { stream += 4; len = nb; }
      }
    }
    const bool one_pass = a.kind == kPlain || a.kind == kBss || a.kind == kBoolPlain;
    s_stream = stream; s_len = err ? 0 : len; s_bw = bw; s_err = err;
    s_pos = 0; s_produced = 0; s_nruns = 0;
    s_done = (err != kErrNone || one_pass) ? 1 : 0;
    if (a.kind == kPlain) {
      const int64_t have = len / a.width;
      if (need > have) { s_err = kErrPlainShort; s_produced = 0; }
      else s_produced = need;
    } else if (a.kind == kBoolPlain) {
      if (need > len * 8) s_err = kErrBoolShort;           // ensureBitsAvailable (boolean_decoder.go:57-63)
      else s_produced = need;
    } else if (a.kind == kBss) {                         // validateByteStreamSplitPageData, Decode, DecodeSpaced
      const int64_t w = a.width;
      const int64_t to_read = need < len / w ? need : len / w;
      if (pg.num_values * w < len) s_err = kErrBssSize;
      else if (len % w) s_err = kErrBssAlign;
      else if (to_read * w > 0x7fffffffLL) s_err = kErrBssEof;
      else if (a.valid && to_read < need) s_err = kErrBssShort;
      else s_produced = to_read;                         // dense: min(num_values, stride)
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
    // the window starts at the 16-byte aligned start of the next header
    const uintptr_t sbeg = reinterpret_cast<uintptr_t>(a.data) + stream;
    const uintptr_t a0 = (sbeg + s_pos) & ~(uintptr_t)15;
    load_window(win, sbeg, sbeg + len, a0);
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
    // RleBooleanDecoder.DecodeToBitmap: a short stream is io.ErrUnexpectedEOF after the values delivered
    if (a.kind == kBoolRle && s_err == kErrNone && produced < need) s_err = kErrBoolEof;
    const int64_t slots = slots_written(a.valid, pg, a.tile_cnt, a.plan.tile_base[p], a.plan.tile_base[p + 1], need, produced,
                                        err_delivers_nothing(s_err));
    PageState ps;
    ps.stream = stream; ps.stream_len = len; ps.need = need; ps.produced = produced; ps.slots = slots;
    ps.nruns = s_nruns; ps.bw = bw; ps.err = s_err; ps.pad = (int32_t)s_arg;
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

// The runs of tile `tile` (ti = tile_info[tile]) that hold every rank it needs are [ti.y, tile_last_run]: from the
// run holding its first rank to the run holding the next tile's first rank, or the page's last run for its last tile.
__device__ __forceinline__ int64_t tile_last_run(const PqArgs& a, int64_t tile, int2 ti, int32_t nruns) {
  const int64_t p = ti.x, lo = ti.y;
  int64_t hi = tile + 1 < a.plan.tile_base[p + 1] ? a.tile_info[tile + 1].y : nruns - 1;
  if (hi < lo) hi = lo;
  return hi;
}

// the run of runs[lo..hi] that holds dense rank `rank`
__device__ __forceinline__ uint2 find_run(const uint2* runs, int64_t lo, int64_t hi, int64_t rank) {
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if ((int64_t)(runs[mid].x & ~kLiteralFlag) <= rank) lo = mid; else hi = mid - 1;
  }
  return runs[lo];
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
  const int tid = threadIdx.x;
  const uint2* runs = a.runs + (KIND == kPlain || KIND == kRank || KIND == kBss ? 0 : a.plan.run_base[p]);
  const uint8_t* stream = a.data + ps.stream;
  T* out = reinterpret_cast<T*>(a.out) + pg.out;

  const int64_t rhi = tile_last_run(a, tile, ti, ps.nruns);

  int64_t rank_base = SPACED ? a.tile_cnt[tile] : s0;   // the tile's first dense rank
#pragma unroll
  for (int q = 0; q < kTile / kRleThreads; ++q) {
    const int64_t s = s0 + q * kRleThreads + tid;
    const bool in = s < limit;
    bool v = in;
    int64_t rank = s;
    if (SPACED) rank = spaced_rank(in, a.valid, pg.out + s, warp_tot, rank_base, v);
    if (!in) continue;
    if (!v) { out[s] = (T)0; continue; }
    uint32_t idx;
    if (KIND == kPlain) {
      out[s] = load_unaligned<T>(stream + rank * (int64_t)sizeof(T));
      continue;
    } else if (KIND == kRank) {
      out[s] = (T)rank;
      continue;
    } else if (KIND == kBss) {
      // byte j of rank r is stream[j * stride + r]: consecutive lanes read consecutive bytes of each stream
      const int64_t stride = ps.stream_len / (int64_t)sizeof(T);
      T v = 0;
#pragma unroll
      for (int j = 0; j < (int)sizeof(T); ++j) v |= (T)__ldg(stream + j * stride + rank) << (8 * j);
      out[s] = v;
      continue;
    } else {
      const uint2 r = find_run(runs, ti.y, rhi, rank);
      idx = (r.x & kLiteralFlag) ? unpack_at(stream + r.y, rank - (int64_t)(r.x & ~kLiteralFlag), ps.bw) : r.y;
    }
    if (KIND == kLevels) {
      out[s] = (T)idx;
    } else if (KIND == kIndex) {
      if ((int64_t)idx < a.dict_len) {
        out[s] = (T)idx;
      } else {
        out[s] = (T)-1;
        atomicMin(a.bad, (unsigned long long)(pg.out + s));
      }
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
  int64_t end;              // bytes of the stream the walk consumed (bytesRead() once every value is decoded)
  uint32_t vpm;
  int32_t err;
};

struct DeltaArgs {
  const ag_pq_page* pages;
  const int64_t* mb_base;   // [n_pages + 1]: first miniblock descriptor of every page
  const int64_t* tile_base; // [n_pages + 1]: first output tile of every page
  int64_t n_pages;
  const uint8_t* data;
  const int64_t* skip;      // may be NULL: per page, bytes before the stream (a DELTA_BYTE_ARRAY page's suffix lengths)
  const uint8_t* valid;     // NULL = every slot valid
  DeltaPage* st;
  DeltaMini* mb;
  int64_t* tile_cnt;        // spaced only: valid bits per tile, then the tile's first dense rank
  unsigned long long* tile_sum;   // per tile: sum of its deltas, then (after tile_sum_scan_kernel) of the page's deltas before it
  int64_t* d_decoded;       // may be NULL
  int width;                // 4 (INT32) or 8 (INT64)
  void* out;
};

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
  const int64_t skip = a.skip ? min(a.skip[p], pg.len) : 0;
  const uint8_t* page = a.data + pg.data + skip;
  const int64_t len = pg.len - skip;

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
    // the window starts at the 16-byte aligned start of the next block header
    const uintptr_t sbeg = reinterpret_cast<uintptr_t>(page);
    const uintptr_t a0 = (sbeg + w.pos) & ~(uintptr_t)15;
    load_window(win, sbeg, sbeg + len, a0);
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
    const int64_t slots = slots_written(a.valid, pg, a.tile_cnt, t0, t1, need, produced, err == kDErrShort);
    DeltaPage ps;
    ps.first = s_first; ps.produced = produced; ps.slots = slots; ps.arg0 = w.arg0; ps.arg1 = w.arg1; ps.end = w.pos;
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
// Spaced slots map to dense ranks through spaced_rank.  T is the physical width, so every sum wraps like the reference's
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
  const int tid = threadIdx.x;
  if (s0 >= ps.slots) {                                          // block-uniform
    if (!WRITE && tid == 0) a.tile_sum[tile] = 0;
    return;
  }
  const uint8_t* page = a.data + pg.data + (a.skip ? min(a.skip[p], pg.len) : 0);
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
    if (SPACED) rank = spaced_rank(in, a.valid, pg.out + s, warp_cnt, rank_base, v);
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

// one block per page: per-tile sums (of deltas, or of BYTE_ARRAY lengths) -> the sum of the page's tiles before each
// tile, wrapping at 64 bits
__global__ void __launch_bounds__(kRleThreads)
tile_sum_scan_kernel(const int64_t* tile_base, unsigned long long* sums) {
  __shared__ unsigned long long warp_sum[kRleThreads / 32];
  segment_excl_scan(sums, tile_base[blockIdx.x], tile_base[blockIdx.x + 1], warp_sum);
}

template <typename T, bool SPACED>
ag_status launch_delta_values(const DeltaArgs& a, int64_t n_tiles, cudaStream_t st) {
  delta_values_kernel<T, SPACED, false><<<(unsigned)n_tiles, kRleThreads, 0, st>>>(a);
  AG_TRY(check_launch("delta_values_kernel"));
  tile_sum_scan_kernel<<<(unsigned)a.n_pages, kRleThreads, 0, st>>>(a.tile_base, a.tile_sum);
  AG_TRY(check_launch("tile_sum_scan_kernel"));
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

// ---------------------------------------------------------------- host side of every page driver ----
// A checked page table and the plan the device reads: pages | desc_base[n+1] | tile_base[n+1], where desc_base is
// every page's first descriptor (runs, or DELTA_BINARY_PACKED miniblocks) and tile_base its first 1024-slot tile.
struct PagePlan {
  std::vector<uint8_t> bytes;         // a caller may append its own page data before upload_plan
  int64_t n_pages = 0, n_desc = 0, n_tiles = 0;
  int64_t data_end = 0, slot_end = 0; // one past the last page byte / output slot
  bool any_data = false;              // some page has bytes
  int64_t* desc_base() { return reinterpret_cast<int64_t*>(bytes.data() + (size_t)n_pages * sizeof(ag_pq_page)); }
  int64_t* tile_base() { return desc_base() + n_pages + 1; }
};

// Checks `pages` and plans them; cap(page) is the number of descriptors a page may need.  No page gives an empty plan.
template <typename Cap>
static inline ag_status plan_pages(const char* fn, const ag_pq_page* pages, int64_t n_pages, Cap cap, PagePlan* p) {
  if (n_pages < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative page count", fn);
  if (n_pages > 0 && !pages) AG_FAIL(AG_ERR_INVALID, "%s: NULL page table", fn);
  const size_t pb = (size_t)n_pages * sizeof(ag_pq_page);
  p->n_pages = n_pages;
  p->bytes.assign(pb + 2 * (size_t)(n_pages + 1) * 8, 0);
  if (n_pages) memcpy(p->bytes.data(), pages, pb);
  int64_t *desc_base = p->desc_base(), *tile_base = p->tile_base();
  for (int64_t i = 0; i < n_pages; ++i) {
    const ag_pq_page& g = pages[i];
    if (g.data < 0 || g.len < 0 || g.num_values < 0 || g.out < 0 || g.num_values > 0x7fffffffLL || g.len > 0xffffffffLL)
      AG_FAIL(AG_ERR_INVALID, "%s: page %lld: negative field, more than 2^31-1 values or more than 2^32-1 bytes", fn, (long long)i);
    desc_base[i + 1] = desc_base[i] + cap(g);
    tile_base[i + 1] = tile_base[i] + (g.num_values + kTile - 1) / kTile;
    p->data_end = std::max(p->data_end, g.data + g.len);
    p->slot_end = std::max(p->slot_end, g.out + g.num_values);
    p->any_data |= g.len > 0;
  }
  p->n_desc = desc_base[n_pages];
  p->n_tiles = tile_base[n_pages];
  return AG_OK;
}

// Uploads the plan to device memory `d` (p.bytes.size() bytes) and returns its device views.
static inline ag_status upload_plan(const PagePlan& p, uint8_t* d, cudaStream_t st, PqPlan* out) {
  AG_TRY(h2d(d, p.bytes.data(), p.bytes.size(), st));
  out->pages = reinterpret_cast<const ag_pq_page*>(d);
  out->run_base = reinterpret_cast<const int64_t*>(d + (size_t)p.n_pages * sizeof(ag_pq_page));
  out->tile_base = out->run_base + p.n_pages + 1;
  out->n_pages = p.n_pages;
  out->n_tiles = p.n_tiles;
  return AG_OK;
}

// spaced calls: the valid bits of every tile into tile_cnt
static inline ag_status launch_tile_counts(const PqPlan& plan, const uint8_t* valid, int64_t* tile_cnt, cudaStream_t st) {
  if (!valid || plan.n_tiles == 0) return AG_OK;
  PqArgs c{};
  c.plan = plan; c.valid = valid; c.tile_cnt = tile_cnt;
  pq_tile_count_kernel<<<grid_for(plan.n_tiles, kRleThreads / 32, 8), kRleThreads, 0, st>>>(c);
  return check_launch("pq_tile_count_kernel");
}

// The end of a driver: copies the per-page states back, synchronises `st` once, fills h_decoded (host, may be NULL),
// fails on the lowest failing page with the text text(page, state, buf, size) gives, then on the lowest out-of-range
// dictionary index in *d_bad (NULL: the call looks up no dictionary).
template <typename S, typename Text>
ag_status read_back(const char* fn, const S* d_st, int64_t n_pages, const unsigned long long* d_bad, int64_t* h_decoded,
                    cudaStream_t st, Text text) {
  std::vector<S> hs((size_t)n_pages);
  int64_t bad = AG_NO_ERROR_POS;
  AG_TRY(d2h(hs.data(), d_st, (size_t)n_pages * sizeof(S), st));
  if (d_bad) AG_TRY(d2h(&bad, d_bad, 8, st));
  AG_TRY(sync(st));
  if (h_decoded)
    for (int64_t i = 0; i < n_pages; ++i) h_decoded[i] = hs[i].slots;
  for (int64_t i = 0; i < n_pages; ++i)
    if (hs[i].err != 0) {
      char msg[200];
      text(i, hs[i], msg, sizeof msg);
      AG_FAIL(AG_ERR_INVALID, "%s: page %lld: %s (%lld values decoded)", fn, (long long)i, msg, (long long)hs[i].slots);
    }
  if (bad != AG_NO_ERROR_POS) AG_FAIL(AG_ERR_INVALID, "%s: invalid index values found for dictionary converter (output slot %lld)", fn, (long long)bad);
  return AG_OK;
}

// One call of a fixed-width or DELTA_BINARY_PACKED page entry point.  `pages` is host memory; the other pointers are
// host memory in a host flavour and device memory in a device flavour.
struct PqCall {
  const char* fn;           // message prefix
  int job;                  // fixed.cu: what runs after pass 1
  int ptype;                // AG_PQ_TYPE_* where the error texts depend on it, else 0
  int width;                // bytes per output slot (booleans: 1)
  int fixed_bw;             // levels: bits.Len(max_level); RLE booleans: 1
  int v1;                   // levels: 4-byte length prefix
  bool bitmap;              // booleans: `out` is a bitmap
  const uint8_t* data;
  const ag_pq_page* pages;
  int64_t n_pages;
  const uint8_t* valid;     // NULL = every slot valid
  const void* dict;
  int64_t dict_len;         // 0 unless the pages are dictionary-encoded
  void* out;
};

// A device flavour: decodes `c`, fills h_decoded (host, may be NULL), synchronises `st` once.
typedef ag_status (*pq_pages_dev_fn)(const PqCall& c, int64_t* d_decoded, int64_t* h_decoded, int64_t* d_bad_pos, cudaStream_t st);

// host flavour: stage the page bytes, validity and dictionary, decode, copy back only the slots each page wrote.  A
// boolean bitmap's bytes up to the last page's last slot go up and come back whole, so every bit the call does not
// write keeps its value.
static inline ag_status pq_pages_host(pq_pages_dev_fn dev, const PqCall& c, int64_t* decoded, int64_t* bad_pos) {
  const char* fn = c.fn;
  PagePlan plan;
  AG_TRY(plan_pages(fn, c.pages, c.n_pages, [](const ag_pq_page&) { return (int64_t)0; }, &plan));
  if (c.n_pages == 0) return AG_OK;
  if (plan.data_end > 0 && !c.data) AG_FAIL(AG_ERR_INVALID, "%s: NULL page data", fn);
  if (plan.slot_end > 0 && !c.out) AG_FAIL(AG_ERR_INVALID, "%s: NULL output", fn);
  if (c.dict_len > 0 && !c.dict) AG_FAIL(AG_ERR_INVALID, "%s: NULL dictionary", fn);
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  const size_t vbytes = c.valid ? (size_t)((plan.slot_end + 7) >> 3) : 0;
  const size_t dbytes = (size_t)c.dict_len * c.width;
  const size_t obytes = c.bitmap ? (size_t)((plan.slot_end + 7) >> 3) : (size_t)plan.slot_end * c.width;
  Carve sc;
  const size_t o_data = sc.take((size_t)plan.data_end), o_valid = sc.take(vbytes), o_dict = sc.take(dbytes);
  const size_t o_out = sc.take(obytes), o_bad = sc.take(8);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, sc.size));
  AG_TRY(h2d(d + o_data, c.data, (size_t)plan.data_end, cs));
  AG_TRY(h2d(d + o_valid, c.valid, vbytes, cs));
  AG_TRY(h2d(d + o_dict, c.dict, dbytes, cs));
  // *bad_pos is copied back whatever happens: it reads AG_NO_ERROR_POS when the call fails before any kernel runs
  static const int64_t kNone = AG_NO_ERROR_POS;
  AG_TRY(h2d(d + o_bad, &kNone, 8, cs));
  if (c.bitmap) AG_TRY(h2d(d + o_out, c.out, obytes, cs));
  PqCall dc = c;
  dc.data = d + o_data;
  dc.valid = vbytes ? d + o_valid : nullptr;
  dc.dict = dbytes ? d + o_dict : nullptr;
  dc.out = d + o_out;
  std::vector<int64_t> dec((size_t)c.n_pages, 0);   // stays 0 when the call fails before decoding
  const ag_status rc = dev(dc, nullptr, dec.data(), reinterpret_cast<int64_t*>(d + o_bad), cs);
  // a decode error still delivers the values decoded before it
  if (rc != AG_OK && rc != AG_ERR_INVALID) return rc;
  if (decoded) memcpy(decoded, dec.data(), (size_t)c.n_pages * 8);
  if (c.bitmap) {
    AG_TRY(d2h(c.out, d + o_out, obytes, cs));
  } else {
    for (int64_t i = 0; i < c.n_pages; ++i) {
      const size_t off = (size_t)c.pages[i].out * c.width;
      AG_TRY(d2h((uint8_t*)c.out + off, d + o_out + off, (size_t)dec[i] * c.width, cs));
    }
  }
  if (bad_pos) AG_TRY(d2h(bad_pos, d + o_bad, 8, cs));
  const ag_status rs = sync(cs);
  return rc != AG_OK ? rc : rs;
}

}  // namespace

}  // namespace ag
