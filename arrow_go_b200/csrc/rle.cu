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

enum PqKind { kLevels = 0, kDict = 1, kPlain = 2 };

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

__device__ __forceinline__ int block_excl_scan(int v, int* warp_tot, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_tot[wid] = x;
  __syncthreads();
  int off = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kRleThreads / 32; ++w) {
    const int t = warp_tot[w];
    off += (w < wid) ? t : 0;
    tot += t;
  }
  __syncthreads();
  *total = tot;
  return off + x - v;
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
  int64_t need = pg.num_values;
  if (a.valid) {
    const int64_t t0 = a.plan.tile_base[p], t1 = a.plan.tile_base[p + 1];
    int64_t run = 0;
    for (int64_t t = t0; t < t1; t += kRleThreads) {
      const int c = (t + tid < t1) ? (int)a.tile_cnt[t + tid] : 0;
      int tot;
      const int ex = block_excl_scan(c, warp_tot, &tot);
      if (t + tid < t1) a.tile_cnt[t + tid] = run + ex;   // now the tile's first dense rank
      run += tot;
    }
    need = run;
  }

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
      slots = pg.num_values;
      if (produced < need) {
        const int64_t t0 = a.plan.tile_base[p], t1 = a.plan.tile_base[p + 1];
        int64_t t = t0;
        while (t + 1 < t1 && a.tile_cnt[t + 1] <= produced) ++t;
        int64_t rank = a.tile_cnt[t];
        int64_t s = (t - t0) * kTile;
        for (;; ++s) {                                           // the produced-th valid slot lies in tile t
          if (bit_is_set(a.valid, pg.out + s)) { if (rank == produced) break; ++rank; }
        }
        slots = s;
      }
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
  const ag_status rc = parquet_pages_dev(kind, fixed_bw, v1, width, dbytes ? d + o_dict : nullptr, dict_len, d, pages, n_pages,
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

}  // extern "C"
