// fixed.cu — the fixed-width Parquet page driver: definition / repetition levels, dictionary-encoded and PLAIN spaced
// 4- and 8-byte values, BOOLEAN (PLAIN bit-packed, RLE) into an Arrow boolean bitmap, and INT32 / INT64 / FLOAT /
// DOUBLE / INT96 / FIXED_LEN_BYTE_ARRAY (PLAIN, dictionary, BYTE_STREAM_SPLIT) into `width` bytes per slot.
//   RleDecoder.Next / GetBatch                                   parquet/internal/utils/rle.go:123-169,203-239
//   LevelDecoder.SetData / SetDataV2 / Decode                    parquet/internal/encoding/levels.go:188-297
//   dictDecoder.SetData / decode / decodeSpaced                  decoder.go:125-160 over
//                                                                TypedRleDecoder.GetBatchWithDict[Spaced] (utils/typed_rle_dict.go:143-236)
//   PlainDecoder.DecodeSpaced                                    plain_encoding_types.go:98 -> spacedExpand (decoder.go:209)
//   PlainBooleanDecoder.DecodeToBitmap / decodeSpacedToBitmap   parquet/internal/encoding/boolean_decoder.go:264-304
//   RleBooleanDecoder.SetData / DecodeToBitmap                   boolean_decoder.go:321-341,382-417
//   PlainDecoder[T] (INT96 too)                                  plain_encoding_types.go:61-110
//   PlainFixedLenByteArrayDecoder, ByteStreamSplitFixedLenByteArrayDecoder   fixed_len_byte_array_decoder.go
//   validateByteStreamSplitPageData, ByteStreamSplitDecoder[T]   byte_stream_split.go:98-250
//   accepted encodings per physical type                         typed_encoder.go:250-291,432-437,538-552,714-727
//
// Every call runs the passes of pq_decode.cuh first: pq_tile_count_kernel (spaced), then pq_runs_kernel, one block per
// page, which scans the spaced rank bases, walks the runs of level, dictionary and RLE pages and checks the pages of
// the pass-1 kinds this file adds (kBss, kBoolPlain, kBoolRle).  What runs after it:
//   - levels: pq_expand_kernel<kLevels> into int16.
//   - PLAIN and dictionary pages of 4- and 8-byte values: pq_expand_kernel<kPlain / kDict>, for
//     ag_parquet_plain_decode_spaced and ag_parquet_dict_decode as for the fixed_decode pages of those widths.
//   - BYTE_STREAM_SPLIT pages of 4- and 8-byte values: pq_expand_kernel<kBss>, one thread per slot assembling its value
//     in a register from one byte of each stream; consecutive threads read consecutive bytes of every stream and store
//     consecutive values.
//   - other widths, and BYTE_STREAM_SPLIT of other widths: the source of a slot is its dense rank (dense: the slot
//     itself; spaced: pq_expand_kernel<kRank>) or its dictionary index (pq_expand_kernel<kIndex>), one int32 per slot.
//     fx_copy_kernel then writes the output in aligned 16-byte pieces, consecutive threads on consecutive pieces, each
//     piece assembled byte by byte from its sources (PLAIN: data[rank * width + j], dictionary: dict[index * width + j],
//     BYTE_STREAM_SPLIT: data[j * stride + rank]).  A piece at either end of a tile is stored byte by byte, so no
//     byte outside the slots a page decoded is written.
//   - booleans: fx_bool_kernel, one block per 1024-slot tile.  Each thread finds its slot's value bit (PLAIN: bit
//     `rank` of the page; RLE: the run holding `rank`, found by find_run), a ballot per warp packs 32 slots into
//     shared memory, and one thread per aligned 32-bit output word stores it.  A word shared with a neighbouring tile
//     or page, or with slots the call does not write, is merged with atomicAnd / atomicOr.
#include <string.h>

#include <algorithm>
#include <vector>

#include "pq_decode.cuh"

namespace ag {

namespace {

constexpr int kCopyChunk = 16384;   // output bytes per fx_copy_kernel block and step

enum FxSrc { kSrcPlain = 0, kSrcDict = 1, kSrcBss = 2 };

// what runs after pass 1
enum FxJob { kJobPlainT = 0, kJobDictT = 1, kJobPlainW = 2, kJobDictW = 3, kJobBss = 4, kJobBoolPlain = 5, kJobBoolRle = 6, kJobBssT = 7, kJobLevels = 8 };

struct FxArgs {
  PqPlan plan;
  const PageState* st;
  const uint8_t* data;
  const uint8_t* valid;     // NULL = every slot valid
  const int32_t* map;       // per slot: dense rank or dictionary index; NULL = the slot itself
  const uint8_t* dict;
  int64_t dict_len;
  int64_t width;
  uint8_t* out;
};

// grid (tiles, chunks): block (t, y) writes the output bytes [t0 + y * kCopyChunk, ...) of tile t, stepping by
// gridDim.y chunks
template <int SRC>
__global__ void __launch_bounds__(kRleThreads)
fx_copy_kernel(FxArgs a) {
  const int64_t tile = blockIdx.x;
  const int64_t p = find_page(a.plan.tile_base, a.plan.n_pages, tile);
  const ag_pq_page pg = a.plan.pages[p];
  const PageState ps = a.st[p];
  const int64_t s0 = (tile - a.plan.tile_base[p]) * kTile;
  const int64_t s1 = min(s0 + (int64_t)kTile, ps.slots);
  if (s0 >= s1) return;                                          // block-uniform
  const int64_t w = a.width;
  const int64_t t0 = (pg.out + s0) * w, t1 = (pg.out + s1) * w;   // the tile's output bytes
  const uint8_t* src_base = SRC == kSrcDict ? a.dict : a.data + ps.stream;
  const int64_t step = SRC == kSrcBss ? ps.stream_len / w : 1;   // source distance of bytes j and j + 1 of a value
  // source offset of byte 0 of slot s's value, or -1 for a slot that holds zeros
  auto source = [&](int64_t s) -> int64_t {
    if (a.valid && !bit_is_set(a.valid, pg.out + s)) return -1;
    const int64_t r = a.map ? (int64_t)a.map[pg.out + s] : s;
    if (SRC == kSrcDict) return (r >= 0 && r < a.dict_len) ? r * w : -1;
    return SRC == kSrcBss ? r : r * w;
  };
  const uintptr_t ob = reinterpret_cast<uintptr_t>(a.out);
  for (int64_t lo = t0 + (int64_t)blockIdx.y * kCopyChunk; lo < t1; lo += (int64_t)gridDim.y * kCopyChunk) {
    const int64_t hi = min(lo + (int64_t)kCopyChunk, t1);
    const int64_t first = (int64_t)(((ob + lo) & ~(uintptr_t)15) - ob);   // first aligned piece touching [lo, hi)
    for (int64_t q0 = first + (int64_t)threadIdx.x * 16; q0 < hi; q0 += (int64_t)kRleThreads * 16) {
      const int64_t b0 = q0 > lo ? q0 : lo;
      const int64_t rel = b0 - t0;
      int64_t s = s0 + rel / w;
      int64_t j = rel - (s - s0) * w;
      int64_t src = source(s);
      uint32_t v[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const int64_t o = q0 + k;
        if (o >= b0 && o < hi) {
          if (src >= 0) v[k >> 2] |= (uint32_t)__ldg(src_base + src + j * step) << (8 * (k & 3));
          if (++j == w) {
            j = 0;
            ++s;
            if (o + 1 < hi) src = source(s);
          }
        }
      }
      if (q0 >= lo && q0 + 16 <= hi) {
        *reinterpret_cast<uint4*>(a.out + q0) = make_uint4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          const int64_t o = q0 + k;
          if (o >= lo && o < hi) a.out[o] = (uint8_t)(v[k >> 2] >> (8 * (k & 3)));
        }
      }
    }
  }
}

// one block per tile of 1024 slots of one page; a.out is the output bitmap
template <bool RLE, bool SPACED>
__global__ void __launch_bounds__(kRleThreads)
fx_bool_kernel(PqArgs a) {
  __shared__ int warp_tot[kRleThreads / 32];
  __shared__ uint32_t tbits[kTile / 32];                         // bit i = value of the tile's slot i
  const int64_t tile = blockIdx.x;
  const int2 ti = a.tile_info[tile];
  const int64_t p = ti.x;
  const ag_pq_page pg = a.plan.pages[p];
  const PageState ps = a.st[p];
  const int64_t s0 = (tile - a.plan.tile_base[p]) * kTile;
  const int64_t limit = ps.slots;
  if (s0 >= limit) return;                                       // block-uniform
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const uint2* runs = a.runs + (RLE ? a.plan.run_base[p] : 0);
  const uint8_t* stream = a.data + ps.stream;
  const int64_t rhi = tile_last_run(a, tile, ti, ps.nruns);

  int64_t rank_base = SPACED ? a.tile_cnt[tile] : s0;
#pragma unroll
  for (int q = 0; q < kTile / kRleThreads; ++q) {
    const int64_t s = s0 + q * kRleThreads + tid;
    bool v = s < limit;
    int64_t rank = s;
    if (SPACED) rank = spaced_rank(s < limit, a.valid, pg.out + s, warp_tot, rank_base, v);
    bool bit = false;
    if (v) {
      if (!RLE) {
        bit = (__ldg(stream + (rank >> 3)) >> (rank & 7)) & 1;
      } else {
        const uint2 r = find_run(runs, ti.y, rhi, rank);
        // a repeated value is true when any bit of its byte is set (rle.go:161-165 keeps the whole byte)
        bit = (r.x & kLiteralFlag) ? unpack_at(stream + r.y, rank - (int64_t)(r.x & ~kLiteralFlag), 1) != 0u : r.y != 0u;
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, bit);
    if (lane == 0) tbits[q * (kRleThreads / 32) + wid] = m;
  }
  __syncthreads();

  // output words: absolute bits [b0, b1) of the word-aligned base
  const int64_t s1 = min(s0 + (int64_t)kTile, limit);
  const uintptr_t ob = reinterpret_cast<uintptr_t>(a.out);
  uint32_t* words = reinterpret_cast<uint32_t*>(ob & ~(uintptr_t)3);
  const int64_t b0 = (int64_t)(ob & 3) * 8 + pg.out + s0, b1 = b0 + (s1 - s0);
  const int64_t w0 = b0 >> 5, nw = ((b1 - 1) >> 5) - w0 + 1;
  auto tw = [&](int64_t k) -> uint32_t { return (k >= 0 && k < kTile / 32) ? tbits[k] : 0u; };
  for (int64_t i = tid; i < nw; i += kRleThreads) {
    const int64_t wb = (w0 + i) * 32;                            // absolute bit of the word's bit 0
    const int64_t rel = wb - b0;                                 // tile slot at the word's bit 0 (>= -31)
    const uint32_t val = rel >= 0 ? __funnelshift_r(tw(rel >> 5), tw((rel >> 5) + 1), (int)(rel & 31)) : tw(0) << (int)(-rel);
    uint32_t mask = 0xffffffffu;
    if (wb < b0) mask &= 0xffffffffu << (int)(b0 - wb);
    if (wb + 32 > b1) mask &= 0xffffffffu >> (int)(wb + 32 - b1);
    if (mask == 0xffffffffu) {
      words[w0 + i] = val;
    } else {
      atomicAnd(words + w0 + i, ~mask);
      atomicOr(words + w0 + i, val & mask);
    }
  }
}

int pass1_kind(int job) {
  switch (job) {
    case kJobPlainT: case kJobPlainW: return kPlain;
    case kJobDictT: return kDict;
    case kJobDictW: return kIndex;
    case kJobBss: case kJobBssT: return kBss;
    case kJobBoolPlain: return kBoolPlain;
    case kJobLevels: return kLevels;
    default: return kBoolRle;
  }
}

void fx_err_text(const PageState& s, const ag_pq_page& pg, int ptype, int width, char* buf, size_t n) {
  switch (s.err) {
    case kErrPlainShort:
      if (ptype == AG_PQ_TYPE_INT96)
        snprintf(buf, n, "parquet: eof exception decode plain INT96, nvals: %lld, nbytes: %lld, datalen: %lld", (long long)s.need,
                 (long long)s.need * 12, (long long)pg.len);
      else if (ptype == AG_PQ_TYPE_FIXED_LEN_BYTE_ARRAY) snprintf(buf, n, "parquet: eof exception");
      else snprintf(buf, n, "%s", err_text(s.err));
      break;
    case kErrBssSize:
      snprintf(buf, n, "data size (%lld) is too small for the number of values in in BYTE_STREAM_SPLIT (%lld)", (long long)pg.len,
               (long long)pg.num_values);
      break;
    case kErrBssAlign:
      if (ptype == AG_PQ_TYPE_FIXED_LEN_BYTE_ARRAY)
        snprintf(buf, n, "ByteStreamSplit data size %lld not aligned with type FIXED_LEN_BYTE_ARRAY and byte_width: %d", (long long)pg.len, width);
      else snprintf(buf, n, "ByteStreamSplit data size %lld not aligned with byte_width: %d", (long long)pg.len, width);
      break;
    case kErrBssEof: snprintf(buf, n, "parquet: eof exception"); break;
    case kErrBssShort: snprintf(buf, n, "parquet: number of values / definitions levels read did not match"); break;
    case kErrBoolShort:
      snprintf(buf, n, "parquet: boolean data has %lld bits available, need %lld: unexpected EOF", (long long)pg.len * 8, (long long)s.need);
      break;
    case kErrBoolLength: snprintf(buf, n, "invalid length - %lld (corrupt data page?)", (long long)pg.len); break;
    case kErrBoolBytes: snprintf(buf, n, "received invalid number of bytes - %u (corrupt data page?)", (unsigned)s.pad); break;
    case kErrBoolEof: snprintf(buf, n, "unexpected EOF"); break;
    default: snprintf(buf, n, "%s", err_text(s.err)); break;
  }
}

// pq_expand_kernel<K> over the call's 4- or 8-byte values
template <int K>
ag_status expand_wide(const PqArgs& a, bool spaced, cudaStream_t st) {
  if (a.width == 4) return spaced ? launch_expand<K, uint32_t, true>(a, st) : launch_expand<K, uint32_t, false>(a, st);
  return spaced ? launch_expand<K, unsigned long long, true>(a, st) : launch_expand<K, unsigned long long, false>(a, st);
}

// The device work of every entry point of this file.  `c.pages` is host memory; everything else device memory on
// `st`.  Synchronises `st` once.  h_decoded (host, may be NULL) receives the per-page decoded counts.
ag_status fx_pages_dev(const PqCall& c, int64_t* d_decoded, int64_t* h_decoded, int64_t* d_bad_pos, cudaStream_t st) {
  const char* fn = c.fn;
  const int kind = pass1_kind(c.job);
  const bool has_runs = kind == kLevels || kind == kDict || kind == kIndex || kind == kBoolRle;
  PagePlan plan;
  AG_TRY(plan_pages(fn, c.pages, c.n_pages, [&](const ag_pq_page& g) { return has_runs ? std::min(g.num_values, g.len) : (int64_t)0; }, &plan));
  if (c.n_pages == 0) {
    // no index is looked at: *d_bad_pos is still overwritten
    if (!d_bad_pos) return AG_OK;
    static const int64_t kNone = AG_NO_ERROR_POS;
    AG_TRY(h2d(d_bad_pos, &kNone, 8, st));
    return sync(st);
  }
  const int64_t n_tiles = plan.n_tiles;
  const bool dict = c.job == kJobDictT || c.job == kJobDictW;
  // jobs whose expansion stores whole 2-, 4- or 8-byte elements
  const bool typed = c.job == kJobLevels || c.job == kJobPlainT || c.job == kJobDictT || c.job == kJobBssT;
  if (n_tiles > 0 && !c.out) AG_FAIL(AG_ERR_INVALID, "%s: NULL output", fn);
  if (plan.any_data && !c.data) AG_FAIL(AG_ERR_INVALID, "%s: NULL page data", fn);
  if (c.dict_len > 0 && !c.dict) AG_FAIL(AG_ERR_INVALID, "%s: NULL dictionary", fn);
  if (c.job == kJobDictT && c.dict && (reinterpret_cast<uintptr_t>(c.dict) & (c.width - 1)))
    AG_FAIL(AG_ERR_INVALID, "%s: dictionary not aligned to its value width", fn);
  if (typed && c.out && (reinterpret_cast<uintptr_t>(c.out) & (c.width - 1)))
    AG_FAIL(AG_ERR_INVALID, "%s: output not aligned to its element width", fn);
  const bool mapped = c.job == kJobDictW || ((c.job == kJobPlainW || c.job == kJobBss) && c.valid);

  Carve sc;
  const size_t o_plan = sc.take(plan.bytes.size());
  const size_t o_st = sc.take((size_t)c.n_pages * sizeof(PageState));
  const size_t o_tc = sc.take(c.valid ? (size_t)n_tiles * 8 : 0);
  const size_t o_ti = sc.take((size_t)n_tiles * 8);
  const size_t o_bad = sc.take(8);
  const size_t o_runs = sc.take((size_t)plan.n_desc * 8);
  const size_t o_map = sc.take(mapped ? (size_t)plan.slot_end * 4 : 0);
  // this call synchronises `st` anyway, so its device scratch may live in a Temps
  Temps t(st);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, sc.size));
  int32_t* map = mapped ? reinterpret_cast<int32_t*>(d + o_map) : nullptr;
  PqArgs a{};
  AG_TRY(upload_plan(plan, d + o_plan, st, &a.plan));
  a.data = c.data;
  a.valid = c.valid;
  a.st = reinterpret_cast<PageState*>(d + o_st);
  a.tile_cnt = c.valid ? reinterpret_cast<int64_t*>(d + o_tc) : nullptr;
  a.tile_info = reinterpret_cast<int2*>(d + o_ti);
  a.bad = reinterpret_cast<unsigned long long*>(d_bad_pos ? (void*)d_bad_pos : (void*)(d + o_bad));
  a.runs = plan.n_desc ? reinterpret_cast<uint2*>(d + o_runs) : nullptr;
  a.d_decoded = d_decoded;
  a.kind = kind; a.fixed_bw = c.fixed_bw; a.v1 = c.v1; a.width = c.width;
  a.dict_len = c.dict_len; a.dict = c.dict; a.out = mapped ? (void*)map : c.out;
  AG_TRY(launch_tile_counts(a.plan, c.valid, a.tile_cnt, st));
  pq_runs_kernel<<<(unsigned)c.n_pages, kRleThreads, 0, st>>>(a);
  AG_TRY(check_launch("pq_runs_kernel"));
  const bool sp = c.valid != nullptr;
  switch (c.job) {
    case kJobLevels: AG_TRY((launch_expand<kLevels, int16_t, false>(a, st))); break;
    case kJobPlainT: AG_TRY(expand_wide<kPlain>(a, sp, st)); break;
    case kJobDictT: AG_TRY(expand_wide<kDict>(a, sp, st)); break;
    case kJobBssT: AG_TRY(expand_wide<kBss>(a, sp, st)); break;
    case kJobPlainW: case kJobDictW: case kJobBss: {
      if (c.job == kJobDictW) AG_TRY((sp ? launch_expand<kIndex, int32_t, true>(a, st) : launch_expand<kIndex, int32_t, false>(a, st)));
      else if (mapped) AG_TRY((launch_expand<kRank, int32_t, true>(a, st)));
      if (n_tiles == 0) break;
      FxArgs f;
      f.plan = a.plan; f.st = a.st; f.data = c.data; f.valid = c.valid; f.map = map;
      f.dict = static_cast<const uint8_t*>(c.dict); f.dict_len = c.dict_len; f.width = c.width;
      f.out = static_cast<uint8_t*>(c.out);
      const int64_t chunks = std::min<int64_t>(((int64_t)kTile * c.width + kCopyChunk - 1) / kCopyChunk, 65535);
      const dim3 grid((unsigned)n_tiles, (unsigned)chunks);
      if (c.job == kJobPlainW) fx_copy_kernel<kSrcPlain><<<grid, kRleThreads, 0, st>>>(f);
      else if (c.job == kJobDictW) fx_copy_kernel<kSrcDict><<<grid, kRleThreads, 0, st>>>(f);
      else fx_copy_kernel<kSrcBss><<<grid, kRleThreads, 0, st>>>(f);
      AG_TRY(check_launch("fx_copy_kernel"));
      break;
    }
    default:
      if (n_tiles == 0) break;
      if (c.job == kJobBoolPlain) {
        if (sp) fx_bool_kernel<false, true><<<(unsigned)n_tiles, kRleThreads, 0, st>>>(a);
        else fx_bool_kernel<false, false><<<(unsigned)n_tiles, kRleThreads, 0, st>>>(a);
      } else {
        if (sp) fx_bool_kernel<true, true><<<(unsigned)n_tiles, kRleThreads, 0, st>>>(a);
        else fx_bool_kernel<true, false><<<(unsigned)n_tiles, kRleThreads, 0, st>>>(a);
      }
      AG_TRY(check_launch("fx_bool_kernel"));
      break;
  }
  return read_back(fn, a.st, c.n_pages, dict ? a.bad : nullptr, h_decoded, st,
                   [&](int64_t i, const PageState& s, char* buf, size_t n) { fx_err_text(s, c.pages[i], c.ptype, c.width, buf, n); });
}

// ---- argument checks of the entry points, each giving the call's PqCall ----
int bit_len(int v) { int n = 0; while (v) { ++n; v >>= 1; } return n; }

ag_status levels_args(int max_level, int encoding, PqCall* c) {
  if (encoding == AG_PQ_LEVELS_BIT_PACKED) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "levels_decode: deprecated BIT_PACKED levels are not implemented");
  if (encoding != AG_PQ_LEVELS_V1_RLE && encoding != AG_PQ_LEVELS_V2_RLE) AG_FAIL(AG_ERR_INVALID, "levels_decode: unknown level encoding %d", encoding);
  if (max_level < 0 || max_level > 0xffff) AG_FAIL(AG_ERR_INVALID, "levels_decode: max_level must be 0..65535 (bit width 0..16)");
  *c = PqCall{};
  c->fn = "levels_decode"; c->job = kJobLevels; c->width = 2; c->fixed_bw = bit_len(max_level); c->v1 = encoding == AG_PQ_LEVELS_V1_RLE;
  return AG_OK;
}

// dict_decode (kJobDictT) and plain_decode_spaced (kJobPlainT): 4- or 8-byte values
ag_status wide_args(const char* fn, int job, int value_width, int64_t dict_len, PqCall* c) {
  if (value_width != 4 && value_width != 8) AG_FAIL(AG_ERR_INVALID, "%s: value_width must be 4 or 8", fn);
  if (job == kJobDictT && dict_len < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative dictionary length", fn);
  *c = PqCall{};
  c->fn = fn; c->job = job; c->width = value_width; c->dict_len = job == kJobDictT ? dict_len : 0;
  return AG_OK;
}

ag_status fixed_args(int ptype, int type_length, int encoding, int64_t dict_len, PqCall* c) {
  const char* fn = "fixed_decode";
  int w;
  switch (ptype) {
    case AG_PQ_TYPE_INT32: case AG_PQ_TYPE_FLOAT: w = 4; break;
    case AG_PQ_TYPE_INT64: case AG_PQ_TYPE_DOUBLE: w = 8; break;
    case AG_PQ_TYPE_INT96: w = 12; break;
    case AG_PQ_TYPE_FIXED_LEN_BYTE_ARRAY:
      if (type_length < 1) AG_FAIL(AG_ERR_INVALID, "%s: FIXED_LEN_BYTE_ARRAY type_length must be >= 1, got %d", fn, type_length);
      w = type_length;
      break;
    default: AG_FAIL(AG_ERR_INVALID, "%s: physical type %d is not INT32, INT64, INT96, FLOAT, DOUBLE or FIXED_LEN_BYTE_ARRAY", fn, ptype);
  }
  const bool wide = w == 4 || w == 8;
  int job;
  if (encoding == AG_PQ_ENC_PLAIN) job = wide ? kJobPlainT : kJobPlainW;
  else if (encoding == AG_PQ_ENC_PLAIN_DICTIONARY || encoding == AG_PQ_ENC_RLE_DICTIONARY) job = wide ? kJobDictT : kJobDictW;
  else if (encoding == AG_PQ_ENC_BYTE_STREAM_SPLIT && ptype != AG_PQ_TYPE_INT96) job = wide ? kJobBssT : kJobBss;
  else AG_FAIL(AG_ERR_INVALID, "%s: encoding %d is not accepted for physical type %d", fn, encoding, ptype);
  const bool dict = job == kJobDictT || job == kJobDictW;
  if (dict && dict_len < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative dictionary length", fn);
  *c = PqCall{};
  c->fn = fn; c->job = job; c->ptype = ptype; c->width = w; c->dict_len = dict ? dict_len : 0;
  return AG_OK;
}

ag_status bool_args(int encoding, PqCall* c) {
  if (encoding != AG_PQ_ENC_PLAIN && encoding != AG_PQ_ENC_RLE)
    AG_FAIL(AG_ERR_INVALID, "bool_decode: encoding %d is not accepted for BOOLEAN (PLAIN or RLE)", encoding);
  *c = PqCall{};
  c->fn = "bool_decode"; c->job = encoding == AG_PQ_ENC_PLAIN ? kJobBoolPlain : kJobBoolRle; c->width = 1; c->bitmap = true;
  c->fixed_bw = encoding == AG_PQ_ENC_RLE ? 1 : 0;
  return AG_OK;
}


}  // namespace

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_parquet_levels_decode_dev(int max_level, int encoding, const uint8_t* d_data, const ag_pq_page* pages, int64_t n_pages,
                                       int16_t* d_out, int64_t* d_decoded, ag_stream_t s) {
  AG_TRY(ensure_init());
  PqCall c;
  AG_TRY(levels_args(max_level, encoding, &c));
  c.data = d_data; c.pages = pages; c.n_pages = n_pages; c.out = d_out;
  return fx_pages_dev(c, d_decoded, nullptr, nullptr, resolve_stream(s));
}

ag_status ag_parquet_levels_decode(int max_level, int encoding, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages,
                                   int16_t* out, int64_t* decoded) {
  AG_TRY(ensure_init());
  PqCall c;
  AG_TRY(levels_args(max_level, encoding, &c));
  c.data = data; c.pages = pages; c.n_pages = n_pages; c.out = out;
  return pq_pages_host(fx_pages_dev, c, decoded, nullptr);
}

ag_status ag_parquet_dict_decode_dev(int value_width, const void* d_dict, int64_t dict_len, const uint8_t* d_data, const ag_pq_page* pages,
                                     int64_t n_pages, const uint8_t* d_valid, void* d_out, int64_t* d_decoded, int64_t* d_bad_pos, ag_stream_t s) {
  AG_TRY(ensure_init());
  PqCall c;
  AG_TRY(wide_args("dict_decode", kJobDictT, value_width, dict_len, &c));
  c.data = d_data; c.pages = pages; c.n_pages = n_pages; c.valid = d_valid; c.dict = d_dict; c.out = d_out;
  return fx_pages_dev(c, d_decoded, nullptr, d_bad_pos, resolve_stream(s));
}

ag_status ag_parquet_dict_decode(int value_width, const void* dict, int64_t dict_len, const uint8_t* data, const ag_pq_page* pages,
                                 int64_t n_pages, const uint8_t* valid, void* out, int64_t* decoded, int64_t* bad_pos) {
  AG_TRY(ensure_init());
  if (bad_pos) *bad_pos = AG_NO_ERROR_POS;
  PqCall c;
  AG_TRY(wide_args("dict_decode", kJobDictT, value_width, dict_len, &c));
  c.data = data; c.pages = pages; c.n_pages = n_pages; c.valid = valid; c.dict = dict; c.out = out;
  return pq_pages_host(fx_pages_dev, c, decoded, bad_pos);
}

ag_status ag_parquet_plain_decode_spaced_dev(int value_width, const uint8_t* d_data, const ag_pq_page* pages, int64_t n_pages,
                                             const uint8_t* d_valid, void* d_out, ag_stream_t s) {
  AG_TRY(ensure_init());
  PqCall c;
  AG_TRY(wide_args("plain_decode_spaced", kJobPlainT, value_width, 0, &c));
  c.data = d_data; c.pages = pages; c.n_pages = n_pages; c.valid = d_valid; c.out = d_out;
  return fx_pages_dev(c, nullptr, nullptr, nullptr, resolve_stream(s));
}

ag_status ag_parquet_plain_decode_spaced(int value_width, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages,
                                         const uint8_t* valid, void* out) {
  AG_TRY(ensure_init());
  PqCall c;
  AG_TRY(wide_args("plain_decode_spaced", kJobPlainT, value_width, 0, &c));
  c.data = data; c.pages = pages; c.n_pages = n_pages; c.valid = valid; c.out = out;
  return pq_pages_host(fx_pages_dev, c, nullptr, nullptr);
}

ag_status ag_parquet_bool_decode_dev(int encoding, const uint8_t* d_data, const ag_pq_page* pages, int64_t n_pages, const uint8_t* d_valid,
                                     uint8_t* d_out_bits, int64_t* d_decoded, ag_stream_t s) {
  AG_TRY(ensure_init());
  PqCall c;
  AG_TRY(bool_args(encoding, &c));
  c.data = d_data; c.pages = pages; c.n_pages = n_pages; c.valid = d_valid; c.out = d_out_bits;
  return fx_pages_dev(c, d_decoded, nullptr, nullptr, resolve_stream(s));
}

ag_status ag_parquet_bool_decode(int encoding, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages, const uint8_t* valid,
                                 uint8_t* out_bits, int64_t* decoded) {
  AG_TRY(ensure_init());
  PqCall c;
  AG_TRY(bool_args(encoding, &c));
  c.data = data; c.pages = pages; c.n_pages = n_pages; c.valid = valid; c.out = out_bits;
  return pq_pages_host(fx_pages_dev, c, decoded, nullptr);
}

ag_status ag_parquet_fixed_decode_dev(int physical_type, int type_length, int encoding, const uint8_t* d_data, const ag_pq_page* pages,
                                      int64_t n_pages, const uint8_t* d_valid, const void* d_dict, int64_t dict_len, void* d_out,
                                      int64_t* d_decoded, int64_t* d_bad_pos, ag_stream_t s) {
  AG_TRY(ensure_init());
  PqCall c;
  AG_TRY(fixed_args(physical_type, type_length, encoding, dict_len, &c));
  c.data = d_data; c.pages = pages; c.n_pages = n_pages; c.valid = d_valid; c.dict = d_dict; c.out = d_out;
  return fx_pages_dev(c, d_decoded, nullptr, d_bad_pos, resolve_stream(s));
}

ag_status ag_parquet_fixed_decode(int physical_type, int type_length, int encoding, const uint8_t* data, const ag_pq_page* pages,
                                  int64_t n_pages, const uint8_t* valid, const void* dict, int64_t dict_len, void* out, int64_t* decoded,
                                  int64_t* bad_pos) {
  AG_TRY(ensure_init());
  if (bad_pos) *bad_pos = AG_NO_ERROR_POS;
  PqCall c;
  AG_TRY(fixed_args(physical_type, type_length, encoding, dict_len, &c));
  c.data = data; c.pages = pages; c.n_pages = n_pages; c.valid = valid; c.dict = dict; c.out = out;
  return pq_pages_host(fx_pages_dev, c, decoded, bad_pos);
}

}  // extern "C"
