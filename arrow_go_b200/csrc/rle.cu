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

#include "pq_decode.cuh"

namespace ag {

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
  a.skip = nullptr;
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
