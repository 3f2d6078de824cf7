// rle.cu — DELTA_BINARY_PACKED INT32 / INT64 Parquet pages on the device (deltaBitPackDecoder,
// parquet/internal/encoding/delta_bit_packing.go:72-316).  The RLE/bit-packed decoders (levels, dictionary indices)
// and the PLAIN spaced decoder run through fixed.cu's driver.
//
// The delta passes reuse pq_decode.cuh's tile counts, window and tile layout: delta_walk_kernel (one block per page)
// parses the header and walks the block chain into one 16-byte descriptor per miniblock the page needs;
// delta_values_kernel sums each tile's deltas, tile_sum_scan_kernel scans the sums per page, and delta_values_kernel
// unpacks again, block-scans and writes.  Every value is the first value plus a prefix sum of the deltas, modulo the
// physical width.
#include "pq_decode.cuh"

namespace ag {

// DELTA_BINARY_PACKED pages.  `c.pages` is host memory; everything else is device memory on `st`.  Synchronises `st`
// once to read the per-page error codes back; h_decoded (host, may be NULL) receives the per-page decoded counts.
// Launches: tile counts (spaced), the block walk, the tile sums, the per-page scan of the tile sums, and the
// unpack-scan-write pass.
static ag_status delta_pages_dev(const PqCall& c, int64_t* d_decoded, int64_t* h_decoded, int64_t*, cudaStream_t st) {
  const char* fn = c.fn;
  PagePlan plan;   // descriptors: miniblocks, each holding >= 32 deltas
  AG_TRY(plan_pages(fn, c.pages, c.n_pages, [](const ag_pq_page& g) { return (g.num_values + 31) / 32; }, &plan));
  if (c.n_pages == 0) return AG_OK;
  const int64_t n_tiles = plan.n_tiles;
  if (n_tiles > 0 && !c.out) AG_FAIL(AG_ERR_INVALID, "%s: NULL output", fn);
  if (plan.any_data && !c.data) AG_FAIL(AG_ERR_INVALID, "%s: NULL page data", fn);
  if (c.out && (reinterpret_cast<uintptr_t>(c.out) & (c.width - 1))) AG_FAIL(AG_ERR_INVALID, "%s: output not aligned to its element width", fn);

  Carve sc;
  const size_t o_plan = sc.take(plan.bytes.size());
  const size_t o_st = sc.take((size_t)c.n_pages * sizeof(DeltaPage));
  const size_t o_tc = sc.take(c.valid ? (size_t)n_tiles * 8 : 0);
  const size_t o_ts = sc.take((size_t)n_tiles * 8);
  const size_t o_mb = sc.take((size_t)plan.n_desc * sizeof(DeltaMini));
  // this call synchronises `st` anyway, so its device scratch may live in a Temps
  Temps t(st);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, sc.size));
  PqPlan pl;
  AG_TRY(upload_plan(plan, d + o_plan, st, &pl));
  DeltaArgs a;
  a.pages = pl.pages;
  a.mb_base = pl.run_base;
  a.tile_base = pl.tile_base;
  a.n_pages = c.n_pages;
  a.data = c.data;
  a.skip = nullptr;
  a.valid = c.valid;
  a.st = reinterpret_cast<DeltaPage*>(d + o_st);
  a.mb = reinterpret_cast<DeltaMini*>(d + o_mb);
  a.tile_cnt = c.valid ? reinterpret_cast<int64_t*>(d + o_tc) : nullptr;
  a.tile_sum = reinterpret_cast<unsigned long long*>(d + o_ts);
  a.d_decoded = d_decoded;
  a.width = c.width;
  a.out = c.out;
  AG_TRY(launch_tile_counts(pl, c.valid, a.tile_cnt, st));
  delta_walk_kernel<<<(unsigned)c.n_pages, kRleThreads, 0, st>>>(a);
  AG_TRY(check_launch("delta_walk_kernel"));
  if (n_tiles) {
    AG_TRY(visit_width(8 * c.width, [&](auto tag) -> ag_status {
      using T = typename decltype(tag)::type;
      if constexpr (sizeof(T) >= 4) return c.valid ? launch_delta_values<T, true>(a, n_tiles, st) : launch_delta_values<T, false>(a, n_tiles, st);
      else AG_FAIL(AG_ERR_INVALID, "%s: value_width must be 4 or 8", fn);
    }, [&] { AG_FAIL(AG_ERR_INVALID, "%s: value_width must be 4 or 8", fn); }));
  }
  return read_back(fn, a.st, c.n_pages, nullptr, h_decoded, st,
                   [](int64_t, const DeltaPage& s, char* buf, size_t n) { delta_err_text(s, buf, n); });
}

static ag_status delta_args(int value_width, PqCall* c) {
  if (value_width != 4 && value_width != 8) AG_FAIL(AG_ERR_INVALID, "delta_decode: value_width must be 4 (INT32) or 8 (INT64)");
  *c = PqCall{};
  c->fn = "delta_decode"; c->width = value_width;
  return AG_OK;
}

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_parquet_delta_decode_dev(int value_width, const uint8_t* d_data, const ag_pq_page* pages, int64_t n_pages,
                                      const uint8_t* d_valid, void* d_out, int64_t* d_decoded, ag_stream_t s) {
  AG_TRY(ensure_init());
  PqCall c;
  AG_TRY(delta_args(value_width, &c));
  c.data = d_data; c.pages = pages; c.n_pages = n_pages; c.valid = d_valid; c.out = d_out;
  return delta_pages_dev(c, d_decoded, nullptr, nullptr, resolve_stream(s));
}

ag_status ag_parquet_delta_decode(int value_width, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages,
                                  const uint8_t* valid, void* out, int64_t* decoded) {
  AG_TRY(ensure_init());
  PqCall c;
  AG_TRY(delta_args(value_width, &c));
  c.data = data; c.pages = pages; c.n_pages = n_pages; c.valid = valid; c.out = out;
  return pq_pages_host(delta_pages_dev, c, decoded, nullptr);
}

}  // extern "C"
