// lz_exec.cuh — what the Parquet page decompressors (snappy.cu, zstd.cu, gzip.cu, lz4.cu) share.  Internal, not part of
// the ABI.
//
//   pq_dst_overlap_check  overlapping dst ranges of an ag_pq_compressed batch (the SNAPPY compressor checks it too)
//   pq_compressed_check   the argument checks of an ag_pq_compressed batch, AG_ERR_INVALID before any launch
//   pq_decompress_dev     the device flavour: the checks, then the codec
//   pq_decompress_host    the host flavour: the checks, stage src, run the codec, copy back only written bytes
//   lz_plan / lz_upload   the page table and the codec's per-page bounds as prefix arrays, in one upload
//   lz_exec_launch        the executor (lz_exec.cu): a page's output from element descriptors {first output byte,
//                         literal source / copy offset, kind}
//   lz_read_back          the end of a call: per-page states back, one synchronisation, the lowest failing page
#pragma once

#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <vector>

#include "host_stage.cuh"

namespace ag {

// AG_ERR_INVALID naming the two lowest pages whose [dst, dst + dst_len) ranges overlap (empty ranges overlap nothing).
// Shared with the compressor (snappy_encode.cu), where dst_len is the capacity.
static inline ag_status pq_dst_overlap_check(const char* fn, const ag_pq_compressed* pages, int64_t n_pages) {
  std::vector<int64_t> order;
  for (int64_t i = 0; i < n_pages; ++i)
    if (pages[i].dst_len > 0) order.push_back(i);
  std::sort(order.begin(), order.end(), [&](int64_t x, int64_t y) { return pages[x].dst < pages[y].dst || (pages[x].dst == pages[y].dst && x < y); });
  for (size_t k = 1; k < order.size(); ++k) {
    const ag_pq_compressed &u = pages[order[k - 1]], &v = pages[order[k]];
    if (v.dst < u.dst + u.dst_len) {
      const int64_t x = std::min(order[k - 1], order[k]), y = std::max(order[k - 1], order[k]);
      AG_FAIL(AG_ERR_INVALID, "%s: pages %lld and %lld: overlapping dst ranges", fn, (long long)x, (long long)y);
    }
  }
  return AG_OK;
}

// Argument checks shared by every codec and both flavours; every one is AG_ERR_INVALID before any launch.  `src` and
// `dst` are the compressed data and the output, in host or device memory; only whether they are NULL matters.
// *src_end / *dst_end: the bytes of `src` / `dst` the batch spans.
static inline ag_status pq_compressed_check(const char* fn, const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages,
                                            const uint8_t* dst, int64_t* src_end, int64_t* dst_end) {
  *src_end = *dst_end = 0;
  if (n_pages < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative page count", fn);
  if (n_pages == 0) return AG_OK;
  if (!pages) AG_FAIL(AG_ERR_INVALID, "%s: NULL page table", fn);
  for (int64_t i = 0; i < n_pages; ++i) {
    const ag_pq_compressed& g = pages[i];
    if (g.src < 0 || g.src_len < 0 || g.dst < 0 || g.dst_len < 0 || g.src_len > 0xffffffffLL || g.dst_len > 0xffffffffLL)
      AG_FAIL(AG_ERR_INVALID, "%s: page %lld: negative field or more than 2^32-1 bytes", fn, (long long)i);
    *src_end = std::max(*src_end, g.src + g.src_len);
    *dst_end = std::max(*dst_end, g.dst + g.dst_len);
  }
  AG_TRY(pq_dst_overlap_check(fn, pages, n_pages));
  if (*src_end > 0 && !src) AG_FAIL(AG_ERR_INVALID, "%s: NULL compressed data", fn);
  if (*dst_end > 0 && !dst) AG_FAIL(AG_ERR_INVALID, "%s: NULL output", fn);
  return AG_OK;
}

// A codec: decompresses a checked, non-empty batch into device `dst`.  `pages` is host memory; everything else is
// device memory on `st`.  Fills h_written (host, may be NULL) with the bytes per page and synchronises `st` once.
typedef ag_status (*pq_codec_dev_fn)(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst,
                                     int64_t* d_written, int64_t* h_written, cudaStream_t st);

// device flavour: check, decompress
static inline ag_status pq_decompress_dev(const char* fn, pq_codec_dev_fn dev, const uint8_t* src, const ag_pq_compressed* pages,
                                          int64_t n_pages, uint8_t* dst, int64_t* d_written, cudaStream_t st) {
  int64_t src_end, dst_end;
  AG_TRY(pq_compressed_check(fn, src, pages, n_pages, dst, &src_end, &dst_end));
  if (n_pages == 0) return AG_OK;
  return dev(src, pages, n_pages, dst, d_written, nullptr, st);
}

// host flavour: check, stage the compressed bytes, decompress, copy back only the bytes each page wrote
static inline ag_status pq_decompress_host(const char* fn, pq_codec_dev_fn dev, const uint8_t* src, const ag_pq_compressed* pages,
                                           int64_t n_pages, uint8_t* dst, int64_t* written) {
  int64_t src_end, dst_end;
  AG_TRY(pq_compressed_check(fn, src, pages, n_pages, dst, &src_end, &dst_end));
  if (n_pages == 0) return AG_OK;
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  Carve sc;
  sc.take((size_t)src_end);
  const size_t o_dst = sc.take((size_t)dst_end);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, sc.size));
  AG_TRY(h2d(d, src, (size_t)src_end, cs));
  std::vector<int64_t> w((size_t)n_pages, 0);                    // stays 0 when the call fails before decoding
  const ag_status rc = dev(d, pages, n_pages, d + o_dst, nullptr, w.data(), cs);
  // a corrupt page still delivers the bytes it decoded before the failure
  if (rc != AG_OK && rc != AG_ERR_INVALID) return rc;
  if (written) memcpy(written, w.data(), (size_t)n_pages * 8);
  for (int64_t i = 0; i < n_pages; ++i) AG_TRY(d2h(dst + pages[i].dst, d + o_dst + pages[i].dst, (size_t)w[i], cs));
  const ag_status rs = sync(cs);
  return rc != AG_OK ? rc : rs;
}

// The plan a codec's kernels read: pages | K prefix arrays [n_pages + 1], one per per-page bound (element
// descriptors, literal bytes, ...).  total[k] is bound k over the batch, what the codec carves its scratch by.
template <size_t K>
struct LzPlan {
  std::vector<uint8_t> bytes;
  int64_t n_pages = 0;
  std::array<int64_t, K> total{};
};

// Its device views after lz_upload: base[k] is prefix array k.
template <size_t K>
struct LzPlanDev {
  const ag_pq_compressed* pages;
  std::array<const int64_t*, K> base;
};

// Plans a checked batch; bounds(page) gives the K bounds of one page as a std::array<int64_t, K>.
template <size_t K, typename Bounds>
static inline LzPlan<K> lz_plan(const ag_pq_compressed* pages, int64_t n_pages, Bounds bounds) {
  LzPlan<K> p;
  const size_t pb = (size_t)n_pages * sizeof(ag_pq_compressed), n1 = (size_t)n_pages + 1;
  p.n_pages = n_pages;
  p.bytes.assign(pb + K * n1 * 8, 0);
  memcpy(p.bytes.data(), pages, pb);
  int64_t* base = reinterpret_cast<int64_t*>(p.bytes.data() + pb);
  for (int64_t i = 0; i < n_pages; ++i) {
    const std::array<int64_t, K> b = bounds(pages[i]);
    for (size_t k = 0; k < K; ++k) base[k * n1 + i + 1] = base[k * n1 + i] + b[k];
  }
  for (size_t k = 0; k < K; ++k) p.total[k] = base[k * n1 + n_pages];
  return p;
}

// Uploads the plan to device memory `d` (p.bytes.size() bytes) and returns its device views.
template <size_t K>
static inline ag_status lz_upload(const LzPlan<K>& p, uint8_t* d, cudaStream_t st, LzPlanDev<K>* out) {
  AG_TRY(h2d(d, p.bytes.data(), p.bytes.size(), st));
  out->pages = reinterpret_cast<const ag_pq_compressed*>(d);
  const int64_t* base = reinterpret_cast<const int64_t*>(d + (size_t)p.n_pages * sizeof(ag_pq_compressed));
  for (size_t k = 0; k < K; ++k) out->base[k] = base + k * (size_t)(p.n_pages + 1);
  return AG_OK;
}

// The end of a call: copies the per-page states back, synchronises `st` once, fills h_written (host, may be NULL) from
// state.written, and fails on the lowest page that text(page, state, buf, size) writes a non-empty text for.
template <typename S, typename Text>
ag_status lz_read_back(const char* fn, const S* d_st, int64_t n_pages, int64_t* h_written, cudaStream_t st, Text text) {
  std::vector<S> hs((size_t)n_pages);
  AG_TRY(d2h(hs.data(), d_st, (size_t)n_pages * sizeof(S), st));
  AG_TRY(sync(st));
  if (h_written)
    for (int64_t i = 0; i < n_pages; ++i) h_written[i] = hs[i].written;
  for (int64_t i = 0; i < n_pages; ++i) {
    char msg[200] = "";
    text(i, hs[i], msg, sizeof msg);
    if (msg[0]) AG_FAIL(AG_ERR_INVALID, "%s: page %lld: %s (%lld bytes written)", fn, (long long)i, msg, (long long)hs[i].written);
  }
  return AG_OK;
}

// The text of a stream whose own output size is not the page's dst_len.
static inline void size_text(char* buf, size_t n, int64_t dst_len, int64_t got) {
  snprintf(buf, n, "parquet: metadata said %lld bytes uncompressed data page, got %lld bytes", (long long)dst_len, (long long)got);
}

constexpr int kLzThreads = 256;
constexpr int kLzBatch = 2048;                            // output bytes per execute step
constexpr unsigned long long kFromLit = 1ull << 61;       // execute: source byte is the page's literal buffer [low bits]
constexpr unsigned long long kFromDst = 1ull << 62;       // execute: source byte is dst[low bits]
constexpr unsigned long long kFromSrc = 1ull << 63;       // execute: source byte is the page's compressed byte [low bits]
constexpr unsigned long long kLzPosMask = kFromLit - 1;

enum LzKind : uint8_t { kLzCopy = 0, kLzSrc = 1, kLzLit = 2 };

struct LzExec {
  const ag_pq_compressed* pages;
  const int64_t* elem_base;   // [n_pages + 1]: first element descriptor of every page
  const uint8_t* src;         // kLzSrc literals: byte e_ref of the page's compressed bytes
  const uint8_t* lit;         // kLzLit literals: byte lit_base[p] + e_ref (NULL when no element is kLzLit)
  const int64_t* lit_base;
  uint8_t* dst;
  const int64_t* done;        // page p: done[p * stride] output bytes to write, done[p * stride + 1] elements
  int stride;
  const uint32_t* e_out;      // element: first output byte, within the page
  const uint32_t* e_ref;      // literal: byte offset of its bytes in its source; copy: the offset (any length)
  const uint8_t* e_lit;       // LzKind
};

// Launches lz_exec_kernel, one block per page, on `st`.
ag_status lz_exec_launch(const LzExec& x, int64_t n_pages, cudaStream_t st);

}  // namespace ag
