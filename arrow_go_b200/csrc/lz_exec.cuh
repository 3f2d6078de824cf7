// lz_exec.cuh — what the Parquet page decompressors (snappy.cu, zstd.cu, gzip.cu, lz4.cu) share.  Internal, not part of
// the ABI.
//
//   pq_compressed_check   the argument checks of an ag_pq_compressed batch, AG_ERR_INVALID before any launch
//   pq_decompress_host    the host-pointer flavour: stage src, run the device flavour, copy back only written bytes
//   lz_exec_page          the executor: a page's output from element descriptors {first output byte, literal source /
//                         copy offset, kind}, in 2048-byte batches with pointer jumping over in-batch sources
#pragma once

#include <string.h>

#include <algorithm>
#include <vector>

#include "host_stage.cuh"

namespace ag {

// Argument checks shared by every codec and both flavours; every one is AG_ERR_INVALID before any launch.
// *src_end / *dst_end: the bytes of `src` / `dst` the batch spans.
static inline ag_status pq_compressed_check(const char* fn, const ag_pq_compressed* pages, int64_t n_pages, int64_t* src_end,
                                            int64_t* dst_end) {
  *src_end = *dst_end = 0;
  if (n_pages < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative page count", fn);
  if (n_pages == 0) return AG_OK;
  if (!pages) AG_FAIL(AG_ERR_INVALID, "%s: NULL page table", fn);
  std::vector<int64_t> order;
  for (int64_t i = 0; i < n_pages; ++i) {
    const ag_pq_compressed& g = pages[i];
    if (g.src < 0 || g.src_len < 0 || g.dst < 0 || g.dst_len < 0 || g.src_len > 0xffffffffLL || g.dst_len > 0xffffffffLL)
      AG_FAIL(AG_ERR_INVALID, "%s: page %lld: negative field or more than 2^32-1 bytes", fn, (long long)i);
    *src_end = std::max(*src_end, g.src + g.src_len);
    *dst_end = std::max(*dst_end, g.dst + g.dst_len);
    if (g.dst_len > 0) order.push_back(i);
  }
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

// The device flavour of a codec: decompresses into device `dst`, fills h_written (host, may be NULL) with the bytes per
// page, synchronises `st` once.
typedef ag_status (*pq_codec_dev_fn)(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst,
                                     int64_t* d_written, int64_t* h_written, cudaStream_t st);

// host flavour: stage the compressed bytes, decompress, copy back only the bytes each page wrote
static inline ag_status pq_decompress_host(const char* fn, pq_codec_dev_fn dev, const uint8_t* src, const ag_pq_compressed* pages,
                                           int64_t n_pages, uint8_t* dst, int64_t* written) {
  int64_t src_end, dst_end;
  AG_TRY(pq_compressed_check(fn, pages, n_pages, &src_end, &dst_end));
  if (n_pages == 0) return AG_OK;
  if (src_end > 0 && !src) AG_FAIL(AG_ERR_INVALID, "%s: NULL compressed data", fn);
  if (dst_end > 0 && !dst) AG_FAIL(AG_ERR_INVALID, "%s: NULL output", fn);
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

// One block (kLzThreads) writes page p's output in batches of kLzBatch bytes, in order.  Each element produces at
// least one byte.  Byte j of a copy at `pos` with offset r is dst[pos - r + (j mod r)], so every output byte names
// one source byte: a literal byte, an output byte before the batch (read back from dst, written by this block), or
// an earlier byte of the same batch, which pointer jumping in shared memory resolves.
__device__ __forceinline__ void lz_exec_page(const LzExec& a, int64_t p) {
  __shared__ uint32_t s_out[kLzBatch + 1], s_ref[kLzBatch + 1];
  __shared__ uint8_t s_lit[kLzBatch + 1];
  __shared__ unsigned long long s_src[kLzBatch];
  const int64_t written = a.done[p * a.stride], nelem = a.done[p * a.stride + 1];
  if (written <= 0 || nelem <= 0) return;                        // block-uniform
  const ag_pq_compressed pg = a.pages[p];
  const uint8_t* in = a.src + pg.src;
  const uint8_t* lit = a.lit ? a.lit + a.lit_base[p] : nullptr;
  uint8_t* out = a.dst + pg.dst;
  const int64_t eb = a.elem_base[p];
  const int tid = threadIdx.x;
  int64_t e0 = 0;                                                // the element holding the batch's first byte
  for (int64_t B = 0; B < written; B += kLzBatch) {
    const int nb = (int)(written - B < kLzBatch ? written - B : kLzBatch);
    // elements e0 .. e0 + nl - 1 hold every byte of [B, B + kLzBatch] (each element produces at least one byte)
    const int nl = (int)(nelem - e0 < kLzBatch + 1 ? nelem - e0 : kLzBatch + 1);
    for (int k = tid; k < nl; k += kLzThreads) {
      s_out[k] = a.e_out[eb + e0 + k];
      s_ref[k] = a.e_ref[eb + e0 + k];
      s_lit[k] = a.e_lit[eb + e0 + k];
    }
    __syncthreads();
    auto holder = [&](uint32_t pos) {                            // last loaded element starting at or before pos
      int lo = 0, hi = nl - 1;
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (s_out[mid] <= pos) lo = mid; else hi = mid - 1;
      }
      return lo;
    };
    for (int b = tid; b < nb; b += kLzThreads) {
      const uint32_t pos = (uint32_t)(B + b);
      const int e = holder(pos);
      const uint32_t j = pos - s_out[e], r = s_ref[e];
      unsigned long long s;
      if (s_lit[e]) {
        s = (s_lit[e] == kLzSrc ? kFromSrc : kFromLit) | (unsigned long long)(r + j);
      } else {
        const uint32_t q = s_out[e] - r + (j < r ? j : j % r);
        s = (int64_t)q < B ? kFromDst | q : (unsigned long long)((int64_t)q - B);
      }
      s_src[b] = s;
    }
    __syncthreads();
    while (true) {                                               // pointer jumping to a byte outside the batch
      bool pend = false;
      for (int b = tid; b < nb; b += kLzThreads) {
        const unsigned long long v = s_src[b];
        if (v < kFromLit) {
          const unsigned long long w = s_src[v];
          s_src[b] = w;
          pend |= w < kFromLit;
        }
      }
      if (!__syncthreads_or(pend)) break;
    }
    for (int b = tid; b < nb; b += kLzThreads) {
      const unsigned long long v = s_src[b];
      // dst bytes before the batch were written by this block before the last barrier: a plain (coherent) load
      out[B + b] = (v & kFromSrc) ? __ldg(in + (v & kLzPosMask)) : (v & kFromLit) ? lit[v & kLzPosMask] : out[v & kLzPosMask];
    }
    e0 += holder((uint32_t)(B + kLzBatch < written ? B + kLzBatch : written - 1));
    __syncthreads();
  }
}

}  // namespace ag
