// snappy.cu — raw Snappy decompression of Parquet SNAPPY pages on the device.
//   serializedPageReader.decompress   parquet/file/page_reader.go:597-621 -> compress.Decode (parquet/compress/compress.go:107)
//                                     -> snappyCodec.DecodeWithError (parquet/compress/snappy.go:43-45)
//   element checks                    golang/snappy's decode (ErrCorrupt)
//
// A call decompresses a batch of pages (ag_pq_compressed descriptors, one device buffer of compressed bytes) in two
// launches, both one block per page:
//   1. snappy_parse_kernel: reads the preamble, then streams the compressed bytes through the shared-memory window of
//      pq_window.cuh in spans of 1024 candidate element starts.  Every thread decodes the element that would start at
//      each of its 4 positions (length, output length, offset); the element chain through the span is found by
//      span_chain's pointer doubling over those next-positions (a reach bitmask, log2(elements) rounds), and a block
//      scan of the chain's output lengths gives each element its output position.  Each element is validated here and
//      written as a 9-byte descriptor {output position, literal source / copy offset, literal flag}, so a failing page
//      knows how many bytes its valid elements produce before anything is executed.  A literal longer than the window
//      moves the next span (and window) past it without loading it.
//   2. lz_exec_kernel (lz_exec.cu, shared with every codec): walks the page's output in 2048-byte batches.  Byte j of a copy at `pos` is
//      dst[pos - off + (j mod off)], so every output byte names one source byte: a compressed byte (literals), an
//      output byte before the batch (read back from dst, which the same block wrote, L2-resident), or an earlier byte
//      of the same batch.  Pointer jumping in shared memory resolves the last kind, so overlapping copies and copies of
//      copies in one batch (offset 1 runs, the offset-8 copies of int64 columns) are as parallel as literals.
// Roofline.  compressed bytes read + decompressed bytes written.  This design also writes and reads 9 B per element
// descriptor and reads each copied byte once more (from L2).
#include <string.h>

#include <algorithm>
#include <vector>

#include "lz_exec.cuh"
#include "pq_window.cuh"

namespace ag {

namespace {

constexpr int kLook = 4;                    // bytes an element header reaches past its tag byte
constexpr unsigned long long kCntOne = 1ull << 48;   // parse scan: element count in bits 48.., output bytes below
constexpr unsigned long long kLenMask = kCntOne - 1;
constexpr unsigned long long kLenClamp = 1ull << 33; // any longer element is corrupt (dst_len <= 2^32-1)

constexpr const char* kFn = "snappy_decompress";     // message prefix

enum SnapErr : int { kSnOk = 0, kSnCorrupt = 1, kSnSize = 2 };

struct SnapPage {           // written by snappy_parse_kernel, read by lz_exec_kernel and the host
  int64_t written;          // output bytes of the page's valid elements (LzExec::done)
  int64_t nelem;            // element descriptors written
  int64_t preamble;         // the stream's uncompressed length (kSnSize names it)
  int32_t err;
  int32_t pad;
};

struct SnapArgs {
  const ag_pq_compressed* pages;
  const int64_t* elem_base;   // [n_pages + 1]: first element descriptor of every page
  const uint8_t* src;
  uint8_t* dst;
  SnapPage* st;
  uint32_t* e_out;            // element: first output byte, within the page
  uint32_t* e_ref;            // literal: byte offset of its bytes in the page's stream; copy: the offset
  uint8_t* e_lit;             // 1 = literal
  int64_t* d_written;         // may be NULL
};

// one block per page: preamble, element chain, validation, element descriptors
__global__ void __launch_bounds__(kPqThreads)
snappy_parse_kernel(SnapArgs a) {
  __shared__ uint4 win[kWinVec];
  __shared__ uint16_t jmp[2][kSpan];         // next chain position 2^r elements on (kSpan: leaves the span)
  __shared__ uint32_t reach[kSpan / 32];     // span positions on the element chain
  __shared__ unsigned long long warp_tot[kPqThreads / 32];
  __shared__ int64_t s_pos, s_next, s_written, s_nelem, s_pre, s_fail_out, s_fail_idx;
  __shared__ int s_err, s_done, s_fail;
  const int64_t p = blockIdx.x;
  const ag_pq_compressed pg = a.pages[p];
  const int tid = threadIdx.x;
  const uint8_t* in = a.src + pg.src;
  const int64_t len = pg.src_len, dlen = pg.dst_len;
  const int64_t eb = a.elem_base[p], cap = a.elem_base[p + 1] - eb;

  if (tid == 0) {
    int err = kSnOk;
    int64_t pos = 0;
    unsigned long long v = 0;
    if (len != 0 || dlen != 0) {                                 // an empty v2 value region has no preamble
      if (!read_uvarint([&](int64_t i) { return (uint32_t)__ldg(in + i); }, pos, len, &v) || v > 0xffffffffull) err = kSnCorrupt;
      else if ((int64_t)v != dlen) err = kSnSize;
    }
    s_pos = pos; s_pre = (int64_t)v; s_err = err; s_written = 0; s_nelem = 0;
    s_done = err != kSnOk || pos >= len;
  }

  const uint8_t* wb = reinterpret_cast<const uint8_t*>(win);
  const uintptr_t sbeg = reinterpret_cast<uintptr_t>(in);
  int64_t wlo = INT64_MIN / 2;                                   // stream offset of the window's first byte
  while (true) {
    __syncthreads();
    if (s_done) break;
    const int64_t cur = s_pos;
    if ((cur + kSpan + kLook < len ? cur + kSpan + kLook : len) > wlo + kWinBytes) {
      const uintptr_t a0 = (sbeg + cur) & ~(uintptr_t)15;      // the window starts at the span's aligned start
      load_window(win, sbeg, sbeg + len, a0);
      wlo = (int64_t)a0 - (int64_t)sbeg;
    }
    auto byte_at = [&](int64_t i) -> uint32_t { return i < len ? (uint32_t)wb[i - wlo] : 0u; };

    // ---- the element that would start at each of this thread's positions ----
    uint32_t J[kPer], ref[kPer];
    unsigned long long olen[kPer], elen[kPer];
    bool lit[kPer], bad[kPer], ends[kPer];
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const int q = tid * kPer + k;
      const int64_t i = cur + q;
      J[k] = kSpan; ref[k] = 0; olen[k] = 0; elen[k] = 0; lit[k] = false; bad[k] = true;
      if (i < len) {
        const uint32_t tag = byte_at(i);
        unsigned long long hdr, L;
        switch (tag & 3) {
          case 0: {
            const uint32_t m = tag >> 2;
            if (m < 60) {
              hdr = 1; L = m + 1;
            } else {                                             // length-1 in the next 1..4 bytes, little-endian
              const int nb = (int)m - 59;
              unsigned long long x = 0;
              for (int b = 0; b < nb; ++b) x |= (unsigned long long)byte_at(i + 1 + b) << (8 * b);
              hdr = 1 + nb; L = x + 1;
            }
            lit[k] = true;
            ref[k] = (uint32_t)(i + (int64_t)hdr);
            break;
          }
          case 1: hdr = 2; L = 4 + ((tag >> 2) & 7); ref[k] = ((tag >> 5) << 8) | byte_at(i + 1); break;
          case 2: hdr = 3; L = 1 + (tag >> 2); ref[k] = byte_at(i + 1) | byte_at(i + 2) << 8; break;
          default:
            hdr = 5; L = 1 + (tag >> 2);
            ref[k] = byte_at(i + 1) | byte_at(i + 2) << 8 | byte_at(i + 3) << 16 | byte_at(i + 4) << 24;
            break;
        }
        const unsigned long long e = hdr + (lit[k] ? L : 0ull);
        bad[k] = (unsigned long long)(len - i) < e;              // length, literal bytes or offset cut off
        elen[k] = e;
        olen[k] = L < kLenClamp ? L : kLenClamp;
        if (!bad[k] && (unsigned long long)q + e < kSpan && i + (int64_t)e < len) J[k] = (uint32_t)(q + e);
      }
      ends[k] = J[k] == kSpan;
      jmp[0][q] = (uint16_t)J[k];
    }
    if (tid == 0) s_fail = kSpan;
    span_chain(J, jmp, reach);

    // ---- output positions, validation, descriptors ----
    bool on[kPer];
    unsigned long long loc = 0;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      on[k] = bit_on(reach, tid * kPer + k);
      if (on[k]) loc += kCntOne | olen[k];
    }
    unsigned long long tot;
    const unsigned long long ex = block_excl_scan(loc, warp_tot, &tot);
    const int64_t w0 = s_written, n0 = s_nelem;
    unsigned long long run = ex;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      if (!on[k]) continue;
      const unsigned long long o = (unsigned long long)w0 + (run & kLenMask);
      const bool fail = bad[k] || o > (unsigned long long)dlen || olen[k] > (unsigned long long)dlen - o ||
                        (!lit[k] && (ref[k] == 0 || ref[k] > o));
      if (fail) atomicMin(&s_fail, tid * kPer + k);
      run += kCntOne | olen[k];
    }
    __syncthreads();
    const int fq = s_fail;
    run = ex;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      if (!on[k]) continue;
      const int q = tid * kPer + k;
      const int64_t o = w0 + (int64_t)(run & kLenMask), idx = n0 + (int64_t)(run >> 48);
      if (q < fq) {
        if (idx < cap) {
          a.e_out[eb + idx] = (uint32_t)o;
          a.e_ref[eb + idx] = ref[k];
          a.e_lit[eb + idx] = lit[k] ? 1 : 0;
        }
        if (ends[k]) s_next = cur + q + (int64_t)elen[k];
      } else if (q == fq) {
        s_fail_out = o; s_fail_idx = idx;
      }
      run += kCntOne | olen[k];
    }
    __syncthreads();
    if (tid == 0) {
      if (fq < kSpan) {
        s_err = kSnCorrupt; s_written = s_fail_out; s_nelem = s_fail_idx; s_done = 1;
      } else {
        s_written = w0 + (int64_t)(tot & kLenMask); s_nelem = n0 + (int64_t)(tot >> 48);
        s_pos = s_next;
        s_done = s_next >= len;
      }
    }
  }

  if (tid == 0) {
    int err = s_err;
    int64_t written = s_written, nelem = s_nelem;
    if (err == kSnOk && written != dlen) err = kSnCorrupt;      // the stream ends before the output is full
    if (err == kSnSize) written = nelem = 0;
    SnapPage ps;
    ps.written = written; ps.nelem = nelem < cap ? nelem : cap; ps.preamble = s_pre; ps.err = err; ps.pad = 0;
    a.st[p] = ps;
    if (a.d_written) a.d_written[p] = written;
  }
}

}  // namespace

// Decompresses a checked, non-empty batch of pages (pq_codec_dev_fn).
static ag_status snappy_dev(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst, int64_t* d_written,
                            int64_t* h_written, cudaStream_t st) {
  // plan: pages | elem_base[n+1].  A valid element takes >= 2 compressed bytes and produces >= 1 output byte.
  const LzPlan<1> plan = lz_plan<1>(pages, n_pages, [](const ag_pq_compressed& g) {
    return std::array<int64_t, 1>{std::min(g.src_len / 2, g.dst_len)};
  });
  const int64_t n_elem = plan.total[0];
  Carve sc;
  sc.take(plan.bytes.size());
  const size_t off_st = sc.take((size_t)n_pages * sizeof(SnapPage)), off_out = sc.take((size_t)n_elem * 4), off_ref = sc.take((size_t)n_elem * 4);
  const size_t off_lit = sc.take((size_t)n_elem);
  // this call synchronises `st` anyway, so its device scratch may live in a Temps
  Temps t(st);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, sc.size));
  LzPlanDev<1> pl;
  AG_TRY(lz_upload(plan, d, st, &pl));
  SnapArgs a;
  a.pages = pl.pages;
  a.elem_base = pl.base[0];
  a.src = src;
  a.dst = dst;
  a.st = reinterpret_cast<SnapPage*>(d + off_st);
  a.e_out = reinterpret_cast<uint32_t*>(d + off_out);
  a.e_ref = reinterpret_cast<uint32_t*>(d + off_ref);
  a.e_lit = d + off_lit;
  a.d_written = d_written;
  snappy_parse_kernel<<<(unsigned)n_pages, kPqThreads, 0, st>>>(a);
  AG_TRY(check_launch("snappy_parse_kernel"));
  LzExec x;
  x.pages = a.pages; x.elem_base = a.elem_base; x.src = src; x.lit = nullptr; x.lit_base = nullptr; x.dst = dst;
  x.done = reinterpret_cast<const int64_t*>(a.st); x.stride = sizeof(SnapPage) / 8;
  x.e_out = a.e_out; x.e_ref = a.e_ref; x.e_lit = a.e_lit;
  AG_TRY(lz_exec_launch(x, n_pages, st));
  return lz_read_back(kFn, a.st, n_pages, h_written, st, [&](int64_t i, const SnapPage& s, char* buf, size_t n) {
    if (s.err == kSnSize) size_text(buf, n, pages[i].dst_len, s.preamble);
    else if (s.err == kSnCorrupt) snprintf(buf, n, "parquet: could not decompress page: snappy: corrupt input");
  });
}

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_parquet_snappy_decompress_dev(const uint8_t* d_src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* d_dst,
                                           int64_t* d_written, ag_stream_t s) {
  AG_TRY(ensure_init());
  return pq_decompress_dev(kFn, snappy_dev, d_src, pages, n_pages, d_dst, d_written, resolve_stream(s));
}

ag_status ag_parquet_snappy_decompress(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst,
                                       int64_t* written) {
  AG_TRY(ensure_init());
  return pq_decompress_host(kFn, snappy_dev, src, pages, n_pages, dst, written);
}

}  // extern "C"
