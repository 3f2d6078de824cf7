// lz4.cu — LZ4 block decompression of Parquet LZ4_RAW pages on the device.
//   serializedPageReader.decompress   parquet/file/page_reader.go:597-621 -> compress.Decode (parquet/compress/compress.go:107)
//                                     -> lz4RawCodec.DecodeWithError (parquet/compress/lz4_raw.go:63-70) -> lz4.UncompressBlock
//   sequence checks                   pierrec/lz4 v4's block decoder (ErrInvalidSourceShortBuffer)
//
// A call decompresses a batch of pages (ag_pq_compressed descriptors, one device buffer of compressed bytes) in two
// launches, both one block per page, in the shape of snappy.cu:
//   1. lz4_parse_kernel: streams the compressed bytes through the shared-memory window of pq_window.cuh in spans of
//      1024 candidate token positions.  Every thread decodes the sequence that would start at each of its 4 positions
//      (token, literal length, offset, match length; an extension run is read from the window up to kExt bytes), the
//      sequence chain through the span is found by span_chain, and a block scan of the chain's output lengths and
//      element counts gives each sequence its output position and its first descriptor.  A sequence is one kLzSrc
//      literal (none when its literal run is empty) and one kLzCopy match (none when it ends the stream).  Every element
//      is validated here, so a failing page knows how many bytes its valid elements produce before anything executes.
//      A sequence that leaves the window (an extension run longer than kExt, or literals that carry its offset past the
//      window) ends the span: its thread finishes it from global memory and the next span starts after it.
//   2. lz_exec_kernel: the shared executor of lz_exec.cu, unchanged (the 16-bit offsets fit e_ref).
// Roofline.  compressed bytes read + decompressed bytes written.  This design also writes and reads 9 B per element
// descriptor and reads each copied byte once more (from L2).
#include <string.h>

#include <algorithm>
#include <vector>

#include "lz_exec.cuh"
#include "pq_window.cuh"

namespace ag {

namespace {

constexpr int kExt = 16;                    // extension bytes a window decode reads; a longer run leaves the window
constexpr int kLook = 2 * kExt + 3;         // bytes past a span a short sequence's header reaches (token, runs, offset)
constexpr unsigned long long kCntOne = 1ull << 48;   // parse scan: descriptor count in bits 48.., output bytes below
constexpr unsigned long long kLenMask = kCntOne - 1;

constexpr const char* kFn = "lz4_raw_decompress";    // message prefix

enum Lz4Err : int { kL4Ok = 0, kL4Corrupt = 1, kL4Size = 2 };
enum SeqState : int { kSqOk = 0, kSqBadLit = 1, kSqBadMatch = 2, kSqOut = 3 };

struct Lz4Page {            // written by lz4_parse_kernel, read by lz_exec_kernel and the host
  int64_t written;          // output bytes of the page's valid elements (LzExec::done)
  int64_t nelem;            // element descriptors written
  int64_t got;              // a clean stream's output bytes (kL4Size names them)
  int32_t err;
  int32_t pad;
};

struct Lz4Args {
  const ag_pq_compressed* pages;
  const int64_t* elem_base;   // [n_pages + 1]: first element descriptor of every page
  const uint8_t* src;
  uint8_t* dst;
  Lz4Page* st;
  uint32_t* e_out;            // element: first output byte, within the page
  uint32_t* e_ref;            // literal: byte offset of its bytes in the page's stream; match: the offset
  uint8_t* e_lit;             // LzKind
  int64_t* d_written;         // may be NULL
};

struct Seq {
  unsigned long long ll, ml;  // literal and match bytes (ml == 0: the sequence ends the stream)
  int64_t lit, end;           // stream offsets of the literals and of the next token
  uint32_t off;
  int state;                  // SeqState
};

// The sequence whose token is at i < len.  byte_at(j) is the byte at stream offset j, -1 past the input and -2 past
// what the caller holds (kSqOut); an extension run of `cap` bytes of 255 is kSqOut too.
template <typename B>
__device__ __forceinline__ Seq lz4_seq(B byte_at, int64_t i, int64_t len, int64_t cap) {
  Seq s;
  s.ml = 0; s.off = 0; s.end = len;
  const int t = byte_at(i);
  int64_t p = i + 1;
  auto run = [&](unsigned long long& n, int bad) -> int {      // extension bytes, each added, up to the first < 255
    for (int64_t k = 0;; ++k) {
      if (k == cap) return kSqOut;
      const int b = byte_at(p);
      if (b == -2) return kSqOut;
      if (b < 0) return bad;
      ++p;
      n += (unsigned)b;
      if (b != 255) return kSqOk;
    }
  };
  s.ll = (unsigned)t >> 4;
  s.state = s.ll == 15 ? run(s.ll, kSqBadLit) : kSqOk;
  s.lit = p;
  if (s.state != kSqOk) return s;
  if ((unsigned long long)(len - p) < s.ll) { s.state = kSqBadLit; return s; }
  p += (int64_t)s.ll;
  if (p == len) {                                                // the input ends after the literals
    s.state = (t & 15) ? kSqBadMatch : kSqOk;
    return s;
  }
  if (len - p < 2) { s.state = kSqBadMatch; return s; }
  const int b0 = byte_at(p), b1 = byte_at(p + 1);
  if (b0 == -2 || b1 == -2) { s.state = kSqOut; return s; }
  s.off = (uint32_t)b0 | (uint32_t)b1 << 8;
  p += 2;
  s.ml = (unsigned)(t & 15);
  s.state = s.ml == 15 ? run(s.ml, kSqBadMatch) : kSqOk;
  s.ml += 4;
  s.end = p;
  return s;
}

// 0: both elements of a sequence placed at output byte o are valid; kSqBadLit / kSqBadMatch: the element that fails
__device__ __forceinline__ int lz4_check(int state, unsigned long long ll, unsigned long long ml, uint32_t off,
                                         unsigned long long o, unsigned long long dlen) {
  if (state == kSqBadLit || ll > dlen - o) return kSqBadLit;
  if (state == kSqBadMatch || (ml && (off == 0 || off > o + ll || ml > dlen - o - ll))) return kSqBadMatch;
  return kSqOk;
}

// one block per page: sequence chain, validation, element descriptors
__global__ void __launch_bounds__(kPqThreads)
lz4_parse_kernel(Lz4Args a) {
  __shared__ uint4 win[kWinVec];
  __shared__ uint16_t jmp[2][kSpan];         // next chain position 2^r sequences on (kSpan: leaves the span)
  __shared__ uint32_t reach[kSpan / 32];     // span positions on the sequence chain
  __shared__ unsigned long long warp_tot[kPqThreads / 32];
  __shared__ int64_t s_pos, s_next, s_written, s_nelem, s_fail_out, s_fail_idx, s_xw, s_xn;
  __shared__ int s_err, s_done, s_fail, s_xfail;
  const int64_t p = blockIdx.x;
  const ag_pq_compressed pg = a.pages[p];
  const int tid = threadIdx.x;
  const uint8_t* in = a.src + pg.src;
  const int64_t len = pg.src_len, dlen = pg.dst_len;
  const int64_t eb = a.elem_base[p], cap = a.elem_base[p + 1] - eb;

  if (tid == 0) {
    s_pos = 0; s_err = kL4Ok; s_written = 0; s_nelem = 0;
    s_done = len == 0;
  }

  // descriptors of the valid elements of a sequence at output byte o, first descriptor idx; -> descriptors written
  auto emit = [&](const Seq& s, int64_t o, int64_t idx, int fail) -> int {
    int n = 0;
    if (fail != kSqBadLit && s.ll) {
      if (idx < cap) { a.e_out[eb + idx] = (uint32_t)o; a.e_ref[eb + idx] = (uint32_t)s.lit; a.e_lit[eb + idx] = kLzSrc; }
      ++n;
    }
    if (fail == kSqOk && s.ml) {
      if (idx + n < cap) { a.e_out[eb + idx + n] = (uint32_t)(o + (int64_t)s.ll); a.e_ref[eb + idx + n] = s.off; a.e_lit[eb + idx + n] = kLzCopy; }
      ++n;
    }
    return n;
  };

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
    const int64_t wend = wlo + kWinBytes;
    auto byte_at = [&](int64_t j) -> int { return j >= len ? -1 : j >= wend ? -2 : (int)wb[j - wlo]; };

    // ---- the sequence that would start at each of this thread's positions ----
    uint32_t J[kPer], nxt[kPer], ll[kPer], ml[kPer], off[kPer], lrel[kPer];
    int state[kPer];
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const int q = tid * kPer + k;
      const int64_t i = cur + q;
      J[k] = kSpan; nxt[k] = 0; ll[k] = 0; ml[k] = 0; off[k] = 0; lrel[k] = 0; state[k] = kSqBadLit;
      if (i < len) {
        const Seq s = lz4_seq(byte_at, i, len, kExt);
        state[k] = s.state;
        if (s.state != kSqOut) {                                 // in the window: lengths below 2^13
          ll[k] = (uint32_t)s.ll; ml[k] = (uint32_t)s.ml; off[k] = s.off; lrel[k] = (uint32_t)(s.lit - i);
          nxt[k] = (uint32_t)(q + (s.end - i));
          if (s.state == kSqOk && s.ml && nxt[k] < kSpan && s.end < len) J[k] = nxt[k];
        }
      }
      jmp[0][q] = (uint16_t)J[k];
    }
    if (tid == 0) { s_fail = kSpan; s_xfail = 0; s_xw = 0; s_xn = 0; }
    span_chain(J, jmp, reach);

    // ---- output positions, validation, descriptors ----
    bool on[kPer];
    unsigned long long loc = 0;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      on[k] = bit_on(reach, tid * kPer + k);
      if (on[k] && state[k] != kSqOut) loc += kCntOne * ((ll[k] != 0) + (ml[k] != 0)) | (ll[k] + ml[k]);
    }
    unsigned long long tot;
    const unsigned long long ex = block_excl_scan(loc, warp_tot, &tot);
    const int64_t w0 = s_written, n0 = s_nelem;
    unsigned long long run = ex;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      if (!on[k] || state[k] == kSqOut) continue;
      const unsigned long long o = (unsigned long long)w0 + (run & kLenMask);
      if (lz4_check(state[k], ll[k], ml[k], off[k], o, (unsigned long long)dlen) != kSqOk) atomicMin(&s_fail, tid * kPer + k);
      run += kCntOne * ((ll[k] != 0) + (ml[k] != 0)) | (ll[k] + ml[k]);
    }
    __syncthreads();
    const int fq = s_fail;
    run = ex;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      if (!on[k]) continue;
      const int q = tid * kPer + k;
      if (q > fq) break;
      const int64_t o = w0 + (int64_t)(run & kLenMask), idx = n0 + (int64_t)(run >> 48), i = cur + q;
      if (state[k] == kSqOut) {                                  // the chain's last sequence: finish it from global memory
        const Seq s = lz4_seq([&](int64_t j) -> int { return j < len ? (int)__ldg(in + j) : -1; }, i, len, INT64_MAX);
        const int f = lz4_check(s.state, s.ll, s.ml, s.off, (unsigned long long)o, (unsigned long long)dlen);
        s_xn = emit(s, o, idx, f);
        s_xw = f == kSqBadLit ? 0 : f == kSqBadMatch ? (int64_t)s.ll : (int64_t)(s.ll + s.ml);
        s_xfail = f != kSqOk;
        s_next = s.end;
        break;
      }
      Seq s;
      s.ll = ll[k]; s.ml = ml[k]; s.off = off[k]; s.lit = i + lrel[k]; s.state = state[k];
      const int f = q == fq ? lz4_check(state[k], ll[k], ml[k], off[k], (unsigned long long)o, (unsigned long long)dlen) : kSqOk;
      const int n = emit(s, o, idx, f);
      if (q == fq) {
        s_fail_out = o + (f == kSqBadMatch ? (int64_t)ll[k] : 0); s_fail_idx = idx + n;
      } else if (!ml[k] || nxt[k] >= kSpan || cur + nxt[k] >= len) {
        s_next = cur + nxt[k];                                   // the chain leaves the span, or the stream ends here
      }
      run += kCntOne * ((ll[k] != 0) + (ml[k] != 0)) | (ll[k] + ml[k]);
    }
    __syncthreads();
    if (tid == 0) {
      if (fq < kSpan) {
        s_err = kL4Corrupt; s_written = s_fail_out; s_nelem = s_fail_idx; s_done = 1;
      } else {
        s_written = w0 + (int64_t)(tot & kLenMask) + s_xw; s_nelem = n0 + (int64_t)(tot >> 48) + s_xn;
        if (s_xfail) {
          s_err = kL4Corrupt; s_done = 1;
        } else {
          s_pos = s_next;
          s_done = s_next >= len;
        }
      }
    }
  }

  if (tid == 0) {
    int err = s_err;
    int64_t written = s_written, nelem = s_nelem, got = 0;
    if (err == kL4Ok && written != dlen) {
      if (len == 0) {
        err = kL4Corrupt;                                        // an empty block with output to fill
      } else {
        err = kL4Size; got = written; written = nelem = 0;
      }
    }
    Lz4Page ps;
    ps.written = written; ps.nelem = nelem < cap ? nelem : cap; ps.got = got; ps.err = err; ps.pad = 0;
    a.st[p] = ps;
    if (a.d_written) a.d_written[p] = written;
  }
}

}  // namespace

// Decompresses a checked, non-empty batch of pages (pq_codec_dev_fn).
static ag_status lz4_raw_dev(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst, int64_t* d_written,
                             int64_t* h_written, cudaStream_t st) {
  // plan: pages | elem_base[n+1].  Every sequence but the last takes >= 3 compressed bytes and makes <= 2 elements;
  // every valid element produces >= 1 output byte.
  const LzPlan<1> plan = lz_plan<1>(pages, n_pages, [](const ag_pq_compressed& g) {
    return std::array<int64_t, 1>{std::min(g.dst_len, 2 * (g.src_len / 3) + 2)};
  });
  const int64_t n_elem = plan.total[0];
  Carve sc;
  sc.take(plan.bytes.size());
  const size_t off_st = sc.take((size_t)n_pages * sizeof(Lz4Page)), off_out = sc.take((size_t)n_elem * 4), off_ref = sc.take((size_t)n_elem * 4);
  const size_t off_lit = sc.take((size_t)n_elem);
  // this call synchronises `st` anyway, so its device scratch may live in a Temps
  Temps t(st);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, sc.size));
  LzPlanDev<1> pl;
  AG_TRY(lz_upload(plan, d, st, &pl));
  Lz4Args a;
  a.pages = pl.pages;
  a.elem_base = pl.base[0];
  a.src = src;
  a.dst = dst;
  a.st = reinterpret_cast<Lz4Page*>(d + off_st);
  a.e_out = reinterpret_cast<uint32_t*>(d + off_out);
  a.e_ref = reinterpret_cast<uint32_t*>(d + off_ref);
  a.e_lit = d + off_lit;
  a.d_written = d_written;
  lz4_parse_kernel<<<(unsigned)n_pages, kPqThreads, 0, st>>>(a);
  AG_TRY(check_launch("lz4_parse_kernel"));
  LzExec x;
  x.pages = a.pages; x.elem_base = a.elem_base; x.src = src; x.lit = nullptr; x.lit_base = nullptr; x.dst = dst;
  x.done = reinterpret_cast<const int64_t*>(a.st); x.stride = sizeof(Lz4Page) / 8;
  x.e_out = a.e_out; x.e_ref = a.e_ref; x.e_lit = a.e_lit;
  AG_TRY(lz_exec_launch(x, n_pages, st));
  return lz_read_back(kFn, a.st, n_pages, h_written, st, [&](int64_t i, const Lz4Page& s, char* buf, size_t n) {
    if (s.err == kL4Size) size_text(buf, n, pages[i].dst_len, s.got);
    else if (s.err == kL4Corrupt) snprintf(buf, n, "parquet: could not decompress page: lz4: invalid source or destination buffer too short");
  });
}

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_parquet_lz4_raw_decompress_dev(const uint8_t* d_src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* d_dst,
                                            int64_t* d_written, ag_stream_t s) {
  AG_TRY(ensure_init());
  return pq_decompress_dev(kFn, lz4_raw_dev, d_src, pages, n_pages, d_dst, d_written, resolve_stream(s));
}

ag_status ag_parquet_lz4_raw_decompress(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst,
                                        int64_t* written) {
  AG_TRY(ensure_init());
  return pq_decompress_host(kFn, lz4_raw_dev, src, pages, n_pages, dst, written);
}

}  // extern "C"
