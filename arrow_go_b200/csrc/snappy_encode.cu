// snappy_encode.cu — raw Snappy compression of Parquet SNAPPY pages on the device.
//   serializedPageWriter.Compress   parquet/file/page_writer.go:229-233 (CompressBound, then EncodeLevel)
//                                   -> snappyCodec.Encode / CompressBound (parquet/compress/snappy.go:27-33, 51-53)
//
// The parse is fixed (include/arrowgpu.h states it; tests/snappy_encode_model.py pins it byte for byte): every page is
// cut into 64 KiB fragments, each with its own 4096-entry hash table and copies only within itself, walked in windows
// of 32 candidate positions where the first position whose latest same-hash predecessor holds the same 4 bytes starts
// a match.  A call is two launches:
//   1. snappy_match_kernel: one warp per fragment, kMatchWarps fragments per block, a uint16 table per warp in shared
//      memory.  Each lane hashes one position of the window; its candidate is the highest lower lane with the same
//      hash (__match_any_sync masked below the lane), else the table entry.  The first matching lane comes from a
//      ballot; lanes up to it insert their positions, the highest lane of each hash writing.  A match is extended 32
//      bytes per step with a ballot.  The warp writes the fragment's elements to scratch at a fixed stride.
//   2. snappy_assemble_kernel: one block per page writes the preamble and moves the page's fragments into place in
//      order, with 16-byte stores where the destination is aligned.
// Scratch bound of a fragment of m bytes.  Its elements are (literal, copy) pairs and one last literal.  A copy of
// n >= 4 bytes takes at most n - 1 bytes (3 per 64- or 60-byte piece, 2 or 3 for the last piece of 4..64).  A literal
// of k bytes takes k + 1 (k <= 60), k + 2 (k <= 256) or k + 3 bytes (k <= 65536).  So a pair costs at most what it
// covers plus 1 when k > 60 (the pair covers >= 65 bytes) or plus 2 when k > 256 (>= 261 bytes), at most 1 per 65
// bytes covered, and the last literal adds at most 3: m + m / 65 + 3 bytes.  Summed over a page's fragments with
// the preamble this stays below ag_parquet_snappy_max_size's 32 + n + n / 6.
// Scratch: kFragStride (66,560) bytes per fragment, about the input's size, plus 4 bytes per fragment.
// Roofline.  input read + output written; this design adds the fragments' elements written to scratch and read back.
#include "lz_exec.cuh"

namespace ag {

namespace {

constexpr int kFrag = 1 << 16;                       // bytes per fragment
constexpr int kTableBits = 12;                       // 4096-entry hash table per fragment
constexpr int kMatchWarps = 4;                       // fragments per block of the match kernel
constexpr int kAsmThreads = 256;
constexpr uint32_t kEmpty = 0xffff;                  // no position (every candidate position is below 65533)
constexpr int64_t kFragBound = kFrag + kFrag / 65 + 3;
constexpr int64_t kFragStride = (kFragBound + 15) / 16 * 16;

constexpr const char* kFn = "snappy_compress";

struct SnapFrag {            // one fragment: its input bytes (absolute offset in src) and their count
  int64_t src;
  int64_t len;
};

__device__ __forceinline__ uint32_t load32(const uint8_t* p) {
  return (uint32_t)__ldg(p) | (uint32_t)__ldg(p + 1) << 8 | (uint32_t)__ldg(p + 2) << 16 | (uint32_t)__ldg(p + 3) << 24;
}

// one literal of k bytes from `in` at out[op..]; returns the new op (warp-uniform)
__device__ __forceinline__ int emit_literal(uint8_t* out, int op, const uint8_t* in, int k, int lane) {
  if (k == 0) return op;
  const uint32_t n = (uint32_t)k - 1;
  const int hdr = n < 60 ? 1 : n < 256 ? 2 : 3;
  if (lane == 0) {
    out[op] = (uint8_t)(n < 60 ? n << 2 : n < 256 ? 60 << 2 : 61 << 2);
    if (hdr > 1) out[op + 1] = (uint8_t)n;
    if (hdr > 2) out[op + 2] = (uint8_t)(n >> 8);
  }
  for (int j = lane; j < k; j += 32) out[op + hdr + j] = __ldg(in + j);
  return op + hdr + k;
}

// the copy of n >= 4 bytes at offset `off` in golang/snappy's forms; returns the new op (warp-uniform)
__device__ __forceinline__ int emit_copy(uint8_t* out, int op, uint32_t off, int n, int lane) {
  const int chunks = n >= 68 ? (n - 68) / 64 + 1 : 0;          // 64-byte pieces, 2-byte offset
  for (int j = lane; j < chunks; j += 32) {
    out[op + 3 * j] = 63 << 2 | 2;
    out[op + 3 * j + 1] = (uint8_t)off;
    out[op + 3 * j + 2] = (uint8_t)(off >> 8);
  }
  op += 3 * chunks;
  n -= 64 * chunks;
  if (n > 64) {                                                  // 65..67 left: a 60-byte piece first
    if (lane == 0) { out[op] = 59 << 2 | 2; out[op + 1] = (uint8_t)off; out[op + 2] = (uint8_t)(off >> 8); }
    op += 3;
    n -= 60;
  }
  if (n < 12 && off < 2048) {
    if (lane == 0) { out[op] = (uint8_t)((off >> 8) << 5 | (n - 4) << 2 | 1); out[op + 1] = (uint8_t)off; }
    return op + 2;
  }
  if (lane == 0) { out[op] = (uint8_t)((n - 1) << 2 | 2); out[op + 1] = (uint8_t)off; out[op + 2] = (uint8_t)(off >> 8); }
  return op + 3;
}

// one warp per fragment: its elements at scratch + f * kFragStride, their byte count in frag_out[f]
__global__ void __launch_bounds__(kMatchWarps * 32)
snappy_match_kernel(const SnapFrag* frags, int64_t n_frags, const uint8_t* src, uint8_t* scratch, uint32_t* frag_out) {
  __shared__ uint16_t table[kMatchWarps][1 << kTableBits];
  const int lane = threadIdx.x & 31;
  const int64_t f = (int64_t)blockIdx.x * kMatchWarps + (threadIdx.x >> 5);
  if (f >= n_frags) return;                                      // warp-uniform; no block barrier follows
  uint16_t* tb = table[threadIdx.x >> 5];
  uint32_t* tb32 = reinterpret_cast<uint32_t*>(tb);
  for (int i = lane; i < (1 << kTableBits) / 2; i += 32) tb32[i] = kEmpty | kEmpty << 16;
  __syncwarp();
  const SnapFrag fr = frags[f];
  const uint8_t* in = src + fr.src;
  const int m = (int)fr.len, nc = m - 3;                         // candidate positions p: p + 4 <= m
  uint8_t* out = scratch + f * kFragStride;
  const unsigned below = (1u << lane) - 1;
  int op = 0, lit = 0, cur = 0;
  while (cur < nc) {
    const int p = cur + lane;
    const bool valid = p < nc;
    const uint32_t x = valid ? load32(in + p) : 0u;
    const uint32_t h = (x * 0x1E35A7BDu) >> (32 - kTableBits);
    const unsigned peers = __match_any_sync(0xffffffffu, valid ? h : 0x10000u + lane);
    const unsigned lower = peers & below;
    const int q = lower ? cur + 31 - __clz(lower) : valid ? (int)tb[h] : (int)kEmpty;
    const bool hit = valid && q != (int)kEmpty && load32(in + q) == x;
    const unsigned ball = __ballot_sync(0xffffffffu, hit);
    const int first = ball ? __ffs(ball) - 1 : 31;
    const unsigned upto = first == 31 ? 0xffffffffu : (2u << first) - 1;
    __syncwarp();                                                // every lane has read the table
    if (valid && lane <= first && (peers & upto) >> lane == 1u) tb[h] = (uint16_t)p;
    __syncwarp();
    if (!ball) {
      cur += 32;
      continue;
    }
    const int pm = cur + first, qm = __shfl_sync(0xffffffffu, q, first);
    int n = 4;
    while (true) {
      const int i = pm + n + lane;
      const bool diff = i >= m || __ldg(in + qm + n + lane) != __ldg(in + i);
      const unsigned b = __ballot_sync(0xffffffffu, diff);
      if (b) { n += __ffs(b) - 1; break; }
      n += 32;
    }
    op = emit_literal(out, op, in + lit, pm - lit, lane);
    op = emit_copy(out, op, (uint32_t)(pm - qm), n, lane);
    cur = lit = pm + n;
  }
  op = emit_literal(out, op, in + lit, m - lit, lane);
  if (lane == 0) frag_out[f] = (uint32_t)op;
}

// out[0..len) = in[0..len), `in` 4-byte aligned (a fragment's scratch); 16-byte stores where `out` is aligned
__device__ __forceinline__ void block_move(uint8_t* out, const uint8_t* in, int64_t len) {
  const int tid = threadIdx.x;
  const int64_t head = std::min<int64_t>(len, (16 - (reinterpret_cast<uintptr_t>(out) & 15)) & 15);
  const int64_t mid = (len - head) / 16, tail = head + mid * 16;
  if (tid < head) out[tid] = in[tid];
  const uintptr_t sa = reinterpret_cast<uintptr_t>(in + head);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(sa & ~(uintptr_t)3);
  const int sh = (int)(sa & 3) * 8;
  uint4* o = reinterpret_cast<uint4*>(out + head);
  for (int64_t k = tid; k < mid; k += kAsmThreads) {
    const uint32_t* s = w + 4 * k;
    const uint32_t a0 = s[0], a1 = s[1], a2 = s[2], a3 = s[3], a4 = sh ? s[4] : 0u;
    o[k] = make_uint4(__funnelshift_r(a0, a1, sh), __funnelshift_r(a1, a2, sh), __funnelshift_r(a2, a3, sh),
                      __funnelshift_r(a3, a4, sh));
  }
  for (int64_t j = tail + tid; j < len; j += kAsmThreads) out[j] = in[j];
}

// one block per page: the preamble, then the page's fragments in order
__global__ void __launch_bounds__(kAsmThreads)
snappy_assemble_kernel(const ag_pq_compressed* pages, const int64_t* frag_base, const uint8_t* scratch,
                       const uint32_t* frag_out, uint8_t* dst, int64_t* d_written) {
  const int64_t p = blockIdx.x;
  const ag_pq_compressed pg = pages[p];
  uint8_t* out = dst + pg.dst;
  int64_t pos = 0;
  for (uint64_t v = (uint64_t)pg.src_len;; v >>= 7) {            // uvarint(src_len)
    if (threadIdx.x == 0) out[pos] = (uint8_t)(v >= 0x80 ? (v & 0x7f) | 0x80 : v);
    ++pos;
    if (v < 0x80) break;
  }
  for (int64_t f = frag_base[p]; f < frag_base[p + 1]; ++f) {
    const int64_t len = frag_out[f];
    block_move(out + pos, scratch + f * kFragStride, len);
    pos += len;
  }
  if (d_written && threadIdx.x == 0) d_written[p] = pos;
}

int64_t max_size(int64_t n) { return 32 + n + n / 6; }

// Argument checks, every one AG_ERR_INVALID before any launch.  *src_end / *dst_end: the bytes the batch spans.
ag_status check_compress(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, const uint8_t* dst,
                         int64_t* src_end, int64_t* dst_end) {
  *src_end = *dst_end = 0;
  if (n_pages < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative page count", kFn);
  if (n_pages == 0) return AG_OK;
  if (!pages) AG_FAIL(AG_ERR_INVALID, "%s: NULL page table", kFn);
  if (n_pages > 0x7fffffff) AG_FAIL(AG_ERR_INVALID, "%s: more than 2^31-1 pages", kFn);
  for (int64_t i = 0; i < n_pages; ++i) {
    const ag_pq_compressed& g = pages[i];
    if (g.src < 0 || g.src_len < 0 || g.dst < 0 || g.dst_len < 0)
      AG_FAIL(AG_ERR_INVALID, "%s: page %lld: negative field", kFn, (long long)i);
    if (g.src_len > 0xffffffffLL)
      AG_FAIL(AG_ERR_INVALID, "%s: page %lld: more than 2^32-1 bytes of input", kFn, (long long)i);
    if (g.dst_len < max_size(g.src_len))
      AG_FAIL(AG_ERR_INVALID, "%s: page %lld: capacity %lld below the bound %lld", kFn, (long long)i, (long long)g.dst_len,
              (long long)max_size(g.src_len));
    *src_end = std::max(*src_end, g.src + g.src_len);
    *dst_end = std::max(*dst_end, g.dst + g.dst_len);
  }
  AG_TRY(pq_dst_overlap_check(kFn, pages, n_pages));
  if (*src_end > 0 && !src) AG_FAIL(AG_ERR_INVALID, "%s: NULL input", kFn);
  if (!dst) AG_FAIL(AG_ERR_INVALID, "%s: NULL output", kFn);
  return AG_OK;
}

// Compresses a checked, non-empty batch on `st` without synchronising it: the tables and scratch are stream-ordered.
ag_status snappy_compress_dev(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst, int64_t* d_written,
                              cudaStream_t st) {
  std::vector<SnapFrag> frags;
  std::vector<int64_t> base((size_t)n_pages + 1, 0);
  for (int64_t i = 0; i < n_pages; ++i) {
    for (int64_t s = 0; s < pages[i].src_len; s += kFrag)
      frags.push_back(SnapFrag{pages[i].src + s, std::min<int64_t>(kFrag, pages[i].src_len - s)});
    base[(size_t)i + 1] = (int64_t)frags.size();
  }
  const int64_t n_frags = (int64_t)frags.size();
  TableImage img(st);
  const size_t o_pages = img.add(std::vector<ag_pq_compressed>(pages, pages + n_pages));
  const size_t o_base = img.add(base), o_frags = img.add(frags);
  AG_TRY(img.upload(kFn));
  Carve sc;
  const size_t o_scr = sc.take((size_t)n_frags * kFragStride + 16), o_len = sc.take((size_t)n_frags * 4);
  uint8_t* d = nullptr;
  AG_TRY(dev_alloc_async(reinterpret_cast<void**>(&d), sc.size, st));
  uint8_t* scratch = d + o_scr;
  uint32_t* frag_out = reinterpret_cast<uint32_t*>(d + o_len);
  if (n_frags) {
    snappy_match_kernel<<<(unsigned)((n_frags + kMatchWarps - 1) / kMatchWarps), kMatchWarps * 32, 0, st>>>(
        img.at<SnapFrag>(o_frags), n_frags, src, scratch, frag_out);
    const ag_status rc = check_launch("snappy_match_kernel");
    if (rc != AG_OK) { dev_free_async(d, st); return rc; }
  }
  snappy_assemble_kernel<<<(unsigned)n_pages, kAsmThreads, 0, st>>>(img.at<ag_pq_compressed>(o_pages), img.at<int64_t>(o_base),
                                                                     scratch, frag_out, dst, d_written);
  const ag_status rc = check_launch("snappy_assemble_kernel");
  dev_free_async(d, st);
  return rc;
}

}  // namespace

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_parquet_snappy_max_size(int64_t n, int64_t* size) {
  if (n < 0 || n > 0xffffffffLL) AG_FAIL(AG_ERR_INVALID, "snappy_max_size: %lld bytes outside 0..2^32-1", (long long)n);
  if (!size) AG_FAIL(AG_ERR_INVALID, "snappy_max_size: NULL size");
  *size = max_size(n);
  return AG_OK;
}

ag_status ag_parquet_snappy_compress_dev(const uint8_t* d_src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* d_dst,
                                         int64_t* d_written, ag_stream_t s) {
  AG_TRY(ensure_init());
  int64_t src_end, dst_end;
  AG_TRY(check_compress(d_src, pages, n_pages, d_dst, &src_end, &dst_end));
  if (n_pages == 0) return AG_OK;
  return snappy_compress_dev(d_src, pages, n_pages, d_dst, d_written, resolve_stream(s));
}

ag_status ag_parquet_snappy_compress(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst,
                                     int64_t* written) {
  AG_TRY(ensure_init());
  int64_t src_end, dst_end;
  AG_TRY(check_compress(src, pages, n_pages, dst, &src_end, &dst_end));
  if (n_pages == 0) return AG_OK;
  // stage the input, compress, copy back the written counts and then only the bytes each page wrote
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  Carve sc;
  const size_t o_src = sc.take((size_t)src_end), o_dst = sc.take((size_t)dst_end), o_w = sc.take((size_t)n_pages * 8);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, sc.size));
  AG_TRY(h2d(d + o_src, src, (size_t)src_end, cs));
  int64_t* d_w = reinterpret_cast<int64_t*>(d + o_w);
  AG_TRY(snappy_compress_dev(d + o_src, pages, n_pages, d + o_dst, d_w, cs));
  std::vector<int64_t> w((size_t)n_pages);
  AG_TRY(d2h(w.data(), d_w, (size_t)n_pages * 8, cs));
  AG_TRY(sync(cs));
  for (int64_t i = 0; i < n_pages; ++i) AG_TRY(d2h(dst + pages[i].dst, d + o_dst + pages[i].dst, (size_t)w[i], cs));
  if (written) memcpy(written, w.data(), (size_t)n_pages * 8);
  return sync(cs);
}

}  // extern "C"
