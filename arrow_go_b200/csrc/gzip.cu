// gzip.cu — GZIP decompression (RFC 1952 members, RFC 1951 DEFLATE) of Parquet GZIP pages on the device.
//   serializedPageReader.decompress   parquet/file/page_reader.go:597-621 -> compress.Decode (parquet/compress/compress.go:107)
//                                     -> gzipCodec.DecodeWithError (parquet/compress/gzip.go:51-79)
//
// A call decompresses a batch of pages (ag_pq_compressed descriptors, one device buffer of compressed bytes).  Within a
// page a DEFLATE block starts only where the previous one ends, so the parallelism is the batch.  Three launches:
//   1. gz_inflate_kernel, one warp per page, kWarps pages per block.  Lane 0 walks the member headers and the block
//      headers and decodes every symbol through a 64-bit bit buffer; the warp builds the decode tables of a dynamic
//      block in shared memory (counts per length, canonical first codes, then every lane fills the primary-table
//      entries of its own symbols).  The fixed tables are built once per block.  Literals go to the page's literal
//      scratch at their output position (one kLzLit element per run), a length/distance pair becomes a kLzCopy element,
//      a stored block one kLzSrc element over the compressed bytes.  Per member it records the output range and the
//      stored CRC32 and ISIZE; per page the first decode event.
//   2. lz_exec_kernel, one block per page: the executor shared with every codec (lz_exec.cu).
//   3. gz_crc_kernel, one block per member: every thread CRCs a contiguous 64-byte slice with a table in shared memory;
//      the slice CRCs combine in a tree (a warp by shuffles, then the warps), multiplying by x^(8·len) mod P with one
//      constant per level.  A member whose CRC32 or ISIZE differs sets the page's lowest failing member by atomicMin.
// Roofline.  compressed bytes read + decompressed bytes written.  This design also writes and reads the literals once
// more, 9 B per element, and reads the output once more for the CRC.
#include "lz_exec.cuh"

namespace ag {

namespace {

constexpr const char* kFn = "gzip_decompress";  // message prefix
constexpr int kWarps = 4;                 // pages per block of gz_inflate_kernel
constexpr int kPrim = 10;                 // primary decode-table bits; longer codes decode canonically
constexpr int kNameMax = 512;             // FNAME / FCOMMENT: at most kNameMax - 1 bytes before the NUL
constexpr int kCrcThreads = 256, kCrcSlice = 64, kCrcChunk = kCrcThreads * kCrcSlice;
constexpr int kCrcSplit = 16;             // blocks per page of gz_crc_kernel
constexpr uint32_t kPoly = 0xEDB88320u;   // CRC-32 (IEEE), reflected

// Decode events, in the order of include/arrowgpu.h's list (0 = none).
enum GEvent : int {
  kGOk = 0, kGEof, kGExceed, kGHeader, kGBlockType, kGStored, kGCodeLengths, kGHuffman, kGSymbol, kGDistance
};

struct GMember {                // one member with its trailer read; output offsets within the page
  int64_t out0, out1;
  uint32_t crc, isize;
};

struct GPage {                  // written by gz_inflate_kernel, read by lz_exec_kernel (LzExec::done) and the host
  int64_t written;              // output bytes before the first decode event, at most dst_len
  int64_t nelem;
  int64_t total;                // output bytes of the stream before the first decode event (may pass dst_len by one element)
  int32_t event;                // GEvent
  int32_t nmem;
  int32_t ck_bad;               // lowest member with a CRC32 or ISIZE mismatch (INT32_MAX: none)
  int32_t pad;
};

struct GArgs {
  const ag_pq_compressed* pages;
  const int64_t* lit_base;      // [n_pages + 1] literal scratch bytes
  const int64_t* elem_base;     // execute elements
  const int64_t* mem_base;      // member records
  int64_t n_pages;
  const uint8_t* src;
  const uint8_t* dst;
  GPage* st;
  GMember* mem;
  uint8_t* lit;
  uint32_t* e_out;
  uint32_t* e_ref;
  uint8_t* e_lit;
  int64_t* d_written;           // may be NULL
  uint32_t x2n[32];             // x^(2^k) mod P
  uint32_t slice_shift[9];      // x^(8 · kCrcSlice · 2^k) mod P
};

__constant__ uint16_t c_len_base[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                        31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_len_bits[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dist_base[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                         193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dist_bits[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_clen_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// a · b mod P, polynomials over GF(2) in the reflected representation (x^0 is bit 31)
__host__ __device__ inline uint32_t mulmodp(uint32_t a, uint32_t b) {
  uint32_t p = 0;
  for (uint32_t m = 1u << 31; m; m >>= 1) {
    if (a & m) p ^= b;
    b = (b & 1) ? (b >> 1) ^ kPoly : b >> 1;
  }
  return p;
}

// x^(n · 2^k) mod P
__host__ __device__ inline uint32_t x2nmodp(const uint32_t* x2n, uint64_t n, int k) {
  uint32_t p = 1u << 31;
  for (; n; n >>= 1, ++k)
    if (n & 1) p = mulmodp(x2n[k & 31], p);
  return p;
}

__device__ __forceinline__ uint32_t ld(const uint8_t* p) { return __ldg(p); }

// LSB-first bit reader over in[0, len); bits past len read as zeros (pos > 8 · len is a truncation)
struct BitIn {
  const uint8_t* in;
  int64_t len, pos, base;       // pos: next bit; base: bit position of buf's bit 0 (a multiple of 8, <= pos)
  unsigned long long buf;
  __device__ __forceinline__ void fill() {
    const int64_t b0 = pos >> 3;
    base = b0 << 3;
    unsigned long long v = 0;
    if (b0 + 8 <= len) {
#pragma unroll
      for (int i = 0; i < 8; ++i) v |= (unsigned long long)ld(in + b0 + i) << (8 * i);
    } else {
      for (int i = 0; i < 8 && b0 + i < len; ++i) v |= (unsigned long long)ld(in + b0 + i) << (8 * i);
    }
    buf = v;
  }
  __device__ __forceinline__ uint32_t peek(int n) {              // n <= 32
    if (pos + n > base + 64) fill();
    return (uint32_t)(buf >> (pos - base)) & (uint32_t)((1ull << n) - 1);
  }
  __device__ __forceinline__ uint32_t take(int n) {
    const uint32_t v = peek(n);
    pos += n;
    return v;
  }
  __device__ __forceinline__ bool over() const { return pos > 8 * len; }
};

struct HufT {                   // a canonical Huffman decode table
  uint16_t prim[1 << kPrim];    // the next kPrim bits -> sym | length << 9 (0: no code of <= kPrim bits)
  uint16_t sym[288];            // symbols by (length, symbol)
  uint16_t first[16], count[16], index[16];   // per length: first canonical code, codes, first position in sym
};

struct WarpSmem {
  HufT lit, dist;               // the code-length code is built in `lit` before the literal/length code
  uint8_t lens[320];
  int cnt[16], next[16];
  int ok, nlit, ndist;
};

struct FixedSmem {
  HufT lit, dist;
};

// Builds `t` from lens[0, n) with the whole warp.  A code must be complete; a single code of length 1 is accepted
// (zlib and Go's compress/flate agree), and so is no code at all when `may_be_empty` (a distance code that a block
// never uses).  False on an over-subscribed or incomplete code.
__device__ bool hbuild(const uint8_t* lens, int n, HufT& t, bool may_be_empty, WarpSmem& w) {
  const int lane = threadIdx.x & 31;
  if (lane < 16) w.cnt[lane] = 0;
  for (int i = lane; i < (1 << kPrim); i += 32) t.prim[i] = 0;
  __syncwarp();
  for (int s = lane; s < n; s += 32)
    if (lens[s]) atomicAdd(&w.cnt[lens[s]], 1);
  __syncwarp();
  if (lane == 0) {
    int left = 1, total = 0, code = 0, idx = 0;
    bool ok = true;
    for (int L = 1; L <= 15; ++L) {
      left = 2 * left - w.cnt[L];
      if (left < 0) ok = false;
      code = (code + (L > 1 ? w.cnt[L - 1] : 0)) << 1;
      t.first[L] = (uint16_t)code; t.count[L] = (uint16_t)w.cnt[L]; t.index[L] = (uint16_t)idx;
      w.next[L] = idx;
      idx += w.cnt[L];
      total += w.cnt[L];
    }
    if (ok && left > 0) ok = (total == 1 && w.cnt[1] == 1) || (total == 0 && may_be_empty);
    w.ok = ok;
  }
  __syncwarp();
  if (!w.ok) return false;
  for (int b0 = 0; b0 < n; b0 += 32) {                           // symbols in order: the rank within each length
    const int s = b0 + lane;
    const int L = s < n ? lens[s] : 0;
    const unsigned peers = __match_any_sync(0xffffffffu, L);
    const int at = L ? w.next[L] : 0;
    __syncwarp();
    if (L) {
      const int idx = at + __popc(peers & ((1u << lane) - 1));
      t.sym[idx] = (uint16_t)s;
      if (L <= kPrim) {
        const uint32_t code = t.first[L] + (uint32_t)(idx - t.index[L]);
        for (uint32_t r = __brev(code) >> (32 - L); r < (1u << kPrim); r += 1u << L) t.prim[r] = (uint16_t)(s | L << 9);
      }
      if (lane == __ffs(peers) - 1) w.next[L] = at + __popc(peers);
    }
    __syncwarp();
  }
  return true;
}

// one symbol, or -1 for a bit sequence that is no code (nothing consumed)
__device__ __forceinline__ int hdecode(BitIn& b, const HufT& t) {
  const uint32_t bits = b.peek(15);
  const uint32_t e = t.prim[bits & ((1u << kPrim) - 1)];
  if (e) {
    b.pos += e >> 9;
    return (int)(e & 511);
  }
  uint32_t code = __brev(bits & ((1u << kPrim) - 1)) >> (32 - kPrim);
  for (int L = kPrim + 1; L <= 15; ++L) {
    code = (code << 1) | ((bits >> (L - 1)) & 1);
    const uint32_t c = code - t.first[L];
    if (c < t.count[L]) {
      b.pos += L;
      return t.sym[t.index[L] + c];
    }
  }
  return -1;
}

// Lane 0's walk over one page.  Every emitted element starts below dst_len; a literal byte lands in the literal
// scratch at its output position, so a run's element points at its own first byte.
struct Walk {
  BitIn b;
  int64_t dlen, out, m0, run, ne, ecap, mcap, q;
  int nmem, ev, phase;
  bool in_member, last;
};

__device__ __forceinline__ void emit(const GArgs& a, int64_t eb, Walk& w, int64_t out, uint32_t ref, uint8_t kind) {
  if (out < w.dlen && w.ne < w.ecap) {
    a.e_out[eb + w.ne] = (uint32_t)out; a.e_ref[eb + w.ne] = ref; a.e_lit[eb + w.ne] = kind;
    ++w.ne;
  }
}

__device__ __forceinline__ void close_run(const GArgs& a, int64_t eb, Walk& w) {
  if (w.run >= 0) emit(a, eb, w, w.run, (uint32_t)w.run, kLzLit);
  w.run = -1;
}

// The symbols of one Huffman block up to its end-of-block code; returns a GEvent.
__device__ __forceinline__ int inflate_block(const GArgs& a, int64_t eb, uint8_t* lit, Walk& w, const HufT& lt, const HufT& dt) {
  BitIn b = w.b;
  int64_t out = w.out, run = w.run;
  const int64_t dlen = w.dlen;
  int ev = kGOk;
  while (true) {
    const int sym = hdecode(b, lt);
    if (b.over()) { ev = kGEof; break; }
    if (sym < 0) { ev = kGSymbol; break; }
    if (sym < 256) {
      if (out >= dlen) { ev = kGExceed; break; }
      lit[out] = (uint8_t)sym;
      if (run < 0) run = out;
      ++out;
      continue;
    }
    if (sym == 256) break;
    if (sym >= 286) { ev = kGSymbol; break; }
    const uint32_t len = c_len_base[sym - 257] + b.take(c_len_bits[sym - 257]);
    if (b.over()) { ev = kGEof; break; }
    const int ds = hdecode(b, dt);
    if (b.over()) { ev = kGEof; break; }
    if (ds < 0 || ds >= 30) { ev = kGSymbol; break; }
    const uint32_t dist = c_dist_base[ds] + b.take(c_dist_bits[ds]);
    if (b.over()) { ev = kGEof; break; }
    if ((int64_t)dist > out - w.m0) { ev = kGDistance; break; }
    w.run = run;
    close_run(a, eb, w);
    run = -1;
    emit(a, eb, w, out, dist, kLzCopy);
    out += len;
    if (out > dlen) { ev = kGExceed; break; }
  }
  w.b = b; w.out = out; w.run = run;
  return ev;
}

enum GReq : int { kReqDone = 0, kReqClen, kReqTables };

// Lane 0: runs the walk until it needs the warp to build tables (kReqClen / kReqTables) or the page is done.
__device__ __forceinline__ int walk_step(const GArgs& a, int64_t eb, uint8_t* lit, GMember* M, Walk& w, WarpSmem& s,
                                         const FixedSmem& fx) {
  const uint8_t* in = w.b.in;
  const int64_t len = w.b.len;
  if (w.phase == kReqClen) {                                     // the code-length code is built: the code lengths
    w.phase = 0;
    if (!s.ok) { w.ev = kGHuffman; return kReqDone; }
    const int n = s.nlit + s.ndist;
    int i = 0;
    while (i < n) {
      const int sym = hdecode(w.b, s.lit);
      if (w.b.over()) { w.ev = kGEof; return kReqDone; }
      if (sym < 0) { w.ev = kGCodeLengths; return kReqDone; }
      if (sym < 16) { s.lens[i++] = (uint8_t)sym; continue; }
      int rep, v = 0;
      if (sym == 16) {
        if (i == 0) { w.ev = kGCodeLengths; return kReqDone; }
        v = s.lens[i - 1];
        rep = 3 + (int)w.b.take(2);
      } else if (sym == 17) {
        rep = 3 + (int)w.b.take(3);
      } else {
        rep = 11 + (int)w.b.take(7);
      }
      if (w.b.over()) { w.ev = kGEof; return kReqDone; }
      if (i + rep > n) { w.ev = kGCodeLengths; return kReqDone; }
      for (int k = 0; k < rep; ++k) s.lens[i++] = (uint8_t)v;
    }
    w.phase = kReqTables;
    return kReqTables;
  }
  if (w.phase == kReqTables) {                                   // the literal/length and distance codes are built
    w.phase = 0;
    if (!s.ok) { w.ev = kGHuffman; return kReqDone; }
    w.ev = inflate_block(a, eb, lit, w, s.lit, s.dist);
    if (w.ev) return kReqDone;
  }
  while (true) {
    if (!w.in_member) {                                          // a member header, or the end of the stream
      int64_t q = w.q;
      if (q == len) return kReqDone;
      if (len - q < 10) { w.ev = kGEof; return kReqDone; }
      if (ld(in + q) != 0x1f || ld(in + q + 1) != 0x8b || ld(in + q + 2) != 8) { w.ev = kGHeader; return kReqDone; }
      const uint32_t flg = ld(in + q + 3);
      const int64_t h0 = q;
      q += 10;
      if (flg & 4) {                                             // FEXTRA
        if (len - q < 2) { w.ev = kGEof; return kReqDone; }
        const int64_t xlen = ld(in + q) | ld(in + q + 1) << 8;
        q += 2;
        if (len - q < xlen) { w.ev = kGEof; return kReqDone; }
        q += xlen;
      }
      for (int f = 8; f <= 16; f += 8) {                         // FNAME, FCOMMENT
        if (!(flg & f)) continue;
        for (int i = 0;; ++i, ++q) {
          if (i >= kNameMax) { w.ev = kGHeader; return kReqDone; }
          if (q >= len) { w.ev = kGEof; return kReqDone; }
          if (ld(in + q) == 0) { ++q; break; }
        }
      }
      if (flg & 2) {                                             // FHCRC
        if (len - q < 2) { w.ev = kGEof; return kReqDone; }
        uint32_t c = 0xFFFFFFFFu;
        for (int64_t i = h0; i < q; ++i) {
          c ^= ld(in + i);
          for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ kPoly : c >> 1;
        }
        if (((~c) & 0xFFFF) != (ld(in + q) | ld(in + q + 1) << 8)) { w.ev = kGHeader; return kReqDone; }
        q += 2;
      }
      w.in_member = true; w.last = false;
      w.b.pos = 8 * q;
      w.m0 = w.out;
    }
    if (w.last) {                                                // the trailer, at the next byte boundary
      const int64_t q = (w.b.pos + 7) >> 3;
      if (len - q < 8) { w.ev = kGEof; return kReqDone; }
      if (w.nmem < w.mcap) {
        GMember m;
        m.out0 = w.m0; m.out1 = w.out;
        m.crc = ld(in + q) | ld(in + q + 1) << 8 | ld(in + q + 2) << 16 | ld(in + q + 3) << 24;
        m.isize = ld(in + q + 4) | ld(in + q + 5) << 8 | ld(in + q + 6) << 16 | ld(in + q + 7) << 24;
        M[w.nmem++] = m;
      }
      w.q = q + 8;
      w.in_member = false;
      continue;
    }
    const uint32_t hdr = w.b.take(3);
    if (w.b.over()) { w.ev = kGEof; return kReqDone; }
    w.last = hdr & 1;
    const int type = hdr >> 1;
    if (type == 0) {                                             // stored
      w.b.pos = (w.b.pos + 7) & ~7ll;
      const uint32_t n = w.b.take(16), nn = w.b.take(16);
      if (w.b.over()) { w.ev = kGEof; return kReqDone; }
      if (n != (~nn & 0xFFFF)) { w.ev = kGStored; return kReqDone; }
      if (w.b.pos + 8 * (int64_t)n > 8 * len) { w.ev = kGEof; return kReqDone; }
      if (n > 0) {
        close_run(a, eb, w);
        emit(a, eb, w, w.out, (uint32_t)(w.b.pos >> 3), kLzSrc);
        w.out += n;
        w.b.pos += 8 * (int64_t)n;
        if (w.out > w.dlen) { w.ev = kGExceed; return kReqDone; }
      }
    } else if (type == 1) {                                      // fixed Huffman
      w.ev = inflate_block(a, eb, lit, w, fx.lit, fx.dist);
      if (w.ev) return kReqDone;
    } else if (type == 2) {                                      // dynamic Huffman: HLIT, HDIST, HCLEN, the code-length code
      const uint32_t h = w.b.take(14);
      if (w.b.over()) { w.ev = kGEof; return kReqDone; }
      const int nlit = 257 + (h & 31), ndist = 1 + ((h >> 5) & 31), nclen = 4 + (h >> 10);
      if (nlit > 286 || ndist > 30) { w.ev = kGCodeLengths; return kReqDone; }
      for (int i = 0; i < 19; ++i) s.lens[c_clen_order[i]] = i < nclen ? (uint8_t)w.b.take(3) : 0;
      if (w.b.over()) { w.ev = kGEof; return kReqDone; }
      s.nlit = nlit; s.ndist = ndist;
      w.phase = kReqClen;
      return kReqClen;
    } else {
      w.ev = kGBlockType;
      return kReqDone;
    }
  }
}

__device__ void fixed_lens(uint8_t* lens, bool dist) {
  const int lane = threadIdx.x & 31;
  for (int s = lane; s < 288; s += 32) lens[s] = dist ? 5 : s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
  __syncwarp();
}

__global__ void __launch_bounds__(32 * kWarps)
gz_inflate_kernel(GArgs a) {
  __shared__ WarpSmem sm[kWarps];
  __shared__ FixedSmem fx;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  WarpSmem& s = sm[warp];
  if (warp == 0) {                                               // the fixed codes, once per block
    fixed_lens(s.lens, false);
    hbuild(s.lens, 288, fx.lit, false, s);
    __syncwarp();
    fixed_lens(s.lens, true);
    hbuild(s.lens, 32, fx.dist, false, s);
  }
  __syncthreads();
  const int64_t p = (int64_t)blockIdx.x * kWarps + warp;
  if (p >= a.n_pages) return;
  const ag_pq_compressed pg = a.pages[p];
  const int64_t eb = a.elem_base[p];
  uint8_t* lit = a.lit + a.lit_base[p];
  GMember* M = a.mem + a.mem_base[p];
  Walk w;
  w.b.in = a.src + pg.src; w.b.len = pg.src_len; w.b.pos = 0; w.b.base = -64; w.b.buf = 0;   // base: forces the first fill
  w.dlen = pg.dst_len; w.out = 0; w.m0 = 0; w.run = -1; w.ne = 0; w.q = 0;
  w.ecap = a.elem_base[p + 1] - eb; w.mcap = a.mem_base[p + 1] - a.mem_base[p];
  w.nmem = 0; w.ev = kGOk; w.phase = 0; w.in_member = false; w.last = false;
  while (true) {
    int req = kReqDone;
    if (lane == 0) req = walk_step(a, eb, lit, M, w, s, fx);
    req = __shfl_sync(0xffffffffu, req, 0);
    if (req == kReqDone) break;
    __syncwarp();
    bool ok;
    if (req == kReqClen) ok = hbuild(s.lens, 19, s.lit, false, s);
    else ok = s.lens[256] != 0 && hbuild(s.lens, s.nlit, s.lit, false, s) && hbuild(s.lens + s.nlit, s.ndist, s.dist, true, s);
    if (lane == 0) s.ok = ok;
    __syncwarp();
  }
  if (lane == 0) {
    close_run(a, eb, w);
    GPage ps;
    ps.total = w.out;
    ps.written = w.out < w.dlen ? w.out : w.dlen;
    ps.nelem = w.ne;
    ps.event = w.ev; ps.nmem = w.nmem; ps.ck_bad = INT32_MAX; ps.pad = 0;
    a.st[p] = ps;
    if (a.d_written) a.d_written[p] = ps.written;
  }
}

// CRC32 of every recorded member's output.  The member is read as if left-padded with zeros to whole chunks: zeros
// before the first byte leave a zero CRC register unchanged, so every slice is exactly kCrcSlice bytes and every tree
// level multiplies by one constant.  crc32(M) = x^(8n)·0xFFFFFFFF + R(M) + 0xFFFFFFFF, R the register from zero.
__global__ void __launch_bounds__(kCrcThreads)
gz_crc_kernel(GArgs a) {
  __shared__ uint32_t tab[256];
  __shared__ uint32_t part[kCrcThreads / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  {
    uint32_t c = (uint32_t)t;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ kPoly : c >> 1;
    tab[t] = c;
  }
  __syncthreads();
  const int64_t p = blockIdx.x;
  const int nmem = a.st[p].nmem;
  const GMember* M = a.mem + a.mem_base[p];
  const uint8_t* page = a.dst + a.pages[p].dst;
  for (int m = blockIdx.y; m < nmem; m += gridDim.y) {
    const GMember mb = M[m];
    const uint8_t* d = page + mb.out0;
    const int64_t n = mb.out1 - mb.out0, pad = (kCrcChunk - n % kCrcChunk) % kCrcChunk;
    uint32_t acc = 0;                                            // thread 0's running register over whole chunks
    for (int64_t v0 = 0; v0 < n + pad; v0 += kCrcChunk) {
      const int64_t hi = v0 + (int64_t)(t + 1) * kCrcSlice - pad;
      int64_t i = hi - kCrcSlice;
      if (i < 0) i = 0;
      uint32_t r = 0;
      for (; i < hi; ++i) r = tab[(r ^ __ldg(d + i)) & 255] ^ (r >> 8);
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        const uint32_t o = __shfl_down_sync(0xffffffffu, r, 1 << k);
        if ((lane & ((2 << k) - 1)) == 0) r = mulmodp(a.slice_shift[k], r) ^ o;
      }
      if (lane == 0) part[warp] = r;
      __syncthreads();
      if (t == 0) {
        uint32_t c = part[0];
        for (int k = 1; k < kCrcThreads / 32; ++k) c = mulmodp(a.slice_shift[5], c) ^ part[k];
        acc = mulmodp(a.slice_shift[8], acc) ^ c;
      }
      __syncthreads();
    }
    if (t == 0) {
      const uint32_t crc = mulmodp(x2nmodp(a.x2n, (uint64_t)n, 3), 0xFFFFFFFFu) ^ acc ^ 0xFFFFFFFFu;
      if (crc != mb.crc || (uint32_t)n != mb.isize) atomicMin(&a.st[p].ck_bad, m);
    }
  }
}

const char* const kEventText[] = {"",          "unexpected EOF", "",        "gzip: invalid header", "gzip: block type",
                                  "gzip: stored length", "gzip: code lengths", "gzip: huffman", "gzip: symbol", "gzip: distance"};

// Decompresses a checked, non-empty batch of pages (pq_codec_dev_fn).
ag_status gzip_dev(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst, int64_t* d_written,
                   int64_t* h_written, cudaStream_t st) {
  // plan: pages | three prefix arrays [n+1].  Bounds from the table, per page (sl = src_len, dl = dst_len):
  //   literals   a literal is stored only at an output position below dl: dl bytes;
  //   elements   every element starts below dl at its own position, so at most dl.  Also: copies C <= dl / 3 + 1 (each
  //              produces >= 3 bytes, one may cross dl); a non-empty stored block S takes >= 5 bytes of its own (LEN,
  //              NLEN, a byte), S <= sl / 5; a literal run ends at a copy, a stored block or the end, so runs <= C + S + 1;
  //   members    a member takes >= 20 bytes (10 header, 2 for the shortest block, 8 trailer): sl / 20 + 1.
  const LzPlan<3> plan = lz_plan<3>(pages, n_pages, [](const ag_pq_compressed& g) {
    const int64_t sl = g.src_len, dl = g.dst_len;
    return std::array<int64_t, 3>{dl, std::min(dl, 2 * (dl / 3 + 1) + 2 * (sl / 5) + 1), sl / 20 + 1};
  });
  const int64_t n_lit = plan.total[0], n_elem = plan.total[1], n_mem = plan.total[2];
  Carve sc;
  sc.take(plan.bytes.size());
  const size_t o_st = sc.take((size_t)n_pages * sizeof(GPage)), o_mem = sc.take((size_t)n_mem * sizeof(GMember));
  const size_t o_lit = sc.take((size_t)n_lit);
  const size_t o_eo = sc.take((size_t)n_elem * 4), o_er = sc.take((size_t)n_elem * 4), o_ek = sc.take((size_t)n_elem);
  // this call synchronises `st` anyway, so its device scratch may live in a Temps
  Temps t(st);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, sc.size));
  LzPlanDev<3> pl;
  AG_TRY(lz_upload(plan, d, st, &pl));
  GArgs a;
  a.pages = pl.pages;
  a.lit_base = pl.base[0]; a.elem_base = pl.base[1]; a.mem_base = pl.base[2];
  a.n_pages = n_pages;
  a.src = src; a.dst = dst;
  a.st = reinterpret_cast<GPage*>(d + o_st);
  a.mem = reinterpret_cast<GMember*>(d + o_mem);
  a.lit = d + o_lit;
  a.e_out = reinterpret_cast<uint32_t*>(d + o_eo); a.e_ref = reinterpret_cast<uint32_t*>(d + o_er); a.e_lit = d + o_ek;
  a.d_written = d_written;
  a.x2n[0] = 1u << 30;                                           // x^1
  for (int k = 1; k < 32; ++k) a.x2n[k] = mulmodp(a.x2n[k - 1], a.x2n[k - 1]);
  for (int k = 0; k < 9; ++k) a.slice_shift[k] = x2nmodp(a.x2n, (uint64_t)kCrcSlice << k, 3);
  gz_inflate_kernel<<<(unsigned)((n_pages + kWarps - 1) / kWarps), 32 * kWarps, 0, st>>>(a);
  AG_TRY(check_launch("gz_inflate_kernel"));
  LzExec x;
  x.pages = a.pages; x.elem_base = a.elem_base; x.src = src; x.lit = a.lit; x.lit_base = a.lit_base; x.dst = dst;
  x.done = reinterpret_cast<const int64_t*>(a.st); x.stride = sizeof(GPage) / 8;
  x.e_out = a.e_out; x.e_ref = a.e_ref; x.e_lit = a.e_lit;
  AG_TRY(lz_exec_launch(x, n_pages, st));
  gz_crc_kernel<<<dim3((unsigned)n_pages, kCrcSplit), kCrcThreads, 0, st>>>(a);
  AG_TRY(check_launch("gz_crc_kernel"));
  // The first event in stream order: a member's checksum is checked at its trailer, before anything the walk met after
  // it, so a mismatch wins; then the walk's event; then a clean stream that is short of dst_len.
  return lz_read_back(kFn, a.st, n_pages, h_written, st, [&](int64_t i, const GPage& s, char* buf, size_t n) {
    const int64_t dl = pages[i].dst_len;
    char what[96];
    if (s.ck_bad != INT32_MAX) snprintf(what, sizeof what, "gzip: invalid checksum");
    else if (s.event == kGExceed) snprintf(what, sizeof what, "codec: gzip: decoded data exceeds destination size %lld", (long long)dl);
    else if (s.event != kGOk) snprintf(what, sizeof what, "%s", kEventText[s.event]);
    else if (s.total < dl) snprintf(what, sizeof what, "%s", s.total == 0 ? "EOF" : "unexpected EOF");
    else return;
    snprintf(buf, n, "parquet: could not decompress page: %s", what);
  });
}

}  // namespace

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_parquet_gzip_decompress_dev(const uint8_t* d_src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* d_dst,
                                         int64_t* d_written, ag_stream_t s) {
  AG_TRY(ensure_init());
  return pq_decompress_dev(kFn, gzip_dev, d_src, pages, n_pages, d_dst, d_written, resolve_stream(s));
}

ag_status ag_parquet_gzip_decompress(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst,
                                     int64_t* written) {
  AG_TRY(ensure_init());
  return pq_decompress_host(kFn, gzip_dev, src, pages, n_pages, dst, written);
}

}  // extern "C"
