// zstd.cu — ZSTD decompression (RFC 8878) of Parquet ZSTD pages on the device.
//   serializedPageReader.decompress   parquet/file/page_reader.go:597-621 -> compress.Decode (parquet/compress/compress.go:107)
//                                     -> zstdCodec.DecodeWithError (parquet/compress/zstd.go:115-118), getdecoder (:100-105)
//
// A call decompresses a batch of pages (ag_pq_compressed descriptors, one device buffer of compressed bytes).  The
// parallelism comes from the batch: every zstd block (<= 128 KiB of output) and every Huffman stream is independent
// once the headers are known.  Six launches:
//   1. zstd_walk_kernel, one thread per page: frame headers, zstd-block headers and the literals / sequences section
//      headers, one descriptor per zstd block.  The only dependence between zstd blocks (Treeless literals, Repeat
//      sequence modes) becomes the index of the zstd block whose table description is in effect.  Literal and
//      sequence scratch offsets are assigned here.
//   2. zstd_literals_kernel, one warp per zstd block: builds the Huffman decode table in shared memory from the
//      description in effect, then one lane per stream (1 or 4) decodes the literals into the literal scratch.
//   3. zstd_sequences_kernel, one warp per zstd block: builds the LL / OF / ML decode tables in shared memory (again from
//      the descriptions in effect), then one lane decodes the (literal length, match length, offset value) triples.
//   4. zstd_resolve_kernel, one thread per page: repeat offsets in order within each frame, the offset / literal /
//      block / content-size checks, the first failing zstd block, and the execute elements.
//   5. lz_exec_kernel, one block per page: the executor shared with every codec (lz_exec.cu).
//   6. zstd_xxh64_kernel, one warp per checksummed frame: XXH64 of the frame's output (4 lanes, one per accumulator).
// Roofline.  compressed bytes read + decompressed bytes written.  This design also writes and reads 12 B per sequence,
// 9 B per element (2 per sequence), the Huffman literals once more, and reads each copied byte once more (from L2).
#include "lz_exec.cuh"

namespace ag {

namespace {

constexpr const char* kFn = "zstd_decompress";  // message prefix
constexpr uint32_t kMagic = 0xFD2FB528u;
constexpr uint32_t kBlockMax = 1u << 17;
constexpr int kWarps = 4;              // warps per thread block of the literals / sequences kernels
constexpr int kPageSplit = 16;         // thread blocks per page of those kernels

// Checks, in the order of include/arrowgpu.h's list (0 = none).
enum ZCheck : int {
  kZOk = 0, kZTruncated, kZMagic, kZFrameHeader, kZDictionary, kZBlockType, kZBlockSize, kZLiterals, kZHuffman, kZFse,
  kZSequences, kZOffset, kZContentSize, kZPageSize
};
enum ZErr : int { kZErrNone = 0, kZErrCorrupt = 1, kZErrSize = 2 };

struct ZBlk {                 // one zstd block, page-relative offsets
  uint32_t start;             // first content byte in the page's compressed bytes
  uint32_t size;              // Block_Size (RLE: bytes of output)
  uint32_t end;               // one past the last content byte
  uint32_t lit_off;           // raw literals: their first byte; Huffman: first byte after the literals header
  uint32_t lit_end;           // one past the literals section
  uint32_t regen;             // literals
  uint32_t lit_base;          // Huffman / RLE literals: offset in the page's literal scratch
  uint32_t seq_off;           // first byte after the sequence count and modes byte
  uint32_t nseq;
  uint32_t frame;             // frame index within the page
  int64_t seq_base;           // first triple in the page's sequence scratch
  int32_t huf_from;           // zstd block whose Huffman description is in effect (-1: none)
  int32_t from[3];            // zstd block whose LL / OF / ML table is in effect (-1: none)
  uint8_t type, lit_type, streams, modes;
  uint8_t err_hdr, err_lit, err_seq, lit_stored;
};

struct ZFrame {
  uint32_t first, nblk;       // zstd blocks [first, first + nblk) of the page
  int64_t fcs;                // content size, -1 when absent
  uint64_t window;
  uint32_t ck;                // stored checksum
  int32_t has_ck;             // checksum flag set and checksum read
  int32_t complete;           // the last zstd block was seen
  int32_t verify;             // set by resolve: the frame's output is out and has a checksum to compare
  int64_t out0, out1;         // set by resolve: the frame's output range in the page
};

struct ZPage {                // written by the kernels, read by lz_exec_kernel (LzExec::done) and the host
  int64_t written;
  int64_t nelem;
  int64_t got;                // kZErrSize: the size the frames give
  int32_t err, check;
  int32_t nblk, nframe;
  int32_t walk_fail, walk_check;  // the zstd block the walk stopped at (-1: none)
  int32_t ck_bad;             // lowest frame with a checksum mismatch (INT32_MAX: none)
  int32_t pad;
};

struct ZArgs {
  const ag_pq_compressed* pages;
  const int64_t* blk_base;    // [n_pages + 1] per page: zstd-block descriptors
  const int64_t* frame_base;  // frame descriptors
  const int64_t* lit_base;    // literal scratch bytes
  const int64_t* seq_base;    // sequence triples
  const int64_t* elem_base;   // execute elements
  const uint8_t* src;
  uint8_t* dst;
  ZPage* st;
  ZBlk* blk;
  ZFrame* fr;
  uint8_t* lit;
  uint32_t* s_ll;
  uint32_t* s_ml;
  uint32_t* s_of;
  uint32_t* e_out;
  uint32_t* e_ref;
  uint8_t* e_lit;
  int64_t* d_written;         // may be NULL
};

__constant__ uint32_t c_ll_base[36] = {0,  1,  2,  3,  4,  5,  6,  7,  8,  9,  10,  11,  12,  13,  14,   15,   16,   18,
                                       20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
__constant__ uint8_t c_ll_bits[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1,
                                      1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
__constant__ uint32_t c_ml_base[53] = {3,  4,  5,  6,  7,  8,  9,  10, 11, 12,  13,  14,  15,  16,   17,   18,   19,   20,
                                       21, 22, 23, 24, 25, 26, 27, 28, 29, 30,  31,  32,  33,  34,   35,   37,   39,   41,
                                       43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539};
__constant__ uint8_t c_ml_bits[53] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                                      0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
__constant__ int8_t c_ll_default[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2,
                                        2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
__constant__ int8_t c_of_default[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
__constant__ int8_t c_ml_default[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                        1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
// per symbol type LL, OF, ML: max accuracy log, max symbol, predefined accuracy log
__constant__ int c_max_log[3] = {9, 8, 9};
__constant__ int c_max_sym[3] = {35, 31, 52};
__constant__ int c_def_log[3] = {6, 5, 6};

__device__ __forceinline__ uint32_t ld(const uint8_t* p) { return __ldg(p); }
__device__ __forceinline__ uint32_t le_at(const uint8_t* p, int n) {
  uint32_t v = 0;
  for (int i = 0; i < n; ++i) v |= ld(p + i) << (8 * i);
  return v;
}

// RFC 8878 backward bitstream over buf[0, len): the highest set bit of the last byte is the padding marker.  pos counts
// the bits not yet consumed; bits below 0 read as zeros (pos < 0 is an overflow).
struct BitBack {
  const uint8_t* buf;
  int64_t len, pos, cbase;
  unsigned long long c;
  __device__ bool init(const uint8_t* b, int64_t n) {
    buf = b; len = n; cbase = INT64_MIN / 4; c = 0;
    if (n <= 0) return false;
    const uint32_t last = ld(b + n - 1);
    if (last == 0) return false;
    pos = 8 * (n - 1) + (31 - __clz(last));
    return true;
  }
  __device__ void refill() {
    cbase = (((pos + 7) >> 3) << 3) - 64;
    c = 0;
    const int64_t b0 = cbase >> 3;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int64_t q = b0 + i;
      if (q >= 0 && q < len) c |= (unsigned long long)ld(buf + q) << (8 * i);
    }
  }
  __device__ __forceinline__ uint32_t peek(int n) {
    if (n == 0) return 0;
    const int64_t p = pos - n;
    if (p < cbase || pos > cbase + 64) refill();
    return (uint32_t)((c >> (p - cbase)) & ((1ull << n) - 1));
  }
  __device__ __forceinline__ uint32_t read(int n) {
    const uint32_t v = peek(n);
    pos -= n;
    return v;
  }
};

// bits [pos, pos + n) of buf[0, len), little-endian forward; bytes past len read as zeros
__device__ uint32_t bits_fwd(const uint8_t* buf, int64_t len, int64_t pos, int n) {
  unsigned long long v = 0;
  const int64_t b0 = pos >> 3;
  for (int i = 0; i < 5; ++i)
    if (b0 + i < len) v |= (unsigned long long)ld(buf + b0 + i) << (8 * i);
  return (uint32_t)((v >> (pos & 7)) & ((1ull << n) - 1));
}

struct FseEntry { uint8_t sym, nb; uint16_t base; };

// FSE table description (RFC 8878 4.1.1) -> normalized counts; returns the bytes used or -1
__device__ int read_ncount(const uint8_t* buf, int64_t len, int max_log, int max_sym, int16_t* norm, int* nsym, int* al_out) {
  if (len <= 0) return -1;
  int64_t pos = 0;
  const int al = (int)bits_fwd(buf, len, 0, 4) + 5;
  pos = 4;
  if (al > max_log) return -1;
  int remaining = (1 << al) + 1, threshold = 1 << al, nbits = al + 1, sym = 0;
  bool prev0 = false;
  while (remaining > 1) {
    if (sym > max_sym) return -1;
    if (prev0) {
      int n0 = sym;
      while (bits_fwd(buf, len, pos, 2) == 3) { n0 += 3; pos += 2; if (pos > 8 * len) return -1; }
      n0 += (int)bits_fwd(buf, len, pos, 2);
      pos += 2;
      if (n0 > max_sym) return -1;
      while (sym < n0) norm[sym++] = 0;
      if (pos > 8 * len) return -1;
    }
    const int mx = 2 * threshold - 1 - remaining;
    const int low = (int)bits_fwd(buf, len, pos, nbits - 1);
    int count;
    if (low < mx) {
      count = low;
      pos += nbits - 1;
    } else {
      count = (int)bits_fwd(buf, len, pos, nbits);
      if (count >= threshold) count -= mx;
      pos += nbits;
    }
    count -= 1;
    remaining -= count < 0 ? -count : count;
    norm[sym++] = (int16_t)count;
    prev0 = count == 0;
    if (remaining < threshold) {
      if (remaining <= 1) break;
      nbits = 32 - __clz(remaining);
      threshold = 1 << (nbits - 1);
    }
    if (pos > 8 * len) return -1;
  }
  if (remaining != 1 || pos > 8 * len) return -1;
  *nsym = sym;
  *al_out = al;
  return (int)((pos + 7) >> 3);
}

// decode table of a normalized distribution; false when the spread does not close
__device__ bool fse_build(const int16_t* norm, int nsym, int al, FseEntry* t, uint16_t* next) {
  const int size = 1 << al;
  int high = size - 1;
  for (int s = 0; s < nsym; ++s) {
    if (norm[s] == -1) { t[high--].sym = (uint8_t)s; next[s] = 1; }
    else next[s] = (uint16_t)(norm[s] > 0 ? norm[s] : 0);
  }
  const int step = (size >> 1) + (size >> 3) + 3;
  int pos = 0;
  for (int s = 0; s < nsym; ++s)
    for (int i = 0; i < norm[s]; ++i) {
      t[pos].sym = (uint8_t)s;
      pos = (pos + step) & (size - 1);
      while (pos > high) pos = (pos + step) & (size - 1);
    }
  if (pos != 0) return false;
  for (int u = 0; u < size; ++u) {
    const int s = t[u].sym;
    const int x = next[s]++;
    const int nb = al - (31 - __clz(x));
    t[u].nb = (uint8_t)nb;
    t[u].base = (uint16_t)((x << nb) - size);
  }
  return true;
}

__device__ void fse_default(int k, int16_t* norm, int* nsym, int* al) {
  const int8_t* d = k == 0 ? c_ll_default : k == 1 ? c_of_default : c_ml_default;
  const int n = k == 0 ? 36 : k == 1 ? 29 : 53;
  for (int s = 0; s < n; ++s) norm[s] = d[s];
  *nsym = n;
  *al = c_def_log[k];
}

// ------------------------------------------------------------------------------------------------------------- walk
// One thread per page.  Frame and zstd-block headers, the literals and sequences section headers of compressed blocks.
__global__ void __launch_bounds__(32)
zstd_walk_kernel(ZArgs a) {
  if (threadIdx.x != 0) return;
  const int64_t p = blockIdx.x;
  const ag_pq_compressed pg = a.pages[p];
  const uint8_t* in = a.src + pg.src;
  const int64_t len = pg.src_len, dlen = pg.dst_len;
  ZBlk* B = a.blk + a.blk_base[p];
  ZFrame* F = a.fr + a.frame_base[p];
  const int64_t bcap = a.blk_base[p + 1] - a.blk_base[p], fcap = a.frame_base[p + 1] - a.frame_base[p];
  const int64_t lcap = a.lit_base[p + 1] - a.lit_base[p];
  int64_t seq_room = a.seq_base[p + 1] - a.seq_base[p];
  ZPage ps;
  ps.written = 0; ps.nelem = 0; ps.got = 0; ps.err = kZErrNone; ps.check = kZOk; ps.nblk = 0; ps.nframe = 0;
  ps.walk_fail = -1; ps.walk_check = kZOk; ps.ck_bad = INT32_MAX; ps.pad = 0;
  if (len == 0 && dlen == 0) { a.st[p] = ps; return; }
  int64_t pos = 0, lit_used = 0, seq_used = 0, fcs_sum = 0;
  int nblk = 0, nfr = 0;
  bool all_fcs = true;
  int fail = kZOk;
  while (pos < len && fail == kZOk) {
    if (len - pos < 4) { fail = kZTruncated; break; }
    const uint32_t magic = le_at(in + pos, 4);
    if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) {                   // skippable frame
      if (len - pos < 8 || (uint64_t)(len - pos - 8) < le_at(in + pos + 4, 4)) { fail = kZTruncated; break; }
      pos += 8 + (int64_t)le_at(in + pos + 4, 4);
      continue;
    }
    if (magic != kMagic) { fail = kZMagic; break; }
    pos += 4;
    if (pos >= len) { fail = kZTruncated; break; }
    const uint32_t fhd = ld(in + pos);
    const int fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, ck = (fhd >> 2) & 1, did_flag = fhd & 3;
    if ((fhd >> 3) & 1) { fail = kZFrameHeader; break; }
    const int dsz = did_flag == 3 ? 4 : did_flag;
    const int fsz = fcs_flag == 0 ? single : (2 << (fcs_flag - 1));
    if (pos + 1 + (1 - single) + dsz + fsz > len) { fail = kZTruncated; break; }
    int64_t q = pos + 1;
    uint64_t window = 0;
    if (!single) {
      const uint32_t wd = ld(in + q);
      const int wlog = 10 + (int)(wd >> 3);
      window = (1ull << wlog) + ((1ull << wlog) >> 3) * (wd & 7);
      ++q;
    }
    const uint32_t did = le_at(in + q, dsz);
    q += dsz;
    if (did != 0) { fail = kZDictionary; break; }
    int64_t fcs = -1;
    if (fsz) {
      unsigned long long v = 0;
      for (int i = 0; i < fsz; ++i) v |= (unsigned long long)ld(in + q + i) << (8 * i);
      if (fsz == 2) v += 256;
      fcs = v > (1ull << 62) ? (1ll << 62) : (int64_t)v;         // any larger size fails the same checks
    }
    q += fsz;
    if (single) window = (uint64_t)fcs;
    pos = q;
    const uint32_t bmax = window < kBlockMax ? (uint32_t)window : kBlockMax;
    if (fcs < 0) all_fcs = false; else fcs_sum += fcs;
    ZFrame f;
    f.first = nblk; f.nblk = 0; f.fcs = fcs; f.window = window; f.ck = 0; f.has_ck = 0; f.complete = 0; f.verify = 0;
    f.out0 = f.out1 = 0;
    int last_huf = -1, last_from[3] = {-1, -1, -1};
    while (true) {
      if (pos + 3 > len) { fail = kZTruncated; break; }
      const uint32_t bh = le_at(in + pos, 3);
      const int last = bh & 1, btype = (bh >> 1) & 3;
      const uint32_t bsize = bh >> 3;
      if (btype == 3) { fail = kZBlockType; break; }
      if (bsize > bmax) { fail = kZBlockSize; break; }
      const int64_t stored = btype == 1 ? 1 : bsize;
      if (pos + 3 + stored > len) { fail = kZTruncated; break; }
      if (nblk >= bcap || nfr >= fcap) { fail = kZTruncated; break; }   // not reached: a block takes >= 3 bytes
      ZBlk b;
      memset(&b, 0, sizeof b);
      b.type = (uint8_t)btype; b.start = (uint32_t)(pos + 3); b.size = bsize; b.end = (uint32_t)(pos + 3 + stored);
      b.frame = (uint32_t)nfr; b.huf_from = -1; b.from[0] = b.from[1] = b.from[2] = -1;
      if (btype == 2) {
        // ---- literals section header ----
        const uint8_t* d = in + b.start;
        const int64_t dl = bsize;
        int err = kZOk;
        int lt = 0, sf = 0, hl = 0, ns = 0;
        uint32_t regen = 0, comp = 0;
        if (dl < 1) err = kZLiterals;
        else {
          const uint32_t b0 = ld(d);
          lt = b0 & 3; sf = (b0 >> 2) & 3;
          if (lt < 2) {
            if (sf == 0 || sf == 2) { regen = b0 >> 3; hl = 1; }
            else if (sf == 1) { if (dl < 2) err = kZLiterals; else { regen = (b0 >> 4) + (ld(d + 1) << 4); hl = 2; } }
            else { if (dl < 3) err = kZLiterals; else { regen = (b0 >> 4) + (ld(d + 1) << 4) + (ld(d + 2) << 12); hl = 3; } }
          } else {
            hl = sf == 0 || sf == 1 ? 3 : sf == 2 ? 4 : 5;
            if (dl < hl) err = kZLiterals;
            else {
              unsigned long long v = 0;
              for (int i = 0; i < hl; ++i) v |= (unsigned long long)ld(d + i) << (8 * i);
              const int bits = sf <= 1 ? 10 : sf == 2 ? 14 : 18;
              regen = (uint32_t)((v >> 4) & ((1u << bits) - 1));
              comp = (uint32_t)(v >> (4 + bits));
              ns = sf == 0 ? 1 : 4;
            }
          }
        }
        int64_t lend = 0;
        if (err == kZOk) {
          if (regen > kBlockMax) err = kZLiterals;
          lend = lt == 0 ? hl + (int64_t)regen : lt == 1 ? hl + 1 : hl + (int64_t)comp;
          if (lt >= 2 && ns == 4 && regen < 6) err = kZLiterals;
          if (lend > dl) err = kZLiterals;
        }
        // ---- sequences section header ----
        uint32_t nseq = 0;
        int modes = 0;
        int64_t s = lend;
        if (err == kZOk) {
          if (s >= dl) err = kZSequences;
          else {
            const uint32_t c0 = ld(d + s);
            if (c0 < 128) { nseq = c0; s += 1; }
            else if (c0 < 255) { if (s + 2 > dl) err = kZSequences; else { nseq = ((c0 - 128) << 8) + ld(d + s + 1); s += 2; } }
            else { if (s + 3 > dl) err = kZSequences; else { nseq = ld(d + s + 1) + (ld(d + s + 2) << 8) + 0x7F00; s += 3; } }
          }
          if (err == kZOk) {
            if (nseq == 0) {
              if (s != dl) err = kZSequences;
            } else {
              if (s >= dl) err = kZSequences;
              else {
                modes = (int)ld(d + s);
                if (modes & 3) err = kZSequences;
                s += 1;
                if (err == kZOk && (int64_t)nseq > seq_room) err = kZSequences;
              }
            }
          }
        }
        b.err_hdr = (uint8_t)err;
        if (err == kZOk) {
          b.lit_type = (uint8_t)lt; b.streams = (uint8_t)ns; b.regen = regen;
          b.lit_off = b.start + (uint32_t)hl; b.lit_end = b.start + (uint32_t)lend;
          b.nseq = nseq; b.modes = (uint8_t)modes; b.seq_off = b.start + (uint32_t)s;
          if (lt >= 1) {
            b.lit_base = (uint32_t)(lit_used < lcap ? lit_used : lcap);
            b.lit_stored = lit_used + (int64_t)regen <= lcap;
            lit_used += regen;
          }
          if (lt == 2) last_huf = nblk;
          if (lt >= 2) b.huf_from = lt == 2 ? nblk : last_huf;
          if (nseq > 0) {
            for (int k = 0; k < 3; ++k) {
              const int m = (modes >> (6 - 2 * k)) & 3;
              b.from[k] = m == 3 ? last_from[k] : nblk;
              last_from[k] = b.from[k];
            }
            b.seq_base = seq_used;
            seq_used += nseq;
            seq_room -= nseq;
          }
        }
      }
      B[nblk] = b;
      ++nblk; ++f.nblk;
      pos += 3 + stored;
      if (last) { f.complete = 1; break; }
    }
    if (fail == kZOk && ck) {
      if (pos + 4 > len) fail = kZTruncated;
      else { f.ck = le_at(in + pos, 4); f.has_ck = 1; pos += 4; }
    }
    if (f.nblk > 0) F[nfr++] = f;
  }
  ps.nblk = nblk; ps.nframe = nfr;
  if (fail != kZOk) { ps.walk_fail = nblk; ps.walk_check = fail; }
  else if (all_fcs && fcs_sum != dlen) { ps.err = kZErrSize; ps.got = fcs_sum; }
  a.st[p] = ps;
}

// ---------------------------------------------------------------------------------------------------------- literals
struct HufSmem {
  uint16_t table[1 << 11];    // sym | nbits << 8
  uint8_t w[256];
  uint16_t start[256];
  int max_bits, nsym, used, err;
  int16_t norm[256];
  FseEntry ft[64];
  uint16_t next[256];
};

// Huffman tree description at d[0, len) -> table; lane 0 parses, the warp fills.  Returns the bytes used or -1.
__device__ int huf_build(const uint8_t* d, int64_t len, HufSmem& h) {
  const int lane = threadIdx.x & 31;
  if (lane == 0) {
    int err = 0, n = 0, used = 0;
    if (len < 1) err = 1;
    const uint32_t hb = err ? 0 : ld(d);
    if (!err && hb < 128) {
      if (1 + (int64_t)hb > len) err = 1;
      int nsym = 0, al = 0, u = -1;
      if (!err) u = read_ncount(d + 1, hb, 6, 255, h.norm, &nsym, &al);
      if (u < 0 || !fse_build(h.norm, nsym, al, h.ft, h.next)) err = 1;
      BitBack bb;
      if (!err && !bb.init(d + 1 + u, (int64_t)hb - u)) err = 1;
      if (!err) {
        uint32_t s1 = bb.read(al), s2 = bb.read(al);
        while (true) {
          if (n > 253) { err = 1; break; }
          h.w[n++] = h.ft[s1].sym;
          s1 = h.ft[s1].base + bb.read(h.ft[s1].nb);
          if (bb.pos < 0) { h.w[n++] = h.ft[s2].sym; break; }
          if (n > 253) { err = 1; break; }
          h.w[n++] = h.ft[s2].sym;
          s2 = h.ft[s2].base + bb.read(h.ft[s2].nb);
          if (bb.pos < 0) { h.w[n++] = h.ft[s1].sym; break; }
        }
      }
      used = 1 + (int)hb;
    } else if (!err) {
      n = (int)hb - 127;
      used = 1 + (n + 1) / 2;
      if (used > len) err = 1;
      for (int i = 0; i < n && !err; ++i) {
        const uint32_t b = ld(d + 1 + i / 2);
        h.w[i] = (uint8_t)((i & 1) ? b & 15 : b >> 4);
      }
    }
    uint32_t total = 0;
    for (int i = 0; i < n && !err; ++i) {
      if (h.w[i] > 11) err = 1;
      else if (h.w[i]) total += 1u << (h.w[i] - 1);
    }
    int mb = 0;
    if (!err) {
      if (total == 0) err = 1;
      else {
        mb = 32 - __clz(total);
        const uint32_t rest = (1u << mb) - total;
        if (mb > 11 || (rest & (rest - 1))) err = 1;
        else h.w[n++] = (uint8_t)(32 - __clz(rest));
      }
    }
    if (!err) {
      int ones = 0;
      for (int i = 0; i < n; ++i) ones += h.w[i] == 1;
      if (ones < 2 || (ones & 1)) err = 1;
    }
    if (!err) {                                                   // canonical order: weight ascending, then symbol
      uint32_t rank[13] = {0};
      for (int i = 0; i < n; ++i) if (h.w[i]) rank[h.w[i]] += 1u << (h.w[i] - 1);
      uint32_t acc = 0;
      for (int wt = 1; wt <= 12; ++wt) { const uint32_t c = rank[wt]; rank[wt] = acc; acc += c; }
      for (int i = 0; i < n; ++i)
        if (h.w[i]) { h.start[i] = (uint16_t)rank[h.w[i]]; rank[h.w[i]] += 1u << (h.w[i] - 1); }
    }
    h.err = err; h.max_bits = mb; h.nsym = n; h.used = used;
  }
  __syncwarp();
  if (h.err) return -1;
  const int mb = h.max_bits, n = h.nsym;
  for (int i = 0; i < n; ++i) {
    const int wt = h.w[i];
    if (!wt) continue;
    const uint16_t e = (uint16_t)(i | (mb + 1 - wt) << 8);
    for (int j = lane; j < (1 << (wt - 1)); j += 32) h.table[h.start[i] + j] = e;
  }
  __syncwarp();
  return h.used;
}

// one Huffman stream: n symbols, consumed exactly
__device__ bool huf_stream(const uint8_t* d, int64_t len, int64_t n, const HufSmem& h, uint8_t* out) {
  BitBack bb;
  if (!bb.init(d, len)) return false;
  const int mb = h.max_bits;
  for (int64_t i = 0; i < n; ++i) {
    const uint16_t e = h.table[bb.peek(mb)];
    if (out) out[i] = (uint8_t)(e & 255);
    bb.pos -= e >> 8;
    if (bb.pos < 0) return false;
  }
  return bb.pos == 0;
}

__global__ void __launch_bounds__(32 * kWarps)
zstd_literals_kernel(ZArgs a) {
  __shared__ HufSmem sm[kWarps];
  __shared__ int ok[kWarps][4];
  const int64_t p = blockIdx.x;
  const ZPage ps = a.st[p];
  if (ps.err != kZErrNone) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  HufSmem& h = sm[warp];
  const uint8_t* in = a.src + a.pages[p].src;
  ZBlk* B = a.blk + a.blk_base[p];
  uint8_t* lit = a.lit + a.lit_base[p];
  for (int i = blockIdx.y * kWarps + warp; i < ps.nblk; i += gridDim.y * kWarps) {
    const ZBlk b = B[i];
    if (b.type != 2 || b.err_hdr || b.lit_type == 0) continue;
    if (b.lit_type == 1) {
      if (b.lit_stored) {
        const uint8_t v = (uint8_t)ld(in + b.lit_off);
        for (uint32_t j = lane; j < b.regen; j += 32) lit[b.lit_base + j] = v;
      }
      continue;
    }
    int err = 0;
    int64_t body = b.lit_off;
    if (b.huf_from < 0) err = 1;
    else {
      const ZBlk& t = B[b.huf_from];
      const int used = huf_build(in + t.lit_off, (int64_t)t.lit_end - t.lit_off, h);
      if (used < 0) err = 1;
      else if (b.lit_type == 2) body += used;
    }
    if (!err) {
      const int64_t blen = (int64_t)b.lit_end - body;
      uint8_t* out = b.lit_stored ? lit + b.lit_base : nullptr;
      if (b.streams == 1) {
        if (lane == 0) ok[warp][0] = huf_stream(in + body, blen, b.regen, h, out);
        __syncwarp();
        err = !ok[warp][0];
      } else {
        if (blen < 6) err = 1;
        else {
          const uint8_t* jt = in + body;
          const int64_t s0 = le_at(jt, 2), s1 = le_at(jt + 2, 2), s2 = le_at(jt + 4, 2);
          const int64_t s3 = blen - 6 - s0 - s1 - s2;
          if (s3 < 0) err = 1;
          else {
            const int64_t seg = ((int64_t)b.regen + 3) / 4;
            if (lane < 4) {
              const int64_t off = 6 + (lane > 0 ? s0 : 0) + (lane > 1 ? s1 : 0) + (lane > 2 ? s2 : 0);
              const int64_t sl = lane == 0 ? s0 : lane == 1 ? s1 : lane == 2 ? s2 : s3;
              const int64_t cnt = lane < 3 ? seg : (int64_t)b.regen - 3 * seg;
              ok[warp][lane] = huf_stream(jt + off, sl, cnt, h, out ? out + lane * seg : nullptr);
            }
            __syncwarp();
            err = !(ok[warp][0] && ok[warp][1] && ok[warp][2] && ok[warp][3]);
          }
        }
      }
    }
    if (lane == 0 && err) B[i].err_lit = kZHuffman;
    __syncwarp();
  }
}

// --------------------------------------------------------------------------------------------------------- sequences
struct SeqSmem {
  FseEntry t[3][512];
  int16_t norm[64];
  uint16_t next[64];
  int al[3];
};

// builds symbol type k's table from the description of block `b` at cursor *cur (mode m); false on a bad description
__device__ int seq_table(const uint8_t* in, const ZBlk& b, int k, int m, int64_t* cur, SeqSmem& s) {
  if (m == 0) {
    int nsym, al;
    fse_default(k, s.norm, &nsym, &al);
    fse_build(s.norm, nsym, al, s.t[k], s.next);
    s.al[k] = al;
    return kZOk;
  }
  if (m == 1) {
    if (*cur >= b.end) return kZSequences;
    const uint32_t sym = ld(in + *cur);
    if ((int)sym > c_max_sym[k]) return kZSequences;
    s.t[k][0].sym = (uint8_t)sym; s.t[k][0].nb = 0; s.t[k][0].base = 0;
    s.al[k] = 0;
    *cur += 1;
    return kZOk;
  }
  int nsym, al;
  const int used = read_ncount(in + *cur, (int64_t)b.end - *cur, c_max_log[k], c_max_sym[k], s.norm, &nsym, &al);
  if (used < 0 || *cur + used > b.end) return kZFse;
  if (!fse_build(s.norm, nsym, al, s.t[k], s.next)) return kZFse;
  s.al[k] = al;
  *cur += used;
  return kZOk;
}

// the description of symbol type k in block b (whose mode for k is not Repeat): skip the ones before it, build it
__device__ int seq_table_from(const uint8_t* in, const ZBlk& b, int k, SeqSmem& s) {
  int64_t cur = b.seq_off;
  for (int j = 0; j < k; ++j) {
    const int m = (b.modes >> (6 - 2 * j)) & 3;
    if (m == 1) cur += 1;
    else if (m == 2) {
      int nsym, al;
      const int used = read_ncount(in + cur, (int64_t)b.end - cur, c_max_log[j], c_max_sym[j], s.norm, &nsym, &al);
      if (used < 0) return kZFse;
      cur += used;
    }
  }
  return seq_table(in, b, k, (b.modes >> (6 - 2 * k)) & 3, &cur, s);
}

__global__ void __launch_bounds__(32 * kWarps)
zstd_sequences_kernel(ZArgs a) {
  __shared__ SeqSmem sm[kWarps];
  const int64_t p = blockIdx.x;
  const ZPage ps = a.st[p];
  if (ps.err != kZErrNone) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane != 0) return;
  SeqSmem& s = sm[warp];
  const uint8_t* in = a.src + a.pages[p].src;
  ZBlk* B = a.blk + a.blk_base[p];
  const int64_t sb = a.seq_base[p];
  for (int i = blockIdx.y * kWarps + warp; i < ps.nblk; i += gridDim.y * kWarps) {
    const ZBlk b = B[i];
    if (b.type != 2 || b.err_hdr || b.nseq == 0) continue;
    int err = kZOk;
    int64_t cur = b.seq_off;
    for (int k = 0; k < 3 && err == kZOk; ++k) {
      const int m = (b.modes >> (6 - 2 * k)) & 3;
      if (m != 3) err = seq_table(in, b, k, m, &cur, s);
      else if (b.from[k] < 0) err = kZSequences;
      else err = seq_table_from(in, B[b.from[k]], k, s);
    }
    BitBack bb;
    if (err == kZOk && !bb.init(in + cur, (int64_t)b.end - cur)) err = kZSequences;
    if (err == kZOk) {
      uint32_t stl = bb.read(s.al[0]), sto = bb.read(s.al[1]), stm = bb.read(s.al[2]);
      uint32_t* ll = a.s_ll + sb + b.seq_base;
      uint32_t* ml = a.s_ml + sb + b.seq_base;
      uint32_t* of = a.s_of + sb + b.seq_base;
      for (uint32_t q = 0; q < b.nseq; ++q) {
        const FseEntry el = s.t[0][stl], eo = s.t[1][sto], em = s.t[2][stm];
        const int ofc = eo.sym;
        const uint32_t ofv = (1u << ofc) + bb.read(ofc);
        const uint32_t mlv = c_ml_base[em.sym] + bb.read(c_ml_bits[em.sym]);
        const uint32_t llv = c_ll_base[el.sym] + bb.read(c_ll_bits[el.sym]);
        ll[q] = llv; ml[q] = mlv; of[q] = ofv;
        if (q + 1 < b.nseq) {
          stl = el.base + bb.read(el.nb);
          stm = em.base + bb.read(em.nb);
          sto = eo.base + bb.read(eo.nb);
        }
        if (bb.pos < 0) { err = kZSequences; break; }
      }
      if (err == kZOk && bb.pos != 0) err = kZSequences;
    }
    if (err) B[i].err_seq = (uint8_t)err;
  }
}

// ----------------------------------------------------------------------------------------------------------- resolve
// One thread per page: the zstd blocks in order.  Repeat offsets, the execution checks, the first failing block, the
// execute elements (only those ending at or before dst_len).
__global__ void __launch_bounds__(32)
zstd_resolve_kernel(ZArgs a) {
  if (threadIdx.x != 0) return;
  const int64_t p = blockIdx.x;
  ZPage ps = a.st[p];
  const ag_pq_compressed pg = a.pages[p];
  const int64_t dlen = pg.dst_len;
  if (ps.err != kZErrNone || (pg.src_len == 0 && dlen == 0)) {
    if (a.d_written) a.d_written[p] = 0;
    return;
  }
  const ZBlk* B = a.blk + a.blk_base[p];
  ZFrame* F = a.fr + a.frame_base[p];
  const int64_t eb = a.elem_base[p], ecap = a.elem_base[p + 1] - eb, sb = a.seq_base[p];
  int64_t pos = 0, ne = 0;
  int fail = -1, check = kZOk, over = -1;
  int64_t over_pos = 0, over_ne = 0;
  auto emit = [&](int64_t out, int64_t n, uint32_t ref, uint8_t kind) {
    if (n > 0 && out + n <= dlen && ne < ecap) {
      a.e_out[eb + ne] = (uint32_t)out; a.e_ref[eb + ne] = ref; a.e_lit[eb + ne] = kind;
      ++ne;
    }
  };
  for (int fi = 0; fi < ps.nframe && fail < 0; ++fi) {
    ZFrame f = F[fi];
    const int64_t f0 = pos;
    const uint64_t bmax = f.window < kBlockMax ? f.window : kBlockMax;
    uint32_t rep0 = 1, rep1 = 4, rep2 = 8;
    for (uint32_t bi = 0; bi < f.nblk; ++bi) {
      const int k = (int)(f.first + bi);
      const ZBlk b = B[k];
      const int64_t start = pos, ne0 = ne;
      int err = b.err_hdr ? b.err_hdr : b.err_lit ? b.err_lit : b.err_seq;
      if (!err) {
        if (b.type == 0) {
          emit(pos, b.size, b.start, kLzSrc);
          pos += b.size;
        } else if (b.type == 1) {
          emit(pos, b.size > 0 ? 1 : 0, b.start, kLzSrc);
          emit(pos + 1, (int64_t)b.size - 1, 1, kLzCopy);
          pos += b.size;
        } else {
          const uint32_t* ll = a.s_ll + sb + b.seq_base;
          const uint32_t* ml = a.s_ml + sb + b.seq_base;
          const uint32_t* of = a.s_of + sb + b.seq_base;
          const uint8_t lk = b.lit_type == 0 ? kLzSrc : kLzLit;
          const uint32_t lref = b.lit_type == 0 ? b.lit_off : b.lit_base;
          uint32_t lp = 0;
          for (uint32_t q = 0; q < b.nseq; ++q) {
            const uint32_t l = ll[q], m = ml[q], v = of[q];
            if ((uint64_t)lp + l > b.regen) { err = kZSequences; break; }
            emit(pos, l, lref + lp, lk);
            pos += l; lp += l;
            uint32_t off;
            if (v > 3) {
              off = v - 3; rep2 = rep1; rep1 = rep0; rep0 = off;
            } else {
              const uint32_t idx = v - 1 + (l == 0);
              if (idx == 0) off = rep0;
              else if (idx == 1) { off = rep1; rep1 = rep0; rep0 = off; }
              else if (idx == 2) { off = rep2; rep2 = rep1; rep1 = rep0; rep0 = off; }
              else { off = rep0 - 1; rep2 = rep1; rep1 = rep0; rep0 = off; }
            }
            if (off == 0 || (int64_t)off > pos - f0 || (uint64_t)off > f.window) { err = kZOffset; break; }
            emit(pos, m, off, kLzCopy);
            pos += m;
          }
          if (!err) {
            emit(pos, (int64_t)b.regen - lp, lref + lp, lk);
            pos += (int64_t)b.regen - lp;
            if ((uint64_t)(pos - start) > bmax) err = kZBlockSize;
          }
        }
      }
      if (!err && f.fcs >= 0 && (pos - f0 > f.fcs || (f.complete && bi + 1 == f.nblk && pos - f0 != f.fcs))) err = kZContentSize;
      if (err) { fail = k; check = err; pos = start; ne = ne0; break; }
      if (over < 0 && pos > dlen) { over = k; over_pos = start; over_ne = ne0; }
    }
    if (fail >= 0) break;
    F[fi].out0 = f0; F[fi].out1 = pos;
    F[fi].verify = f.has_ck;
  }
  if (fail < 0 && ps.walk_fail >= 0) { fail = ps.walk_fail; check = ps.walk_check; }
  if (fail < 0) {
    if (pos != dlen) { ps.err = kZErrSize; ps.got = pos; ps.written = 0; ps.nelem = 0; }
    else { ps.written = pos; ps.nelem = ne; }
  } else {
    ps.err = kZErrCorrupt; ps.check = check;
    if (over >= 0 && over < fail) { ps.check = kZPageSize; ps.written = over_pos; ps.nelem = over_ne; }
    else { ps.written = pos; ps.nelem = ne; }
  }
  if (ps.err == kZErrSize) for (int fi = 0; fi < ps.nframe; ++fi) F[fi].verify = 0;
  else for (int fi = 0; fi < ps.nframe; ++fi) if (F[fi].verify && F[fi].out1 > ps.written) F[fi].verify = 0;
  a.st[p] = ps;
  if (a.d_written) a.d_written[p] = ps.written;
}

// ------------------------------------------------------------------------------------------------------------- xxh64
constexpr unsigned long long kP1 = 11400714785074694791ull, kP2 = 14029467366897019727ull, kP3 = 1609587929392839161ull,
                             kP4 = 9650029242287828579ull, kP5 = 2870177450012600261ull;
__device__ __forceinline__ unsigned long long rotl64(unsigned long long x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ unsigned long long xround(unsigned long long acc, unsigned long long v) {
  return rotl64(acc + v * kP2, 31) * kP1;
}
__device__ __forceinline__ unsigned long long ld64(const uint8_t* p) {
  unsigned long long v = 0;
  for (int i = 0; i < 8; ++i) v |= (unsigned long long)p[i] << (8 * i);
  return v;
}

// One warp per frame that has a checksum to compare: lanes 0..3 own the four accumulators (sequential by definition).
__global__ void __launch_bounds__(32 * kWarps)
zstd_xxh64_kernel(ZArgs a) {
  const int64_t p = blockIdx.x;
  const ZPage ps = a.st[p];
  if (ps.err == kZErrSize) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const ZFrame* F = a.fr + a.frame_base[p];
  const uint8_t* out = a.dst + a.pages[p].dst;
  for (int fi = blockIdx.y * kWarps + warp; fi < ps.nframe; fi += gridDim.y * kWarps) {
    const ZFrame f = F[fi];
    if (!f.verify) continue;
    const uint8_t* d = out + f.out0;
    const int64_t n = f.out1 - f.out0, stripes = n / 32;
    unsigned long long v = 0;
    if (lane < 4) {
      v = lane == 0 ? kP1 + kP2 : lane == 1 ? kP2 : lane == 2 ? 0ull : 0ull - kP1;
      for (int64_t s = 0; s < stripes; ++s) v = xround(v, ld64(d + 32 * s + 8 * lane));
    }
    const unsigned long long v0 = __shfl_sync(0xffffffffu, v, 0), v1 = __shfl_sync(0xffffffffu, v, 1),
                             v2 = __shfl_sync(0xffffffffu, v, 2), v3 = __shfl_sync(0xffffffffu, v, 3);
    if (lane == 0) {
      unsigned long long h;
      if (n >= 32) {
        h = rotl64(v0, 1) + rotl64(v1, 7) + rotl64(v2, 12) + rotl64(v3, 18);
        h = (h ^ xround(0, v0)) * kP1 + kP4;
        h = (h ^ xround(0, v1)) * kP1 + kP4;
        h = (h ^ xround(0, v2)) * kP1 + kP4;
        h = (h ^ xround(0, v3)) * kP1 + kP4;
      } else {
        h = kP5;
      }
      h += (unsigned long long)n;
      int64_t i = stripes * 32;
      for (; i + 8 <= n; i += 8) h = rotl64(h ^ xround(0, ld64(d + i)), 27) * kP1 + kP4;
      if (i + 4 <= n) {
        const unsigned long long w = (unsigned long long)d[i] | (unsigned long long)d[i + 1] << 8 |
                                     (unsigned long long)d[i + 2] << 16 | (unsigned long long)d[i + 3] << 24;
        h = rotl64(h ^ (w * kP1), 23) * kP2 + kP3;
        i += 4;
      }
      for (; i < n; ++i) h = rotl64(h ^ ((unsigned long long)d[i] * kP5), 11) * kP1;
      h ^= h >> 33; h *= kP2; h ^= h >> 29; h *= kP3; h ^= h >> 32;
      if ((uint32_t)h != f.ck) atomicMin(&a.st[p].ck_bad, fi);
    }
  }
}

const char* const kCheckName[] = {"", "truncated", "bad magic", "frame header", "dictionary", "block type", "block size", "literals",
                                  "huffman", "fse", "sequences", "offset", "content size", "page size"};

// Decompresses a checked, non-empty batch of pages (pq_codec_dev_fn).
ag_status zstd_dev(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst, int64_t* d_written,
                   int64_t* h_written, cudaStream_t st) {
  // plan: pages | five prefix arrays [n+1].  Bounds from the table: a zstd block takes >= 3 compressed bytes, a frame
  // >= 8; a sequence produces >= 3 output bytes; literals are output bytes; an element produces >= 1 output byte and
  // there are at most 2 per sequence and 2 per zstd block.
  const LzPlan<5> plan = lz_plan<5>(pages, n_pages, [](const ag_pq_compressed& g) {
    const int64_t sl = g.src_len, dl = g.dst_len;
    return std::array<int64_t, 5>{sl / 3, sl / 8, dl, dl / 3, std::min(dl, 2 * (dl / 3) + 2 * (sl / 3))};
  });
  const int64_t n_blk = plan.total[0], n_frame = plan.total[1], n_lit = plan.total[2], n_seq = plan.total[3], n_elem = plan.total[4];
  Carve sc;
  sc.take(plan.bytes.size());
  const size_t o_st = sc.take((size_t)n_pages * sizeof(ZPage)), o_blk = sc.take((size_t)n_blk * sizeof(ZBlk));
  const size_t o_fr = sc.take((size_t)n_frame * sizeof(ZFrame)), o_lit = sc.take((size_t)n_lit);
  const size_t o_ll = sc.take((size_t)n_seq * 4), o_ml = sc.take((size_t)n_seq * 4), o_of = sc.take((size_t)n_seq * 4);
  const size_t o_eo = sc.take((size_t)n_elem * 4), o_er = sc.take((size_t)n_elem * 4), o_ek = sc.take((size_t)n_elem);
  // this call synchronises `st` anyway, so its device scratch may live in a Temps
  Temps t(st);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, sc.size));
  LzPlanDev<5> pl;
  AG_TRY(lz_upload(plan, d, st, &pl));
  ZArgs a;
  a.pages = pl.pages;
  a.blk_base = pl.base[0]; a.frame_base = pl.base[1]; a.lit_base = pl.base[2]; a.seq_base = pl.base[3]; a.elem_base = pl.base[4];
  a.src = src; a.dst = dst;
  a.st = reinterpret_cast<ZPage*>(d + o_st);
  a.blk = reinterpret_cast<ZBlk*>(d + o_blk);
  a.fr = reinterpret_cast<ZFrame*>(d + o_fr);
  a.lit = d + o_lit;
  a.s_ll = reinterpret_cast<uint32_t*>(d + o_ll); a.s_ml = reinterpret_cast<uint32_t*>(d + o_ml); a.s_of = reinterpret_cast<uint32_t*>(d + o_of);
  a.e_out = reinterpret_cast<uint32_t*>(d + o_eo); a.e_ref = reinterpret_cast<uint32_t*>(d + o_er); a.e_lit = d + o_ek;
  a.d_written = d_written;
  const dim3 split((unsigned)n_pages, kPageSplit);
  zstd_walk_kernel<<<(unsigned)n_pages, 32, 0, st>>>(a);
  AG_TRY(check_launch("zstd_walk_kernel"));
  zstd_literals_kernel<<<split, 32 * kWarps, 0, st>>>(a);
  AG_TRY(check_launch("zstd_literals_kernel"));
  zstd_sequences_kernel<<<split, 32 * kWarps, 0, st>>>(a);
  AG_TRY(check_launch("zstd_sequences_kernel"));
  zstd_resolve_kernel<<<(unsigned)n_pages, 32, 0, st>>>(a);
  AG_TRY(check_launch("zstd_resolve_kernel"));
  LzExec x;
  x.pages = a.pages; x.elem_base = a.elem_base; x.src = src; x.lit = a.lit; x.lit_base = a.lit_base; x.dst = dst;
  x.done = reinterpret_cast<const int64_t*>(a.st); x.stride = sizeof(ZPage) / 8;
  x.e_out = a.e_out; x.e_ref = a.e_ref; x.e_lit = a.e_lit;
  AG_TRY(lz_exec_launch(x, n_pages, st));
  zstd_xxh64_kernel<<<split, 32 * kWarps, 0, st>>>(a);
  AG_TRY(check_launch("zstd_xxh64_kernel"));
  return lz_read_back(kFn, a.st, n_pages, h_written, st, [&](int64_t i, const ZPage& s, char* buf, size_t n) {
    if (s.err == kZErrSize) size_text(buf, n, pages[i].dst_len, s.got);
    else if (s.ck_bad != INT32_MAX) snprintf(buf, n, "parquet: could not decompress page: zstd: checksum mismatch");
    else if (s.err == kZErrCorrupt) snprintf(buf, n, "parquet: could not decompress page: zstd: %s", kCheckName[s.check]);
  });
}

}  // namespace

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_parquet_zstd_decompress_dev(const uint8_t* d_src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* d_dst,
                                         int64_t* d_written, ag_stream_t s) {
  AG_TRY(ensure_init());
  return pq_decompress_dev(kFn, zstd_dev, d_src, pages, n_pages, d_dst, d_written, resolve_stream(s));
}

ag_status ag_parquet_zstd_decompress(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst,
                                     int64_t* written) {
  AG_TRY(ensure_init());
  return pq_decompress_host(kFn, zstd_dev, src, pages, n_pages, dst, written);
}

}  // extern "C"
