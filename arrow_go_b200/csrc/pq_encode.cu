// pq_encode.cu — Parquet page encoders on the device: the RLE/bit-packed hybrid stream (RleEncoder,
// parquet/internal/utils/rle.go:314-445) for definition levels, dictionary indices and RLE booleans, and
// DELTA_BINARY_PACKED INT32 / INT64 (deltaBitPackEncoder, parquet/internal/encoding/delta_bit_packing.go:362-494).
//
// RLE/bit-packed: a parallel restatement of the sequential greedy encoder (tests/pq_encode_model.py is its
// specification).  Values are buffered in groups of 8 from an origin (the page start, or the end of the last repeated
// run), so a repeated run starts exactly at the first group, on the origin's 8-alignment, whose values are all equal,
// and runs to the end of that equal run, which is the next origin.  An equal run [a, b) entered with residue r (the
// origin mod 8) is caught iff a + ((r - a) mod 8) + 8 <= b, and then leaves residue b mod 8: every run of 8 or more is a
// map Z8 -> Z8 and the residue chain is a scan of those maps.  The groups between an origin and the next caught group
// are literal runs of at most 63 groups; the tail is a repeated run when no literal is pending and its < 8 values are
// equal, else one zero-padded literal group.
//
// rle_encode_kernel, one block per page, streams the page in tiles of kEncTile values (16 consecutive values per
// thread) through shared memory with a 16-value halo before and 8 after, and carries (origin, its stream offset, the
// start of the run still open at the tile's end, the first group start not yet decided) from tile to tile.  Per tile:
// a max-scan of run heads gives every run's start; a scan of the long runs' maps gives each thread's entry residue
// and so the caught runs; a max-scan of their ends gives each thread's origin; a sum-scan of stretch sizes (literal
// groups and headers, then the repeated run) gives every write offset.  Then each thread writes the repeated runs it
// closes and the literal groups starting in its values, and thread 0 writes the few groups held back by the previous
// tile's open run and, on the last tile, the tail.  HBM traffic: values read once plus stream bytes written once (the
// halo re-reads 24 values per 4096 from L2).
//
// DELTA_BINARY_PACKED: delta_encode_kernel, one block per page, gives each warp one block of deltas per step: the
// block's min delta, each miniblock's width (deltas wrap at the physical width), the block's size, a scan of the 8
// warps' sizes, then the header and bit-packed miniblocks.  Values are read from global memory (L1 / L2 serve the
// repeats); HBM traffic: values read once plus encoded bytes written once.
//
// BYTE_ARRAY (PLAIN, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY) from Arrow offsets, data and validity, over 1024-slot
// tiles of every page: ba_check_kernel (offsets and validity only: slot errors, per-tile sums) and tile_sum_scan_kernel,
// then the call's one synchronisation reads the per-page error words; ba_last_scan_kernel (DELTA: each tile's previous
// valid slot) and ba_dense_kernel (dense lengths, DELTA prefixes)
// feeds delta_encode_kernel<int32_t> through device page tables; ba_bytes_kernel writes each section in aligned 16-byte
// pieces.  BaCall below describes the order.
#include <climits>

#include "pq_decode.cuh"

namespace ag {

namespace {

constexpr int kEncItems = 16;                       // consecutive values per thread
constexpr int kEncTile = kPqThreads * kEncItems;    // values per tile
constexpr int kHaloLo = 16, kHaloHi = 8;
constexpr int kWin = kHaloLo + kEncTile + kHaloHi;  // values held in shared memory per tile
constexpr uint32_t kMapId = 0x76543210u;            // identity Z8 -> Z8 map, one nibble per residue
constexpr long long kNone = AG_NO_ERROR_POS;

__device__ __forceinline__ int skew(int j) { return j + (j >> 4); }  // 16 values per thread: no bank conflicts

// exclusive block scan of one value per thread under an associative `op` (in thread order, or in reverse order with
// REV); *total is the whole block's reduction
template <bool REV, typename V, typename Op>
__device__ __forceinline__ V block_scan_op(V v, V id, Op op, V* warp_tot, V* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  V x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const V y = REV ? __shfl_down_sync(0xffffffffu, x, o) : __shfl_up_sync(0xffffffffu, x, o);
    if (REV ? lane + o < 32 : lane >= o) x = REV ? op(x, y) : op(y, x);
  }
  V ex = REV ? __shfl_down_sync(0xffffffffu, x, 1) : __shfl_up_sync(0xffffffffu, x, 1);
  if (REV ? lane == 31 : lane == 0) ex = id;
  if (REV ? lane == 0 : lane == 31) warp_tot[wid] = x;
  __syncthreads();
  V pre = id, tot = id;
#pragma unroll
  for (int w = 0; w < kPqThreads / 32; ++w) {
    const V t = warp_tot[REV ? kPqThreads / 32 - 1 - w : w];
    if (REV ? kPqThreads / 32 - 1 - w > wid : w < wid) pre = op(pre, t);
    tot = op(tot, t);
  }
  __syncthreads();
  *total = tot;
  return op(pre, ex);
}

// f then g, maps Z8 -> Z8 held one nibble per residue
__device__ __forceinline__ uint32_t map_then(uint32_t f, uint32_t g) {
  uint32_t h = 0;
#pragma unroll
  for (int r = 0; r < 8; ++r) h |= ((g >> (4 * ((f >> (4 * r)) & 15u))) & 15u) << (4 * r);
  return h;
}

// the map of the equal run [a, b): residue r catches it iff a + ((r - a) mod 8) + 8 <= b, and then becomes b mod 8
__device__ __forceinline__ uint32_t run_map(int64_t a, int64_t b) {
  uint32_t m = 0;
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int64_t c = a + ((r - (int)(a & 7)) & 7);
    m |= (uint32_t)(c + 8 <= b ? (int)(b & 7) : r) << (4 * r);
  }
  return m;
}

__device__ __forceinline__ int varint_len(unsigned long long v) {
  int n = 1;
  while (v >= 0x80) { v >>= 7; ++n; }
  return n;
}
__device__ __forceinline__ int64_t put_varint(uint8_t* p, int64_t pos, unsigned long long v) {
  while (v >= 0x80) { p[pos++] = (uint8_t)(v | 0x80); v >>= 7; }
  p[pos++] = (uint8_t)v;
  return pos;
}
__device__ __forceinline__ unsigned long long zigzag(long long v) { return ((unsigned long long)v << 1) ^ (unsigned long long)(v >> 63); }

// LSB-first bit writer: appends w <= 32 bits, storing every completed byte at p[pos++]
struct BitPut {
  uint8_t* p;
  int64_t pos;
  unsigned long long acc = 0;
  int nbits = 0;
  __device__ __forceinline__ void put(unsigned long long x, int w) {
    acc |= (x & ((1ull << w) - 1ull)) << nbits;   // w <= 32 and nbits < 8: fits
    nbits += w;
    while (nbits >= 8) { p[pos++] = (uint8_t)acc; acc >>= 8; nbits -= 8; }
  }
};

struct RleEncArgs {
  const ag_pq_enc_page* pages;
  const void* values;
  uint8_t* out;
  int64_t* lengths;               // may be NULL
  unsigned long long* bad;        // lowest element offset holding a value wider than bw
  int bw, form;
};

template <int INPUT>
__device__ __forceinline__ uint32_t enc_load(const void* values, int64_t e) {
  if constexpr (INPUT == AG_PQ_RLE_IN_U32) return static_cast<const uint32_t*>(values)[e];
  else if constexpr (INPUT == AG_PQ_RLE_IN_I16) return (uint32_t)(int32_t) static_cast<const int16_t*>(values)[e];  // < 0: too wide
  else return (static_cast<const uint8_t*>(values)[e >> 3] >> (e & 7)) & 1u;
}

// 8 values from window slot j on, bit-packed into bw bytes at st[pos]
__device__ __forceinline__ void put_group(uint8_t* st, int64_t pos, const uint32_t* sv, int j, int bw) {
  BitPut b{st, pos};
#pragma unroll
  for (int k = 0; k < 8; ++k) b.put(sv[skew(j + k)], bw);
}

template <int INPUT>
__global__ void __launch_bounds__(kPqThreads)
rle_encode_kernel(RleEncArgs a) {
  __shared__ uint32_t sv[kWin + kWin / 16 + 1];
  __shared__ long long wl[kPqThreads / 32];
  __shared__ uint32_t wm[kPqThreads / 32];
  const ag_pq_enc_page pg = a.pages[blockIdx.x];
  const int64_t n = pg.num_values;
  const int bw = a.bw, nrep = (bw + 7) / 8;
  const int64_t run63 = 63 * (int64_t)bw + 1;     // bytes of a full literal run
  const uint32_t mask = bw == 32 ? 0xffffffffu : (1u << bw) - 1u;
  const int prefix = a.form == AG_PQ_RLE_LEN4 ? 4 : a.form == AG_PQ_RLE_WIDTH ? 1 : 0;
  uint8_t* const st = a.out + pg.out + prefix;    // the hybrid stream
  const int tid = threadIdx.x;
  auto lmax = [](long long x, long long y) { return x > y ? x : y; };
  auto lmin = [](long long x, long long y) { return x < y ? x : y; };
  auto lsum = [](long long x, long long y) { return x + y; };

  // carried from tile to tile (every thread holds the same copy)
  int64_t ac = 0;     // start of the run open at the end of the last tile
  int64_t o = 0;      // origin of the open stretch
  int64_t base = 0;   // stream offset of that stretch
  int64_t F = 0;      // first group start of the open stretch not yet decided literal or repeated
  long long bad = kNone;
  int64_t len = 0;
  for (int64_t t0 = 0; t0 < n; t0 += kEncTile) {
    const int64_t t1 = t0 + kEncTile < n ? t0 + kEncTile : n;
    const bool last = t1 == n;
    const int64_t win0 = t0 - kHaloLo;
    __syncthreads();                              // the last tile's readers are done
    for (int j = tid; j < kWin; j += kPqThreads) {
      const int64_t p = win0 + j;
      uint32_t v = 0;
      if (p >= 0 && p < n) {
        v = enc_load<INPUT>(a.values, pg.in + p);
        if (v > mask) {
          if (p >= t0 && p < bad) bad = p;
          v &= mask;
        }
      }
      sv[skew(j)] = v;
    }
    __syncthreads();
    const int64_t s0 = t0 + (int64_t)tid * kEncItems, s1 = s0 + kEncItems < t1 ? s0 + kEncItems : t1;
    auto V = [&](int64_t p) { return sv[skew((int)(p - win0))]; };
    auto head = [&](int64_t i) { return i == 0 || V(i) != V(i - 1); };
    auto ends = [&](int64_t i) { return i + 1 == n || V(i + 1) != V(i); };   // a run ends after i

    // run starts: the last head at or before each of my values
    long long h = -1;
    for (int64_t i = s0; i < s1; ++i) if (head(i)) h = i;
    long long htot;
    const long long hin = lmax(block_scan_op<false>(h, -1ll, lmax, wl, &htot), (long long)ac);

    // the maps of the long runs that end in my values, then my entry residue
    uint32_t m = kMapId;
    {
      int64_t s = hin;
      for (int64_t i = s0; i < s1; ++i) {
        if (head(i)) s = i;
        if (ends(i) && i + 1 - s >= 8) m = map_then(m, run_map(s, i + 1));
      }
    }
    uint32_t mtot;
    const uint32_t mex = block_scan_op<false>(m, kMapId, [](uint32_t f, uint32_t g) { return map_then(f, g); }, wm, &mtot);
    int r = (mex >> (4 * (int)(o & 7))) & 15;

    // my caught runs [c, b) (at most 2 end in 16 values)
    int64_t c0 = 0, b0 = 0, c1 = 0, b1 = 0;
    int nc = 0;
    {
      int64_t s = hin;
      for (int64_t i = s0; i < s1; ++i) {
        if (head(i)) s = i;
        if (ends(i) && i + 1 - s >= 8) {
          const int64_t c = s + ((r - (int)(s & 7)) & 7);
          if (c + 8 <= i + 1) {
            if (nc == 0) { c0 = c; b0 = i + 1; } else { c1 = c; b1 = i + 1; }
            ++nc;
            r = (int)((i + 1) & 7);
          }
        }
      }
    }
    long long btot, ctot;
    const int64_t oin = lmax(block_scan_op<false>(nc ? (long long)(nc == 2 ? b1 : b0) : -1ll, -1ll, lmax, wl, &btot), (long long)o);
    const int64_t cnext = block_scan_op<true>(nc ? (long long)c0 : kNone, kNone, lmin, wl, &ctot);  // first caught c after me
    auto stretch_bytes = [&](int64_t from, int64_t c, int64_t b) {
      const int64_t g = (c - from) >> 3;
      return g * bw + (g + 62) / 63 + varint_len((unsigned long long)(b - c) << 1) + nrep;
    };
    long long bytes = 0;
    if (nc >= 1) bytes += stretch_bytes(oin, c0, b0);
    if (nc == 2) bytes += stretch_bytes(b0, c1, b1);
    long long bsum;
    const int64_t bin = base + block_scan_op<false>(bytes, 0ll, lsum, wl, &bsum);
    const int64_t o_new = lmax(btot, (long long)o), base_new = base + bsum;
    // a caught run ending at t1 leaves the open run starting at the origin t1, whose head the next tile holds
    const int64_t ac_new = lmax(htot, lmax((long long)ac, (long long)o_new));
    const int64_t F_new = o_new + ((ac_new - o_new + 7) & ~(int64_t)7);
    const int64_t lim = last ? n - 7 : F_new;     // group starts below lim are decided (last tile: whole groups)

    // literal groups of the stretch (so, sbase) starting in [x0, x1)
    auto literal = [&](int64_t so, int64_t sbase, int64_t x0, int64_t x1) {
      for (int64_t x = so + ((x0 - so + 7) & ~(int64_t)7); x < x1; x += 8) {
        const int64_t k = (x - so) >> 3;
        put_group(st, sbase + k * bw + k / 63 + 1, sv, (int)(x - win0), bw);
        if (k % 63 == 62) st[sbase + (k / 63) * run63] = 0x7f;
      }
    };
    // closes the stretch (so, sbase) with the caught run [c, b); returns the stream offset after it
    auto close = [&](int64_t so, int64_t sbase, int64_t c, int64_t b) {
      const int64_t g = (c - so) >> 3;
      if (g % 63) st[sbase + (g / 63) * run63] = (uint8_t)(((g % 63) << 1) | 1);
      int64_t pos = put_varint(st, sbase + g * bw + (g + 62) / 63, (unsigned long long)(b - c) << 1);
      const uint32_t v = V(b - 1);
      for (int k = 0; k < nrep; ++k) st[pos++] = (uint8_t)(v >> (8 * k));
      return pos;
    };
    {
      int64_t so = oin, sbase = bin, x0 = s0;
      if (nc >= 1) { literal(so, sbase, x0, c0 < s1 ? c0 : s1); sbase = close(so, sbase, c0, b0); so = x0 = b0; }
      if (nc == 2) { literal(so, sbase, x0, c1 < s1 ? c1 : s1); sbase = close(so, sbase, c1, b1); so = x0 = b1; }
      int64_t x1 = s1 < cnext ? s1 : cnext;
      literal(so, sbase, x0, x1 < lim ? x1 : lim);
    }
    if (tid == 0 && F < t0) {
      // groups the previous tile held back: literal iff the run open there was not caught (any group of a run
      // longer than 16 values is repeated, so they start at t0 - 16 or later)
      int64_t x1 = t0 < ctot ? t0 : ctot;
      literal(o, base, F > win0 ? F : win0, x1 < lim ? x1 : lim);
    }
    if (last && tid == 0) {
      const int64_t full = (n - o_new) >> 3, xe = o_new + 8 * full;
      int64_t G = full;
      len = base_new + G * bw + (G + 62) / 63;
      if (xe < n) {
        bool eq = true;
        for (int64_t i = xe + 1; i < n; ++i) eq &= V(i) == V(xe);
        if (full % 63 == 0 && eq) {
          int64_t pos = put_varint(st, len, (unsigned long long)(n - xe) << 1);
          const uint32_t v = V(xe);
          for (int k = 0; k < nrep; ++k) st[pos++] = (uint8_t)(v >> (8 * k));
          len = pos;
        } else {
          put_group(st, base_new + full * bw + full / 63 + 1, sv, (int)(xe - win0), bw);   // zeros past n
          if (full % 63 == 62) st[base_new + (full / 63) * run63] = 0x7f;
          G = full + 1;
          len = base_new + G * bw + (G + 62) / 63;
        }
      }
      if (G % 63) st[base_new + (G / 63) * run63] = (uint8_t)(((G % 63) << 1) | 1);
    }
    o = o_new; base = base_new; ac = ac_new; F = F_new;
  }
  if (bad != kNone) atomicMin(a.bad, (unsigned long long)(pg.in + bad));
  if (tid == 0) {
    uint8_t* pre = a.out + pg.out;
    if (a.form == AG_PQ_RLE_LEN4)
      for (int k = 0; k < 4; ++k) pre[k] = (uint8_t)((uint64_t)len >> (8 * k));
    else if (a.form == AG_PQ_RLE_WIDTH)
      pre[0] = (uint8_t)bw;
    if (a.lengths) a.lengths[blockIdx.x] = prefix + len;
  }
}

struct DeltaEncArgs {
  const ag_pq_enc_page* pages;
  const void* values;
  uint8_t* out;
  int64_t* lengths;   // may be NULL
  int block, mini;
};

// delta k (k >= 1) of a page, wrapped at T's width and sign-extended
template <typename T>
__device__ __forceinline__ long long delta_of(const T* v, int64_t k) {
  using U = typename std::make_unsigned<T>::type;
  return (long long)(T)(U)((U)v[k] - (U)v[k - 1]);
}

template <typename T>
__global__ void __launch_bounds__(kPqThreads)
delta_encode_kernel(DeltaEncArgs a) {
  constexpr int kWarps = kPqThreads / 32;
  __shared__ long long wsz[kWarps];
  __shared__ long long s_hdr;
  const ag_pq_enc_page pg = a.pages[blockIdx.x];
  const int64_t n = pg.num_values;
  const T* v = static_cast<const T*>(a.values) + pg.in;
  uint8_t* const out = a.out + pg.out;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int block = a.block, mini = a.mini, vpm = block / mini;
  if (threadIdx.x == 0) {
    int64_t pos = put_varint(out, 0, (unsigned long long)block);
    pos = put_varint(out, pos, (unsigned long long)mini);
    pos = put_varint(out, pos, (unsigned long long)n);
    s_hdr = put_varint(out, pos, zigzag(n ? (long long)v[0] : 0ll));
  }
  __syncthreads();
  int64_t run = s_hdr;
  const int64_t nblk = n > 1 ? (n - 2) / block + 1 : 0;
  for (int64_t j0 = 0; j0 < nblk; j0 += kWarps) {
    const int64_t j = j0 + warp;
    const int64_t k0 = 1 + j * block;                 // first delta of the block
    const int64_t cnt = j < nblk ? (n - k0 < block ? n - k0 : block) : 0;
    long long mn = LLONG_MAX;
    for (int64_t k = lane; k < cnt; k += 32) { const long long d = delta_of(v, k0 + k); mn = d < mn ? d : mn; }
#pragma unroll
    for (int s = 16; s; s >>= 1) { const long long y = __shfl_xor_sync(0xffffffffu, mn, s); mn = y < mn ? y : mn; }
    // bit width of miniblock q: deltas wrap like uint64(delta - min)
    auto width = [&](int q) {
      unsigned long long acc = 0;
      const int64_t e = (int64_t)(q + 1) * vpm < cnt ? (int64_t)(q + 1) * vpm : cnt;
      for (int64_t k = (int64_t)q * vpm + lane; k < e; k += 32) acc |= (unsigned long long)delta_of(v, k0 + k) - (unsigned long long)mn;
#pragma unroll
      for (int s = 16; s; s >>= 1) acc |= __shfl_xor_sync(0xffffffffu, acc, s);
      return acc ? 64 - __clzll((long long)acc) : 0;
    };
    long long size = 0;
    if (cnt) {
      size = varint_len(zigzag(mn)) + mini;
      for (int q = 0; q < mini && (int64_t)q * vpm < cnt; ++q) size += (int64_t)width(q) * vpm / 8;
    }
    if (lane == 0) wsz[warp] = size;
    __syncthreads();
    long long ex = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) { ex += w < warp ? wsz[w] : 0; tot += wsz[w]; }
    __syncthreads();
    if (cnt) {
      int64_t pos = run + ex;
      if (lane == 0) pos = put_varint(out, pos, zigzag(mn));
      pos = __shfl_sync(0xffffffffu, pos, 0);
      const int64_t wpos = pos;
      pos += mini;
      for (int q = 0; q < mini; ++q) {
        const int w = (int64_t)q * vpm < cnt ? width(q) : 0;
        if (lane == 0) out[wpos + q] = (uint8_t)w;
        if ((int64_t)q * vpm >= cnt) continue;
        // lanes pack groups of 8 deltas (zeros past the block's last delta) into w bytes each
        for (int g = lane; g < vpm / 8; g += 32) {
          BitPut b{out, pos + (int64_t)g * w};
          for (int k = 0; k < 8; ++k) {
            const int64_t kk = (int64_t)q * vpm + 8 * g + k;
            const unsigned long long u = kk < cnt ? (unsigned long long)delta_of(v, k0 + kk) - (unsigned long long)mn : 0ull;
            if (w > 32) { b.put(u, 32); b.put(u >> 32, w - 32); } else { b.put(u, w); }
          }
        }
        pos += (int64_t)w * vpm / 8;
      }
    }
    run += tot;
  }
  if (threadIdx.x == 0 && a.lengths) a.lengths[blockIdx.x] = run;
}

// ------------------------------------------------------------------------------------------------ host side ----
int64_t bytes_for_bits(int64_t b) { return (b + 7) / 8; }

// MaxRLEBufferSize + MinRLEBufferSize (rle.go:36-51) plus the form's prefix
int64_t rle_bound(int bw, int form, int64_t n) {
  const int64_t runs = bytes_for_bits(n);
  const int64_t max_size = std::max(runs + runs * bw, runs * (1 + bytes_for_bits(bw)));
  const int64_t min_size = std::max(1 + bytes_for_bits(512 * (int64_t)bw), 5 + bytes_for_bits(bw));
  return max_size + min_size + (form == AG_PQ_RLE_LEN4 ? 4 : form == AG_PQ_RLE_WIDTH ? 1 : 0);
}

// header (4 varints of at most 10 bytes each) + per block: min delta (10) + width bytes + every miniblock at full width
__host__ __device__ int64_t delta_bound(int width, int block, int mini, int64_t n) {
  const int64_t nblk = n > 1 ? (n - 2) / block + 1 : 0;
  return 40 + nblk * (10 + mini + (int64_t)block * width);
}

ag_status check_rle_args(const char* fn, int bw, int form, int input, bool has_input) {
  if (form != AG_PQ_RLE_BARE && form != AG_PQ_RLE_LEN4 && form != AG_PQ_RLE_WIDTH) AG_FAIL(AG_ERR_INVALID, "%s: unknown form %d", fn, form);
  if (!has_input) {
    if (bw < 0 || bw > 32) AG_FAIL(AG_ERR_INVALID, "%s: bit width %d outside 0..32", fn, bw);
    return AG_OK;
  }
  if (input == AG_PQ_RLE_IN_U32) {
    if (bw < 0 || bw > 32) AG_FAIL(AG_ERR_INVALID, "%s: bit width %d outside 0..32 for indices", fn, bw);
  } else if (input == AG_PQ_RLE_IN_I16) {
    if (bw < 0 || bw > 16) AG_FAIL(AG_ERR_INVALID, "%s: bit width %d outside 0..16 for levels", fn, bw);
  } else if (input == AG_PQ_RLE_IN_BITMAP) {
    if (bw != 1) AG_FAIL(AG_ERR_INVALID, "%s: bit width %d for bitmap input (must be 1)", fn, bw);
  } else {
    AG_FAIL(AG_ERR_INVALID, "%s: unknown input kind %d", fn, input);
  }
  return AG_OK;
}

ag_status check_delta_args(const char* fn, int width, int block, int mini) {
  if (width != 4 && width != 8) AG_FAIL(AG_ERR_INVALID, "%s: value_width must be 4 (INT32) or 8 (INT64), got %d", fn, width);
  if (block <= 0 || block % 128) AG_FAIL(AG_ERR_INVALID, "%s: values per block must be a multiple of 128, got %d", fn, block);
  if (mini <= 0 || block % mini) AG_FAIL(AG_ERR_INVALID, "%s: miniblocks per block must divide the block size, got %d miniblocks for %d values", fn, mini, block);
  if ((block / mini) % 32) AG_FAIL(AG_ERR_INVALID, "%s: values per miniblock must be a nonzero multiple of 32, got %d", fn, block / mini);
  return AG_OK;
}

// The page table checked against the bound bound(num_values); *in_end / *out_end: the input elements and output bytes
// the pages reach.
template <typename Bound>
ag_status check_pages(const char* fn, const ag_pq_enc_page* pages, int64_t n_pages, Bound bound, int64_t* in_end, int64_t* out_end) {
  if (n_pages < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative page count", fn);
  if (n_pages > 0 && !pages) AG_FAIL(AG_ERR_INVALID, "%s: NULL page table", fn);
  if (n_pages > 0x7fffffff) AG_FAIL(AG_ERR_INVALID, "%s: more than 2^31-1 pages", fn);
  *in_end = *out_end = 0;
  for (int64_t i = 0; i < n_pages; ++i) {
    const ag_pq_enc_page& p = pages[i];
    if (p.num_values < 0 || p.num_values > 0x7fffffff) AG_FAIL(AG_ERR_INVALID, "%s: page %lld: num_values %lld outside 0..2^31-1", fn, (long long)i, (long long)p.num_values);
    if (p.in < 0 || p.out < 0) AG_FAIL(AG_ERR_INVALID, "%s: page %lld: negative offset", fn, (long long)i);
    const int64_t need = bound(p.num_values);
    if (p.capacity < need) AG_FAIL(AG_ERR_INVALID, "%s: page %lld: capacity %lld below the bound %lld", fn, (long long)i, (long long)p.capacity, (long long)need);
    if (p.num_values) *in_end = std::max(*in_end, p.in + p.num_values);
    *out_end = std::max(*out_end, p.out + p.capacity);
  }
  return AG_OK;
}

ag_status rle_encode_dev(int bw, int form, int input, const void* d_values, const ag_pq_enc_page* pages, int64_t n_pages,
                         uint8_t* d_out, int64_t* d_lengths, int64_t* d_bad_pos, int64_t* h_bad, cudaStream_t st) {
  const char* fn = "rle_encode";
  AG_TRY(check_rle_args(fn, bw, form, input, true));
  int64_t in_end, out_end;
  AG_TRY(check_pages(fn, pages, n_pages, [&](int64_t n) { return rle_bound(bw, form, n); }, &in_end, &out_end));
  if (in_end > 0 && !d_values) AG_FAIL(AG_ERR_INVALID, "%s: NULL values", fn);
  if (out_end > 0 && !d_out) AG_FAIL(AG_ERR_INVALID, "%s: NULL output", fn);
  TableImage img(st);
  const size_t o_pages = img.add(std::vector<ag_pq_enc_page>(pages, pages + n_pages));
  const size_t o_bad = img.add(std::vector<long long>{kNone});
  AG_TRY(img.upload(fn));
  unsigned long long* d_bad = img.at<unsigned long long>(o_bad);
  if (n_pages) {
    RleEncArgs a{img.at<ag_pq_enc_page>(o_pages), d_values, d_out, d_lengths, d_bad, bw, form};
    if (input == AG_PQ_RLE_IN_U32) rle_encode_kernel<AG_PQ_RLE_IN_U32><<<(unsigned)n_pages, kPqThreads, 0, st>>>(a);
    else if (input == AG_PQ_RLE_IN_I16) rle_encode_kernel<AG_PQ_RLE_IN_I16><<<(unsigned)n_pages, kPqThreads, 0, st>>>(a);
    else rle_encode_kernel<AG_PQ_RLE_IN_BITMAP><<<(unsigned)n_pages, kPqThreads, 0, st>>>(a);
    AG_TRY(check_launch("rle_encode_kernel"));
  }
  if (d_bad_pos) AG_CUDA_TRY(cudaMemcpyAsync(d_bad_pos, d_bad, 8, cudaMemcpyDeviceToDevice, st));
  int64_t bad = kNone;
  AG_TRY(d2h(&bad, d_bad, 8, st));
  AG_TRY(sync(st));
  if (h_bad) *h_bad = bad;
  if (bad != kNone) {
    const uint32_t mask = bw == 32 ? 0xffffffffu : (1u << bw) - 1u;
    for (int64_t i = 0; i < n_pages; ++i)
      if (bad >= pages[i].in && bad < pages[i].in + pages[i].num_values)
        AG_FAIL(AG_ERR_INVALID, "%s: page %lld: value at element %lld wider than bit width %d (mask 0x%x)", fn, (long long)i, (long long)bad, bw, mask);
  }
  return AG_OK;
}

ag_status delta_encode_dev(int width, int block, int mini, const void* d_values, const ag_pq_enc_page* pages, int64_t n_pages,
                           uint8_t* d_out, int64_t* d_lengths, cudaStream_t st) {
  const char* fn = "delta_encode";
  AG_TRY(check_delta_args(fn, width, block, mini));
  int64_t in_end, out_end;
  AG_TRY(check_pages(fn, pages, n_pages, [&](int64_t n) { return delta_bound(width, block, mini, n); }, &in_end, &out_end));
  if (in_end > 0 && !d_values) AG_FAIL(AG_ERR_INVALID, "%s: NULL values", fn);
  if (out_end > 0 && !d_out) AG_FAIL(AG_ERR_INVALID, "%s: NULL output", fn);
  if (reinterpret_cast<uintptr_t>(d_values) & (width - 1)) AG_FAIL(AG_ERR_INVALID, "%s: values not aligned to their width", fn);
  if (n_pages == 0) return AG_OK;
  TableImage img(st);
  const size_t o_pages = img.add(std::vector<ag_pq_enc_page>(pages, pages + n_pages));
  AG_TRY(img.upload(fn));
  DeltaEncArgs a{img.at<ag_pq_enc_page>(o_pages), d_values, d_out, d_lengths, block, mini};
  if (width == 4) delta_encode_kernel<int32_t><<<(unsigned)n_pages, kPqThreads, 0, st>>>(a);
  else delta_encode_kernel<int64_t><<<(unsigned)n_pages, kPqThreads, 0, st>>>(a);
  AG_TRY(check_launch("delta_encode_kernel"));
  return sync(st);
}

// host flavour: stage the input the pages reach and an output image as large as their sections, encode, and copy back
// each page's written bytes and the lengths
template <typename Dev>
ag_status encode_host(const ag_pq_enc_page* pages, int64_t n_pages, const void* values, int64_t in_bytes, int64_t out_end,
                      uint8_t* out, int64_t* lengths, Dev dev) {
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  Carve sc;
  const size_t o_in = sc.take((size_t)in_bytes), o_out = sc.take((size_t)out_end), o_len = sc.take((size_t)n_pages * 8);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, sc.size));
  AG_TRY(h2d(d + o_in, values, (size_t)in_bytes, cs));
  int64_t* d_len = reinterpret_cast<int64_t*>(d + o_len);
  const ag_status rc = dev(d + o_in, d + o_out, d_len, (cudaStream_t)cs);
  if (rc != AG_OK) return rc;
  std::vector<int64_t> len((size_t)n_pages);
  AG_TRY(d2h(len.data(), d_len, (size_t)n_pages * 8, cs));
  AG_TRY(sync(cs));
  for (int64_t i = 0; i < n_pages; ++i) AG_TRY(d2h(out + pages[i].out, d + o_out + pages[i].out, (size_t)len[i], cs));
  if (lengths) memcpy(lengths, len.data(), (size_t)n_pages * 8);
  return sync(cs);
}

// ------------------------------------------------------------------------------- BYTE_ARRAY value sections ----
constexpr int kBaItems = kBaTile / kPqThreads;      // 4 consecutive slots per thread
constexpr unsigned long long kBaOk = ~0ull;         // error word of a page that passes
constexpr unsigned long long kBaCap = ~0ull - 1;    // capacity below the bound; every slot error is lower
enum BaErr { kBaNegFirst = 0, kBaDecreasing = 1, kBaTooLong = 2 };   // slot errors: word = slot * 4 + kind

struct BaArgs {
  const ag_pq_enc_page* pages;
  const int64_t* tile_base;       // [n_pages + 1]: first tile of every page
  const int64_t* sum_base;        // [n_pages + 1]: tile_base[p] + p, page p's entries in cnt / bytes
  int64_t n_pages, n_tiles;
  const void* offsets;
  const uint8_t* data;
  const uint8_t* valid;           // NULL: every slot valid
  int enc;
  unsigned long long* err;        // [n_pages] lowest slot error word, kBaCap, or kBaOk
  unsigned long long* cnt;        // per tile valid values, then (scanned) the page's before the tile; the page's
                                  // entry after its tiles holds its total
  unsigned long long* bytes;      // the same for the section bytes (DELTA: suffix bytes, written by the dense pass)
  long long* last;                // [n_tiles] the tile's last valid slot, -1 if none (DELTA: then the page's, up to
                                  // and including the tile)
  int64_t* dense;                 // [n_pages + 1] the page's first dense value; [n_pages] all of them
  int32_t* lens;                  // dense: lengths (DELTA_LENGTH) or suffix lengths (DELTA)
  int32_t* pre;                   // dense: prefix lengths (DELTA)
  ag_pq_enc_page* tab;            // [2 * n_pages] the length streams' pages (DELTA: prefixes, then suffixes)
  int64_t* slen;                  // [2 * n_pages] bytes of those streams
  int64_t* sec;                   // [n_pages] the byte section's offset from the page's out
  uint8_t* out;
  int64_t* lengths;               // may be NULL
  const ag_pq_ba_chunk* chunks;   // NULL, or per page its own offsets and validity (a dictionary call's chunks)
};

__host__ __device__ __forceinline__ int64_t ba_bound(int enc, int64_t n, int64_t span) {
  if (enc == AG_PQ_ENC_PLAIN) return 4 * n + span;
  return (enc == AG_PQ_ENC_DELTA_BYTE_ARRAY ? 2 : 1) * delta_bound(4, 128, 4, n) + span;
}

template <typename O>
__device__ __forceinline__ int64_t off_at(const void* o, int64_t i) { return (int64_t) static_cast<const O*>(o)[i]; }

// the length of the common prefix of x[0, m) and y[0, m), 16 bytes per step
__device__ __forceinline__ int64_t common_prefix(const uint8_t* x, const uint8_t* y, int64_t m) {
  for (int64_t k = 0; k < m; k += 16) {
    const int c = m - k < 16 ? (int)(m - k) : 16;
    const u128 d = window(x + k, c) ^ window(y + k, c);
    if (d) {
      const unsigned long long lo = (unsigned long long)d;
      return k + (lo ? __ffsll((long long)lo) - 1 : 64 + __ffsll((long long)(d >> 64)) - 1) / 8;
    }
  }
  return m;
}

// the tile of block `t`: its page, the page's slot of the thread's first item, the offsets of the thread's items and
// their validity (false past the page).  `offsets` / `valid`: the page's arrays.
struct BaSlots {
  int64_t p, j0;
  ag_pq_enc_page pg;
  int64_t o[kBaItems + 1];
  bool v[kBaItems];
};

template <typename O>
__device__ __forceinline__ void ba_slots(const BaArgs& a, int64_t t, BaSlots& s, const void* offsets, const uint8_t* valid) {
  s.p = find_page(a.tile_base, a.n_pages, t);
  s.pg = a.pages[s.p];
  s.j0 = (t - a.tile_base[s.p]) * kBaTile + threadIdx.x * kBaItems;
#pragma unroll
  for (int q = 0; q <= kBaItems; ++q) {
    const int64_t j = s.j0 + q;
    s.o[q] = j <= s.pg.num_values ? off_at<O>(offsets, s.pg.in + j) : 0;
    if (q < kBaItems) s.v[q] = j < s.pg.num_values && (!valid || bit_is_set(valid, s.pg.in + j));
  }
}

// Checking pass: one thread per page for the capacity (from the page's offsets span), one block per tile for the
// slot errors and the tile's valid count, section bytes (PLAIN, DELTA_LENGTH) and last valid slot.  Reads offsets and
// validity only.
template <typename O>
__global__ void __launch_bounds__(kPqThreads)
ba_check_kernel(BaArgs a) {
  __shared__ long long wl[kPqThreads / 32];
  for (int64_t p = (int64_t)blockIdx.x * kPqThreads + threadIdx.x; p < a.n_pages; p += (int64_t)gridDim.x * kPqThreads) {
    const ag_pq_enc_page pg = a.pages[p];
    const void* o = a.chunks ? a.chunks[p].offsets : a.offsets;
    const int64_t span = pg.num_values ? off_at<O>(o, pg.in + pg.num_values) - off_at<O>(o, pg.in) : 0;
    if (pg.capacity < ba_bound(a.enc, pg.num_values, span)) atomicMin(a.err + p, kBaCap);
  }
  if (blockIdx.x >= a.n_tiles) return;
  const int64_t t = blockIdx.x;
  BaSlots s;
  if (a.chunks) {
    const ag_pq_ba_chunk& ch = a.chunks[find_page(a.tile_base, a.n_pages, t)];
    ba_slots<O>(a, t, s, ch.offsets, ch.valid);
  } else {
    ba_slots<O>(a, t, s, a.offsets, a.valid);
  }
  long long c = 0, b = 0, lst = -1;
  unsigned long long bad = kBaOk;
#pragma unroll
  for (int q = 0; q < kBaItems; ++q) {
    const int64_t j = s.j0 + q;
    if (j >= s.pg.num_values) break;
    const unsigned long long w = (unsigned long long)(s.pg.in + j) * 4;
    const int64_t len = s.o[q + 1] - s.o[q];
    if (j == 0 && s.o[0] < 0) bad = min(bad, w + kBaNegFirst);
    if (len < 0) bad = min(bad, w + kBaDecreasing);
    else if (s.v[q] && len > INT_MAX) bad = min(bad, w + kBaTooLong);
    if (s.v[q]) {
      ++c;
      b += len + (a.enc == AG_PQ_ENC_PLAIN ? 4 : 0);
      lst = s.pg.in + j;
    }
  }
  if (bad != kBaOk) atomicMin(a.err + s.p, bad);
  auto lsum = [](long long x, long long y) { return x + y; };
  auto lmax = [](long long x, long long y) { return x > y ? x : y; };
  long long ctot, btot, ltot;
  block_scan_op<false>(c, 0ll, lsum, wl, &ctot);
  block_scan_op<false>(b, 0ll, lsum, wl, &btot);
  block_scan_op<false>(lst, -1ll, lmax, wl, &ltot);
  if (threadIdx.x == 0) {
    a.cnt[t + s.p] = (unsigned long long)ctot;
    if (a.enc != AG_PQ_ENC_DELTA_BYTE_ARRAY) a.bytes[t + s.p] = (unsigned long long)btot;
    a.last[t] = ltot;
  }
}

// one block: every page's first dense value and the length streams' page tables (input at the page's dense base,
// num_values its valid count, output at its out)
__global__ void __launch_bounds__(kPqThreads)
ba_tables_kernel(BaArgs a) {
  __shared__ long long ws[kPqThreads / 32];
  for (int64_t p = threadIdx.x; p < a.n_pages; p += kPqThreads) a.dense[p] = (int64_t)a.cnt[a.sum_base[p + 1] - 1];
  __syncthreads();
  const int64_t total = segment_excl_scan(a.dense, 0, a.n_pages, ws);
  __syncthreads();
  if (threadIdx.x == 0) a.dense[a.n_pages] = total;
  for (int64_t p = threadIdx.x; p < a.n_pages; p += kPqThreads) {
    const ag_pq_enc_page pg = a.pages[p];
    const ag_pq_enc_page t{a.dense[p], (int64_t)a.cnt[a.sum_base[p + 1] - 1], pg.out, pg.capacity};
    a.tab[p] = t;
    a.tab[a.n_pages + p] = t;
  }
}

// DELTA, one block per page: each tile's last valid slot -> the page's last valid slot at or before the tile (a max-scan
// over the page's tiles), so that a tile after a run of all-null tiles finds its previous value in one load
__global__ void __launch_bounds__(kPqThreads)
ba_last_scan_kernel(const int64_t* tile_base, long long* last) {
  __shared__ long long wl[kPqThreads / 32];
  auto lmax = [](long long x, long long y) { return x > y ? x : y; };
  const int64_t t1 = tile_base[blockIdx.x + 1];
  long long run = -1;
  for (int64_t t = tile_base[blockIdx.x]; t < t1; t += kPqThreads) {
    const int64_t i = t + threadIdx.x;
    const long long x = i < t1 ? last[i] : -1ll;
    long long tot;
    const long long ex = block_scan_op<false>(x, -1ll, lmax, wl, &tot);
    if (i < t1) last[i] = lmax(lmax(run, ex), x);
    run = lmax(run, tot);
  }
}

// DELTA_LENGTH / DELTA: the valid values' lengths as dense int32; DELTA: prefix lengths against the previous valid
// value of the page (across a tile edge, the page's last valid slot before the tile, from ba_last_scan_kernel) and
// suffix lengths, and the tile's suffix bytes
template <typename O, bool DBA>
__global__ void __launch_bounds__(kPqThreads)
ba_dense_kernel(BaArgs a) {
  __shared__ long long wl[kPqThreads / 32];
  const int64_t t = blockIdx.x;
  BaSlots s;
  ba_slots<O>(a, t, s, a.offsets, a.valid);
  auto lsum = [](long long x, long long y) { return x + y; };
  auto lmax = [](long long x, long long y) { return x > y ? x : y; };
  long long c = 0, lst = -1, tot;
#pragma unroll
  for (int q = 0; q < kBaItems; ++q)
    if (s.v[q]) { ++c; lst = s.pg.in + s.j0 + q; }
  int64_t r = a.dense[s.p] + (int64_t)a.cnt[t + s.p] + block_scan_op<false>(c, 0ll, lsum, wl, &tot);
  long long prev = -1;
  if (DBA) prev = lmax(block_scan_op<false>(lst, -1ll, lmax, wl, &tot), t > a.tile_base[s.p] ? a.last[t - 1] : -1ll);
  long long sb = 0;
#pragma unroll
  for (int q = 0; q < kBaItems; ++q) {
    if (!s.v[q]) continue;
    const int64_t len = s.o[q + 1] - s.o[q];
    int64_t pl = 0;
    if (DBA) {
      if (prev >= 0) {
        const int64_t p0 = off_at<O>(a.offsets, prev), plen = off_at<O>(a.offsets, prev + 1) - p0;
        pl = common_prefix(a.data + p0, a.data + s.o[q], plen < len ? plen : len);
      }
      a.pre[r] = (int32_t)pl;
      prev = s.pg.in + s.j0 + q;
    }
    a.lens[r++] = (int32_t)(len - pl);
    sb += len - pl;
  }
  if (DBA) {
    block_scan_op<false>(sb, 0ll, lsum, wl, &tot);
    if (threadIdx.x == 0) a.bytes[t + s.p] = (unsigned long long)tot;
  }
}

// DELTA: the suffix-length stream starts where the prefix stream ends
__global__ void ba_link_kernel(BaArgs a) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < a.n_pages; p += (int64_t)gridDim.x * blockDim.x)
    a.tab[a.n_pages + p].out = a.tab[p].out + a.slen[p];
}

// every page: its byte section's offset after its length streams, and the bytes it wrote
__global__ void ba_finish_kernel(BaArgs a, int streams) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < a.n_pages; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t sec = (streams > 0 ? a.slen[p] : 0) + (streams > 1 ? a.slen[a.n_pages + p] : 0);
    a.sec[p] = sec;
    if (a.lengths) a.lengths[p] = sec + (int64_t)a.bytes[a.sum_base[p + 1] - 1];
  }
}

// Byte pass, one block per tile: each slot's section bytes (PLAIN: 4-byte length and value; DELTA_LENGTH: value;
// DELTA: suffix) are placed by a scan into shared memory, then threads fill the tile's section in 16-byte pieces
// aligned in `out`: a binary search finds the slot under a piece's first byte, the piece is assembled in a register
// from 16-byte loads shifted into place, and stored whole (pieces cut by the tile's ends: byte by byte).
template <typename O, int ENC>
__global__ void __launch_bounds__(kPqThreads)
ba_bytes_kernel(BaArgs a) {
  __shared__ long long wl[kPqThreads / 32];
  __shared__ int64_t soff[kBaTile + 1];   // tile slot -> its first byte, relative to the tile's
  __shared__ int64_t ssrc[kBaTile];       // tile slot -> its first data byte placed
  const int64_t t = blockIdx.x;
  const int tid = threadIdx.x;
  BaSlots s;
  ba_slots<O>(a, t, s, a.offsets, a.valid);
  auto lsum = [](long long x, long long y) { return x + y; };
  long long tot;
  int64_t r = 0;
  if (ENC == AG_PQ_ENC_DELTA_BYTE_ARRAY) {
    long long c = 0;
#pragma unroll
    for (int q = 0; q < kBaItems; ++q) c += s.v[q];
    r = a.dense[s.p] + (int64_t)a.cnt[t + s.p] + block_scan_op<false>(c, 0ll, lsum, wl, &tot);
  }
  int64_t z[kBaItems];
  long long sum = 0;
#pragma unroll
  for (int q = 0; q < kBaItems; ++q) {
    z[q] = 0;
    int64_t src = s.o[q];
    if (s.v[q]) {
      z[q] = s.o[q + 1] - s.o[q];
      if (ENC == AG_PQ_ENC_PLAIN) z[q] += 4;
      if (ENC == AG_PQ_ENC_DELTA_BYTE_ARRAY) { const int32_t pl = a.pre[r++]; z[q] -= pl; src += pl; }
    }
    ssrc[tid * kBaItems + q] = src;
    sum += z[q];
  }
  long long run = block_scan_op<false>(sum, 0ll, lsum, wl, &tot);
#pragma unroll
  for (int q = 0; q < kBaItems; ++q) { soff[tid * kBaItems + q] = run; run += z[q]; }
  if (tid == 0) soff[kBaTile] = tot;
  __syncthreads();

  uint8_t* const lo_p = a.out + s.pg.out + a.sec[s.p] + (int64_t)a.bytes[t + s.p];
  const uintptr_t lo_a = reinterpret_cast<uintptr_t>(lo_p), hi_a = lo_a + (uintptr_t)tot;
  for (uintptr_t P = (lo_a & ~(uintptr_t)15) + 16 * (uintptr_t)tid; P < hi_a; P += 16 * kPqThreads) {
    const uintptr_t lo = P > lo_a ? P : lo_a, hi = P + 16 < hi_a ? P + 16 : hi_a;
    int64_t b = (int64_t)(lo - lo_a);
    int l = 0, h = kBaTile - 1;                     // the last slot starting at or before b holds b
    while (l < h) {
      const int m = (l + h + 1) >> 1;
      if (soff[m] <= b) l = m; else h = m - 1;
    }
    u128 acc = 0;
    const int dend = (int)(hi - P);
    for (int d = (int)(lo - P), k; d < dend; d += k, b += k) {
      int64_t w = b - soff[l];
      while (w >= soff[l + 1] - soff[l]) { ++l; w = b - soff[l]; }   // past the slot's bytes, and empty slots
      const int64_t left = soff[l + 1] - soff[l] - w;
      u128 part;
      if (ENC == AG_PQ_ENC_PLAIN && w < 4) {
        k = (int)(4 - w < dend - d ? 4 - w : dend - d);
        const unsigned long long hdr = (unsigned long long)(uint32_t)(soff[l + 1] - soff[l] - 4) >> (8 * w);
        part = (u128)(hdr & ((1ull << (8 * k)) - 1));
      } else {
        k = (int)(left < dend - d ? left : dend - d);
        part = window(a.data + ssrc[l] + (ENC == AG_PQ_ENC_PLAIN ? w - 4 : w), k);
      }
      acc |= part << (8 * d);
    }
    uint8_t* const dst = reinterpret_cast<uint8_t*>(P);
    if (lo == P && hi == P + 16) {
      *reinterpret_cast<uint4*>(dst) = make_uint4((uint32_t)acc, (uint32_t)(acc >> 32), (uint32_t)(acc >> 64), (uint32_t)(acc >> 96));
    } else {
      for (int d = (int)(lo - P); d < dend; ++d) dst[d] = (uint8_t)(acc >> (8 * d));
    }
  }
}

ag_status check_ba_args(const char* fn, int enc, int ow) {
  if (enc != AG_PQ_ENC_PLAIN && enc != AG_PQ_ENC_DELTA_LENGTH_BYTE_ARRAY && enc != AG_PQ_ENC_DELTA_BYTE_ARRAY)
    AG_FAIL(AG_ERR_INVALID, "%s: encoding %d is not PLAIN, DELTA_LENGTH_BYTE_ARRAY or DELTA_BYTE_ARRAY", fn, enc);
  if (ow != 4 && ow != 8) AG_FAIL(AG_ERR_INVALID, "%s: offset_width must be 4 or 8, got %d", fn, ow);
  return AG_OK;
}

// The host checks of a call: arguments, the page table, and the buffers the pages reach.  *in_end: the slots they reach.
ag_status check_ba_call(const char* fn, int enc, int ow, const void* offsets, const uint8_t* data, const ag_pq_enc_page* pages,
                        int64_t n_pages, const uint8_t* out, int64_t* in_end, int64_t* out_end) {
  AG_TRY(check_ba_args(fn, enc, ow));
  AG_TRY(check_pages(fn, pages, n_pages, [](int64_t) { return (int64_t)0; }, in_end, out_end));
  if (*in_end > 0 && !offsets) AG_FAIL(AG_ERR_INVALID, "%s: NULL offsets", fn);
  if (*in_end > 0 && !data) AG_FAIL(AG_ERR_INVALID, "%s: NULL data", fn);
  if (*out_end > 0 && !out) AG_FAIL(AG_ERR_INVALID, "%s: NULL output", fn);
  return AG_OK;
}

// One checked call in two steps: check() runs the checking pass and synchronises `st` once to read the per-page error
// words; encode() then enqueues the rest without synchronising.  Scratch and tables are stream-ordered.
struct BaCall {
  const char* fn;
  int enc, ow;
  const ag_pq_enc_page* pages;
  int64_t n_pages;
  cudaStream_t st;
  TableImage img;
  void* scratch = nullptr;
  void* vals = nullptr;
  BaArgs a{};
  int64_t total = 0;   // valid values of all pages (DELTA_LENGTH, DELTA)
  BaCall(const char* f, int e, int w, const ag_pq_enc_page* p, int64_t n, cudaStream_t s)
      : fn(f), enc(e), ow(w), pages(p), n_pages(n), st(s), img(s) {}
  ~BaCall() { dev_free_async(vals, st); dev_free_async(scratch, st); }

  // chunks: NULL, or a HOST array of one dictionary chunk per page, which then brings its own offsets and validity;
  // errors name the chunk and give the slot in the call's numbering across the chunks
  ag_status check(const void* d_off, const uint8_t* d_valid, int64_t* d_bad_pos, int64_t* h_bad, const ag_pq_ba_chunk* chunks = nullptr) {
    std::vector<int64_t> tb((size_t)n_pages + 1, 0), sb((size_t)n_pages + 1, 0);
    for (int64_t i = 0; i < n_pages; ++i) {
      tb[(size_t)i + 1] = tb[(size_t)i] + (pages[i].num_values + kBaTile - 1) / kBaTile;
      sb[(size_t)i + 1] = tb[(size_t)i + 1] + i + 1;
    }
    const int64_t n_tiles = tb[(size_t)n_pages];
    if (n_tiles > 0x7fffffff) AG_FAIL(AG_ERR_INVALID, "%s: more than 2^31-1 tiles of %d slots", fn, kBaTile);
    const size_t o_pages = img.add(std::vector<ag_pq_enc_page>(pages, pages + n_pages));
    const size_t o_tb = img.add(tb), o_sb = img.add(sb);
    const size_t o_err = img.add(std::vector<unsigned long long>((size_t)n_pages, kBaOk));
    const size_t o_chunks = chunks ? img.add(std::vector<ag_pq_ba_chunk>(chunks, chunks + n_pages)) : 0;
    AG_TRY(img.upload(fn));
    Carve sc;
    const size_t o_cnt = sc.take((size_t)(n_tiles + n_pages) * 8), o_bytes = sc.take((size_t)(n_tiles + n_pages) * 8);
    const size_t o_last = sc.take((size_t)n_tiles * 8), o_dense = sc.take((size_t)(n_pages + 1) * 8);
    const size_t o_tab = sc.take((size_t)n_pages * 2 * sizeof(ag_pq_enc_page)), o_slen = sc.take((size_t)n_pages * 16);
    const size_t o_sec = sc.take((size_t)n_pages * 8);
    AG_TRY(dev_alloc_async(&scratch, sc.size, st));
    uint8_t* d = static_cast<uint8_t*>(scratch);
    AG_CUDA_TRY(cudaMemsetAsync(d, 0, o_last, st));   // cnt and bytes: the pages' total entries start at 0
    a = BaArgs{img.at<ag_pq_enc_page>(o_pages), img.at<int64_t>(o_tb), img.at<int64_t>(o_sb), n_pages, n_tiles, d_off,
               nullptr, d_valid, enc, img.at<unsigned long long>(o_err), reinterpret_cast<unsigned long long*>(d + o_cnt),
               reinterpret_cast<unsigned long long*>(d + o_bytes), reinterpret_cast<long long*>(d + o_last),
               reinterpret_cast<int64_t*>(d + o_dense), nullptr, nullptr, reinterpret_cast<ag_pq_enc_page*>(d + o_tab),
               reinterpret_cast<int64_t*>(d + o_slen), reinterpret_cast<int64_t*>(d + o_sec), nullptr, nullptr,
               chunks ? img.at<ag_pq_ba_chunk>(o_chunks) : nullptr};
    const unsigned grid = (unsigned)std::max<int64_t>(n_tiles, (n_pages + kPqThreads - 1) / kPqThreads);
    if (ow == 4) ba_check_kernel<int32_t><<<grid, kPqThreads, 0, st>>>(a);
    else ba_check_kernel<int64_t><<<grid, kPqThreads, 0, st>>>(a);
    AG_TRY(check_launch("ba_check_kernel"));
    tile_sum_scan_kernel<<<(unsigned)n_pages, kPqThreads, 0, st>>>(a.sum_base, a.cnt);
    AG_TRY(check_launch("tile_sum_scan_kernel"));
    if (enc != AG_PQ_ENC_DELTA_BYTE_ARRAY) {
      tile_sum_scan_kernel<<<(unsigned)n_pages, kPqThreads, 0, st>>>(a.sum_base, a.bytes);
      AG_TRY(check_launch("tile_sum_scan_kernel"));
    }
    if (enc != AG_PQ_ENC_PLAIN) {
      ba_tables_kernel<<<1, kPqThreads, 0, st>>>(a);
      AG_TRY(check_launch("ba_tables_kernel"));
      AG_TRY(d2h(&total, a.dense + n_pages, 8, st));
    }
    std::vector<unsigned long long> err((size_t)n_pages);
    AG_TRY(d2h(err.data(), a.err, (size_t)n_pages * 8, st));
    AG_TRY(sync(st));
    int64_t page = -1;
    for (int64_t i = 0; i < n_pages && page < 0; ++i) if (err[(size_t)i] != kBaOk) page = i;
    const unsigned long long w = page < 0 ? kBaOk : err[(size_t)page];
    int64_t bad = page < 0 || w == kBaCap ? (int64_t)AG_NO_ERROR_POS : (int64_t)(w >> 2);
    if (chunks && bad != (int64_t)AG_NO_ERROR_POS) {
      bad -= chunks[page].offset;
      for (int64_t c = 0; c < page; ++c) bad += chunks[c].length;
    }
    if (h_bad) *h_bad = bad;
    if (d_bad_pos) AG_TRY(h2d(d_bad_pos, &bad, 8, st));
    if (page < 0) return AG_OK;
    const char* unit = chunks ? "chunk" : "page";
    const long long pl = (long long)page, sl = (long long)bad;
    if (w == kBaCap) AG_FAIL(AG_ERR_INVALID, "%s: page %lld: capacity %lld below the bound for its %lld values and their bytes", fn, pl,
                             (long long)pages[page].capacity, (long long)pages[page].num_values);
    if ((w & 3) == kBaNegFirst) AG_FAIL(AG_ERR_INVALID, "%s: %s %lld: negative offset at slot %lld", fn, unit, pl, sl);
    if ((w & 3) == kBaDecreasing) AG_FAIL(AG_ERR_INVALID, "%s: %s %lld: offsets decrease after slot %lld", fn, unit, pl, sl);
    AG_FAIL(AG_ERR_INVALID, "%s: %s %lld: value at slot %lld longer than 2^31-1 bytes", fn, unit, pl, sl);
  }

  ag_status encode(const uint8_t* d_data, uint8_t* d_out, int64_t* d_lengths) {
    a.data = d_data;
    a.out = d_out;
    a.lengths = d_lengths;
    const bool dba = enc == AG_PQ_ENC_DELTA_BYTE_ARRAY;
    const unsigned nt = (unsigned)a.n_tiles, np = (unsigned)n_pages, ng = (unsigned)((n_pages + kPqThreads - 1) / kPqThreads);
    if (enc != AG_PQ_ENC_PLAIN) {
      AG_TRY(dev_alloc_async(&vals, (size_t)total * (dba ? 8 : 4) + 16, st));
      a.lens = static_cast<int32_t*>(vals);
      a.pre = a.lens + total;
      if (nt && dba) {
        ba_last_scan_kernel<<<np, kPqThreads, 0, st>>>(a.tile_base, a.last);
        AG_TRY(check_launch("ba_last_scan_kernel"));
      }
      if (nt) {
        if (ow == 4) dba ? ba_dense_kernel<int32_t, true><<<nt, kPqThreads, 0, st>>>(a) : ba_dense_kernel<int32_t, false><<<nt, kPqThreads, 0, st>>>(a);
        else dba ? ba_dense_kernel<int64_t, true><<<nt, kPqThreads, 0, st>>>(a) : ba_dense_kernel<int64_t, false><<<nt, kPqThreads, 0, st>>>(a);
        AG_TRY(check_launch("ba_dense_kernel"));
      }
      if (dba) {
        tile_sum_scan_kernel<<<np, kPqThreads, 0, st>>>(a.sum_base, a.bytes);
        AG_TRY(check_launch("tile_sum_scan_kernel"));
      }
      delta_encode_kernel<int32_t><<<np, kPqThreads, 0, st>>>(DeltaEncArgs{a.tab, dba ? a.pre : a.lens, d_out, a.slen, 128, 4});
      AG_TRY(check_launch("delta_encode_kernel"));
      if (dba) {
        ba_link_kernel<<<ng, kPqThreads, 0, st>>>(a);
        AG_TRY(check_launch("ba_link_kernel"));
        delta_encode_kernel<int32_t><<<np, kPqThreads, 0, st>>>(DeltaEncArgs{a.tab + n_pages, a.lens, d_out, a.slen + n_pages, 128, 4});
        AG_TRY(check_launch("delta_encode_kernel"));
      }
    }
    ba_finish_kernel<<<ng, kPqThreads, 0, st>>>(a, enc == AG_PQ_ENC_PLAIN ? 0 : dba ? 2 : 1);
    AG_TRY(check_launch("ba_finish_kernel"));
    if (!nt) return AG_OK;
    if (ow == 4) {
      if (enc == AG_PQ_ENC_PLAIN) ba_bytes_kernel<int32_t, AG_PQ_ENC_PLAIN><<<nt, kPqThreads, 0, st>>>(a);
      else if (dba) ba_bytes_kernel<int32_t, AG_PQ_ENC_DELTA_BYTE_ARRAY><<<nt, kPqThreads, 0, st>>>(a);
      else ba_bytes_kernel<int32_t, AG_PQ_ENC_DELTA_LENGTH_BYTE_ARRAY><<<nt, kPqThreads, 0, st>>>(a);
    } else {
      if (enc == AG_PQ_ENC_PLAIN) ba_bytes_kernel<int64_t, AG_PQ_ENC_PLAIN><<<nt, kPqThreads, 0, st>>>(a);
      else if (dba) ba_bytes_kernel<int64_t, AG_PQ_ENC_DELTA_BYTE_ARRAY><<<nt, kPqThreads, 0, st>>>(a);
      else ba_bytes_kernel<int64_t, AG_PQ_ENC_DELTA_LENGTH_BYTE_ARRAY><<<nt, kPqThreads, 0, st>>>(a);
    }
    return check_launch("ba_bytes_kernel");
  }
};

// ------------------------------------------------------------------------------- BYTE_ARRAY dictionaries ----
// The host checks of a dictionary call (before the device is touched); *slots: the call's slots.
ag_status check_ba_dict_call(const char* fn, int ow, const ag_pq_ba_chunk* chunks, int64_t n_chunks, const int64_t* marks, int64_t n_marks,
                             const void* indices, const int64_t* mark_counts, const int64_t* counts, int64_t* slots) {
  if (ow != 4 && ow != 8) AG_FAIL(AG_ERR_INVALID, "%s: offset_width must be 4 or 8, got %d", fn, ow);
  if (n_chunks < 0 || (n_chunks > 0 && !chunks)) AG_FAIL(AG_ERR_INVALID, "%s: bad chunk table", fn);
  int64_t total = 0;
  for (int64_t c = 0; c < n_chunks; ++c) {
    const ag_pq_ba_chunk& ch = chunks[c];
    if (ch.offset < 0 || ch.length < 0) AG_FAIL(AG_ERR_INVALID, "%s: chunk %lld: negative offset or length", fn, (long long)c);
    if (ch.length == 0) continue;
    if (!ch.offsets || !ch.data || !ch.first) AG_FAIL(AG_ERR_INVALID, "%s: chunk %lld: NULL offsets, data or first bitmap", fn, (long long)c);
    if (reinterpret_cast<uintptr_t>(ch.first) & 3) AG_FAIL(AG_ERR_INVALID, "%s: chunk %lld: the first bitmap must be 4-byte aligned", fn, (long long)c);
    if (ch.length > INT_MAX - total) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "%s: more than 2^31-1 slots per call", fn);
    total += ch.length;
  }
  if (n_marks < 0 || (n_marks > 0 && (!marks || !mark_counts))) AG_FAIL(AG_ERR_INVALID, "%s: bad mark table", fn);
  for (int64_t j = 0; j < n_marks; ++j)
    if (marks[j] < 0 || marks[j] > total)
      AG_FAIL(AG_ERR_INVALID, "%s: mark %lld at slot %lld outside 0..%lld", fn, (long long)j, (long long)marks[j], (long long)total);
  if (!counts) AG_FAIL(AG_ERR_INVALID, "%s: NULL counts", fn);
  if (total > 0 && !indices) AG_FAIL(AG_ERR_INVALID, "%s: NULL indices", fn);
  *slots = total;
  return AG_OK;
}

// One dictionary call over device chunks: the checking pass over every chunk as a page of its own arrays (one
// synchronisation; it never reads `data`), then `checked` (which may still fill in the chunks' data), then hash.cu's
// dictionary kernels.
template <typename Checked>
ag_status ba_dict_call(const char* fn, int ow, const ag_pq_ba_chunk* chunks, int64_t n_chunks, int64_t slots, const int64_t* marks,
                       int64_t n_marks, uint32_t* indices, int64_t* mark_counts, int64_t* counts, int64_t* d_bad_pos, int64_t* h_bad,
                       cudaStream_t st, Checked checked) {
  if (slots == 0) {
    if (h_bad) *h_bad = AG_NO_ERROR_POS;
    static const int64_t kNoPos = AG_NO_ERROR_POS;
    if (d_bad_pos) AG_TRY(h2d(d_bad_pos, &kNoPos, 8, st));
    AG_TRY(checked((int64_t)0));
    return ba_dict_encode_dev(BaDictPlan{ow, nullptr, nullptr, nullptr, nullptr, nullptr, n_chunks, 0, 0, 0}, chunks, marks, n_marks,
                              indices, mark_counts, counts, st);
  }
  std::vector<ag_pq_enc_page> pages((size_t)n_chunks);
  for (int64_t c = 0; c < n_chunks; ++c) pages[(size_t)c] = ag_pq_enc_page{chunks[c].offset, chunks[c].length, 0, INT64_MAX};
  // DELTA_LENGTH_BYTE_ARRAY: the checking pass that also finds every page's (chunk's) first dense slot
  BaCall c(fn, AG_PQ_ENC_DELTA_LENGTH_BYTE_ARRAY, ow, pages.data(), n_chunks, st);
  AG_TRY(c.check(nullptr, nullptr, d_bad_pos, h_bad, chunks));
  AG_TRY(checked(c.total));
  const BaDictPlan p{ow, nullptr, nullptr, c.a.tile_base, c.a.cnt, c.a.dense, n_chunks, c.a.n_tiles, slots, c.total};
  return ba_dict_encode_dev(p, chunks, marks, n_marks, indices, mark_counts, counts, st);
}

}  // namespace

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_parquet_rle_max_size(int bit_width, int form, int64_t num_values, int64_t* size) {
  AG_TRY(ensure_init());
  AG_TRY(check_rle_args("rle_max_size", bit_width, form, 0, false));
  if (num_values < 0 || num_values > 0x7fffffff) AG_FAIL(AG_ERR_INVALID, "rle_max_size: num_values %lld outside 0..2^31-1", (long long)num_values);
  if (!size) AG_FAIL(AG_ERR_INVALID, "rle_max_size: NULL size");
  *size = rle_bound(bit_width, form, num_values);
  return AG_OK;
}

ag_status ag_parquet_rle_encode_dev(int bit_width, int form, int input, const void* d_values, const ag_pq_enc_page* pages,
                                    int64_t n_pages, uint8_t* d_out, int64_t* d_lengths, int64_t* d_bad_pos, ag_stream_t s) {
  AG_TRY(ensure_init());
  return rle_encode_dev(bit_width, form, input, d_values, pages, n_pages, d_out, d_lengths, d_bad_pos, nullptr, resolve_stream(s));
}

ag_status ag_parquet_rle_encode(int bit_width, int form, int input, const void* values, const ag_pq_enc_page* pages,
                                int64_t n_pages, uint8_t* out, int64_t* lengths, int64_t* bad_pos) {
  AG_TRY(ensure_init());
  if (bad_pos) *bad_pos = AG_NO_ERROR_POS;
  AG_TRY(check_rle_args("rle_encode", bit_width, form, input, true));
  int64_t in_end, out_end;
  AG_TRY(check_pages("rle_encode", pages, n_pages, [&](int64_t n) { return rle_bound(bit_width, form, n); }, &in_end, &out_end));
  if (in_end > 0 && !values) AG_FAIL(AG_ERR_INVALID, "rle_encode: NULL values");
  if (out_end > 0 && !out) AG_FAIL(AG_ERR_INVALID, "rle_encode: NULL output");
  const int64_t in_bytes = input == AG_PQ_RLE_IN_BITMAP ? (in_end + 7) / 8 : in_end * (input == AG_PQ_RLE_IN_I16 ? 2 : 4);
  return encode_host(pages, n_pages, values, in_bytes, out_end, out, lengths, [&](const uint8_t* dv, uint8_t* dout, int64_t* dlen, cudaStream_t st) {
    return rle_encode_dev(bit_width, form, input, dv, pages, n_pages, dout, dlen, nullptr, bad_pos, st);
  });
}

ag_status ag_parquet_delta_max_size(int value_width, int block_size, int miniblocks, int64_t num_values, int64_t* size) {
  AG_TRY(ensure_init());
  AG_TRY(check_delta_args("delta_max_size", value_width, block_size, miniblocks));
  if (num_values < 0 || num_values > 0x7fffffff) AG_FAIL(AG_ERR_INVALID, "delta_max_size: num_values %lld outside 0..2^31-1", (long long)num_values);
  if (!size) AG_FAIL(AG_ERR_INVALID, "delta_max_size: NULL size");
  *size = delta_bound(value_width, block_size, miniblocks, num_values);
  return AG_OK;
}

ag_status ag_parquet_delta_encode_dev(int value_width, int block_size, int miniblocks, const void* d_values, const ag_pq_enc_page* pages,
                                      int64_t n_pages, uint8_t* d_out, int64_t* d_lengths, ag_stream_t s) {
  AG_TRY(ensure_init());
  return delta_encode_dev(value_width, block_size, miniblocks, d_values, pages, n_pages, d_out, d_lengths, resolve_stream(s));
}

ag_status ag_parquet_delta_encode(int value_width, int block_size, int miniblocks, const void* values, const ag_pq_enc_page* pages,
                                  int64_t n_pages, uint8_t* out, int64_t* lengths) {
  AG_TRY(ensure_init());
  AG_TRY(check_delta_args("delta_encode", value_width, block_size, miniblocks));
  int64_t in_end, out_end;
  AG_TRY(check_pages("delta_encode", pages, n_pages, [&](int64_t n) { return delta_bound(value_width, block_size, miniblocks, n); }, &in_end, &out_end));
  if (in_end > 0 && !values) AG_FAIL(AG_ERR_INVALID, "delta_encode: NULL values");
  if (out_end > 0 && !out) AG_FAIL(AG_ERR_INVALID, "delta_encode: NULL output");
  return encode_host(pages, n_pages, values, in_end * value_width, out_end, out, lengths, [&](const uint8_t* dv, uint8_t* dout, int64_t* dlen, cudaStream_t st) {
    return delta_encode_dev(value_width, block_size, miniblocks, dv, pages, n_pages, dout, dlen, st);
  });
}

ag_status ag_parquet_byte_array_max_size(int encoding, int64_t num_values, int64_t value_bytes, int64_t* size) {
  AG_TRY(check_ba_args("byte_array_max_size", encoding, 4));
  if (num_values < 0 || num_values > 0x7fffffff) AG_FAIL(AG_ERR_INVALID, "byte_array_max_size: num_values %lld outside 0..2^31-1", (long long)num_values);
  if (value_bytes < 0 || value_bytes > (1ll << 62)) AG_FAIL(AG_ERR_INVALID, "byte_array_max_size: value_bytes %lld outside 0..2^62", (long long)value_bytes);
  if (!size) AG_FAIL(AG_ERR_INVALID, "byte_array_max_size: NULL size");
  *size = ba_bound(encoding, num_values, value_bytes);
  return AG_OK;
}

ag_status ag_parquet_byte_array_encode_dev(int encoding, int offset_width, const void* d_offsets, const uint8_t* d_data,
                                           const uint8_t* d_valid, const ag_pq_enc_page* pages, int64_t n_pages, uint8_t* d_out,
                                           int64_t* d_lengths, int64_t* d_bad_pos, ag_stream_t s) {
  AG_TRY(ensure_init());
  const char* fn = "byte_array_encode";
  int64_t in_end, out_end;
  AG_TRY(check_ba_call(fn, encoding, offset_width, d_offsets, d_data, pages, n_pages, d_out, &in_end, &out_end));
  const cudaStream_t st = resolve_stream(s);
  if (n_pages == 0) {
    static const int64_t kNoPos = AG_NO_ERROR_POS;
    return d_bad_pos ? h2d(d_bad_pos, &kNoPos, 8, st) : AG_OK;
  }
  BaCall c(fn, encoding, offset_width, pages, n_pages, st);
  AG_TRY(c.check(d_offsets, d_valid, d_bad_pos, nullptr));
  return c.encode(d_data, d_out, d_lengths);
}

ag_status ag_parquet_byte_array_encode(int encoding, int offset_width, const void* offsets, const uint8_t* data, const uint8_t* valid,
                                       const ag_pq_enc_page* pages, int64_t n_pages, uint8_t* out, int64_t* lengths, int64_t* bad_pos) {
  AG_TRY(ensure_init());
  const char* fn = "byte_array_encode";
  if (bad_pos) *bad_pos = AG_NO_ERROR_POS;
  int64_t in_end, out_end;
  AG_TRY(check_ba_call(fn, encoding, offset_width, offsets, data, pages, n_pages, out, &in_end, &out_end));
  if (n_pages == 0) return AG_OK;
  // Stage the slots the pages reach, [s0, in_end) with s0 a multiple of 8 so the validity bytes keep their bit phase.
  // Staged buffers are addressed through pointers moved back by their first element, so the kernels see the caller's
  // slot and data indices.
  int64_t s0 = in_end;
  for (int64_t i = 0; i < n_pages; ++i) if (pages[i].num_values) s0 = std::min(s0, pages[i].in);
  s0 &= ~(int64_t)7;
  const int64_t n_off = in_end > 0 ? in_end - s0 + 1 : 0, n_vb = valid && in_end > 0 ? (in_end - s0 + 7) / 8 : 0;
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  Carve sc;
  const size_t o_off = sc.take((size_t)(n_off * offset_width)), o_vb = sc.take((size_t)n_vb);
  const size_t o_out = sc.take((size_t)out_end), o_len = sc.take((size_t)n_pages * 8);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, sc.size));
  AG_TRY(h2d(d + o_off, static_cast<const uint8_t*>(offsets) + s0 * offset_width, (size_t)(n_off * offset_width), cs));
  AG_TRY(h2d(d + o_vb, valid + s0 / 8, (size_t)n_vb, cs));
  int64_t* d_len = reinterpret_cast<int64_t*>(d + o_len);
  BaCall c(fn, encoding, offset_width, pages, n_pages, cs);
  AG_TRY(c.check(d + o_off - s0 * offset_width, valid ? d + o_vb - s0 / 8 : nullptr, nullptr, bad_pos));
  // the checks passed, so every page's bytes lie between its first and last offsets
  auto off = [&](int64_t i) {
    return offset_width == 4 ? (int64_t) static_cast<const int32_t*>(offsets)[i] : static_cast<const int64_t*>(offsets)[i];
  };
  int64_t lo = INT64_MAX, hi = 0;
  for (int64_t i = 0; i < n_pages; ++i)
    if (pages[i].num_values) { lo = std::min(lo, off(pages[i].in)); hi = std::max(hi, off(pages[i].in + pages[i].num_values)); }
  if (hi < lo) lo = hi;
  uint8_t* dd;
  AG_TRY(t.alloc_t(&dd, (size_t)(hi - lo)));
  AG_TRY(h2d(dd, data + lo, (size_t)(hi - lo), cs));
  AG_TRY(c.encode(dd - lo, d + o_out, d_len));
  std::vector<int64_t> len((size_t)n_pages);
  AG_TRY(d2h(len.data(), d_len, (size_t)n_pages * 8, cs));
  AG_TRY(sync(cs));
  for (int64_t i = 0; i < n_pages; ++i) AG_TRY(d2h(out + pages[i].out, d + o_out + pages[i].out, (size_t)len[(size_t)i], cs));
  if (lengths) memcpy(lengths, len.data(), (size_t)n_pages * 8);
  return sync(cs);
}

ag_status ag_parquet_byte_array_dict_encode_dev(int offset_width, const ag_pq_ba_chunk* chunks, int64_t n_chunks, const int64_t* marks,
                                                int64_t n_marks, uint32_t* d_indices, int64_t* d_mark_counts, int64_t* d_counts,
                                                int64_t* d_bad_pos, ag_stream_t s) {
  const char* fn = "byte_array_dict_encode";
  int64_t slots;
  AG_TRY(check_ba_dict_call(fn, offset_width, chunks, n_chunks, marks, n_marks, d_indices, d_mark_counts, d_counts, &slots));
  AG_TRY(ensure_init());
  return ba_dict_call(fn, offset_width, chunks, n_chunks, slots, marks, n_marks, d_indices, d_mark_counts, d_counts, d_bad_pos, nullptr,
                      resolve_stream(s), [](int64_t) { return AG_OK; });
}

ag_status ag_parquet_byte_array_dict_encode(int offset_width, const ag_pq_ba_chunk* chunks, int64_t n_chunks, const int64_t* marks,
                                            int64_t n_marks, uint32_t* indices, int64_t* mark_counts, int64_t* counts, int64_t* bad_pos) {
  const char* fn = "byte_array_dict_encode";
  if (bad_pos) *bad_pos = AG_NO_ERROR_POS;
  int64_t slots;
  AG_TRY(check_ba_dict_call(fn, offset_width, chunks, n_chunks, marks, n_marks, indices, mark_counts, counts, &slots));
  AG_TRY(ensure_init());
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  // Each chunk's offsets, validity bytes, first words and (once the checking pass has passed) data are staged at
  // pointers moved back by their first element, so the kernels see the chunk's own slot numbering.  The data staged is
  // [offsets[offset], offsets[offset + length]), which holds every value once the offsets are checked.
  const int ow = offset_width;
  std::vector<ag_pq_ba_chunk> dc((size_t)n_chunks);
  for (int64_t c = 0; c < n_chunks; ++c) {
    const ag_pq_ba_chunk& ch = chunks[c];
    ag_pq_ba_chunk& d = dc[(size_t)c];
    d = ch;
    if (ch.length == 0) continue;
    const int64_t v0 = ch.offset >> 3, nv = ch.valid ? ((ch.offset + ch.length + 7) >> 3) - v0 : 0;
    const int64_t f0 = ch.offset >> 5, nf = ((ch.offset + ch.length + 31) >> 5) - f0;
    uint8_t *o, *v = nullptr, *f;
    AG_TRY(t.alloc_t(&o, (size_t)(ch.length + 1) * ow));
    AG_TRY(h2d(o, static_cast<const uint8_t*>(ch.offsets) + ch.offset * ow, (size_t)(ch.length + 1) * ow, cs));
    if (ch.valid) { AG_TRY(t.alloc_t(&v, (size_t)nv)); AG_TRY(h2d(v, ch.valid + v0, (size_t)nv, cs)); }
    AG_TRY(t.alloc_t(&f, (size_t)nf * 4));
    d.offsets = o - ch.offset * ow;
    d.valid = ch.valid ? v - v0 : nullptr;
    d.data = nullptr;
    d.first = f - f0 * 4;
  }
  Carve sc;
  const size_t o_idx = sc.take((size_t)slots * 4), o_mc = sc.take((size_t)n_marks * 16), o_cnt = sc.take(24);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, sc.size));
  int64_t valid = 0;
  auto stage_data = [&](int64_t nv) {
    valid = nv;
    for (int64_t c = 0; c < n_chunks; ++c) {
      const ag_pq_ba_chunk& ch = chunks[c];
      if (ch.length == 0) continue;
      auto off = [&](int64_t i) {
        return ow == 4 ? (int64_t) static_cast<const int32_t*>(ch.offsets)[i] : static_cast<const int64_t*>(ch.offsets)[i];
      };
      const int64_t lo = off(ch.offset), hi = off(ch.offset + ch.length);
      uint8_t* dd;
      AG_TRY(t.alloc_t(&dd, (size_t)(hi - lo)));
      AG_TRY(h2d(dd, ch.data + lo, (size_t)(hi - lo), cs));
      dc[(size_t)c].data = dd - lo;
    }
    return AG_OK;
  };
  AG_TRY(ba_dict_call(fn, ow, dc.data(), n_chunks, slots, marks, n_marks, reinterpret_cast<uint32_t*>(d + o_idx),
                      reinterpret_cast<int64_t*>(d + o_mc), reinterpret_cast<int64_t*>(d + o_cnt), nullptr, bad_pos, cs, stage_data));
  AG_TRY(d2h(indices, d + o_idx, (size_t)valid * 4, cs));
  AG_TRY(d2h(mark_counts, d + o_mc, (size_t)n_marks * 16, cs));
  AG_TRY(d2h(counts, d + o_cnt, 24, cs));
  for (int64_t c = 0; c < n_chunks; ++c) {
    const ag_pq_ba_chunk& ch = chunks[c];
    if (ch.length == 0) continue;
    const int64_t f0 = ch.offset >> 5, nf = ((ch.offset + ch.length + 31) >> 5) - f0;
    AG_TRY(d2h(ch.first + f0 * 4, dc[(size_t)c].first + f0 * 4, (size_t)nf * 4, cs));
  }
  return sync(cs);
}

}  // extern "C"
