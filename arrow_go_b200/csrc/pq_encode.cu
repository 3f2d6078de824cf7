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
#include <climits>

#include "host_stage.cuh"
#include "pq_window.cuh"

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
int64_t delta_bound(int width, int block, int mini, int64_t n) {
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

}  // extern "C"
