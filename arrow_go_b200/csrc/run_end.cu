// run_end.cu — run_end_encode / run_end_decode for fixed-width and boolean columns on sm_90a.
//
// Replaces the fixed-width and boolean loops of arrow/compute/internal/kernels/vector_run_end_encode.go:
// CountNumberOfRuns (:114-141), PreallocOutput (:143-180) and WriteEncodedRuns (:86-112) for the encode, and
// decodeBool / decodeFixedWidth ExpandAllRuns (:591-719) for the decode.
//
// Run rule (vector_run_end_encode.go:96-105): rows i-1 and i share a run iff their validity bits are equal and their
// values compare equal with the physical type's `==` — also under a null (the payload is read whatever the validity).
// Floats use IEEE ==: every NaN row starts a run, +0.0 and -0.0 share one.  Run r has run_ends[r] = the first row of
// run r+1 (n for the last run), values[r] = the value of its first row and validity bit r = that row's validity.
//
// Rows are handled in GROUPS: the G rows of one 16-byte load (G = 16 / sizeof(T)) or of one 32-bit word of a boolean
// column (G = 32).  Groups are numbered on the 16-byte grid of the values buffer, so every interior group is one
// aligned vector load: group q holds rows q*G - h .. q*G - h + G-1, h = the row phase of `vals` inside its 16 bytes.
// Rows outside [0, n) of the first and last group are masked.  A group's first row is compared with the last row of
// the group before it (the previous lane's, through a shuffle; lane 0 loads it).
//
// Encode: a count kernel (one streaming pass: runs and null runs), then one single-pass compaction with the decoupled
// look-back of filter.cu (lookback.cuh).  A block tile is 8 warps x kRSteps warp steps x 32 groups; the boundary
// rows of a warp step get consecutive ranks, a boundary of rank r > 0 at row i writes run_ends[r-1] = i, every
// boundary writes values[r]; the validity bits (and a boolean column's value bits) of the tile's runs are gathered in
// shared memory and written as whole words, atomicOr only on the tile's two edge words.
// Bytes: two reads of the column (count + encode) + runs x (value width + run-end width) written.
//
// Decode: output tiles of kDTileRows rows.  A one-thread kernel finds the runs [first, last] that cover
// [offset, offset+length); a second kernel binary-searches, one thread per tile and all tiles at once, the run of each
// tile's first row in run_ends[first..last].  A decode block stages the run ends of its tile, clipped to the tile,
// in shared memory with each run's validity (and BOOL value) bit (at most kDTileRows + 1 of them: a valid run is at
// least one row long); each thread resolves its rows against that segment and writes 16-byte vectors, boolean output
// and validity as whole 32-bit words.  The run ends of [first, last] are checked to increase strictly (every block checks
// its share); malformed run ends lower the error word and never make a kernel read or write out of bounds.
// Bytes: runs x (value width + run-end width) read + length x value width written.
#include "common.cuh"
#include "lookback.cuh"

namespace ag {

constexpr int kRThreads = 256;
constexpr int kRWarps = kRThreads / 32;
constexpr int kRSteps = 8;                                 // warp steps per tile
constexpr int kRGroupsPerTile = kRWarps * kRSteps * 32;    // 2048 groups: 32 KB of fixed-width values
constexpr int kCountSteps = 4;                             // warp steps per iteration of the count kernel
constexpr int kDTileRows = 4096;
constexpr int kDThreads = 256;

// ---------------------------------------------------------------- groups ----------------
template <typename T> struct GroupOf {              // fixed-width values
  static constexpr int G = 16 / (int)sizeof(T);
  T v[G];
};
struct BoolGroup {                                  // boolean values: one 32-bit word
  static constexpr int G = 32;
  uint32_t v;
};

struct EncodeParams {
  const void* vals;          // element 0 of the span (vals + offset); boolean: the bitmap, rows at bit vbit
  int64_t vbit;              // boolean values: bit offset of row 0
  int h;                     // row phase of `vals` inside its 16 bytes (0 for booleans)
  const uint8_t* valid;      // may be NULL
  int64_t voff;              // bit offset of row 0 in `valid`
  int64_t n;
  void* run_ends;            // R[capacity]
  void* out;                 // T[capacity], or a pre-zeroed 4-byte aligned bitmap of ceil(capacity/32) words
  uint32_t* out_valid;       // pre-zeroed, 4-byte aligned, ceil(capacity/32) words (may be NULL)
  int64_t capacity;
  unsigned long long* counts;   // [0] runs, [1] null runs
  unsigned long long* status;
  unsigned long long* gstatus;
  int64_t n_groups, n_tiles;
};

template <typename T>
__device__ __forceinline__ bool same_value(T a, T b) { return a == b; }   // IEEE == for floats (NaN != NaN, -0 == +0)

// 32 bits of an LSB-first bitmap from bit `bit` (may be negative), reading only bytes [lo, hi); other bits are 0.
// bitmap_load32 with its edge path inlined: the out-of-line call costs the encode kernels a spill.
__device__ __forceinline__ uint32_t load_bits32(const uint8_t* __restrict__ base, int64_t bit, int64_t lo, int64_t hi) {
  const int64_t mis = (int64_t)(reinterpret_cast<uintptr_t>(base) & 3);
  const uint8_t* abase = base - mis;
  const int64_t abit = bit + mis * 8;
  const int64_t w = abit >> 5;
  const int sh = (int)(abit & 31);
  lo += mis; hi += mis;
  const int64_t b0 = w * 4;
  uint32_t w0, w1;
  if (b0 >= lo && b0 + 8 <= hi) {
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(abase + b0);
    w0 = wp[0]; w1 = wp[1];
  } else {
    w0 = w1 = 0u;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int64_t b = b0 + k;
      const uint32_t v = (b >= lo && b < hi) ? (uint32_t)abase[b] : 0u;
      if (k < 4) w0 |= v << (8 * k); else w1 |= v << (8 * (k - 4));
    }
  }
  return sh ? __funnelshift_r(w0, w1, sh) : w0;
}

// Load group q: its values, the validity bits of its rows (bit e = row q*G-h+e; all ones without a bitmap) and the
// in-range mask.
template <typename T>
__device__ __forceinline__ void load_group(const EncodeParams& p, int64_t q, GroupOf<T>& g, uint32_t& m, uint32_t& range) {
  constexpr int G = GroupOf<T>::G;
  const int64_t row0 = q * G - p.h;
  const T* base = reinterpret_cast<const T*>(p.vals);
  if (row0 >= 0 && row0 + G <= p.n) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(base + row0));
    memcpy(g.v, &u, 16);
    range = G == 32 ? 0xffffffffu : ((1u << G) - 1u);
  } else {
    range = 0;
#pragma unroll
    for (int e = 0; e < G; ++e) {
      const int64_t r = row0 + e;
      g.v[e] = T(0);
      if (r >= 0 && r < p.n) { g.v[e] = base[r]; range |= 1u << e; }
    }
  }
  m = p.valid ? load_bits32(p.valid, p.voff + row0, p.voff >> 3, (p.voff + p.n + 7) >> 3) : 0xffffffffu;
}
__device__ __forceinline__ void load_group(const EncodeParams& p, int64_t q, BoolGroup& g, uint32_t& m, uint32_t& range) {
  const int64_t row0 = q * 32;
  const int64_t rem = p.n - row0;
  range = rem >= 32 ? 0xffffffffu : bit_range_mask(0, (int)rem);
  const uint8_t* bits = reinterpret_cast<const uint8_t*>(p.vals);
  g.v = load_bits32(bits, p.vbit + row0, p.vbit >> 3, (p.vbit + p.n + 7) >> 3);
  m = p.valid ? load_bits32(p.valid, p.voff + row0, p.voff >> 3, (p.voff + p.n + 7) >> 3) : 0xffffffffu;
}

template <typename T> __device__ __forceinline__ T last_of(const GroupOf<T>& g) { return g.v[GroupOf<T>::G - 1]; }
__device__ __forceinline__ uint32_t last_of(const BoolGroup& g) { return g.v >> 31; }

// Value and validity of row r (0 <= r < n), loaded directly: the predecessor of a warp step's first group.
template <typename T>
__device__ __forceinline__ T load_row(const EncodeParams& p, int64_t r, const GroupOf<T>*) { return reinterpret_cast<const T*>(p.vals)[r]; }
__device__ __forceinline__ uint32_t load_row(const EncodeParams& p, int64_t r, const BoolGroup*) {
  return (uint32_t)bit_is_set(reinterpret_cast<const uint8_t*>(p.vals), p.vbit + r);
}

// Boundary bits of a group (bit e: row q*G-h+e starts a run).  prev_v / prev_m: the row before the group's first row
// (unused for the group of row 0, which always starts a run).
template <typename T>
__device__ __forceinline__ uint32_t boundaries(const GroupOf<T>& g, uint32_t m, uint32_t range, T prev_v, uint32_t prev_m, int64_t row0) {
  constexpr int G = GroupOf<T>::G;
  uint32_t b = 0;
#pragma unroll
  for (int e = 0; e < G; ++e) {
    const T pv = e == 0 ? prev_v : g.v[e - 1];
    const uint32_t pm = e == 0 ? prev_m : (m >> (e - 1)) & 1u;
    const bool first = row0 + e == 0;
    if (first || pm != ((m >> e) & 1u) || !same_value(pv, g.v[e])) b |= 1u << e;
  }
  return b & range;
}
__device__ __forceinline__ uint32_t boundaries(const BoolGroup& g, uint32_t m, uint32_t range, uint32_t prev_v, uint32_t prev_m, int64_t row0) {
  const uint32_t dv = g.v ^ ((g.v << 1) | prev_v);
  const uint32_t dm = m ^ ((m << 1) | prev_m);
  return (dv | dm | (row0 == 0 ? 1u : 0u)) & range;
}

template <typename T> struct GroupTraits { using Group = GroupOf<T>; using Elem = T; };
struct BoolTag {};
template <> struct GroupTraits<BoolTag> { using Group = BoolGroup; using Elem = uint32_t; };

// One warp step over groups q0 + lane: the boundary bits and the null-run starts of this lane's group.
template <typename V>
__device__ __forceinline__ void step_bounds(const EncodeParams& p, int64_t q, int lane, typename GroupTraits<V>::Group& g,
                                            uint32_t& m, uint32_t& b) {
  using Group = typename GroupTraits<V>::Group;
  using E = typename GroupTraits<V>::Elem;
  constexpr int G = Group::G;
  uint32_t range = 0;
  if (q < p.n_groups) load_group(p, q, g, m, range);
  else { m = 0; memset(&g, 0, sizeof(g)); }
  const int64_t row0 = q * G - (int64_t)p.h;
  E pv = __shfl_up_sync(0xffffffffu, last_of(g), 1);
  uint32_t pm = __shfl_up_sync(0xffffffffu, (m >> (G - 1)) & 1u, 1);
  if (lane == 0 && row0 >= 1 && row0 - 1 < p.n) {
    pv = load_row(p, row0 - 1, (const Group*)nullptr);
    pm = p.valid ? (uint32_t)bit_is_set(p.valid, p.voff + row0 - 1) : 1u;
  }
  b = (q < p.n_groups) ? boundaries(g, m, range, pv, pm, row0) : 0u;
}

// L2 prefetch of a warp's kRSteps warp steps from group q0 (lanes 0, 8, 16, 24: one 128-byte line each per step) and
// of their validity bytes.
template <int G>
__device__ __forceinline__ void prefetch_tile(const EncodeParams& p, int64_t q0, int lane) {
  const char* vbase = G == 32 ? reinterpret_cast<const char*>(p.vals) + ((p.vbit + q0 * 32) >> 3)
                              : reinterpret_cast<const char*>(p.vals) + (q0 * G - p.h) * (16 / G);
  const int64_t vbytes = G == 32 ? (p.vbit + p.n + 7) / 8 - (p.vbit + q0 * 32) / 8 : (p.n - (q0 * G - p.h)) * (16 / G);
#pragma unroll
  for (int s = 0; s < kRSteps; ++s) {
    const int64_t off = (int64_t)s * 32 * (G == 32 ? 4 : 16) + lane * (G == 32 ? 4 : 16);
    if (off < vbytes) asm volatile("prefetch.global.L2 [%0];" :: "l"(vbase + off));
  }
  if (p.valid) {
    const int64_t bit = p.voff + q0 * G - p.h;
    const int64_t byte = (bit < 0 ? 0 : bit) >> 3, end = (p.voff + p.n + 7) >> 3;
    const int64_t off = byte + lane * 16;   // lanes 0, 8, 16, 24: the 512 bytes from the warp's first validity byte
    if (off < end) asm volatile("prefetch.global.L2 [%0];" :: "l"(p.valid + off));
  }
}

// ---------------------------------------------------------------- count -----------------
template <typename V>
__global__ void __launch_bounds__(kRThreads)
run_end_count_kernel(const EncodeParams p) {
  using Group = typename GroupTraits<V>::Group;
  const int lane = threadIdx.x & 31;
  unsigned long long runs = 0, null_runs = 0;
  const int64_t stride = (int64_t)gridDim.x * kRThreads;
  // whole warps iterate together (the shuffles need every lane)
  // each warp takes kCountSteps consecutive warp steps per iteration: that many loads in flight per thread
  for (int64_t q0 = ((int64_t)blockIdx.x * kRThreads + (threadIdx.x & ~31)) * kCountSteps; q0 < p.n_groups; q0 += stride * kCountSteps) {
    Group g[kCountSteps]; uint32_t m[kCountSteps], b[kCountSteps];
#pragma unroll
    for (int u = 0; u < kCountSteps; ++u) step_bounds<V>(p, q0 + u * 32 + lane, lane, g[u], m[u], b[u]);
#pragma unroll
    for (int u = 0; u < kCountSteps; ++u) {
      runs += __popc(b[u]);
      null_runs += __popc(b[u] & ~m[u]);
    }
  }
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) {
    runs += __shfl_xor_sync(0xffffffffu, runs, s);
    null_runs += __shfl_xor_sync(0xffffffffu, null_runs, s);
  }
  __shared__ unsigned long long sm[2][kRWarps];
  if (lane == 0) { sm[0][threadIdx.x >> 5] = runs; sm[1][threadIdx.x >> 5] = null_runs; }
  __syncthreads();
  if (threadIdx.x < 2) {
    unsigned long long t = 0;
#pragma unroll
    for (int w = 0; w < kRWarps; ++w) t += sm[threadIdx.x][w];
    if (t) atomicAdd(p.counts + threadIdx.x, t);
  }
}

// ---------------------------------------------------------------- encode ----------------
// Tile t = groups [t * kRGroupsPerTile, ...); warp w owns kRSteps consecutive warp steps of it.  Static tile order
// (block b: tiles b, b+G, ...) and one resident wave (cooperative launch), as filter_kernel.
template <typename V, typename R>
__global__ void __launch_bounds__(kRThreads, 2)
run_end_encode_kernel(const EncodeParams p) {
  using Group = typename GroupTraits<V>::Group;
  constexpr int G = Group::G;
  constexpr bool kBool = std::is_same<V, BoolTag>::value;
  constexpr int kStageWords = kRGroupsPerTile * G / 32 + 2;   // the tile's runs, from the word of its first rank
  __shared__ uint32_t s_valid[kStageWords];
  __shared__ uint32_t s_bits[kBool ? kStageWords : 1];
  __shared__ uint32_t s_warp[kRWarps];
  __shared__ unsigned long long s_base;
  __shared__ unsigned long long s_null_runs;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  R* __restrict__ run_ends = reinterpret_cast<R*>(p.run_ends);
  const long long cap_words = (p.capacity + 31) >> 5;
  if (threadIdx.x == 0) s_null_runs = 0;
  __syncthreads();
  for (int64_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    for (int i = threadIdx.x; i < kStageWords; i += kRThreads) { s_valid[i] = 0u; if (kBool) s_bits[i] = 0u; }
    Group g[kRSteps];
    uint32_t m[kRSteps], b[kRSteps];
    const int64_t q0 = tile * kRGroupsPerTile + (int64_t)warp * kRSteps * 32;
#pragma unroll
    for (int s = 0; s < kRSteps; ++s) step_bounds<V>(p, q0 + s * 32 + lane, lane, g[s], m[s], b[s]);
    // the block's next tile heads for L2 now, so that HBM streams while this tile waits for its prefix
    if (tile + gridDim.x < p.n_tiles && (lane & 7) == 0) prefetch_tile<G>(p, q0 + (int64_t)gridDim.x * kRGroupsPerTile, lane);
    // ranks: row order is (warp, step, lane, bit)
    uint32_t excl[kRSteps];
    uint32_t warp_total = 0, nulls = 0;
#pragma unroll
    for (int s = 0; s < kRSteps; ++s) {
      const uint32_t c = __popc(b[s]);
      nulls += __popc(b[s] & ~m[s]);
      uint32_t incl = c;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
      }
      excl[s] = warp_total + incl - c;
      warp_total += __shfl_sync(0xffffffffu, incl, 31);
    }
    nulls = __reduce_add_sync(0xffffffffu, nulls);
    if (lane == 0) { s_warp[warp] = warp_total; if (nulls) atomicAdd(&s_null_runs, (unsigned long long)nulls); }
    __syncthreads();
    uint32_t warp_base = 0, tile_total = 0;
#pragma unroll
    for (int w = 0; w < kRWarps; ++w) {
      const uint32_t t = s_warp[w];
      if (w < warp) warp_base += t;
      tile_total += t;
    }
    if (warp == 0) {
      const unsigned long long base = lookback<true>(p.status, p.gstatus, tile, tile_total, lane);
      if (lane == 0) {
        s_base = base;
        if (tile == p.n_tiles - 1) {   // the last tile knows the number of runs: the last run end is n
          const unsigned long long total = base + tile_total;
          p.counts[0] = total;
          if ((long long)total - 1 < p.capacity) run_ends[total - 1] = (R)p.n;
        }
      }
    }
    __syncthreads();
    const unsigned long long tbase = s_base;
    const unsigned long long word0 = tbase >> 5;
#pragma unroll
    for (int s = 0; s < kRSteps; ++s) {
      const unsigned long long r0 = tbase + warp_base + excl[s];
      const int64_t row0 = (q0 + s * 32 + lane) * G - (int64_t)p.h;
      if constexpr (kBool) {
        // a BOOL group is one register: walk its boundary bits
        uint32_t bits = b[s];
        unsigned long long r = r0;
        while (bits) {
          const int e = __ffs(bits) - 1;
          bits &= bits - 1;
          if (r > 0 && (long long)r <= p.capacity) run_ends[r - 1] = (R)(row0 + e);
          if ((long long)r < p.capacity) {
            const unsigned sw = (unsigned)((r >> 5) - word0);
            if (p.out_valid && ((m[s] >> e) & 1u)) atomicOr(&s_valid[sw], 1u << (r & 31));
            if ((g[s].v >> e) & 1u) atomicOr(&s_bits[sw], 1u << (r & 31));
          }
          ++r;
        }
      } else {
        // e unrolled, so the values stay in registers
#pragma unroll
        for (int e = 0; e < G; ++e) {
          if (!((b[s] >> e) & 1u)) continue;
          const unsigned long long r = r0 + __popc(b[s] & ((1u << e) - 1u));
          if (r > 0 && (long long)r <= p.capacity) run_ends[r - 1] = (R)(row0 + e);
          if ((long long)r >= p.capacity) continue;
          if (p.out_valid && ((m[s] >> e) & 1u)) atomicOr(&s_valid[(unsigned)((r >> 5) - word0)], 1u << (r & 31));
          reinterpret_cast<typename GroupTraits<V>::Elem*>(p.out)[r] = g[s].v[e];
        }
      }
    }
    __syncthreads();
    // the tile's words: [word0, last word of its last run]; edge words are shared with the neighbouring tiles
    if (tile_total > 0) {
      const unsigned long long last = (tbase + tile_total - 1) >> 5;
      const int nw = (int)(last - word0 + 1);
      for (int i = threadIdx.x; i < nw; i += kRThreads) {
        const unsigned long long wi = word0 + i;
        if ((long long)wi >= cap_words) break;
        const bool edge = i == 0 || i == nw - 1;
        if (p.out_valid) {
          if (edge) { if (s_valid[i]) atomicOr(p.out_valid + wi, s_valid[i]); }
          else p.out_valid[wi] = s_valid[i];
        }
        if constexpr (kBool) {
          uint32_t* bout = reinterpret_cast<uint32_t*>(p.out);
          if (edge) { if (s_bits[i]) atomicOr(bout + wi, s_bits[i]); }
          else bout[wi] = s_bits[i];
        }
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0 && s_null_runs) atomicAdd(p.counts + 1, s_null_runs);
}

static ag_status encode_params(int type, const void* vals, const uint8_t* valid, int64_t offset, int64_t n, EncodeParams* p,
                               const char* who) {
  if (n < 0 || offset < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative length or offset", who);
  if (n > 0 && !vals) AG_FAIL(AG_ERR_INVALID, "%s: NULL values", who);
  *p = EncodeParams{};
  p->valid = valid; p->voff = offset; p->n = n;
  if (type == AG_TYPE_BOOL) {
    p->vals = vals; p->vbit = offset; p->h = 0;
    p->n_groups = (n + 31) / 32;
    return AG_OK;
  }
  const int w = type_width(type);
  if (w == 0) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "%s: type id %d (boolean and the 10 numeric types only)", who, type);
  const char* base = static_cast<const char*>(vals) + offset * w;
  if ((uintptr_t)base % w) AG_FAIL(AG_ERR_INVALID, "%s: values not aligned to the element width", who);
  const int G = 16 / w;
  p->h = (int)(((uintptr_t)base & 15) / w);
  p->vals = base;
  p->n_groups = (n + p->h + G - 1) / G;
  return AG_OK;
}

// Visit the value type: BoolTag or the exact numeric type.
template <typename F>
static ag_status visit_value(int type, F&& f, const char* who) {
  if (type == AG_TYPE_BOOL) return f(TypeTag<BoolTag>{});
  return visit_type(type, f, [&] { AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "%s: type id %d (boolean and the 10 numeric types only)", who, type); });
}
template <typename F>
static ag_status visit_run_end(int run_end_type, F&& f, const char* who) {
  switch (run_end_type) {
    case AG_TYPE_INT16: return f(TypeTag<int16_t>{});
    case AG_TYPE_INT32: return f(TypeTag<int32_t>{});
    case AG_TYPE_INT64: return f(TypeTag<int64_t>{});
    default: AG_FAIL(AG_ERR_INVALID, "%s: bad run end type %d", who, run_end_type);
  }
}
static ag_status check_run_end_length(int run_end_type, int64_t n, const char* who) {   // validateRunEndType :437-444
  const int64_t mx = run_end_type == AG_TYPE_INT16 ? INT16_MAX : (run_end_type == AG_TYPE_INT32 ? INT32_MAX : INT64_MAX);
  if (n > mx) AG_FAIL(AG_ERR_INVALID, "%s: cannot run-end encode arrays with more elements than the run end type can hold: %lld", who, (long long)mx);
  return AG_OK;
}

ag_status run_end_count_dev(int type, const void* vals, const uint8_t* valid, int64_t offset, int64_t n, int64_t* d_counts, cudaStream_t st) {
  if (!d_counts) AG_FAIL(AG_ERR_INVALID, "run_end_count: NULL counts");
  EncodeParams p;
  AG_TRY(encode_params(type, vals, valid, offset, n, &p, "run_end_count"));
  p.counts = reinterpret_cast<unsigned long long*>(d_counts);
  AG_CUDA_TRY(cudaMemsetAsync(d_counts, 0, 2 * sizeof(int64_t), st));
  if (n == 0) return AG_OK;
  return visit_value(type, [&](auto tag) {
    using V = typename decltype(tag)::type;
    const int grid = grid_for(p.n_groups, kRThreads * kCountSteps, 8);
    run_end_count_kernel<V><<<grid, kRThreads, 0, st>>>(p);
    return check_launch("run_end_count_kernel");
  }, "run_end_count");
}

ag_status run_end_encode_dev(int type, int run_end_type, const void* vals, const uint8_t* valid, int64_t offset, int64_t n,
                             void* run_ends, void* out, uint8_t* out_valid, int64_t capacity, int64_t* d_counts, cudaStream_t st) {
  const char* who = "run_end_encode";
  if (!d_counts) AG_FAIL(AG_ERR_INVALID, "%s: NULL counts", who);
  if (capacity < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative capacity", who);
  EncodeParams p;
  AG_TRY(encode_params(type, vals, valid, offset, n, &p, who));
  AG_TRY(visit_run_end(run_end_type, [](auto) { return AG_OK; }, who));
  AG_TRY(check_run_end_length(run_end_type, n, who));
  if (capacity > 0 && (!run_ends || !out)) AG_FAIL(AG_ERR_INVALID, "%s: NULL run_ends / values output", who);
  if (valid && capacity > 0 && !out_valid) AG_FAIL(AG_ERR_INVALID, "%s: an input with a validity bitmap needs an output validity bitmap", who);
  if (out_valid && ((uintptr_t)out_valid & 3)) AG_FAIL(AG_ERR_INVALID, "%s: out_valid must be 4-byte aligned", who);
  if (type == AG_TYPE_BOOL && ((uintptr_t)out & 3)) AG_FAIL(AG_ERR_INVALID, "%s: boolean output bitmap must be 4-byte aligned", who);
  if (type != AG_TYPE_BOOL && ((uintptr_t)out % type_width(type))) AG_FAIL(AG_ERR_INVALID, "%s: output not aligned to the element width", who);
  p.run_ends = run_ends; p.out = out; p.capacity = capacity;
  p.out_valid = valid ? reinterpret_cast<uint32_t*>(out_valid) : nullptr;
  p.counts = reinterpret_cast<unsigned long long*>(d_counts);
  AG_CUDA_TRY(cudaMemsetAsync(d_counts, 0, 2 * sizeof(int64_t), st));
  if (n == 0) return AG_OK;
  const size_t cap_bytes = (size_t)((capacity + 31) >> 5) * 4;
  if (p.out_valid && cap_bytes) AG_CUDA_TRY(cudaMemsetAsync(p.out_valid, 0, cap_bytes, st));
  if (type == AG_TYPE_BOOL && cap_bytes) AG_CUDA_TRY(cudaMemsetAsync(out, 0, cap_bytes, st));
  Workspace* ws;
  AG_TRY(get_workspace(st, &ws));
  WorkspaceLock ws_lock(ws);
  p.n_tiles = (p.n_groups + kRGroupsPerTile - 1) / kRGroupsPerTile;
  const size_t n_status = (size_t)p.n_tiles + (size_t)((p.n_tiles + 31) >> 5);
  AG_TRY(ensure_tile_status(ws, n_status, st));
  p.status = ws->tile_status;
  p.gstatus = p.status + p.n_tiles;
  AG_CUDA_TRY(cudaMemsetAsync(p.status, 0, n_status * sizeof(unsigned long long), st));
  return visit_value(type, [&](auto vtag) {
    using V = typename decltype(vtag)::type;
    return visit_run_end(run_end_type, [&](auto rtag) {
      using R = typename decltype(rtag)::type;
      const void* fn = (const void*)run_end_encode_kernel<V, R>;
      void* args[] = {(void*)&p};
      AG_CUDA_TRY(cudaLaunchCooperativeKernel(fn, dim3(grid_one_wave(run_end_encode_kernel<V, R>, kRThreads, p.n_tiles)), dim3(kRThreads), args, 0, st));
      return check_launch("run_end_encode_kernel");
    }, who);
  }, who);
}

// ---------------------------------------------------------------- decode ----------------
struct DecodeParams {
  const void* run_ends;      // R[n_runs]
  int64_t n_runs;
  const void* vals;          // the values child's buffer (element 0)
  const uint8_t* valid;      // may be NULL
  int64_t voff;              // the values child's offset
  int64_t offset, length;    // the logical slice
  void* out;                 // T[length] at offset 0, or a boolean bitmap of ceil(length/32) words
  uint32_t* out_valid;       // ceil(length/32) words (NULL when `valid` is NULL)
  unsigned long long* null_count;
  long long* err;            // error word: lowered to the index of the first malformed run end found
  int64_t* bounds;           // [0] first, [1] last run of the slice; -1 when the slice is malformed
  int64_t* tile_first;       // [t]: the run that covers the first row of output tile t
  int64_t n_tiles;
};

template <typename R>
__device__ __forceinline__ int64_t upper_bound_runs(const R* re, int64_t lo, int64_t hi, int64_t x) {   // first p in [lo, hi) with re[p] > x
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if ((int64_t)re[mid] > x) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// One thread: the runs covering the first and the last row of the slice.
template <typename R>
__global__ void run_end_bounds_kernel(const DecodeParams p) {
  const R* re = reinterpret_cast<const R*>(p.run_ends);
  const int64_t a = p.offset, b = p.offset + p.length - 1;
  const int64_t first = upper_bound_runs(re, 0, p.n_runs, a);
  const int64_t last = upper_bound_runs(re, 0, p.n_runs, b);
  long long bad = AG_NO_ERROR_POS;
  if (first >= p.n_runs || last >= p.n_runs) bad = p.n_runs;                       // the run ends stop before offset+length
  else if (last < first || last - first + 1 > p.length) bad = first;                // not strictly increasing
  else if (first > 0 && (int64_t)re[first - 1] > a) bad = first;
  else if (last > first && (int64_t)re[last - 1] > b) bad = last;
  if (bad != AG_NO_ERROR_POS) {
    atomicMin(p.err, bad);
    p.bounds[0] = p.bounds[1] = -1;
  } else {
    p.bounds[0] = first;
    p.bounds[1] = last;
  }
}

// One thread per output tile: the run that covers its first row, searched in run_ends[first..last] (all tiles at once,
// so the dependent loads of the searches overlap).
template <typename R>
__global__ void __launch_bounds__(kDThreads)
run_end_tile_first_kernel(const DecodeParams p) {
  const int64_t t = (int64_t)blockIdx.x * kDThreads + threadIdx.x;
  const int64_t first = p.bounds[0], last = p.bounds[1];
  if (t >= p.n_tiles || first < 0) return;
  const int64_t a = p.offset + t * kDTileRows;
  const int64_t hi = first + t * kDTileRows + 1;   // a valid run covers at least one row
  p.tile_first[t] = upper_bound_runs(reinterpret_cast<const R*>(p.run_ends), first, hi < last + 1 ? hi : last + 1, a);
}

template <typename V, typename R>
__global__ void __launch_bounds__(kDThreads)
run_end_decode_kernel(const DecodeParams p) {
  using E = typename GroupTraits<V>::Elem;
  constexpr bool kBool = std::is_same<V, BoolTag>::value;
  constexpr int G = GroupTraits<V>::Group::G;
  constexpr int kGroups = kDTileRows / G;
  __shared__ int32_t s_end[kDTileRows + 1];   // the tile's run ends, clipped to the tile and made tile-relative
  __shared__ uint8_t s_flag[kDTileRows + 1];  // bit 0: the run's validity, bit 1: a BOOL run's value
  __shared__ int64_t s_p0;
  __shared__ int s_seg;
  const R* re = reinterpret_cast<const R*>(p.run_ends);
  const int64_t first = p.bounds[0], last = p.bounds[1];
  if (first < 0) return;
  const int64_t tile = blockIdx.x;
  // this block's share of the strict-increase check: run ends (i-1, i), i in (first, last]
  for (int64_t i = first + 1 + tile * kDTileRows + threadIdx.x; i <= last && i < first + 1 + (tile + 1) * kDTileRows; i += kDThreads)
    if ((int64_t)re[i - 1] >= (int64_t)re[i]) atomicMin(p.err, (long long)i);
  const int64_t row0 = tile * kDTileRows;
  const int rows = (int)(p.length - row0 < kDTileRows ? p.length - row0 : kDTileRows);
  const int64_t a = p.offset + row0;
  if (threadIdx.x == 0) {
    // runs p0 .. p1: from the run of the tile's first row to the run of the next tile's first row (which may start
    // exactly there: its clipped end is then `rows` like its predecessor's, and no row picks it)
    const int64_t p0 = p.tile_first[tile];
    const int64_t p1 = tile + 1 < p.n_tiles ? p.tile_first[tile + 1] : last;
    const int64_t len = p1 - p0 + 1;
    int seg = (int)(len >= 1 && len <= kDTileRows + 1 ? len : 0);
    if (p0 < first || p1 > last || seg == 0) { atomicMin(p.err, (long long)(p0 < first ? first : p0)); seg = 0; }
    s_p0 = p0;
    s_seg = seg;
  }
  __syncthreads();
  const int seg = s_seg;
  if (seg == 0) return;
  const int64_t p0 = s_p0;
  for (int k = threadIdx.x; k < seg; k += kDThreads) {
    const int64_t e = (int64_t)re[p0 + k] - a;   // clipped to [0, rows]
    s_end[k] = (int32_t)(e < 0 ? 0 : (e > rows ? rows : e));
    const int64_t run = p.voff + p0 + k;
    uint32_t f = p.valid ? (uint32_t)bit_is_set(p.valid, run) : 1u;
    if constexpr (kBool) f |= (uint32_t)bit_is_set(reinterpret_cast<const uint8_t*>(p.vals), run) << 1;
    s_flag[k] = (uint8_t)f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const E* vals = reinterpret_cast<const E*>(p.vals);
  unsigned long long nulls = 0;
  const bool vec_out = !kBool && (((uintptr_t)p.out & 15) == 0);
  for (int gi = threadIdx.x; gi < (kGroups + 31) / 32 * 32; gi += kDThreads) {   // whole warps: the shuffles need every lane
    const int j0 = gi * G;
    uint32_t vbits = 0, mbits = 0;
    if (gi < kGroups && j0 < rows) {
      // the run of row j0: the first k with s_end[k] > j0
      int lo = 0, hi = seg - 1;
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (s_end[mid] > j0) hi = mid; else lo = mid + 1; }
      int k = lo;
      E v[kBool ? 1 : G];
      const int n_here = rows - j0 < G ? rows - j0 : G;
      for (int e = 0; e < G; ++e) {
        if (e < n_here) {
          while (k < seg - 1 && s_end[k] <= j0 + e) ++k;
          const uint32_t f = s_flag[k];
          mbits |= (f & 1u) << e;
          nulls += (f & 1u) ^ 1u;
          if constexpr (kBool) vbits |= (f >> 1) << e;
          else v[e] = vals[p.voff + p0 + k];
        } else if constexpr (!kBool) {
          v[e] = E(0);
        }
      }
      if constexpr (kBool) {
        reinterpret_cast<uint32_t*>(p.out)[(row0 + j0) >> 5] = vbits;
      } else {
        E* o = reinterpret_cast<E*>(p.out) + row0 + j0;
        if (vec_out && n_here == G) {
          uint4 u;
          memcpy(&u, v, 16);
          *reinterpret_cast<uint4*>(o) = u;
        } else {
          for (int e = 0; e < n_here; ++e) o[e] = v[e];
        }
      }
    }
    if (p.out_valid) {
      // the 32 / G lanes that share a validity word OR their bits together; the lowest writes it
      uint32_t w = mbits << (j0 & 31);
      if constexpr (G < 32) {
#pragma unroll
        for (int s = 1; s < 32 / G; s <<= 1) w |= __shfl_xor_sync(0xffffffffu, w, s);
      }
      if ((lane & (32 / G - 1)) == 0 && gi < kGroups && j0 < rows) p.out_valid[(row0 + j0) >> 5] = w;
    }
  }
  if (p.valid) {
    nulls = __reduce_add_sync(0xffffffffu, (unsigned)nulls);
    if (lane == 0 && nulls) atomicAdd(p.null_count, nulls);
  }
}

ag_status run_end_decode_dev(int type, int run_end_type, const void* run_ends, int64_t n_runs, const void* vals, const uint8_t* valid,
                             int64_t values_offset, int64_t offset, int64_t length, void* out, uint8_t* out_valid,
                             int64_t* d_null_count, int64_t* d_error_word, cudaStream_t st) {
  const char* who = "run_end_decode";
  if (!d_null_count || !d_error_word) AG_FAIL(AG_ERR_INVALID, "%s: NULL null_count / error word", who);
  if (n_runs < 0 || values_offset < 0 || offset < 0 || length < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative length or offset", who);
  AG_TRY(visit_value(type, [](auto) { return AG_OK; }, who));
  AG_TRY(visit_run_end(run_end_type, [](auto) { return AG_OK; }, who));
  AG_CUDA_TRY(cudaMemsetAsync(d_null_count, 0, sizeof(int64_t), st));
  if (length == 0) return AG_OK;
  if (!run_ends || !vals || !out) AG_FAIL(AG_ERR_INVALID, "%s: NULL run_ends / values / output", who);
  if (valid && !out_valid) AG_FAIL(AG_ERR_INVALID, "%s: a values child with a validity bitmap needs an output validity bitmap", who);
  if (out_valid && ((uintptr_t)out_valid & 3)) AG_FAIL(AG_ERR_INVALID, "%s: out_valid must be 4-byte aligned", who);
  if (type == AG_TYPE_BOOL && ((uintptr_t)out & 3)) AG_FAIL(AG_ERR_INVALID, "%s: boolean output bitmap must be 4-byte aligned", who);
  if (type != AG_TYPE_BOOL && ((uintptr_t)out % type_width(type))) AG_FAIL(AG_ERR_INVALID, "%s: output not aligned to the element width", who);
  Workspace* ws;
  AG_TRY(get_workspace(st, &ws));
  WorkspaceLock ws_lock(ws);
  DecodeParams p{};
  p.run_ends = run_ends; p.n_runs = n_runs; p.vals = vals; p.valid = valid; p.voff = values_offset;
  p.offset = offset; p.length = length; p.out = out; p.out_valid = valid ? reinterpret_cast<uint32_t*>(out_valid) : nullptr;
  p.null_count = reinterpret_cast<unsigned long long*>(d_null_count);
  p.err = reinterpret_cast<long long*>(d_error_word);
  p.bounds = ws->scalars;   // [0], [1]: first / last run
  p.n_tiles = (length + kDTileRows - 1) / kDTileRows;
  AG_TRY(ensure_tile_status(ws, (size_t)p.n_tiles, st));
  p.tile_first = reinterpret_cast<int64_t*>(ws->tile_status);
  return visit_value(type, [&](auto vtag) {
    using V = typename decltype(vtag)::type;
    return visit_run_end(run_end_type, [&](auto rtag) {
      using R = typename decltype(rtag)::type;
      run_end_bounds_kernel<R><<<1, 1, 0, st>>>(p);
      AG_TRY(check_launch("run_end_bounds_kernel"));
      run_end_tile_first_kernel<R><<<(unsigned)((p.n_tiles + kDThreads - 1) / kDThreads), kDThreads, 0, st>>>(p);
      AG_TRY(check_launch("run_end_tile_first_kernel"));
      run_end_decode_kernel<V, R><<<(unsigned)p.n_tiles, kDThreads, 0, st>>>(p);
      return check_launch("run_end_decode_kernel");
    }, who);
  }, who);
}

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_run_end_count_dev(int type, const void* d_vals, const uint8_t* d_valid, int64_t offset, int64_t n, int64_t* d_counts, ag_stream_t s) {
  AG_TRY(ensure_init());
  return run_end_count_dev(type, d_vals, d_valid, offset, n, d_counts, resolve_stream(s));
}
ag_status ag_run_end_encode_dev(int type, int run_end_type, const void* d_vals, const uint8_t* d_valid, int64_t offset, int64_t n,
                                void* d_run_ends, void* d_out, uint8_t* d_out_valid, int64_t capacity, int64_t* d_counts, ag_stream_t s) {
  AG_TRY(ensure_init());
  return run_end_encode_dev(type, run_end_type, d_vals, d_valid, offset, n, d_run_ends, d_out, d_out_valid, capacity, d_counts, resolve_stream(s));
}
ag_status ag_run_end_decode_dev(int type, int run_end_type, const void* d_run_ends, int64_t n_runs, const void* d_vals, const uint8_t* d_valid,
                                int64_t values_offset, int64_t offset, int64_t length, void* d_out, uint8_t* d_out_valid,
                                int64_t* d_null_count, int64_t* d_error_word, ag_stream_t s) {
  AG_TRY(ensure_init());
  return run_end_decode_dev(type, run_end_type, d_run_ends, n_runs, d_vals, d_valid, values_offset, offset, length, d_out, d_out_valid,
                            d_null_count, d_error_word, resolve_stream(s));
}

}  // extern "C"
