// scan.cu — cumulative_sum / cumulative_sum_checked in ONE pass over HBM.
//
// Replaces cumulativeSumNoNulls / WithNulls (+Checked) of
// arrow/compute/internal/kernels/vector_cumulative.go:228-330 (driver cumulativeSumSpans :332-368,
// state :100-145, checked adders :147-206):
//   out[i] = start + sum of the VALID in[j], j <= i;  a null input gives a null output slot (value
//   left at 0, like the reference's freshly allocated buffer); unless SkipNulls, every slot after the
//   first null is null as well (state.encounteredNull) and nothing accumulates past it; the checked
//   flavour fails with "overflow" at the first running sum that leaves the type's range.
// Chunked input is one logical sequence (cumulativeSumExecChunked :385-410): the running value and
// the encountered-null flag live in a small device-resident state block that every call reads and
// updates, so a chunked column is a chain of launches on one stream with no host round trip.
//
// Roofline: HBM, 2 x sizeof(T) algorithmic bytes per row (read once, write once).
// Algorithm: single-pass scan with decoupled look-back over 32 KB tiles, one kernel for every call
// (cumsum_stream_kernel below: checked or not, with or without a validity bitmap, any element-aligned operands).
//   * warp w of a tile owns a contiguous 4 KB segment, loaded coalesced and transposed through
//     swizzled shared memory so that each lane owns 128 contiguous bytes: one local scan and ONE warp
//     scan per tile;
//   * tile status, three levels: every tile publishes its AGGREGATE; the last tile of a group of 128
//     publishes the GROUP aggregate (it needs only its own group's tile aggregates, so it never waits
//     on earlier groups); the last tile of a super-group of 32 groups publishes the INCLUSIVE prefix.
//     Tile i gathers <= 127 tile aggregates (four per lane), <= 31 group aggregates (one per lane) and
//     one inclusive prefix, and folds them in a FIXED order — the association of a floating-point sum
//     is a function of (data, n) only, never of timing.  The only serial hand-off happens once per
//     4096 tiles (128 MB of input); a first version with one inclusive prefix per 128 tiles left
//     every resident block stalled behind each hand-off;
//   * every status word carries its own flag and is written exactly once, so there is no torn
//     flag/value pair to guard against (a 64-bit accumulator is split over 32-bit payloads);
//   * static tile order + cooperative launch (one resident wave): a tile only ever waits on lower
//     tiles, which resident blocks reach in increasing order.
// Unchecked integers accumulate modulo 2^64, which is all the wrapped result needs; the checked flavour
// accumulates an exact 96-bit value (64-bit wrap + carry count) and compares the running sum with the
// type's range per element.  Floats accumulate in their own type from -0.0 (the identity of IEEE addition);
// outputs and carried state are bit-exact with tests/cumsum_float_ref.py, the step-by-step model of this
// fold order, on any input; bit-exact with the reference's left-to-right loop, signed zeros included,
// whenever every partial sum is exactly representable; within the summation bound of the fold's depth
// otherwise.  The carried state is the last tile's excl + tile_total, which can differ by rounding from
// the last output slot (excl + ((warp_excl + lane_excl) + x...)); the reference's state is its last output
// (DESIGN.md).
#include "common.cuh"

#include <limits>

namespace ag {
namespace {

constexpr int kScThreads = 256;
constexpr int kScWarps = kScThreads / 32;
constexpr int kScRows = 8;                              // 16-byte vectors per lane per tile
constexpr int kScTileBytes = kScThreads * kScRows * 16;  // 32 KB of input
constexpr int kScGroup = 128;                           // tiles per look-back group
constexpr int kScSuper = 32;                            // groups per super-group (the serial chain steps once per 4096 tiles)
constexpr unsigned long long kScFlag = 1ull << 32;      // payload in bits 0..31, flag in bit 32

struct CumsumState {  // device-resident, 32 bytes: include/arrowgpu.h ag_cumsum_state
  unsigned long long lo;  // running value: wrapped 64-bit integer sum, or the float / double bit pattern
  long long hi;           // carries of the exact integer sum (0 for floats)
  long long encountered_null;
  long long null_count;   // null slots written so far (all chunks of the sequence)
};

// ---- accumulators ---------------------------------------------------------------------------
struct AccX { unsigned long long lo; int hi; };  // exact: value = hi * 2^64 + lo

template <typename T> struct IsFp { static constexpr bool v = false; };
template <> struct IsFp<float> { static constexpr bool v = true; };
template <> struct IsFp<double> { static constexpr bool v = true; };

template <typename T, bool kFp = IsFp<T>::v> struct Pol;

template <typename T>
struct Pol<T, false> {  // integers
  using A = AccX;
  static constexpr int K = 3;
  static constexpr bool kSigned = T(-1) < T(0);
  static __device__ __forceinline__ A zero() { return A{0ull, 0}; }
  static __device__ __forceinline__ A add(A a, A b) {
    A r;
    r.lo = a.lo + b.lo;
    r.hi = a.hi + b.hi + (r.lo < a.lo ? 1 : 0);
    return r;
  }
  static __device__ __forceinline__ A add_elem(A a, T x) {
    A b;
    b.lo = (unsigned long long)(long long)x;  // sign / zero extension to 64 bits
    if (!kSigned) b.lo = (unsigned long long)x;
    b.hi = (kSigned && x < T(0)) ? -1 : 0;
    return add(a, b);
  }
  static __device__ __forceinline__ T value(A a) { return (T)a.lo; }
  static __device__ __forceinline__ bool out_of_range(A a) {
    if (sizeof(T) == 8) {
      if (kSigned) return a.hi != (((long long)a.lo < 0) ? -1 : 0);
      return a.hi != 0;
    }
    // exact value fits 64 bits comfortably for narrower types (|sum| < 2^32 * 2^31)
    const long long v = (long long)a.lo;
    if (a.hi != (v < 0 ? -1 : 0)) return true;
    return v < (long long)std::numeric_limits<T>::lowest() || v > (long long)std::numeric_limits<T>::max();
  }
  static __device__ __forceinline__ A shfl_up(A a, int d) {
    A r;
    r.lo = __shfl_up_sync(0xffffffffu, a.lo, d);
    r.hi = __shfl_up_sync(0xffffffffu, a.hi, d);
    return r;
  }
  static __device__ __forceinline__ A shfl(A a, int src) {
    A r;
    r.lo = __shfl_sync(0xffffffffu, a.lo, src);
    r.hi = __shfl_sync(0xffffffffu, a.hi, src);
    return r;
  }
  static __device__ __forceinline__ A shfl_xor(A a, int m) {
    A r;
    r.lo = __shfl_xor_sync(0xffffffffu, a.lo, m);
    r.hi = __shfl_xor_sync(0xffffffffu, a.hi, m);
    return r;
  }
  static __device__ __forceinline__ void to_words(A a, unsigned (&w)[3]) { w[0] = (unsigned)a.lo; w[1] = (unsigned)(a.lo >> 32); w[2] = (unsigned)a.hi; }
  static __device__ __forceinline__ A from_words(const unsigned (&w)[3]) { return A{(unsigned long long)w[0] | ((unsigned long long)w[1] << 32), (int)w[2]}; }
  static __device__ __forceinline__ A from_state(const CumsumState& s) { return A{s.lo, (int)s.hi}; }
  static __device__ __forceinline__ void to_state(A a, CumsumState* s) { s->lo = a.lo; s->hi = a.hi; }
};

template <typename T>
struct PolWrap {  // unchecked integers: the sum modulo 2^64 is all the result needs
  using A = unsigned long long;
  static constexpr int K = 2;
  static constexpr bool kSigned = T(-1) < T(0);
  static __device__ __forceinline__ A zero() { return 0ull; }
  static __device__ __forceinline__ A add(A a, A b) { return a + b; }
  static __device__ __forceinline__ A add_elem(A a, T x) { return a + (kSigned ? (A)(long long)x : (A)x); }
  static __device__ __forceinline__ T value(A a) { return (T)a; }
  static __device__ __forceinline__ T offset_add(T off, T local) { return (T)((A)off + (A)local); }  // modulo 2^w
  static __device__ __forceinline__ bool out_of_range(A) { return false; }
  static __device__ __forceinline__ A shfl_up(A a, int d) { return __shfl_up_sync(0xffffffffu, a, d); }
  static __device__ __forceinline__ A shfl(A a, int src) { return __shfl_sync(0xffffffffu, a, src); }
  static __device__ __forceinline__ void to_words(A a, unsigned (&w)[3]) { w[0] = (unsigned)a; w[1] = (unsigned)(a >> 32); }
  static __device__ __forceinline__ A from_words(const unsigned (&w)[3]) { return (A)w[0] | ((A)w[1] << 32); }
  static __device__ __forceinline__ A from_state(const CumsumState& s) { return s.lo; }
  static __device__ __forceinline__ void to_state(A a, CumsumState* s) {
    // keep the exact-sum convention of the state block: hi = sign extension of the wrapped low word is
    // NOT the exact carry count, so an unchecked call leaves hi consistent with "value = lo" only
    s->lo = a;
    s->hi = (kSigned && (long long)a < 0) ? -1 : 0;
  }
};

template <typename T, bool kChecked> struct PolSel { using type = Pol<T>; };
template <> struct PolSel<uint8_t, false> { using type = PolWrap<uint8_t>; };
template <> struct PolSel<int8_t, false> { using type = PolWrap<int8_t>; };
template <> struct PolSel<uint16_t, false> { using type = PolWrap<uint16_t>; };
template <> struct PolSel<int16_t, false> { using type = PolWrap<int16_t>; };
template <> struct PolSel<uint32_t, false> { using type = PolWrap<uint32_t>; };
template <> struct PolSel<int32_t, false> { using type = PolWrap<int32_t>; };
template <> struct PolSel<unsigned long long, false> { using type = PolWrap<unsigned long long>; };
template <> struct PolSel<long long, false> { using type = PolWrap<long long>; };

template <typename T>
struct Pol<T, true> {  // float / double: accumulate in the value type
  using A = T;
  static constexpr int K = sizeof(T) == 8 ? 2 : 1;
  // -0.0 is the identity of IEEE addition (+0.0 is not: -0.0 + +0.0 = +0.0), so the padded lanes, entries and
  // accumulators that start from it leave every sum's bits alone, the sign of a zero included
  static __device__ __forceinline__ A zero() { return T(-0.0); }
  static __device__ __forceinline__ A add(A a, A b) {
    if constexpr (sizeof(T) == 8) return __dadd_rn(a, b); else return __fadd_rn(a, b);
  }
  static __device__ __forceinline__ A add_elem(A a, T x) { return add(a, x); }
  static __device__ __forceinline__ T value(A a) { return a; }
  static __device__ __forceinline__ T offset_add(T off, T local) { return add(off, local); }
  static __device__ __forceinline__ bool out_of_range(A) { return false; }  // checkedAdder default: plain add
  static __device__ __forceinline__ A shfl_up(A a, int d) { return __shfl_up_sync(0xffffffffu, a, d); }
  static __device__ __forceinline__ A shfl(A a, int src) { return __shfl_sync(0xffffffffu, a, src); }
  static __device__ __forceinline__ A shfl_xor(A a, int m) { return __shfl_xor_sync(0xffffffffu, a, m); }
  static __device__ __forceinline__ void to_words(A a, unsigned (&w)[3]) {
    if constexpr (sizeof(T) == 8) { const unsigned long long b = (unsigned long long)__double_as_longlong(a); w[0] = (unsigned)b; w[1] = (unsigned)(b >> 32); }
    else w[0] = __float_as_uint(a);
  }
  static __device__ __forceinline__ A from_words(const unsigned (&w)[3]) {
    if constexpr (sizeof(T) == 8) return __longlong_as_double((long long)((unsigned long long)w[0] | ((unsigned long long)w[1] << 32)));
    else return __uint_as_float(w[0]);
  }
  static __device__ __forceinline__ A from_state(const CumsumState& s) {
    if constexpr (sizeof(T) == 8) return __longlong_as_double((long long)s.lo); else return __uint_as_float((unsigned)s.lo);
  }
  static __device__ __forceinline__ void to_state(A a, CumsumState* s) {
    if constexpr (sizeof(T) == 8) s->lo = (unsigned long long)__double_as_longlong(a); else s->lo = __float_as_uint(a);
    s->hi = 0;
  }
};

__device__ __forceinline__ void st_word(unsigned long long* p, unsigned v) { *reinterpret_cast<volatile unsigned long long*>(p) = kScFlag | v; }

struct CumsumParams {
  const void* in;
  void* out;
  const uint8_t* valid;   // may be NULL
  int64_t voff;
  int64_t n;
  int skip_nulls;
  const long long* first_null;   // device: first null row of this call (n when none); NULL when valid == NULL
  CumsumState* state;
  long long* first_bad;          // may be NULL when !checked
  uint8_t* out_valid;            // may be NULL (then there are no nulls anywhere in the sequence)
  int64_t ooff;
  unsigned long long* agg;       // [n_tiles][S]    S = StatusEntry<K>::kStride words per entry
  unsigned long long* gagg;      // [n_groups][S]   aggregate of a whole group
  unsigned long long* sincl;     // [n_super][S]    inclusive prefix at the end of a super-group
  int64_t n_tiles;
};

// ---- the scan kernel ------------------------------------------------------------------------------
// Profiled on a block-synchronous shape (one warp of each block doing the look-back between two block barriers):
// most warp samples sit at the barrier behind the look-back and that warp spends 92 % of its time inside it (half
// waiting for flags of tiles that other blocks are reducing at the same moment, half in ~600 dependent instructions
// of one warp) — every resident block is in the same phase, so nothing on the SM covers that wait, which took longer
// than the tile's HBM time.  This kernel takes the look-back off the critical path:
//   * a block = 8 compute warps + 1 LOOK-BACK warp.  In iteration j the compute warps reduce tile j
//     and finalize tile j-1 while the look-back warp resolves the prefix of tile j-1 (whose aggregate,
//     and those of its predecessors in other blocks, were published an iteration ago: the polls hit);
//     one block barrier per tile joins them;
//   * tiles arrive by cp.async (16 bytes per thread, no staging registers) straight into the SWIZZLED
//     position of a 3-stage shared-memory ring (loading / being reduced / waiting for its prefix); a
//     warp only ever touches its own 4 KB segment of a stage, so the ring needs __syncwarp only;
//   * the look-back reads a whole status entry per load, issues all its polls as one batch
//     and folds them with interleaved warp scans: ~1 L2 round trip + ~150 instructions;
//   * interior tiles run a branch-free body (base pointer + immediate offsets).
// Operands that are only element-aligned (Arrow slices, later chunks of a chunked output) take block-uniform side
// paths in the load and store stages; the aligned path is unchanged by them.
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, int bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
// 4- / 8-byte pieces for an input that is only element-aligned (an Arrow slice): same destination layout, more copies
template <int kB>
__device__ __forceinline__ void cp_async_small_zfill(uint32_t dst, const void* src, int bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2, %3;" ::"r"(dst), "l"(src), "n"(kB), "r"(bytes) : "memory");
}
// A 16-byte vector stored to an address aligned only to its lowest set bit `mis & -mis` (>= sizeof(T)), in the widest
// pieces that alignment allows
template <typename W>
__device__ __forceinline__ void st_pieces_as(unsigned char* dst, const uint4& v) {
  const W* s = reinterpret_cast<const W*>(&v);
#pragma unroll
  for (int q = 0; q < 16 / (int)sizeof(W); ++q) __stcs(reinterpret_cast<W*>(dst) + q, s[q]);
}
template <typename T>
__device__ __forceinline__ void st_pieces(unsigned char* dst, const uint4& v, int mis) {
  if (sizeof(T) >= 8 || (mis & 7) == 0) st_pieces_as<unsigned long long>(dst, v);
  else if (sizeof(T) >= 4 || (mis & 3) == 0) st_pieces_as<unsigned>(dst, v);
  else if (sizeof(T) >= 2 || (mis & 1) == 0) st_pieces_as<unsigned short>(dst, v);
  else st_pieces_as<unsigned char>(dst, v);
}
// a shared-memory read the compiler must not reuse from before the atomic that announced it
template <typename A> __device__ __forceinline__ A ld_shared_volatile(const A& a) { return *reinterpret_cast<const volatile A*>(&a); }
__device__ __forceinline__ AccX ld_shared_volatile(const AccX& a) {
  const volatile AccX& v = a;
  return AccX{v.lo, v.hi};
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int kPending> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(kPending) : "memory"); }

// One status entry = K flagged 64-bit words, fetched with one volatile load per 16 bytes (every word carries its own
// flag, so it does not matter whether the words are observed at the same instant).  kStride words apart, so that every
// entry of a multi-word accumulator starts on a 16-byte boundary.
template <int K> struct StatusEntry;
template <> struct StatusEntry<1> {
  static constexpr int kStride = 1;
  unsigned long long w0;
  __device__ __forceinline__ void load(const unsigned long long* p) { asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(w0) : "l"(p) : "memory"); }
  __device__ __forceinline__ bool ready() const { return (w0 & kScFlag) != 0; }
  __device__ __forceinline__ void words(unsigned (&w)[3]) const { w[0] = (unsigned)w0; w[1] = 0u; w[2] = 0u; }
  __device__ __forceinline__ void set_ready_zero() { w0 = kScFlag; }
};
template <> struct StatusEntry<2> {
  static constexpr int kStride = 2;
  unsigned long long w0, w1;
  __device__ __forceinline__ void load(const unsigned long long* p) {
    asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(p) : "memory");
  }
  __device__ __forceinline__ bool ready() const { return ((w0 & w1) & kScFlag) != 0; }
  __device__ __forceinline__ void words(unsigned (&w)[3]) const { w[0] = (unsigned)w0; w[1] = (unsigned)w1; w[2] = 0u; }
  __device__ __forceinline__ void set_ready_zero() { w0 = kScFlag; w1 = kScFlag; }
};
template <> struct StatusEntry<3> {  // the exact 96-bit integer sum: 32 bytes, the fourth word is never written
  static constexpr int kStride = 4;
  unsigned long long w0, w1, w2, w3;
  __device__ __forceinline__ void load(const unsigned long long* p) {
    asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(p) : "memory");
    asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(w2), "=l"(w3) : "l"(p + 2) : "memory");
  }
  __device__ __forceinline__ bool ready() const { return ((w0 & w1 & w2) & kScFlag) != 0; }
  __device__ __forceinline__ void words(unsigned (&w)[3]) const { w[0] = (unsigned)w0; w[1] = (unsigned)w1; w[2] = (unsigned)w2; }
  __device__ __forceinline__ void set_ready_zero() { w0 = kScFlag; w1 = kScFlag; w2 = kScFlag; }
};

// The look-back of one tile, executed by a whole warp.  Returns the tile's exclusive prefix (all lanes) after publishing
// whatever this tile owes the others (its group aggregate, the super-group prefix).  Built for latency: whole entries
// per load, every poll of a level in one batch, the four tile-aggregate scans interleaved.
template <typename P>
__device__ __forceinline__ typename P::A cumsum_lookback(const CumsumParams& p, int64_t tile, typename P::A tile_total,
                                                         typename P::A start, int lane) {
  using A = typename P::A;
  constexpr int K = P::K;
  constexpr int S = StatusEntry<K>::kStride;
  constexpr int R = kScGroup / 32;
  const int64_t g = tile / kScGroup;
  const int qpos = (int)(tile - g * kScGroup);
  const int64_t sg = g / kScSuper;
  const int gq = (int)(g - sg * kScSuper);
  const unsigned long long* a_src = p.agg + (g * kScGroup + lane) * S;
  const unsigned long long* g_src = p.gagg + (sg * kScSuper + lane) * S;
  const unsigned long long* s_src = p.sincl + (sg > 0 ? sg - 1 : 0) * S;
  StatusEntry<K> ea[R], eg, es;
  bool need_a[R];
#pragma unroll
  for (int r = 0; r < R; ++r) need_a[r] = r * 32 + lane < qpos;
  const bool need_g = lane < gq, need_s = sg > 0;
  // first batch: everything at once (one L2 round trip when all flags are up, the common case)
#pragma unroll
  for (int r = 0; r < R; ++r) { if (need_a[r]) ea[r].load(a_src + r * 32 * S); else ea[r].set_ready_zero(); }
  if (need_g) eg.load(g_src); else eg.set_ready_zero();
  if (need_s) es.load(s_src); else es.set_ready_zero();
  while (true) {
    bool ok = true;
#pragma unroll
    for (int r = 0; r < R; ++r) ok = ok && ea[r].ready();
    if (__all_sync(0xffffffffu, ok)) break;
#pragma unroll
    for (int r = 0; r < R; ++r) if (need_a[r] && !ea[r].ready()) ea[r].load(a_src + r * 32 * S);
  }
  A x[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    unsigned w[3];
    ea[r].words(w);
    x[r] = need_a[r] ? P::from_words(w) : P::zero();
  }
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const A up = P::shfl_up(x[r], d);
      if (lane >= d) x[r] = P::add(up, x[r]);
    }
  }
  A part = P::zero();
#pragma unroll
  for (int r = 0; r < R; ++r) part = P::add(part, P::shfl(x[r], 31));
  if (qpos == kScGroup - 1 && lane == 0) {  // group aggregate: needs nothing older than this group
    unsigned wg[3] = {0u, 0u, 0u};
    P::to_words(P::add(part, tile_total), wg);
#pragma unroll
    for (int k = 0; k < K; ++k) st_word(p.gagg + g * S + k, wg[k]);
  }
  while (!__all_sync(0xffffffffu, eg.ready() && es.ready())) {
    if (need_g && !eg.ready()) eg.load(g_src);
    if (need_s && !es.ready()) es.load(s_src);
  }
  unsigned w[3];
  eg.words(w);
  A gpart = need_g ? P::from_words(w) : P::zero();
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const A up = P::shfl_up(gpart, d);
    if (lane >= d) gpart = P::add(up, gpart);
  }
  gpart = P::shfl(gpart, 31);
  es.words(w);
  const A base = need_s ? P::from_words(w) : start;
  const A excl = P::add(P::add(base, gpart), part);
  if (lane == 0 && qpos == kScGroup - 1 && gq == kScSuper - 1) {
    unsigned wi[3] = {0u, 0u, 0u};
    P::to_words(P::add(excl, tile_total), wi);
#pragma unroll
    for (int k = 0; k < K; ++k) st_word(p.sincl + sg * S + k, wi[k]);
  }
  return excl;
}

constexpr int kScStreamThreads = kScThreads + 32;  // 8 compute warps + the look-back warp
constexpr int kScStreamStages = 3;
constexpr int kScStreamBlocksPerSm = 2;            // 2 x (3 x 32 KB) of the SM's 227 KB

// kChecked (integers only): the exact 96-bit running sum, compared with T's range at every valid row; the lowest row
// that leaves it goes to first_bad
template <typename T, bool kHasValid, bool kChecked>
__global__ void __launch_bounds__(kScStreamThreads, kScStreamBlocksPerSm)
cumsum_stream_kernel(const CumsumParams p) {
  using P = typename PolSel<T, kChecked>::type;
  using A = typename P::A;
  constexpr int S = StatusEntry<P::K>::kStride;
  constexpr int N = 16 / sizeof(T);
  constexpr int E = kScRows * N;                  // rows owned by one lane (128 contiguous bytes)
  constexpr int kTileRows = kScTileBytes / sizeof(T);
  constexpr int kSegRows = kTileRows / kScWarps;
  constexpr int VW = (E + 31) / 32;               // validity words per lane
  extern __shared__ __align__(128) unsigned char s_ring[];  // 3 stages x 32 KB
  __shared__ A s_warp[2][kScWarps];
  __shared__ A s_excl[2];
  __shared__ unsigned s_arrived[2];
  __shared__ CumsumState s_state;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool looker = warp == kScWarps;
  if (threadIdx.x < 2) s_arrived[threadIdx.x] = 0u;
  const unsigned char* __restrict__ in = reinterpret_cast<const unsigned char*>(p.in);
  unsigned char* __restrict__ out = reinterpret_cast<unsigned char*>(p.out);
  const int64_t n_bytes = p.n * (int64_t)sizeof(T);
  const int out_mis = (int)(reinterpret_cast<uintptr_t>(out) & 15);  // 0, or a multiple of sizeof(T) (block-uniform)
  auto store16 = [&](int64_t g, const uint4& v) {  // bytes [g, g + 16) of the output, all inside it
    if (out_mis) st_pieces<T>(out + g, v, out_mis);
    else __stcs(reinterpret_cast<uint4*>(out + g), v);
  };

  if (threadIdx.x == 0) s_state = *p.state;
  __syncthreads();
  const A start = P::from_state(s_state);
  if (!p.skip_nulls && s_state.encountered_null != 0) {
    // an earlier chunk of the sequence met a null: every slot of this call is null (value 0) and the
    // carried state stays as it is
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    for (int64_t b = ((int64_t)blockIdx.x * kScStreamThreads + threadIdx.x) * 16; b < n_bytes; b += (int64_t)gridDim.x * kScStreamThreads * 16) {
      if (b + 16 <= n_bytes) store16(b, z);
      else for (int64_t j = b; j < n_bytes; ++j) out[j] = 0;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { CumsumState ns = s_state; P::to_state(start, &ns); *p.state = ns; }
    return;
  }

  // validity of the E rows a lane owns, 32 at a time: rows at or past `limit` (the first null when nulls are not
  // skipped) and past n contribute nothing.  Returns whether every row counts (the common case).
  int64_t limit = p.n;
  if (kHasValid && !p.skip_nulls) limit = *p.first_null;
  const int64_t vlo = p.voff >> 3, vhi = (p.voff + p.n + 7) >> 3;
  auto lane_validity = [&](int64_t tile, unsigned (&vbits)[VW]) -> bool {
    if (!kHasValid) return true;
    const int64_t t0 = tile * kTileRows + (int64_t)(warp & (kScWarps - 1)) * kSegRows + (int64_t)lane * E;
    bool dense = true;
#pragma unroll
    for (int w = 0; w < VW; ++w) {
      const int64_t e0 = t0 + w * 32;
      unsigned m = (e0 < p.n) ? bitmap_load32(p.valid, p.voff + e0, vlo, vhi) : 0u;
      const int64_t room = limit - e0;
      if (room < 32) m &= (room <= 0) ? 0u : ((1u << (int)room) - 1u);
      constexpr unsigned kFull = (E >= 32) ? 0xffffffffu : ((1u << (E & 31)) - 1u);
      m &= kFull;
      vbits[w] = m;
      dense = dense && m == kFull;
    }
    return dense;
  };

  // byte offsets of this lane inside a 4 KB warp segment
  //   striped (coalesced) vector k:  logical (k*32 + lane) * 16, parked at its owner's row, chunk ^ (owner & 7)
  //   blocked chunk c of row `lane`: lane*128 + ((c ^ (lane & 7)) << 4)
  const uint32_t ring = (uint32_t)__cvta_generic_to_shared(s_ring);
  const uint32_t seg_off = (uint32_t)(warp & (kScWarps - 1)) * 4096u;
  const uint32_t str_even = (uint32_t)(((lane & ~7) | ((lane & 7) ^ (lane >> 3))) << 4);  // k even; k odd: ^ 64; + k*512
  const uint32_t blk_row = (uint32_t)lane * 128u;
  const uint32_t blk_x = (uint32_t)(lane & 7) << 4;

  const int in_mis = (int)(reinterpret_cast<uintptr_t>(in) & 15);   // 0, or a multiple of sizeof(T) (block-uniform)
  auto prefetch = [&](int64_t tile, int stage) {
    const uint32_t dst0 = ring + (uint32_t)stage * kScTileBytes + seg_off;
    const int64_t g0 = tile * kScTileBytes + seg_off + (int64_t)lane * 16;
    if (sizeof(T) < 4 && (in_mis & 3)) {
      // 1- / 2-byte elements below 4-byte alignment: cp.async has no piece that small, so plain loads fill the same
      // slots (the __syncwarp after cp_async_wait orders these stores too: a warp only touches its own segment)
      const T* src = reinterpret_cast<const T*>(in);
#pragma unroll 4  // fully unrolled, the 16-bit kernels' loads in flight raise their register count by ~15
      for (int k = 0; k < kScRows; ++k) {
        const int64_t e = (g0 + k * 512) / (int64_t)sizeof(T);
        __align__(16) T v[N];
#pragma unroll
        for (int i = 0; i < N; ++i) v[i] = e + i < p.n ? src[e + i] : T(0);
        *reinterpret_cast<uint4*>(s_ring + (dst0 - ring) + (str_even ^ ((k & 1) << 6)) + k * 512) = *reinterpret_cast<const uint4*>(v);
      }
    } else if (in_mis) {
      // element-aligned input: the 16-byte slots of the ring are filled by two 8-byte or four 4-byte copies
#pragma unroll
      for (int k = 0; k < kScRows; ++k) {
        const uint32_t d = dst0 + (str_even ^ ((k & 1) << 6)) + k * 512;
        const int64_t g = g0 + k * 512;
        if ((in_mis & 7) == 0) {
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            const int64_t room = n_bytes - (g + q * 8);
            const int bytes = room >= 8 ? 8 : (room > 0 ? (int)room : 0);
            cp_async_small_zfill<8>(d + q * 8, bytes > 0 ? in + g + q * 8 : in, bytes);
          }
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int64_t room = n_bytes - (g + q * 4);
            const int bytes = room >= 4 ? 4 : (room > 0 ? (int)room : 0);
            cp_async_small_zfill<4>(d + q * 4, bytes > 0 ? in + g + q * 4 : in, bytes);
          }
        }
      }
    } else if (g0 - (int64_t)lane * 16 + 4096 <= n_bytes) {
#pragma unroll
      for (int k = 0; k < kScRows; ++k) cp_async16(dst0 + (str_even ^ ((k & 1) << 6)) + k * 512, in + g0 + k * 512);
    } else {  // the segment crosses the end of the input: zero-fill what is not there
#pragma unroll
      for (int k = 0; k < kScRows; ++k) {
        const int64_t g = g0 + k * 512;
        const int64_t room = n_bytes - g;
        const int bytes = room >= 16 ? 16 : (room > 0 ? (int)room : 0);
        cp_async16_zfill(dst0 + (str_even ^ ((k & 1) << 6)) + k * 512, bytes > 0 ? in + g : in, bytes);
      }
    }
  };

  const int64_t G = gridDim.x;
  const int64_t mine = ((int64_t)blockIdx.x < p.n_tiles) ? (p.n_tiles - blockIdx.x + G - 1) / G : 0;  // tiles of this block
  if (!looker) { if (mine > 0) prefetch(blockIdx.x, 0); cp_async_commit(); }
  A lane_excl_cur = P::zero(), warp_excl_cur = P::zero();
  long long my_bad = AG_NO_ERROR_POS;  // checked: lowest row of this lane whose running sum left T's range
  // validity words of the rows this lane owns: fetched once per tile, in its reduction, and carried to its finalization
  // one iteration later; `dense` is made warp-uniform so a warp runs ONE of the two loops, not both under divergence
  unsigned vb_cur[VW], vb_prev[VW];
  bool dense_cur = true, dense_prev = true;
#pragma unroll
  for (int w = 0; w < VW; ++w) { vb_cur[w] = 0u; vb_prev[w] = 0u; }
  int st_r = 0, st_f = kScStreamStages - 1;   // stage of the tile being reduced (j % 3) / finalized ((j-1) % 3)
  // iteration j: reduce tile j (j < mine), look-back + finalize tile j-1 (j >= 1)
  for (int64_t j = 0; j <= mine; ++j) {
    const int64_t tile_r = blockIdx.x + j * G, tile_f = tile_r - G;
    const int br = (int)(j & 1), bf = br ^ 1;
    A lane_excl_next = P::zero();
    if (!looker) {
      const int st_n = st_r + 1 == kScStreamStages ? 0 : st_r + 1;
      if (j + 1 < mine) prefetch(tile_r + G, st_n);  // that stage held tile j-2: finalized, by this warp, an iteration ago
      cp_async_commit();
      if (j < mine) {
        cp_async_wait<1>();
        __syncwarp();
        const unsigned char* seg = s_ring + st_r * kScTileBytes + seg_off;
        uint4 raw[kScRows];
#pragma unroll
        for (int c = 0; c < kScRows; ++c) raw[c] = *reinterpret_cast<const uint4*>(seg + blk_row + (((uint32_t)c << 4) ^ blk_x));
        const T* o = reinterpret_cast<const T*>(raw);
        A tot = P::zero();
        dense_cur = __all_sync(0xffffffffu, lane_validity(tile_r, vb_cur));
        if (dense_cur) {
#pragma unroll
          for (int i = 0; i < E; ++i) tot = P::add_elem(tot, o[i]);
        } else {
#pragma unroll
          for (int i = 0; i < E; ++i) if ((vb_cur[i >> 5] >> (i & 31)) & 1u) tot = P::add_elem(tot, o[i]);
        }
        A incl = tot;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const A up = P::shfl_up(incl, d);
          if (lane >= d) incl = P::add(up, incl);
        }
        lane_excl_next = P::shfl_up(incl, 1);
        if (lane == 0) lane_excl_next = P::zero();
        if (lane == 31) {
          // the LAST warp to deliver its total publishes the tile aggregate: no barrier between a tile's reduction
          // and the moment other blocks can see it (their look-backs wait on exactly this word)
          s_warp[br][warp] = incl;
          __threadfence_block();
          if (atomicAdd(&s_arrived[br], 1u) == kScWarps - 1) {
            __threadfence_block();
            s_arrived[br] = 0u;
            A tile_total = P::zero();
#pragma unroll
            for (int wi = 0; wi < kScWarps; ++wi) tile_total = P::add(tile_total, ld_shared_volatile(s_warp[br][wi]));
            unsigned w[3] = {0u, 0u, 0u};
            P::to_words(tile_total, w);
#pragma unroll
            for (int k = 0; k < P::K; ++k) st_word(p.agg + tile_r * S + k, w[k]);
          }
        }
      }
    } else if (j >= 1) {
      A tile_total = P::zero();
#pragma unroll
      for (int wi = 0; wi < kScWarps; ++wi) tile_total = P::add(tile_total, s_warp[bf][wi]);
      const A excl = cumsum_lookback<P>(p, tile_f, tile_total, start, lane);
      if (lane == 0) {
        s_excl[bf] = excl;
        if (tile_f == p.n_tiles - 1) {
          CumsumState ns = s_state;
          P::to_state(P::add(excl, tile_total), &ns);
          if (kHasValid && *p.first_null < p.n) ns.encountered_null = 1;
          *p.state = ns;
        }
      }
    }
    __syncthreads();
    if (!looker) {
      A warp_excl_next = P::zero();
      if (j < mine) {
        A tile_total = P::zero();
#pragma unroll
        for (int wi = 0; wi < kScWarps; ++wi) {
          if (wi == warp) warp_excl_next = tile_total;
          tile_total = P::add(tile_total, s_warp[br][wi]);
        }
      }
      if (j >= 1) {
        unsigned char* seg = s_ring + st_f * kScTileBytes + seg_off;
        uint4 raw[kScRows];
#pragma unroll
        for (int c = 0; c < kScRows; ++c) raw[c] = *reinterpret_cast<const uint4*>(seg + blk_row + (((uint32_t)c << 4) ^ blk_x));
        T* o = reinterpret_cast<T*>(raw);
        if constexpr (kChecked) {
          // the exact running sum from the tile's prefix on: every valid row is range-checked
          A run = P::add(P::add(s_excl[bf], warp_excl_cur), lane_excl_cur);
          const int64_t t0 = tile_f * kTileRows + (int64_t)warp * kSegRows + (int64_t)lane * E;
#pragma unroll
          for (int i = 0; i < E; ++i) {
            if (dense_prev || ((vb_prev[i >> 5] >> (i & 31)) & 1u)) {
              run = P::add_elem(run, o[i]);
              o[i] = P::value(run);
              if (P::out_of_range(run) && t0 + i < my_bad) my_bad = t0 + i;
            } else {
              o[i] = T(0);
            }
          }
        } else {
          A run = P::add(warp_excl_cur, lane_excl_cur);
          const T off = P::value(s_excl[bf]);
          if (dense_prev) {
#pragma unroll
            for (int i = 0; i < E; ++i) { run = P::add_elem(run, o[i]); o[i] = P::offset_add(off, P::value(run)); }
          } else {
#pragma unroll
            for (int i = 0; i < E; ++i) {
              if ((vb_prev[i >> 5] >> (i & 31)) & 1u) { run = P::add_elem(run, o[i]); o[i] = P::offset_add(off, P::value(run)); }
              else o[i] = T(0);
            }
          }
        }
#pragma unroll
        for (int c = 0; c < kScRows; ++c) *reinterpret_cast<uint4*>(seg + blk_row + (((uint32_t)c << 4) ^ blk_x)) = raw[c];
        __syncwarp();
        const int64_t g0 = tile_f * kScTileBytes + seg_off + (int64_t)lane * 16;
        if (!out_mis && g0 - (int64_t)lane * 16 + 4096 <= n_bytes) {
#pragma unroll
          for (int k = 0; k < kScRows; ++k)
            __stcs(reinterpret_cast<uint4*>(out + g0 + k * 512), *reinterpret_cast<const uint4*>(seg + (str_even ^ ((k & 1) << 6)) + k * 512));
        } else {
#pragma unroll
          for (int k = 0; k < kScRows; ++k) {
            const int64_t g = g0 + k * 512;
            const uint4 v = *reinterpret_cast<const uint4*>(seg + (str_even ^ ((k & 1) << 6)) + k * 512);
            if (g + 16 <= n_bytes) store16(g, v);
            else {
              const unsigned char* vb = reinterpret_cast<const unsigned char*>(&v);
              for (int q = 0; q < 16; ++q) if (g + q < n_bytes) out[g + q] = vb[q];
            }
          }
        }
        __syncwarp();  // the segment is refilled (cp.async) two iterations from now, by this warp
      }
      lane_excl_cur = lane_excl_next;
      warp_excl_cur = warp_excl_next;
      dense_prev = dense_cur;
#pragma unroll
      for (int w = 0; w < VW; ++w) vb_prev[w] = vb_cur[w];
    }
    st_f = st_r;
    st_r = st_r + 1 == kScStreamStages ? 0 : st_r + 1;
  }
  if constexpr (IsFp<T>::v && !kHasValid) {
    // Without a bitmap the last tile's rows past n arrive zero-filled and enter its lane totals as +0.0, which is not
    // the identity of the fold.  They come after every real row, so no output sees them; only the carried state
    // excl + tile_total can: it reads +0.0 where the real rows give -0.0 + -0.0.  That happens exactly when excl and
    // the last output (excl + the real rows' fold) are both -0.0, so the owner of row n - 1 puts the sign back here,
    // once per call, after the looker's state store (ordered by the last iteration's barrier).
    const int64_t last = p.n - 1, tile = last / kTileRows;
    const int64_t local = last - tile * kTileRows;
    if (p.n % kTileRows != 0 && tile % G == blockIdx.x && !looker && warp == local / kSegRows && lane == (local % kSegRows) / E) {
      const int i = (int)(local % E);
      const unsigned char* seg = s_ring + ((mine - 1) % kScStreamStages) * kScTileBytes + seg_off;
      const T out_last = *reinterpret_cast<const T*>(seg + blk_row + (((uint32_t)(i / N) << 4) ^ blk_x) + (i % N) * sizeof(T));
      const T excl = s_excl[(mine - 1) & 1];
      if (out_last == T(0) && signbit(out_last) && excl == T(0) && signbit(excl)) {
        CumsumState ns = *p.state;
        P::to_state(T(-0.0), &ns);
        *p.state = ns;
      }
    }
  }
  if (kChecked) lower_error_row(my_bad, p.first_bad);
}

// first 0 bit of validity[voff, voff+n): one thread per 32 rows, atomicMin into *first_null (pre-set to n)
__global__ void __launch_bounds__(256)
first_null_kernel(const uint8_t* __restrict__ valid, int64_t voff, int64_t n, long long* first_null) {
  const int64_t vlo = voff >> 3, vhi = (voff + n + 7) >> 3;
  const int64_t n_words = (n + 31) >> 5;
  long long mine = AG_NO_ERROR_POS;
  for (int64_t w = (int64_t)blockIdx.x * 256 + threadIdx.x; w < n_words; w += (int64_t)gridDim.x * 256) {
    uint32_t bits = bitmap_load32(valid, voff + w * 32, vlo, vhi);
    const int64_t room = n - w * 32;
    if (room < 32) bits |= ~((1u << (int)room) - 1u);  // rows past n count as valid
    if (bits != 0xffffffffu) { const long long r = w * 32 + (__ffs(~bits) - 1); if (r < mine) mine = r; break; }  // rows only grow with w
  }
  lower_error_row(mine, first_null);
}

__global__ void set_i64_kernel(long long* p, long long v) { *p = v; }

// Output validity of one call, one thread per aligned 32-bit output word:
//   SkipNulls: the input validity;  otherwise: valid up to the first null, null from there on
//   (vector_cumulative.go:277-289), everything null once an earlier chunk met a null.
// Runs BEFORE cumsum_stream_kernel on the same stream (it needs the state as the call found it) and adds
// the number of null slots it wrote to state->null_count.
__global__ void __launch_bounds__(256)
cumsum_validity_kernel(const uint8_t* __restrict__ valid, int64_t voff, int64_t n, int skip_nulls, const long long* first_null,
                       CumsumState* state, uint32_t* __restrict__ out_words, int shift, int64_t n_words) {
  const bool dead = !skip_nulls && state->encountered_null != 0;
  const int64_t limit = dead ? 0 : ((valid && !skip_nulls) ? *first_null : n);
  const int64_t vlo = voff >> 3, vhi = (voff + n + 7) >> 3;
  long long nulls = 0;
  for (int64_t w = (int64_t)blockIdx.x * 256 + threadIdx.x; w < n_words; w += (int64_t)gridDim.x * 256) {
    const int64_t e0 = (w << 5) - shift;
    uint32_t v = 0xffffffffu;
    if (valid) v = bitmap_load32(valid, voff + e0, vlo, vhi);
    const int64_t room = limit - e0;  // rows e0+j with j >= room are null
    if (room < 32) v &= (room <= 0) ? 0u : ((1u << (int)room) - 1u);
    const int64_t lo64 = -e0, hi64 = n - e0;
    const int lo = lo64 > 0 ? (int)lo64 : 0;
    const int hi = hi64 < 32 ? (int)hi64 : 32;
    if (hi > lo) {
      const uint32_t m = bit_range_mask(lo, hi);
      bitmap_store32_masked(out_words + w, v, m);
      nulls += __popc(~v & m);
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) nulls += __shfl_xor_sync(0xffffffffu, nulls, d);
  if ((threadIdx.x & 31) == 0 && nulls) atomicAdd(reinterpret_cast<unsigned long long*>(&state->null_count), (unsigned long long)nulls);
}

template <typename T, bool kChecked>
ag_status launch_cumsum(CumsumParams& p, cudaStream_t st) {
  constexpr int S = StatusEntry<PolSel<T, kChecked>::type::K>::kStride;  // words per status entry
  constexpr int kTileRows = kScTileBytes / sizeof(T);
  Workspace* ws;
  AG_TRY(get_workspace(st, &ws));
  WorkspaceLock ws_lock(ws);
  p.n_tiles = (p.n + kTileRows - 1) / kTileRows;
  const int64_t n_groups = (p.n_tiles + kScGroup - 1) / kScGroup;
  const int64_t n_super = (n_groups + kScSuper - 1) / kScSuper;
  const size_t words = (size_t)(p.n_tiles + n_groups + n_super) * S;
  AG_TRY(ensure_tile_status(ws, words, st));
  p.agg = ws->tile_status;
  p.gagg = p.agg + p.n_tiles * S;
  p.sincl = p.gagg + n_groups * S;
  AG_CUDA_TRY(cudaMemsetAsync(ws->tile_status, 0, words * sizeof(unsigned long long), st));
  if (p.valid) {
    long long* fn = reinterpret_cast<long long*>(ws->scalars) + 8;  // slot 8 of the per-stream scalars
    set_i64_kernel<<<1, 1, 0, st>>>(fn, (long long)p.n);
    const int grid = grid_for((p.n + 31) >> 5, 256 * 4, 8);
    first_null_kernel<<<grid, 256, 0, st>>>(p.valid, p.voff, p.n, fn);
    AG_TRY(check_launch("first_null_kernel"));
    p.first_null = fn;
  }
  if (p.out_valid) {
    uint8_t* first = p.out_valid + (p.ooff >> 3);
    const uintptr_t a = reinterpret_cast<uintptr_t>(first);
    uint32_t* words = reinterpret_cast<uint32_t*>(a & ~(uintptr_t)3);
    const int shift = (int)(a & 3) * 8 + (int)(p.ooff & 7);
    const int64_t n_words = (p.n + shift + 31) >> 5;
    cumsum_validity_kernel<<<grid_for(n_words, 256, 8), 256, 0, st>>>(p.valid, p.voff, p.n, p.skip_nulls, p.first_null, p.state, words, shift, n_words);
    AG_TRY(check_launch("cumsum_validity_kernel"));
  }
  constexpr int kRing = kScStreamStages * kScTileBytes;
  static std::atomic<unsigned> attr_set{0u}, attr_set_v{0u};  // per instantiation, one bit per device
  const void* fn = p.valid ? (const void*)cumsum_stream_kernel<T, true, kChecked> : (const void*)cumsum_stream_kernel<T, false, kChecked>;
  AG_TRY(ensure_dynamic_smem(fn, kRing, p.valid ? &attr_set_v : &attr_set));
  int per_sm = 0;
  AG_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kScStreamThreads, kRing));
  if (per_sm < 1) per_sm = 1;
  const int64_t cap = (int64_t)sm_count() * per_sm;
  const int grid = (int)(p.n_tiles < cap ? p.n_tiles : cap);
  void* args[] = {(void*)&p};
  AG_CUDA_TRY(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(kScStreamThreads), args, kRing, st));
  return check_launch("cumsum_stream_kernel");
}

__global__ void cumsum_state_init_kernel(CumsumState* s, unsigned long long lo, long long hi) {
  s->lo = lo; s->hi = hi; s->encountered_null = 0; s->null_count = 0;
}

}  // namespace

ag_status cumulative_sum_dev(int type, const void* in, const uint8_t* valid, int64_t voff, int64_t n, int skip_nulls, int checked,
                             void* out, uint8_t* out_valid, int64_t ooff, void* d_state, int64_t* d_first_bad, cudaStream_t st) {
  if (n < 0 || voff < 0 || ooff < 0) AG_FAIL(AG_ERR_INVALID, "cumulative_sum: negative length or offset");
  if (type_width(type) == 0) AG_FAIL(AG_ERR_TYPE, "cumulative_sum: input type must be numeric, got type id %d", type);
  if (!d_state) AG_FAIL(AG_ERR_INVALID, "cumulative_sum: NULL state");
  if (checked && !d_first_bad) AG_FAIL(AG_ERR_INVALID, "cumulative_sum: the checked flavour needs an error word");
  if (n == 0) return AG_OK;
  if (!in || !out) AG_FAIL(AG_ERR_INVALID, "cumulative_sum: NULL operand");
  if (valid && !out_valid) AG_FAIL(AG_ERR_INVALID, "cumulative_sum: an input with a validity bitmap needs an output validity bitmap");
  CumsumParams p{};
  p.out_valid = out_valid; p.ooff = ooff;
  p.in = in; p.out = out; p.valid = valid; p.voff = voff; p.n = n; p.skip_nulls = skip_nulls;
  p.first_null = nullptr; p.state = static_cast<CumsumState*>(d_state); p.first_bad = (long long*)d_first_bad;
  // the type id was validated above; anything else would run as float64
  return visit_type(type, [&](auto tag) {
    using T = typename decltype(tag)::type;
    if constexpr (!IsFp<T>::v) {  // floats: the checked adder is the plain one
      if (checked) return launch_cumsum<T, true>(p, st);
    }
    return launch_cumsum<T, false>(p, st);
  }, [&] { return launch_cumsum<double, false>(p, st); });
}

ag_status cumulative_sum_state_init(void* d_state, int type, const void* start_host, cudaStream_t st) {
  if (!d_state) AG_FAIL(AG_ERR_INVALID, "cumulative_sum: NULL state");
  const int w = type_width(type);
  if (w == 0) AG_FAIL(AG_ERR_TYPE, "cumulative_sum: input type must be numeric, got type id %d", type);
  unsigned long long lo = 0;
  long long hi = 0;
  if (start_host) {
    visit_type(type, [&](auto tag) {
      using T = typename decltype(tag)::type;
      if constexpr (std::is_floating_point<T>::value) {
        memcpy(&lo, start_host, sizeof(T));  // bit pattern (float in the low 32 bits)
      } else {
        const T v = *(const T*)start_host;
        lo = (unsigned long long)v;  // sign-extends a signed start value
        if constexpr (std::is_signed<T>::value) hi = v < 0 ? -1 : 0;
      }
      return AG_OK;
    }, [] { return AG_OK; });  // the type id was validated above
  }
  cumsum_state_init_kernel<<<1, 1, 0, st>>>(static_cast<CumsumState*>(d_state), lo, hi);
  return check_launch("cumsum_state_init_kernel");
}

}  // namespace ag

using namespace ag;

extern "C" ag_status ag_cumulative_sum_state_init_dev(void* d_state, int type, const void* start_host, ag_stream_t s) {
  AG_TRY(ensure_init());
  return cumulative_sum_state_init(d_state, type, start_host, resolve_stream(s));
}

extern "C" ag_status ag_cumulative_sum_dev(int type, const void* d_in, const uint8_t* d_valid, int64_t valid_offset, int64_t n,
                                           int skip_nulls, int checked, void* d_out, uint8_t* d_out_valid, int64_t out_valid_offset,
                                           void* d_state, int64_t* d_first_bad, ag_stream_t s) {
  AG_TRY(ensure_init());
  return cumulative_sum_dev(type, d_in, d_valid, valid_offset, n, skip_nulls, checked, d_out, d_out_valid, out_valid_offset,
                            d_state, d_first_bad, resolve_stream(s));
}
