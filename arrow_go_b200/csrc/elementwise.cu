// elementwise.cu — scalar arithmetic kernels on sm_90a.
//
// Replaces arithmetic_{binary,arr_scalar,scalar_arr,unary_same_types,unary_diff_type}_{avx2,sse4}
// (arrow/compute/internal/kernels/_lib/base_arithmetic.cc:465-483) under ScalarBinary /
// ScalarUnary (kernels/helpers.go:42-60,193-236: every slot is computed, nulls included), and
// the pure-Go checked integer kernels (kernels/base_arithmetic.go:84-108,154-161,249-294) under
// ScalarBinaryNotNull (helpers.go:284-380).
//
// Roofline: HBM.  arr⊕arr moves 3 x width bytes per row (24 B for float64), arr⊕scalar 2 x width.
// One add per 24 bytes -> no tensor cores, no shared-memory reuse: the job is to keep
// >= 64 KB of 128-bit loads in flight per SM and to write with full 128-byte lines.
//
// Layout: 256-thread blocks, one resident wave (SMs x occupancy); a block streams contiguous
// 4096-row tiles, each thread moving 4 independent 16-byte vectors per operand at a time
// (ld.global.cs / st.global.cs — streaming, evict first: every byte is touched once).  A chunked
// call is ONE launch per 256 aligned spans.  Pointers that are only element-aligned (Arrow
// slices, Appendix D of SURVEY.md) keep the 128-bit accesses: the tile aligns on its output and
// funnel-shifts the inputs (shift_combine below); same arithmetic, same bits.
#include "common.cuh"
#include "elem_ops.cuh"

#include <algorithm>
#include <stdlib.h>
#include <type_traits>
#include <vector>

namespace ag {

constexpr int kEwThreads = 256;
constexpr int kEwUnroll = 4;
constexpr int kEwBlocksPerSM = 8;

template <typename T, int N> struct alignas(16) Vec { T v[N]; };

template <typename T>
__device__ __forceinline__ Vec<T, 16 / sizeof(T)> ldv(const T* p, int64_t vi) {
  const uint4 r = __ldcs(reinterpret_cast<const uint4*>(p) + vi);
  return *reinterpret_cast<const Vec<T, 16 / sizeof(T)>*>(&r);
}
template <typename T>
__device__ __forceinline__ void stv(T* p, int64_t vi, const Vec<T, 16 / sizeof(T)>& v) {
  __stcs(reinterpret_cast<uint4*>(p) + vi, *reinterpret_cast<const uint4*>(&v));
}

// ---- element-aligned operands (Arrow slices: base + offset*width is only element-aligned) ----------------------
// The kernels align on the OUTPUT (a few head elements go through the scalar path) and read a misaligned input as
// aligned 16-byte vectors: output vector v needs bytes [mb, mb+16) of the aligned pair (v, v+1).  Lane j loads aligned
// vector v_j and takes v_j+1 from lane j+1 by shuffle (lane 31 from lane 0's NEXT vector, which the same warp loads
// anyway), so HBM still sees every byte once and every access is a full 128-bit transaction — cf. the reference's
// prefix / suffix handling around its SIMD body, _lib/scalar_comparison.cc:72-95.
__device__ __forceinline__ uint4 shift_combine(const uint4 a, const uint4 b, int mb) {
  uint32_t w0, w1, w2, w3, w4;
  switch (mb >> 2) {
    case 0: w0 = a.x; w1 = a.y; w2 = a.z; w3 = a.w; w4 = b.x; break;
    case 1: w0 = a.y; w1 = a.z; w2 = a.w; w3 = b.x; w4 = b.y; break;
    case 2: w0 = a.z; w1 = a.w; w2 = b.x; w3 = b.y; w4 = b.z; break;
    default: w0 = a.w; w1 = b.x; w2 = b.y; w3 = b.z; w4 = b.w; break;
  }
  const int s = (mb & 3) * 8;
  return make_uint4(__funnelshift_r(w0, w1, s), __funnelshift_r(w1, w2, s), __funnelshift_r(w2, w3, s), __funnelshift_r(w3, w4, s));
}
// next aligned vector of every lane: lanes 0..30 read their right neighbour's `cur`, lane 31 reads lane 0's `nxt`
__device__ __forceinline__ uint4 neighbour_vector(const uint4 cur, const uint4 nxt, int lane) {
  const uint4 t = lane == 0 ? nxt : cur;
  const int src = (lane + 1) & 31;
  return make_uint4(__shfl_sync(0xffffffffu, t.x, src), __shfl_sync(0xffffffffu, t.y, src), __shfl_sync(0xffffffffu, t.z, src),
                    __shfl_sync(0xffffffffu, t.w, src));
}

// ---------------------------------------------------------------- binary -----------
static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ---------------------------------------------------------------- batched spans -----
// One launch for up to kSpanTable aligned spans of a chunked call (iterateExecSpans, executor.go:757-863,
// yields ~2 spans per chunk boundary; the reference runs its kernel once per span on one
// goroutine — here a span costs nothing extra).  Work is cut into tiles of kBinaryTileBytes per
// operand; the span table travels in the launch parameters, so the call puts nothing on the stream
// but the kernel, and every thread finds its tile's span in the table itself (a block-uniform index:
// the constant cache broadcasts it) by walking forward from its previous tile's span.
constexpr int kSpanTile = 4096;        // rows per tile of the checked kernels
constexpr int kSpanTileBytes = 32768;  // bytes per operand per tile of the unary kernel (4096 float64 rows)
// Bytes per operand per tile of binary_spans_kernel (2048 float64 rows).  Its blocks claim tiles, so the last tiles set
// how far apart the blocks finish: 16 KB tiles ran the 200-span float64 Add 0.7 % faster than 32 KB tiles and 3.3 %
// faster than 64 KB tiles on an H100 80GB HBM3 at 700 W.
constexpr int kBinaryTileBytes = 16384;

// Rows before the first 16-byte boundary of `out` (the span head).  Tiles start there, so inside a tile the output is
// always vector-aligned: a chunked call whose slices share one misalignment (pos*width off a 16-byte boundary on every
// operand — what executeSpans produces) runs entirely on the aligned path.
static __host__ __device__ __forceinline__ long long span_head(const void* out, int width, long long n) {
  const int N = 16 / width;
  const long long h = (N - (long long)((reinterpret_cast<uintptr_t>(out) & 15) / width)) & (N - 1);
  return h < n ? h : n;
}
// true when an array input of the span is not 16-byte aligned at the row where the output is
static inline bool span_needs_shift(int shape, const void* l, const void* r, const void* out, int width, long long n) {
  const uintptr_t hb = (uintptr_t)(span_head(out, width, n) * width);
  return (shape != AG_SHAPE_SA && ((reinterpret_cast<uintptr_t>(l) + hb) & 15)) ||
         (shape != AG_SHAPE_AS && ((reinterpret_cast<uintptr_t>(r) + hb) & 15));
}
static inline long long span_tiles(const void* out, int width, long long n, int tile_bytes) {
  const long long rows = tile_bytes / width;
  const long long body = n - span_head(out, width, n);
  const long long t = (body + rows - 1) / rows;
  return t > 0 ? t : 1;
}

struct SpanDesc {
  const void* l;
  const void* r;
  void* out;
  long long n;
  long long first_tile;  // number of tiles of this launch before this span
};

// Spans per launch of a chunked call: 256 x 40 B = 10 KB of launch parameters, copied at every launch, which holds the
// ~2 spans per chunk boundary of a 100-chunk column in one launch.  A call with more spans runs as several launches.
constexpr int kSpanTable = 256;
template <int kSpans> struct SpanTable { SpanDesc s[kSpans]; };

// kSpans: table capacity — 1 for the contiguous call and a single-span chunked call, kSpanTable otherwise.
// kShift: some span has an input that is not 16-byte aligned where its output is (the host checks); the common
// all-aligned call keeps the lean kernel (no shuffle path, 3 resident blocks per SM).
// Blocks claim tiles from the counter `next_tile` (zero at launch), one claim ahead so that the atomic's latency hides
// behind a tile: a block on a slower SM takes fewer tiles instead of finishing last.  The block that makes the last
// claim (each block makes one claim past the end) sets the counter back to zero for the next launch on the stream.
template <typename T, typename Op, int kShape, int kSpans, bool kShift>
__global__ void __launch_bounds__(kEwThreads, kShift ? 2 : 3)
binary_spans_kernel(const __grid_constant__ SpanTable<kSpans> table, int n_spans, long long total_tiles, T scalar,
                    unsigned* __restrict__ next_tile) {
  constexpr int N = 16 / sizeof(T);
  __shared__ unsigned s_tile[2];
  const auto claim = [&] {
    const unsigned t = atomicAdd(next_tile, 1u);
    if (t == total_tiles + gridDim.x - 1) *next_tile = 0;
    return t;
  };
  if (threadIdx.x == 0) s_tile[0] = claim();
  __syncthreads();
  int s = 0;
  for (int k = 0;; ++k) {
    const unsigned tile = s_tile[k & 1];
    if (tile >= total_tiles) break;
    if (threadIdx.x == 0) s_tile[(k + 1) & 1] = claim();
    while (kSpans > 1 && s + 1 < n_spans && table.s[s + 1].first_tile <= tile) ++s;   // a block's claims only grow: n_spans steps in all
    const SpanDesc sp = table.s[s];
    constexpr int kTile = kBinaryTileBytes / (int)sizeof(T);
    const long long head = span_head(sp.out, (int)sizeof(T), sp.n);
    const int t_in = (int)(tile - sp.first_tile);   // a span of 2^31 tiles would be 64 TB per operand
    if (t_in == 0 && threadIdx.x < head) {   // the few rows before the output's first 16-byte boundary
      const T* l0 = reinterpret_cast<const T*>(sp.l);
      const T* r0 = reinterpret_cast<const T*>(sp.r);
      reinterpret_cast<T*>(sp.out)[threadIdx.x] =
          Op::template apply<T>(kShape == AG_SHAPE_SA ? scalar : l0[threadIdx.x], kShape == AG_SHAPE_AS ? scalar : r0[threadIdx.x]);
    }
    const long long e0 = head + (long long)t_in * kTile;
    const long long rest = sp.n - e0;
    const int len = (int)(rest < kTile ? (rest > 0 ? rest : 0) : kTile);
    const T* l = reinterpret_cast<const T*>(sp.l) + (kShape == AG_SHAPE_SA ? 0 : e0);
    const T* r = reinterpret_cast<const T*>(sp.r) + (kShape == AG_SHAPE_AS ? 0 : e0);
    T* out = reinterpret_cast<T*>(sp.out) + e0;
    const bool vec = !kShift || (((kShape == AG_SHAPE_SA ? 0 : reinterpret_cast<uintptr_t>(l)) |
                                  (kShape == AG_SHAPE_AS ? 0 : reinterpret_cast<uintptr_t>(r))) & 15) == 0;
    if (vec) {
      const int nvec = len / N;
      constexpr int kIters = kTile / N / kEwThreads;  // vectors per thread in a full tile
#pragma unroll
      for (int b = 0; b < kIters; b += kEwUnroll) {
        Vec<T, N> a[kEwUnroll], c[kEwUnroll];
#pragma unroll
        for (int k = 0; k < kEwUnroll; ++k) {
          const int vi = (b + k) * kEwThreads + threadIdx.x;
          if (vi < nvec) {
            if (kShape != AG_SHAPE_SA) a[k] = ldv(l, vi);
            if (kShape != AG_SHAPE_AS) c[k] = ldv(r, vi);
          }
        }
#pragma unroll
        for (int k = 0; k < kEwUnroll; ++k) {
          const int vi = (b + k) * kEwThreads + threadIdx.x;
          if (vi < nvec) {
            Vec<T, N> o;
#pragma unroll
            for (int e = 0; e < N; ++e)
              o.v[e] = Op::template apply<T>(kShape == AG_SHAPE_SA ? scalar : a[k].v[e], kShape == AG_SHAPE_AS ? scalar : c[k].v[e]);
            stv(out, vi, o);
          }
        }
      }
      const int i = nvec * N + threadIdx.x;
      if (i < len) out[i] = Op::template apply<T>(kShape == AG_SHAPE_SA ? scalar : l[i], kShape == AG_SHAPE_AS ? scalar : r[i]);
    } else if constexpr (kShift) {
      // element-aligned inputs: the output is aligned, shift the inputs (see shift_combine)
      constexpr int ho = 0;                   // tiles start on an output vector boundary (span_head)
      const int nvec = len / N;
      {
        const int i = nvec * N + threadIdx.x;  // < N tail rows, last tile of the span only
        if (i < len) out[i] = Op::template apply<T>(kShape == AG_SHAPE_SA ? scalar : l[i], kShape == AG_SHAPE_AS ? scalar : r[i]);
      }
      const int mbl = kShape == AG_SHAPE_SA ? 0 : (int)(reinterpret_cast<uintptr_t>(l + ho) & 15);
      const int mbr = kShape == AG_SHAPE_AS ? 0 : (int)(reinterpret_cast<uintptr_t>(r + ho) & 15);
      const uint4* __restrict__ lf = reinterpret_cast<const uint4*>(reinterpret_cast<const char*>(l + ho) - mbl);
      const uint4* __restrict__ rf = reinterpret_cast<const uint4*>(reinterpret_cast<const char*>(r + ho) - mbr);
      uint4* __restrict__ ob = reinterpret_cast<uint4*>(out + ho);
      const int lane = threadIdx.x & 31;
      const int nl = nvec + (mbl ? 1 : 0), nr = nvec + (mbr ? 1 : 0);   // a shifted operand reads one vector more
      constexpr int kWarpVecs = 32 * kEwUnroll;
      for (int base = (threadIdx.x >> 5) * kWarpVecs; base < nvec; base += (kEwThreads / 32) * kWarpVecs) {
        uint4 a[kEwUnroll + 1], c[kEwUnroll + 1];
#pragma unroll
        for (int k = 0; k < kEwUnroll; ++k) {
          const int vi = base + k * 32 + lane;
          a[k] = make_uint4(0, 0, 0, 0); c[k] = make_uint4(0, 0, 0, 0);
          if (kShape != AG_SHAPE_SA && vi < nl) a[k] = __ldcs(lf + vi);
          if (kShape != AG_SHAPE_AS && vi < nr) c[k] = __ldcs(rf + vi);
        }
        a[kEwUnroll] = make_uint4(0, 0, 0, 0); c[kEwUnroll] = make_uint4(0, 0, 0, 0);
        if (lane == 0) {   // the vector after this warp's last one
          if (mbl && base + kWarpVecs < nl) a[kEwUnroll] = __ldcs(lf + base + kWarpVecs);
          if (mbr && base + kWarpVecs < nr) c[kEwUnroll] = __ldcs(rf + base + kWarpVecs);
        }
#pragma unroll
        for (int k = 0; k < kEwUnroll; ++k) {
          const int vi = base + k * 32 + lane;
          uint4 av = a[k], cv = c[k];
          if (mbl) av = shift_combine(a[k], neighbour_vector(a[k], a[k + 1], lane), mbl);
          if (mbr) cv = shift_combine(c[k], neighbour_vector(c[k], c[k + 1], lane), mbr);
          if (vi < nvec) {
            const Vec<T, N>& x = *reinterpret_cast<const Vec<T, N>*>(&av);
            const Vec<T, N>& y = *reinterpret_cast<const Vec<T, N>*>(&cv);
            Vec<T, N> o;
#pragma unroll
            for (int e = 0; e < N; ++e)
              o.v[e] = Op::template apply<T>(kShape == AG_SHAPE_SA ? scalar : x.v[e], kShape == AG_SHAPE_AS ? scalar : y.v[e]);
            __stcs(ob + vi, *reinterpret_cast<const uint4*>(&o));
          }
        }
      }
    }
    __syncthreads();   // every thread has read s_tile[k & 1] before thread 0 stores claim k + 2 there
  }
}

// One launch of binary_spans_kernel over the host table `spans` of 1..kSpanTable spans (first_tile counted from this
// launch's first span).  `scalar_host` is the host scalar of an AS / SA call; `chunked` marks a call that came in
// through the span entry point.
struct SpanLaunch {
  const SpanDesc* spans;
  int n_spans;
  long long tiles;
  const void* scalar_host;
  bool shift;  // span_needs_shift for some span
  bool chunked;
};

template <typename T, typename Op, int kShape, int kSpans>
static ag_status launch_table_t(const SpanLaunch& a, T scalar, cudaStream_t st) {
  SpanTable<kSpans> table{};
  for (int i = 0; i < a.n_spans; ++i) table.s[i] = a.spans[i];
  Workspace* ws = nullptr;
  AG_TRY(get_workspace(st, &ws));
  WorkspaceLock lk(ws);   // the tile counter is the stream's ticket: one kernel sequence at a time
  const auto go = [&](auto kernel) {
    kernel<<<grid_one_wave(kernel, kEwThreads, a.tiles), kEwThreads, 0, st>>>(table, a.n_spans, a.tiles, scalar, ws->ticket);
    return check_launch("binary_spans_kernel");
  };
  return a.shift ? go(binary_spans_kernel<T, Op, kShape, kSpans, true>) : go(binary_spans_kernel<T, Op, kShape, kSpans, false>);
}

template <typename T, typename Op, int kShape>
static ag_status launch_spans_t(const SpanLaunch& a, cudaStream_t st) {
  const T scalar = kShape == AG_SHAPE_AA ? T(0) : *reinterpret_cast<const T*>(a.scalar_host);
  return a.n_spans == 1 ? launch_table_t<T, Op, kShape, 1>(a, scalar, st) : launch_table_t<T, Op, kShape, kSpanTable>(a, scalar, st);
}

template <typename T, typename Op>
static ag_status launch_binary_shape(int shape, const SpanLaunch& a, cudaStream_t st) {
  return visit_shape(shape, [&](auto s) { return launch_spans_t<T, Op, decltype(s)::value>(a, st); },
                     [&] { AG_FAIL(AG_ERR_INVALID, "arith: bad operand shape %d", shape); });
}

static ag_status launch_binary(int type, int8_t op, int shape, const SpanLaunch& a, cudaStream_t st) {
  return visit_storage_type(type, [&](auto tag) {
    using T = typename decltype(tag)::type;
    switch (op) {
      // the *_CHECKED aliases are the plain loops here, like the reference's native code
      // (base_arithmetic.cc:445-462); the checking variants are ag_arith_checked.
      case AG_OP_ADD: case AG_OP_ADD_CHECKED: return launch_binary_shape<T, OpAdd>(shape, a, st);
      case AG_OP_SUB: case AG_OP_SUB_CHECKED: return launch_binary_shape<T, OpSub>(shape, a, st);
      case AG_OP_MUL: case AG_OP_MUL_CHECKED: return launch_binary_shape<T, OpMul>(shape, a, st);
      case AG_OP_BIT_AND: case AG_OP_BIT_OR: case AG_OP_BIT_XOR:
        if constexpr (std::is_integral<T>::value) {
          if (op == AG_OP_BIT_AND) return launch_binary_shape<T, OpBitAnd>(shape, a, st);
          if (op == AG_OP_BIT_OR) return launch_binary_shape<T, OpBitOr>(shape, a, st);
          return launch_binary_shape<T, OpBitXor>(shape, a, st);
        } else {
          AG_FAIL(AG_ERR_TYPE, "arith: bitwise ops take integer types");
        }
      default:
        AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "arith: binary op %d has no native kernel%s", (int)op,
                a.chunked ? "" : " (the reference has none either)");
    }
  }, [&] { AG_FAIL(AG_ERR_TYPE, "arith: unsupported type id %d", type); });
}

// The contiguous call: one span by value through the same tile kernel (contiguous 16 KB tiles per
// block iteration streamed faster than a grid-strided loop), any element alignment.
ag_status arith_binary_dev(int type, int8_t op, int shape, const void* l, const void* r, void* out, int64_t n, cudaStream_t st) {
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "arith: negative length");
  if (n == 0) return AG_OK;
  const int w = type_width(type);
  if (w == 0) AG_FAIL(AG_ERR_TYPE, "arith: unsupported type id %d", type);
  const uintptr_t m = (uintptr_t)(w - 1);
  if (((uintptr_t)out & m) || (shape != AG_SHAPE_SA && ((uintptr_t)l & m)) || (shape != AG_SHAPE_AS && ((uintptr_t)r & m)))
    AG_FAIL(AG_ERR_INVALID, "arith: operand not aligned to its element width");
  const void* lp = shape == AG_SHAPE_SA ? nullptr : l;
  const void* rp = shape == AG_SHAPE_AS ? nullptr : r;
  const void* scalar_host = shape == AG_SHAPE_AS ? r : (shape == AG_SHAPE_SA ? l : nullptr);
  const SpanDesc one{lp, rp, out, (long long)n, 0};
  return launch_binary(type, op, shape, SpanLaunch{&one, 1, span_tiles(out, w, n, kBinaryTileBytes), scalar_host, span_needs_shift(shape, lp, rp, out, w, n), false}, st);
}

// spans: HOST array of {l, r, out, n} with DEVICE pointers (the scalar side is a HOST pointer to
// one element and must be the same pointer in every span).  The non-empty spans run kSpanTable at a time, one launch
// each; every span is checked before the first launch.
ag_status arith_binary_spans_dev(int type, int8_t op, int shape, const ag_span3* spans, int64_t n_spans, cudaStream_t st) {
  if (n_spans < 0) AG_FAIL(AG_ERR_INVALID, "arith_spans: negative span count");
  const int w = type_width(type);
  if (w == 0) AG_FAIL(AG_ERR_TYPE, "arith: unsupported type id %d", type);
  std::vector<SpanDesc> desc;
  desc.reserve((size_t)n_spans);
  const void* scalar_host = nullptr;
  const uintptr_t m = (uintptr_t)(w - 1);
  for (int64_t i = 0; i < n_spans; ++i) {
    const ag_span3& s = spans[i];
    if (s.n < 0) AG_FAIL(AG_ERR_INVALID, "arith_spans: negative length");
    if (s.n == 0) continue;
    if (!s.l || !s.r || !s.out) AG_FAIL(AG_ERR_INVALID, "arith_spans: NULL operand in span %lld", (long long)i);
    if (((uintptr_t)s.out & m) || (shape != AG_SHAPE_SA && ((uintptr_t)s.l & m)) || (shape != AG_SHAPE_AS && ((uintptr_t)s.r & m)))
      AG_FAIL(AG_ERR_INVALID, "arith_spans: operand not aligned to its element width");
    if (shape == AG_SHAPE_AS) scalar_host = s.r;
    if (shape == AG_SHAPE_SA) scalar_host = s.l;
    desc.push_back(SpanDesc{s.l, s.r, s.out, (long long)s.n, 0});
  }
  for (size_t first = 0; first < desc.size(); first += kSpanTable) {
    const int cnt = (int)std::min(desc.size() - first, (size_t)kSpanTable);
    long long tiles = 0;
    bool shift = false;
    for (int i = 0; i < cnt; ++i) {
      SpanDesc& d = desc[first + i];
      d.first_tile = tiles;
      shift = shift || span_needs_shift(shape, d.l, d.r, d.out, w, d.n);
      tiles += span_tiles(d.out, w, d.n, kBinaryTileBytes);
    }
    AG_TRY(launch_binary(type, op, shape, SpanLaunch{desc.data() + first, cnt, tiles, scalar_host, shift, true}, st));
  }
  return AG_OK;
}

// ---------------------------------------------------------------- unary ------------
// Same shape as binary_spans_kernel: tiles of 32 KB that start on the output's first 16-byte boundary; a warp owns 128
// consecutive vectors of a tile (4 x 16-byte loads in flight per lane); kShift adds the shuffle / funnel-shift read of an
// input that is not 16-byte aligned where the output is (an Arrow slice).
template <typename T, typename Op, bool kShift>
__global__ void __launch_bounds__(kEwThreads)
unary_vec_kernel(const T* __restrict__ in, T* __restrict__ out, int64_t n) {
  constexpr int N = 16 / sizeof(T);
  constexpr int kTile = kSpanTileBytes / (int)sizeof(T);
  const long long head = span_head(out, (int)sizeof(T), n);
  if (blockIdx.x == 0 && threadIdx.x < head) out[threadIdx.x] = Op::template apply<T, T>(in[threadIdx.x]);
  const int64_t body = n - head;
  const int64_t n_tiles = (body + kTile - 1) / kTile;
  const int lane = threadIdx.x & 31;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t e0 = head + tile * kTile;
    const int len = (int)((n - e0 < kTile) ? (n - e0) : kTile);
    const T* ip = in + e0;
    T* op = out + e0;
    const int nvec = len / N;
    {
      const int i = nvec * N + threadIdx.x;   // < N tail rows, last tile only
      if (i < len) op[i] = Op::template apply<T, T>(ip[i]);
    }
    const int mb = kShift ? (int)(reinterpret_cast<uintptr_t>(ip) & 15) : 0;
    const uint4* __restrict__ vf = reinterpret_cast<const uint4*>(reinterpret_cast<const char*>(ip) - mb);
    uint4* __restrict__ ob = reinterpret_cast<uint4*>(op);
    const int nin = nvec + (mb ? 1 : 0);
    constexpr int kWarpVecs = 32 * kEwUnroll;
    for (int base = (threadIdx.x >> 5) * kWarpVecs; base < nvec; base += (kEwThreads / 32) * kWarpVecs) {
      uint4 a[kEwUnroll + 1];
#pragma unroll
      for (int k = 0; k < kEwUnroll; ++k) {
        const int vi = base + k * 32 + lane;
        a[k] = make_uint4(0, 0, 0, 0);
        if (vi < nin) a[k] = __ldcs(vf + vi);
      }
      a[kEwUnroll] = make_uint4(0, 0, 0, 0);
      if (kShift && mb && lane == 0 && base + kWarpVecs < nin) a[kEwUnroll] = __ldcs(vf + base + kWarpVecs);
#pragma unroll
      for (int k = 0; k < kEwUnroll; ++k) {
        const int vi = base + k * 32 + lane;
        uint4 av = a[k];
        if (kShift && mb) av = shift_combine(a[k], neighbour_vector(a[k], a[k + 1], lane), mb);
        if (vi < nvec) {
          const Vec<T, N>& x = *reinterpret_cast<const Vec<T, N>*>(&av);
          Vec<T, N> o;
#pragma unroll
          for (int e = 0; e < N; ++e) o.v[e] = Op::template apply<T, T>(x.v[e]);
          __stcs(ob + vi, *reinterpret_cast<const uint4*>(&o));
        }
      }
    }
  }
}

template <typename TI, typename TO, typename Op>
__global__ void __launch_bounds__(kEwThreads)
unary_scalar_kernel(const TI* __restrict__ in, TO* __restrict__ out, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * kEwThreads;
  for (int64_t i = (int64_t)blockIdx.x * kEwThreads + threadIdx.x; i < n; i += stride)
    out[i] = Op::template apply<TO, TI>(in[i]);
}

template <typename T, typename Op>
static ag_status launch_unary_same_t(const void* in, void* out, int64_t n, cudaStream_t st) {
  const int64_t tiles = span_tiles(out, (int)sizeof(T), n, kSpanTileBytes);
  if (span_needs_shift(AG_SHAPE_AS, in, nullptr, out, (int)sizeof(T), n)) {   // "array op scalar" = one array input
    const int grid = grid_one_wave(unary_vec_kernel<T, Op, true>, kEwThreads, tiles);
    unary_vec_kernel<T, Op, true><<<grid, kEwThreads, 0, st>>>((const T*)in, (T*)out, n);
  } else {
    const int grid = grid_one_wave(unary_vec_kernel<T, Op, false>, kEwThreads, tiles);
    unary_vec_kernel<T, Op, false><<<grid, kEwThreads, 0, st>>>((const T*)in, (T*)out, n);
  }
  return check_launch("unary_kernel");
}

template <typename T>
static ag_status launch_unary_same_op(int8_t op, const void* in, void* out, int64_t n, cudaStream_t st) {
  switch (op) {
    case AG_OP_ABS: case AG_OP_ABS_CHECKED: return launch_unary_same_t<T, UAbs>(in, out, n, st);
    case AG_OP_NEGATE: return launch_unary_same_t<T, UNeg>(in, out, n, st);
    case AG_OP_NEGATE_CHECKED: return launch_unary_same_t<T, UNegChecked>(in, out, n, st);
    case AG_OP_SIGN: return launch_unary_same_t<T, USign>(in, out, n, st);
    case AG_OP_BIT_NOT:
      if constexpr (std::is_integral<T>::value) return launch_unary_same_t<T, UBitNot>(in, out, n, st);
      else AG_FAIL(AG_ERR_TYPE, "arith: bit_wise_not takes integer types");
    default: AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "arith: unary op %d has no native kernel", (int)op);
  }
}

ag_status arith_unary_same_dev(int type, int8_t op, const void* in, void* out, int64_t n, cudaStream_t st) {
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "arith: negative length");
  if (n == 0) return AG_OK;
  return visit_type(type, [&](auto tag) { return launch_unary_same_op<typename decltype(tag)::type>(op, in, out, n, st); },
                    [&] { AG_FAIL(AG_ERR_TYPE, "arith: unsupported type id %d", type); });
}

template <typename TI>
static ag_status launch_sign_diff(int otype, const void* in, void* out, int64_t n, cudaStream_t st) {
  const int grid = grid_for(n, kEwThreads * kEwUnroll, kEwBlocksPerSM);
  return visit_type(otype, [&](auto tag) {
    using TO = typename decltype(tag)::type;
    unary_scalar_kernel<TI, TO, USign><<<grid, kEwThreads, 0, st>>>((const TI*)in, (TO*)out, n);
    return check_launch("sign_diff_kernel");
  }, [&] { AG_FAIL(AG_ERR_TYPE, "arith: unsupported output type id %d", otype); });
}

ag_status arith_unary_diff_dev(int itype, int otype, int8_t op, const void* in, void* out, int64_t n, cudaStream_t st) {
  if (op != AG_OP_SIGN) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "arith: unary_diff_type only implements SIGN (base_arithmetic.cc:427-438)");
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "arith: negative length");
  if (n == 0) return AG_OK;
  const auto not_int = [&] { AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "arith: sign with differing types needs an integer input"); };
  return visit_type(itype, [&](auto tag) {
    using TI = typename decltype(tag)::type;
    if constexpr (std::is_integral<TI>::value) return launch_sign_diff<TI>(otype, in, out, n, st);
    else return not_int();
  }, not_int);
}

// ---------------------------------------------------------------- checked ----------
// kNotNull: ScalarBinaryNotNull slot semantics (null slots written as 0, not computed);
// otherwise ScalarBinary (every slot computed — MUL_CHECKED, base_arithmetic.go:279-286).
template <typename ST, typename Op, int kShape, bool kNotNull, bool kHasValid>
__global__ void __launch_bounds__(kEwThreads)
checked_kernel(const ST* __restrict__ l, const uint8_t* __restrict__ lvalid, int64_t loff,
               const ST* __restrict__ r, const uint8_t* __restrict__ rvalid, int64_t roff,
               ST* __restrict__ out, int64_t n, ST scalar, long long* __restrict__ first_bad) {
  // A warp's rows in one step are 32 consecutive rows starting at a multiple of 32, so the 32
  // validity bits are ONE window of each bitmap (a warp-uniform load) instead of 32 byte loads.
  // One row per thread per iteration at full occupancy measured faster than a 4-way unrolled variant.
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * kEwThreads;
  const int64_t l_lo = loff >> 3, l_hi = (loff + n + 7) >> 3, r_lo = roff >> 3, r_hi = (roff + n + 7) >> 3;
  long long my_bad = AG_NO_ERROR_POS;
  const int64_t n_up = (n + 31) & ~(int64_t)31;  // keep whole warps in the loop (the window load is warp-uniform)
  for (int64_t i = (int64_t)blockIdx.x * kEwThreads + threadIdx.x; i < n_up; i += stride) {
    bool valid = i < n;
    if (kNotNull && kHasValid) {  // the no-bitmap instantiation stays small (24 registers, full occupancy)
      const int64_t row32 = i - lane;
      uint32_t w = 0xffffffffu;
      if (kShape != AG_SHAPE_SA && lvalid) w &= bitmap_load32(lvalid, loff + row32, l_lo, l_hi);
      if (kShape != AG_SHAPE_AS && rvalid) w &= bitmap_load32(rvalid, roff + row32, r_lo, r_hi);
      valid = valid && ((w >> lane) & 1);
    }
    ST o = 0;
    if (valid) {
      const ST a = (kShape == AG_SHAPE_SA) ? scalar : l[i];
      const ST b = (kShape == AG_SHAPE_AS) ? scalar : r[i];
      bool bad;
      o = Op::apply(a, b, bad);
      if (bad && (long long)i < my_bad) my_bad = (long long)i;
    }
    if (i < n) out[i] = o;
  }
  lower_error_row(my_bad, first_bad);
}


// Vectorised form of checked_kernel for 16-byte aligned operands: the Add tile loop (contiguous
// 4096-row tiles, 4 x 16-byte vectors in flight per operand) with the validity bits of a lane's
// N rows taken from one 32-bit window of each bitmap.
template <typename ST, typename Op, int kShape, bool kNotNull, bool kHasValid>
__global__ void __launch_bounds__(kEwThreads)
checked_tile_kernel(const ST* __restrict__ l, const uint8_t* __restrict__ lvalid, int64_t loff,
                    const ST* __restrict__ r, const uint8_t* __restrict__ rvalid, int64_t roff,
                    ST* __restrict__ out, int64_t n, ST scalar, long long* __restrict__ first_bad) {
  constexpr int N = 16 / sizeof(ST);
  constexpr uint32_t kNMask = (N >= 32) ? 0xffffffffu : ((1u << N) - 1u);
  const int lane = threadIdx.x & 31;
  const int64_t l_lo = loff >> 3, l_hi = (loff + n + 7) >> 3, r_lo = roff >> 3, r_hi = (roff + n + 7) >> 3;
  const int64_t n_tiles = (n + kSpanTile - 1) / kSpanTile;
  long long my_bad = AG_NO_ERROR_POS;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t e0 = tile * kSpanTile;
    const int len = (int)((n - e0 < kSpanTile) ? (n - e0) : kSpanTile);
    const int nvec = len / N;
    constexpr int kIters = (kSpanTile / N + kEwThreads - 1) / kEwThreads;
#pragma unroll
    for (int b0 = 0; b0 < kIters; b0 += kEwUnroll) {
      Vec<ST, N> a[kEwUnroll], b[kEwUnroll];
      uint32_t vbits[kEwUnroll];
      // A warp owns kEwUnroll*32 CONSECUTIVE vectors of the chunk (k-th load = vectors k*32 .. k*32+31 of
      // them), i.e. kEwUnroll*32*N consecutive rows = kEwUnroll*N validity words: lane j fetches word j
      // (and j+32 for the 1-byte types) of both bitmaps ONCE per chunk and the lanes pick their bits out
      // of it with a shuffle — the per-load version spent more issue slots on bitmap addressing than on
      // the arithmetic.
      const int vbase = b0 * kEwThreads + (threadIdx.x >> 5) * (kEwUnroll * 32);  // first vector of this warp in the tile
      constexpr int kWords = kEwUnroll * N;                                      // <= 64
      uint32_t wv0 = 0xffffffffu, wv1 = 0xffffffffu;
      if (kNotNull && kHasValid) {
        const int64_t wrow0 = e0 + (int64_t)vbase * N;
        if (lane < kWords && wrow0 + (int64_t)lane * 32 < e0 + len) {
          if (kShape != AG_SHAPE_SA && lvalid) wv0 &= bitmap_load32(lvalid, loff + wrow0 + lane * 32, l_lo, l_hi);
          if (kShape != AG_SHAPE_AS && rvalid) wv0 &= bitmap_load32(rvalid, roff + wrow0 + lane * 32, r_lo, r_hi);
        }
        if (kWords > 32 && lane + 32 < kWords && wrow0 + (int64_t)(lane + 32) * 32 < e0 + len) {
          if (kShape != AG_SHAPE_SA && lvalid) wv1 &= bitmap_load32(lvalid, loff + wrow0 + (lane + 32) * 32, l_lo, l_hi);
          if (kShape != AG_SHAPE_AS && rvalid) wv1 &= bitmap_load32(rvalid, roff + wrow0 + (lane + 32) * 32, r_lo, r_hi);
        }
      }
#pragma unroll
      for (int k = 0; k < kEwUnroll; ++k) {
        const int vi = vbase + k * 32 + lane;
        vbits[k] = kNMask;
        if (kNotNull && kHasValid) {
          const int word = k * N + ((lane * N) >> 5);  // warp-relative validity word of this lane's N rows
          uint32_t w = __shfl_sync(0xffffffffu, wv0, word & 31);
          if (kWords > 32) { const uint32_t w1 = __shfl_sync(0xffffffffu, wv1, word & 31); if (word >= 32) w = w1; }
          vbits[k] = (w >> ((lane * N) & 31)) & kNMask;
        }
        if (vi < nvec) {
          if (kShape != AG_SHAPE_SA) a[k] = ldv(l + e0, vi);
          if (kShape != AG_SHAPE_AS) b[k] = ldv(r + e0, vi);
        }
      }
#pragma unroll
      for (int k = 0; k < kEwUnroll; ++k) {
        const int vi = vbase + k * 32 + lane;
        if (vi < nvec) {
          Vec<ST, N> o;
#pragma unroll
          for (int e = 0; e < N; ++e) {
            o.v[e] = 0;
            if ((vbits[k] >> e) & 1) {
              bool bad;
              o.v[e] = Op::apply(kShape == AG_SHAPE_SA ? scalar : a[k].v[e], kShape == AG_SHAPE_AS ? scalar : b[k].v[e], bad);
              const long long row = (long long)(e0 + (int64_t)vi * N + e);
              if (bad && row < my_bad) my_bad = row;
            }
          }
          stv(out + e0, vi, o);
        }
      }
    }
    // tail of the last tile (< N rows)
    const int i = nvec * N + threadIdx.x;
    if (i < len) {
      const int64_t row = e0 + i;
      bool valid = true;
      if (kNotNull && kHasValid) {
        if (kShape != AG_SHAPE_SA && lvalid) valid = bit_is_set(lvalid, loff + row);
        if (kShape != AG_SHAPE_AS && rvalid) valid = valid && bit_is_set(rvalid, roff + row);
      }
      ST o = 0;
      if (valid) {
        bool bad;
        o = Op::apply(kShape == AG_SHAPE_SA ? scalar : l[row], kShape == AG_SHAPE_AS ? scalar : r[row], bad);
        if (bad && (long long)row < my_bad) my_bad = (long long)row;
      }
      out[row] = o;
    }
  }
  lower_error_row(my_bad, first_bad);
}

template <typename ST, typename Op, bool kNotNull>
static ag_status launch_checked_shape(int shape, const void* l, const uint8_t* lvalid, int64_t loff,
                                      const void* r, const uint8_t* rvalid, int64_t roff,
                                      void* out, int64_t n, int64_t* d_first_bad, cudaStream_t st) {
  const int grid = grid_for(n, kEwThreads * kEwUnroll, kEwBlocksPerSM);
  long long* fb = reinterpret_cast<long long*>(d_first_bad);
  const bool hv = kNotNull && ((shape != AG_SHAPE_SA && lvalid) || (shape != AG_SHAPE_AS && rvalid));
  const bool vec = aligned16(out) && (shape == AG_SHAPE_SA || aligned16(l)) && (shape == AG_SHAPE_AS || aligned16(r));
  return visit_shape(shape, [&](auto s) {
    constexpr int kShape = decltype(s)::value;
    // the scalar side passes no array and no bitmap; only the kHasValid instantiation gets the bitmaps
    const ST* lp = kShape == AG_SHAPE_SA ? nullptr : (const ST*)l;
    const ST* rp = kShape == AG_SHAPE_AS ? nullptr : (const ST*)r;
    const ST scalar = kShape == AG_SHAPE_AS ? *(const ST*)r : (kShape == AG_SHAPE_SA ? *(const ST*)l : ST(0));
    const bool lbits = hv && kShape != AG_SHAPE_SA, rbits = hv && kShape != AG_SHAPE_AS;
    const uint8_t* lv = lbits ? lvalid : nullptr;
    const uint8_t* rv = rbits ? rvalid : nullptr;
    const int64_t lo = lbits ? loff : 0, ro = rbits ? roff : 0;
    const auto go = [&](auto tile_kernel, auto row_kernel) {
      if (vec)
        tile_kernel<<<grid_one_wave(tile_kernel, kEwThreads, (n + kSpanTile - 1) / kSpanTile), kEwThreads, 0, st>>>(lp, lv, lo, rp, rv, ro, (ST*)out, n, scalar, fb);
      else
        row_kernel<<<grid, kEwThreads, 0, st>>>(lp, lv, lo, rp, rv, ro, (ST*)out, n, scalar, fb);
      return check_launch("checked_kernel");
    };
    if (hv) return go(checked_tile_kernel<ST, Op, kShape, kNotNull, true>, checked_kernel<ST, Op, kShape, kNotNull, true>);
    return go(checked_tile_kernel<ST, Op, kShape, kNotNull, false>, checked_kernel<ST, Op, kShape, kNotNull, false>);
  }, [&] { AG_FAIL(AG_ERR_INVALID, "arith_checked: bad operand shape %d", shape); });
}

template <typename ST>
static ag_status launch_checked_op(int8_t op, int shape, const void* l, const uint8_t* lvalid, int64_t loff,
                                   const void* r, const uint8_t* rvalid, int64_t roff,
                                   void* out, int64_t n, int64_t* d_first_bad, cudaStream_t st) {
  switch (op) {
    case AG_OP_ADD_CHECKED: return launch_checked_shape<ST, ChkAdd<ST>, true>(shape, l, lvalid, loff, r, rvalid, roff, out, n, d_first_bad, st);
    case AG_OP_SUB_CHECKED: return launch_checked_shape<ST, ChkSub<ST>, true>(shape, l, lvalid, loff, r, rvalid, roff, out, n, d_first_bad, st);
    case AG_OP_MUL_CHECKED: return launch_checked_shape<ST, ChkMul<ST>, false>(shape, l, lvalid, loff, r, rvalid, roff, out, n, d_first_bad, st);
    case AG_OP_DIV: case AG_OP_DIV_CHECKED: return launch_checked_shape<ST, ChkDiv<ST>, true>(shape, l, lvalid, loff, r, rvalid, roff, out, n, d_first_bad, st);
    case AG_OP_SHIFT_LEFT: return launch_checked_shape<ST, ChkShift<ST, true, false>, true>(shape, l, lvalid, loff, r, rvalid, roff, out, n, d_first_bad, st);
    case AG_OP_SHIFT_RIGHT: return launch_checked_shape<ST, ChkShift<ST, false, false>, true>(shape, l, lvalid, loff, r, rvalid, roff, out, n, d_first_bad, st);
    case AG_OP_SHIFT_LEFT_CHECKED: return launch_checked_shape<ST, ChkShift<ST, true, true>, true>(shape, l, lvalid, loff, r, rvalid, roff, out, n, d_first_bad, st);
    case AG_OP_SHIFT_RIGHT_CHECKED: return launch_checked_shape<ST, ChkShift<ST, false, true>, true>(shape, l, lvalid, loff, r, rvalid, roff, out, n, d_first_bad, st);
    default: AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "arith_checked: op %d is not a checked integer op", (int)op);
  }
}

template <typename FT>
static ag_status launch_checked_fdiv(int8_t op, int shape, const void* l, const uint8_t* lvalid, int64_t loff,
                                     const void* r, const uint8_t* rvalid, int64_t roff,
                                     void* out, int64_t n, int64_t* d_first_bad, cudaStream_t st) {
  switch (op) {
    case AG_OP_DIV: return launch_checked_shape<FT, ChkFDiv<FT, false>, true>(shape, l, lvalid, loff, r, rvalid, roff, out, n, d_first_bad, st);
    case AG_OP_DIV_CHECKED: return launch_checked_shape<FT, ChkFDiv<FT, true>, true>(shape, l, lvalid, loff, r, rvalid, roff, out, n, d_first_bad, st);
    default: AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "arith_checked: op %d on a floating point type (only DIV / DIV_CHECKED have NotNull float kernels)", (int)op);
  }
}

ag_status arith_checked_dev(int type, int8_t op, int shape, const void* l, const uint8_t* lvalid, int64_t loff,
                            const void* r, const uint8_t* rvalid, int64_t roff,
                            void* out, int64_t n, int64_t* d_first_bad, cudaStream_t st) {
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "arith_checked: negative length");
  if (n == 0) return AG_OK;
  // null scalar: "fast path if one side is entirely null" (helpers.go:287,314,341) — output untouched
  if ((shape == AG_SHAPE_SA && !l) || (shape == AG_SHAPE_AS && !r)) return AG_OK;
  return visit_type(type, [&](auto tag) {
    using T = typename decltype(tag)::type;
    if constexpr (std::is_floating_point<T>::value) return launch_checked_fdiv<T>(op, shape, l, lvalid, loff, r, rvalid, roff, out, n, d_first_bad, st);
    else return launch_checked_op<T>(op, shape, l, lvalid, loff, r, rvalid, roff, out, n, d_first_bad, st);
  }, [&] { AG_FAIL(AG_ERR_TYPE, "arith_checked: type id %d is not a numeric type", type); });
}

// AbsoluteValueChecked / NegateChecked on signed integers (base_arithmetic.go:295-340): ScalarUnary,
// i.e. every slot; v == MinInt -> errOverflow.
template <typename ST, bool kAbs>
__global__ void __launch_bounds__(kEwThreads)
unary_checked_kernel(const ST* __restrict__ in, ST* __restrict__ out, int64_t n, long long* __restrict__ first_bad) {
  using U = typename std::make_unsigned<ST>::type;
  constexpr ST tmin = (ST)((U)1 << (sizeof(ST) * 8 - 1));
  const int64_t stride = (int64_t)gridDim.x * kEwThreads;
  long long my_bad = AG_NO_ERROR_POS;
  for (int64_t i = (int64_t)blockIdx.x * kEwThreads + threadIdx.x; i < n; i += stride) {
    const ST v = in[i];
    if (v == tmin && (long long)i < my_bad) my_bad = (long long)i;
    out[i] = kAbs ? UAbs::apply<ST, ST>(v) : UNeg::apply<ST, ST>(v);
  }
  lower_error_row(my_bad, first_bad);
}

template <typename ST>
static ag_status launch_unary_checked(int8_t op, const void* in, void* out, int64_t n, int64_t* d_first_bad, cudaStream_t st) {
  const int64_t need = (n + kEwThreads * kEwUnroll - 1) / (kEwThreads * kEwUnroll);
  if (op == AG_OP_ABS_CHECKED)
    unary_checked_kernel<ST, true><<<grid_one_wave(unary_checked_kernel<ST, true>, kEwThreads, need), kEwThreads, 0, st>>>((const ST*)in, (ST*)out, n, (long long*)d_first_bad);
  else
    unary_checked_kernel<ST, false><<<grid_one_wave(unary_checked_kernel<ST, false>, kEwThreads, need), kEwThreads, 0, st>>>((const ST*)in, (ST*)out, n, (long long*)d_first_bad);
  return check_launch("unary_checked_kernel");
}

ag_status arith_unary_checked_dev(int type, int8_t op, const void* in, void* out, int64_t n, int64_t* d_first_bad, cudaStream_t st) {
  if (op != AG_OP_ABS_CHECKED && op != AG_OP_NEGATE_CHECKED) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "arith_unary_checked: op %d", (int)op);
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "arith: negative length");
  if (n == 0) return AG_OK;
  // unsigned / floating: cannot overflow; an unknown type id is refused by arith_unary_same_dev
  const auto unchecked = [&] { return arith_unary_same_dev(type, op, in, out, n, st); };
  return visit_type(type, [&](auto tag) {
    using T = typename decltype(tag)::type;
    if constexpr (std::is_integral<T>::value && std::is_signed<T>::value) return launch_unary_checked<T>(op, in, out, n, d_first_bad, st);
    else return unchecked();
  }, unchecked);
}

__global__ void reset_error_word_kernel(long long* w) { *w = AG_NO_ERROR_POS; }

ag_status error_word_reset(int64_t* d_word, cudaStream_t st) {
  reset_error_word_kernel<<<1, 1, 0, st>>>((long long*)d_word);
  return check_launch("reset_error_word_kernel");
}

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_arith_binary_dev(int type, int8_t op, int shape, const void* l, const void* r, void* out, int64_t n, ag_stream_t s) {
  AG_TRY(ensure_init());
  return arith_binary_dev(type, op, shape, l, r, out, n, resolve_stream(s));
}
ag_status ag_arith_binary_spans_dev(int type, int8_t op, int shape, const ag_span3* spans, int64_t n_spans, ag_stream_t s) {
  AG_TRY(ensure_init());
  if (n_spans > 0 && !spans) AG_FAIL(AG_ERR_INVALID, "arith_spans: NULL span table");
  return arith_binary_spans_dev(type, op, shape, spans, n_spans, resolve_stream(s));
}
ag_status ag_arith_unary_same_dev(int type, int8_t op, const void* in, void* out, int64_t n, ag_stream_t s) {
  AG_TRY(ensure_init());
  return arith_unary_same_dev(type, op, in, out, n, resolve_stream(s));
}
ag_status ag_arith_unary_diff_dev(int itype, int otype, int8_t op, const void* in, void* out, int64_t n, ag_stream_t s) {
  AG_TRY(ensure_init());
  return arith_unary_diff_dev(itype, otype, op, in, out, n, resolve_stream(s));
}
ag_status ag_arith_checked_dev(int type, int8_t op, int shape, const void* l, const uint8_t* lvalid, int64_t loff,
                               const void* r, const uint8_t* rvalid, int64_t roff,
                               void* out, int64_t n, int64_t* d_first_bad, ag_stream_t s) {
  AG_TRY(ensure_init());
  if (!d_first_bad) AG_FAIL(AG_ERR_INVALID, "arith_checked: NULL error word");
  return arith_checked_dev(type, op, shape, l, lvalid, loff, r, rvalid, roff, out, n, d_first_bad, resolve_stream(s));
}
ag_status ag_arith_unary_checked_dev(int type, int8_t op, const void* in, void* out, int64_t n, int64_t* d_first_bad, ag_stream_t s) {
  AG_TRY(ensure_init());
  if (!d_first_bad) AG_FAIL(AG_ERR_INVALID, "arith_unary_checked: NULL error word");
  return arith_unary_checked_dev(type, op, in, out, n, d_first_bad, resolve_stream(s));
}
ag_status ag_error_word_reset_dev(int64_t* d_word, ag_stream_t s) {
  AG_TRY(ensure_init());
  return error_word_reset(d_word, resolve_stream(s));
}

}  // extern "C"
