// minmax.cu — integer min/max of a column in one pass.
//
// Replaces {int,uint}{8,16,32,64}_max_min_{avx2,sse4,neon} (internal/utils/_lib/min_max.c:23-125;
// Go entry points GetMinMaxInt32 ... internal/utils/min_max.go, pure-Go loops :25-210) — the
// reduction Parquet column statistics run over every value page
// (parquet/metadata/statistics_types.gen.go:160-190,464-490).  n == 0 returns (MAX, MIN) of the
// type, the reference's initial values (min_max.c:24-25).  Order-independent => bit-exact.
//
// Roofline: HBM, sizeof(T) algorithmic bytes per row.  Same shape as sum_kernel: a one-wave grid
// of 256-thread blocks streams contiguous 32 KB tiles with 8 16-byte loads in flight per thread;
// warp shuffle tree -> block -> partials -> last block (ticket).  Inputs that are only
// element-aligned (Arrow slices) peel up to 15 bytes at the head; the vector body starts at the
// first 16-byte boundary.
#include "host_stage.cuh"

#include <string.h>
#include <limits>

namespace ag {
namespace {

constexpr int kMmThreads = 256;
constexpr int kMmLoads = 8;
constexpr int kMmAcc = 4;

template <typename T> struct MinMax { T lo, hi; };

template <typename T>
__device__ __forceinline__ void fold(MinMax<T>& m, T v) { m.lo = v < m.lo ? v : m.lo; m.hi = v > m.hi ? v : m.hi; }

template <typename T>
__device__ __forceinline__ T shfl_xor_any(T v, int mask) {
  if constexpr (sizeof(T) == 8) {
    unsigned long long u = (unsigned long long)v;
    u = __shfl_xor_sync(0xffffffffu, u, mask);
    return (T)u;
  } else {
    int u = (int)v;  // sign / zero extension round-trips through the conversion back to T
    u = __shfl_xor_sync(0xffffffffu, u, mask);
    return (T)u;
  }
}

template <typename T>
__device__ __forceinline__ MinMax<T> block_minmax(MinMax<T> m, T* s_lo, T* s_hi) {
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) {
    const T a = shfl_xor_any(m.lo, d), b = shfl_xor_any(m.hi, d);
    m.lo = a < m.lo ? a : m.lo;
    m.hi = b > m.hi ? b : m.hi;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { s_lo[warp] = m.lo; s_hi[warp] = m.hi; }
  __syncthreads();
  if (warp == 0) {
    m.lo = lane < kMmThreads / 32 ? s_lo[lane] : std::numeric_limits<T>::max();
    m.hi = lane < kMmThreads / 32 ? s_hi[lane] : std::numeric_limits<T>::lowest();
#pragma unroll
    for (int d = 4; d >= 1; d >>= 1) {
      const T a = shfl_xor_any(m.lo, d), b = shfl_xor_any(m.hi, d);
      m.lo = a < m.lo ? a : m.lo;
      m.hi = b > m.hi ? b : m.hi;
    }
  }
  __syncthreads();
  return m;  // valid in thread 0
}

template <typename T>
__global__ void __launch_bounds__(kMmThreads)
minmax_kernel(const T* __restrict__ in, size_t n, size_t head, unsigned long long* __restrict__ partials,
              unsigned* __restrict__ ticket, T* __restrict__ out) {
  constexpr int N = 16 / sizeof(T);
  constexpr int kTileVecs = kMmThreads * kMmLoads;
  __shared__ T s_lo[8], s_hi[8];
  __shared__ bool is_last;
  MinMax<T> acc[kMmAcc];  // independent chains: a 64-bit min/max is a compare + two selects deep
#pragma unroll
  for (int k = 0; k < kMmAcc; ++k) acc[k] = MinMax<T>{std::numeric_limits<T>::max(), std::numeric_limits<T>::lowest()};
  const uint4* body = reinterpret_cast<const uint4*>(in + head);  // 16-byte aligned by construction
  const size_t n_vecs = (n - head) / N;
  const size_t n_tiles = (n_vecs + kTileVecs - 1) / kTileVecs;
  for (size_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const size_t v0 = tile * kTileVecs + threadIdx.x;
    uint4 raw[kMmLoads];
    if (v0 + (size_t)(kMmLoads - 1) * kMmThreads < n_vecs) {  // full tile: no per-load predicates
#pragma unroll
      for (int k = 0; k < kMmLoads; ++k) raw[k] = __ldcs(body + v0 + (size_t)k * kMmThreads);
#pragma unroll
      for (int k = 0; k < kMmLoads; ++k) {
        const T* e = reinterpret_cast<const T*>(&raw[k]);
#pragma unroll
        for (int j = 0; j < N; ++j) fold(acc[(k * N + j) % kMmAcc], e[j]);
      }
    } else {
#pragma unroll
      for (int k = 0; k < kMmLoads; ++k) {
        const size_t vi = v0 + (size_t)k * kMmThreads;
        if (vi < n_vecs) {
          raw[k] = __ldcs(body + vi);
          const T* e = reinterpret_cast<const T*>(&raw[k]);
#pragma unroll
          for (int j = 0; j < N; ++j) fold(acc[j % kMmAcc], e[j]);
        }
      }
    }
  }
  MinMax<T> m = acc[0];
#pragma unroll
  for (int k = 1; k < kMmAcc; ++k) { m.lo = acc[k].lo < m.lo ? acc[k].lo : m.lo; m.hi = acc[k].hi > m.hi ? acc[k].hi : m.hi; }
  if (blockIdx.x == 0) {  // element-granular head (before the first 16-byte boundary) and tail
    const size_t tail0 = head + n_vecs * N;
    for (size_t i = threadIdx.x; i < head; i += kMmThreads) fold(m, in[i]);
    for (size_t i = tail0 + threadIdx.x; i < n; i += kMmThreads) fold(m, in[i]);
  }
  m = block_minmax(m, s_lo, s_hi);
  if (gridDim.x == 1) {
    if (threadIdx.x == 0) { out[0] = m.lo; out[1] = m.hi; }
    return;
  }
  if (threadIdx.x == 0) {
    partials[2 * blockIdx.x] = (unsigned long long)m.lo;
    partials[2 * blockIdx.x + 1] = (unsigned long long)m.hi;
    __threadfence();
    is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  MinMax<T> r{std::numeric_limits<T>::max(), std::numeric_limits<T>::lowest()};
  for (unsigned i = threadIdx.x; i < gridDim.x; i += kMmThreads) {
    const T a = (T)__ldcg(partials + 2 * i), b = (T)__ldcg(partials + 2 * i + 1);
    r.lo = a < r.lo ? a : r.lo;
    r.hi = b > r.hi ? b : r.hi;
  }
  r = block_minmax(r, s_lo, s_hi);
  if (threadIdx.x == 0) { out[0] = r.lo; out[1] = r.hi; *ticket = 0; }
}

template <typename T>
__global__ void minmax_empty_kernel(T* out) { out[0] = std::numeric_limits<T>::max(); out[1] = std::numeric_limits<T>::lowest(); }

template <typename T>
ag_status launch_minmax(const void* d_in, size_t n, void* d_out, cudaStream_t st) {
  if (n == 0) {
    minmax_empty_kernel<T><<<1, 1, 0, st>>>((T*)d_out);
    return check_launch("minmax_empty_kernel");
  }
  constexpr int N = 16 / sizeof(T);
  const uintptr_t a = reinterpret_cast<uintptr_t>(d_in);
  if (a % sizeof(T)) AG_FAIL(AG_ERR_INVALID, "min_max: values pointer is not element-aligned");
  size_t head = ((16 - a % 16) % 16) / sizeof(T);
  if (head > n) head = n;
  Workspace* ws;
  AG_TRY(get_workspace(st, &ws));
  WorkspaceLock ws_lock(ws);
  const size_t n_vecs = (n - head) / N;
  size_t want = (n_vecs + (size_t)kMmThreads * kMmLoads - 1) / ((size_t)kMmThreads * kMmLoads);
  if (want < 1) want = 1;
  // exactly one wave of resident blocks (min/max is order-independent, so the grid may follow the
  // device): a fixed grid of 8 blocks per SM runs more than one wave at this kernel's 48 registers
  int grid = grid_one_wave(minmax_kernel<T>, kMmThreads, (int64_t)want);
  if (grid > kMaxPartials / 2) grid = kMaxPartials / 2;
  minmax_kernel<T><<<grid, kMmThreads, 0, st>>>((const T*)d_in, n, head, (unsigned long long*)ws->partials, ws->ticket, (T*)d_out);
  return check_launch("minmax_kernel");
}

}  // namespace

ag_status min_max_dev(int type, const void* d_in, int64_t n, void* d_out, cudaStream_t st) {
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "min_max: negative length");
  if (!d_out) AG_FAIL(AG_ERR_INVALID, "min_max: NULL output");
  if (n > 0 && !d_in) AG_FAIL(AG_ERR_INVALID, "min_max: NULL values");
  const auto not_int = [&] {
    AG_FAIL(AG_ERR_TYPE, "min_max: type id %d is not an integer type (internal/utils/min_max.go covers the 8 integer types)", type);
  };
  return visit_type(type, [&](auto tag) {
    using T = typename decltype(tag)::type;
    if constexpr (std::is_integral<T>::value) return launch_minmax<T>(d_in, (size_t)n, d_out, st);
    else return not_int();
  }, not_int);
}

}  // namespace ag

using namespace ag;

extern "C" ag_status ag_min_max_dev(int type, const void* d_values, int64_t n, void* d_min_max, ag_stream_t s) {
  AG_TRY(ensure_init());
  return min_max_dev(type, d_values, n, d_min_max, resolve_stream(s));
}

// Host flavour: stage the column (the copy is >100x the kernel), same kernel, two elements back.
extern "C" ag_status ag_min_max(int type, const void* values, int64_t n, void* min_out, void* max_out) {
  AG_TRY(ensure_init());
  const int w = type_width(type);
  if (w == 0 || type_is_float(type)) AG_FAIL(AG_ERR_TYPE, "min_max: type id %d is not an integer type", type);
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "min_max: negative length");
  if (!min_out || !max_out) AG_FAIL(AG_ERR_INVALID, "min_max: NULL result pointer");
  if (n > 0 && !values) AG_FAIL(AG_ERR_INVALID, "min_max: NULL values");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  const size_t nbytes = (size_t)n * w;
  const size_t bytes = (nbytes + 15) & ~(size_t)15;   // the two results follow the values, 16-byte aligned
  uint8_t* d_in;
  AG_TRY(t.alloc_t(&d_in, bytes + 16));
  const size_t chunk = (size_t)64 << 20;
  for (size_t off = 0; off < nbytes; off += chunk)
    AG_TRY(h2d(d_in + off, (const uint8_t*)values + off, nbytes - off < chunk ? nbytes - off : chunk, cs));
  AG_TRY(min_max_dev(type, d_in, n, d_in + bytes, cs));
  unsigned char res[16];
  AG_TRY(d2h(res, d_in + bytes, 2 * (size_t)w, cs));
  AG_TRY(sync(cs));
  memcpy(min_out, res, (size_t)w);
  memcpy(max_out, res + w, (size_t)w);
  return AG_OK;
}
