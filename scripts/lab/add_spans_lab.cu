// add_spans_lab.cu — standalone copy of the chunked Add's tile loop (binary_spans_kernel<double, OpAdd, AA>, the
// all-aligned instantiation in arrow_go_b200/csrc/elementwise.cu) that stamps %globaltimer when each block starts and
// when it has finished its last tile, under two tile schedules: the grid-stride order and tiles claimed from a counter
// (the product's).  Not part of the product: scripts/add_gap.py compiles it into a temporary shared library and
// reports how far apart the blocks finish, as a share of the kernel's time.  Keep the loop in step with the product.
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr int kThreads = 256;
constexpr int kUnroll = 4;
constexpr int kTileBytes = 16384;   // kBinaryTileBytes

struct SpanDesc {
  const void* l;
  const void* r;
  void* out;
  long long n;
  long long first_tile;
};

__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

long long span_head(const void* out, long long n) {
  const long long h = (2 - (long long)((reinterpret_cast<uintptr_t>(out) & 15) / 8)) & 1;
  return h < n ? h : n;
}
__device__ __forceinline__ long long span_head_d(const void* out, long long n) {
  const long long h = (2 - (long long)((reinterpret_cast<uintptr_t>(out) & 15) / 8)) & 1;
  return h < n ? h : n;
}

constexpr int kSpans = 256;
struct SpanTable { SpanDesc s[kSpans]; };

// kClaimed: blocks claim tiles from a counter one claim ahead (the product's schedule); otherwise the grid-stride order
// tile = blockIdx.x, blockIdx.x + gridDim.x, ...
template <bool kClaimed>
__global__ void __launch_bounds__(kThreads, 3)
spans_lab_kernel(const __grid_constant__ SpanTable table, int n_spans, long long total_tiles, unsigned* __restrict__ next_tile,
                 unsigned long long* __restrict__ stamps) {
  constexpr int N = 2;
  constexpr int kTile = kTileBytes / 8;
  if (threadIdx.x == 0) stamps[2 * blockIdx.x] = globaltimer();
  __shared__ unsigned s_tile[2];
  const auto claim = [&] {
    const unsigned t = atomicAdd(next_tile, 1u);
    if (t == total_tiles + gridDim.x - 1) *next_tile = 0;
    return t;
  };
  if (threadIdx.x == 0) s_tile[0] = kClaimed ? claim() : blockIdx.x;
  __syncthreads();
  int s = 0;
  for (int k = 0;; ++k) {
    const long long tile = kClaimed ? (long long)s_tile[k & 1] : (long long)blockIdx.x + (long long)k * gridDim.x;
    if (tile >= total_tiles) break;
    if (kClaimed && threadIdx.x == 0) s_tile[(k + 1) & 1] = claim();
    while (s + 1 < n_spans && table.s[s + 1].first_tile <= tile) ++s;
    const SpanDesc sp = table.s[s];
    const long long head = span_head_d(sp.out, sp.n);
    const int t_in = (int)(tile - sp.first_tile);
    const double* l0 = reinterpret_cast<const double*>(sp.l);
    const double* r0 = reinterpret_cast<const double*>(sp.r);
    if (t_in == 0 && threadIdx.x < head) reinterpret_cast<double*>(sp.out)[threadIdx.x] = l0[threadIdx.x] + r0[threadIdx.x];
    const long long e0 = head + (long long)t_in * kTile;
    const long long rest = sp.n - e0;
    const int len = (int)(rest < kTile ? (rest > 0 ? rest : 0) : kTile);
    const uint4* l = reinterpret_cast<const uint4*>(l0 + e0);
    const uint4* r = reinterpret_cast<const uint4*>(r0 + e0);
    uint4* out = reinterpret_cast<uint4*>(reinterpret_cast<double*>(sp.out) + e0);
    const int nvec = len / N;
    constexpr int kIters = kTile / N / kThreads;
#pragma unroll
    for (int b = 0; b < kIters; b += kUnroll) {
      uint4 a[kUnroll], c[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const int vi = (b + u) * kThreads + threadIdx.x;
        if (vi < nvec) { a[u] = __ldcs(l + vi); c[u] = __ldcs(r + vi); }
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const int vi = (b + u) * kThreads + threadIdx.x;
        if (vi < nvec) {
          const double2 x = *reinterpret_cast<const double2*>(&a[u]);
          const double2 y = *reinterpret_cast<const double2*>(&c[u]);
          const double2 o = make_double2(x.x + y.x, x.y + y.y);
          __stcs(out + vi, *reinterpret_cast<const uint4*>(&o));
        }
      }
    }
    const int i = nvec * N + threadIdx.x;
    if (i < len) reinterpret_cast<double*>(sp.out)[e0 + i] = l0[e0 + i] + r0[e0 + i];
    if (kClaimed) __syncthreads();
  }
  __syncthreads();
  if (threadIdx.x == 0) stamps[2 * blockIdx.x + 1] = globaltimer();
}

}  // namespace

extern "C" {

// Blocks the product would launch for `tiles` tiles: one resident wave.
int add_spans_lab_grid(long long tiles) {
  int dev = 0, sms = 0, per_sm = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, spans_lab_kernel<true>, kThreads, 0) != cudaSuccess)
    return -1;
  const long long cap = (long long)sms * per_sm;
  return (int)(tiles < cap ? tiles : cap);
}

// Runs the Add over the spans {l, r, out, n} (device pointers, float64, at most 256 spans) `reps` times with the
// grid-stride (claimed = 0) or the claimed (claimed = 1) tile schedule.  stamps: host array of reps * grid * 2
// (start, end) nanosecond values.  Returns 0, or the CUDA error code.
int add_spans_lab_run(const void* const* l, const void* const* r, void* const* out, const long long* n, int n_spans, int reps,
                      int claimed, unsigned long long* stamps) {
  if (n_spans < 1 || n_spans > kSpans) return (int)cudaErrorInvalidValue;
  SpanTable t{};
  long long tiles = 0;
  for (int i = 0; i < n_spans; ++i) {
    t.s[i] = SpanDesc{l[i], r[i], out[i], n[i], tiles};
    const long long body = n[i] - span_head(out[i], n[i]);
    const long long k = (body + kTileBytes / 8 - 1) / (kTileBytes / 8);
    tiles += k > 0 ? k : 1;
  }
  const int grid = add_spans_lab_grid(tiles);
  unsigned* counter = nullptr;
  unsigned long long* ds = nullptr;
  cudaError_t e = grid > 0 ? cudaSuccess : cudaErrorInvalidValue;
  if (e == cudaSuccess) e = cudaMalloc(&counter, sizeof(unsigned));
  if (e == cudaSuccess) e = cudaMemset(counter, 0, sizeof(unsigned));
  if (e == cudaSuccess) e = cudaMalloc(&ds, sizeof(unsigned long long) * 2 * grid);
  for (int k = 0; k < reps && e == cudaSuccess; ++k) {
    if (claimed) spans_lab_kernel<true><<<grid, kThreads>>>(t, n_spans, tiles, counter, ds);
    else spans_lab_kernel<false><<<grid, kThreads>>>(t, n_spans, tiles, counter, ds);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpy(stamps + (size_t)k * 2 * grid, ds, sizeof(unsigned long long) * 2 * grid, cudaMemcpyDeviceToHost);
  }
  cudaFree(counter);
  cudaFree(ds);
  return (int)e;
}

}  // extern "C"
