// reduce.cu — arrow/math Sum on sm_90a.
//
// Replaces sum_{float64,int64,uint64}_{avx2,sse4,neon} (arrow/math/_lib/float64.c:20-26,
// int64.c:21-27, uint64.c; Go entry Float64Funcs.Sum arrow/math/float64.go:34-39).
// Validity bitmaps are ignored, exactly like the reference (it sums values[offset:offset+len]).
//
// Roofline: HBM.  8 algorithmic bytes per row, ~0.125 flop/byte.
//
// float64: every accumulator is a (sum, error) pair updated with Knuth's TwoSum (6 dependent-free flops per element,
// far below what the FP64 pipe can do while the kernel waits on HBM), and partial results are merged the same way.
// With the errors summed in floating point this is Ogita, Rump and Oishi's Sum2: |res - S| <= 2 eps |S| +
// gamma_n^2 sum|x| (eps = 2^-53, gamma_n = n eps / (1 - n eps); the 2 covers the final rounding of s + c).  So the
// result is within 1 ULP of the exactly rounded sum while gamma_n^2 sum|x| is small against eps |S| — 0 ULP from
// math.fsum at 100M N(0,1) rows (tests/test_gpu_sum.py), where the reference's own three association orders (AVX2 /
// SSE4 / pure Go, SURVEY §3.4) sit tens to hundreds of ULP apart — and can be many ULP off on badly conditioned data.
// Whenever every partial sum is exact (the reference's tests, integer-valued data) the result is bit-identical to the
// reference in any order.  Non-finite inputs: any NaN, or +inf and -inf together, give NaN; infinities or an overflow
// of one sign give that infinity.  Unspecified, as in the reference's AVX2 order: finite inputs whose partial sums
// overflow with both signs may give NaN, and then the class may differ from the reference's.  tests/sum_f64_ref.py
// models this kernel's association bit for bit, so a change to the order below changes that model with it.
// ag_sum_f64_reforder reproduces the AVX2 order bit for bit on any input.  Integers wrap (any order is exact).
//
// Shape of the reduction (fixed => the float64 result is a pure function of (data, n)):
//   * the input is viewed as PAIRS (x[2j], x[2j+1]); an odd last element is folded in at the end;
//   * G = sum_grid(n) blocks of 256 threads (at most 132 x 8, a constant); block b streams the
//     contiguous 2048-pair (32 KB) tiles b, b+G, ...; in a tile thread t owns pairs t, t+256, ...
//     with 8 pair-loads in flight, load k feeding accumulator pair k % 4 (8 chains per thread);
//   * thread sum -> warp xor-shuffle tree -> block tree (fixed) -> partials[G];
//   * the last block to finish (ticket) reduces partials[] with the same fixed tree.
// 16-byte aligned inputs use 128-bit ld.global.cs; 8-byte aligned ones use two 64-bit loads
// with the SAME pair->thread mapping, so alignment never changes the result.
#include "host_stage.cuh"

#include <type_traits>


namespace ag {

constexpr int kSumThreads = 256;
constexpr int kSumLoads = 8;                                  // 16-byte pair loads in flight per thread
constexpr int kSumAcc = 4;                                    // accumulator pairs per thread (slot = load % 4)
constexpr int kSumTilePairs = kSumThreads * kSumLoads;        // 2048 pairs = 32 KB per block iteration
constexpr int kSumBlocksPerSM = 8;
constexpr int kSumSMs = 132;                                  // H100 SXM
constexpr int kSumMaxBlocks = kSumSMs * kSumBlocksPerSM;      // fixed (not queried): the result must not depend on the device

// float64 keeps (sum, error) pairs: 64 registers per thread, 4 resident blocks per SM -> its one-wave grid is 132 x 4
template <typename T> constexpr int sum_blocks_per_sm() { return std::is_floating_point<T>::value ? 4 : kSumBlocksPerSM; }

template <typename T>
static inline int sum_grid(size_t n_pairs) {
  // small inputs get few blocks (latency), big ones the fixed one-wave grid
  size_t want = (n_pairs + kSumTilePairs - 1) / kSumTilePairs;
  if (want < 1) want = 1;
  static_assert(kSumMaxBlocks <= kMaxPartials, "one 16-byte partial per block");
  constexpr size_t cap = kSumSMs * sum_blocks_per_sm<T>();
  if (want > cap) want = cap;
  return (int)want;
}

template <typename T> struct Pair { T x, y; };

template <typename T, bool kAligned>
__device__ __forceinline__ Pair<T> load_pair(const T* __restrict__ in, size_t j) {
  Pair<T> p;
  if (kAligned) {
    const ulonglong2 v = __ldcs(reinterpret_cast<const ulonglong2*>(in) + j);
    p.x = *reinterpret_cast<const T*>(&v.x);
    p.y = *reinterpret_cast<const T*>(&v.y);
  } else {
    p.x = __ldcs(in + 2 * j);
    p.y = __ldcs(in + 2 * j + 1);
  }
  return p;
}

template <typename T>
__device__ __forceinline__ T shfl_xor_t(T v, int m) {
  unsigned long long u = *reinterpret_cast<unsigned long long*>(&v);
  u = __shfl_xor_sync(0xffffffffu, u, m);
  return *reinterpret_cast<T*>(&u);
}

// Accumulator: integers are a plain wrapping sum; float64 carries the rounding error of every addition (TwoSum:
// s + x = t + e exactly) in a second word.  16 bytes either way, which is the partials slot size.
template <typename T> struct Acc {
  T s;
  __device__ __forceinline__ void zero() { s = T(0); }
  __device__ __forceinline__ void add(T x) { s = s + x; }
  __device__ __forceinline__ void merge(const Acc& o) { s = s + o.s; }
  __device__ __forceinline__ Acc shfl_xor(int m) const { Acc r; r.s = shfl_xor_t(s, m); return r; }
  __device__ __forceinline__ T value() const { return s; }
  __device__ __forceinline__ ulonglong2 raw() const { return make_ulonglong2(*reinterpret_cast<const unsigned long long*>(&s), 0ull); }
  static __device__ __forceinline__ Acc from_raw(const ulonglong2 v) { Acc r; r.s = *reinterpret_cast<const T*>(&v.x); return r; }
};
template <> struct Acc<double> {
  double s, c;
  __device__ __forceinline__ void zero() { s = 0.0; c = 0.0; }
  __device__ __forceinline__ void add(double x) {
    const double t = __dadd_rn(s, x);
    const double z = __dsub_rn(t, s);
    const double e = __dadd_rn(__dsub_rn(s, __dsub_rn(t, z)), __dsub_rn(x, z));
    s = t;
    c = __dadd_rn(c, e);
  }
  __device__ __forceinline__ void merge(const Acc& o) { add(o.s); c = __dadd_rn(c, o.c); }
  __device__ __forceinline__ Acc shfl_xor(int m) const { Acc r; r.s = shfl_xor_t(s, m); r.c = shfl_xor_t(c, m); return r; }
  // s is the plain IEEE sum of its chain: once it is ±inf or NaN it stays non-finite through every later add / merge,
  // and only then can c be NaN (TwoSum's inf - inf), so a non-finite s is the result as it stands.
  __device__ __forceinline__ double value() const { return isfinite(s) ? __dadd_rn(s, c) : s; }
  __device__ __forceinline__ ulonglong2 raw() const { return make_ulonglong2((unsigned long long)__double_as_longlong(s), (unsigned long long)__double_as_longlong(c)); }
  static __device__ __forceinline__ Acc from_raw(const ulonglong2 v) { Acc r; r.s = __longlong_as_double((long long)v.x); r.c = __longlong_as_double((long long)v.y); return r; }
};

// ---- cross-GPU exchange fused into the reduction (multi-GPU global Sum, SURVEY §8e) -------------------------
// Every rank owns a MAILBOX in its HBM: 2 buffers (epoch parity) x world slots of {flag, sum, error}.  The thread that
// holds a rank's final (sum, error) pair stores it straight into slot[rank] of EVERY rank's mailbox (peer stores over
// NVLink), publishes the epoch as the flag behind a system-scope fence, then waits for the world's flags in its own
// mailbox and folds the pairs in RANK ORDER — so the collective costs one NVLink store + one poll inside the kernel
// that computed the sum: no second launch, no host synchronisation, identical bits on every rank.  A rank can be at
// most one epoch ahead of the slowest one (it cannot finish epoch e before everyone has written e), hence two buffers.
// Called by every lane of warp 0 of the block that holds the final pair (valid in lane 0).  Lane r talks to rank r:
// the world's stores, flag releases and polls are in flight together (one NVLink round trip, not `world` of them); the
// fold itself stays sequential in rank order so every rank computes the same bits.  Returns the total in every lane.
template <typename T>
__device__ __forceinline__ Acc<T> exchange_sum(Acc<T> mine, const SumExchange& x) {
  const int lane = threadIdx.x & 31;
  const int buf = (int)(x.epoch & 1ull);
  ulonglong2 me = mine.raw();
  me.x = __shfl_sync(0xffffffffu, me.x, 0);
  me.y = __shfl_sync(0xffffffffu, me.y, 0);
  Acc<T> g; g.zero();
  for (int r0 = 0; r0 < x.world; r0 += 32) {
    const int r = r0 + lane;
    if (r < x.world) {
      MailSlot* m = x.peers[r] + buf * x.world + x.rank;
      m->s = me.x;
      m->c = me.y;
      __threadfence_system();
      asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(&m->flag), "l"(x.epoch) : "memory");
    }
  }
  for (int r0 = 0; r0 < x.world; r0 += 32) {
    const int r = r0 + lane;
    ulonglong2 v = make_ulonglong2(0ull, 0ull);
    if (r < x.world) {
      MailSlot* m = x.local + buf * x.world + r;
      unsigned long long f;
      do {
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(f) : "l"(&m->flag) : "memory");
      } while (f != x.epoch);
      v.x = *reinterpret_cast<volatile unsigned long long*>(&m->s);
      v.y = *reinterpret_cast<volatile unsigned long long*>(&m->c);
    }
    const int cnt = x.world - r0 < 32 ? x.world - r0 : 32;
    for (int k = 0; k < cnt; ++k) {   // rank order
      ulonglong2 o;
      o.x = __shfl_sync(0xffffffffu, v.x, k);
      o.y = __shfl_sync(0xffffffffu, v.y, k);
      g.merge(Acc<T>::from_raw(o));
    }
  }
  return g;
}

// fixed tree over the 256 threads of a block; result valid in thread 0
template <typename T>
__device__ __forceinline__ Acc<T> block_tree_sum(Acc<T> v, Acc<T>* smem /* >= 8 */) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v.merge(v.shfl_xor(m));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  Acc<T> r; r.zero();
  if (warp == 0) {
    if (lane < kSumThreads / 32) r = smem[lane];
#pragma unroll
    for (int m = 4; m >= 1; m >>= 1) r.merge(r.shfl_xor(m));
  }
  __syncthreads();
  return r;
}

template <typename T, bool kAligned>
__global__ void __launch_bounds__(kSumThreads, std::is_floating_point<T>::value ? 4 : 5)
sum_kernel(const T* __restrict__ in, size_t n, ulonglong2* __restrict__ partials, unsigned* __restrict__ ticket,
           T* __restrict__ out, const SumExchange xch) {
  __shared__ Acc<T> smem[8];
  __shared__ bool is_last;
  const size_t n_pairs = n >> 1;
  const size_t n_tiles = (n_pairs + kSumTilePairs - 1) / kSumTilePairs;
  Acc<T> ax[kSumAcc], ay[kSumAcc];
#pragma unroll
  for (int k = 0; k < kSumAcc; ++k) { ax[k].zero(); ay[k].zero(); }
  // Block b streams the contiguous 32 KB tiles b, b+G, b+2G, ...; inside a tile thread t owns
  // pairs t, t+256, ... (8 independent 16-byte loads in flight), load k feeds accumulator k % 4.
  for (size_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const size_t j0 = tile * kSumTilePairs + threadIdx.x;
    if (j0 + (size_t)(kSumLoads - 1) * kSumThreads < n_pairs) {
      Pair<T> p[kSumLoads];
#pragma unroll
      for (int k = 0; k < kSumLoads; ++k) p[k] = load_pair<T, kAligned>(in, j0 + (size_t)k * kSumThreads);
#pragma unroll
      for (int k = 0; k < kSumLoads; ++k) { ax[k % kSumAcc].add(p[k].x); ay[k % kSumAcc].add(p[k].y); }
    } else {
#pragma unroll
      for (int k = 0; k < kSumLoads; ++k) {
        const size_t jj = j0 + (size_t)k * kSumThreads;
        if (jj < n_pairs) {
          const Pair<T> p = load_pair<T, kAligned>(in, jj);
          ax[k % kSumAcc].add(p.x); ay[k % kSumAcc].add(p.y);
        }
      }
    }
  }
  // ((x0+y0)+(x1+y1)) + ((x2+y2)+(x3+y3))
#pragma unroll
  for (int k = 0; k < kSumAcc; ++k) ax[k].merge(ay[k]);
  ax[0].merge(ax[1]); ax[2].merge(ax[3]); ax[0].merge(ax[2]);
  Acc<T> v = block_tree_sum(ax[0], smem);

  if (gridDim.x == 1) {
    if (threadIdx.x < 32) {
      if (threadIdx.x == 0 && (n & 1)) v.add(in[n - 1]);
      if (xch.world > 1) v = exchange_sum(v, xch);
      if (threadIdx.x == 0) *out = v.value();
    }
    return;
  }
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = v.raw();
    __threadfence();
    const unsigned t = atomicAdd(ticket, 1u);
    is_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // fixed-order reduction of the partials: thread t takes t, t+256, ... then the block tree
  Acc<T> acc; acc.zero();
  for (unsigned i = threadIdx.x; i < gridDim.x; i += kSumThreads) {
    acc.merge(Acc<T>::from_raw(__ldcg(partials + i)));
  }
  acc = block_tree_sum(acc, smem);
  if (threadIdx.x < 32) {
    if (threadIdx.x == 0) {
      if (n & 1) acc.add(in[n - 1]);
      *ticket = 0;  // leave the workspace ready for the next launch on this stream
    }
    if (xch.world > 1) acc = exchange_sum(acc, xch);
    if (threadIdx.x == 0) *out = acc.value();
  }
}

// Reference association order (float64_avx2_amd64.s:36-43,86-174): 32 interleaved serial
// chains over the first n&~31 elements — lane j of ONE warp owns chain j, so every load is a
// fully coalesced 256-byte row — combined as (y0+y4)+(y2+y6) + (y1+y5)+(y3+y7) per ymm lane,
// lo128+hi128, hadd, then the n&31 tail sequentially.  n < 32: purely sequential.
// Latency-bound by design (n/32 dependent DADDs); bit-exact with the reference on any input.
__global__ void __launch_bounds__(32) sum_f64_reforder_kernel(const double* __restrict__ in, size_t n, double* out) {
  const int lane = threadIdx.x;
  const size_t body = (n > 31) ? (n & ~(size_t)31) : 0;
  double acc = 0.0;
  size_t k = 0;
  // 8 independent loads in flight per lane; the adds stay in chain order
  for (; k + 8 * 32 <= body; k += 8 * 32) {
    double v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = __ldcs(in + k + u * 32 + lane);
#pragma unroll
    for (int u = 0; u < 8; ++u) acc = __dadd_rn(acc, v[u]);
  }
  for (; k < body; k += 32) acc = __dadd_rn(acc, __ldcs(in + k + lane));
  double s = 0.0;
  if (body) {
    // lane j = 4*y + q  (ymm register y, 64-bit lane q)
    // t_y = acc[y] + acc[y+4]  for y in 0..3            -> xor 16
    double t = __dadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, 16));
    // u0 = t0 + t2, u1 = t1 + t3                         -> xor 8 (valid in y<2)
    double u = __dadd_rn(t, __shfl_xor_sync(0xffffffffu, t, 8));
    // v = u0 + u1                                         -> xor 4 (valid in y==0, lanes q=0..3)
    double v = __dadd_rn(u, __shfl_xor_sync(0xffffffffu, u, 4));
    // w0 = v[0]+v[2], w1 = v[1]+v[3]                      -> xor 2
    double w = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 2));
    // hadd: w0 + w1                                       -> xor 1
    s = __dadd_rn(w, __shfl_xor_sync(0xffffffffu, w, 1));
  }
  if (lane == 0) {
    for (size_t i = body; i < n; ++i) s = __dadd_rn(s, in[i]);
    *out = s;
  }
}

// n == 0 with an exchange: the rank still has to take part, with a zero pair
__global__ void sum_exchange_only_kernel(unsigned long long* out, const SumExchange xch, int is_f64) {   // <<<1, 32>>>
  if (is_f64) { Acc<double> z; z.zero(); z = exchange_sum(z, xch); if (threadIdx.x == 0) *reinterpret_cast<double*>(out) = z.value(); }
  else { Acc<unsigned long long> z; z.zero(); z = exchange_sum(z, xch); if (threadIdx.x == 0) *out = z.value(); }
}

template <typename T>
ag_status launch_sum(const T* d_in, size_t n, T* d_res, cudaStream_t st, const SumExchange* xch) {
  SumExchange x{};
  x.world = 1;
  if (xch) x = *xch;
  if (n == 0) {
    if (x.world > 1) {
      sum_exchange_only_kernel<<<1, 32, 0, st>>>(reinterpret_cast<unsigned long long*>(d_res), x, std::is_floating_point<T>::value ? 1 : 0);
      return check_launch("sum_exchange_only_kernel");
    }
    AG_CUDA_TRY(cudaMemsetAsync(d_res, 0, sizeof(T), st));
    return AG_OK;
  }
  if ((reinterpret_cast<uintptr_t>(d_in) & 7) != 0) AG_FAIL(AG_ERR_INVALID, "sum: input is not 8-byte aligned");
  Workspace* ws;
  AG_TRY(get_workspace(st, &ws));
  WorkspaceLock ws_lock(ws);
  const bool aligned = (reinterpret_cast<uintptr_t>(d_in) & 15) == 0;
  const int grid = sum_grid<T>(n >> 1);
  if (aligned)
    sum_kernel<T, true><<<grid, kSumThreads, 0, st>>>(d_in, n, (ulonglong2*)ws->partials, ws->ticket, d_res, x);
  else
    sum_kernel<T, false><<<grid, kSumThreads, 0, st>>>(d_in, n, (ulonglong2*)ws->partials, ws->ticket, d_res, x);
  return check_launch("sum_kernel");
}

// Host-pointer flavour: stage the whole column to HBM with chunked async copies (the copy is
// >100x the kernel time, so there is nothing to gain from overlapping the reduction), then run
// exactly the same kernel as the device flavour => identical bits.
template <typename T, typename F>
static ag_status host_sum(const T* buf, size_t n, T* res, F&& launch) {
  if (!res) AG_FAIL(AG_ERR_INVALID, "sum: NULL result pointer");
  AG_TRY(ensure_init());
  if (n == 0) { *res = T(0); return AG_OK; }
  if (!buf) AG_FAIL(AG_ERR_INVALID, "sum: NULL buffer");
  CallStream cs;  // a private pooled stream per call keeps concurrent host calls independent
  AG_TRY(cs.acquire());
  Temps t(cs);
  T* d_in;
  AG_TRY(t.alloc_t(&d_in, n * sizeof(T) + sizeof(T)));
  T* d_res = d_in + n;
  const size_t chunk = (size_t)8 << 20;  // elements (64 MiB)
  for (size_t off = 0; off < n; off += chunk)
    AG_TRY(h2d(d_in + off, buf + off, (n - off < chunk ? n - off : chunk) * sizeof(T), cs));
  AG_TRY(launch(d_in, n, d_res, cs));
  AG_TRY(d2h(res, d_res, sizeof(T), cs));
  return sync(cs);
}

static ag_status launch_reforder(const double* d_in, size_t n, double* d_res, cudaStream_t st) {
  if (n == 0) { AG_CUDA_TRY(cudaMemsetAsync(d_res, 0, sizeof(double), st)); return AG_OK; }
  sum_f64_reforder_kernel<<<1, 32, 0, st>>>(d_in, n, d_res);
  return check_launch("sum_f64_reforder_kernel");
}

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_sum_f64_dev(const double* d, size_t n, double* d_res, ag_stream_t s) {
  AG_TRY(ensure_init());
  return launch_sum<double>(d, n, d_res, resolve_stream(s), nullptr);
}
ag_status ag_sum_i64_dev(const int64_t* d, size_t n, int64_t* d_res, ag_stream_t s) {
  AG_TRY(ensure_init());
  // wrapping two's-complement sum == unsigned sum (int64.c:21-27)
  return launch_sum<unsigned long long>((const unsigned long long*)d, n, (unsigned long long*)d_res, resolve_stream(s), nullptr);
}
ag_status ag_sum_u64_dev(const uint64_t* d, size_t n, uint64_t* d_res, ag_stream_t s) {
  AG_TRY(ensure_init());
  return launch_sum<unsigned long long>((const unsigned long long*)d, n, (unsigned long long*)d_res, resolve_stream(s), nullptr);
}
ag_status ag_sum_f64_reforder_dev(const double* d, size_t n, double* d_res, ag_stream_t s) {
  AG_TRY(ensure_init());
  return launch_reforder(d, n, d_res, resolve_stream(s));
}

// ---- global Sum over the ranks of a communicator (comm.cu): the local reduction and the cross-GPU fold are ONE kernel
ag_status ag_sum_i64_global_dev(ag_comm_t comm, const int64_t* d, size_t n, int64_t* d_res, ag_stream_t s) {
  AG_TRY(ensure_init());
  cudaStream_t st = resolve_stream(s);
  SumExchange x;
  AG_TRY(comm_next_exchange(comm, &x));
  return launch_sum<unsigned long long>((const unsigned long long*)d, n, (unsigned long long*)d_res, st, &x);
}
ag_status ag_sum_u64_global_dev(ag_comm_t comm, const uint64_t* d, size_t n, uint64_t* d_res, ag_stream_t s) {
  return ag_sum_i64_global_dev(comm, (const int64_t*)d, n, (int64_t*)d_res, s);
}
ag_status ag_sum_f64_global_dev(ag_comm_t comm, const double* d, size_t n, double* d_res, ag_stream_t s) {
  AG_TRY(ensure_init());
  cudaStream_t st = resolve_stream(s);
  SumExchange x;
  AG_TRY(comm_next_exchange(comm, &x));
  return launch_sum<double>(d, n, d_res, st, &x);
}
// the north_star's literal form: per-GPU Sum, then ncclAllReduce of the 8-byte result on the same stream (no host sync)
ag_status ag_sum_i64_global_nccl_dev(ag_comm_t comm, const int64_t* d, size_t n, int64_t* d_res, ag_stream_t s) {
  AG_TRY(ensure_init());
  cudaStream_t st = resolve_stream(s);
  AG_TRY(launch_sum<unsigned long long>((const unsigned long long*)d, n, (unsigned long long*)d_res, st, nullptr));
  return comm_nccl_allreduce_sum_i64(comm, d_res, 1, st);
}

ag_status ag_sum_f64(const double* buf, size_t n, double* res) {
  return host_sum<double>(buf, n, res, [](const double* d, size_t m, double* r, cudaStream_t st) { return launch_sum<double>(d, m, r, st, nullptr); });
}
ag_status ag_sum_i64(const int64_t* buf, size_t n, int64_t* res) {
  return host_sum<unsigned long long>((const unsigned long long*)buf, n, (unsigned long long*)res,
      [](const unsigned long long* d, size_t m, unsigned long long* r, cudaStream_t st) { return launch_sum<unsigned long long>(d, m, r, st, nullptr); });
}
ag_status ag_sum_u64(const uint64_t* buf, size_t n, uint64_t* res) {
  return host_sum<unsigned long long>((const unsigned long long*)buf, n, (unsigned long long*)res,
      [](const unsigned long long* d, size_t m, unsigned long long* r, cudaStream_t st) { return launch_sum<unsigned long long>(d, m, r, st, nullptr); });
}
ag_status ag_sum_f64_reforder(const double* buf, size_t n, double* res) {
  return host_sum<double>(buf, n, res, [](const double* d, size_t m, double* r, cudaStream_t st) { return launch_reforder(d, m, r, st); });
}

}  // extern "C"
