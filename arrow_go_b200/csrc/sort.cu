// sort.cu — sort_indices for one fixed-width column on sm_90a (SURVEY §8f rank 3).
//
// Replaces kernels.SortIndices for a single key (arrow/compute/internal/kernels/vector_sort.go:385-481,
// arraySortOneColumnRange vector_sort_internal.go:250-300): a STABLE permutation of 0..n-1 laid out as
//     NullsAtEnd   : [ finite values in key order | NaNs in row order | nulls in row order ]
//     NullsAtStart : [ nulls in row order | NaNs in row order | finite values in key order ]
// (partitionNullsOnly + partitionNullLikes, vector_sort_internal.go:36-150, then a stable sort of the finite range
// with compareOrdered: ascending or descending, ties keep row order, -0.0 == +0.0; vector_sort_physical.go,
// vector_sort_support.go:100-170).  Output: uint64 row indices, like the reference.
//
// Algorithm: least-significant-digit radix sort over (key, row) pairs, 8-bit digits.
//   key' is an order-preserving unsigned image of the value (sign bias for signed ints; floats: 2^(w-1) +- magnitude,
//   which folds -0.0 onto +0.0 and keeps trailing zero bits on both sides of zero), complemented for Descending so that
//   an ascending stable sort of key' gives the descending order with ties still in row order.  The sorted key is
//       key = (key' - min key') >> tz,   tz = trailing bits on which every finite key' agrees,
//   still order preserving, and only ceil(bits(max - min) - tz) / 8) digits can differ: a column of small integers
//   (whatever their sign), or of doubles holding integers, needs one to four passes instead of eight.
//   K0  one pass over the column: min / max / OR of differences of key' over the finite rows + NaN and null counts
//       -> read back (40 bytes) so the host can lay out the three regions and pick the digits;
//   K1  class pass, only when the column has NaNs or nulls: stable 3-way partition of the rows into the region order
//       above, materialising the pairs (a column without them feeds the first digit pass straight from the source);
//   K2+ one pass per digit on the finite region: tile histogram (shared-memory atomics, [tile][bin]) -> scan over the
//       tiles (segment sums, then each segment rescans itself) -> scatter with a stable in-tile rank (digit groups from
//       one ballot per bit + per-warp digit counters, tile staged in shared memory); the last pass writes the uint64
//       row indices straight into `out`.
// Roofline: HBM; per digit pass 8 (histogram read) + 12 + 12 bytes/row for 64-bit keys (first pass from the source:
// 8 + 8 + 12; last pass: 8 + 12 + 8); the gathers are never random (pairs move with their rows).  The API is synchronous
// in one spot: the 40-byte read-back after K0.
#include "common.cuh"

#include <string.h>
#include <type_traits>
#include <vector>

namespace ag {

constexpr int kSoThreads = 512;
constexpr int kSoPerThread = 8;
constexpr int kSoTile = kSoThreads * kSoPerThread;   // 4096 rows per tile
constexpr int kSoWarps = kSoThreads / 32;
constexpr int kSoWarpRows = kSoTile / kSoWarps;      // 256 consecutive rows per warp
constexpr int kSoBins = 256;

struct SortSource {
  const void* vals;        // element 0 of the values buffer
  const uint8_t* valid;    // validity bitmap (may be NULL)
  int64_t voff;            // element offset of the slice (values and bitmap)
  int64_t n;
  int descending;
  int nulls_first;
};

// order-preserving unsigned image of a value; *cls = 0 finite, 1 NaN
template <typename T, typename K>
__device__ __forceinline__ K sort_key(T v, int descending, int* cls) {
  K k;
  *cls = 0;
  if constexpr (std::is_same<T, float>::value) {
    // sign-magnitude -> offset binary: 2^31 +- magnitude.  Unlike the usual "flip all bits of the negatives" image this
    // keeps the trailing zero bits of the magnitude on both sides of zero (a float column holding small integers then
    // loses its constant low digits to the `tz` shift whatever the signs), and -0.0 lands on +0.0 by itself
    // (compareOrdered: -0.0 == +0.0).
    const uint32_t b = __float_as_uint(v), mag = b & 0x7fffffffu;
    if (mag > 0x7f800000u) *cls = 1;
    k = (K)((b & 0x80000000u) ? (0x80000000u - mag) : (0x80000000u | mag));
  } else if constexpr (std::is_same<T, double>::value) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(v), mag = b & 0x7fffffffffffffffull;
    if (mag > 0x7ff0000000000000ull) *cls = 1;
    k = (K)((b >> 63) ? (0x8000000000000000ull - mag) : (0x8000000000000000ull | mag));
  } else if constexpr (std::is_signed<T>::value) {
    using U = typename std::make_unsigned<T>::type;
    k = (K)(U)((U)v ^ (U)((U)1 << (sizeof(T) * 8 - 1)));
  } else {
    k = (K)v;
  }
  if (descending) {
    // complement inside the value's own width so narrower types keep their zero high bits
    if constexpr (sizeof(T) < sizeof(K)) k = (K)(~k & (((K)1 << (sizeof(T) * 8)) - 1));
    else k = (K)~k;
  }
  return k;
}

// region index of a row class under the null placement: the class pass sorts by this "digit"
__device__ __forceinline__ int class_digit(int cls /*0 finite,1 NaN,2 null*/, int nulls_first) { return nulls_first ? 2 - cls : cls; }

// key = (key' - kmin) >> tz
struct SortXform { unsigned long long kmin; int tz; };

// ---------------------------------------------------------------- K0: statistics of key'
// stats: [0] min, [1] max, [2] OR of (key' ^ key' of row 0) over the FINITE rows; [3] NaN rows, [4] null rows.
// (Row 0 as the reference even when it is not finite: a bit then merely looks varying, which costs a pass, not a result.)
template <typename T, typename K>
__global__ void __launch_bounds__(kSoThreads)
sort_prep_kernel(const SortSource src, unsigned long long* __restrict__ stats) {
  const T* __restrict__ vals = reinterpret_cast<const T*>(src.vals) + src.voff;
  int c0;
  const K ref = sort_key<T, K>(vals[0], src.descending, &c0);
  K mn = (K)~(K)0, mx = 0, vr = 0;
  unsigned n_nan = 0, n_null = 0;
  const int64_t ntiles = (src.n + kSoTile - 1) / kSoTile;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    T v[kSoPerThread];
#pragma unroll
    for (int e = 0; e < kSoPerThread; ++e) {      // 8 loads in flight per thread
      const int64_t i = tile * kSoTile + e * kSoThreads + threadIdx.x;
      v[e] = i < src.n ? __ldcs(vals + i) : T(0);
    }
#pragma unroll
    for (int e = 0; e < kSoPerThread; ++e) {
      const int64_t i = tile * kSoTile + e * kSoThreads + threadIdx.x;
      if (i < src.n) {
        int cls;
        const K k = sort_key<T, K>(v[e], src.descending, &cls);
        if (src.valid && !bit_is_set(src.valid, src.voff + i)) cls = 2;
        if (cls == 0) { mn = k < mn ? k : mn; mx = k > mx ? k : mx; vr |= k ^ ref; }
        n_nan += cls == 1;
        n_null += cls == 2;
      }
    }
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    const K omn = __shfl_xor_sync(0xffffffffu, mn, m), omx = __shfl_xor_sync(0xffffffffu, mx, m);
    mn = omn < mn ? omn : mn; mx = omx > mx ? omx : mx;
    vr |= __shfl_xor_sync(0xffffffffu, vr, m);
    n_nan += __shfl_xor_sync(0xffffffffu, n_nan, m);
    n_null += __shfl_xor_sync(0xffffffffu, n_null, m);
  }
  if ((threadIdx.x & 31) == 0) {
    if (mn <= mx) {
      atomicMin(&stats[0], (unsigned long long)mn);
      atomicMax(&stats[1], (unsigned long long)mx);
      if (vr) atomicOr(&stats[2], (unsigned long long)vr);
    }
    if (n_nan) atomicAdd(&stats[3], (unsigned long long)n_nan);
    if (n_null) atomicAdd(&stats[4], (unsigned long long)n_null);
  }
}

// ---------------------------------------------------------------- shared pieces of a pass
// class pass: tile_hist layout [bin][tile] (one contiguous row per bin, scanned by one block per bin; three bins)
__global__ void __launch_bounds__(kSoThreads)
sort_scan_bins_kernel(unsigned* __restrict__ tile_hist, int64_t ntiles, const unsigned* __restrict__ tot) {
  __shared__ unsigned long long s_w[kSoWarps];
  __shared__ unsigned long long s_base;
  // first position of this bin = rows of all lower bins (tot: per-bin totals of the pass, at most 256 of them)
  {
    unsigned long long v = (threadIdx.x < blockIdx.x) ? (unsigned long long)tot[threadIdx.x] : 0ull;   // blockIdx.x <= 255 < kSoThreads
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long b = 0;
      for (int w = 0; w < kSoWarps; ++w) b += s_w[w];
      s_base = b;
    }
    __syncthreads();
  }
  unsigned* row = tile_hist + (int64_t)blockIdx.x * ntiles;
  const int64_t per = (ntiles + kSoThreads - 1) / kSoThreads;
  const int64_t lo = (int64_t)threadIdx.x * per, hi = lo + per < ntiles ? lo + per : ntiles;
  unsigned long long sum = 0;
  for (int64_t i = lo; i < hi; ++i) sum += row[i];
  unsigned long long inc = sum;
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long o = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += o;
  }
  if (lane == 31) s_w[threadIdx.x >> 5] = inc;
  __syncthreads();
  unsigned long long base = s_base;
  for (int w = 0; w < (threadIdx.x >> 5); ++w) base += s_w[w];
  unsigned long long run = base + inc - sum;
  for (int64_t i = lo; i < hi; ++i) {
    const unsigned c = row[i];
    row[i] = (unsigned)run;     // positions fit 32 bits (n < 2^32)
    run += c;
  }
}

// Digit passes keep their tile histograms as [tile][256] (one coalesced 1 KB row per tile for the histogram kernel's
// write and the scatter's read) and scan them over the tiles in two steps: per-segment column sums, then every segment
// rescans its own tiles from (rows of lower bins) + (rows of this bin in lower segments).
constexpr int kSoSegThreads = 256;   // one thread per bin
__global__ void __launch_bounds__(kSoSegThreads)
sort_digit_segsum_kernel(const unsigned* __restrict__ th, int64_t ntiles, int64_t tiles_per_seg, unsigned* __restrict__ seg_sums) {
  const int64_t lo = (int64_t)blockIdx.x * tiles_per_seg, hi = lo + tiles_per_seg < ntiles ? lo + tiles_per_seg : ntiles;
  unsigned sum = 0;
#pragma unroll 8
  for (int64_t t = lo; t < hi; ++t) sum += th[t * 256 + threadIdx.x];
  seg_sums[(int64_t)blockIdx.x * 256 + threadIdx.x] = sum;
}

__global__ void __launch_bounds__(kSoSegThreads)
sort_digit_apply_kernel(unsigned* __restrict__ th, int64_t ntiles, int64_t tiles_per_seg, const unsigned* __restrict__ seg_sums,
                        const unsigned* __restrict__ tot) {
  __shared__ unsigned s_w[kSoSegThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // exclusive scan of the 256 bin totals: first position of this thread's bin
  const unsigned c = tot[threadIdx.x];
  unsigned inc = c;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned o = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += o;
  }
  if (lane == 31) s_w[warp] = inc;
  __syncthreads();
  unsigned run = inc - c;
  for (int w = 0; w < warp; ++w) run += s_w[w];
  // rows of this bin in the segments below
#pragma unroll 8
  for (int64_t sgm = 0; sgm < (int64_t)blockIdx.x; ++sgm) run += seg_sums[sgm * 256 + threadIdx.x];
  const int64_t lo = (int64_t)blockIdx.x * tiles_per_seg, hi = lo + tiles_per_seg < ntiles ? lo + tiles_per_seg : ntiles;
#pragma unroll 8
  for (int64_t t = lo; t < hi; ++t) {
    const unsigned k = th[t * 256 + threadIdx.x];
    th[t * 256 + threadIdx.x] = run;     // positions fit 32 bits (n < 2^32)
    run += k;
  }
}

// Stable rank of every element of a tile inside its digit: warp w owns rows [256w, 256w+256) of the tile and walks them
// 32 at a time; lanes with equal digits form a group, the group's lowest lane advances the warp's counter of that digit,
// and a lane's rank is the counter before the step plus its position inside the group.  The groups come from one ballot
// per digit bit (peers = lanes that agree with me on every bit): `match.any` does the same in one instruction but keeps the
// ADU pipe busy for tens of cycles per warp instruction and bounded the whole scatter when profiled.
// After the walk the warp counters of a digit are turned into exclusive offsets (thread b handles digit b).
// digits[e] for e = 0..7 are the digits of rows 256w + 32e + lane; rank[e] receives the rank inside (warp, digit).
// s_cnt: [kSoWarps][256] counters; on return s_cnt[w][b] = rows of digit b in warps < w, tile_count[b] in s_tot.
template <int kBits, bool kFull = false>
__device__ __forceinline__ void tile_rank(const int (&digits)[kSoPerThread], const bool (&live)[kSoPerThread], unsigned (&rank)[kSoPerThread],
                                          unsigned* s_cnt, unsigned* s_tot) {
  constexpr int nbins = 1 << kBits;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < kSoWarps * 256; i += kSoThreads) s_cnt[i] = 0;
  __syncthreads();
  unsigned* mine = s_cnt + warp * 256;
  const unsigned lt = (1u << lane) - 1u;
#pragma unroll
  for (int e = 0; e < kSoPerThread; ++e) {
    const int d = digits[e];
    // rows past the end (only the highest lanes of the last step of the last tile) join no group
    unsigned peers = kFull ? 0xffffffffu : __ballot_sync(0xffffffffu, live[e]);
#pragma unroll
    for (int b = 0; b < kBits; ++b) {
      // lanes whose bit b equals mine: and -> predicate, ballot, complement under the predicate (4 SASS instructions per
      // bit; the C++ form `bit ? m : ~m` compiled to 6)
      unsigned m;
      asm volatile("{\n"
                   "  .reg .pred p;\n"
                   "  .reg .b32 t;\n"
                   "  and.b32 t, %1, %2;\n"
                   "  setp.ne.u32 p, t, 0;\n"
                   "  vote.sync.ballot.b32 %0, p, 0xffffffff;\n"
                   "  @!p not.b32 %0, %0;\n"
                   "}\n" : "=r"(m) : "r"(d), "r"(1 << b));
      peers &= m;
    }
    unsigned old = 0;
    const int leader = __ffs(peers) - 1;
    if ((kFull || live[e]) && lane == leader) { old = mine[d]; mine[d] = old + __popc(peers); }
    old = __shfl_sync(0xffffffffu, old, leader & 31);
    rank[e] = old + __popc(peers & lt);
    __syncwarp();
  }
  __syncthreads();
  if (threadIdx.x < nbins) {
    unsigned run = 0;
#pragma unroll
    for (int w = 0; w < kSoWarps; ++w) {
      const unsigned c = s_cnt[w * 256 + threadIdx.x];
      s_cnt[w * 256 + threadIdx.x] = run;
      run += c;
    }
    s_tot[threadIdx.x] = run;
  }
  __syncthreads();
}

// ---------------------------------------------------------------- K1: class pass (source arrays -> pairs)
template <typename T, typename K>
__global__ void __launch_bounds__(kSoThreads)
sort_class_hist_kernel(const SortSource src, unsigned* __restrict__ tile_hist, int64_t ntiles) {
  __shared__ unsigned s_c[4];
  const T* __restrict__ vals = reinterpret_cast<const T*>(src.vals) + src.voff;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    if (threadIdx.x < 4) s_c[threadIdx.x] = 0;
    __syncthreads();
    unsigned c[3] = {0, 0, 0};
#pragma unroll 4
    for (int e = 0; e < kSoPerThread; ++e) {
      const int64_t i = tile * kSoTile + e * kSoThreads + threadIdx.x;
      if (i < src.n) {
        int cls;
        (void)sort_key<T, K>(vals[i], 0, &cls);
        if (src.valid && !bit_is_set(src.valid, src.voff + i)) cls = 2;
        ++c[class_digit(cls, src.nulls_first)];
      }
    }
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      unsigned v = c[b];
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
      if ((threadIdx.x & 31) == 0 && v) atomicAdd(&s_c[b], v);
    }
    __syncthreads();
    if (threadIdx.x < 3) tile_hist[(int64_t)threadIdx.x * ntiles + tile] = s_c[threadIdx.x];
    __syncthreads();
  }
}

template <typename T, typename K>
__global__ void __launch_bounds__(kSoThreads)
sort_class_scatter_kernel(const SortSource src, const SortXform xf, const unsigned* __restrict__ tile_off, int64_t ntiles, K* __restrict__ keys_out,
                          unsigned* __restrict__ idx_out) {
  __shared__ unsigned s_cnt[kSoWarps * 256];
  __shared__ unsigned s_tot[256];
  __shared__ unsigned s_base[4];
  const T* __restrict__ vals = reinterpret_cast<const T*>(src.vals) + src.voff;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    int digits[kSoPerThread];
    bool live[kSoPerThread];
    unsigned rank[kSoPerThread];
    K key[kSoPerThread];
    const int64_t row0 = tile * kSoTile + warp * kSoWarpRows + lane;
#pragma unroll
    for (int e = 0; e < kSoPerThread; ++e) {
      const int64_t i = row0 + e * 32;
      live[e] = i < src.n;
      digits[e] = 0; key[e] = 0;
      if (live[e]) {
        int cls;
        key[e] = sort_key<T, K>(__ldcs(vals + i), src.descending, &cls);
        if (src.valid && !bit_is_set(src.valid, src.voff + i)) cls = 2;
        key[e] = cls ? (K)0 : (K)((key[e] - (K)xf.kmin) >> xf.tz);
        digits[e] = class_digit(cls, src.nulls_first);
      }
    }
    if (threadIdx.x < 3) s_base[threadIdx.x] = tile_off[(int64_t)threadIdx.x * ntiles + tile];
    tile_rank<2>(digits, live, rank, s_cnt, s_tot);
#pragma unroll
    for (int e = 0; e < kSoPerThread; ++e) {
      if (live[e]) {
        const unsigned pos = s_base[digits[e]] + s_cnt[warp * 256 + digits[e]] + rank[e];
        keys_out[pos] = key[e];
        idx_out[pos] = (unsigned)(row0 + e * 32);
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- K2: digit passes
// kFromSource: the pass reads the column itself (no NaN / null rows: pair i is (key(vals[i]), i)), otherwise the pair
// buffers of the previous pass.  T is only used with kFromSource.
template <typename T, typename K, bool kFromSource>
__device__ __forceinline__ K pass_key(const SortSource& src, const SortXform& xf, const K* __restrict__ keys, int64_t lo, int64_t i) {
  if constexpr (kFromSource) {
    int cls;
    const K k = sort_key<T, K>(__ldcs(reinterpret_cast<const T*>(src.vals) + src.voff + i), src.descending, &cls);
    return (K)((k - (K)xf.kmin) >> xf.tz);
  } else {
    return __ldcs(keys + lo + i);
  }
}

// tot[256]: per-bin totals of the pass (zeroed by the host), accumulated per block and flushed once
template <typename T, typename K, bool kFromSource>
__global__ void __launch_bounds__(kSoThreads)
sort_digit_hist_kernel(const SortSource src, const SortXform xf, const K* __restrict__ keys, int64_t lo, int64_t n, int shift,
                       unsigned* __restrict__ tile_hist, int64_t ntiles, unsigned* __restrict__ tot) {
  __shared__ unsigned s_h[kSoBins];
  unsigned acc = 0;                      // thread b < 256: rows of digit b in this block's tiles
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    if (threadIdx.x < kSoBins) s_h[threadIdx.x] = 0;
    __syncthreads();
    K kk[kSoPerThread];
#pragma unroll
    for (int e = 0; e < kSoPerThread; ++e) {      // every load of the tile in flight before the first atomic
      const int64_t i = tile * kSoTile + e * kSoThreads + threadIdx.x;
      kk[e] = i < n ? pass_key<T, K, kFromSource>(src, xf, keys, lo, i) : (K)0;
    }
#pragma unroll
    for (int e = 0; e < kSoPerThread; ++e) {
      const int64_t i = tile * kSoTile + e * kSoThreads + threadIdx.x;
      if (i < n) atomicAdd(&s_h[(int)((kk[e] >> shift) & 0xff)], 1u);
    }
    __syncthreads();
    if (threadIdx.x < kSoBins) {
      const unsigned c = s_h[threadIdx.x];
      tile_hist[tile * kSoBins + threadIdx.x] = c;      // [tile][bin]
      acc += c;
    }
    __syncthreads();
  }
  if (threadIdx.x < kSoBins && acc) atomicAdd(&tot[threadIdx.x], acc);
}

// The scatter stages the tile in shared memory in digit order first (position = exclusive bin offset inside the tile +
// rows of the digit in earlier warps + rank), then walks the staged tile with consecutive threads: rows of one digit
// are consecutive there AND consecutive in the destination, so the global writes are contiguous runs issued by
// neighbouring lanes instead of 16 isolated 8-byte stores per bin.
// kLast: the final pass writes the uint64 row indices into `out64` (positions are absolute) and drops the keys.
template <typename T, typename K, bool kFromSource, bool kLast>
__global__ void __launch_bounds__(kSoThreads, 2)     // 64 registers: two 512-thread blocks per SM (71 in one variant left one)
sort_digit_scatter_kernel(const SortSource src, const SortXform xf, const K* __restrict__ keys_in, const unsigned* __restrict__ idx_in, int64_t lo,
                          int64_t n, int shift, const unsigned* __restrict__ tile_off, int64_t ntiles, K* __restrict__ keys_out,
                          unsigned* __restrict__ idx_out, unsigned long long* __restrict__ out64) {
  extern __shared__ __align__(16) unsigned char s_dyn[];
  K* s_key = reinterpret_cast<K*>(s_dyn);                                   // [kSoTile] staged keys, digit order
  unsigned* s_idx = reinterpret_cast<unsigned*>(s_dyn + sizeof(K) * kSoTile);  // [kSoTile]
  unsigned* s_cnt = s_idx + kSoTile;                                        // [kSoWarps][256]
  __shared__ unsigned s_tot[kSoBins];
  __shared__ unsigned s_excl[kSoBins];     // exclusive offset of a digit inside the staged tile
  __shared__ unsigned s_base[kSoBins];     // global position of the tile's first row of a digit, minus its staged offset
  __shared__ unsigned s_w[kSoBins / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // one tile; kFull (4096 rows) drops every per-row range test — all tiles but possibly the last
  auto do_tile = [&](int64_t tile, auto full_tag) {
    constexpr bool kFull = decltype(full_tag)::value;
    int digits[kSoPerThread];
    bool live[kSoPerThread];
    unsigned rank[kSoPerThread];
    K key[kSoPerThread];
    unsigned idx[kSoPerThread];
    const int64_t row0 = tile * kSoTile + warp * kSoWarpRows + lane;
    const int len = kFull ? kSoTile : (int)(n - tile * kSoTile);
#pragma unroll
    for (int e = 0; e < kSoPerThread; ++e) {
      const int64_t i = row0 + e * 32;
      live[e] = kFull || i < n;
      key[e] = 0; idx[e] = 0; digits[e] = 0;
      if (live[e]) {
        key[e] = pass_key<T, K, kFromSource>(src, xf, keys_in, lo, i);
        idx[e] = kFromSource ? (unsigned)i : __ldcs(idx_in + lo + i);
        digits[e] = (int)((key[e] >> shift) & 0xff);
      }
    }
    if (threadIdx.x < kSoBins) s_base[threadIdx.x] = tile_off[tile * kSoBins + threadIdx.x];     // [tile][bin]
    tile_rank<8, kFull>(digits, live, rank, s_cnt, s_tot);
    // exclusive scan of the 256 digit totals of the tile (one digit per thread of the first 8 warps)
    {
      const unsigned c = threadIdx.x < kSoBins ? s_tot[threadIdx.x] : 0u;
      unsigned inc = c;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const unsigned o = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += o;
      }
      if (lane == 31 && warp < kSoBins / 32) s_w[warp] = inc;
      __syncthreads();
      if (threadIdx.x < kSoBins) {
        unsigned wb = 0;
        for (int w = 0; w < warp; ++w) wb += s_w[w];
        s_excl[threadIdx.x] = wb + inc - c;
        s_base[threadIdx.x] -= wb + inc - c;      // destination of staged element j of this digit = s_base[d] + j (mod 2^32)
      }
    }
    __syncthreads();
#pragma unroll
    for (int e = 0; e < kSoPerThread; ++e) {
      if (live[e]) {
        const unsigned p = s_excl[digits[e]] + s_cnt[warp * 256 + digits[e]] + rank[e];
        s_key[p] = key[e];
        s_idx[p] = idx[e];
      }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < len; j += kSoThreads) {
      const K k = s_key[j];
      const int d = (int)((k >> shift) & 0xff);
      const int64_t pos = lo + (unsigned)(s_base[d] + (unsigned)j);
      if constexpr (kLast) {
        __stcs(out64 + pos, (unsigned long long)s_idx[j]);
      } else {
        keys_out[pos] = k;
        idx_out[pos] = s_idx[j];
      }
    }
    __syncthreads();
  };
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    if ((tile + 1) * (int64_t)kSoTile <= n) do_tile(tile, std::true_type());
    else do_tile(tile, std::false_type());
  }
}

__global__ void __launch_bounds__(kSoThreads)
sort_widen_kernel(const unsigned* __restrict__ idx, int64_t n, unsigned long long* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * kSoThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kSoThreads) out[i] = idx[i];
}
__global__ void __launch_bounds__(kSoThreads)
sort_iota_kernel(int64_t n, unsigned long long* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * kSoThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kSoThreads) out[i] = (unsigned long long)i;
}

template <typename T, typename K, bool kFromSource>
static ag_status launch_digit_pass(const SortSource& src, const SortXform& xf, const K* keys_in, const unsigned* idx_in, int64_t lo, int64_t fn, int shift,
                                   unsigned* tile_hist, unsigned* seg_sums, unsigned* tot, K* keys_out, unsigned* idx_out, unsigned long long* out64,
                                   bool last, cudaStream_t st) {
  constexpr size_t kScatterSmem = (sizeof(K) + 4) * (size_t)kSoTile + (size_t)kSoWarps * 256 * 4;
  static std::atomic<unsigned> attr_a{0u}, attr_b{0u};   // per instantiation, one bit per device
  AG_TRY(ensure_dynamic_smem((const void*)sort_digit_scatter_kernel<T, K, kFromSource, false>, (int)kScatterSmem, &attr_a));
  AG_TRY(ensure_dynamic_smem((const void*)sort_digit_scatter_kernel<T, K, kFromSource, true>, (int)kScatterSmem, &attr_b));
  const int64_t ftiles = (fn + kSoTile - 1) / kSoTile;
  const int fgrid = grid_for(fn, kSoTile, 8);
  sort_digit_hist_kernel<T, K, kFromSource><<<fgrid, kSoThreads, 0, st>>>(src, xf, keys_in, lo, fn, shift, tile_hist, ftiles, tot);
  AG_TRY(check_launch("sort_digit_hist_kernel"));
  int64_t nseg = 2 * (int64_t)sm_count();
  if (nseg > ftiles) nseg = ftiles;
  const int64_t tps = (ftiles + nseg - 1) / nseg;
  nseg = (ftiles + tps - 1) / tps;
  sort_digit_segsum_kernel<<<(int)nseg, kSoSegThreads, 0, st>>>(tile_hist, ftiles, tps, seg_sums);
  AG_TRY(check_launch("sort_digit_segsum_kernel"));
  sort_digit_apply_kernel<<<(int)nseg, kSoSegThreads, 0, st>>>(tile_hist, ftiles, tps, seg_sums, tot);
  AG_TRY(check_launch("sort_digit_apply_kernel"));
  if (last)
    sort_digit_scatter_kernel<T, K, kFromSource, true><<<fgrid, kSoThreads, kScatterSmem, st>>>(src, xf, keys_in, idx_in, lo, fn, shift, tile_hist, ftiles, keys_out, idx_out, out64);
  else
    sort_digit_scatter_kernel<T, K, kFromSource, false><<<fgrid, kSoThreads, kScatterSmem, st>>>(src, xf, keys_in, idx_in, lo, fn, shift, tile_hist, ftiles, keys_out, idx_out, out64);
  return check_launch("sort_digit_scatter_kernel");
}

template <typename T, typename K>
static ag_status sort_indices_t(const SortSource& src, unsigned long long* d_out, int64_t* nulls_out, int64_t* nans_out, cudaStream_t st) {
  constexpr int ND = (int)sizeof(K);
  const int64_t n = src.n;
  const int64_t ntiles = (n + kSoTile - 1) / kSoTile;
  const size_t key_bytes = ((size_t)n * sizeof(K) + 255) & ~(size_t)255;
  const size_t idx_bytes = ((size_t)n * 4 + 255) & ~(size_t)255;
  const size_t th_bytes = ((size_t)256 * ntiles * 4 + 255) & ~(size_t)255;
  const size_t seg_bytes = (size_t)2 * sm_count() * 256 * 4;
  // statistics, then one row of bin totals per pass (+ the class pass), then the per-segment column sums of a pass
  const size_t head0 = (8 * 8 + (size_t)(ND + 1) * 256 * 4 + 255) & ~(size_t)255;
  const size_t head = head0 + ((seg_bytes + 255) & ~(size_t)255);
  void* scratch = nullptr;
  AG_TRY(dev_alloc_async(&scratch, head + 2 * key_bytes + 2 * idx_bytes + th_bytes, st));
  char* base = reinterpret_cast<char*>(scratch);
  unsigned long long* d_stats = reinterpret_cast<unsigned long long*>(base);
  unsigned* d_tot = reinterpret_cast<unsigned*>(base + 64);
  unsigned* d_seg = reinterpret_cast<unsigned*>(base + head0);
  K* keys[2] = {reinterpret_cast<K*>(base + head), reinterpret_cast<K*>(base + head + key_bytes)};
  unsigned* idx[2] = {reinterpret_cast<unsigned*>(base + head + 2 * key_bytes), reinterpret_cast<unsigned*>(base + head + 2 * key_bytes + idx_bytes)};
  unsigned* tile_hist = reinterpret_cast<unsigned*>(base + head + 2 * key_bytes + 2 * idx_bytes);
  ag_status rc = AG_OK;
  do {
    unsigned long long h[8] = {~0ull, 0, 0, 0, 0, 0, 0, 0};
    if (cudaMemsetAsync(base, 0, head0, st) != cudaSuccess ||
        cudaMemcpyAsync(d_stats, h, 8, cudaMemcpyHostToDevice, st) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "statistics init", __FILE__, __LINE__); break; }
    const int grid = grid_for(n, kSoTile, 8);
    sort_prep_kernel<T, K><<<grid, kSoThreads, 0, st>>>(src, d_stats);
    if ((rc = check_launch("sort_prep_kernel")) != AG_OK) break;
    if (cudaMemcpyAsync(h, d_stats, 5 * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "statistics read-back", __FILE__, __LINE__); break; }
    const unsigned long long n_nan = h[3], n_null = h[4], n_fin = (unsigned long long)n - n_nan - n_null;
    if (nulls_out) *nulls_out = (int64_t)n_null;
    if (nans_out) *nans_out = (int64_t)n_nan;
    // the key transform and the digits that can differ
    SortXform xf{0, 0};
    int nd = 0;
    if (n_fin > 1 && h[1] > h[0]) {
      xf.kmin = h[0];
      while (xf.tz < 8 * ND - 1 && !((h[2] >> xf.tz) & 1ull)) ++xf.tz;     // h[2] != 0 here (max > min)
      unsigned long long r = (h[1] - h[0]) >> xf.tz;
      int bits = 0;
      while (r) { ++bits; r >>= 1; }
      nd = (bits + 7) / 8;
    }
    const bool classes = (n_nan + n_null) > 0;
    const int64_t fn = (int64_t)n_fin;
    const int64_t fin_lo = (int64_t)(src.nulls_first ? n_null + n_nan : 0);
    if (classes) {
      // ---- K1: class pass -> pairs in buffer 0, region layout in class-digit order
      unsigned cls_cnt[3];
      cls_cnt[src.nulls_first ? 2 : 0] = (unsigned)n_fin; cls_cnt[1] = (unsigned)n_nan; cls_cnt[src.nulls_first ? 0 : 2] = (unsigned)n_null;
      unsigned* d_cls_tot = d_tot + (size_t)ND * 256;
      if (cudaMemcpyAsync(d_cls_tot, cls_cnt, sizeof(cls_cnt), cudaMemcpyHostToDevice, st) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "class totals", __FILE__, __LINE__); break; }
      sort_class_hist_kernel<T, K><<<grid, kSoThreads, 0, st>>>(src, tile_hist, ntiles);
      if ((rc = check_launch("sort_class_hist_kernel")) != AG_OK) break;
      sort_scan_bins_kernel<<<3, kSoThreads, 0, st>>>(tile_hist, ntiles, d_cls_tot);
      if ((rc = check_launch("sort_scan_bins_kernel")) != AG_OK) break;
      sort_class_scatter_kernel<T, K><<<grid, kSoThreads, 0, st>>>(src, xf, tile_hist, ntiles, keys[0], idx[0]);
      if ((rc = check_launch("sort_class_scatter_kernel")) != AG_OK) break;
    }
    // ---- K2: digit passes over the finite region
    int cur = 0;
    for (int d = 0; d < nd; ++d) {
      const bool last = d == nd - 1;
      if (d == 0 && !classes)
        rc = launch_digit_pass<T, K, true>(src, xf, nullptr, nullptr, 0, fn, 0, tile_hist, d_seg, d_tot, keys[0], idx[0], d_out, last, st);
      else
        rc = launch_digit_pass<K, K, false>(src, xf, keys[cur], idx[cur], fin_lo, fn, 8 * d, tile_hist, d_seg, d_tot + (size_t)d * 256, keys[cur ^ 1], idx[cur ^ 1], d_out, last, st);
      if (rc != AG_OK) break;
      if (!(d == 0 && !classes)) cur ^= 1;     // a source pass writes buffer 0
    }
    if (rc != AG_OK) break;
    if (nd == 0) {
      // every finite key equal (or at most one finite row): the class order is the answer
      if (classes) sort_widen_kernel<<<grid_for(n, kSoThreads * 8, 8), kSoThreads, 0, st>>>(idx[0], n, d_out);
      else sort_iota_kernel<<<grid_for(n, kSoThreads * 8, 8), kSoThreads, 0, st>>>(n, d_out);
      rc = check_launch("sort_widen_kernel");
    } else if (classes) {
      // NaN / null rows stayed in buffer 0
      const int64_t olo = src.nulls_first ? 0 : fn, ohi = src.nulls_first ? fin_lo : n;
      sort_widen_kernel<<<grid_for(ohi - olo, kSoThreads * 8, 8), kSoThreads, 0, st>>>(idx[0] + olo, ohi - olo, d_out + olo);
      rc = check_launch("sort_widen_kernel");
    }
  } while (0);
  const ag_status frc = dev_free_async(scratch, st);
  return rc != AG_OK ? rc : frc;
}

ag_status sort_indices_dev(int type, const void* vals, const uint8_t* valid, int64_t voff, int64_t n, int order, int null_placement,
                           uint64_t* d_out, int64_t* nulls_out, int64_t* nans_out, cudaStream_t st) {
  if (n < 0 || voff < 0) AG_FAIL(AG_ERR_INVALID, "sort_indices: negative length or offset");
  if (order != 0 && order != 1) AG_FAIL(AG_ERR_INVALID, "sort_indices: order must be 0 (ascending) or 1 (descending)");
  if (null_placement != 0 && null_placement != 1) AG_FAIL(AG_ERR_INVALID, "sort_indices: null placement must be 0 (at end) or 1 (at start)");
  if (nulls_out) *nulls_out = 0;
  if (nans_out) *nans_out = 0;
  if (n == 0) return AG_OK;
  if (!vals || !d_out) AG_FAIL(AG_ERR_INVALID, "sort_indices: NULL values/output");
  if (n >= (1ll << 32)) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "sort_indices: more than 2^32-1 rows per call");
  SortSource src{vals, valid, voff, n, order, null_placement};
  unsigned long long* out = reinterpret_cast<unsigned long long*>(d_out);
  return visit_type(type, [&](auto tag) {
    using T = typename decltype(tag)::type;
    using K = typename std::conditional<sizeof(T) == 8, unsigned long long, uint32_t>::type;
    return sort_indices_t<T, K>(src, out, nulls_out, nans_out, st);
  }, [&] { AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "sort_indices: unsupported type id %d (fixed-width numeric columns only)", type); });
}

}  // namespace ag

using namespace ag;

extern "C" ag_status ag_sort_indices_dev(int type, const void* d_vals, const uint8_t* d_valid, int64_t offset, int64_t n, int order,
                                         int null_placement, uint64_t* d_out, int64_t* null_count, int64_t* nan_count, ag_stream_t s) {
  AG_TRY(ensure_init());
  return sort_indices_dev(type, d_vals, d_valid, offset, n, order, null_placement, d_out, null_count, nan_count, resolve_stream(s));
}
