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
#include "host_stage.cuh"

#include <algorithm>
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
// Where a pass reads its (key, row) pairs:
//   kPairs       the pair buffers of the previous pass;
//   kFromSource  the column itself (no NaN / null rows: pair i is (key(vals[i]), i));
//   kFromWords   a packed key word of the multi-key sort, in row order: pair i is (words[i], i);
//   kGather      the next packed key word, through the permutation so far: pair i is (words[row_i], row_i) with row_i
//                from the pair buffers of the previous pass (an 8-byte random read per row).
// T is only used with kFromSource.
constexpr int kPairs = 0, kFromSource = 1, kFromWords = 2, kGather = 3;
template <typename T, typename K, int kMode>
__device__ __forceinline__ K pass_key(const SortSource& src, const SortXform& xf, const K* __restrict__ keys, const unsigned* __restrict__ idx,
                                      int64_t lo, int64_t i) {
  if constexpr (kMode == kFromSource) {
    int cls;
    const K k = sort_key<T, K>(__ldcs(reinterpret_cast<const T*>(src.vals) + src.voff + i), src.descending, &cls);
    return (K)((k - (K)xf.kmin) >> xf.tz);
  } else if constexpr (kMode == kGather) {
    return __ldg(keys + __ldcs(idx + lo + i));
  } else {
    return __ldcs(keys + lo + i);
  }
}

// tot[256]: per-bin totals of the pass (zeroed by the host), accumulated per block and flushed once
template <typename T, typename K, int kMode>
__global__ void __launch_bounds__(kSoThreads)
sort_digit_hist_kernel(const SortSource src, const SortXform xf, const K* __restrict__ keys, const unsigned* __restrict__ idx, int64_t lo, int64_t n,
                       int shift, unsigned* __restrict__ tile_hist, int64_t ntiles, unsigned* __restrict__ tot) {
  __shared__ unsigned s_h[kSoBins];
  unsigned acc = 0;                      // thread b < 256: rows of digit b in this block's tiles
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    if (threadIdx.x < kSoBins) s_h[threadIdx.x] = 0;
    __syncthreads();
    K kk[kSoPerThread];
#pragma unroll
    for (int e = 0; e < kSoPerThread; ++e) {      // every load of the tile in flight before the first atomic
      const int64_t i = tile * kSoTile + e * kSoThreads + threadIdx.x;
      kk[e] = i < n ? pass_key<T, K, kMode>(src, xf, keys, idx, lo, i) : (K)0;
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
template <typename T, typename K, int kMode, bool kLast>
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
        if constexpr (kMode == kGather) {
          idx[e] = __ldcs(idx_in + lo + i);
          key[e] = __ldg(keys_in + idx[e]);
        } else {
          key[e] = pass_key<T, K, kMode>(src, xf, keys_in, idx_in, lo, i);
          idx[e] = (kMode == kFromSource || kMode == kFromWords) ? (unsigned)i : __ldcs(idx_in + lo + i);
        }
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

template <typename T, typename K, int kMode>
static ag_status launch_digit_pass(const SortSource& src, const SortXform& xf, const K* keys_in, const unsigned* idx_in, int64_t lo, int64_t fn, int shift,
                                   unsigned* tile_hist, unsigned* seg_sums, unsigned* tot, K* keys_out, unsigned* idx_out, unsigned long long* out64,
                                   bool last, cudaStream_t st) {
  constexpr size_t kScatterSmem = (sizeof(K) + 4) * (size_t)kSoTile + (size_t)kSoWarps * 256 * 4;
  static std::atomic<unsigned> attr_a{0u}, attr_b{0u};   // per instantiation, one bit per device
  AG_TRY(ensure_dynamic_smem((const void*)sort_digit_scatter_kernel<T, K, kMode, false>, (int)kScatterSmem, &attr_a));
  AG_TRY(ensure_dynamic_smem((const void*)sort_digit_scatter_kernel<T, K, kMode, true>, (int)kScatterSmem, &attr_b));
  const int64_t ftiles = (fn + kSoTile - 1) / kSoTile;
  const int fgrid = grid_for(fn, kSoTile, 8);
  sort_digit_hist_kernel<T, K, kMode><<<fgrid, kSoThreads, 0, st>>>(src, xf, keys_in, idx_in, lo, fn, shift, tile_hist, ftiles, tot);
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
    sort_digit_scatter_kernel<T, K, kMode, true><<<fgrid, kSoThreads, kScatterSmem, st>>>(src, xf, keys_in, idx_in, lo, fn, shift, tile_hist, ftiles, keys_out, idx_out, out64);
  else
    sort_digit_scatter_kernel<T, K, kMode, false><<<fgrid, kSoThreads, kScatterSmem, st>>>(src, xf, keys_in, idx_in, lo, fn, shift, tile_hist, ftiles, keys_out, idx_out, out64);
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
        rc = launch_digit_pass<T, K, kFromSource>(src, xf, nullptr, nullptr, 0, fn, 0, tile_hist, d_seg, d_tot, keys[0], idx[0], d_out, last, st);
      else
        rc = launch_digit_pass<K, K, kPairs>(src, xf, keys[cur], idx[cur], fin_lo, fn, 8 * d, tile_hist, d_seg, d_tot + (size_t)d * 256, keys[cur ^ 1], idx[cur ^ 1], d_out, last, st);
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

// ================================================================ several keys over chunked columns
// The keys of a row are packed into one B-bit integer whose ascending order is the lexicographic order of the keys, and
// the digit passes above sort that integer.  Key j contributes, most significant key first, the field
//     class code (0..2 bits) | value (vbits)
// class code: the row's class among {finite, NaN, null} numbered in placement order over the classes the column holds
// (one class: no bits); value: (key' - min key') >> tz for finite rows (the transform of the single-key sort), 0 for
// NaN and null rows, so that those tie on the key and fall through to the next one.
//   P0  one launch (blockIdx.y = key): min / max / OR / AND of key' over the finite rows, NaN and null rows of every key
//       -> one read-back so the host can size the fields;
//   P1  one launch: every row's packed key, written once as W = ceil(B/64) uint64 words (one uint32 word if B <= 32);
//   P2+ the digit passes, least significant digit of word 0 first; the first pass of every later word gathers that word
//       through the permutation so far (kGather), the last pass writes the uint64 row indices.
// Rows are numbered across chunks.  Both kernels walk a span table: the row ranges inside which every key column stays
// in one chunk (cut wherever a chunk of any key ends, like IterateExecSpans); a tile of 4096 rows never crosses a span
// and blocks find their span by binary search over the spans' first tiles, so a table of many small chunks is still
// one launch per kernel.
struct SkChunk { const void* vals; const uint8_t* valid; int64_t offset; int64_t row0; };   // row0: first row of the chunk
struct SkSpan { int64_t row0; int64_t len; int64_t first_tile; };
struct SkKey {
  int type, descending;
  int cls_bits, vbits, tz;
  int code[3];                  // class code of finite / NaN / null rows
  unsigned long long kmin;
};
constexpr int kSkStats = 8;     // per key: [0] min, [1] max, [2] OR, [3] AND of key' (finite rows), [4] NaN rows, [5] null rows

// key' of element li (offset included) of a chunk; *cls = 0 finite, 1 NaN, 2 null.  BOOL: the data bit.
__device__ __forceinline__ unsigned long long sk_load(int type, const SkChunk& c, int64_t li, int descending, int* cls) {
  using U = unsigned long long;
  U k = 0;
  *cls = 0;
  switch (type) {
    case AG_TYPE_BOOL: k = (U)bit_is_set(reinterpret_cast<const uint8_t*>(c.vals), li) ^ (U)(descending != 0); break;
    case AG_TYPE_UINT8: k = sort_key<uint8_t, U>(reinterpret_cast<const uint8_t*>(c.vals)[li], descending, cls); break;
    case AG_TYPE_INT8: k = sort_key<int8_t, U>(reinterpret_cast<const int8_t*>(c.vals)[li], descending, cls); break;
    case AG_TYPE_UINT16: k = sort_key<uint16_t, U>(reinterpret_cast<const uint16_t*>(c.vals)[li], descending, cls); break;
    case AG_TYPE_INT16: k = sort_key<int16_t, U>(reinterpret_cast<const int16_t*>(c.vals)[li], descending, cls); break;
    case AG_TYPE_UINT32: k = sort_key<uint32_t, U>(reinterpret_cast<const uint32_t*>(c.vals)[li], descending, cls); break;
    case AG_TYPE_INT32: k = sort_key<int32_t, U>(reinterpret_cast<const int32_t*>(c.vals)[li], descending, cls); break;
    case AG_TYPE_UINT64: k = sort_key<U, U>(reinterpret_cast<const U*>(c.vals)[li], descending, cls); break;
    case AG_TYPE_INT64: k = sort_key<long long, U>(reinterpret_cast<const long long*>(c.vals)[li], descending, cls); break;
    case AG_TYPE_FLOAT32: k = sort_key<float, U>(reinterpret_cast<const float*>(c.vals)[li], descending, cls); break;
    default: k = sort_key<double, U>(reinterpret_cast<const double*>(c.vals)[li], descending, cls); break;
  }
  if (c.valid && !bit_is_set(c.valid, li)) *cls = 2;
  return k;
}

// the span of a tile: the last span whose first tile is <= tile
__device__ __forceinline__ int sk_span_of(const SkSpan* __restrict__ spans, int nspans, int64_t tile) {
  int lo = 0, hi = nspans - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (spans[mid].first_tile <= tile) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// P0.  span_chunk[s * nkeys + j]: the chunk (index into `chunks`) of key j over span s.
__global__ void __launch_bounds__(kSoThreads)
sort_keys_prep_kernel(const SkKey* __restrict__ keys, const SkChunk* __restrict__ chunks, const SkSpan* __restrict__ spans,
                      const int* __restrict__ span_chunk, int nspans, int nkeys, int64_t ntiles, unsigned long long* __restrict__ stats) {
  const int j = blockIdx.y;
  const int type = keys[j].type, descending = keys[j].descending;
  unsigned long long mn = ~0ull, mx = 0, vor = 0, vand = ~0ull;
  unsigned n_nan = 0, n_null = 0;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int s = sk_span_of(spans, nspans, tile);
    const SkSpan sp = spans[s];
    const SkChunk c = chunks[span_chunk[(int64_t)s * nkeys + j]];
    const int64_t r0 = sp.row0 + (tile - sp.first_tile) * kSoTile;
    const int64_t len = min((int64_t)kSoTile, sp.row0 + sp.len - r0);
    const int64_t base = c.offset + (r0 - c.row0);
#pragma unroll
    for (int e = 0; e < kSoPerThread; ++e) {
      const int64_t i = e * kSoThreads + threadIdx.x;
      if (i < len) {
        int cls;
        const unsigned long long k = sk_load(type, c, base + i, descending, &cls);
        if (cls == 0) { mn = k < mn ? k : mn; mx = k > mx ? k : mx; vor |= k; vand &= k; }
        n_nan += cls == 1;
        n_null += cls == 2;
      }
    }
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    const unsigned long long omn = __shfl_xor_sync(0xffffffffu, mn, m), omx = __shfl_xor_sync(0xffffffffu, mx, m);
    mn = omn < mn ? omn : mn; mx = omx > mx ? omx : mx;
    vor |= __shfl_xor_sync(0xffffffffu, vor, m);
    vand &= __shfl_xor_sync(0xffffffffu, vand, m);
    n_nan += __shfl_xor_sync(0xffffffffu, n_nan, m);
    n_null += __shfl_xor_sync(0xffffffffu, n_null, m);
  }
  if ((threadIdx.x & 31) == 0) {
    unsigned long long* st = stats + (int64_t)j * kSkStats;
    if (mn <= mx) {
      atomicMin(&st[0], mn);
      atomicMax(&st[1], mx);
      atomicOr(&st[2], vor);
      atomicAnd(&st[3], vand);
    }
    if (n_nan) atomicAdd(&st[4], (unsigned long long)n_nan);
    if (n_null) atomicAdd(&st[5], (unsigned long long)n_null);
  }
}

// P1.  Word w of row r is words[w * n + r]; fields are emitted from the least significant key up.
template <typename W>
__global__ void __launch_bounds__(kSoThreads, 2)
sort_keys_pack_kernel(const SkKey* __restrict__ keys, const SkChunk* __restrict__ chunks, const SkSpan* __restrict__ spans,
                      const int* __restrict__ span_chunk, int nspans, int nkeys, int64_t ntiles, int64_t n, W* __restrict__ words) {
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int s = sk_span_of(spans, nspans, tile);
    const SkSpan sp = spans[s];
    const int64_t r0 = sp.row0 + (tile - sp.first_tile) * kSoTile;
    const int64_t len = min((int64_t)kSoTile, sp.row0 + sp.len - r0);
    for (int e = 0; e < kSoPerThread; ++e) {
      const int64_t i = e * kSoThreads + threadIdx.x;
      if (i >= len) break;
      const int64_t r = r0 + i;
      unsigned long long cur = 0;
      int sh = 0;
      W* out = words + r;
      // OR `width` (<= 64) bits of v in at bit `sh` of the current word; store each word once, when it is full
      auto emit = [&](unsigned long long v, int width) {
        if (width == 0) return;
        cur |= v << sh;
        if (sh + width >= 64) {
          *out = (W)cur;
          out += n;
          cur = sh ? v >> (64 - sh) : 0ull;
          sh = sh + width - 64;
        } else {
          sh += width;
        }
      };
      for (int j = nkeys - 1; j >= 0; --j) {
        const SkKey kd = keys[j];
        if (kd.cls_bits + kd.vbits == 0) continue;
        const SkChunk c = chunks[span_chunk[(int64_t)s * nkeys + j]];
        int cls;
        const unsigned long long k = sk_load(kd.type, c, c.offset + (r - c.row0), kd.descending, &cls);
        emit(cls ? 0ull : (k - kd.kmin) >> kd.tz, kd.vbits);
        emit((unsigned long long)(cls == 0 ? kd.code[0] : cls == 1 ? kd.code[1] : kd.code[2]), kd.cls_bits);
      }
      if (sh) *out = (W)cur;
    }
  }
}

namespace {
struct SkPlan {
  std::vector<SkKey> keys;
  std::vector<SkChunk> chunks;
  std::vector<SkSpan> spans;
  std::vector<int> span_chunk;
  int64_t ntiles = 0;
};

// Chunk table and span table of the keys (host only).  Empty chunks never own a span.
static void sk_build_tables(int nkeys, const ag_sort_key* keys, int64_t n, SkPlan* p) {
  std::vector<int> base(nkeys);
  std::vector<int64_t> cuts;
  for (int j = 0; j < nkeys; ++j) {
    base[j] = (int)p->chunks.size();
    int64_t row = 0;
    for (int c = 0; c < keys[j].nchunks; ++c) {
      const ag_sort_chunk& ch = keys[j].chunks[c];
      p->chunks.push_back(SkChunk{ch.vals, ch.valid, ch.offset, row});
      row += ch.length;
      cuts.push_back(row);
    }
  }
  std::sort(cuts.begin(), cuts.end());
  cuts.erase(std::unique(cuts.begin(), cuts.end()), cuts.end());
  std::vector<int> at(nkeys, 0);   // current chunk of each key
  int64_t row0 = 0;
  for (int64_t cut : cuts) {
    if (cut <= row0) continue;
    const int64_t len = cut - row0;
    p->spans.push_back(SkSpan{row0, len, p->ntiles});
    p->ntiles += (len + kSoTile - 1) / kSoTile;
    for (int j = 0; j < nkeys; ++j) {
      while (keys[j].chunks[at[j]].length == 0 || p->chunks[base[j] + at[j]].row0 + keys[j].chunks[at[j]].length <= row0) ++at[j];
      p->span_chunk.push_back(base[j] + at[j]);
    }
    row0 = cut;
  }
  (void)n;
}

static int bit_length(unsigned long long v) { int b = 0; while (v) { ++b; v >>= 1; } return b; }
}  // namespace

// The digit passes over the packed words.  K = uint32 when the key fits 32 bits (one word), else uint64.
template <typename K>
static ag_status sk_digit_passes(const K* words, int64_t n, int bits, char* body, size_t words_bytes, unsigned* d_tot, unsigned* d_seg,
                                 unsigned long long* d_out, cudaStream_t st) {
  const size_t key_bytes = ((size_t)n * sizeof(K) + 255) & ~(size_t)255;
  const size_t idx_bytes = ((size_t)n * 4 + 255) & ~(size_t)255;
  K* keys[2] = {reinterpret_cast<K*>(body + words_bytes), reinterpret_cast<K*>(body + words_bytes + key_bytes)};
  unsigned* idx[2] = {reinterpret_cast<unsigned*>(body + words_bytes + 2 * key_bytes), reinterpret_cast<unsigned*>(body + words_bytes + 2 * key_bytes + idx_bytes)};
  unsigned* tile_hist = reinterpret_cast<unsigned*>(body + words_bytes + 2 * key_bytes + 2 * idx_bytes);
  const SortSource none{nullptr, nullptr, 0, n, 0, 0};
  const SortXform xf{0, 0};
  const int nwords = (bits + 8 * (int)sizeof(K) - 1) / (8 * (int)sizeof(K));
  int pass = 0, cur = 0;
  const int npasses = [&] { int t = 0; for (int w = 0; w < nwords; ++w) t += (std::min(bits - 64 * w, 8 * (int)sizeof(K)) + 7) / 8; return t; }();
  for (int w = 0; w < nwords; ++w) {
    const K* word = words + (size_t)w * n;
    const int nd = (std::min(bits - 64 * w, 8 * (int)sizeof(K)) + 7) / 8;
    for (int d = 0; d < nd; ++d, ++pass) {
      const bool last = pass == npasses - 1;
      unsigned* tot = d_tot + (size_t)pass * 256;
      if (pass == 0) {
        AG_TRY((launch_digit_pass<K, K, kFromWords>(none, xf, word, nullptr, 0, n, 0, tile_hist, d_seg, tot, keys[0], idx[0], d_out, last, st)));
        continue;     // the first pass writes buffer 0
      }
      if constexpr (sizeof(K) == 8) {   // a 32-bit key is one word: nothing to gather
        if (d == 0) {
          AG_TRY((launch_digit_pass<K, K, kGather>(none, xf, word, idx[cur], 0, n, 0, tile_hist, d_seg, tot, keys[cur ^ 1], idx[cur ^ 1], d_out, last, st)));
          cur ^= 1;
          continue;
        }
      }
      AG_TRY((launch_digit_pass<K, K, kPairs>(none, xf, keys[cur], idx[cur], 0, n, 8 * d, tile_hist, d_seg, tot, keys[cur ^ 1], idx[cur ^ 1], d_out, last, st)));
      cur ^= 1;
    }
  }
  return AG_OK;
}

ag_status check_chunk_list(const char* who, int j, int nchunks, const ag_sort_chunk* chunks, int64_t nrows, const char* rows_name) {
  if (nchunks < 0 || (nchunks > 0 && !chunks)) AG_FAIL(AG_ERR_INVALID, "%s %d: bad chunk list", who, j);
  int64_t rows = 0;
  for (int c = 0; c < nchunks; ++c) {
    const ag_sort_chunk& ch = chunks[c];
    if (ch.offset < 0 || ch.length < 0) AG_FAIL(AG_ERR_INVALID, "%s %d: negative chunk offset or length", who, j);
    if (ch.length > 0 && !ch.vals) AG_FAIL(AG_ERR_INVALID, "%s %d: NULL chunk values", who, j);
    rows += ch.length;
  }
  if (rows != nrows)
    AG_FAIL(AG_ERR_INVALID, "%s %d: chunk row count %lld does not match %s %lld", who, j, (long long)rows, rows_name, (long long)nrows);
  return AG_OK;
}

ag_status sort_indices_keys_check(int nkeys, const ag_sort_key* keys, int64_t n) {
  if (nkeys < 1 || !keys) AG_FAIL(AG_ERR_INVALID, "sort_indices: must provide at least one sort key");
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "sort_indices: negative length");
  for (int j = 0; j < nkeys; ++j) {
    const ag_sort_key& k = keys[j];
    if (k.order != 0 && k.order != 1) AG_FAIL(AG_ERR_INVALID, "sort_indices: sort key %d: order must be 0 (ascending) or 1 (descending)", j);
    if (k.null_placement != 0 && k.null_placement != 1) AG_FAIL(AG_ERR_INVALID, "sort_indices: sort key %d: null placement must be 0 (at end) or 1 (at start)", j);
    AG_TRY(check_chunk_list("sort_indices: sort key", j, k.nchunks, k.chunks, n, "column length"));
    if (k.type != AG_TYPE_BOOL && type_width(k.type) == 0)
      AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "sort_indices: sort key %d: unsupported type id %d (boolean and numeric columns only)", j, k.type);
  }
  if (n >= (1ll << 32)) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "sort_indices: more than 2^32-1 rows per call");
  return AG_OK;
}

ag_status sort_indices_keys_dev(int nkeys, const ag_sort_key* keys, int64_t n, uint64_t* d_out, cudaStream_t st) {
  AG_TRY(sort_indices_keys_check(nkeys, keys, n));
  if (n == 0) return AG_OK;
  if (!d_out) AG_FAIL(AG_ERR_INVALID, "sort_indices: NULL output");

  SkPlan p;
  sk_build_tables(nkeys, keys, n, &p);
  for (int j = 0; j < nkeys; ++j) {
    SkKey k{};
    k.type = keys[j].type;
    k.descending = keys[j].order;
    p.keys.push_back(k);
  }
  // head: statistics | key plans | chunks | spans | span chunks
  std::vector<unsigned long long> stats((size_t)nkeys * kSkStats, 0);
  for (int j = 0; j < nkeys; ++j) { stats[j * kSkStats + 0] = ~0ull; stats[j * kSkStats + 3] = ~0ull; }
  TableImage head(st);
  const size_t o_stats = head.add(stats), o_keys = head.add(p.keys), o_chunks = head.add(p.chunks), o_spans = head.add(p.spans),
               o_sc = head.add(p.span_chunk);
  AG_TRY(head.upload("sort key tables"));
  unsigned long long* d_stats = head.at<unsigned long long>(o_stats);
  SkKey* d_keys = head.at<SkKey>(o_keys);
  const SkChunk* d_chunks = head.at<const SkChunk>(o_chunks);
  const SkSpan* d_spans = head.at<const SkSpan>(o_spans);
  const int* d_sc = head.at<const int>(o_sc);
  const int nspans = (int)p.spans.size();
  unsigned long long* out = reinterpret_cast<unsigned long long*>(d_out);
  void* body = nullptr;
  ag_status rc = AG_OK;
  do {
    // ---- P0: statistics of every key, one read-back
    const dim3 pgrid((unsigned)grid_for(n, kSoTile, std::max(1, 8 / nkeys)), (unsigned)nkeys);
    sort_keys_prep_kernel<<<pgrid, kSoThreads, 0, st>>>(d_keys, d_chunks, d_spans, d_sc, nspans, nkeys, p.ntiles, d_stats);
    if ((rc = check_launch("sort_keys_prep_kernel")) != AG_OK) break;
    std::vector<unsigned long long> hs((size_t)nkeys * kSkStats);
    if (cudaMemcpyAsync(hs.data(), d_stats, hs.size() * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "statistics read-back", __FILE__, __LINE__); break; }
    // ---- plan: the field of every key
    int bits = 0;
    for (int j = 0; j < nkeys; ++j) {
      SkKey& k = p.keys[j];
      const unsigned long long* s = &hs[(size_t)j * kSkStats];
      const unsigned long long n_nan = s[4], n_null = s[5], n_fin = (unsigned long long)n - n_nan - n_null;
      // classes in placement order (NullsAtEnd: finite, NaN, null; NullsAtStart: null, NaN, finite), absent ones skipped
      const int order[3] = {keys[j].null_placement ? 2 : 0, 1, keys[j].null_placement ? 0 : 2};
      const unsigned long long count[3] = {n_fin, n_nan, n_null};
      int present = 0;
      for (int c : order) if (count[c]) k.code[c] = present++;
      k.cls_bits = present == 3 ? 2 : present == 2 ? 1 : 0;
      if (n_fin > 1 && s[1] > s[0]) {
        k.kmin = s[0];
        const unsigned long long varying = s[2] ^ s[3];
        while (!((varying >> k.tz) & 1ull)) ++k.tz;
        k.vbits = bit_length((s[1] - s[0]) >> k.tz);
      }
      bits += k.cls_bits + k.vbits;
    }
    if (bits == 0) {   // every row ties on every key
      sort_iota_kernel<<<grid_for(n, kSoThreads * 8, 8), kSoThreads, 0, st>>>(n, out);
      rc = check_launch("sort_iota_kernel");
      break;
    }
    if (cudaMemcpyAsync(d_keys, p.keys.data(), (size_t)nkeys * sizeof(SkKey), cudaMemcpyHostToDevice, st) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "sort key plans", __FILE__, __LINE__); break; }
    // body: totals of every pass | segment sums | packed words | pairs x2 | indices x2 | tile histograms
    const bool narrow = bits <= 32;
    const size_t kw = narrow ? 4 : 8;
    const int nwords = narrow ? 1 : (bits + 63) / 64;
    const int npasses_max = nwords * 8;
    const size_t tot_bytes = ((size_t)npasses_max * 256 * 4 + 255) & ~(size_t)255;
    const size_t seg_bytes = ((size_t)2 * sm_count() * 256 * 4 + 255) & ~(size_t)255;
    const size_t words_bytes = ((size_t)nwords * n * kw + 255) & ~(size_t)255;
    const size_t pair_bytes = 2 * (((size_t)n * kw + 255) & ~(size_t)255) + 2 * (((size_t)n * 4 + 255) & ~(size_t)255);
    const int64_t ntiles = (n + kSoTile - 1) / kSoTile;
    const size_t th_bytes = (size_t)256 * ntiles * 4;
    if ((rc = dev_alloc_async(&body, tot_bytes + seg_bytes + words_bytes + pair_bytes + th_bytes, st)) != AG_OK) break;
    char* bd = reinterpret_cast<char*>(body);
    unsigned* d_tot = reinterpret_cast<unsigned*>(bd);
    unsigned* d_seg = reinterpret_cast<unsigned*>(bd + tot_bytes);
    char* wbase = bd + tot_bytes + seg_bytes;
    if (cudaMemsetAsync(d_tot, 0, tot_bytes, st) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "pass totals", __FILE__, __LINE__); break; }
    // ---- P1: pack
    const int grid = grid_for(p.ntiles * kSoTile, kSoTile, 8);
    if (narrow) sort_keys_pack_kernel<uint32_t><<<grid, kSoThreads, 0, st>>>(d_keys, d_chunks, d_spans, d_sc, nspans, nkeys, p.ntiles, n, reinterpret_cast<uint32_t*>(wbase));
    else sort_keys_pack_kernel<unsigned long long><<<grid, kSoThreads, 0, st>>>(d_keys, d_chunks, d_spans, d_sc, nspans, nkeys, p.ntiles, n, reinterpret_cast<unsigned long long*>(wbase));
    if ((rc = check_launch("sort_keys_pack_kernel")) != AG_OK) break;
    // ---- P2+: digit passes
    if (narrow) rc = sk_digit_passes<uint32_t>(reinterpret_cast<const uint32_t*>(wbase), n, bits, wbase, words_bytes, d_tot, d_seg, out, st);
    else rc = sk_digit_passes<unsigned long long>(reinterpret_cast<const unsigned long long*>(wbase), n, bits, wbase, words_bytes, d_tot, d_seg, out, st);
  } while (0);
  const ag_status frc = dev_free_async(body, st);
  return rc != AG_OK ? rc : frc;
}

}  // namespace ag

using namespace ag;

extern "C" ag_status ag_sort_indices_dev(int type, const void* d_vals, const uint8_t* d_valid, int64_t offset, int64_t n, int order,
                                         int null_placement, uint64_t* d_out, int64_t* null_count, int64_t* nan_count, ag_stream_t s) {
  AG_TRY(ensure_init());
  return sort_indices_dev(type, d_vals, d_valid, offset, n, order, null_placement, d_out, null_count, nan_count, resolve_stream(s));
}

extern "C" ag_status ag_sort_indices_keys_dev(int nkeys, const ag_sort_key* keys, int64_t n, uint64_t* d_out, ag_stream_t s) {
  AG_TRY(ensure_init());
  return sort_indices_keys_dev(nkeys, keys, n, d_out, resolve_stream(s));
}
