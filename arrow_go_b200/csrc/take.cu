// take.cu — gather (Take) on sm_90a.
//
// Replaces PrimitiveTake (arrow/compute/internal/kernels/vector_selection.go:1162-1192) =
// checkIndexBounds (kernels/helpers.go:929-981) + primitiveTakeImpl (:878-988):
//     out[i]       = values[idx[i]]                         for slots valid in idx and in values
//     out_valid[i] = idxValid[i] ∧ valuesValid[idx[i]]
//     other slots keep the allocator's zero (we write 0)
// Indices of width 1/2/4/8 bytes are reinterpreted as unsigned after the bounds check
// (:1147-1159); only VALID index slots are bounds-checked (helpers.go:942); the error names the
// first offender in row order (:944-955) — here: atomicMin over the offending rows.
//
// Two shapes, same results:
//
//  * direct (take_kernel): one pass, bounds check fused, 4 independent gathers in flight per thread.
//    Right whenever the gathers already have locality: values table that fits L2, small calls, and
//    sorted / reverse-sorted / clustered indices — the inputs the reference special-cases by 32-point
//    sampling (vector_selection.go:897-911); here a 1024-point probe kernel decides on the device.
//
//  * windowed (take_partition_kernel -> take_window_gather_kernel -> take_unpermute_kernel), for random
//    indices into a table much larger than L2.  A random 8-byte read costs a whole DRAM line, whatever the number
//    of loads in flight, while the same gather from an L2-resident table is bound by L2 sector requests,
//    one per gathered row.  So:
//      A  partition each 8192-row tile of the indices by table window (8 MB of values): tile-local
//         counting sort in shared memory -> window-local indices in bucket order (4 B/row), the
//         position of every row in that order (2 B/row) and the per-tile bucket offsets;
//      B  sweep the windows in order: blocks draw chunks (window, 32..256 consecutive tiles) from a
//         global counter, so at any moment the whole grid gathers from about three neighbouring
//         windows (24 MB, half of H100's 50 MB L2) that stay in L2; the runs of a chunk are walked as one concatenated sequence, so
//         every lane works whatever the run length; gathered values land in `out` in bucket order;
//      C  un-permute every tile of `out` in place through shared memory (and emit the validity words).
//    DRAM traffic ≈ 4+4+2 (A) + 4+8+8·(table rows / n) (B) + 8+2+8 (C) ≈ 48 B/row at table rows = n,
//    against 20 B/row algorithmic.
//
// Roofline: HBM.  Algorithmic 4 + 8 + 8 = 20 B/row for int64 values and int32 indices.
//
// Direct layout: a block iteration covers 1024 consecutive rows; thread t handles rows t, t+256,
// t+512, t+768 so index loads and output stores are coalesced.  A warp's rows in one step are 32
// consecutive rows starting at a multiple of 32, so the output validity word is one __ballot_sync.
#include "common.cuh"

#include <atomic>

namespace ag {

constexpr int kTkThreads = 256;
constexpr int kTkUnroll = 4;

struct TakeParams {
  const void* vals;       // element 0 of the values buffer
  const uint8_t* vvalid;
  int64_t voff;
  unsigned long long vlen;
  const void* idx;
  const uint8_t* ivalid;
  int64_t ioff;
  int64_t n;
  int idx_signed;
  int bounds_check;
  void* out;
  uint32_t* out_valid;    // 4-byte aligned, offset 0 (may be NULL)
  long long* bad_pos;     // lowered with atomicMin (may be NULL when !bounds_check)
  const int* route;       // device word written by take_probe_kernel (NULL: unconditional)
};

constexpr int kRouteDirect = 1;
constexpr int kRouteWindowed = 2;

template <typename V, typename I>
__global__ void __launch_bounds__(kTkThreads)
take_kernel(const TakeParams p) {
  const V* __restrict__ vals = reinterpret_cast<const V*>(p.vals) + p.voff;
  const I* __restrict__ idx = reinterpret_cast<const I*>(p.idx);
  V* __restrict__ out = reinterpret_cast<V*>(p.out);
  const int lane = threadIdx.x & 31;
  const int64_t step = (int64_t)gridDim.x * kTkThreads * kTkUnroll;
  long long my_bad = AG_NO_ERROR_POS;
  if (p.route && *p.route != kRouteDirect) return;
  for (int64_t base = (int64_t)blockIdx.x * kTkThreads * kTkUnroll; base < p.n; base += step) {
    I ix[kTkUnroll];
    bool ok[kTkUnroll];
#pragma unroll
    for (int k = 0; k < kTkUnroll; ++k) {
      const int64_t i = base + k * kTkThreads + threadIdx.x;
      ok[k] = i < p.n;
      ix[k] = 0;
      if (ok[k]) {
        ix[k] = __ldcs(idx + i);
        if (p.ivalid) ok[k] = bit_is_set(p.ivalid, p.ioff + i);
      }
    }
    V v[kTkUnroll];
#pragma unroll
    for (int k = 0; k < kTkUnroll; ++k) {
      v[k] = V(0);
      if (ok[k]) {
        if (take_index_oob(ix[k], p.vlen, p.idx_signed)) {
          ok[k] = false;  // never dereference; with bounds_check the whole call fails anyway
          if (p.bounds_check) {
            const long long i = base + k * kTkThreads + threadIdx.x;
            if (i < my_bad) my_bad = i;
          }
        } else {
          if (p.vvalid) ok[k] = bit_is_set(p.vvalid, p.voff + (int64_t)ix[k]);
          if (ok[k]) v[k] = vals[ix[k]];
        }
      }
    }
#pragma unroll
    for (int k = 0; k < kTkUnroll; ++k) {
      const int64_t i = base + k * kTkThreads + threadIdx.x;
      if (i < p.n) __stcs(out + i, v[k]);
      if (p.out_valid) {
        const int64_t w = (base + k * kTkThreads + (threadIdx.x & ~31)) >> 5;  // warp-uniform
        store_valid_word(p.out_valid, w, __ballot_sync(0xffffffffu, ok[k]), p.n, lane);
      }
    }
  }
  if (p.bounds_check) lower_error_row(my_bad, p.bad_pos);
}

// booleanTakeImpl (vector_selection.go:990-1074): out bit i = values bit [voff + idx[i]]; same
// validity and bounds rules.  A warp's 32 rows of one step form one output word (ballot).
template <typename I>
__global__ void __launch_bounds__(kTkThreads)
take_bool_kernel(const TakeParams p) {
  const uint8_t* __restrict__ vals = reinterpret_cast<const uint8_t*>(p.vals);
  const I* __restrict__ idx = reinterpret_cast<const I*>(p.idx);
  uint32_t* __restrict__ out = reinterpret_cast<uint32_t*>(p.out);
  const int lane = threadIdx.x & 31;
  const int64_t step = (int64_t)gridDim.x * kTkThreads;
  long long my_bad = AG_NO_ERROR_POS;
  for (int64_t base = (int64_t)blockIdx.x * kTkThreads; base < p.n; base += step) {
    const int64_t i = base + threadIdx.x;
    bool ok = i < p.n, bit = false;
    if (ok) {
      const I ix = idx[i];
      if (p.ivalid) ok = bit_is_set(p.ivalid, p.ioff + i);
      if (ok) {
        if (take_index_oob(ix, p.vlen, p.idx_signed)) {
          ok = false;
          if (p.bounds_check && (long long)i < my_bad) my_bad = (long long)i;
        } else {
          if (p.vvalid) ok = bit_is_set(p.vvalid, p.voff + (int64_t)ix);
          if (ok) bit = bit_is_set(vals, p.voff + (int64_t)ix);
        }
      }
    }
    const int64_t w = (base + (threadIdx.x & ~31)) >> 5;
    const uint32_t dbits = __ballot_sync(0xffffffffu, bit);
    const uint32_t vbits = __ballot_sync(0xffffffffu, ok);
    store_bool_words(out, p.out_valid, w, dbits, vbits, p.n, lane);
  }
  if (p.bounds_check) lower_error_row(my_bad, p.bad_pos);
}

static ag_status launch_take_bool(int idx_width, const TakeParams& p, cudaStream_t st) {
  const int64_t need = (p.n + kTkThreads - 1) / kTkThreads;
  return visit_width(idx_width, [&](auto tag) {
    const auto kernel = take_bool_kernel<typename decltype(tag)::type>;
    kernel<<<grid_one_wave(kernel, kTkThreads, need), kTkThreads, 0, st>>>(p);
    return check_launch("take_bool_kernel");
  }, [&] { AG_FAIL(AG_ERR_INDEX, "take: invalid indices byte width"); });
}

template <typename V>
static ag_status launch_take_v(int idx_width, const TakeParams& p, cudaStream_t st) {
  const int64_t need = (p.n + kTkThreads * kTkUnroll - 1) / (kTkThreads * kTkUnroll);
  return visit_width(idx_width, [&](auto tag) {
    const auto kernel = take_kernel<V, typename decltype(tag)::type>;
    kernel<<<grid_one_wave(kernel, kTkThreads, need), kTkThreads, 0, st>>>(p);
    return check_launch("take_kernel");
  }, [&] { AG_FAIL(AG_ERR_INDEX, "take: invalid indices byte width"); });  // vector_selection.go:1157
}


// =================================================================== windowed take
constexpr int kWinTile = 8192;        // rows per tile: positions fit 13 bits, one tile of int64 = 64 KB of shared memory
constexpr int kWinMaxBuckets = 1022;  // + the no-gather bucket + the end slot = 1024 shared-memory counters
constexpr int kWinAThreads = 512;
constexpr int kWinBThreads = 256;

struct TakeWindowPlan {
  int shift;        // log2(rows per window)
  int nb;           // table windows
  int nslots;       // nb + 2: bucket nb holds rows that gather nothing (null / out-of-range index), slot nb+1 = tile length
  int64_t ntiles;
  int64_t tpad;     // ntiles rounded up to 256 (every chunk size divides it)
  int ct;           // tiles per chunk of pass B
  int bgrid;        // blocks of pass B
};

// Routing probe: 1024 evenly spaced adjacent index pairs.  When most of them already point into the same few cache
// lines (sorted, reverse-sorted, clustered, or constant indices) the direct kernel streams the table at full speed
// and the windowed path would only add traffic.  The reference makes the same decision on the host by sampling 32
// points (vector_selection.go:897-911); the choice never changes a result.
template <typename I>
__global__ void __launch_bounds__(1024) take_probe_kernel(const I* __restrict__ idx, int64_t n, int near_rows, int* route) {
  const int64_t stride = (n - 1) / 1024;
  const int64_t i = (int64_t)threadIdx.x * stride;
  bool near = false;
  if (i + 1 < n) {
    const I a = idx[i], b = idx[i + 1];
    const I d = a > b ? (I)(a - b) : (I)(b - a);   // unsigned distance; a negative signed index just looks far away
    near = d <= (I)near_rows;
  }
  const int cnt = __syncthreads_count(near);
  if (threadIdx.x == 0) *route = cnt >= 768 ? kRouteDirect : kRouteWindowed;
}

// Pass A.  One tile per block iteration: load 8192 indices (coalesced), count them per table window with shared
// memory atomics (the returned old value is the row's rank inside its bucket), exclusive-scan the <= 1024 counters,
// scatter window-local indices into bucket order in shared memory, write them out coalesced.  The bounds check of
// checkIndexBounds is fused here (valid slots only).
struct PartitionShared {
  uint32_t hist[kWinMaxBuckets + 2];
  alignas(16) uint32_t sorted[kWinTile];
  uint32_t wsum[kWinAThreads / 32];
};

// One tile.  kFull: 8192 rows and a 16-byte aligned index pointer -> no per-row range tests, 128-bit loads.
// All per-row arithmetic is 32-bit: lim32 = min(limit, 2^32 - 1) (a 64-bit index is first tested against the 64-bit
// limit and then narrowed, since a row that passes is < 2^32 only when the table is; otherwise the window-local index
// and the bucket come from the 64-bit value).
template <typename I, bool kValid, bool kFull>
__device__ __forceinline__ void partition_tile(const TakeParams& p, const TakeWindowPlan& w, PartitionShared& sh, const I* __restrict__ idx,
                                               int64_t tile, unsigned long long limit, uint32_t* __restrict__ sorted, uint16_t* __restrict__ perm,
                                               uint16_t* __restrict__ off, uint32_t& bad_local) {
  constexpr int QUADS = kWinTile / (4 * kWinAThreads);
  constexpr int SPER = (kWinMaxBuckets + 2 + kWinAThreads - 1) / kWinAThreads;
  const int lane = threadIdx.x & 31;
  const int64_t base = tile * kWinTile;
  const int len = kFull ? kWinTile : (int)min((int64_t)kWinTile, p.n - base);
  const uint32_t nb = (uint32_t)w.nb;
  const int shift = w.shift;
  const bool all_fit = limit > 0xffffffffull;                 // every 32-bit index is in range
  const uint32_t lim32 = all_fit ? 0xffffffffu : (uint32_t)limit;
  for (int b = threadIdx.x; b < w.nslots; b += kWinAThreads) sh.hist[b] = 0;
  __syncthreads();
  I ix[QUADS][4];
  uint32_t bk[QUADS][4];   // bucket << 13 | rank within the bucket  (bucket <= 1023: 10 bits)
#pragma unroll
  for (int q = 0; q < QUADS; ++q) {
    const int r0 = q * (4 * kWinAThreads) + 4 * threadIdx.x;
    if (kFull) {
      const I* src = idx + base + r0;
      if constexpr (sizeof(I) == 4) {
        const uint4 v = __ldcs(reinterpret_cast<const uint4*>(src));
        ix[q][0] = v.x; ix[q][1] = v.y; ix[q][2] = v.z; ix[q][3] = v.w;
      } else {
        const ulonglong2 v0 = __ldcs(reinterpret_cast<const ulonglong2*>(src));
        const ulonglong2 v1 = __ldcs(reinterpret_cast<const ulonglong2*>(src) + 1);
        ix[q][0] = v0.x; ix[q][1] = v0.y; ix[q][2] = v1.x; ix[q][3] = v1.y;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) ix[q][j] = r0 + j < len ? idx[base + r0 + j] : (I)0;
    }
  }
#pragma unroll
  for (int q = 0; q < QUADS; ++q) {
    const int r0 = q * (4 * kWinAThreads) + 4 * threadIdx.x;
    uint32_t vbits = 0xfu;
    if (kValid) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if ((!kFull && r0 + j >= len) || !bit_is_set(p.ivalid, p.ioff + base + r0 + j)) vbits &= ~(1u << j);
    } else if (!kFull) {
#pragma unroll
      for (int j = 0; j < 4; ++j) if (r0 + j >= len) vbits &= ~(1u << j);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bool live = (!kValid && kFull) ? true : (bool)((vbits >> j) & 1u);   // row exists and its index slot is valid
      bool oob;
      uint32_t b;
      if constexpr (sizeof(I) == 4) {
        oob = (uint32_t)ix[q][j] >= lim32 && !all_fit;        // one 32-bit compare
        b = shift < 32 ? (uint32_t)ix[q][j] >> shift : 0u;
      } else {
        oob = (unsigned long long)ix[q][j] >= limit;
        b = (uint32_t)((unsigned long long)ix[q][j] >> shift);
      }
      if (live && oob) bad_local = min(bad_local, (uint32_t)(r0 + j));
      if (!live || oob) b = nb;
      bk[q][j] = 0;
      if (kFull || r0 + j < len) bk[q][j] = (b << 13) | atomicAdd(&sh.hist[b], 1u);
    }
  }
  __syncthreads();
  {
    uint32_t loc[SPER];
    uint32_t s = 0;
#pragma unroll
    for (int j = 0; j < SPER; ++j) {
      const int b = threadIdx.x * SPER + j;
      loc[j] = b < w.nslots ? sh.hist[b] : 0u;
      s += loc[j];
    }
    uint32_t inc = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t o = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += o;
    }
    if (lane == 31) sh.wsum[threadIdx.x >> 5] = inc;
    __syncthreads();
    uint32_t wbase = 0;
    for (int q = 0; q < (threadIdx.x >> 5); ++q) wbase += sh.wsum[q];
    uint32_t run = wbase + inc - s;
#pragma unroll
    for (int j = 0; j < SPER; ++j) {
      const int b = threadIdx.x * SPER + j;
      if (b < w.nslots) sh.hist[b] = run;
      run += loc[j];
    }
  }
  __syncthreads();
  for (int b = threadIdx.x; b < w.nslots; b += kWinAThreads) off[tile * w.nslots + b] = (uint16_t)sh.hist[b];
  const uint32_t wmask32 = shift < 32 ? ((1u << shift) - 1u) : 0xffffffffu;
#pragma unroll
  for (int q = 0; q < QUADS; ++q) {
    const int r0 = q * (4 * kWinAThreads) + 4 * threadIdx.x;
    uint32_t pos[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      pos[j] = 0;
      if (kFull || r0 + j < len) {
        pos[j] = sh.hist[bk[q][j] >> 13] + (bk[q][j] & 8191u);
        sh.sorted[pos[j]] = (uint32_t)ix[q][j] & wmask32;    // low 32 bits hold the whole window-local index (shift <= 32)
      }
    }
    if (kFull || r0 + 4 <= len) {
      *reinterpret_cast<uint2*>(perm + base + r0) = make_uint2(pos[0] | (pos[1] << 16), pos[2] | (pos[3] << 16));
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) if (r0 + j < len) perm[base + r0 + j] = (uint16_t)pos[j];
    }
  }
  __syncthreads();
  {
    const int nv = len >> 2;
    uint4* dst = reinterpret_cast<uint4*>(sorted + base);        // scratch: 256-byte aligned, base is a multiple of 8192
    const uint4* src = reinterpret_cast<const uint4*>(sh.sorted);
    for (int i = threadIdx.x; i < nv; i += kWinAThreads) dst[i] = src[i];
    const int r = (nv << 2) + threadIdx.x;
    if (!kFull && r < len) sorted[base + r] = sh.sorted[r];
  }
  __syncthreads();
}

template <typename I, bool kValid>
__global__ void __launch_bounds__(kWinAThreads, 2)
take_partition_kernel(const TakeParams p, const TakeWindowPlan w, uint32_t* __restrict__ sorted, uint16_t* __restrict__ perm,
                      uint16_t* __restrict__ off) {
  // thread t owns rows 4t..4t+3 of each 2048-row quarter of the tile: 128-bit index loads, 64-bit perm stores
  __shared__ PartitionShared sh;
  if (*p.route != kRouteWindowed) return;
  const I* __restrict__ idx = reinterpret_cast<const I*>(p.idx);
  // one unsigned compare does the whole bounds check: a negative signed index is >= 2^(bits-1) as unsigned
  unsigned long long limit = p.vlen;
  if (p.idx_signed && sizeof(I) < 8 && limit > (1ull << (sizeof(I) * 8 - 1))) limit = 1ull << (sizeof(I) * 8 - 1);
  if (p.idx_signed && sizeof(I) == 8 && limit > (1ull << 63)) limit = 1ull << 63;
  const bool vec_ok = (reinterpret_cast<uintptr_t>(idx) & 15) == 0;
  long long my_bad = AG_NO_ERROR_POS;
  for (int64_t tile = blockIdx.x; tile < w.ntiles; tile += gridDim.x) {
    uint32_t bad_local = 0xffffffffu;
    const bool full = vec_ok && (tile + 1) * (int64_t)kWinTile <= p.n;
    if (full) partition_tile<I, kValid, true>(p, w, sh, idx, tile, limit, sorted, perm, off, bad_local);
    else partition_tile<I, kValid, false>(p, w, sh, idx, tile, limit, sorted, perm, off, bad_local);
    if (bad_local != 0xffffffffu && tile * kWinTile + bad_local < my_bad) my_bad = tile * kWinTile + bad_local;
  }
  if (p.bounds_check) lower_error_row(my_bad, p.bad_pos);
}

// off[tile][slot] -> offT[slot][tile] (pass A writes one contiguous row per tile, pass B reads one contiguous run of
// tiles per bucket); tiles in [ntiles, tpad) read as empty.
__global__ void take_offsets_transpose_kernel(const uint16_t* __restrict__ off, uint16_t* __restrict__ offT, int64_t ntiles, int nslots,
                                              int64_t tpad, const int* route) {
  __shared__ uint16_t t[32][33];
  if (*route != kRouteWindowed) return;
  const int64_t t0 = (int64_t)blockIdx.x * 32;
  const int s0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int64_t tt = t0 + j;
    const int ss = s0 + threadIdx.x;
    t[j][threadIdx.x] = (tt < ntiles && ss < nslots) ? off[tt * nslots + ss] : (uint16_t)0;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int ss = s0 + j;
    const int64_t tt = t0 + threadIdx.x;
    if (ss < nslots && tt < tpad) offT[(int64_t)ss * tpad + tt] = tt < ntiles ? t[threadIdx.x][j] : (uint16_t)0;
  }
}

// Pass B.  Chunk = (window b, CT consecutive tiles).  Chunks are claimed in (b, tile) order from one global counter
// (next claim issued a chunk ahead), so the in-flight chunks are a contiguous range of that order: the grid works
// inside a few neighbouring windows at any moment.  Thread t < CT loads the run [off[b][tile], off[b+1][tile]) of its
// tile; a block scan turns the CT run lengths into one concatenated element space, which the block walks 4 x 256
// elements at a time (binary search for the first run, then forward).
template <typename V, int CT>
__global__ void __launch_bounds__(kWinBThreads)
take_window_gather_kernel(const TakeParams p, const TakeWindowPlan w, const uint32_t* __restrict__ sorted,
                          const uint16_t* __restrict__ offT, unsigned long long* counter) {
  static_assert(CT <= kWinBThreads, "one run descriptor per thread");
  __shared__ uint32_t s_start[CT + 1];
  __shared__ long long s_src[CT];
  __shared__ uint32_t s_w[kWinBThreads / 32];
  __shared__ unsigned long long s_claim[2];
  if (*p.route != kRouteWindowed) return;
  const V* __restrict__ vals = reinterpret_cast<const V*>(p.vals) + p.voff;
  V* __restrict__ gathered = reinterpret_cast<V*>(p.out);
  const int lane = threadIdx.x & 31;
  const int64_t cpb = w.tpad / CT;
  const int64_t nchunks = cpb * w.nb;
  if (threadIdx.x == 0) s_claim[0] = atomicAdd(counter, 1ull);
  __syncthreads();
  for (int it = 0;; ++it) {
    const int64_t chunk = (int64_t)s_claim[it & 1];
    if (chunk >= nchunks) break;
    if (threadIdx.x == 0) s_claim[(it + 1) & 1] = atomicAdd(counter, 1ull);
    const int64_t b = chunk / cpb;
    const int64_t t0 = (chunk - b * cpb) * CT;
    uint32_t len = 0, o0 = 0;
    if (threadIdx.x < CT) {
      o0 = offT[b * w.tpad + t0 + threadIdx.x];
      len = (uint32_t)offT[(b + 1) * w.tpad + t0 + threadIdx.x] - o0;
    }
    uint32_t inc = len;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t o = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += o;
    }
    if (lane == 31) s_w[threadIdx.x >> 5] = inc;
    __syncthreads();
    uint32_t wbase = 0;
    for (int q = 0; q < (threadIdx.x >> 5); ++q) wbase += s_w[q];
    const uint32_t start = wbase + inc - len;
    if (threadIdx.x < CT) {
      s_start[threadIdx.x] = start;
      s_src[threadIdx.x] = (long long)(t0 + threadIdx.x) * kWinTile + o0 - start;
      if (threadIdx.x == CT - 1) s_start[CT] = start + len;
    }
    __syncthreads();
    const uint32_t total = s_start[CT];
    const V* __restrict__ win = vals + ((unsigned long long)b << w.shift);
    int r = 0;
    {
      int lo = 0, hi = CT;  // largest r with s_start[r] <= threadIdx.x
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (s_start[mid] <= threadIdx.x) lo = mid; else hi = mid;
      }
      r = lo;
    }
    for (uint32_t e = threadIdx.x; e < total; e += 4 * kWinBThreads) {
      long long a[4];
      uint32_t l[4];
      bool h[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t ee = e + k * kWinBThreads;
        h[k] = ee < total;
        if (h[k]) {
          while (s_start[r + 1] <= ee) ++r;
          a[k] = s_src[r] + ee;
          l[k] = __ldcs(sorted + a[k]);       // streamed once: evict first, the window lines should stay
        }
      }
      V v[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) if (h[k]) v[k] = win[l[k]];
#pragma unroll
      for (int k = 0; k < 4; ++k) if (h[k]) __stcs(gathered + a[k], v[k]);
    }
    __syncthreads();
  }
}

// Pass C.  out[row] = gathered[perm[row]] inside each tile, in place (the whole tile sits in shared memory between the
// read and the write).  Rows of the no-gather bucket (position >= its start) get value 0 and validity 0.
template <typename V, int kWinCThreads, int kPerSm>
__global__ void __launch_bounds__(kWinCThreads, kPerSm)
take_unpermute_kernel(const TakeParams p, const TakeWindowPlan w, const uint16_t* __restrict__ perm, const uint16_t* __restrict__ off) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  V* s_vals = reinterpret_cast<V*>(s_raw);
  constexpr int PER = kWinTile / kWinCThreads;
  if (*p.route != kRouteWindowed) return;
  V* __restrict__ out = reinterpret_cast<V*>(p.out);
  const bool vec_ok = (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  const int lane = threadIdx.x & 31;
  for (int64_t tile = blockIdx.x; tile < w.ntiles; tile += gridDim.x) {
    const int64_t base = tile * kWinTile;
    const int len = (int)min((int64_t)kWinTile, p.n - base);
    const uint32_t null_start = off[tile * w.nslots + w.nb];
    uint16_t pm[PER];
#pragma unroll
    for (int k = 0; k < PER; ++k) {
      const int r = k * kWinCThreads + threadIdx.x;
      pm[k] = r < len ? perm[base + r] : (uint16_t)0;
    }
    if (len == kWinTile && vec_ok) {
      const uint4* src = reinterpret_cast<const uint4*>(out + base);
      uint4* dst = reinterpret_cast<uint4*>(s_raw);
      for (int i = threadIdx.x; i < (int)(kWinTile * sizeof(V) / 16); i += kWinCThreads) dst[i] = __ldcs(src + i);
    } else {
      for (int r = threadIdx.x; r < len; r += kWinCThreads) s_vals[r] = out[base + r];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < PER; ++k) {
      const int r = k * kWinCThreads + threadIdx.x;
      const bool ok = r < len && pm[k] < null_start;
      if (r < len) __stcs(out + base + r, ok ? s_vals[pm[k]] : V(0));
      if (p.out_valid) {
        const uint32_t bits = __ballot_sync(0xffffffffu, ok);
        const int64_t wd = (base + k * kWinCThreads + (threadIdx.x & ~31)) >> 5;
        const int64_t rem = p.n - (wd << 5);
        if (lane == 0 && rem > 0) {
          if (rem >= 32) p.out_valid[wd] = bits;
          else bitmap_store32_masked(p.out_valid + wd, bits, bit_range_mask(0, (int)rem));
        }
      }
    }
    __syncthreads();
  }
}

// ---- routing policy -------------------------------------------------------------------------------------------
// mode 0 = automatic, 1 = always direct, 2 = windowed whenever the shapes allow it (tests).  Automatic: the table must
// be well beyond what L2 keeps (so random gathers really go to DRAM), the call large enough that the window sweep
// amortises (pass B needs a few thousand tiles to keep a whole grid inside two or three windows), and there must be
// at least one gathered row per 8 table rows (below that most DRAM lines are touched once either way).
// Windows are at least `window_bytes` (8 MB: three of them in pass B's 24 MB) and, in automatic mode, large enough that
// there are at most kWinAutoBuckets of them: the per-tile bucket offsets grow with windows x tiles.  On an H100 (100M
// random int32 indices into 100M int64 rows / 1B into 1B): 8 MB windows 2.27 / 36.7 ms, 16 MB 2.89 / 32.7 ms, 32 MB
// 3.20 / 32.6 ms; the rule picks 8 MB and 32 MB.  No other sizes were swept.
static constexpr unsigned long long kWinAutoBuckets = 256;
static std::atomic<int> g_take_mode{0};
static std::atomic<long long> g_take_min_rows{32ll << 20};
static std::atomic<long long> g_take_min_table_bytes{160ll << 20};
static std::atomic<long long> g_take_window_bytes{8ll << 20};

static bool plan_windowed(int bit_width, int idx_width, const TakeParams& p, TakeWindowPlan* w) {
  const int mode = g_take_mode.load(std::memory_order_relaxed);
  if (mode == 1) return false;
  if (bit_width != 8 && bit_width != 16 && bit_width != 32 && bit_width != 64) return false;
  if (idx_width != 32 && idx_width != 64) return false;
  if (p.vvalid) return false;                      // values validity is a second random read: direct path
  if (p.n < 2 || p.n >= (1ll << 40) || p.vlen < 2 || p.vlen >= (1ull << 48)) return false;
  const int wbytes = bit_width / 8;
  if (mode == 0) {
    if (p.n < g_take_min_rows.load(std::memory_order_relaxed)) return false;
    if ((long long)p.vlen * wbytes < g_take_min_table_bytes.load(std::memory_order_relaxed)) return false;
    if ((unsigned long long)p.n * 8 < p.vlen) return false;
  }
  const long long window = g_take_window_bytes.load(std::memory_order_relaxed);
  int shift = 4;
  while (((long long)wbytes << shift) < window && shift < 31) ++shift;
  unsigned long long nb = (p.vlen + (1ull << shift) - 1) >> shift;
  while (mode == 0 && nb > kWinAutoBuckets && shift < 32) { ++shift; nb = (p.vlen + (1ull << shift) - 1) >> shift; }
  while (nb > (unsigned long long)kWinMaxBuckets && shift < 32) { ++shift; nb = (p.vlen + (1ull << shift) - 1) >> shift; }
  if (nb > (unsigned long long)kWinMaxBuckets) return false;
  w->shift = shift;
  w->nb = (int)nb;
  w->nslots = w->nb + 2;
  w->ntiles = (p.n + kWinTile - 1) / kWinTile;
  w->tpad = (w->ntiles + 255) / 256 * 256;
  // in-flight footprint of pass B = (blocks x tiles per chunk / tiles) windows; keep it within ~24 MB, half of H100's L2
  const double windows_in_l2 = (double)(24ll << 20) / (double)((long long)wbytes << shift);
  const int full_grid = sm_count() * 8;
  double ct = windows_in_l2 * (double)w->ntiles / (double)full_grid;
  int c = 32;
  while (c < 256 && c * 1.5 < ct) c *= 2;
  w->ct = c;
  const double cpb = (double)w->tpad / c;
  long long g = (long long)(windows_in_l2 * cpb);
  if (g < sm_count()) g = sm_count();
  if (g > full_grid) g = full_grid;
  w->bgrid = (int)g;
  return true;
}

template <typename V>
static ag_status launch_window_gather(const TakeParams& p, const TakeWindowPlan& w, const uint32_t* sorted, const uint16_t* offT,
                                      unsigned long long* counter, cudaStream_t st) {
  switch (w.ct) {
    case 32: take_window_gather_kernel<V, 32><<<w.bgrid, kWinBThreads, 0, st>>>(p, w, sorted, offT, counter); break;
    case 64: take_window_gather_kernel<V, 64><<<w.bgrid, kWinBThreads, 0, st>>>(p, w, sorted, offT, counter); break;
    case 128: take_window_gather_kernel<V, 128><<<w.bgrid, kWinBThreads, 0, st>>>(p, w, sorted, offT, counter); break;
    default: take_window_gather_kernel<V, 256><<<w.bgrid, kWinBThreads, 0, st>>>(p, w, sorted, offT, counter); break;
  }
  return check_launch("take_window_gather_kernel");
}

template <typename V>
static ag_status launch_unpermute(const TakeParams& p, const TakeWindowPlan& w, const uint16_t* perm, const uint16_t* off, cudaStream_t st) {
  // 3 blocks x 512 threads per SM: a tile is 64 KB of shared memory whatever the block size, and three tiles in flight
  // overlap one block's load phase with another's store phase better than two
  static std::atomic<unsigned> attr_set{0u};  // one bit per device
  const int smem = kWinTile * (int)sizeof(V);
  AG_TRY(ensure_dynamic_smem((const void*)take_unpermute_kernel<V, 512, 3>, smem, &attr_set));
  const int64_t cap = (int64_t)sm_count() * 3;
  take_unpermute_kernel<V, 512, 3><<<(int)(w.ntiles < cap ? w.ntiles : cap), 512, smem, st>>>(p, w, perm, off);
  return check_launch("take_unpermute_kernel");
}

// probe -> direct kernel (runs only when the probe says so) -> A, transpose, B, C (run only otherwise).  Everything is
// stream-ordered; the host never waits.
template <typename V>
static ag_status take_windowed(int idx_width, TakeParams p, const TakeWindowPlan& w, cudaStream_t st) {
  void* scratch = nullptr;
  const size_t sorted_bytes = ((size_t)p.n * 4 + 255) & ~(size_t)255;
  const size_t perm_bytes = ((size_t)p.n * 2 + 255) & ~(size_t)255;
  const size_t off_bytes = ((size_t)w.nslots * (size_t)w.tpad * 2 + 255) & ~(size_t)255;
  AG_TRY(dev_alloc_async(&scratch, 256 + sorted_bytes + perm_bytes + 2 * off_bytes, st));
  char* base = reinterpret_cast<char*>(scratch);
  int* route = reinterpret_cast<int*>(base);
  unsigned long long* counter = reinterpret_cast<unsigned long long*>(base + 64);
  uint32_t* sorted = reinterpret_cast<uint32_t*>(base + 256);
  uint16_t* perm = reinterpret_cast<uint16_t*>(base + 256 + sorted_bytes);
  uint16_t* off = reinterpret_cast<uint16_t*>(base + 256 + sorted_bytes + perm_bytes);
  uint16_t* offT = reinterpret_cast<uint16_t*>(base + 256 + sorted_bytes + perm_bytes + off_bytes);
  ag_status rc = AG_OK;
  do {
    if (cudaMemsetAsync(base, 0, 256, st) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "cudaMemsetAsync", __FILE__, __LINE__); break; }
    const int near_rows = 256 / (int)sizeof(V);    // adjacent indices within two cache lines of each other
    if (g_take_mode.load(std::memory_order_relaxed) == 2) {
      const int forced = kRouteWindowed;
      if (cudaMemcpyAsync(route, &forced, sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "cudaMemcpyAsync", __FILE__, __LINE__); break; }
    } else if (idx_width == 32) {
      take_probe_kernel<uint32_t><<<1, 1024, 0, st>>>(reinterpret_cast<const uint32_t*>(p.idx), p.n, near_rows, route);
      if ((rc = check_launch("take_probe_kernel")) != AG_OK) break;
    } else {
      take_probe_kernel<unsigned long long><<<1, 1024, 0, st>>>(reinterpret_cast<const unsigned long long*>(p.idx), p.n, near_rows, route);
      if ((rc = check_launch("take_probe_kernel")) != AG_OK) break;
    }
    p.route = route;
    if ((rc = launch_take_v<V>(idx_width, p, st)) != AG_OK) break;
    const int64_t acap = (int64_t)sm_count() * 2;
    const int agrid = (int)(w.ntiles < acap ? w.ntiles : acap);
    if (idx_width == 32) {
      if (p.ivalid) take_partition_kernel<uint32_t, true><<<agrid, kWinAThreads, 0, st>>>(p, w, sorted, perm, off);
      else take_partition_kernel<uint32_t, false><<<agrid, kWinAThreads, 0, st>>>(p, w, sorted, perm, off);
    } else {
      if (p.ivalid) take_partition_kernel<unsigned long long, true><<<agrid, kWinAThreads, 0, st>>>(p, w, sorted, perm, off);
      else take_partition_kernel<unsigned long long, false><<<agrid, kWinAThreads, 0, st>>>(p, w, sorted, perm, off);
    }
    if ((rc = check_launch("take_partition_kernel")) != AG_OK) break;
    const dim3 tg((unsigned)(w.tpad / 32), (unsigned)((w.nslots + 31) / 32));
    take_offsets_transpose_kernel<<<tg, dim3(32, 8), 0, st>>>(off, offT, w.ntiles, w.nslots, w.tpad, route);
    if ((rc = check_launch("take_offsets_transpose_kernel")) != AG_OK) break;
    if ((rc = launch_window_gather<V>(p, w, sorted, offT, counter, st)) != AG_OK) break;
    if ((rc = launch_unpermute<V>(p, w, perm, off, st)) != AG_OK) break;
  } while (0);
  const ag_status frc = dev_free_async(scratch, st);
  return rc != AG_OK ? rc : frc;
}

ag_status take_primitive_dev(int bit_width, const void* vals, const uint8_t* vvalid, int64_t voff, int64_t vlen,
                             int idx_width, int idx_signed, const void* idx, const uint8_t* ivalid, int64_t ioff,
                             int64_t n, int bounds_check, void* out, uint8_t* out_valid, int64_t* d_bad_pos, cudaStream_t st) {
  if (n < 0 || voff < 0 || ioff < 0 || vlen < 0) AG_FAIL(AG_ERR_INVALID, "take: negative length or offset");
  if (n == 0) return AG_OK;
  if (!idx || !out) AG_FAIL(AG_ERR_INVALID, "take: NULL indices/output");
  if (!vals && vlen > 0) AG_FAIL(AG_ERR_INVALID, "take: NULL values");
  if (bounds_check && !d_bad_pos) AG_FAIL(AG_ERR_INVALID, "take: bounds_check needs an error word");
  if (out_valid && (reinterpret_cast<uintptr_t>(out_valid) & 3)) AG_FAIL(AG_ERR_INVALID, "take: out_valid must be 4-byte aligned");
  if ((vvalid || ivalid) && !out_valid)
    AG_FAIL(AG_ERR_INVALID, "take: inputs may have nulls but no output validity buffer was given (vector_selection.go:1175)");
  TakeParams p{};
  p.vals = vals; p.vvalid = vvalid; p.voff = voff; p.vlen = (unsigned long long)vlen;
  p.idx = idx; p.ivalid = ivalid; p.ioff = ioff; p.n = n;
  p.idx_signed = idx_signed; p.bounds_check = bounds_check;
  p.out = out; p.out_valid = reinterpret_cast<uint32_t*>(out_valid); p.bad_pos = reinterpret_cast<long long*>(d_bad_pos);
  TakeWindowPlan w;
  if (plan_windowed(bit_width, idx_width, p, &w)) {
    // plan_windowed admits 8/16/32/64-bit values only; anything else would run as 64-bit
    return visit_width(bit_width, [&](auto tag) { return take_windowed<typename decltype(tag)::type>(idx_width, p, w, st); },
                       [&] { return take_windowed<unsigned long long>(idx_width, p, w, st); });
  }
  if (bit_width == 1) {
    if (reinterpret_cast<uintptr_t>(out) & 3) AG_FAIL(AG_ERR_INVALID, "take: boolean output bitmap must be 4-byte aligned");
    return launch_take_bool(idx_width, p, st);
  }
  return visit_width(bit_width, [&](auto tag) { return launch_take_v<typename decltype(tag)::type>(idx_width, p, st); },
                     [&] { AG_FAIL(AG_ERR_INVALID, "take: invalid values byte width for take"); });  // vector_selection.go:1190
}

}  // namespace ag

using namespace ag;

extern "C" ag_status ag_take_primitive_dev(int bit_width, const void* vals, const uint8_t* vvalid, int64_t voff, int64_t vlen,
                                           int idx_width, int idx_signed, const void* idx, const uint8_t* ivalid, int64_t ioff,
                                           int64_t n, int bounds_check, void* out, uint8_t* out_valid,
                                           int64_t* d_bad_pos, ag_stream_t s) {
  AG_TRY(ensure_init());
  return take_primitive_dev(bit_width, vals, vvalid, voff, vlen, idx_width, idx_signed, idx, ivalid, ioff, n,
                            bounds_check, out, out_valid, d_bad_pos, resolve_stream(s));
}

extern "C" ag_status ag_take_set_policy(int mode, int64_t min_rows, int64_t min_table_bytes, int64_t window_bytes) {
  if (mode < 0 || mode > 2) AG_FAIL(AG_ERR_INVALID, "ag_take_set_policy: mode must be 0 (auto), 1 (direct) or 2 (windowed)");
  g_take_mode.store(mode);
  if (min_rows > 0) g_take_min_rows.store(min_rows);
  if (min_table_bytes > 0) g_take_min_table_bytes.store(min_table_bytes);
  if (window_bytes >= 4096) g_take_window_bytes.store(window_bytes);
  return AG_OK;
}
