// filter.cu — stream compaction (Filter, GetTakeIndices) on sm_90a.
//
// Replaces PrimitiveFilter (arrow/compute/internal/kernels/vector_selection.go:449-520) =
// getFilterOutputSize (:57-81) + primitiveFilterImpl (:267-395) + filterWriter (:397-421), and
// GetTakeIndices (:102-236).  Row rule restated from the reference's default branch
// (:321-392; the block-level fast paths :303-320 are shortcuts of it):
//     selected  = mask ∧ maskValid            -> emit value, validity = valuesValid (or 1)
//     EmitNulls ∧ ¬maskValid                  -> emit null  (value 0 :417-421, validity 0)
//     anything else                           -> dropped
// Output is stable (row order preserved), so it is bit-identical to the reference's.
//
// Roofline: HBM.  Algorithmic bytes/row for int64 at selectivity s: 8 + 1/8 + 8s.  Values are
// fetched only for emitted rows (predicated 8-byte loads; DRAM moves the touched 32-byte
// sectors), so at low selectivity the kernel can move FEWER bytes than that figure.
//
// Single pass, decoupled look-back over 32K-row BLOCK tiles:
//   * phase 1 puts the tile's 1024 mask words in shared memory (bitmap mask: coalesced word
//     loads; fused compare: the values are streamed once and __ballot_sync packs the predicate);
//   * block scan of the word popcounts -> tile aggregate published in a 64-bit status word
//     (2 flag bits + 62-bit count, one store => a reader never sees a flag without its value);
//     warp 0 resolves the tile's exclusive prefix with a two-level look-back (`lookback`, lookback.cuh): two
//     or three dependent L2 round trips whatever the number of tiles in flight;
//   * phase 2 is warp-cooperative: for each word, lane j owns row 32k+j; the lanes whose bit is
//     set load (8 words in flight per lane) and store to out[base_k + rank], rank = popc of the
//     lower set bits, so the writes of one step are contiguous.  Only the sectors of selected
//     rows are fetched;
//   * output validity bits are compacted with __reduce_or_sync and merged into pre-zeroed
//     words with at most two atomicOr per step.
#include "common.cuh"
#include "lookback.cuh"

#include <stdlib.h>
#include <type_traits>

namespace ag {

constexpr int kFThreads = 256;
constexpr int kFWarps = kFThreads / 32;
constexpr int kFTileRows = 32768;               // rows per BLOCK tile
constexpr int kFTileWords = kFTileRows / 32;    // 1024 mask words per tile
constexpr int kFWordsPerThread = kFTileWords / kFThreads;  // 4

struct FilterParams {
  const void* vals;          // element 0 of the values buffer (NULL in index mode)
  const uint8_t* vvalid;     // values validity (may be NULL)
  int64_t voff;
  const uint8_t* mask;       // NULL in fused-compare mode
  const uint8_t* mvalid;     // mask validity (may be NULL)
  int64_t moff;
  int64_t n;
  int emit_nulls;
  void* out;
  uint32_t* out_valid;       // 4-byte aligned, pre-zeroed for ceil(capacity/32) words (may be NULL)
  int64_t capacity;          // rows the output buffers can hold
  unsigned long long* status;  // one status word per tile
  unsigned long long* gstatus; // one status word per group of 32 tiles
  long long* out_len;
  int64_t n_tiles;
};

struct FCmpEq { template <typename T> static __device__ __forceinline__ bool apply(T a, T b) { return a == b; } };
struct FCmpNe { template <typename T> static __device__ __forceinline__ bool apply(T a, T b) { return a != b; } };
struct FCmpGt { template <typename T> static __device__ __forceinline__ bool apply(T a, T b) { return a > b; } };
struct FCmpGe { template <typename T> static __device__ __forceinline__ bool apply(T a, T b) { return a >= b; } };
struct FCmpLt { template <typename T> static __device__ __forceinline__ bool apply(T a, T b) { return b > a; } };
struct FCmpLe { template <typename T> static __device__ __forceinline__ bool apply(T a, T b) { return b >= a; } };

// kMode 0: copy values of type V selected by a bitmap mask.
// kMode 1: write row indices as V (GetTakeIndices).
// kMode 2: boolean VALUES: `vals` is an LSB-first bitmap (bit voff+row), `out` a pre-zeroed bitmap;
//          selected bits are compacted exactly like the validity bits (V is a dummy uint32_t).
//
// Tile assignment is STATIC (block b owns tiles b, b+G, ...): a tile only waits on lower tiles,
// every block walks its tiles in increasing order and the grid is launched cooperatively as ONE
// resident wave (cudaLaunchCooperativeKernel fails instead of deadlocking if it could not be).
//
// Schedule: a block = 8 compute warps + 1 LOOK-BACK warp; mask words double-buffered.  In iteration j the compute
// warps run phase 1 of tile j (light: 4 KB of mask, warp-local — warp w loads and counts ITS 128 words) and then
// phase 2 of tile j-1 (heavy: the gathers and stores); the last warp through phase 1 publishes the tile's
// aggregate, and the look-back warp resolves tile j's prefix while phase 2 of tile j-1 streams.  One block
// barrier per tile.  (The block-synchronous shape — all warps wait while warp 0 looks back — ran at 0.885.)
constexpr int kFiThreads = kFThreads + 32;
constexpr int kFWarpWords = kFTileWords / kFWarps;   // 128 mask words per compute warp

template <typename V, int kMode, bool kValidity>
__global__ void __launch_bounds__(kFiThreads)
filter_kernel(const FilterParams p) {
  __shared__ uint32_t s_emit_b[2][kFTileWords];
  __shared__ uint32_t s_sel_b[2][kFTileWords];
  __shared__ uint32_t s_base_b[2][kFTileWords];   // exclusive offset of each word inside its WARP's 128 words
  __shared__ uint32_t s_warp_tot_b[2][kFWarps];
  __shared__ uint32_t s_total[2];
  __shared__ unsigned long long s_tile_base_b[2];
  __shared__ unsigned s_arrived[2];
  __shared__ unsigned s_ready[2];                 // iteration number + 1 of the tile whose total is in s_total
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool looker = warp == kFWarps;
  const V* __restrict__ vals = reinterpret_cast<const V*>(p.vals) + (kMode == 0 ? p.voff : 0);
  V* __restrict__ out = reinterpret_cast<V*>(p.out);
  const uint8_t* __restrict__ bvals = reinterpret_cast<const uint8_t*>(p.vals);  // kMode 2
  uint32_t* __restrict__ bout = reinterpret_cast<uint32_t*>(p.out);             // kMode 2
  const int64_t m_lo = p.moff >> 3, m_hi = (p.moff + p.n + 7) >> 3;
  const long long cap_words = (p.capacity + 31) >> 5;
  if (threadIdx.x < 2) { s_arrived[threadIdx.x] = 0u; s_ready[threadIdx.x] = 0u; }
  __syncthreads();
  const int64_t G = gridDim.x;
  const int64_t mine = ((int64_t)blockIdx.x < p.n_tiles) ? (p.n_tiles - blockIdx.x + G - 1) / G : 0;
  // iteration j: phase 1 + look-back of tile j (j < mine), phase 2 of tile j-1 (j >= 1)
  for (int64_t j = 0; j <= mine; ++j) {
    const int br = (int)(j & 1), bf = br ^ 1;
    if (looker) {
      if (j < mine) {
        const int64_t tile = blockIdx.x + j * G;
        if (lane == 0) { while (*reinterpret_cast<volatile unsigned*>(&s_ready[br]) != (unsigned)(j + 1)) {} }
        __syncwarp();
        __threadfence_block();
        const unsigned long long total = *reinterpret_cast<volatile uint32_t*>(&s_total[br]);
        const unsigned long long excl = lookback<false>(p.status, p.gstatus, tile, total, lane);
        if (lane == 0) {
          s_tile_base_b[br] = excl;
          if (tile == p.n_tiles - 1) *p.out_len = (long long)(excl + total);
        }
      }
      __syncthreads();
      continue;
    }
    if (j < mine) {
      // ---- phase 1: this warp's 128 mask words -> shared memory, popcount scan inside the warp ----
      const int64_t tile = blockIdx.x + j * G;
      const int64_t trow0 = tile * kFTileRows;
      uint32_t cnt[kFWordsPerThread];
      uint32_t tsum = 0;
#pragma unroll
      for (int k = 0; k < kFWordsPerThread; ++k) {
        const int word = warp * kFWarpWords + lane * kFWordsPerThread + k;  // 16 consecutive mask bytes per lane
        const int64_t row0 = trow0 + (int64_t)word * 32;
        uint32_t sel = 0, nul = 0;
        if (row0 < p.n) {
          const int64_t rem = p.n - row0;
          const uint32_t range = rem >= 32 ? 0xffffffffu : bit_range_mask(0, (int)rem);
          const uint32_t m = bitmap_load32(p.mask, p.moff + row0, m_lo, m_hi);
          uint32_t mv = 0xffffffffu;
          if (p.mvalid) mv = bitmap_load32(p.mvalid, p.moff + row0, m_lo, m_hi);
          sel = m & mv & range;
          if (p.emit_nulls) nul = ~mv & range;
        }
        s_sel_b[br][word] = sel;
        s_emit_b[br][word] = sel | nul;
        cnt[k] = __popc(sel | nul);
        tsum += cnt[k];
      }
      uint32_t incl = tsum;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
      }
      uint32_t run = incl - tsum;
#pragma unroll
      for (int k = 0; k < kFWordsPerThread; ++k) { s_base_b[br][warp * kFWarpWords + lane * kFWordsPerThread + k] = run; run += cnt[k]; }
      if (lane == 31) {
        // last warp in: tile total, aggregate published, the look-back warp released (no barrier on the way)
        s_warp_tot_b[br][warp] = incl;
        __threadfence_block();
        if (atomicAdd(&s_arrived[br], 1u) == kFWarps - 1) {
          __threadfence_block();
          s_arrived[br] = 0u;
          uint32_t tot = 0;
#pragma unroll
          for (int w = 0; w < kFWarps; ++w) tot += reinterpret_cast<volatile uint32_t*>(s_warp_tot_b[br])[w];
          s_total[br] = tot;
          st_status(p.status + tile, kFlagAgg | (unsigned long long)tot);
          __threadfence_block();
          *reinterpret_cast<volatile unsigned*>(&s_ready[br]) = (unsigned)(j + 1);
        }
      }
      __syncwarp();  // phase 2 (next iteration) reads the words other lanes of this warp wrote
    }
    if (j >= 1) {
    const int64_t tile = blockIdx.x + (j - 1) * G;
    const int64_t trow0 = tile * kFTileRows;
    const uint32_t* s_emit = s_emit_b[bf];
    const uint32_t* s_sel = s_sel_b[bf];
    const uint32_t* s_base = s_base_b[bf];
    uint32_t warp_base = 0, tile_total = 0;
#pragma unroll
    for (int w = 0; w < kFWarps; ++w) {
      const uint32_t t = s_warp_tot_b[bf][w];
      if (w < warp) warp_base += t;
      tile_total += t;
    }
    // ---- phase 2: compaction; warp w owns words w*128 .. w*128+127, 32 words at a time ----------
    if (tile_total != 0) {
      const unsigned long long tbase = s_tile_base_b[bf] + warp_base;
#pragma unroll 1
      for (int g0 = warp * kFWarpWords; g0 < (warp + 1) * kFWarpWords; g0 += 32) {
        const uint32_t my_emit = s_emit[g0 + lane];
        const unsigned group_cnt = __reduce_add_sync(0xffffffffu, __popc(my_emit));
        if (group_cnt == 0) continue;
        if (group_cnt <= 256) {
          // SPARSE group (<= 25 % selected): lane j walks the set bits of ITS word, so all 32 lanes
          // have loads in flight (4 per lane) instead of the ~3 active lanes of a warp-wide step.
          // Each lane's rows land in consecutive output slots; neighbouring lanes' runs are adjacent.
          const uint32_t my_sel = s_sel[g0 + lane];
          const int64_t wrow = trow0 + (int64_t)(g0 + lane) * 32;
          unsigned long long pos = tbase + s_base[g0 + lane];
          uint32_t bits = my_emit;
          while (bits) {
            int r[4];
            V v[4];
            int cnt = 0;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              r[u] = -1;
              v[u] = V(0);
              if (bits) {
                r[u] = __ffs(bits) - 1;
                bits &= bits - 1;
                ++cnt;
                if ((my_sel >> r[u]) & 1) {
                  if (kMode == 1) v[u] = (V)(wrow + r[u]);
                  else if (kMode == 2) v[u] = (V)bit_is_set(bvals, p.voff + wrow + r[u]);
                  else v[u] = __ldcs(vals + wrow + r[u]);
                }
              }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              if (r[u] >= 0 && (long long)(pos + u) < p.capacity) {
                if (kMode == 2) { if (v[u]) atomicOr(bout + ((pos + u) >> 5), 1u << ((pos + u) & 31)); }
                else out[pos + u] = v[u];
                if (kValidity && ((my_sel >> r[u]) & 1)) {
                  const bool vb = (kMode != 1 && p.vvalid) ? bit_is_set(p.vvalid, p.voff + wrow + r[u]) : true;
                  if (vb) atomicOr(p.out_valid + ((pos + u) >> 5), 1u << ((pos + u) & 31));
                }
              }
            }
            pos += cnt;
          }
          continue;
        }
        // DENSE group: warp-wide steps, lane j owns row 32k+j (coalesced), 8 words in flight
#pragma unroll 1
        for (int j0 = g0; j0 < g0 + 32; j0 += 8) {
          V v[8];
          uint32_t w_emit[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            w_emit[u] = s_emit[j0 + u];
            const uint32_t w_sel = s_sel[j0 + u];
            const int64_t row = trow0 + (int64_t)(j0 + u) * 32 + lane;
            v[u] = V(0);
            if ((w_sel >> lane) & 1) {
              if (kMode == 1) v[u] = (V)row;
              else if (kMode == 2) v[u] = (V)bit_is_set(bvals, p.voff + row);
              else v[u] = __ldcs(vals + row);  // last use: evict-first
            }
          }
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            if (w_emit[u] == 0) continue;  // warp-uniform
            const unsigned long long b = tbase + s_base[j0 + u];
            const bool e = (w_emit[u] >> lane) & 1;
            const unsigned rank = __popc(w_emit[u] & ((1u << lane) - 1u));
            const unsigned long long pos = b + rank;
            if (kMode == 2) {
              const uint32_t dpat = __reduce_or_sync(0xffffffffu, (e && v[u]) ? (1u << rank) : 0u);
              if (lane == 0 && dpat) {
                const unsigned sh = (unsigned)(b & 31);
                const unsigned long long wi = b >> 5;
                if ((long long)wi < cap_words) atomicOr(bout + wi, dpat << sh);
                if (sh && (dpat >> (32 - sh)) && (long long)(wi + 1) < cap_words) atomicOr(bout + wi + 1, dpat >> (32 - sh));
              }
            } else if (e && (long long)pos < p.capacity) out[pos] = v[u];
            if (kValidity) {
              const int64_t row = trow0 + (int64_t)(j0 + u) * 32 + lane;
              uint32_t vb = 0;
              if (e && ((s_sel[j0 + u] >> lane) & 1)) vb = (kMode != 1 && p.vvalid) ? (uint32_t)bit_is_set(p.vvalid, p.voff + row) : 1u;
              const uint32_t pattern = __reduce_or_sync(0xffffffffu, vb << rank);  // rank < 32 whenever vb != 0
              if (lane == 0 && pattern) {
                const unsigned sh = (unsigned)(b & 31);
                const unsigned long long wi = b >> 5;
                if ((long long)wi < cap_words) atomicOr(p.out_valid + wi, pattern << sh);
                if (sh && (pattern >> (32 - sh)) && (long long)(wi + 1) < cap_words) atomicOr(p.out_valid + wi + 1, pattern >> (32 - sh));
              }
            }
          }
        }
      }
    }
    }  // j >= 1
    __syncthreads();
  }
}

template <typename V, int kMode>
static ag_status launch_filter_t(FilterParams& p, cudaStream_t st) {
  Workspace* ws;
  AG_TRY(get_workspace(st, &ws));
  WorkspaceLock ws_lock(ws);
  p.n_tiles = (p.n + kFTileRows - 1) / kFTileRows;
  const size_t n_status = (size_t)p.n_tiles + (size_t)((p.n_tiles + 31) >> 5);
  AG_TRY(ensure_tile_status(ws, n_status, st));
  p.status = ws->tile_status;
  p.gstatus = p.status + p.n_tiles;
  AG_CUDA_TRY(cudaMemsetAsync(p.status, 0, n_status * sizeof(unsigned long long), st));
  if (p.out_valid) AG_CUDA_TRY(cudaMemsetAsync(p.out_valid, 0, (size_t)((p.capacity + 31) >> 5) * 4, st));
  if (kMode == 2 && p.capacity > 0) AG_CUDA_TRY(cudaMemsetAsync(p.out, 0, (size_t)((p.capacity + 31) >> 5) * 4, st));
  void* args[] = {(void*)&p};
  if (p.out_valid)
    AG_CUDA_TRY(cudaLaunchCooperativeKernel((const void*)filter_kernel<V, kMode, true>,
                                            dim3(grid_one_wave(filter_kernel<V, kMode, true>, kFiThreads, p.n_tiles)), dim3(kFiThreads), args, 0, st));
  else
    AG_CUDA_TRY(cudaLaunchCooperativeKernel((const void*)filter_kernel<V, kMode, false>,
                                            dim3(grid_one_wave(filter_kernel<V, kMode, false>, kFiThreads, p.n_tiles)), dim3(kFiThreads), args, 0, st));
  return check_launch("filter_kernel");
}

static ag_status check_filter_args(const FilterParams& p, const char* who) {
  if (p.n < 0 || p.moff < 0 || p.voff < 0 || p.capacity < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative length or offset", who);
  if (!p.out_len) AG_FAIL(AG_ERR_INVALID, "%s: NULL out_len", who);
  if (p.out_valid && (reinterpret_cast<uintptr_t>(p.out_valid) & 3)) AG_FAIL(AG_ERR_INVALID, "%s: out_valid must be 4-byte aligned", who);
  return AG_OK;
}

ag_status filter_primitive_dev(int bit_width, const void* vals, const uint8_t* vvalid, int64_t voff,
                               const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n,
                               int null_selection, void* out, uint8_t* out_valid, int64_t capacity,
                               int64_t* d_out_len, cudaStream_t st) {
  FilterParams p{};
  p.vals = vals; p.vvalid = vvalid; p.voff = voff; p.mask = mask; p.mvalid = mvalid; p.moff = moff; p.n = n;
  p.emit_nulls = (null_selection == AG_EMIT_NULLS) && mvalid != nullptr;
  p.out = out; p.out_valid = reinterpret_cast<uint32_t*>(out_valid); p.capacity = capacity;
  p.out_len = reinterpret_cast<long long*>(d_out_len);
  AG_TRY(check_filter_args(p, "filter"));
  if (n > 0 && !mask) AG_FAIL(AG_ERR_INVALID, "filter: NULL mask");
  if (null_selection != AG_DROP_NULLS && null_selection != AG_EMIT_NULLS) AG_FAIL(AG_ERR_INVALID, "filter: bad null_selection %d", null_selection);
  if ((vvalid || p.emit_nulls) && !out_valid && capacity > 0)
    AG_FAIL(AG_ERR_INVALID, "filter: the output can contain nulls but no output validity buffer was given (vector_selection.go:473)");
  if (n == 0) { AG_CUDA_TRY(cudaMemsetAsync(d_out_len, 0, sizeof(int64_t), st)); return AG_OK; }
  if (!vals || (!out && capacity > 0)) AG_FAIL(AG_ERR_INVALID, "filter: NULL values/output");
  if (bit_width == 1) {
    // boolean values: the output data bitmap is compacted like the validity bits.  (The reference's
    // boolFilterWriter.WriteValue never advances its position, vector_selection.go:433-436; we
    // implement the documented semantics, identical to every other width.)
    if ((uintptr_t)out & 3) AG_FAIL(AG_ERR_INVALID, "filter: boolean output bitmap must be 4-byte aligned");
    return launch_filter_t<uint32_t, 2>(p, st);
  }
  return visit_width(bit_width, [&](auto tag) {
    using V = typename decltype(tag)::type;
    const uintptr_t am = sizeof(V) - 1;
    if (((uintptr_t)vals & am) || ((uintptr_t)out & am)) AG_FAIL(AG_ERR_INVALID, "filter: buffers not aligned to the element width");
    return launch_filter_t<V, 0>(p, st);
  }, [&] { AG_FAIL(AG_ERR_TYPE, "filter: invalid values bit width %d", bit_width); });
}

ag_status take_indices_dev(int index_width, const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n,
                           int null_selection, void* out_idx, uint8_t* out_valid, int64_t capacity,
                           int64_t* d_out_len, cudaStream_t st) {
  FilterParams p{};
  p.mask = mask; p.mvalid = mvalid; p.moff = moff; p.n = n;
  p.emit_nulls = (null_selection == AG_EMIT_NULLS) && mvalid != nullptr;
  p.out = out_idx; p.out_valid = reinterpret_cast<uint32_t*>(out_valid); p.capacity = capacity;
  p.out_len = reinterpret_cast<long long*>(d_out_len);
  AG_TRY(check_filter_args(p, "take_indices"));
  if (n > 0 && !mask) AG_FAIL(AG_ERR_INVALID, "take_indices: NULL mask");
  if (p.emit_nulls && !out_valid && capacity > 0)
    AG_FAIL(AG_ERR_INVALID, "take_indices: EMIT_NULLS with a mask validity bitmap needs an output validity bitmap (a null mask slot would otherwise read as row 0)");
  if (n == 0) { AG_CUDA_TRY(cudaMemsetAsync(d_out_len, 0, sizeof(int64_t), st)); return AG_OK; }
  if (index_width == 16) {
    if (n >= 65535) AG_FAIL(AG_ERR_INVALID, "take_indices: uint16 indices need n < 65535 (vector_selection.go:229-231)");
    return launch_filter_t<uint16_t, 1>(p, st);
  }
  if (index_width == 32) {
    if (n >= 4294967295ll) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "take_indices: filter length exceeds UINT32_MAX (vector_selection.go:233-235)");
    return launch_filter_t<uint32_t, 1>(p, st);
  }
  AG_FAIL(AG_ERR_TYPE, "take_indices: index width must be 16 or 32");
}

// ---------------------------------------------------------------- fused compare + filter ----
// Greater/…(values, scalar) -> Filter in ONE kernel (config 3 of BASELINE.json): no intermediate
// mask in HBM and every value is read from HBM exactly once (8 + 8s bytes/row).
//
// A 16K-row block tile is 16 "segments" of 1024 rows (2 per compute warp).  Phase 1, per segment: lane j
// loads rows 32k+j (32 coalesced 256-byte requests in flight, requested one segment AHEAD of the votes,
// across tile boundaries too), __ballot_sync packs the predicate words, every lane tracks the running count
// from the ballots and the selected values go straight from registers into the segment's staging area in
// SHARED memory.  Phase 2 copies each staged segment to out[] with fully coalesced stores.  A segment that
// selects more rows than its staging area holds (kSegCap, > 21 % of 1024) is compacted by re-reading it.
//
// Schedule.  The block-synchronous shape —
// 8 warps stream a tile, meet, warp 0 resolves the look-back, all copy out — left every resident block in
// the same phase, so nothing covered the look-back, whatever the occupancy,
// the look-back width or the tile claiming order.  Here the look-back is off the critical path:
//   * a block = 8 compute warps + 1 LOOK-BACK warp, staging areas double-buffered;
//   * iteration j: the compute warps run phase 1 of tile j and then phase 2 of tile j-1, while the look-back
//     warp resolves the prefix of tile j-1; one block barrier per tile joins them;
//   * a tile's aggregate is published by the LAST compute warp to finish its segments (shared-memory counter):
//     other blocks see it a whole phase-2 + look-back ahead of the moment they need it.
constexpr int kSegRows = 1024;
constexpr int kSegCap = 224;                              // staged values per segment
constexpr int kFuTileRows = 16384;
constexpr int kFuSegs = kFuTileRows / kSegRows;           // 16
constexpr int kFuSegsPerWarp = kFuSegs / kFWarps;         // 2
constexpr int kFuThreads = kFThreads + 32;                // + the look-back warp
constexpr int kFuEmitWords = kFuTileRows / 32;            // 512

template <typename T>
struct FusedBuffers {   // one of the two staging buffers (dynamic shared memory)
  uint32_t emit[kFuEmitWords];   // predicate words (overflow path only)
  uint32_t cnt[kFuSegs];         // rows selected per segment
  uint32_t excl[kFuSegs];        // exclusive offsets inside the tile
  T stage[kFuSegs][kSegCap];
};

template <typename T, typename Cmp>
__global__ void __launch_bounds__(kFuThreads, 2)
fused_filter_kernel(const T* __restrict__ vals, T scalar, int64_t n, T* __restrict__ out, int64_t capacity,
                    unsigned long long* status, unsigned long long* gstatus, long long* out_len, int64_t n_tiles) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FusedBuffers<T>* bufs = reinterpret_cast<FusedBuffers<T>*>(smem_raw);   // [2]
  __shared__ unsigned long long s_tile_base[2];
  __shared__ uint32_t s_total[2];
  __shared__ unsigned s_arrived[2], s_ready[2], s_done[2];   // sequence-numbered: tile j of this block <-> j + 1
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool looker = warp == kFWarps;
  if (threadIdx.x < 2) { s_arrived[threadIdx.x] = 0u; s_ready[threadIdx.x] = 0u; s_done[threadIdx.x] = 0u; }
  __syncthreads();
  const int64_t G = gridDim.x;
  const int64_t mine = ((int64_t)blockIdx.x < n_tiles) ? (n_tiles - blockIdx.x + G - 1) / G : 0;
  // No block barrier from here on: compute warps and the look-back warp meet through s_ready (a tile's total is in)
  // and s_done (its base is out), so a warp that is ahead is never held back by one that is behind.
  if (looker) {
    for (int64_t j = 0; j < mine; ++j) {
      const int64_t tile = blockIdx.x + j * G;
      const int b = (int)(j & 1);
      if (lane == 0) { while (*reinterpret_cast<volatile unsigned*>(&s_ready[b]) != (unsigned)(j + 1)) {} }
      __syncwarp();
      __threadfence_block();
      const unsigned long long total = *reinterpret_cast<volatile uint32_t*>(&s_total[b]);
      const unsigned long long excl = lookback<false>(status, gstatus, tile, total, lane);
      if (lane == 0) {
        s_tile_base[b] = excl;
        if (tile == n_tiles - 1) *out_len = (long long)(excl + total);
        __threadfence_block();
        *reinterpret_cast<volatile unsigned*>(&s_done[b]) = (unsigned)(j + 1);
      }
    }
    return;
  }

  T v[32];
  auto issue = [&](int64_t t, int sub) {
    const int64_t wrow0 = t * kFuTileRows + (int64_t)(sub * kFWarps + warp) * kSegRows;
    if (wrow0 + kSegRows <= n) {
#pragma unroll
      for (int k = 0; k < 32; ++k) v[k] = __ldcs(vals + wrow0 + k * 32 + lane);
    } else {
#pragma unroll
      for (int k = 0; k < 32; ++k) {
        const int64_t row = wrow0 + k * 32 + lane;
        v[k] = (row < n) ? __ldcs(vals + row) : scalar;
      }
    }
  };
  if (mine > 0) issue(blockIdx.x, 0);
  // iteration j: phase 1 of tile j (j < mine); phase 2 of tile j-1 (j >= 1)
  for (int64_t j = 0; j <= mine; ++j) {
    const int64_t tile_r = blockIdx.x + j * G, tile_f = tile_r - G;
    const int br = (int)(j & 1), bf = br ^ 1;
    {
      if (j < mine) {
        FusedBuffers<T>& B = bufs[br];
        const int64_t trow0 = tile_r * kFuTileRows;
#pragma unroll 1
        for (int sub = 0; sub < kFuSegsPerWarp; ++sub) {
          const int seg = sub * kFWarps + warp;
          const int64_t wrow0 = trow0 + (int64_t)seg * kSegRows;
          __syncwarp();  // keep every load ahead of the first vote
          // Every lane sees every ballot, so each lane tracks the running count itself: the slot of a selected row is
          // (rows selected in earlier words) + (selected rows below it in its word).  No scan and no shuffles; values
          // go from registers straight into the staging area (slots past kSegCap are dropped: overflow path).
          T* stage = B.stage[seg];
          uint32_t myword = 0;
          unsigned running = 0;
          const uint32_t lt = (1u << lane) - 1u;
          if (wrow0 + kSegRows <= n) {  // interior segment: no per-row range test
#pragma unroll
            for (int k = 0; k < 32; ++k) {
              const bool pr = Cmp::template apply<T>(v[k], scalar);
              const uint32_t bits = __ballot_sync(0xffffffffu, pr);
              if (lane == k) myword = bits;
              const unsigned pos = running + __popc(bits & lt);
              if (pr && pos < kSegCap) stage[pos] = v[k];
              running += __popc(bits);
            }
          } else {
#pragma unroll
            for (int k = 0; k < 32; ++k) {
              const int64_t row = wrow0 + k * 32 + lane;
              const bool pr = row < n && Cmp::template apply<T>(v[k], scalar);
              const uint32_t bits = __ballot_sync(0xffffffffu, pr);
              if (lane == k) myword = bits;
              const unsigned pos = running + __popc(bits & lt);
              if (pr && pos < kSegCap) stage[pos] = v[k];
              running += __popc(bits);
            }
          }
          B.emit[seg * 32 + lane] = myword;
          if (lane == 0) B.cnt[seg] = running;
          if (sub + 1 < kFuSegsPerWarp) issue(tile_r, sub + 1);
          else if (j + 1 < mine) issue(tile_r + G, 0);
        }
        if (lane == 0) {
          // last warp in: segment offsets, tile total, aggregate published (no barrier on the way)
          __threadfence_block();
          if (atomicAdd(&s_arrived[br], 1u) == kFWarps - 1) {
            __threadfence_block();
            s_arrived[br] = 0u;
            uint32_t run = 0;
#pragma unroll
            for (int sg = 0; sg < kFuSegs; ++sg) {
              const uint32_t c = reinterpret_cast<volatile uint32_t*>(B.cnt)[sg];
              B.excl[sg] = run;
              run += c;
            }
            s_total[br] = run;
            st_status(status + tile_r, kFlagAgg | (unsigned long long)run);
            __threadfence_block();
            *reinterpret_cast<volatile unsigned*>(&s_ready[br]) = (unsigned)(j + 1);
          }
        }
      }
    }
    if (j >= 1) {
      // ---- phase 2: staged segments -> out[] with coalesced stores --------------------------------
      if (lane == 0) { while (*reinterpret_cast<volatile unsigned*>(&s_done[bf]) != (unsigned)j) {} }
      __syncwarp();
      __threadfence_block();
      FusedBuffers<T>& B = bufs[bf];
      const int64_t trow0 = tile_f * kFuTileRows;
      const unsigned long long tbase = *reinterpret_cast<volatile unsigned long long*>(&s_tile_base[bf]);
#pragma unroll 1
      for (int sub = 0; sub < kFuSegsPerWarp; ++sub) {
        const int seg = sub * kFWarps + warp;
        const unsigned total = B.cnt[seg];
        if (total == 0) continue;
        const unsigned long long base = tbase + reinterpret_cast<volatile uint32_t*>(B.excl)[seg];
        if (total <= kSegCap) {
          const T* stage = B.stage[seg];
          for (unsigned i = lane; i < total; i += 32)
            if ((long long)(base + i) < capacity) out[base + i] = stage[i];
        } else {
          // overflow: re-read the segment's selected rows (they are at worst in L2)
          const uint32_t myword = B.emit[seg * 32 + lane];
          const unsigned cnt = __popc(myword);
          unsigned incl = cnt;
#pragma unroll
          for (int d = 1; d < 32; d <<= 1) {
            const unsigned t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
          }
          const unsigned my_excl = incl - cnt;
          const int64_t wrow0 = trow0 + (int64_t)seg * kSegRows;
#pragma unroll 4
          for (int k = 0; k < 32; ++k) {
            const uint32_t w = __shfl_sync(0xffffffffu, myword, k);
            const unsigned off = __shfl_sync(0xffffffffu, my_excl, k);
            if ((w >> lane) & 1) {
              const unsigned long long pos = base + off + __popc(w & ((1u << lane) - 1u));
              if ((long long)pos < capacity) out[pos] = __ldcs(vals + wrow0 + k * 32 + lane);
            }
          }
        }
      }
      __syncwarp();  // this warp's staging areas of buffer bf are rewritten two iterations from now
    }
  }
}

template <typename T, typename Cmp>
static ag_status launch_fused_t(const void* vals, const void* scalar_host, int64_t n, void* out, int64_t capacity,
                                int64_t* d_out_len, cudaStream_t st) {
  Workspace* ws;
  AG_TRY(get_workspace(st, &ws));
  WorkspaceLock ws_lock(ws);
  const int64_t n_tiles = (n + kFuTileRows - 1) / kFuTileRows;
  const size_t n_status = (size_t)n_tiles + (size_t)((n_tiles + 31) >> 5);
  AG_TRY(ensure_tile_status(ws, n_status, st));
  AG_CUDA_TRY(cudaMemsetAsync(ws->tile_status, 0, n_status * sizeof(unsigned long long), st));
  const size_t smem = 2 * sizeof(FusedBuffers<T>);
  static std::atomic<unsigned> attr_set{0u};  // per instantiation, one bit per device
  const void* fn = (const void*)fused_filter_kernel<T, Cmp>;
  AG_TRY(ensure_dynamic_smem(fn, (int)smem, &attr_set));
  int per_sm = 0;
  AG_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kFuThreads, smem));
  if (per_sm < 1) per_sm = 1;
  int64_t grid = (int64_t)sm_count() * per_sm;
  if (grid > n_tiles) grid = n_tiles;
  const T* a_vals = (const T*)vals;
  T a_scalar = *(const T*)scalar_host;
  T* a_out = (T*)out;
  unsigned long long* a_status = ws->tile_status;
  unsigned long long* a_gstatus = ws->tile_status + n_tiles;
  long long* a_len = (long long*)d_out_len;
  int64_t a_n = n, a_cap = capacity, a_tiles = n_tiles;
  void* args[] = {&a_vals, &a_scalar, &a_n, &a_out, &a_cap, &a_status, &a_gstatus, &a_len, &a_tiles};
  AG_CUDA_TRY(cudaLaunchCooperativeKernel(fn, dim3((unsigned)grid), dim3(kFuThreads), args, smem, st));
  return check_launch("fused_filter_kernel");
}

template <typename T>
static ag_status launch_fused_cmp(int cmp, const void* vals, const void* scalar_host, int64_t n, void* out, int64_t capacity,
                                  int64_t* d_out_len, cudaStream_t st) {
  switch (cmp) {
    case AG_CMP_EQ: return launch_fused_t<T, FCmpEq>(vals, scalar_host, n, out, capacity, d_out_len, st);
    case AG_CMP_NE: return launch_fused_t<T, FCmpNe>(vals, scalar_host, n, out, capacity, d_out_len, st);
    case AG_CMP_GT: return launch_fused_t<T, FCmpGt>(vals, scalar_host, n, out, capacity, d_out_len, st);
    case AG_CMP_GE: return launch_fused_t<T, FCmpGe>(vals, scalar_host, n, out, capacity, d_out_len, st);
    case AG_CMP_LT: return launch_fused_t<T, FCmpLt>(vals, scalar_host, n, out, capacity, d_out_len, st);
    case AG_CMP_LE: return launch_fused_t<T, FCmpLe>(vals, scalar_host, n, out, capacity, d_out_len, st);
    default: AG_FAIL(AG_ERR_INVALID, "filter_compare: bad operator %d", cmp);
  }
}

ag_status filter_compare_scalar_dev(int type, int cmp, const void* vals, const void* scalar_host, int64_t n,
                                    void* out, int64_t capacity, int64_t* d_out_len, cudaStream_t st) {
  if (n < 0 || capacity < 0) AG_FAIL(AG_ERR_INVALID, "filter_compare: negative length");
  if (!d_out_len || !scalar_host) AG_FAIL(AG_ERR_INVALID, "filter_compare: NULL argument");
  if (n == 0) { AG_CUDA_TRY(cudaMemsetAsync(d_out_len, 0, sizeof(int64_t), st)); return AG_OK; }
  if (!vals || (!out && capacity > 0)) AG_FAIL(AG_ERR_INVALID, "filter_compare: NULL values/output");
  const auto not_fused = [&] {
    AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "filter_compare: fused path covers 32/64-bit types; use compare + filter for type id %d", type);
  };
  return visit_type(type, [&](auto tag) {
    using T = typename decltype(tag)::type;
    if constexpr (sizeof(T) >= 4) return launch_fused_cmp<T>(cmp, vals, scalar_host, n, out, capacity, d_out_len, st);
    else return not_fused();
  }, not_fused);
}

// ---------------------------------------------------------------- output size ------
// getFilterOutputSize (vector_selection.go:57-81): popcount(mask ∧ valid) | popcount(mask ∨ ¬valid)
__global__ void __launch_bounds__(kFThreads)
filter_count_kernel(const uint8_t* __restrict__ mask, const uint8_t* __restrict__ mvalid, int64_t moff, int64_t n,
                    int emit_nulls, unsigned long long* __restrict__ count) {
  const int64_t n_words = (n + 31) >> 5;
  const int64_t lo = moff >> 3, hi = (moff + n + 7) >> 3;
  const int64_t stride = (int64_t)gridDim.x * kFThreads;
  unsigned long long c = 0;
  for (int64_t w = (int64_t)blockIdx.x * kFThreads + threadIdx.x; w < n_words; w += stride) {
    const int64_t rem = n - (w << 5);
    const uint32_t range = rem >= 32 ? 0xffffffffu : bit_range_mask(0, (int)rem);
    const uint32_t m = bitmap_load32(mask, moff + (w << 5), lo, hi);
    uint32_t mv = 0xffffffffu;
    if (mvalid) mv = bitmap_load32(mvalid, moff + (w << 5), lo, hi);
    const uint32_t v = emit_nulls ? (m | ~mv) : (m & mv);
    c += __popc(v & range);
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) c += __shfl_xor_sync(0xffffffffu, c, m);
  __shared__ unsigned long long sm[kFWarps];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
#pragma unroll
    for (int i = 0; i < kFWarps; ++i) t += sm[i];
    if (t) atomicAdd(count, t);
  }
}

ag_status filter_output_size_dev(const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n,
                                 int null_selection, int64_t* d_out_len, cudaStream_t st) {
  if (n < 0 || moff < 0) AG_FAIL(AG_ERR_INVALID, "filter_output_size: negative length or offset");
  if (!d_out_len) AG_FAIL(AG_ERR_INVALID, "filter_output_size: NULL result");
  AG_CUDA_TRY(cudaMemsetAsync(d_out_len, 0, sizeof(int64_t), st));
  if (n == 0) return AG_OK;
  if (!mask) AG_FAIL(AG_ERR_INVALID, "filter_output_size: NULL mask");
  const int grid = grid_for((n + 31) >> 5, kFThreads * 4, 4);
  filter_count_kernel<<<grid, kFThreads, 0, st>>>(mask, mvalid, moff, n, null_selection == AG_EMIT_NULLS, (unsigned long long*)d_out_len);
  return check_launch("filter_count_kernel");
}

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_filter_output_size_dev(const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n,
                                    int null_selection, int64_t* d_out_len, ag_stream_t s) {
  AG_TRY(ensure_init());
  return filter_output_size_dev(mask, mvalid, moff, n, null_selection, d_out_len, resolve_stream(s));
}
ag_status ag_filter_primitive_dev(int bit_width, const void* vals, const uint8_t* vvalid, int64_t voff,
                                  const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n,
                                  int null_selection, void* out, uint8_t* out_valid, int64_t out_capacity,
                                  int64_t* d_out_len, ag_stream_t s) {
  AG_TRY(ensure_init());
  return filter_primitive_dev(bit_width, vals, vvalid, voff, mask, mvalid, moff, n, null_selection, out, out_valid,
                              out_capacity, d_out_len, resolve_stream(s));
}
ag_status ag_filter_compare_scalar_dev(int type, int cmp, const void* d_vals, const void* scalar_host, int64_t n,
                                       void* d_out, int64_t out_capacity, int64_t* d_out_len, ag_stream_t s) {
  AG_TRY(ensure_init());
  return filter_compare_scalar_dev(type, cmp, d_vals, scalar_host, n, d_out, out_capacity, d_out_len, resolve_stream(s));
}
ag_status ag_take_indices_dev(int index_width, const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n,
                              int null_selection, void* out_idx, uint8_t* out_valid, int64_t out_capacity,
                              int64_t* d_out_len, ag_stream_t s) {
  AG_TRY(ensure_init());
  return take_indices_dev(index_width, mask, mvalid, moff, n, null_selection, out_idx, out_valid, out_capacity,
                          d_out_len, resolve_stream(s));
}

}  // extern "C"
