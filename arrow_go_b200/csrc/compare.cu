// compare.cu — scalar comparisons -> LSB-first bitmap on sm_90a.
//
// Replaces comparison_{equal,not_equal,greater,greater_equal}_{arr_arr,arr_scalar,scalar_arr}
// _{avx2,sse4} (arrow/compute/internal/kernels/_lib/scalar_comparison.cc:63-256) and the Go
// driver compareKernel (kernels/scalar_comparisons.go:199-218): the output pointer addresses
// the byte holding the first result bit and `offset % 8` is the bit position inside it; bits
// outside [offset, offset+n) are preserved (set_bit_to, scalar_comparison.cc:59-61).
// LT / LE run as GT / GE with operands flipped (arrow/compute/scalar_compare.go:73-99).
//
// Roofline: HBM.  arr⊕scalar on int64 reads 8 B and writes 1/8 B per row (8.125 B/row).
//
// Layout: the output is processed in ALIGNED 32-bit words so that no two threads ever touch
// the same word.  A warp owns a tile of 32 consecutive words (1024 rows): in step k every lane
// loads row (32*(w0+k) + lane - shift) — one coalesced 256-byte request for 8-byte values —
// and __ballot_sync packs the 32 predicates into word k, which lane k keeps.  After 32 steps
// lane k stores word w0+k: one coalesced 128-byte store per warp per 1024 rows.  Words that
// straddle the ends of the range are merged byte-wise (bitmap_store32_masked), so bytes the
// reference would not touch are not touched.
#include "common.cuh"
#include "elem_ops.cuh"

#include <type_traits>

namespace ag {

constexpr int kCmpThreads = 256;
constexpr int kCmpFastBatch = 16;  // interior tiles: loads in flight per lane before the votes
constexpr int kCmpBatch = 8;   // loads in flight per lane before the votes (16 -> 90 regs, 2 blocks/SM: measured slower)

template <typename T, typename Cmp, int kShape>
__global__ void __launch_bounds__(kCmpThreads)
compare_kernel(const T* __restrict__ l, const T* __restrict__ r, T scalar,
               uint32_t* __restrict__ out_words, int shift, int64_t n, int64_t n_words) {
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * (kCmpThreads / 32);
  const int64_t warp_id = (int64_t)blockIdx.x * (kCmpThreads / 32) + (threadIdx.x >> 5);
  const int64_t n_tiles = (n_words + 31) >> 5;
  for (int64_t tile = warp_id; tile < n_tiles; tile += warps_total) {
    const int64_t w0 = tile << 5;
    uint32_t myword = 0;
    const int64_t e_first = (w0 << 5) - shift;  // row of bit 0 of the tile's first word
    if (e_first >= 0 && e_first + 1024 <= n) {
      // interior tile: every row is in range — no per-row bounds tests, pointers advance by 32 rows
      const T* lp = (kShape != AG_SHAPE_SA) ? l + e_first + lane : nullptr;
      const T* rp = (kShape != AG_SHAPE_AS) ? r + e_first + lane : nullptr;
#pragma unroll
      for (int kb = 0; kb < 32; kb += kCmpFastBatch) {
        T a[kCmpFastBatch], b[kCmpFastBatch];
#pragma unroll
        for (int u = 0; u < kCmpFastBatch; ++u) {
          a[u] = (kShape != AG_SHAPE_SA) ? __ldcs(lp + (kb + u) * 32) : scalar;
          b[u] = (kShape != AG_SHAPE_AS) ? __ldcs(rp + (kb + u) * 32) : scalar;
        }
        __syncwarp();  // scheduling fence: issue the whole batch of loads before the first vote
#pragma unroll
        for (int u = 0; u < kCmpFastBatch; ++u) {
          const uint32_t bits = __ballot_sync(0xffffffffu, Cmp::template apply<T>(a[u], b[u]));
          if (lane == kb + u) myword = bits;
        }
      }
    } else {
#pragma unroll
      for (int kb = 0; kb < 32; kb += kCmpBatch) {
        T a[kCmpBatch], b[kCmpBatch];
        bool inr[kCmpBatch];
#pragma unroll
        for (int u = 0; u < kCmpBatch; ++u) {
          const int64_t e = ((w0 + kb + u) << 5) + lane - shift;
          inr[u] = (e >= 0) && (e < n);
          a[u] = scalar; b[u] = scalar;
          if (inr[u]) {
            if (kShape != AG_SHAPE_SA) a[u] = __ldcs(l + e);
            if (kShape != AG_SHAPE_AS) b[u] = __ldcs(r + e);
          }
        }
#pragma unroll
        for (int u = 0; u < kCmpBatch; ++u) {
          const uint32_t bits = __ballot_sync(0xffffffffu, inr[u] && Cmp::template apply<T>(a[u], b[u]));
          if (lane == kb + u) myword = bits;
        }
      }
    }
    const int64_t w = w0 + lane;
    if (w < n_words) {
      // rows covered by word w: e = 32w + b - shift, keep bits with 0 <= e < n
      const int64_t lo64 = (int64_t)shift - (w << 5);
      const int64_t hi64 = n + (int64_t)shift - (w << 5);
      const int lo = lo64 > 0 ? (int)lo64 : 0;
      const int hi = hi64 < 32 ? (int)hi64 : 32;
      if (hi > lo) bitmap_store32_masked(out_words + w, myword, bit_range_mask(lo, hi));
    }
  }
}

template <typename T, typename Cmp>
static ag_status launch_cmp_shape(int shape, const void* l, const void* r, uint8_t* out_bits, int64_t n, int bit_offset, cudaStream_t st) {
  const uintptr_t p = reinterpret_cast<uintptr_t>(out_bits);
  uint32_t* words = reinterpret_cast<uint32_t*>(p & ~(uintptr_t)3);
  const int shift = (int)(p & 3) * 8 + (bit_offset & 7);
  const int64_t n_words = (n + shift + 31) >> 5;
  const int64_t blocks_needed = (((n_words + 31) >> 5) + kCmpThreads / 32 - 1) / (kCmpThreads / 32);
  return visit_shape(shape, [&](auto s) {
    constexpr int kShape = decltype(s)::value;
    const T scalar = kShape == AG_SHAPE_AS ? *(const T*)r : (kShape == AG_SHAPE_SA ? *(const T*)l : T(0));
    const int grid = grid_one_wave(compare_kernel<T, Cmp, kShape>, kCmpThreads, blocks_needed);
    compare_kernel<T, Cmp, kShape><<<grid, kCmpThreads, 0, st>>>(kShape == AG_SHAPE_SA ? nullptr : (const T*)l,
                                                                  kShape == AG_SHAPE_AS ? nullptr : (const T*)r, scalar, words, shift, n, n_words);
    return check_launch("compare_kernel");
  }, [&] { AG_FAIL(AG_ERR_INVALID, "compare: bad operand shape %d", shape); });
}

ag_status compare_dev(int type, int cmp, int shape, const void* l, const void* r, uint8_t* out, int64_t n, int off, cudaStream_t st) {
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "compare: negative length");
  if (n == 0) return AG_OK;
  if (!out) AG_FAIL(AG_ERR_INVALID, "compare: NULL output bitmap");
  const int w = type_width(type);
  if (w == 0) AG_FAIL(AG_ERR_TYPE, "compare: unsupported type id %d", type);
  if (cmp == AG_CMP_LT || cmp == AG_CMP_LE) {
    // a < b == b > a ; a <= b == b >= a  (scalar_compare.go:73-99)
    const void* t = l; l = r; r = t;
    shape = (shape == AG_SHAPE_AS) ? AG_SHAPE_SA : (shape == AG_SHAPE_SA ? AG_SHAPE_AS : AG_SHAPE_AA);
    cmp = (cmp == AG_CMP_LT) ? AG_CMP_GT : AG_CMP_GE;
  }
  const uintptr_t m = (uintptr_t)(w - 1);
  if ((shape != AG_SHAPE_SA && ((uintptr_t)l & m)) || (shape != AG_SHAPE_AS && ((uintptr_t)r & m)))
    AG_FAIL(AG_ERR_INVALID, "compare: operand not aligned to its element width");
  const auto launch = [&](auto cmp_tag) {
    return [&, cmp_tag](auto tag) { return launch_cmp_shape<typename decltype(tag)::type, decltype(cmp_tag)>(shape, l, r, out, n, off, st); };
  };
  const auto bad_type = [&] { AG_FAIL(AG_ERR_TYPE, "compare: unsupported type id %d", type); };
  // ==/!= only look at the bits: they run on the storage type
  switch (cmp) {
    case AG_CMP_EQ: return visit_storage_type(type, launch(CmpEq{}), bad_type);
    case AG_CMP_NE: return visit_storage_type(type, launch(CmpNe{}), bad_type);
    case AG_CMP_GT: return visit_type(type, launch(CmpGt{}), bad_type);
    case AG_CMP_GE: return visit_type(type, launch(CmpGe{}), bad_type);
    default: AG_FAIL(AG_ERR_INVALID, "compare: bad operator %d", cmp);
  }
}

}  // namespace ag

using namespace ag;

extern "C" ag_status ag_compare_dev(int type, int cmp, int shape, const void* l, const void* r,
                                    uint8_t* out, int64_t n, int bit_offset, ag_stream_t s) {
  AG_TRY(ensure_init());
  return compare_dev(type, cmp, shape, l, r, out, n, bit_offset, resolve_stream(s));
}
