// bitmap.cu — validity / boolean bitmap kernels on sm_90a.
//
// Replaces bitmap_aligned_{and,or,and_not,xor}_{avx2,sse4} (arrow/bitutil/_lib/bitmap_ops.c:24-46)
// and the Go code around them: alignedBitmapOp / unalignedBitmapOp (arrow/bitutil/bitmaps.go:
// 527-591), BitmapAnd/Or/Xor/AndNot/Xnor (:601-639), CopyBitmap / InvertBitmap (:483-491),
// SetBitsTo (arrow/bitutil/bitutil.go:158), CountSetBits (:89); the Kleene word lambdas of
// arrow/compute/internal/kernels/scalar_boolean.go:29-65,103-105,180-182,290-292.
//
// These are what propagateNulls (arrow/compute/executor.go:237-349) and the boolean kernels
// run on.  A bitmap is 1/64 of its value column, so the kernels are launch/latency bound at
// record-batch sizes; they are written for exactness with arbitrary bit offsets on every
// operand: one thread per ALIGNED 32-bit output word, inputs fetched as two aligned words +
// funnel shift, edge words merged byte-wise so no byte outside [offset, offset+n) is written.
#include "common.cuh"
#include "elem_ops.cuh"

namespace ag {

constexpr int kBmThreads = 256;

struct BitmapArg {
  const uint8_t* p;   // may be NULL => all ones
  int64_t off;        // bit offset of element 0
};

template <int kOp, int kNIn>
__global__ void __launch_bounds__(kBmThreads)
bitmap_word_kernel(BitmapArg i0, BitmapArg i1, BitmapArg i2, BitmapArg i3,
                   uint32_t* __restrict__ out_words, int shift, int64_t n, int64_t n_words) {
  const int64_t stride = (int64_t)gridDim.x * kBmThreads;
  for (int64_t w = (int64_t)blockIdx.x * kBmThreads + threadIdx.x; w < n_words; w += stride) {
    const int64_t e0 = (w << 5) - shift;  // element index of bit 0 of this output word (may be < 0)
    uint32_t v[4] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
    const BitmapArg in[4] = {i0, i1, i2, i3};
#pragma unroll
    for (int k = 0; k < kNIn; ++k) {
      if (in[k].p) {
        const int64_t lo_byte = in[k].off >> 3;
        const int64_t hi_byte = (in[k].off + n + 7) >> 3;
        v[k] = bitmap_load32(in[k].p, in[k].off + e0, lo_byte, hi_byte);
      }
    }
    const uint32_t o = word_op<kOp>(v[0], v[1], v[2], v[3]);
    const int64_t lo64 = -e0, hi64 = n - e0;
    const int lo = lo64 > 0 ? (int)lo64 : 0;
    const int hi = hi64 < 32 ? (int)hi64 : 32;
    if (hi > lo) bitmap_store32_masked(out_words + w, o, bit_range_mask(lo, hi));
  }
}

template <int kOp, int kNIn>
static ag_status launch_word(BitmapArg a, BitmapArg b, BitmapArg c, BitmapArg d,
                             uint8_t* out, int64_t ooff, int64_t n, cudaStream_t st) {
  if (n == 0) return AG_OK;
  uint8_t* first = out + (ooff >> 3);
  const uintptr_t p = reinterpret_cast<uintptr_t>(first);
  uint32_t* words = reinterpret_cast<uint32_t*>(p & ~(uintptr_t)3);
  const int shift = (int)(p & 3) * 8 + (int)(ooff & 7);
  const int64_t n_words = (n + shift + 31) >> 5;
  const int grid = grid_for(n_words, kBmThreads, 8);
  bitmap_word_kernel<kOp, kNIn><<<grid, kBmThreads, 0, st>>>(a, b, c, d, words, shift, n, n_words);
  return check_launch("bitmap_word_kernel");
}

ag_status bitmap_op_dev(int bitop, const uint8_t* l, int64_t loff, const uint8_t* r, int64_t roff,
                        uint8_t* out, int64_t ooff, int64_t n, cudaStream_t st) {
  if (n < 0 || loff < 0 || roff < 0 || ooff < 0) AG_FAIL(AG_ERR_INVALID, "bitmap_op: negative length or offset");
  if (n == 0) return AG_OK;
  if (!l || !r || !out) AG_FAIL(AG_ERR_INVALID, "bitmap_op: NULL bitmap");
  const BitmapArg a{l, loff}, b{r, roff}, z{nullptr, 0};
  switch (bitop) {
    case AG_BITOP_AND: return launch_word<W_AND, 2>(a, b, z, z, out, ooff, n, st);
    case AG_BITOP_OR: return launch_word<W_OR, 2>(a, b, z, z, out, ooff, n, st);
    case AG_BITOP_XOR: return launch_word<W_XOR, 2>(a, b, z, z, out, ooff, n, st);
    case AG_BITOP_ANDNOT: return launch_word<W_ANDNOT, 2>(a, b, z, z, out, ooff, n, st);
    case AG_BITOP_XNOR: return launch_word<W_XNOR, 2>(a, b, z, z, out, ooff, n, st);
    default: AG_FAIL(AG_ERR_INVALID, "bitmap_op: bad op %d", bitop);
  }
}

ag_status bitmap_copy_dev(const uint8_t* src, int64_t soff, int64_t n, uint8_t* dst, int64_t doff, bool invert, cudaStream_t st) {
  if (n < 0 || soff < 0 || doff < 0) AG_FAIL(AG_ERR_INVALID, "bitmap_copy: negative length or offset");
  if (n == 0) return AG_OK;
  if (!src || !dst) AG_FAIL(AG_ERR_INVALID, "bitmap_copy: NULL bitmap");
  const BitmapArg a{src, soff}, z{nullptr, 0};
  if (invert) return launch_word<W_INVERT, 1>(a, z, z, z, dst, doff, n, st);
  return launch_word<W_COPY, 1>(a, z, z, z, dst, doff, n, st);
}

ag_status bitmap_set_dev(uint8_t* bits, int64_t off, int64_t n, int value, cudaStream_t st) {
  if (n < 0 || off < 0) AG_FAIL(AG_ERR_INVALID, "bitmap_set: negative length or offset");
  if (n == 0) return AG_OK;
  if (!bits) AG_FAIL(AG_ERR_INVALID, "bitmap_set: NULL bitmap");
  const BitmapArg z{nullptr, 0};
  if (value) return launch_word<W_SET1, 0>(z, z, z, z, bits, off, n, st);
  return launch_word<W_SET0, 0>(z, z, z, z, bits, off, n, st);
}

ag_status kleene_dev(int kop, const uint8_t* lvalid, const uint8_t* ldata, int64_t loff,
                     const uint8_t* rvalid, const uint8_t* rdata, int64_t roff,
                     uint8_t* out_valid, uint8_t* out_data, int64_t ooff, int64_t n, cudaStream_t st) {
  if (n < 0 || loff < 0 || roff < 0 || ooff < 0) AG_FAIL(AG_ERR_INVALID, "kleene: negative length or offset");
  if (n == 0) return AG_OK;
  if (!ldata || !rdata || !out_valid || !out_data) AG_FAIL(AG_ERR_INVALID, "kleene: NULL bitmap");
  const BitmapArg lv{lvalid, loff}, ld{ldata, loff}, rv{rvalid, roff}, rd{rdata, roff};
  // two launches (validity word, data word): the two outputs may sit on different 4-byte
  // phases, and each launch owns whole aligned words of ITS output.
  switch (kop) {
    case AG_KLEENE_AND:
      AG_TRY((launch_word<W_KAND_V, 4>(lv, ld, rv, rd, out_valid, ooff, n, st)));
      return launch_word<W_KAND_D, 4>(lv, ld, rv, rd, out_data, ooff, n, st);
    case AG_KLEENE_OR:
      AG_TRY((launch_word<W_KOR_V, 4>(lv, ld, rv, rd, out_valid, ooff, n, st)));
      return launch_word<W_KOR_D, 4>(lv, ld, rv, rd, out_data, ooff, n, st);
    case AG_KLEENE_ANDNOT:
      AG_TRY((launch_word<W_KANDNOT_V, 4>(lv, ld, rv, rd, out_valid, ooff, n, st)));
      return launch_word<W_KANDNOT_D, 4>(lv, ld, rv, rd, out_data, ooff, n, st);
    default: AG_FAIL(AG_ERR_INVALID, "kleene: bad op %d", kop);
  }
}

// ---------------------------------------------------------------- popcount ---------
// CountSetBits(buf, offset, n) (bitutil.go:89-135).  Integer adds: order-free, exact.
__global__ void __launch_bounds__(kBmThreads)
popcount_kernel(const uint8_t* __restrict__ bits, int64_t off, int64_t n, unsigned long long* __restrict__ count) {
  // logical 32-bit windows of the range [off, off+n)
  const int64_t n_words = (n + 31) >> 5;
  const int64_t lo_byte = off >> 3, hi_byte = (off + n + 7) >> 3;
  const int64_t stride = (int64_t)gridDim.x * kBmThreads;
  unsigned long long c = 0;
  for (int64_t w = (int64_t)blockIdx.x * kBmThreads + threadIdx.x; w < n_words; w += stride) {
    uint32_t v = bitmap_load32(bits, off + (w << 5), lo_byte, hi_byte);
    const int64_t rem = n - (w << 5);
    if (rem < 32) v &= bit_range_mask(0, (int)rem);
    c += __popc(v);
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) c += __shfl_xor_sync(0xffffffffu, c, m);
  __shared__ unsigned long long sm[kBmThreads / 32];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
#pragma unroll
    for (int i = 0; i < kBmThreads / 32; ++i) t += sm[i];
    if (t) atomicAdd(count, t);
  }
}

ag_status bitmap_popcount_dev(const uint8_t* bits, int64_t off, int64_t n, int64_t* d_count, cudaStream_t st) {
  if (n < 0 || off < 0) AG_FAIL(AG_ERR_INVALID, "popcount: negative length or offset");
  if (!d_count) AG_FAIL(AG_ERR_INVALID, "popcount: NULL result");
  AG_CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int64_t), st));
  if (n == 0) return AG_OK;
  if (!bits) AG_FAIL(AG_ERR_INVALID, "popcount: NULL bitmap");
  const int grid = grid_for((n + 31) >> 5, kBmThreads * 4, 4);
  popcount_kernel<<<grid, kBmThreads, 0, st>>>(bits, off, n, (unsigned long long*)d_count);
  return check_launch("popcount_kernel");
}

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_bitmap_op_dev(int bitop, const uint8_t* l, int64_t loff, const uint8_t* r, int64_t roff,
                           uint8_t* out, int64_t ooff, int64_t n, ag_stream_t s) {
  AG_TRY(ensure_init());
  return bitmap_op_dev(bitop, l, loff, r, roff, out, ooff, n, resolve_stream(s));
}
ag_status ag_bitmap_copy_dev(const uint8_t* src, int64_t soff, int64_t n, uint8_t* dst, int64_t doff, ag_stream_t s) {
  AG_TRY(ensure_init());
  return bitmap_copy_dev(src, soff, n, dst, doff, false, resolve_stream(s));
}
ag_status ag_bitmap_invert_dev(const uint8_t* src, int64_t soff, int64_t n, uint8_t* dst, int64_t doff, ag_stream_t s) {
  AG_TRY(ensure_init());
  return bitmap_copy_dev(src, soff, n, dst, doff, true, resolve_stream(s));
}
ag_status ag_bitmap_set_dev(uint8_t* bits, int64_t off, int64_t n, int value, ag_stream_t s) {
  AG_TRY(ensure_init());
  return bitmap_set_dev(bits, off, n, value, resolve_stream(s));
}
ag_status ag_bitmap_popcount_dev(const uint8_t* bits, int64_t off, int64_t n, int64_t* d_count, ag_stream_t s) {
  AG_TRY(ensure_init());
  return bitmap_popcount_dev(bits, off, n, d_count, resolve_stream(s));
}
ag_status ag_kleene_dev(int kop, const uint8_t* lvalid, const uint8_t* ldata, int64_t loff,
                        const uint8_t* rvalid, const uint8_t* rdata, int64_t roff,
                        uint8_t* out_valid, uint8_t* out_data, int64_t ooff, int64_t n, ag_stream_t s) {
  AG_TRY(ensure_init());
  return kleene_dev(kop, lvalid, ldata, loff, rvalid, rdata, roff, out_valid, out_data, ooff, n, resolve_stream(s));
}

}  // extern "C"
