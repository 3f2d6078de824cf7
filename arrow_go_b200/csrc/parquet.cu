// parquet.cu — the Parquet column-decode primitives that feed the compute path (SURVEY §8f rank 4): the three SIMD
// leaf loops arrow-go links under parquet/internal, as device kernels, so a reader can decode pages straight into
// device-resident Arrow buffers ("DMA once per record batch" starts at the page, not at the array):
//   unpack32         parquet/internal/utils/_lib/bit_packing_avx2.c:1772-1879 (`unpack32_avx2`: 32 values of num_bits
//                    bits per group, LSB-first, -> uint32; Go driver bit_packing_avx2_amd64.go:34-60 and
//                    BitReader.GetBatch bit_reader.go:539-600) — dictionary indices, RLE/bit-packed hybrid runs, levels;
//   bytes_to_bools   parquet/internal/utils/_lib/unpack_bool.c:21-31 (PLAIN boolean pages -> one byte per value);
//   def levels -> validity bitmap
//                    parquet/internal/bmi/_lib/bitmap_bmi2.c:24-47 (`levels_to_bitmap`: bit i = level[i] > rhs,
//                    `extract_bits` = pext) under file/level_conversion.go:134-176 (defLevelsBatchToBitmap): without a
//                    repeated parent the validity bit of value i is def[i] >= DefLevel; with one, only the slots whose
//                    def level reaches RepeatedAncestorDefLevel produce a bit (pext = stable compaction of bits).
// Roofline: HBM streams.  unpack32 reads num_bits/8 bytes and writes 4 per value; the level conversion is compare.cu's
// int16 > scalar kernel (2 B in, 1 bit out per level) plus, for nested columns, filter.cu's boolean compaction.
#include "host_stage.cuh"

namespace ag {

constexpr int kPqThreads = 256;

// value i occupies bits [i*b, i*b + b) of the little-endian word stream.  A thread produces 4 consecutive values and
// stores them as one 128-bit vector; the <= 2 source words of a value come from aligned 32-bit loads + funnel shift.
__global__ void __launch_bounds__(kPqThreads)
unpack32_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int64_t n, int num_bits) {
  const uint32_t mask = num_bits >= 32 ? 0xffffffffu : ((1u << num_bits) - 1u);
  const int64_t nquads = n >> 2;   // n is a multiple of 32
  for (int64_t q = (int64_t)blockIdx.x * kPqThreads + threadIdx.x; q < nquads; q += (int64_t)gridDim.x * kPqThreads) {
    uint32_t v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const unsigned long long bit = (unsigned long long)(q * 4 + j) * (unsigned)num_bits;
      const int64_t w = (int64_t)(bit >> 5);
      const int sh = (int)(bit & 31);
      const uint32_t lo = in[w];
      // the second word exists whenever the value crosses a word boundary (sh + num_bits > 32), which only happens
      // inside the packed run because every 32-value group ends on a word boundary
      const uint32_t hi = (sh + num_bits > 32) ? in[w + 1] : 0u;
      v[j] = __funnelshift_r(lo, hi, sh) & mask;
    }
    __stcs(reinterpret_cast<uint4*>(out) + q, make_uint4(v[0], v[1], v[2], v[3]));
  }
}

__global__ void __launch_bounds__(kPqThreads)
bytes_to_bools_kernel(const uint8_t* __restrict__ bytes, int64_t len, uint8_t* __restrict__ out, int64_t outlen) {
  // thread = one input byte -> 8 output bytes (one 64-bit store when it fits)
  for (int64_t i = (int64_t)blockIdx.x * kPqThreads + threadIdx.x; i < len; i += (int64_t)gridDim.x * kPqThreads) {
    const unsigned b = bytes[i];
    const int64_t o = i * 8;
    if (o >= outlen) continue;
    if (o + 8 <= outlen && ((reinterpret_cast<uintptr_t>(out) + o) & 7) == 0) {
      unsigned long long v = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) v |= (unsigned long long)((b >> j) & 1u) << (8 * j);
      *reinterpret_cast<unsigned long long*>(out + o) = v;
    } else {
      for (int j = 0; j < 8 && o + j < outlen; ++j) out[o + j] = (uint8_t)((b >> j) & 1u);
    }
  }
}

// bytes_to_bools, bulk part: a thread expands 4 input bytes (one 32-bit load) into 32 output bytes (two 128-bit stores)
__global__ void __launch_bounds__(kPqThreads)
bytes_to_bools4_kernel(const uint32_t* __restrict__ in, int64_t n4, uint4* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * kPqThreads + threadIdx.x; i < n4; i += (int64_t)gridDim.x * kPqThreads) {
    const uint32_t w = __ldcs(in + i);
    uint32_t o[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {           // output word q holds bits 4q .. 4q+3 as bytes
      const uint32_t nib = (w >> (4 * q)) & 0xfu;
      o[q] = (nib & 1u) | ((nib & 2u) << 7) | ((nib & 4u) << 14) | ((nib & 8u) << 21);
    }
    __stcs(out + 2 * i, make_uint4(o[0], o[1], o[2], o[3]));
    __stcs(out + 2 * i + 1, make_uint4(o[4], o[5], o[6], o[7]));
  }
}

// flat definition levels, bulk part: bit i = level[i] > rhs for whole 256-row warp loads.  A lane reads 8 levels with one
// 128-bit load (the generic compare kernel reads 2 bytes per lane per load), four loads in flight; the 8-bit masks of four
// neighbouring lanes are merged by two shuffles into one aligned output word.
__global__ void __launch_bounds__(kPqThreads)
levels_gt_kernel(const uint4* __restrict__ lv, int64_t nvec, int rhs, uint32_t* __restrict__ out_words) {
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = ((int64_t)blockIdx.x * kPqThreads + threadIdx.x) >> 5;
  const int64_t warps = ((int64_t)gridDim.x * kPqThreads) >> 5;
  for (int64_t v0 = warp0 * 128; v0 < nvec; v0 += warps * 128) {     // nvec is a multiple of 32
    uint4 x[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) x[k] = (v0 + k * 32 < nvec) ? __ldcs(lv + v0 + k * 32 + lane) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (v0 + k * 32 >= nvec) break;     // warp-uniform
      const uint32_t wv[4] = {x[k].x, x[k].y, x[k].z, x[k].w};
      uint32_t m = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        m |= ((int)(short)(wv[j] & 0xffffu) > rhs ? 1u : 0u) << (2 * j);
        m |= ((int)(short)(wv[j] >> 16) > rhs ? 1u : 0u) << (2 * j + 1);
      }
      uint32_t v = m << (8 * (lane & 3));
      v |= __shfl_xor_sync(0xffffffffu, v, 1);
      v |= __shfl_xor_sync(0xffffffffu, v, 2);
      if ((lane & 3) == 0) out_words[((v0 + k * 32) >> 2) + (lane >> 2)] = v;
    }
  }
}

ag_status parquet_unpack32_dev(const uint32_t* in, uint32_t* out, int64_t batch_size, int num_bits, int64_t* unpacked, cudaStream_t st) {
  if (unpacked) *unpacked = 0;
  if (batch_size < 0) AG_FAIL(AG_ERR_INVALID, "unpack32: negative batch size");
  if (num_bits < 0 || num_bits > 32) AG_FAIL(AG_ERR_INVALID, "unpack32: num_bits must be 0..32 (bit_packing_avx2.c:1772)");
  const int64_t n = batch_size / 32 * 32;   // whole 32-value groups only, like the reference
  if (unpacked) *unpacked = n;
  if (n == 0) return AG_OK;
  if (!out || (num_bits > 0 && !in)) AG_FAIL(AG_ERR_INVALID, "unpack32: NULL buffer");
  if ((reinterpret_cast<uintptr_t>(out) & 15) || (reinterpret_cast<uintptr_t>(in) & 3)) AG_FAIL(AG_ERR_INVALID, "unpack32: `in` must be 4-byte and `out` 16-byte aligned");
  if (num_bits == 0) { AG_CUDA_TRY(cudaMemsetAsync(out, 0, (size_t)n * 4, st)); return AG_OK; }
  unpack32_kernel<<<grid_for(n / 4, kPqThreads * 4, 8), kPqThreads, 0, st>>>(in, out, n, num_bits);
  return check_launch("unpack32_kernel");
}

ag_status parquet_bytes_to_bools_dev(const uint8_t* bytes, int64_t len, uint8_t* out, int64_t outlen, cudaStream_t st) {
  if (len < 0 || outlen < 0) AG_FAIL(AG_ERR_INVALID, "bytes_to_bools: negative length");
  if (len == 0 || outlen == 0) return AG_OK;
  if (!bytes || !out) AG_FAIL(AG_ERR_INVALID, "bytes_to_bools: NULL buffer");
  // bulk: whole 4-byte groups whose 32 output bytes all exist, when the pointers allow 32- / 128-bit accesses
  int64_t n4 = 0;
  if ((reinterpret_cast<uintptr_t>(bytes) & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0) {
    n4 = len / 4;
    if (n4 * 32 > outlen) n4 = outlen / 32;
  }
  if (n4 > 0) {
    bytes_to_bools4_kernel<<<grid_for(n4, kPqThreads * 4, 8), kPqThreads, 0, st>>>(reinterpret_cast<const uint32_t*>(bytes), n4, reinterpret_cast<uint4*>(out));
    AG_TRY(check_launch("bytes_to_bools4_kernel"));
  }
  const int64_t rest = len - 4 * n4, rest_out = outlen - 32 * n4;
  if (rest > 0 && rest_out > 0) {
    bytes_to_bools_kernel<<<grid_for(rest, kPqThreads * 4, 8), kPqThreads, 0, st>>>(bytes + 4 * n4, rest, out + 32 * n4, rest_out);
    return check_launch("bytes_to_bools_kernel");
  }
  return AG_OK;
}

// d_counts: [0] values read (bits appended), [1] set bits (non-null values)
ag_status parquet_def_levels_to_bitmap_dev(const int16_t* levels, int64_t n, int def_level, int repeated_ancestor_def_level, uint8_t* valid_bits,
                                           int64_t valid_bits_offset, int64_t read_upper_bound, int64_t* d_counts, cudaStream_t st) {
  if (n < 0 || valid_bits_offset < 0) AG_FAIL(AG_ERR_INVALID, "def_levels_to_bitmap: negative length or offset");
  if (!d_counts) AG_FAIL(AG_ERR_INVALID, "def_levels_to_bitmap: NULL counts");
  AG_CUDA_TRY(cudaMemsetAsync(d_counts, 0, 16, st));
  if (n == 0) return AG_OK;   // valid_bits untouched (level_conversion_test.go:58-66)
  if (!levels || !valid_bits) AG_FAIL(AG_ERR_INVALID, "def_levels_to_bitmap: NULL buffer");
  const int16_t rhs = (int16_t)(def_level - 1);
  if (repeated_ancestor_def_level < 0) {
    if (n > read_upper_bound) AG_FAIL(AG_ERR_INVALID, "values read exceed upper bound");   // level_conversion.go:138-140
    // bulk: whole 256-level groups when the output starts on a 32-bit word and the levels on a 16-byte boundary
    int64_t nm = 0;
    uint8_t* first = valid_bits + (valid_bits_offset >> 3);
    if ((valid_bits_offset & 7) == 0 && (reinterpret_cast<uintptr_t>(first) & 3) == 0 && (reinterpret_cast<uintptr_t>(levels) & 15) == 0) nm = n / 256 * 256;
    if (nm > 0) {
      levels_gt_kernel<<<grid_for(nm / 8, kPqThreads * 4, 8), kPqThreads, 0, st>>>(reinterpret_cast<const uint4*>(levels), nm / 8, (int)rhs, reinterpret_cast<uint32_t*>(first));
      AG_TRY(check_launch("levels_gt_kernel"));
    }
    if (n > nm)
      AG_TRY(compare_dev(AG_TYPE_INT16, AG_CMP_GT, AG_SHAPE_AS, levels + nm, &rhs, valid_bits + ((valid_bits_offset + nm) >> 3), n - nm, (int)((valid_bits_offset + nm) & 7), st));
    const long long nn = n;
    AG_CUDA_TRY(cudaMemcpyAsync(d_counts, &nn, 8, cudaMemcpyHostToDevice, st));
    return bitmap_popcount_dev(valid_bits, valid_bits_offset, n, d_counts + 1, st);
  }
  // repeated parent: defined = level > DefLevel-1, present = level > RepeatedAncestorDefLevel-1; the output bits are the
  // defined bits of the present slots, in order (ExtractBits = pext, level_conversion.go:147-158)
  const int16_t rhs2 = (int16_t)(repeated_ancestor_def_level - 1);
  const size_t bm = (size_t)((n + 31) / 32) * 4 + 64;
  uint8_t* tmp = nullptr;
  AG_TRY(dev_alloc_async((void**)&tmp, 3 * bm, st));
  uint8_t *defined = tmp, *present = tmp + bm, *packed = tmp + 2 * bm;
  ag_status rc = AG_OK;
  do {
    if ((rc = compare_dev(AG_TYPE_INT16, AG_CMP_GT, AG_SHAPE_AS, levels, &rhs, defined, n, 0, st)) != AG_OK) break;
    if ((rc = compare_dev(AG_TYPE_INT16, AG_CMP_GT, AG_SHAPE_AS, levels, &rhs2, present, n, 0, st)) != AG_OK) break;
    if (const cudaError_t e = cudaMemsetAsync(packed, 0, bm, st)) { rc = cuda_fail(e, "memset", __FILE__, __LINE__); break; }
    if ((rc = filter_primitive_dev(1, defined, nullptr, 0, present, nullptr, 0, n, AG_DROP_NULLS, packed, nullptr, n, d_counts, st)) != AG_OK) break;
    // the selected count is only known on the device: copy min(count, n) bits — bits past the count are zero in `packed`
    // and the caller's bitmap beyond values_read is unspecified (FirstTimeBitmapWriter), so copy all n candidate bits
    if ((rc = bitmap_copy_dev(packed, 0, n, valid_bits, valid_bits_offset, false, st)) != AG_OK) break;
    rc = bitmap_popcount_dev(packed, 0, n, d_counts + 1, st);
  } while (0);
  cudaFreeAsync(tmp, st);
  return rc;
}

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_parquet_unpack32_dev(const uint32_t* d_in, uint32_t* d_out, int64_t batch_size, int num_bits, int64_t* unpacked, ag_stream_t s) {
  AG_TRY(ensure_init());
  return parquet_unpack32_dev(d_in, d_out, batch_size, num_bits, unpacked, resolve_stream(s));
}
ag_status ag_parquet_bytes_to_bools_dev(const uint8_t* d_bytes, int64_t len, uint8_t* d_out, int64_t outlen, ag_stream_t s) {
  AG_TRY(ensure_init());
  return parquet_bytes_to_bools_dev(d_bytes, len, d_out, outlen, resolve_stream(s));
}
ag_status ag_parquet_def_levels_to_bitmap_dev(const int16_t* d_def_levels, int64_t n, int def_level, int repeated_ancestor_def_level,
                                              uint8_t* d_valid_bits, int64_t valid_bits_offset, int64_t read_upper_bound, int64_t* d_counts,
                                              ag_stream_t s) {
  AG_TRY(ensure_init());
  return parquet_def_levels_to_bitmap_dev(d_def_levels, n, def_level, repeated_ancestor_def_level, d_valid_bits, valid_bits_offset, read_upper_bound,
                                          d_counts, resolve_stream(s));
}

// host-pointer flavours: upload, decode, download (synchronous)
ag_status ag_parquet_unpack32(const uint32_t* in, uint32_t* out, int64_t batch_size, int num_bits, int64_t* unpacked) {
  AG_TRY(ensure_init());
  if (unpacked) *unpacked = 0;
  if (batch_size < 0 || num_bits < 0 || num_bits > 32) AG_FAIL(AG_ERR_INVALID, "unpack32: bad batch size / num_bits");
  const int64_t n = batch_size / 32 * 32;
  if (n == 0) return AG_OK;
  if (!out || (num_bits > 0 && !in)) AG_FAIL(AG_ERR_INVALID, "unpack32: NULL buffer");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  const size_t in_bytes = (size_t)n * num_bits / 8;
  uint32_t *din, *dout;
  AG_TRY(t.alloc_t(&din, in_bytes));
  AG_TRY(t.alloc_t(&dout, (size_t)n * 4));
  AG_TRY(h2d(din, in, in_bytes, cs));
  AG_TRY(parquet_unpack32_dev(din, dout, n, num_bits, unpacked, cs));
  AG_TRY(d2h(out, dout, (size_t)n * 4, cs));
  return sync(cs);
}

ag_status ag_parquet_bytes_to_bools(const uint8_t* bytes, int64_t len, uint8_t* out, int64_t outlen) {
  AG_TRY(ensure_init());
  if (len < 0 || outlen < 0) AG_FAIL(AG_ERR_INVALID, "bytes_to_bools: negative length");
  if (len == 0 || outlen == 0) return AG_OK;
  if (!bytes || !out) AG_FAIL(AG_ERR_INVALID, "bytes_to_bools: NULL buffer");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  const int64_t produced = len * 8 < outlen ? len * 8 : outlen;
  uint8_t *din, *dout;
  AG_TRY(t.alloc_t(&din, (size_t)len));
  AG_TRY(t.alloc_t(&dout, (size_t)produced));
  AG_TRY(h2d(din, bytes, (size_t)len, cs));
  AG_TRY(parquet_bytes_to_bools_dev(din, len, dout, produced, cs));
  AG_TRY(d2h(out, dout, (size_t)produced, cs));
  return sync(cs);
}

ag_status ag_parquet_def_levels_to_bitmap(const int16_t* def_levels, int64_t n, int def_level, int repeated_ancestor_def_level, uint8_t* valid_bits,
                                          int64_t valid_bits_offset, int64_t read_upper_bound, int64_t* values_read, int64_t* null_count) {
  AG_TRY(ensure_init());
  if (values_read) *values_read = 0;
  if (n < 0 || valid_bits_offset < 0) AG_FAIL(AG_ERR_INVALID, "def_levels_to_bitmap: negative length or offset");
  if (n == 0) return AG_OK;
  if (!def_levels || !valid_bits) AG_FAIL(AG_ERR_INVALID, "def_levels_to_bitmap: NULL buffer");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  int16_t* dl; int64_t* dc;
  AG_TRY(t.alloc_t(&dl, (size_t)n * 2));
  AG_TRY(h2d(dl, def_levels, (size_t)n * 2, cs));
  // both device paths write all n bits of [offset, offset + n), so only the edge bytes' neighbours need staging
  OutBitmap ob;
  AG_TRY(ob.stage(t, valid_bits, valid_bits_offset, n));
  AG_TRY(t.alloc_t(&dc, 2 * sizeof(int64_t)));
  AG_TRY(parquet_def_levels_to_bitmap_dev(dl, n, def_level, repeated_ancestor_def_level, ob.d, ob.doff, read_upper_bound, dc, cs));
  int64_t counts[2] = {0, 0};
  AG_TRY(d2h(counts, dc, sizeof(counts), cs));
  AG_TRY(sync(cs));
  if (repeated_ancestor_def_level >= 0 && counts[0] > read_upper_bound) AG_FAIL(AG_ERR_INVALID, "values read exceeded upper bound");
  // bring back only the bytes that hold the values_read bits appended at valid_bits_offset
  AG_TRY(d2h(valid_bits + ob.b0, ob.d, (size_t)(bytes_for_bits(valid_bits_offset + counts[0]) - ob.b0), cs));
  AG_TRY(sync(cs));
  if (values_read) *values_read = counts[0];
  if (null_count) *null_count += counts[0] - counts[1];
  return AG_OK;
}

}  // extern "C"
