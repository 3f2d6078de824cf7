// common.cuh — runtime internals shared by every translation unit of libarrowgpu.so.
// Not part of the public ABI (see include/arrowgpu.h).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <stdio.h>
#include <atomic>
#include <mutex>
#include <type_traits>

#include "../../include/arrowgpu.h"

namespace ag {

// ---------------------------------------------------------------- errors ----------
void set_error(const char* fmt, ...);
ag_status cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define AG_CUDA_TRY(expr)                                                        \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess) return ::ag::cuda_fail(_e, #expr, __FILE__, __LINE__); \
  } while (0)

#define AG_TRY(expr)                     \
  do {                                   \
    ag_status _s = (expr);               \
    if (_s != AG_OK) return _s;          \
  } while (0)

#define AG_FAIL(code, ...)               \
  do {                                   \
    ::ag::set_error(__VA_ARGS__);        \
    return (code);                       \
  } while (0)

// ---------------------------------------------------------------- runtime ---------
// Per-stream scratch: kernels on one stream are serialised by the stream, so one
// workspace per stream is race-free without stream-ordered allocation per call.
struct Workspace {
  // fixed small area
  void* partials;        // kMaxPartials * 16 bytes (sum partials, per-block counters)
  unsigned* ticket;      // last-block-done tickets; kernels leave them at 0
  int64_t* scalars;      // 16 x int64 device scalars (counts, error words)
  // growable area (decoupled look-back tile status for filter / take_indices)
  unsigned long long* tile_status;
  size_t tile_status_cap;  // in elements
  // pinned host mirror of `scalars` for cheap readback
  int64_t* h_scalars;
  // Held by an entry point from get_workspace until its last launch is enqueued: two threads that share a stream
  // (e.g. both pass NULL) may interleave their CALLS but never the launches of one call with another's, so ticket /
  // scalar slots / tile status are always used by one kernel sequence at a time (the stream orders the rest).
  std::mutex* seq_mu;
};
struct WorkspaceLock {
  std::unique_lock<std::mutex> lk;
  explicit WorkspaceLock(Workspace* ws) : lk(*ws->seq_mu) {}
};

constexpr int kMaxPartials = 4096;

ag_status ensure_init();
int sm_count();
cudaStream_t resolve_stream(ag_stream_t s);
int current_device();
int device_count();
ag_status get_workspace(cudaStream_t s, Workspace** ws);
ag_status ensure_tile_status(Workspace* ws, size_t n_tiles, cudaStream_t s);
void count_launch(int n = 1);
ag_status check_launch(const char* what);

// Pooled streams for the synchronous host-pointer entry points (each call owns its streams
// for its duration, so concurrent cgo callers never share a stream or a workspace).
ag_status acquire_call_stream(cudaStream_t* st);
void release_call_stream(cudaStream_t st);
struct CallStream {
  cudaStream_t st = nullptr;
  ag_status acquire() { return acquire_call_stream(&st); }
  ~CallStream() { if (st) release_call_stream(st); }
  operator cudaStream_t() const { return st; }
};

// Device temp allocation (stream-ordered pool).
ag_status dev_alloc_async(void** p, size_t nbytes, cudaStream_t s);
ag_status dev_free_async(void* p, cudaStream_t s);

// ---------------------------------------------------------------- device flavours used across files ----
// The stream-ordered implementations behind the *_dev entry points that the host flavours (host_api.cu) and other
// device code (parquet.cu, hash.cu) call.
// elementwise.cu
ag_status arith_binary_dev(int type, int8_t op, int shape, const void* l, const void* r, void* out, int64_t n, cudaStream_t st);
ag_status arith_unary_same_dev(int type, int8_t op, const void* in, void* out, int64_t n, cudaStream_t st);
ag_status arith_unary_diff_dev(int itype, int otype, int8_t op, const void* in, void* out, int64_t n, cudaStream_t st);
ag_status arith_checked_dev(int type, int8_t op, int shape, const void* l, const uint8_t* lvalid, int64_t loff,
                            const void* r, const uint8_t* rvalid, int64_t roff, void* out, int64_t n, int64_t* d_first_bad, cudaStream_t st);
ag_status error_word_reset(int64_t* d_word, cudaStream_t st);
ag_status arith_unary_checked_dev(int type, int8_t op, const void* in, void* out, int64_t n, int64_t* d_first_bad, cudaStream_t st);
// cast.cu
ag_status cast_numeric_dev(int itype, int otype, const void* in, const uint8_t* valid, int64_t voff, void* out, int64_t n,
                           int allow_int_overflow, int allow_float_truncate, int64_t* first_bad, int64_t row_base, cudaStream_t st);
// scan.cu
ag_status cumulative_sum_dev(int type, const void* in, const uint8_t* valid, int64_t voff, int64_t n, int skip_nulls, int checked,
                             void* out, uint8_t* out_valid, int64_t ooff, void* d_state, int64_t* d_first_bad, cudaStream_t st);
ag_status cumulative_sum_state_init(void* d_state, int type, const void* start_host, cudaStream_t st);
// compare.cu
ag_status compare_dev(int type, int cmp, int shape, const void* l, const void* r, uint8_t* out, int64_t n, int off, cudaStream_t st);
// bitmap.cu
ag_status bitmap_op_dev(int bitop, const uint8_t* l, int64_t loff, const uint8_t* r, int64_t roff, uint8_t* out, int64_t ooff, int64_t n, cudaStream_t st);
ag_status bitmap_copy_dev(const uint8_t* src, int64_t soff, int64_t n, uint8_t* dst, int64_t doff, bool invert, cudaStream_t st);
ag_status bitmap_set_dev(uint8_t* bits, int64_t off, int64_t n, int value, cudaStream_t st);
ag_status bitmap_popcount_dev(const uint8_t* bits, int64_t off, int64_t n, int64_t* d_count, cudaStream_t st);
ag_status kleene_dev(int kop, const uint8_t* lvalid, const uint8_t* ldata, int64_t loff, const uint8_t* rvalid, const uint8_t* rdata,
                     int64_t roff, uint8_t* out_valid, uint8_t* out_data, int64_t ooff, int64_t n, cudaStream_t st);
// filter.cu
ag_status filter_output_size_dev(const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n, int null_selection, int64_t* d_out_len, cudaStream_t st);
ag_status filter_primitive_dev(int bit_width, const void* vals, const uint8_t* vvalid, int64_t voff, const uint8_t* mask, const uint8_t* mvalid,
                               int64_t moff, int64_t n, int null_selection, void* out, uint8_t* out_valid, int64_t capacity, int64_t* d_out_len, cudaStream_t st);
ag_status take_indices_dev(int index_width, const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n, int null_selection,
                           void* out_idx, uint8_t* out_valid, int64_t capacity, int64_t* d_out_len, cudaStream_t st);
// hash.cu
ag_status is_in_dev(int bit_width, const void* vals, const uint8_t* valid, int64_t off, int64_t n, const void* set, const uint8_t* set_valid,
                    int64_t set_off, int64_t set_n, int null_behavior, uint8_t* out_data, uint8_t* out_valid, int64_t* d_null_count, cudaStream_t st);
ag_status unique_dev(int bit_width, const void* vals, const uint8_t* valid, int64_t off, int64_t n, void* out, uint8_t* out_valid, int64_t capacity,
                     int64_t* d_out_len, cudaStream_t st);
ag_status dictionary_encode_dev(int bit_width, const ag_dict_chunk* chunks, int64_t n_chunks, int null_encoding, void* dict,
                                uint8_t* dict_valid, int64_t* d_counts, cudaStream_t st);
// A BYTE_ARRAY dictionary call after pq_encode.cu's checking pass, which counts the valid slots of every kBaTile-slot
// tile of every chunk.  Device tables.
constexpr int kBaTile = 1024;              // slots per tile of every BYTE_ARRAY pass
struct BaDictPlan {
  int ow;                                  // offset width, 4 or 8
  const ag_pq_ba_chunk* chunks;            // [n_chunks] (set by ba_dict_encode_dev from h_chunks)
  const int64_t* row_base;                 // [n_chunks + 1] the first slot of every chunk in the call's numbering (ditto)
  const int64_t* tile_base;                // [n_chunks + 1] the first tile of every chunk
  const unsigned long long* tile_cnt;      // tile t of chunk c, at [t + c]: the chunk's valid slots before the tile
  const int64_t* dense;                    // [n_chunks] the call's valid slots before every chunk
  int64_t n_chunks, n_tiles, slots, valid;
};
// the dictionary kernels of ag_parquet_byte_array_dict_encode_dev; h_chunks and marks are host arrays
ag_status ba_dict_encode_dev(BaDictPlan p, const ag_pq_ba_chunk* h_chunks, const int64_t* marks, int64_t n_marks, uint32_t* indices,
                             int64_t* mark_counts, int64_t* counts, cudaStream_t st);
// run_end.cu
ag_status run_end_count_dev(int type, const void* vals, const uint8_t* valid, int64_t offset, int64_t n, int64_t* d_counts, cudaStream_t st);
ag_status run_end_encode_dev(int type, int run_end_type, const void* vals, const uint8_t* valid, int64_t offset, int64_t n,
                             void* run_ends, void* out, uint8_t* out_valid, int64_t capacity, int64_t* d_counts, cudaStream_t st);
ag_status run_end_decode_dev(int type, int run_end_type, const void* run_ends, int64_t n_runs, const void* vals, const uint8_t* valid,
                             int64_t values_offset, int64_t offset, int64_t length, void* out, uint8_t* out_valid,
                             int64_t* d_null_count, int64_t* d_error_word, cudaStream_t st);
// sort.cu
ag_status sort_indices_dev(int type, const void* vals, const uint8_t* valid, int64_t voff, int64_t n, int order, int null_placement,
                           uint64_t* d_out, int64_t* nulls_out, int64_t* nans_out, cudaStream_t st);
// argument checks of sort_indices_keys_dev (no device work)
ag_status sort_indices_keys_check(int nkeys, const ag_sort_key* keys, int64_t n);
// One column's chunk list against its row count: the list, each chunk's offset, length and values, the sum of the
// lengths.  Messages start with "<who> <j>: "; the row-count one ends with "does not match <rows_name> <nrows>".
ag_status check_chunk_list(const char* who, int j, int nchunks, const ag_sort_chunk* chunks, int64_t nrows, const char* rows_name);
ag_status sort_indices_keys_dev(int nkeys, const ag_sort_key* keys, int64_t n, uint64_t* d_out, cudaStream_t st);
// take.cu
ag_status take_primitive_dev(int bit_width, const void* vals, const uint8_t* vvalid, int64_t voff, int64_t vlen, int idx_width, int idx_signed,
                             const void* idx, const uint8_t* ivalid, int64_t ioff, int64_t n, int bounds_check, void* out, uint8_t* out_valid,
                             int64_t* d_bad_pos, cudaStream_t st);
// take_columns.cu: descriptor checks (no device work) and the gather
ag_status take_columns_check(int ncols, const ag_take_column* cols, int64_t nrows, int idx_width, int64_t idx_offset, int64_t n);
ag_status take_columns_dev(int ncols, const ag_take_column* cols, int64_t nrows, int idx_width, int idx_signed, const void* idx,
                           const uint8_t* idx_valid, int64_t idx_offset, int64_t n, int bounds_check, int64_t* d_bad_pos, cudaStream_t st);
// expr.cu: the checks of the program and its spans (no device work), and the checks followed by one launch
ag_status eval_program_check(const ag_expr_program* prog, int64_t n_spans, const ag_sort_chunk* spans);
ag_status eval_program_dev(const ag_expr_program* prog, int64_t n_spans, const ag_sort_chunk* spans, void* out, uint8_t* out_valid,
                           int64_t* d_error_word, cudaStream_t st);

// ---------------------------------------------------------------- cross-GPU exchange (comm.cu, reduce.cu) ----
struct alignas(32) MailSlot { unsigned long long flag; unsigned long long pad; unsigned long long s; unsigned long long c; };
struct SumExchange {
  MailSlot* const* peers;   // device array [world]: base of every rank's mailbox as addressable from this device
  MailSlot* local;          // this rank's mailbox
  int world, rank;
  unsigned long long epoch; // >= 1, same value on every rank for one collective
};
ag_status comm_next_exchange(ag_comm_t comm, SumExchange* x);   // bumps the communicator's epoch
ag_status comm_nccl_allreduce_sum_i64(ag_comm_t comm, void* d_buf, size_t count, cudaStream_t st);

// ---------------------------------------------------------------- type helpers ----
inline int type_width(int type) {
  switch (type) {
    case AG_TYPE_UINT8: case AG_TYPE_INT8: return 1;
    case AG_TYPE_UINT16: case AG_TYPE_INT16: return 2;
    case AG_TYPE_UINT32: case AG_TYPE_INT32: case AG_TYPE_FLOAT32: return 4;
    case AG_TYPE_UINT64: case AG_TYPE_INT64: case AG_TYPE_FLOAT64: return 8;
    default: return 0;
  }
}
inline bool type_is_signed_int(int type) {
  return type == AG_TYPE_INT8 || type == AG_TYPE_INT16 || type == AG_TYPE_INT32 || type == AG_TYPE_INT64;
}
inline bool type_is_unsigned_int(int type) {
  return type == AG_TYPE_UINT8 || type == AG_TYPE_UINT16 || type == AG_TYPE_UINT32 || type == AG_TYPE_UINT64;
}
inline bool type_is_float(int type) { return type == AG_TYPE_FLOAT32 || type == AG_TYPE_FLOAT64; }

// ---------------------------------------------------------------- kernel dispatch ----
// How an ABI argument picks a kernel instantiation.  Each visitor calls `f` with a TypeTag<T> (visit_shape: a
// std::integral_constant) and returns what `f` returns; a value it does not map goes to `unsupported()` instead,
// so the caller keeps its own status and message.  A caller that takes a subset (integers only, say) checks before
// the call or branches with `if constexpr` inside `f`; the branch also keeps kernels of the other types from
// being instantiated.
template <typename T> struct TypeTag { using type = T; };

// Exact type: each of the 10 numeric type ids as its own C++ type.
template <typename F, typename U>
inline ag_status visit_type(int type, F&& f, U&& unsupported) {
  switch (type) {
    case AG_TYPE_UINT8: return f(TypeTag<uint8_t>{});
    case AG_TYPE_INT8: return f(TypeTag<int8_t>{});
    case AG_TYPE_UINT16: return f(TypeTag<uint16_t>{});
    case AG_TYPE_INT16: return f(TypeTag<int16_t>{});
    case AG_TYPE_UINT32: return f(TypeTag<uint32_t>{});
    case AG_TYPE_INT32: return f(TypeTag<int32_t>{});
    case AG_TYPE_UINT64: return f(TypeTag<unsigned long long>{});
    case AG_TYPE_INT64: return f(TypeTag<long long>{});
    case AG_TYPE_FLOAT32: return f(TypeTag<float>{});
    case AG_TYPE_FLOAT64: return f(TypeTag<double>{});
    default: return unsupported();
  }
}

// Storage type: signed and unsigned integers of one width share the unsigned type; floats stay as they are.  For
// ops whose result bits do not depend on signedness: two's-complement add/sub/mul (base_arithmetic.cc:121-148 makes
// the same move for Multiply), bitwise ops, == and !=.
template <typename F, typename U>
inline ag_status visit_storage_type(int type, F&& f, U&& unsupported) {
  switch (type) {
    case AG_TYPE_UINT8: case AG_TYPE_INT8: return f(TypeTag<uint8_t>{});
    case AG_TYPE_UINT16: case AG_TYPE_INT16: return f(TypeTag<uint16_t>{});
    case AG_TYPE_UINT32: case AG_TYPE_INT32: return f(TypeTag<uint32_t>{});
    case AG_TYPE_UINT64: case AG_TYPE_INT64: return f(TypeTag<unsigned long long>{});
    case AG_TYPE_FLOAT32: return f(TypeTag<float>{});
    case AG_TYPE_FLOAT64: return f(TypeTag<double>{});
    default: return unsupported();
  }
}

// Width: a value or index width of 8/16/32/64 bits as the unsigned integer of that size.
template <typename F, typename U>
inline ag_status visit_width(int bits, F&& f, U&& unsupported) {
  switch (bits) {
    case 8: return f(TypeTag<uint8_t>{});
    case 16: return f(TypeTag<uint16_t>{});
    case 32: return f(TypeTag<uint32_t>{});
    case 64: return f(TypeTag<unsigned long long>{});
    default: return unsupported();
  }
}

// Operand shape of a binary op: AG_SHAPE_AA / AS / SA as a compile-time constant.
template <typename F, typename U>
inline ag_status visit_shape(int shape, F&& f, U&& unsupported) {
  switch (shape) {
    case AG_SHAPE_AA: return f(std::integral_constant<int, AG_SHAPE_AA>{});
    case AG_SHAPE_AS: return f(std::integral_constant<int, AG_SHAPE_AS>{});
    case AG_SHAPE_SA: return f(std::integral_constant<int, AG_SHAPE_SA>{});
    default: return unsupported();
  }
}

inline int64_t bytes_for_bits(int64_t nbits) { return (nbits + 7) >> 3; }

int blocks_per_sm(const void* kernel, int threads);
// Opt a kernel into `bytes` of dynamic shared memory on the calling thread's device, once per device
// (`done` = the caller's per-instantiation bit set; the attribute is per function per context).
static inline ag_status ensure_dynamic_smem(const void* kernel, int bytes, std::atomic<unsigned>* done) {
  const unsigned bit = 1u << (current_device() & 31);
  if (done->load(std::memory_order_acquire) & bit) return AG_OK;
  AG_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done->fetch_or(bit, std::memory_order_release);
  return AG_OK;
}
// One-wave grid for a grid-stride kernel: min(blocks needed, SMs x resident blocks per SM).
template <typename K>
inline int grid_one_wave(K kernel, int threads, int64_t blocks_needed) {
  const int64_t cap = (int64_t)sm_count() * blocks_per_sm(reinterpret_cast<const void*>(kernel), threads);
  if (blocks_needed < 1) blocks_needed = 1;
  return (int)(blocks_needed < cap ? blocks_needed : cap);
}

// Grid sizing: persistent-style grids are multiples of the SM count.
inline int grid_for(int64_t work_items, int items_per_block, int blocks_per_sm) {
  int64_t want = (work_items + items_per_block - 1) / items_per_block;
  int64_t cap = (int64_t)sm_count() * blocks_per_sm;
  if (want < 1) want = 1;
  return (int)(want < cap ? want : cap);
}

// ---------------------------------------------------------------- device helpers --
#ifdef __CUDACC__

// Read 32 bits of an LSB-first bitmap starting at absolute bit position `bit`
// (relative to byte pointer `base`), touching only bytes in [lo_byte, hi_byte).
// Bits that fall outside are returned as 0.  Interior windows are two aligned 32-bit loads and
// a funnel shift; windows that touch the ends of the range go through the (out-of-line) byte-wise
// path so that no byte outside the caller's buffer is ever read.
static __device__ __noinline__ uint32_t bitmap_load32_edge(const uint8_t* abase, int64_t w, int sh, int64_t lo, int64_t hi) {
  uint32_t words[2] = {0u, 0u};
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int64_t b0 = (w + j) * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int64_t b = b0 + k;
      if (b >= lo && b < hi) words[j] |= (uint32_t)abase[b] << (8 * k);
    }
  }
  return sh ? __funnelshift_r(words[0], words[1], sh) : words[0];
}

__device__ __forceinline__ uint32_t bitmap_load32(const uint8_t* __restrict__ base, int64_t bit,
                                                  int64_t lo_byte, int64_t hi_byte) {
  const uintptr_t addr = reinterpret_cast<uintptr_t>(base);
  const int64_t mis = (int64_t)(addr & 3);       // base = abase + mis, abase 4-byte aligned
  const uint8_t* abase = base - mis;
  const int64_t abit = bit + mis * 8;            // bit position relative to abase (floor semantics for negatives)
  const int64_t w = abit >> 5;
  const int sh = (int)(abit & 31);
  const int64_t lo = lo_byte + mis, hi = hi_byte + mis;  // valid byte range relative to abase
  const int64_t b0 = w * 4;
  if (b0 >= lo && b0 + 8 <= hi) {
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(abase + b0);
    const uint32_t w0 = wp[0];
    return sh ? __funnelshift_r(w0, wp[1], sh) : w0;
  }
  return bitmap_load32_edge(abase, w, sh, lo, hi);
}

// mask with bits [a, b) set, 0 <= a <= b <= 32
__device__ __forceinline__ uint32_t bit_range_mask(int a, int b) {
  const uint32_t hi = (b >= 32) ? 0xffffffffu : ((1u << b) - 1u);
  const uint32_t lo = (a >= 32) ? 0xffffffffu : ((1u << a) - 1u);
  return hi & ~lo;
}

// Store the bits of `value` selected by `mask` into the aligned 32-bit word at `wp`,
// preserving every other bit and never touching a byte whose 8 mask bits are all zero
// (edge words of a bitmap may extend past the caller's buffer).
__device__ __forceinline__ void bitmap_store32_masked(uint32_t* wp, uint32_t value, uint32_t mask) {
  if (mask == 0xffffffffu) { *wp = value; return; }
  uint8_t* bp = reinterpret_cast<uint8_t*>(wp);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t m = (mask >> (8 * k)) & 0xffu;
    if (m == 0) continue;
    const uint32_t v = (value >> (8 * k)) & 0xffu;
    if (m == 0xffu) bp[k] = (uint8_t)v;
    else bp[k] = (uint8_t)((bp[k] & ~m) | (v & m));
  }
}

__device__ __forceinline__ bool bit_is_set(const uint8_t* __restrict__ bits, int64_t i) {
  return (bits[i >> 3] >> (i & 7)) & 1;
}

// Lower the warp's lowest failing row into the error word: a shuffle-xor minimum, then one atomicMin from lane 0 when
// some lane saw a failure.  Every lane of the warp calls it.
__device__ __forceinline__ void lower_error_row(long long my_bad, long long* word) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    const long long o = __shfl_xor_sync(0xffffffffu, my_bad, m);
    my_bad = o < my_bad ? o : my_bad;
  }
  if ((threadIdx.x & 31) == 0 && my_bad != AG_NO_ERROR_POS) atomicMin(word, my_bad);
}

// Take's bounds rule for a valid index slot (I: the unsigned type of the index width): out of bounds when the index is
// negative (a signed index type with the sign bit set) or, read as unsigned, >= rows.  take_partition_kernel computes
// the same rule as one unsigned compare against min(rows, 2^(bits-1)) for signed indices.  The operands are references
// so that the kernels keep their register counts: by value, take_kernel needs up to 11 more registers.
// take_columns_kernel spells the rule out: through this helper nvcc reorders its gathers.
template <typename I>
__device__ __forceinline__ bool take_index_oob(const I& ix, const unsigned long long& rows, const int& idx_signed) {
  constexpr I kSignBit = (I)((I)1 << (sizeof(I) * 8 - 1));
  return (idx_signed && (ix & kSignBit)) || (unsigned long long)ix >= rows;
}

// Lane 0 stores word w (a warp's ballot) of an output bitmap of n bits: whole inside the bitmap, masked to the bits
// below n in the last word, not at all past it.
__device__ __forceinline__ void store_valid_word(uint32_t* out_valid, int64_t w, uint32_t bits, int64_t n, int lane) {
  const int64_t rem = n - (w << 5);
  if (lane == 0 && rem > 0) {
    if (rem >= 32) out_valid[w] = bits;
    else bitmap_store32_masked(out_valid + w, bits, bit_range_mask(0, (int)rem));
  }
}

// The same for a boolean output: the data word and, when out_valid is set, the validity word, under one mask.
__device__ __forceinline__ void store_bool_words(uint32_t* out, uint32_t* out_valid, int64_t w, uint32_t dbits, uint32_t vbits,
                                                 int64_t n, int lane) {
  const int64_t rem = n - (w << 5);
  if (lane == 0 && rem > 0) {
    const uint32_t m = rem >= 32 ? 0xffffffffu : bit_range_mask(0, (int)rem);
    bitmap_store32_masked(out + w, dbits, m);
    if (out_valid) bitmap_store32_masked(out_valid + w, vbits, m);
  }
}

// last page p with base[p] <= tile (pages with no tiles share their base with the next page)
__device__ __forceinline__ int64_t find_page(const int64_t* base, int64_t n_pages, int64_t tile) {
  int64_t lo = 0, hi = n_pages - 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (base[mid] <= tile) lo = mid; else hi = mid - 1;
  }
  return lo;
}

using u128 = unsigned __int128;

__device__ __forceinline__ u128 ld16(const uint8_t* p) {
  const uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
  return (u128)v.x | (u128)v.y << 32 | (u128)v.z << 64 | (u128)v.w << 96;
}

// bytes p[0, k), 1 <= k <= 16, in the low bytes: one or two aligned 16-byte loads shifted into place, touching only
// the aligned words that hold those bytes
__device__ __forceinline__ u128 window(const uint8_t* p, int k) {
  const int sh = (int)(reinterpret_cast<uintptr_t>(p) & 15);
  const uint8_t* a = p - sh;
  u128 w = ld16(a) >> (8 * sh);
  if (sh + k > 16) w |= ld16(a + 16) << (8 * (16 - sh));
  return k == 16 ? w : w & (((u128)1 << (8 * k)) - 1);
}

__device__ __forceinline__ uint64_t mix64(uint64_t z) {  // splitmix64 finaliser
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

#endif  // __CUDACC__

}  // namespace ag
