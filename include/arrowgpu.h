/*
 * arrowgpu.h — C ABI of the H100 (sm_90a) implementation of arrow-go's vectorised
 * columnar compute hot path.
 *
 * This header is the drop-in boundary: every entry point replaces one native
 * (c2goasm) inner loop or one pure-Go kernel body of the reference, and is what a
 * cgo package inside arrow-go would bind (see INTEGRATION.md for the Go side).
 * Reference citations are relative to the arrow-go tree (commit b3dacd2a).
 *
 * Conventions
 *   - Plain pointers and sizes only.  No CUDA or torch types appear here.
 *   - Every function returns an ag_status; AG_OK == 0.  ag_last_error() returns the
 *     calling thread's last message.  Status codes map 1:1 onto arrow-go's error
 *     sentinels (arrow/errors.go:21-28).
 *   - Two flavours of every compute entry point:
 *       ag_xxx(...)      HOST pointers.  Synchronous.  The library stages the
 *                        buffers to HBM (pinned, chunked, full-duplex), runs the
 *                        kernel(s) and copies the result back.  This is the form a
 *                        per-span exec.ArrayKernelExec binds.
 *       ag_xxx_dev(...)  DEVICE pointers + a stream.  Asynchronous.  Used when a
 *                        record batch has been uploaded once (ag_upload) and many
 *                        kernels run over it before anything is downloaded.
 *   - `type` arguments are arrow.Type ids (arrow/datatype.go:36-72 ==
 *     kernels/_lib/types.h:20-34); `op` arguments are kernels.ArithmeticOp values
 *     (arrow/compute/internal/kernels/base_arithmetic.go:37-82 ==
 *     _lib/base_arithmetic.cc:31-74).
 *   - Bitmaps are Arrow LSB-first bitmaps addressed by (byte pointer, bit offset).
 *     Bits outside [offset, offset+length) are never modified.
 *   - Value pointers only need element alignment (a slice start is only
 *     element-aligned); 16-byte aligned inputs take the vectorised path.
 *   - All entry points are thread-safe and re-entrant (cgo calls arrive on arbitrary
 *     OS threads, arrow/compute/exec.go:164-170).
 *   - There is NO CPU fallback: without a usable sm_90 device every compute entry
 *     point returns AG_ERR_CUDA.
 */
#ifndef ARROWGPU_H
#define ARROWGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes (arrow/errors.go:21-28) --------------------------------------- */
typedef int ag_status;
#define AG_OK                   0
#define AG_ERR_INVALID          1 /* arrow.ErrInvalid: overflow, divide by zero, length mismatch, bad argument */
#define AG_ERR_INDEX            2 /* arrow.ErrIndex: take index out of bounds */
#define AG_ERR_NOT_IMPLEMENTED  3 /* arrow.ErrNotImplemented */
#define AG_ERR_TYPE             4 /* arrow.ErrType */
#define AG_ERR_CUDA             5 /* device / driver failure (no sentinel in arrow-go; surfaces as ErrInvalid) */
#define AG_ERR_OOM              6 /* device or pinned allocation failed */

/* ---- arrow.Type ids that cross the boundary (arrow/datatype.go:36-72) ----------- */
#define AG_TYPE_NULL     0
#define AG_TYPE_BOOL     1
#define AG_TYPE_UINT8    2
#define AG_TYPE_INT8     3
#define AG_TYPE_UINT16   4
#define AG_TYPE_INT16    5
#define AG_TYPE_UINT32   6
#define AG_TYPE_INT32    7
#define AG_TYPE_UINT64   8
#define AG_TYPE_INT64    9
#define AG_TYPE_FLOAT16 10
#define AG_TYPE_FLOAT32 11
#define AG_TYPE_FLOAT64 12

/* ---- kernels.ArithmeticOp (base_arithmetic.go:37-82) ----------------------------- */
#define AG_OP_ADD             0
#define AG_OP_SUB             1
#define AG_OP_MUL             2
#define AG_OP_DIV             3
#define AG_OP_ABS             4
#define AG_OP_NEGATE          5
#define AG_OP_SIGN           20
#define AG_OP_ADD_CHECKED    21
#define AG_OP_SUB_CHECKED    22
#define AG_OP_MUL_CHECKED    23
#define AG_OP_DIV_CHECKED    24
#define AG_OP_ABS_CHECKED    25
#define AG_OP_NEGATE_CHECKED 26
/* Not ArithmeticOp values: the reference keeps these in separate enums (BitwiseOp scalar_arithmetic.go:183-189,
 * ShiftDir :286-291); one op space here so that they ride the same entry points.
 *   BIT_AND / BIT_OR / BIT_XOR: ag_arith_binary* on the integer types (every slot, like a3: bitwiseKernelOp :191-243
 *     runs the bitmap op over the value buffers); BIT_NOT: ag_arith_unary_same (bitwiseNot :257-259).
 *   SHIFT_*: ag_arith_checked* (ScalarBinaryNotNull slots).  An invalid amount (rhs < 0 or rhs >= bits for unsigned,
 *     rhs >= bits - 1 for SIGNED types — maxShift of shiftKernelSignedImpl :293-296) leaves lhs unchanged; the
 *     _CHECKED flavours also fail the call ("shift amount must be >= 0 and less than precision of type"). */
#define AG_OP_BIT_AND        64
#define AG_OP_BIT_OR         65
#define AG_OP_BIT_XOR        66
#define AG_OP_BIT_NOT        67
#define AG_OP_SHIFT_LEFT     68
#define AG_OP_SHIFT_RIGHT    69
#define AG_OP_SHIFT_LEFT_CHECKED  70
#define AG_OP_SHIFT_RIGHT_CHECKED 71

/* ---- kernels.CompareOperator (kernels/types.go:62-71) ---------------------------- */
#define AG_CMP_EQ 0
#define AG_CMP_NE 1
#define AG_CMP_GT 2
#define AG_CMP_GE 3
#define AG_CMP_LT 4 /* executed as GT with operands flipped, like scalar_compare.go:73-99 */
#define AG_CMP_LE 5 /* executed as GE with operands flipped */

/* operand shapes of the binary entry points (arr_arr / arr_scalar / scalar_arr) */
#define AG_SHAPE_AA 0
#define AG_SHAPE_AS 1
#define AG_SHAPE_SA 2

/* ---- bitmap binary ops (arrow/bitutil/bitmaps.go:601-639) ------------------------ */
#define AG_BITOP_AND     0
#define AG_BITOP_OR      1
#define AG_BITOP_XOR     2
#define AG_BITOP_ANDNOT  3 /* l & ~r */
#define AG_BITOP_XNOR    4
/* Kleene word ops (scalar_boolean.go:103-105,180-182,290-292) */
#define AG_KLEENE_AND     0
#define AG_KLEENE_OR      1
#define AG_KLEENE_ANDNOT  2

/* ---- kernels.NullSelectionBehavior (vector_selection.go:34-39) ------------------- */
#define AG_DROP_NULLS 0
#define AG_EMIT_NULLS 1

/* sentinel written to *first_bad / *bad_pos when no element failed */
#define AG_NO_ERROR_POS INT64_MAX

typedef void* ag_stream_t; /* opaque (a CUDA stream); NULL = the current device's default stream */
typedef void* ag_event_t;  /* opaque (a CUDA event) */
typedef void* ag_comm_t;   /* opaque: one rank of a multi-GPU communicator */

/* ================================================================================= *
 * Runtime, residency, streams
 * ================================================================================= */

/* Initialise one device and its stream pool.  The first call names the process DEFAULT device
 * (device < 0: LOCAL_RANK from the environment, else 0) — all a one-process-per-GPU rank needs.
 * Idempotent; every compute call initialises lazily with device -1 if this was never called.
 * A later ag_init(other) behaves like ag_set_device(other). */
ag_status ag_init(int device);
/* One process driving the whole box (the reference is ONE Go process whose take/filter fan out over
 * goroutines, arrow/compute/selection.go:127-150): initialise every visible device and enable peer
 * access between all pairs.  Then each worker thread picks its device with ag_set_device; streams,
 * pinned and device allocations, and NULL-stream calls follow the calling thread's current device,
 * and a call that is handed a stream always runs on that stream's device. */
ag_status ag_init_all(int* n_devices);
ag_status ag_set_device(int device);
ag_status ag_get_device(int* device);
ag_status ag_shutdown(void);
ag_status ag_device_count(int* count);
ag_status ag_device_info(int* device, int* sm_count, size_t* hbm_bytes, int* cc_major, int* cc_minor);
/* Copies the calling thread's last error message (NUL-terminated) into buf. */
void ag_last_error(char* buf, size_t buflen);
/* Library version string and the number of kernels this process has launched
 * (used by bench.py's gpu_launches and by the loaded-native-code check). */
const char* ag_version(void);
uint64_t ag_kernel_launch_count(void);

/* Pinned host memory: backs a Go memory.Allocator (arrow/memory/allocator.go:23-27);
 * shape follows arrow/memory/internal/cgoalloc/allocator.h:13-18.  64-byte aligned,
 * zero-initialised like memory.GoAllocator / mallocator (calloc). */
ag_status ag_host_alloc(void** ptr, size_t nbytes);
ag_status ag_host_realloc(void** ptr, size_t old_nbytes, size_t new_nbytes);
ag_status ag_host_free(void* ptr);
/* Page-lock memory the caller already owns (e.g. a Mallocator buffer). */
ag_status ag_host_register(void* ptr, size_t nbytes);
ag_status ag_host_unregister(void* ptr);

ag_status ag_dev_alloc(void** dptr, size_t nbytes);   /* stream-ordered pool, zero-filled */
ag_status ag_dev_free(void* dptr);
ag_status ag_dev_memset(void* dptr, int byte, size_t nbytes, ag_stream_t s);
ag_status ag_upload(void* dst_dev, const void* src_host, size_t nbytes, ag_stream_t s);
ag_status ag_download(void* dst_host, const void* src_dev, size_t nbytes, ag_stream_t s);
ag_status ag_copy_dev(void* dst_dev, const void* src_dev, size_t nbytes, ag_stream_t s);

ag_status ag_stream_create(ag_stream_t* s);
ag_status ag_stream_destroy(ag_stream_t s);
ag_status ag_stream_sync(ag_stream_t s);
ag_status ag_event_create(ag_event_t* e);
ag_status ag_event_destroy(ag_event_t e);
ag_status ag_event_record(ag_event_t e, ag_stream_t s);
ag_status ag_event_sync(ag_event_t e);
ag_status ag_event_elapsed_ms(ag_event_t start, ag_event_t stop, float* ms);
/* Writes `nbytes` of a scratch buffer (> L2) so the next timed launch starts cold. */
ag_status ag_flush_l2(ag_stream_t s);

/* ================================================================================= *
 * arrow/math Sum  — replaces sum_{float64,int64,uint64}_{avx2,sse4,neon}
 *   arrow/math/_lib/float64.c:20-26, int64.c:21-27, uint64.c; Go: float64.go:34-39.
 *   Validity is ignored (like the reference); n == 0 gives 0.
 *   Integer sums wrap (two's complement) — bit-exact for any order.
 *   Float64: default mode is a fixed-shape tree of TwoSum (sum, error) pairs (result
 *   is a pure function of data and n, independent of grid/alignment).  Error bound
 *   (Sum2): |res - S| <= 2 eps |S| + gamma_n^2 sum|x|, eps = 2^-53, gamma_n =
 *   n eps / (1 - n eps): within 1 ULP of the exactly rounded sum while gamma_n^2
 *   sum|x| is small against eps |S|; bit-exact with the reference whenever every
 *   partial sum is exact.  Any NaN, or +inf and -inf together, gives NaN; infinities
 *   or an overflow of one sign give that infinity.  Unspecified, as in the reference's
 *   AVX2 order: finite inputs whose partial sums overflow with both signs may give
 *   NaN, and then the class may differ from the reference's.
 *   ag_sum_f64_reforder reproduces the reference AVX2 association order
 *   (float64_avx2_amd64.s:36-43,86-164) bit-for-bit on any input.
 * ================================================================================= */
ag_status ag_sum_f64(const double* buf, size_t n, double* res);
ag_status ag_sum_i64(const int64_t* buf, size_t n, int64_t* res);
ag_status ag_sum_u64(const uint64_t* buf, size_t n, uint64_t* res);
ag_status ag_sum_f64_reforder(const double* buf, size_t n, double* res);
ag_status ag_sum_f64_dev(const double* d_buf, size_t n, double* d_res, ag_stream_t s);
ag_status ag_sum_i64_dev(const int64_t* d_buf, size_t n, int64_t* d_res, ag_stream_t s);
ag_status ag_sum_u64_dev(const uint64_t* d_buf, size_t n, uint64_t* d_res, ag_stream_t s);
ag_status ag_sum_f64_reforder_dev(const double* d_buf, size_t n, double* d_res, ag_stream_t s);

/* ================================================================================= *
 * Multi-GPU (SURVEY §8e): row-range shards, no data-path collective except the global Sum.
 *   Sharding rule: ag_shard_range — ceil-balanced, cuts at multiples of 64 rows (no two shards
 *   share a bitmap word).  Add / compare / filter / take run per shard with no exchange (take
 *   replicates `values`); a bounds / overflow error is the minimum of the shards' error words.
 *   Global Sum: ag_sum_*_global_dev runs the shard's reduction AND the fold over the ranks as
 *   one kernel — the final (sum, error) pair is stored into every rank's HBM mailbox over
 *   NVLink and folded in rank order, so every rank's *d_res holds the same bits, with no
 *   second launch and no host synchronisation.  Every rank of the communicator must make the
 *   call (in the same order when several are in flight).
 *   Setting up the mailboxes:
 *     one process per GPU : ag_comm_local_handle(world, h) on every rank; all-gather the
 *                           AG_COMM_HANDLE_BYTES handles with the caller's own plumbing (MPI,
 *                           torch.distributed, a socket); ag_comm_create(&c, world, rank, handles)
 *     one process, n GPUs : ag_init_all; ag_comm_create_local(comms, n, devices)
 *   NCCL (optional): ag_comm_unique_id on rank 0, broadcast the AG_COMM_ID_BYTES, then
 *   ag_comm_attach_nccl on every rank; ag_sum_i64_global_nccl_dev = per-GPU Sum followed by
 *   ncclAllReduce of the 8-byte result on the same stream.  libnccl.so.2 is dlopen'ed on
 *   first use (AG_ERR_NOT_IMPLEMENTED when the process has none).
 * ================================================================================= */
#define AG_COMM_HANDLE_BYTES 64
#define AG_COMM_ID_BYTES 128
ag_status ag_shard_range(int64_t n_rows, int shard, int n_shards, int64_t* start, int64_t* stop);
ag_status ag_comm_local_handle(int world, void* handle64);
ag_status ag_comm_create(ag_comm_t* comm, int world, int rank, const void* all_handles);
ag_status ag_comm_create_local(ag_comm_t* comms, int n, const int* devices);
ag_status ag_comm_unique_id(void* id128);
ag_status ag_comm_attach_nccl(ag_comm_t comm, const void* id128);
ag_status ag_comm_info(ag_comm_t comm, int* world, int* rank, int* device);
ag_status ag_comm_destroy(ag_comm_t comm);
ag_status ag_sum_i64_global_dev(ag_comm_t comm, const int64_t* d_buf, size_t n, int64_t* d_res, ag_stream_t s);
ag_status ag_sum_u64_global_dev(ag_comm_t comm, const uint64_t* d_buf, size_t n, uint64_t* d_res, ag_stream_t s);
ag_status ag_sum_f64_global_dev(ag_comm_t comm, const double* d_buf, size_t n, double* d_res, ag_stream_t s);
ag_status ag_sum_i64_global_nccl_dev(ag_comm_t comm, const int64_t* d_buf, size_t n, int64_t* d_res, ag_stream_t s);

/* ================================================================================= *
 * Integer min/max — replaces {int,uint}{8,16,32,64}_max_min_{avx2,sse4,neon}
 *   (internal/utils/_lib/min_max.c:23-125; Go: GetMinMaxInt8 ... GetMinMaxUint64,
 *   internal/utils/min_max.go) — the reduction behind Parquet column statistics
 *   (parquet/metadata/statistics_types.gen.go:160-190,464-490).  n == 0 gives the
 *   reference's initial values (type MAX, type MIN).  The device flavour writes
 *   {min, max} as two consecutive elements of the value type.
 * ================================================================================= */
ag_status ag_min_max(int type, const void* values, int64_t n, void* min_out, void* max_out);
ag_status ag_min_max_dev(int type, const void* d_values, int64_t n, void* d_min_max, ag_stream_t s);

/* ================================================================================= *
 * Arithmetic — replaces arithmetic_{binary,arr_scalar,scalar_arr,unary_same_types,
 *   unary_diff_type}_{avx2,sse4} (_lib/base_arithmetic.cc:465-483) and the pure-Go
 *   fallbacks of base_arithmetic.go.  Computed for EVERY slot (ScalarBinary
 *   semantics, helpers.go:193-236).  Ops: ADD/SUB/MUL (+_CHECKED aliases, which for
 *   these entry points are the unchecked loops exactly like the reference's native
 *   code: base_arithmetic.cc:445-462).  Integers wrap.  The scalar operand is a
 *   pointer to one element (host memory in both flavours).
 * ================================================================================= */
ag_status ag_arith_binary(int type, int8_t op, const void* l, const void* r, void* out, int64_t n);
ag_status ag_arith_arr_scalar(int type, int8_t op, const void* l, const void* scalar_r, void* out, int64_t n);
ag_status ag_arith_scalar_arr(int type, int8_t op, const void* scalar_l, const void* r, void* out, int64_t n);
ag_status ag_arith_unary_same(int type, int8_t op, const void* in, void* out, int64_t n);      /* ABS, NEGATE, SIGN (+_CHECKED aliases) */
ag_status ag_arith_unary_diff(int itype, int otype, int8_t op, const void* in, void* out, int64_t n); /* SIGN */
ag_status ag_arith_binary_dev(int type, int8_t op, int shape, const void* d_l, const void* d_r, void* d_out,
                              int64_t n, ag_stream_t s); /* scalar side: HOST pointer to one element */
/* Batched form for chunked arguments: ONE launch (device flavour) / one pipelined transfer
 * schedule (host flavour) for all the aligned spans iterateExecSpans yields for a call
 * (arrow/compute/executor.go:757-863).  A compute.Function that receives whole ChunkedDatums
 * (functions.go:30-41) binds this instead of a per-span kernel.  Results are identical to
 * calling ag_arith_binary[_dev] once per span.  For AS / SA shapes the scalar side of every
 * span must be the same host pointer to one element. */
typedef struct ag_span3 { const void* l; const void* r; void* out; int64_t n; } ag_span3;
ag_status ag_arith_binary_spans(int type, int8_t op, int shape, const ag_span3* spans, int64_t n_spans);
ag_status ag_arith_binary_spans_dev(int type, int8_t op, int shape, const ag_span3* spans, int64_t n_spans, ag_stream_t s);
ag_status ag_arith_unary_same_dev(int type, int8_t op, const void* d_in, void* d_out, int64_t n, ag_stream_t s);
ag_status ag_arith_unary_diff_dev(int itype, int otype, int8_t op, const void* d_in, void* d_out, int64_t n, ag_stream_t s);

/* Checked integer arithmetic with the reference's exact overflow predicate and slot
 * semantics — no native counterpart exists in the reference; this restates
 *   ADD_CHECKED / SUB_CHECKED: base_arithmetic.go:249-278 under ScalarBinaryNotNull
 *       (helpers.go:284-380): only slots valid in BOTH inputs are computed, null slots
 *       are written as 0;
 *   MUL_CHECKED: base_arithmetic.go:84-108,279-286 under ScalarBinary (all slots);
 *   DIV / DIV_CHECKED: base_arithmetic.go:154-161,287-294 (divide by zero -> error),
 *       ScalarBinaryNotNull.
 * lvalid / rvalid may be NULL (= all valid); offsets are bit offsets.  A NULL scalar
 * operand pointer means a null scalar (whole output untouched, status OK).
 * On overflow / divide by zero returns AG_ERR_INVALID and *first_bad (may be NULL)
 * receives the lowest failing row; otherwise AG_NO_ERROR_POS. */
ag_status ag_arith_checked(int type, int8_t op, int shape,
                           const void* l, const uint8_t* lvalid, int64_t loff,
                           const void* r, const uint8_t* rvalid, int64_t roff,
                           void* out, int64_t n, int64_t* first_bad);
/* abs / negate (checked) on signed integers: AbsoluteValueChecked / NegateChecked,
 * base_arithmetic.go:295-340 under ScalarUnary (EVERY slot, null or not): a slot equal to
 * MinInt gives AG_ERR_INVALID "overflow"; other slots as the unchecked kernels.  Unsigned and
 * floating types never fail (they behave like ag_arith_unary_same). */
ag_status ag_arith_unary_checked(int type, int8_t op, const void* in, void* out, int64_t n, int64_t* first_bad);
ag_status ag_arith_unary_checked_dev(int type, int8_t op, const void* d_in, void* d_out, int64_t n, int64_t* d_first_bad, ag_stream_t s);
/* Device flavour: *d_first_bad must be initialised to AG_NO_ERROR_POS by the caller
 * (ag_dev_memset is not enough: use ag_error_word_reset_dev); it is only lowered. */
ag_status ag_arith_checked_dev(int type, int8_t op, int shape,
                               const void* d_l, const uint8_t* d_lvalid, int64_t loff,
                               const void* d_r, const uint8_t* d_rvalid, int64_t roff,
                               void* d_out, int64_t n, int64_t* d_first_bad, ag_stream_t s);
ag_status ag_error_word_reset_dev(int64_t* d_word, ag_stream_t s);

/* ================================================================================= *
 * Numeric casts — replaces cast_type_numeric_{avx2,sse4} (_lib/cast_numeric.cc:22-101, Go
 *   dispatch cast_numeric.go:101-131) for the 10 numeric types, and the checks of
 *   numeric_cast.go that frame it under safe CastOptions (what implicit promotion uses:
 *   compute/exec.go:101-121 -> CastDatum(SafeCastOptions)):
 *     int -> int    intsCanFit/intsInRange (helpers.go:545-653), skipped when AllowIntOverflow
 *     int -> float  checkIntToFloatTrunc   (numeric_cast.go:698-729): |v| <= 2^24 / 2^53
 *     float -> int  checkFloatTrunc        (numeric_cast.go:613-660): OutT(v) converted back != v
 *   the last two skipped when AllowFloatTruncate.  Every slot is converted (nulls too, like
 *   castNumberToNumberUnsafe, helpers.go:690-703); the checks look only at valid slots.
 *   Bit-exact with the reference loops for every input whose converted value is representable
 *   in the output type; out-of-range float -> int is not defined by the reference (its AVX2 body,
 *   SSE4 body and scalar tail disagree) — here: 64-bit truncation (NaN/overflow -> INT64_MIN)
 *   then wrap to the output width, the pure-Go amd64 behaviour.
 *   Checked flavour: AG_ERR_INVALID + lowest failing row in *first_bad (else AG_NO_ERROR_POS).
 * ================================================================================= */
ag_status ag_cast_numeric(int itype, int otype, const void* in, void* out, int64_t n);
ag_status ag_cast_numeric_dev(int itype, int otype, const void* d_in, void* d_out, int64_t n, ag_stream_t s);
ag_status ag_cast_numeric_checked(int itype, int otype, const void* in, const uint8_t* valid, int64_t valid_offset,
                                  void* out, int64_t n, int allow_int_overflow, int allow_float_truncate, int64_t* first_bad);
/* *d_first_bad must hold AG_NO_ERROR_POS (ag_error_word_reset_dev); it is only lowered. */
ag_status ag_cast_numeric_checked_dev(int itype, int otype, const void* d_in, const uint8_t* d_valid, int64_t valid_offset,
                                      void* d_out, int64_t n, int allow_int_overflow, int allow_float_truncate,
                                      int64_t* d_first_bad, ag_stream_t s);

/* ================================================================================= *
 * cumulative_sum / cumulative_sum_checked — replaces cumulativeSum{NoNulls,WithNulls}[Checked]
 *   (arrow/compute/internal/kernels/vector_cumulative.go:228-330; options CumulativeOptions
 *   {Start, SkipNulls} :92-99; chunked input = one logical sequence, :385-410).
 *   out[i] = start + sum of the valid in[j], j <= i.  Null input slot -> null output slot (value 0).
 *   Without skip_nulls every slot after the first null is null too and nothing accumulates past
 *   it.  `checked`: AG_ERR_INVALID "overflow" at the first running sum outside the type's range
 *   (integers only; floats never fail), lowest failing row in *first_bad.
 *   Integers: bit-exact.  Floats: single-pass parallel scan with a fixed (data- and n-determined)
 *   association, bit-exact with its model tests/cumsum_float_ref.py on any input — bit-exact with
 *   the reference's left-to-right loop whenever every partial sum is exactly representable (signed
 *   zeros included), otherwise within the summation error bound of that association (DESIGN.md).
 *   The state carried to the next chunk is the last tile's exclusive prefix + tile total, which may
 *   differ from the last output slot by rounding (the reference carries its last output).
 *
 *   Device flavour: the running value and the encountered-null flag live in a 32-byte device
 *   block (ag_cumsum_state) so that the chunks of a chunked column are a chain of launches on
 *   one stream; initialise it with ag_cumulative_sum_state_init_dev (start_host: pointer to one
 *   element of `type`, or NULL for zero).  d_out_valid (bit offset out_valid_offset) is required
 *   when d_valid is given and otherwise optional (pass it for every chunk when any chunk has
 *   nulls); state.null_count accumulates the null slots written.
 * ================================================================================= */
typedef struct ag_cumsum_state { uint64_t lo; int64_t hi; int64_t encountered_null; int64_t null_count; } ag_cumsum_state;
ag_status ag_cumulative_sum(int type, const void* in, const uint8_t* valid, int64_t valid_offset, int64_t n,
                            const void* start, int skip_nulls, int checked,
                            void* out, uint8_t* out_valid, int64_t* null_count, int64_t* first_bad);
ag_status ag_cumulative_sum_state_init_dev(void* d_state, int type, const void* start_host, ag_stream_t s);
ag_status ag_cumulative_sum_dev(int type, const void* d_in, const uint8_t* d_valid, int64_t valid_offset, int64_t n,
                                int skip_nulls, int checked, void* d_out, uint8_t* d_out_valid, int64_t out_valid_offset,
                                void* d_state, int64_t* d_first_bad, ag_stream_t s);

/* ================================================================================= *
 * Comparisons -> bitmap — replaces comparison_{equal,not_equal,greater,greater_equal}
 *   _{arr_arr,arr_scalar,scalar_arr}_{avx2,sse4} (_lib/scalar_comparison.cc:210-256)
 *   and compareKernel (scalar_comparisons.go:199-218).  `out_bits` points at the byte
 *   holding the first output bit, `bit_offset` is used mod 8 exactly like the
 *   reference; bits outside the written range are preserved.  LT/LE are accepted and
 *   executed by operand flipping.  NaN: every predicate false except NE.
 * ================================================================================= */
ag_status ag_compare(int type, int cmp, int shape, const void* l, const void* r,
                     uint8_t* out_bits, int64_t n, int bit_offset);
ag_status ag_compare_dev(int type, int cmp, int shape, const void* d_l, const void* d_r,
                         uint8_t* d_out_bits, int64_t n, int bit_offset, ag_stream_t s);
/* Named forms with the reference's exact native signature (type,l,r,out,length,offset). */
ag_status ag_cmp_eq_aa(int type, const void* l, const void* r, void* out, int64_t n, int offset);
ag_status ag_cmp_eq_as(int type, const void* l, const void* r, void* out, int64_t n, int offset);
ag_status ag_cmp_eq_sa(int type, const void* l, const void* r, void* out, int64_t n, int offset);
ag_status ag_cmp_ne_aa(int type, const void* l, const void* r, void* out, int64_t n, int offset);
ag_status ag_cmp_ne_as(int type, const void* l, const void* r, void* out, int64_t n, int offset);
ag_status ag_cmp_ne_sa(int type, const void* l, const void* r, void* out, int64_t n, int offset);
ag_status ag_cmp_gt_aa(int type, const void* l, const void* r, void* out, int64_t n, int offset);
ag_status ag_cmp_gt_as(int type, const void* l, const void* r, void* out, int64_t n, int offset);
ag_status ag_cmp_gt_sa(int type, const void* l, const void* r, void* out, int64_t n, int offset);
ag_status ag_cmp_ge_aa(int type, const void* l, const void* r, void* out, int64_t n, int offset);
ag_status ag_cmp_ge_as(int type, const void* l, const void* r, void* out, int64_t n, int offset);
ag_status ag_cmp_ge_sa(int type, const void* l, const void* r, void* out, int64_t n, int offset);

/* ================================================================================= *
 * Bitmaps — replaces bitmap_aligned_{and,or,and_not,xor}_{avx2,sse4}
 *   (arrow/bitutil/_lib/bitmap_ops.c:24-46) plus the Go paths around them:
 *   alignedBitmapOp / unalignedBitmapOp (bitmaps.go:527-591), CopyBitmap /
 *   InvertBitmap (:483-491), SetBitsTo (bitutil.go:158), CountSetBits (:89).
 *   Arbitrary bit offsets on every operand; `out` may alias an input with the same
 *   offset (propagateNulls accumulates in place, executor.go:340-347).
 * ================================================================================= */
ag_status ag_bitmap_op(int bitop, const uint8_t* l, int64_t loff, const uint8_t* r, int64_t roff,
                       uint8_t* out, int64_t ooff, int64_t nbits);
ag_status ag_bitmap_copy(const uint8_t* src, int64_t soff, int64_t nbits, uint8_t* dst, int64_t doff);
ag_status ag_bitmap_invert(const uint8_t* src, int64_t soff, int64_t nbits, uint8_t* dst, int64_t doff);
ag_status ag_bitmap_set(uint8_t* bits, int64_t off, int64_t nbits, int value);
ag_status ag_bitmap_popcount(const uint8_t* bits, int64_t off, int64_t nbits, int64_t* count);
ag_status ag_bitmap_op_dev(int bitop, const uint8_t* d_l, int64_t loff, const uint8_t* d_r, int64_t roff,
                           uint8_t* d_out, int64_t ooff, int64_t nbits, ag_stream_t s);
ag_status ag_bitmap_copy_dev(const uint8_t* d_src, int64_t soff, int64_t nbits, uint8_t* d_dst, int64_t doff, ag_stream_t s);
ag_status ag_bitmap_invert_dev(const uint8_t* d_src, int64_t soff, int64_t nbits, uint8_t* d_dst, int64_t doff, ag_stream_t s);
ag_status ag_bitmap_set_dev(uint8_t* d_bits, int64_t off, int64_t nbits, int value, ag_stream_t s);
/* *d_count is overwritten with the population count of [off, off+nbits). */
ag_status ag_bitmap_popcount_dev(const uint8_t* d_bits, int64_t off, int64_t nbits, int64_t* d_count, ag_stream_t s);

/* Kleene logic on (validity, data) pairs — computeKleene, scalar_boolean.go:29-65 with
 * the word lambdas at :103-105 (and), :180-182 (or), :290-292 (and_not).  lvalid /
 * rvalid may be NULL (= all valid).  Both outputs use bit offset ooff. */
ag_status ag_kleene(int kop, const uint8_t* lvalid, const uint8_t* ldata, int64_t loff,
                    const uint8_t* rvalid, const uint8_t* rdata, int64_t roff,
                    uint8_t* out_valid, uint8_t* out_data, int64_t ooff, int64_t nbits);
ag_status ag_kleene_dev(int kop, const uint8_t* d_lvalid, const uint8_t* d_ldata, int64_t loff,
                        const uint8_t* d_rvalid, const uint8_t* d_rdata, int64_t roff,
                        uint8_t* d_out_valid, uint8_t* d_out_data, int64_t ooff, int64_t nbits, ag_stream_t s);

/* ================================================================================= *
 * Filter — replaces PrimitiveFilter (vector_selection.go:449-520) =
 *   getFilterOutputSize (:57-81) + primitiveFilterImpl (:267-395) + filterWriter
 *   (:397-421), and GetTakeIndices (:102-236).
 *   values: fixed width, bit_width in {8,16,32,64}; `vals` points at element 0 of the
 *   buffer and voff is the element offset (needed for the validity bitmap too).
 *   vvalid / mvalid may be NULL.  Output: stable compaction; out_valid (may be NULL when the
 *   output cannot contain nulls) receives the compacted validity starting at bit 0;
 *   EMIT_NULLS writes value 0 / validity 0 for null mask slots.
 * ================================================================================= */
ag_status ag_filter_output_size(const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n,
                                int null_selection, int64_t* out_len);
ag_status ag_filter_primitive(int bit_width, const void* vals, const uint8_t* vvalid, int64_t voff,
                              const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n,
                              int null_selection, void* out, uint8_t* out_valid,
                              int64_t* out_len, int64_t* out_nulls);
ag_status ag_filter_output_size_dev(const uint8_t* d_mask, const uint8_t* d_mvalid, int64_t moff, int64_t n,
                                    int null_selection, int64_t* d_out_len, ag_stream_t s);
/* out_capacity = number of rows d_out (and d_out_valid) can hold: the exact output length
 * when the caller ran ag_filter_output_size_dev first, or n as an upper bound.  Rows past the
 * capacity are dropped; *d_out_len always receives the full number of emitted rows so a
 * truncation is detectable.  d_out_valid (may be NULL when the output cannot contain nulls:
 * no values validity, and DROP_NULLS or no mask validity) must be 4-byte aligned and hold
 * ceil(out_capacity/32) 32-bit words; it is fully overwritten (Arrow buffers are padded to 64 B). */
ag_status ag_filter_primitive_dev(int bit_width, const void* d_vals, const uint8_t* d_vvalid, int64_t voff,
                                  const uint8_t* d_mask, const uint8_t* d_mvalid, int64_t moff, int64_t n,
                                  int null_selection, void* d_out, uint8_t* d_out_valid, int64_t out_capacity,
                                  int64_t* d_out_len, ag_stream_t s);
/* Fused Greater/…(values, scalar) + Filter: one pass over `values`, no intermediate
 * mask (SURVEY §8d: 8 + 8s bytes/row).  Not a reference entry point — an optimisation
 * the plugin applies to the greater→filter pipeline of config 3; results are identical
 * to ag_compare followed by ag_filter_primitive. */
ag_status ag_filter_compare_scalar_dev(int type, int cmp, const void* d_vals, const void* scalar_host,
                                       int64_t n, void* d_out, int64_t out_capacity, int64_t* d_out_len, ag_stream_t s);
/* GetTakeIndices: mask -> row indices; index_width 16 or 32 bits (the reference picks
 * uint16 when n < 65535 else uint32, vector_selection.go:229-235). */
ag_status ag_take_indices(int index_width, const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n,
                          int null_selection, void* out_idx, uint8_t* out_valid, int64_t* out_len);
ag_status ag_take_indices_dev(int index_width, const uint8_t* d_mask, const uint8_t* d_mvalid, int64_t moff, int64_t n,
                              int null_selection, void* d_out_idx, uint8_t* d_out_valid, int64_t out_capacity,
                              int64_t* d_out_len, ag_stream_t s);

/* ================================================================================= *
 * Take — replaces PrimitiveTake (vector_selection.go:1162-1192) = checkIndexBounds
 *   (helpers.go:929-981) + primitiveTakeImpl (:813-988).
 *   out[i] = values[voff + idx[i]]; out_valid[i] = ivalid[ioff+i] & vvalid[voff+idx[i]].
 *   Null output slots carry value 0 (the reference leaves its zero-initialised
 *   allocation untouched).  idx_width in {8,16,32,64}; idx_signed: indices are
 *   reinterpreted as unsigned after the bounds check (:1147-1159).  With bounds_check,
 *   an out-of-range VALID index gives AG_ERR_INDEX, *bad_pos = lowest offending row and
 *   *bad_index = its value ("%d out of bounds", helpers.go:951).
 * ================================================================================= */
ag_status ag_take_primitive(int bit_width, const void* vals, const uint8_t* vvalid, int64_t voff, int64_t vlen,
                            int idx_width, int idx_signed, const void* idx, const uint8_t* ivalid, int64_t ioff,
                            int64_t n, int bounds_check, void* out, uint8_t* out_valid,
                            int64_t* out_nulls, int64_t* bad_pos, int64_t* bad_index);
/* d_out_valid: 4-byte aligned, offset 0.  *d_bad_pos must have been reset with
 * ag_error_word_reset_dev and is only lowered. */
ag_status ag_take_primitive_dev(int bit_width, const void* d_vals, const uint8_t* d_vvalid, int64_t voff, int64_t vlen,
                                int idx_width, int idx_signed, const void* d_idx, const uint8_t* d_ivalid, int64_t ioff,
                                int64_t n, int bounds_check, void* d_out, uint8_t* d_out_valid,
                                int64_t* d_bad_pos, ag_stream_t s);
/* Routing of large takes (results never depend on it).  Random indices into a values table far larger
 * than L2 go through the windowed path (partition indices by table window of 8 MB or more -> gather window by
 * window out of L2 -> un-permute); sorted / clustered indices and small calls use the direct gather
 * (the reference switches loop shape the same way, vector_selection.go:897-911).
 * mode: 0 automatic (default), 1 always direct, 2 windowed whenever the shapes allow it.
 * min_rows / min_table_bytes / window_bytes: thresholds of the automatic mode and the window size;
 * values <= 0 keep the current setting.  Process-wide. */
ag_status ag_take_set_policy(int mode, int64_t min_rows, int64_t min_table_bytes, int64_t window_bytes);

/* ================================================================================= *
 * is_in / unique for fixed-width values of 1/2/4/8 bytes (SURVEY 8f rank 3) — the memo-table kernels of
 *   kernels/scalar_set_lookup.go:112-413 and kernels/vector_hash.go.  Values are compared by their RAW
 *   BYTES like the reference's memo tables (floats: NaN == NaN of the same payload, -0.0 != +0.0).
 *   is_in: out_data / out_valid are bitmaps at bit offset 0 (4-byte aligned); per row
 *     valid value: in the set -> (true, valid); else INCONCLUSIVE and the set holds a null -> (false, null);
 *                  else (false, valid)
 *     null       : MATCH and the set holds a null -> (true, valid); SKIP, or MATCH without one -> (false, valid);
 *                  else (false, null)                                   (isInKernelExec :373-413)
 *   unique: the distinct values in order of first appearance, a null kept once where it first appears;
 *     *out_len receives the count (capacity n is always enough).
 *   `offset` / `set_offset` are element offsets into both the values buffer and the validity bitmap.
 * ================================================================================= */
#define AG_NULL_MATCH        0
#define AG_NULL_SKIP         1
#define AG_NULL_EMIT_NULL    2
#define AG_NULL_INCONCLUSIVE 3
ag_status ag_is_in(int bit_width, const void* vals, const uint8_t* valid, int64_t offset, int64_t n,
                   const void* set_vals, const uint8_t* set_valid, int64_t set_offset, int64_t set_n, int null_behavior,
                   uint8_t* out_data, uint8_t* out_valid, int64_t* out_nulls);
ag_status ag_is_in_dev(int bit_width, const void* d_vals, const uint8_t* d_valid, int64_t offset, int64_t n,
                       const void* d_set_vals, const uint8_t* d_set_valid, int64_t set_offset, int64_t set_n, int null_behavior,
                       uint8_t* d_out_data, uint8_t* d_out_valid, int64_t* d_null_count, ag_stream_t s);
ag_status ag_unique(int bit_width, const void* vals, const uint8_t* valid, int64_t offset, int64_t n,
                    void* out, uint8_t* out_valid, int64_t* out_len, int64_t* out_nulls);
ag_status ag_unique_dev(int bit_width, const void* d_vals, const uint8_t* d_valid, int64_t offset, int64_t n,
                        void* d_out, uint8_t* d_out_valid, int64_t capacity, int64_t* d_out_len, ag_stream_t s);
/* unique's table policy: a column of more than `small_rows` rows (default 2^21) is first inserted into a table of
 * `small_slots` slots (a power of two, default 2^21 = 32 MB, L2-resident); the full-size table (2n slots) is filled only
 * when more than small_slots/2 distinct values turn up — decided on the device, never changes a result.  0 = default. */
ag_status ag_unique_set_policy(int64_t small_rows, int64_t small_slots);

/* ================================================================================= *
 * dictionary_encode for fixed-width values of 1/2/4/8 bytes — the memo-table kernels of
 *   compute/vector_hash.go:105-121 and kernels/vector_hash.go:144-241 (dictionaryEncodeAction):
 *   output type Dictionary<int32, T> (outputDictionaryType), the dictionary = the distinct values in order of first
 *   appearance over the WHOLE column, keys compared by raw bytes as in unique.  One call encodes every chunk of a
 *   column into one shared dictionary; rows are numbered across the chunks in table order.
 *   null_encoding (DictionaryEncodeOptions.NullEncoding):
 *     AG_NULL_ENCODING_MASK (0)   a null row gets index 0 and a null index slot; the dictionary holds no null;
 *     AG_NULL_ENCODING_ENCODE (1) the null is an ordinary dictionary entry where it first appears (value bytes 0,
 *                                 validity bit clear); the indices have no nulls.   Anything else: AG_ERR_INVALID.
 *   chunks: a HOST array of n_chunks descriptors.  `offset` is an element offset into values and validity; indices
 *     (length int32) and indices_validity (4-byte aligned, ceil(length/32)*4 bytes) are written at offset 0.
 *     indices_validity is written only in Mask mode for a chunk that has a validity bitmap (then it is required).
 *   dict: capacity total rows of the value width; d_dict_valid: ceil(total/8) bytes, written only in Encode mode
 *     (required there when any chunk has a validity bitmap): all ones but the null's bit.
 *   counts (n_chunks + 2 int64): [0] dictionary length, [1] dictionary null count (0 or 1), [2 + c] the null count of
 *     chunk c's indices.
 *   More than 2^31-1 rows in all: AG_ERR_NOT_IMPLEMENTED.  ag_unique_set_policy applies to the table.
 *   Host flavour: every pointer is a host pointer; dict / dict_valid receive only the dictionary's length.
 * ================================================================================= */
#define AG_TYPE_DICTIONARY         29 /* arrow.DICTIONARY (arrow/datatype.go) */
#define AG_NULL_ENCODING_MASK       0
#define AG_NULL_ENCODING_ENCODE     1
typedef struct ag_dict_chunk {
  const void* values;
  const uint8_t* validity;   /* may be NULL */
  int64_t offset;
  int64_t length;
  int32_t* indices;
  uint8_t* indices_validity;
} ag_dict_chunk;
ag_status ag_dictionary_encode(int bit_width, const ag_dict_chunk* chunks, int64_t n_chunks, int null_encoding,
                               void* dict, uint8_t* dict_valid, int64_t* counts);
ag_status ag_dictionary_encode_dev(int bit_width, const ag_dict_chunk* chunks, int64_t n_chunks, int null_encoding,
                                   void* d_dict, uint8_t* d_dict_valid, int64_t* d_counts, ag_stream_t s);

/* ================================================================================= *
 * run_end_encode / run_end_decode for BOOL and the 10 numeric types — the fixed-width and boolean loops of
 *   kernels/vector_run_end_encode.go: CountNumberOfRuns (:114-141) + WriteEncodedRuns (:86-112), and
 *   decodeBool / decodeFixedWidth ExpandAllRuns (:591-719).  Run-end types: AG_TYPE_INT16 / INT32 / INT64; any other
 *   run_end_type is AG_ERR_INVALID "bad run end type" (:567-578).
 * Encode of rows [offset, offset+n) of `vals` (BOOL: an LSB-first bitmap) with optional `valid` (same offset):
 *   rows i-1 and i share a run iff their validity bits are equal AND their values compare equal with the type's ==,
 *   the payload under a null included (:96-105): float NaN rows each start a run, +0.0 and -0.0 share one.
 *   Run r: run_ends[r] = the first row of run r+1 (n for the last run), out[r] = the value (BOOL: bit r) of its first
 *   row, out_valid bit r = that row's validity.  out_valid is written only when `valid` is given (then required).
 *   counts (2 int64): [0] runs, [1] null runs — the true totals even when they exceed `capacity`; runs past
 *   `capacity` are not written.  n > the run-end type's maximum: AG_ERR_INVALID "cannot run-end encode arrays with
 *   more elements than the run end type can hold: <max>" (validateRunEndType :437-444); n == 0: no runs, no error.
 *   Device flavour: out_valid (and a BOOL out) are 4-byte aligned bitmaps of ceil(capacity/32) words, bit 0 = run 0.
 * Decode of the logical slice [offset, offset+length) of a run-end encoded array (run_ends: n_runs entries; the values
 *   child `vals` / `valid` at element offset values_offset, at least values_offset + n_runs elements):
 *   out row j = the value and validity of the run p with run_ends[p-1] <= offset+j < run_ends[p]; the last run is
 *   clipped at offset+length.  out is written at offset 0 (BOOL and out_valid: ceil(length/32) 4-byte aligned words,
 *   bits past length cleared); out_valid is written only when `valid` is given (then required).
 *   Malformed run ends — not strictly increasing over the runs that cover the slice, or a last run end below
 *   offset+length — are AG_ERR_INVALID (host flavour) / lower *d_error_word (device flavour; reset it with
 *   ag_error_word_reset_dev, it is only lowered, to the index of a malformed run end or to n_runs).  Whatever the
 *   input, no read leaves run_ends[0..n_runs) and the values child, and no write leaves the words of [0, length).
 *   The reference does neither: it walks every run to the end of run_ends (:673).
 * Host flavours: every pointer is a host pointer; *null_count (may be NULL) receives the output's null count.
 * ================================================================================= */
#define AG_TYPE_RUN_END_ENCODED    38 /* arrow.RUN_END_ENCODED (arrow/datatype.go) */
ag_status ag_run_end_count(int type, const void* vals, const uint8_t* valid, int64_t offset, int64_t n, int64_t* counts);
ag_status ag_run_end_count_dev(int type, const void* d_vals, const uint8_t* d_valid, int64_t offset, int64_t n, int64_t* d_counts,
                               ag_stream_t s);
ag_status ag_run_end_encode(int type, int run_end_type, const void* vals, const uint8_t* valid, int64_t offset, int64_t n,
                            void* run_ends, void* out, uint8_t* out_valid, int64_t capacity, int64_t* counts);
ag_status ag_run_end_encode_dev(int type, int run_end_type, const void* d_vals, const uint8_t* d_valid, int64_t offset, int64_t n,
                                void* d_run_ends, void* d_out, uint8_t* d_out_valid, int64_t capacity, int64_t* d_counts, ag_stream_t s);
ag_status ag_run_end_decode(int type, int run_end_type, const void* run_ends, int64_t n_runs, const void* vals, const uint8_t* valid,
                            int64_t values_offset, int64_t offset, int64_t length, void* out, uint8_t* out_valid, int64_t* null_count);
ag_status ag_run_end_decode_dev(int type, int run_end_type, const void* d_run_ends, int64_t n_runs, const void* d_vals,
                                const uint8_t* d_valid, int64_t values_offset, int64_t offset, int64_t length, void* d_out,
                                uint8_t* d_out_valid, int64_t* d_null_count, int64_t* d_error_word, ag_stream_t s);

/* ================================================================================= *
 * sort_indices, one fixed-width column (SURVEY 8f rank 3) — replaces kernels.SortIndices for a single
 *   key (vector_sort.go:385-481, vector_sort_internal.go:36-150,250-300): a STABLE permutation of
 *   0..n-1 as uint64 row indices,
 *     null_placement 0 (NullsAtEnd)  : [finite in key order | NaN in row order | null in row order]
 *     null_placement 1 (NullsAtStart): [null in row order | NaN in row order | finite in key order]
 *   order 0 ascending / 1 descending (ties keep row order either way; -0.0 == +0.0).
 *   `offset` is the slice's element offset into both the values buffer and the validity bitmap.
 *   The device flavour synchronises the stream once (a 2 KB histogram read-back decides which radix
 *   passes can be skipped).  n < 2^32 rows per call.
 * ================================================================================= */
ag_status ag_sort_indices(int type, const void* vals, const uint8_t* valid, int64_t offset, int64_t n, int order,
                          int null_placement, uint64_t* out_indices, int64_t* null_count, int64_t* nan_count);
ag_status ag_sort_indices_dev(int type, const void* d_vals, const uint8_t* d_valid, int64_t offset, int64_t n, int order,
                              int null_placement, uint64_t* d_out_indices, int64_t* null_count, int64_t* nan_count, ag_stream_t s);

/* ================================================================================= *
 * sort_indices over several keys, each key column split into chunks — replaces kernels.SortIndices for
 *   record batches, tables and chunked arrays whose key columns are BOOL or one of the 10 numeric types
 *   (arrow/compute/vector_sort.go:30-52,117-200, internal/kernels/vector_sort.go:390-481): a STABLE
 *   lexicographic permutation of 0..n-1 as uint64, rows numbered across chunks.  For each key, first to last:
 *     null_placement 0 (NullsAtEnd)  : [finite in key order | NaN | null]
 *     null_placement 1 (NullsAtStart): [null | NaN | finite in key order]
 *   and ties on a key (NaN and null rows included) are ordered by the next key; ties on every key keep row
 *   order.  -0.0 == +0.0, descending reverses only the finite values, false < true.  This is the partition
 *   rule of radixRecordBatchSortRange (vector_sort_internal.go:170-206) on every input; the reference's chunk
 *   merges and its tail comparator above 8 keys place NaN by order instead (vector_sort_support.go:120-137),
 *   see DESIGN §2.
 *   keys[j]: the column of key j as `nchunks` chunks of `length` rows each (values and validity at element
 *   `offset`; BOOL values are an LSB-first bitmap); every key's chunk lengths sum to n, chunk boundaries may
 *   differ between keys.  The ag_sort_key and ag_sort_chunk arrays are host memory in both flavours; `vals`
 *   and `valid` are host pointers in the host flavour and device pointers in the device flavour.
 *   nkeys < 1, order / null_placement other than 0 / 1, negative offsets or lengths, or chunk lengths that
 *   do not sum to n: AG_ERR_INVALID (vector_sort.go:164-170,390-404); another key type, or n >= 2^32:
 *   AG_ERR_NOT_IMPLEMENTED.  The device flavour synchronises the stream once (the per-key statistics
 *   read-back that sizes the packed key).
 * ================================================================================= */
typedef struct { const void* vals; const uint8_t* valid; int64_t offset; int64_t length; } ag_sort_chunk;
typedef struct { int type; int order; int null_placement; int nchunks; const ag_sort_chunk* chunks; } ag_sort_key;
ag_status ag_sort_indices_keys(int nkeys, const ag_sort_key* keys, int64_t n, uint64_t* out_indices);
ag_status ag_sort_indices_keys_dev(int nkeys, const ag_sort_key* keys, int64_t n, uint64_t* d_out_indices, ag_stream_t s);

/* ================================================================================= *
 * Take over several columns at once — the per-column takes of takeRecordImpl / takeTableImpl and of
 *   FilterRecordBatch / FilterTable (arrow/compute/selection.go:117-204,679-800) in one launch: every column is
 *   gathered by the same n indices, with the rules of ag_take_primitive:
 *     out[i] = the column's row idx[i], rows numbered across its chunks (ag_sort_chunk: values and validity at element
 *       `offset`, BOOL values an LSB-first bitmap); out_valid[i] = idx_valid[idx_offset+i] & the row's validity; value
 *       0 where out_valid is clear.
 *   cols[j]: type BOOL or one of the 10 numeric types, any mix; nchunks chunks whose lengths sum to nrows (empty and
 *   sliced chunks allowed, columns may be chunked differently).  out (BOOL: a bitmap) and out_valid are written at
 *   offset 0.  out_valid may be NULL only when neither the column nor the indices have a validity bitmap.
 *   idx: n indices of idx_width bits (8/16/32/64) starting at element 0, signed when idx_signed; idx_valid (may be
 *   NULL) at bit idx_offset.  Only valid index slots are bounds-checked; negative (signed) or >= nrows is out of
 *   bounds.  With bounds_check: AG_ERR_INDEX "%d out of bounds" with the index of the lowest offending row in
 *   *bad_pos / *bad_index (host flavour), or that row lowered into *d_bad_pos (device flavour; reset it with
 *   ag_error_word_reset_dev).
 *   The ag_take_column and ag_sort_chunk arrays are host memory in both flavours; every other pointer is a host
 *   pointer in the host flavour (out / out_valid receive ceil(n/8) bytes of bitmap) and a device pointer in the
 *   device flavour (out_valid, and a BOOL out, 4-byte aligned, ceil(n/32) words).
 *   Negative offsets or lengths, or chunk lengths that do not sum to nrows: AG_ERR_INVALID; another column type:
 *   AG_ERR_NOT_IMPLEMENTED naming the column.  Both are checked before any device work.
 * ================================================================================= */
typedef struct { int type; int nchunks; const ag_sort_chunk* chunks; void* out; uint8_t* out_valid; } ag_take_column;
ag_status ag_take_columns(int ncols, const ag_take_column* cols, int64_t nrows, int idx_width, int idx_signed, const void* idx,
                          const uint8_t* idx_valid, int64_t idx_offset, int64_t n, int bounds_check, int64_t* bad_pos,
                          int64_t* bad_index);
ag_status ag_take_columns_dev(int ncols, const ag_take_column* cols, int64_t nrows, int idx_width, int idx_signed,
                              const void* d_idx, const uint8_t* d_idx_valid, int64_t idx_offset, int64_t n, int bounds_check,
                              int64_t* d_bad_pos, ag_stream_t s);

/* ================================================================================= *
 * Scalar expressions as one register program — the device half of ExecuteScalarExpression
 * (arrow/compute/exprs/exec.go:542-700) over expression trees (arrow/compute/expression.go: NewLiteral, NewFieldRef,
 * NewCall, Cast).  The host compiler (arrowgpu::compute::ExecuteScalarExpression) binds a tree through the registry,
 * emits it in post-order with registers in Sethi-Ullman order, and runs it with one launch of expr_eval_kernel over
 * every span of a record batch or table.
 *
 *   Registers hold one value per row (any of the 10 numeric types, or BOOL) and a validity bit per row.  Each op
 *   computes what the single-op kernel of its registered function computes in EVERY slot, nulls included:
 *     ADD SUB MUL BIT_AND BIT_OR BIT_XOR             ScalarBinary: every slot; validity = a & b
 *     ADD_CHECKED SUB_CHECKED DIV DIV_CHECKED SHL SHR SHL_CHECKED SHR_CHECKED
 *                                                    ScalarBinaryNotNull: computed where a and b are valid, 0 elsewhere;
 *                                                    overflow / zero divisor (integers: both DIVs; floats: DIV_CHECKED) /
 *                                                    shift out of range (the _CHECKED shifts) fails the program
 *     MUL_CHECKED                                    every slot, fails on overflow in ANY slot (checked multiply)
 *     ABS NEG NEG_UNSIGNED_ZERO SIGN BIT_NOT         every slot; validity = a
 *     ABS_CHECKED NEG_CHECKED                        signed integers, every slot, MinInt fails
 *     EQ NE GT GE LT LE                              BOOL result, every slot; validity = a & b
 *     AND OR XOR AND_NOT / NOT                       BOOL, every slot; validity = a & b / a
 *     KLEENE_AND KLEENE_OR KLEENE_AND_NOT            the Kleene truth tables of scalar_boolean.go:42-46
 *     IS_NULL IS_NOT_NULL IS_NAN                     BOOL result, no nulls
 *     CAST                                           type -> out_type; fails at a valid row as the checked cast does,
 *                                                    unless `flags` allows int overflow / float truncation
 *     LOAD                                           dst <- column a (type = the column's type)
 *     CONST                                          dst <- `bits` (raw little-endian value) in every row, valid iff
 *                                                    flags & 1
 *     NULL_OF                                        dst <- out_type value 0, every row null (a is evaluated first and
 *                                                    its failures count): a checked op with a null literal operand
 *   `type` is the operand type, `out_type` the result type (CAST, NULL_OF: the target; other ops: what the op gives).
 *
 * ag_eval_program[_dev](prog, n_spans, spans, out, out_valid, error):
 *   spans: HOST array of n_spans * prog->n_cols chunk descriptors, span i column j at [i * n_cols + j]; every column of
 *   a span has the span's length, offsets are element offsets (bit offsets for BOOL values and every bitmap) and need
 *   not be multiples of 8; a NULL validity pointer means no nulls.  Output rows start at 0 in span order: `out` holds
 *   the values (BOOL: a bitmap), `out_valid` (may be NULL) the validity; output bitmaps are written in whole 32-bit
 *   words and must be 4-byte aligned.  Device flavour: the span pointers are device pointers and *d_error_word
 *   (reset with ag_error_word_reset_dev) is lowered to the lowest failing output row.  Host flavour: host pointers,
 *   a failing program returns AG_ERR_INVALID "expression failed at row %lld" and stores the row in *first_bad (may
 *   be NULL).  A malformed program — an unknown op, a register or column index out of range, operand types that do
 *   not fit the op, more than AG_EXPR_MAX_* instructions or columns — is AG_ERR_INVALID before any launch.
 * ================================================================================= */
#define AG_EXPR_MAX_REGS   8
#define AG_EXPR_MAX_COLS  16
#define AG_EXPR_MAX_INSTR 128
#define AG_EXPR_LOAD               0
#define AG_EXPR_CONST              1
#define AG_EXPR_NULL_OF            2
#define AG_EXPR_ADD                3
#define AG_EXPR_SUB                4
#define AG_EXPR_MUL                5
#define AG_EXPR_ADD_CHECKED        6
#define AG_EXPR_SUB_CHECKED        7
#define AG_EXPR_MUL_CHECKED        8
#define AG_EXPR_DIV                9
#define AG_EXPR_DIV_CHECKED       10
#define AG_EXPR_BIT_AND           11
#define AG_EXPR_BIT_OR            12
#define AG_EXPR_BIT_XOR           13
#define AG_EXPR_SHL               14
#define AG_EXPR_SHR               15
#define AG_EXPR_SHL_CHECKED       16
#define AG_EXPR_SHR_CHECKED       17
#define AG_EXPR_ABS               18
#define AG_EXPR_NEG               19
#define AG_EXPR_NEG_UNSIGNED_ZERO 20
#define AG_EXPR_SIGN              21
#define AG_EXPR_BIT_NOT           22
#define AG_EXPR_ABS_CHECKED       23
#define AG_EXPR_NEG_CHECKED       24
#define AG_EXPR_EQ                25
#define AG_EXPR_NE                26
#define AG_EXPR_GT                27
#define AG_EXPR_GE                28
#define AG_EXPR_LT                29
#define AG_EXPR_LE                30
#define AG_EXPR_AND               31
#define AG_EXPR_OR                32
#define AG_EXPR_XOR               33
#define AG_EXPR_AND_NOT           34
#define AG_EXPR_KLEENE_AND        35
#define AG_EXPR_KLEENE_OR         36
#define AG_EXPR_KLEENE_AND_NOT    37
#define AG_EXPR_NOT               38
#define AG_EXPR_IS_NULL           39
#define AG_EXPR_IS_NOT_NULL       40
#define AG_EXPR_IS_NAN            41
#define AG_EXPR_CAST              42
#define AG_EXPR_ALLOW_INT_OVERFLOW   1 /* CAST flags */
#define AG_EXPR_ALLOW_FLOAT_TRUNCATE 2
typedef struct ag_expr_instr {
  int32_t op, type, out_type;
  int32_t dst, a, b;   /* registers; LOAD: a = column */
  int32_t flags;       /* CONST: 1 = valid; CAST: AG_EXPR_ALLOW_* */
  uint64_t bits;       /* CONST: the value */
} ag_expr_instr;
typedef struct ag_expr_program {
  int32_t n_instr;
  const ag_expr_instr* instr;  /* host memory */
  int32_t n_cols;
  const int32_t* col_types;    /* host memory: AG_TYPE_BOOL or a numeric type per column */
  int32_t out_reg;
} ag_expr_program;
ag_status ag_eval_program(const ag_expr_program* prog, int64_t n_spans, const ag_sort_chunk* spans, void* out, uint8_t* out_valid,
                          int64_t* first_bad);
ag_status ag_eval_program_dev(const ag_expr_program* prog, int64_t n_spans, const ag_sort_chunk* spans, void* out,
                              uint8_t* out_valid, int64_t* d_error_word, ag_stream_t s);

/* ================================================================================= *
 * Parquet decode primitives (SURVEY 8f rank 4: the feeder side) — the SIMD leaf loops arrow-go links under
 *   parquet/internal, so pages can be decoded into device-resident Arrow buffers.
 *   ag_parquet_unpack32 ↔ unpack32_avx2 (parquet/internal/utils/_lib/bit_packing_avx2.c:1772): values of
 *     num_bits (0..32) bits, LSB-first, 32 per group -> uint32; only whole groups are unpacked
 *     (batch_size/32*32, returned in *unpacked) — the caller handles the tail like BitReader.GetBatch.
 *     d_in 4-byte aligned, d_out 16-byte aligned.
 *   ag_parquet_bytes_to_bools ↔ bytes_to_bools (utils/_lib/unpack_bool.c:21): bit j of byte i -> out[8i+j] (0/1).
 *   ag_parquet_def_levels_to_bitmap ↔ DefLevelsToBitmap (parquet/file/level_conversion.go:134-184 over
 *     levels_to_bitmap / extract_bits, bmi/_lib/bitmap_bmi2.c:24-47): appends validity bits at
 *     valid_bits_offset.  repeated_ancestor_def_level < 0: no repeated parent — bit i = def[i] >= def_level,
 *     values_read = n (error if n > read_upper_bound).  Otherwise only slots with def >= the ancestor level
 *     produce a bit.  *null_count is INCREMENTED by values_read - set bits (like the reference); the device
 *     flavour returns {values_read, set bits} in d_counts[2].  n == 0 leaves valid_bits untouched.
 * ================================================================================= */
ag_status ag_parquet_unpack32(const uint32_t* in, uint32_t* out, int64_t batch_size, int num_bits, int64_t* unpacked);
ag_status ag_parquet_unpack32_dev(const uint32_t* d_in, uint32_t* d_out, int64_t batch_size, int num_bits, int64_t* unpacked, ag_stream_t s);
ag_status ag_parquet_bytes_to_bools(const uint8_t* bytes, int64_t len, uint8_t* out, int64_t outlen);
ag_status ag_parquet_bytes_to_bools_dev(const uint8_t* d_bytes, int64_t len, uint8_t* d_out, int64_t outlen, ag_stream_t s);
ag_status ag_parquet_def_levels_to_bitmap(const int16_t* def_levels, int64_t n, int def_level, int repeated_ancestor_def_level,
                                          uint8_t* valid_bits, int64_t valid_bits_offset, int64_t read_upper_bound,
                                          int64_t* values_read, int64_t* null_count);
ag_status ag_parquet_def_levels_to_bitmap_dev(const int16_t* d_def_levels, int64_t n, int def_level, int repeated_ancestor_def_level,
                                              uint8_t* d_valid_bits, int64_t valid_bits_offset, int64_t read_upper_bound,
                                              int64_t* d_counts, ag_stream_t s);

/* ================================================================================= *
 * Parquet page decode — a batch of pages in one call.  The page payloads (decompressed) sit in one buffer `data`;
 *   `pages` is a HOST array of descriptors in both flavours (like ag_span3):
 *     data        byte offset of the page's stream in `data`
 *     len         bytes available to the stream
 *     num_values  output slots of the page (valid + null slots for a spaced decode)
 *     out         element offset of the page's first slot in `out`; also its bit offset in `valid`
 *   Pages may come in any order and their outputs need not be contiguous.  Runs follow RleDecoder.Next / GetBatch
 *   (parquet/internal/utils/rle.go:123-169,203-239).  A stream that ends cleanly before num_values is not an
 *   error: decoded[i] says how many slots page i wrote (GetBatch's `read`); slots past it are left untouched.
 *   Differences from the reference (DESIGN §2):
 *     - bit widths 0..32 for indices, 0..16 for levels; anything else is AG_ERR_INVALID (the reference rejects
 *       only widths >= 64 and truncates a repeated value wider than 32 bits);
 *     - a truncated literal run, a run count of 0, a varint that runs past the stream / 5 bytes / int32 counts
 *       and a repeated value cut off by the end of the stream are AG_ERR_INVALID naming the page (the reference's
 *       Next() returns false on all but the first).  A truncated literal run still delivers its whole 32-value
 *       groups that are present (bit_reader_test.go:513-566);
 *     - a dictionary index >= dict_len is AG_ERR_INVALID "invalid index values found for dictionary converter"
 *       with the lowest offending output slot in *bad_pos, dense and spaced alike (the reference's dense path
 *       returns a short count instead); the slot holds 0.
 *   The device flavours synchronise `s` once, to read the per-page error codes back; d_decoded (may be NULL) is a
 *   device array of n_pages counts, *d_bad_pos (may be NULL) is overwritten (AG_NO_ERROR_POS when every index
 *   is in range, n_pages == 0 included).  Host flavours: decoded (may be NULL) and bad_pos (may be NULL) are host memory.
 *
 *   ag_parquet_levels_decode: LevelDecoder.SetData / SetDataV2 / Decode (parquet/internal/encoding/levels.go:188-297).
 *     Bit width = bits.Len(max_level).  AG_PQ_LEVELS_V1_RLE: a data page v1's level section, a 4-byte
 *     little-endian length then the stream ("received invalid levels / invalid number of bytes (corrupt data
 *     page?)" when it does not fit); AG_PQ_LEVELS_V2_RLE: the stream alone (len = the v2 header's byte length).
 *     AG_PQ_LEVELS_BIT_PACKED (deprecated) is AG_ERR_NOT_IMPLEMENTED.  Output int16 levels.
 *   ag_parquet_dict_decode: dictDecoder.SetData / decode / decodeSpaced (parquet/internal/encoding/decoder.go:125-160)
 *     over TypedRleDecoder.GetBatchWithDict[Spaced] (utils/typed_rle_dict.go:143-236).  The first byte of a page is
 *     its bit width; an empty page has bit width 0.  value_width 4 or 8 (int32/float, int64/double); `dict` is
 *     aligned to it.  valid == NULL: dense output; otherwise slots whose bit is clear get 0 and the others take the
 *     page's values in order; decoded counts slots.
 *   ag_parquet_plain_decode_spaced: PlainDecoder.DecodeSpaced (plain_encoding_types.go:98) -> spacedExpand
 *     (decoder.go:209) for the PLAIN pages of optional columns (what a writer falls back to once the dictionary
 *     is full).  A page needs value_width bytes per valid slot ("eof exception decode plain" otherwise).  A
 *     required PLAIN page is a plain copy and needs no entry point.
 * ================================================================================= */
typedef struct ag_pq_page {
  int64_t data;
  int64_t len;
  int64_t num_values;
  int64_t out;
} ag_pq_page;
#define AG_PQ_LEVELS_V2_RLE     0
#define AG_PQ_LEVELS_V1_RLE     1
#define AG_PQ_LEVELS_BIT_PACKED 2
ag_status ag_parquet_levels_decode(int max_level, int encoding, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages,
                                   int16_t* out, int64_t* decoded);
ag_status ag_parquet_levels_decode_dev(int max_level, int encoding, const uint8_t* d_data, const ag_pq_page* pages, int64_t n_pages,
                                       int16_t* d_out, int64_t* d_decoded, ag_stream_t s);
ag_status ag_parquet_dict_decode(int value_width, const void* dict, int64_t dict_len, const uint8_t* data, const ag_pq_page* pages,
                                 int64_t n_pages, const uint8_t* valid, void* out, int64_t* decoded, int64_t* bad_pos);
ag_status ag_parquet_dict_decode_dev(int value_width, const void* d_dict, int64_t dict_len, const uint8_t* d_data, const ag_pq_page* pages,
                                     int64_t n_pages, const uint8_t* d_valid, void* d_out, int64_t* d_decoded, int64_t* d_bad_pos, ag_stream_t s);
ag_status ag_parquet_plain_decode_spaced(int value_width, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages,
                                         const uint8_t* valid, void* out);
ag_status ag_parquet_plain_decode_spaced_dev(int value_width, const uint8_t* d_data, const ag_pq_page* pages, int64_t n_pages,
                                             const uint8_t* d_valid, void* d_out, ag_stream_t s);

/* ================================================================================= *
 * DELTA_BINARY_PACKED INT32 / INT64 pages — the same batch-of-pages contract as ag_parquet_dict_decode (host page
 *   table, any page order, valid == NULL for dense output, decoded[i] in slots, the device flavour synchronises `s`
 *   once).  value_width 4 (INT32) or 8 (INT64), anything else AG_ERR_INVALID; `out` aligned to it.
 *   deltaBitPackDecoder (parquet/internal/encoding/delta_bit_packing.go): SetData (:72-133, called with the page's
 *   num_values, file/column_reader.go:527), initBlock (:136-160), unpackNextMini (:162-216), Decode (:264-302),
 *   DecodeSpaced (:305-316).  Each error is AG_ERR_INVALID naming the page, with the reference's message:
 *     - the header (block size, miniblocks per block, total values, first value) is always parsed, even when the
 *       page needs no value: a missing, truncated or over-64-bit varint is "parquet: eof exception"; the block size,
 *       miniblock and values-per-miniblock checks and "invalid delta value count %d for %d buffered values"
 *       (total > 2^32-1 or > num_values) are SetData's; INT32: "initial delta value %d exceeds INT32 range";
 *     - blocks and miniblocks are read lazily, as the reference reads them: only those holding one of the first
 *       min(need, total) - 1 deltas are read ("touched"; need = num_values dense, the page's valid bits spaced).
 *       A touched block: min delta ("parquet: eof exception", INT32: "minimum delta %d exceeds INT32 range"), then
 *       all its width bytes ("failed to read byte").  A touched miniblock: width <= 32 (INT32) / 64 (INT64)
 *       ("delta bit width %d exceeds decoder width %d") and its whole payload of vpm*width/8 bytes present, even
 *       when only part of it is needed ("unexpected EOF").  Widths of miniblocks past the last needed delta are
 *       never looked at, and a stream may end right after the last needed miniblock;
 *     - dense, total < num_values: not an error, decoded = total (Decode's short count);
 *     - spaced, total < valid slots: "parquet: number of values / definition levels read did not match", decoded =
 *       0 and nothing is written (as for a short PLAIN page).
 *   value[k] = value[k-1] + delta + min_delta modulo 2^(8*value_width): every sum wraps at the physical width, so the
 *   result is bit-exact in any summation order, and INT32 is computed in uint32 (the reference accumulates in int64
 *   and truncates, which gives the same bits).
 *   Differences from the reference (DESIGN §2):
 *     - an error inside the block chain still delivers the first value and every miniblock before the failing one;
 *       decoded says how many slots were written (spaced: every slot before the first valid slot whose value was
 *       not delivered), like a truncated literal run.  The reference's Decode returns (0, err).  A header error
 *       delivers no value (spaced: the null slots before the first valid slot get 0);
 *     - the page is decoded in parallel (a block walk, then a prefix sum of the deltas), not miniblock by miniblock.
 * ================================================================================= */
ag_status ag_parquet_delta_decode(int value_width, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages,
                                  const uint8_t* valid, void* out, int64_t* decoded);
ag_status ag_parquet_delta_decode_dev(int value_width, const uint8_t* d_data, const ag_pq_page* pages, int64_t n_pages,
                                      const uint8_t* d_valid, void* d_out, int64_t* d_decoded, ag_stream_t s);

/* ================================================================================= *
 * Page encoders: the value sections of data pages, as arrow-go's writer produces them, from device-resident values.
 *   Batch-of-pages calls in the shape of the decoders: `pages` is a HOST array in both flavours,
 *     in          element offset of the page's first value in `values` (bit offset for bitmap input)
 *     num_values  values to encode, 0 .. 2^31-1
 *     out         byte offset of the page's section in `out`
 *     capacity    bytes available there: at least the call's *_max_size bound for num_values (AG_ERR_INVALID
 *                 naming the page otherwise, before any launch)
 *   Pages may come in any order, share or skip input, and their sections need not be contiguous.  lengths[i] (may be
 *   NULL) receives the bytes page i wrote, prefix included.  Inputs are dense: dictionary indices and DELTA values are
 *   the valid values in order (compact a spaced column with ag_filter_primitive_dev and its validity as the mask).
 *   The device flavours synchronise `s` once (d_lengths and *d_bad_pos are device memory); host flavours stage the
 *   input the pages reach and copy back each page's written bytes.  Without a usable GPU every entry point returns
 *   AG_ERR_CUDA.
 *
 *   ag_parquet_rle_encode: the RLE/bit-packed hybrid stream of RleEncoder.Put / Flush (parquet/internal/utils/
 *     rle.go:314-445), byte for byte: repeated runs of >= 8 caught on the group alignment, literal runs of at most
 *     63 groups, a zero-padded last group.  Used by LevelEncoder (encoding/levels.go:77-169), dictEncoder.WriteIndices
 *     (encoding/encoder.go:293-302) and RleBooleanEncoder (encoding/boolean_encoder.go:185-).
 *     form  AG_PQ_RLE_BARE  the stream alone                        (data page v2 levels)
 *           AG_PQ_RLE_LEN4  4-byte little-endian length, the stream  (data page v1 levels, BOOLEAN RLE pages)
 *           AG_PQ_RLE_WIDTH 1 bit-width byte, the stream             (RLE_DICTIONARY / PLAIN_DICTIONARY data pages)
 *     input AG_PQ_RLE_IN_U32    uint32 dictionary indices, bit width 0..32
 *           AG_PQ_RLE_IN_I16    int16 levels, bit width 0..16
 *           AG_PQ_RLE_IN_BITMAP bits, bit width 1: definition levels of a flat optional column from its validity
 *                               bitmap, or BOOLEAN values
 *     A value wider than the bit width (a negative level included) is AG_ERR_INVALID naming the page, with the lowest
 *     offending element offset (into `values`) in *bad_pos; *bad_pos is AG_NO_ERROR_POS otherwise (may be NULL).  The
 *     reference's BitWriter.WriteValue does not mask and corrupts the neighbouring values (utils/bit_writer.go:115-130).
 *   ag_parquet_rle_max_size: MaxRLEBufferSize + MinRLEBufferSize (rle.go:36-51) plus the form's prefix.
 *   ag_parquet_delta_encode: deltaBitPackEncoder.Put / FlushValues (encoding/delta_bit_packing.go:338,362-494), byte
 *     for byte, with the block shape as a parameter (the reference fixes 128 values in 4 miniblocks; pyarrow writes
 *     INT64 pages with 256/4).  value_width 4 (INT32) or 8 (INT64), `values` aligned to it; deltas wrap at that
 *     width; the width bytes of absent miniblocks of the last block are 0 and the last miniblock is padded with zeros.
 *     A block size that is not a positive multiple of 128, a miniblock count that does not divide it, or values per
 *     miniblock that are not a multiple of 32 is AG_ERR_INVALID (the shapes deltaBitPackDecoder.SetData refuses).
 *   ag_parquet_delta_max_size: 40 header bytes, then per block of deltas 10 + miniblocks + block_size * value_width.
 * ================================================================================= */
typedef struct ag_pq_enc_page {
  int64_t in;
  int64_t num_values;
  int64_t out;
  int64_t capacity;
} ag_pq_enc_page;
#define AG_PQ_RLE_BARE      0
#define AG_PQ_RLE_LEN4      1
#define AG_PQ_RLE_WIDTH     2
#define AG_PQ_RLE_IN_U32    0
#define AG_PQ_RLE_IN_I16    1
#define AG_PQ_RLE_IN_BITMAP 2
ag_status ag_parquet_rle_max_size(int bit_width, int form, int64_t num_values, int64_t* size);
ag_status ag_parquet_rle_encode(int bit_width, int form, int input, const void* values, const ag_pq_enc_page* pages,
                                int64_t n_pages, uint8_t* out, int64_t* lengths, int64_t* bad_pos);
ag_status ag_parquet_rle_encode_dev(int bit_width, int form, int input, const void* d_values, const ag_pq_enc_page* pages,
                                    int64_t n_pages, uint8_t* d_out, int64_t* d_lengths, int64_t* d_bad_pos, ag_stream_t s);
ag_status ag_parquet_delta_max_size(int value_width, int block_size, int miniblocks, int64_t num_values, int64_t* size);
ag_status ag_parquet_delta_encode(int value_width, int block_size, int miniblocks, const void* values, const ag_pq_enc_page* pages,
                                  int64_t n_pages, uint8_t* out, int64_t* lengths);
ag_status ag_parquet_delta_encode_dev(int value_width, int block_size, int miniblocks, const void* d_values, const ag_pq_enc_page* pages,
                                      int64_t n_pages, uint8_t* d_out, int64_t* d_lengths, ag_stream_t s);

/* ================================================================================= *
 * BYTE_ARRAY pages into an Arrow Binary / String (offset_width 4, int32 offsets) or LargeBinary / LargeString
 *   (offset_width 8) array: `offsets` plus one data buffer, as arrow-go's byteArrayRecordReader builds with
 *   array.BinaryBuilder (parquet/file/record_reader.go:902-1030).  The same batch-of-pages contract as
 *   ag_parquet_dict_decode: a host page table, pages in any order, valid == NULL for dense output, pg.out is both the
 *   slot and the bit offset, decoded[i] counts page i's slots, and the device flavour synchronises `s` once.
 *   encoding is the parquet.thrift Encoding of the pages (AG_PQ_ENC_*); any other encoding or offset width is
 *   AG_ERR_INVALID.  Argument checks, AG_ERR_INVALID before any launch: a negative field, a page's slots past
 *   n_slots, and page slot ranges that overlap.
 *   Offsets.  `offsets` holds n_slots + 1 entries of offset_width bytes; offsets[0] = offset_base, and slot i's length
 *   is 0 when it is null, past its page's decoded count or covered by no page, so `offsets` is always a valid Arrow
 *   offsets buffer.  *total = offsets[n_slots] - offset_base.
 *   Data.  out_data is the array's whole data buffer: slot i's bytes go to out_data[offsets[i] .. offsets[i+1]).
 *   offset_base lets one chunk be decoded by chained calls (the dictionary-encoded pages, then the PLAIN pages a
 *   writer fell back to, with offset_base = the first call's total and `offsets` advanced to the second call's first
 *   slot).  When offset_base + *total > out_cap the call returns AG_OK with the offsets and *total written and no byte
 *   of out_data written, so out_data = NULL, out_cap = 0 is a size query.  PLAIN and DELTA_LENGTH_BYTE_ARRAY totals are
 *   bounded by the page bytes; dictionary and DELTA_BYTE_ARRAY totals are not.  The device decides whether the bytes
 *   fit.  With offset_width 4, offset_base + total > 2^31-1 is AG_ERR_INVALID and neither offsets nor data are written
 *   (arrow-go only debug.Asserts this, arrow/array/binarybuilder.go:347).
 *   Encodings (each error is AG_ERR_INVALID "byte_array_decode: page %lld: <message> (%lld values decoded)" naming the
 *   lowest failing page; every other page is decoded in full):
 *     AG_PQ_ENC_PLAIN: PlainByteArrayDecoder.Decode / DecodeSpaced (parquet/internal/encoding/byte_array_decoder.go:
 *       144-189): a 4-byte little-endian length, then the bytes.  "parquet: eof reading bytearray" when a length or a
 *       value is cut off, "parquet: invalid BYTE_ARRAY value" for a negative length.  Bytes after the last value the
 *       page's slots need are not looked at.
 *     AG_PQ_ENC_PLAIN_DICTIONARY / AG_PQ_ENC_RLE_DICTIONARY: dict_offsets (dict_len + 1 entries of offset_width) and
 *       dict_data are what this call produces from the dictionary page with AG_PQ_ENC_PLAIN, dense, offset_base 0
 *       (configureDict, parquet/file/column_reader.go:333-361).  Runs, bit widths, their messages and the
 *       out-of-range index (message, *bad_pos, a slot of length 0) are those of ag_parquet_dict_decode.
 *     AG_PQ_ENC_DELTA_LENGTH_BYTE_ARRAY: DeltaLengthByteArrayDecoder.SetData / Decode (delta_length_byte_array.go:
 *       113-188): every length of the DELTA_BINARY_PACKED INT32 stream is decoded and checked before any value is
 *       delivered (header and chain errors are ag_parquet_delta_decode's messages; "parquet: negative delta byte array
 *       length %d"; "parquet: delta byte array lengths exceed payload size").  The values start at the length
 *       stream's bytesRead(), the end of the miniblock holding the last length.
 *     AG_PQ_ENC_DELTA_BYTE_ARRAY: DeltaByteArrayDecoder.SetData / Decode (delta_byte_array.go:166-303): a stream of
 *       prefix lengths, then a DELTA_LENGTH_BYTE_ARRAY stream of suffixes.  "parquet: delta prefix and suffix length
 *       counts do not match"; "parquet: first delta byte array prefix length must be zero"; "parquet: invalid delta
 *       byte array prefix length %d" (negative, or longer than the previous value).  The previous value resets on
 *       every page and, spaced, is the previous valid value.
 *     A DELTA page with fewer values than valid slots (spaced) is "parquet: number of values / definition levels read
 *     did not match" and delivers nothing; dense, it delivers a short count.  The reference's "delta length / prefix
 *     count exceeds value count" and "not enough ..." checks cannot fire after the stream header's own count check.
 *   No UTF-8 validation, as in the reference.
 *   Differences from the reference (DESIGN §2):
 *     - a PLAIN value or a DELTA_BYTE_ARRAY prefix that fails still delivers the values before it; decoded says how
 *       many slots were written (the reference's Decode returns (0, err) for DELTA_BYTE_ARRAY);
 *     - the dictionary page is decoded in full up front (the reference's dictConverter reads it lazily);
 *     - offset_base + total > 2^31-1 with int32 offsets is an error, not a debug assertion.
 *   The device flavour: *total is host memory, d_decoded and d_bad_pos (may be NULL) device memory, *d_bad_pos is
 *   overwritten.  The host flavour stages `data`, `valid` and the dictionary, and copies back the offsets and only
 *   the bytes it wrote; out_data outside them is untouched.
 * ================================================================================= */
#define AG_PQ_ENC_PLAIN                   0
#define AG_PQ_ENC_PLAIN_DICTIONARY        2
#define AG_PQ_ENC_DELTA_LENGTH_BYTE_ARRAY 6
#define AG_PQ_ENC_DELTA_BYTE_ARRAY        7
#define AG_PQ_ENC_RLE_DICTIONARY          8
ag_status ag_parquet_byte_array_decode(int encoding, int offset_width, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages,
                                       int64_t n_slots, const uint8_t* valid, const void* dict_offsets, const uint8_t* dict_data,
                                       int64_t dict_len, int64_t offset_base, void* offsets, uint8_t* out_data, int64_t out_cap,
                                       int64_t* total, int64_t* decoded, int64_t* bad_pos);
ag_status ag_parquet_byte_array_decode_dev(int encoding, int offset_width, const uint8_t* d_data, const ag_pq_page* pages, int64_t n_pages,
                                           int64_t n_slots, const uint8_t* d_valid, const void* d_dict_offsets, const uint8_t* d_dict_data,
                                           int64_t dict_len, int64_t offset_base, void* d_offsets, uint8_t* d_out_data, int64_t out_cap,
                                           int64_t* total, int64_t* d_decoded, int64_t* d_bad_pos, ag_stream_t s);

/* ================================================================================= *
 * BYTE_ARRAY page encoders: the value sections of data pages from an Arrow Binary / String (offset_width 4) or
 *   LargeBinary / LargeString (offset_width 8) array, as arrow-go's writer produces them.  The page encoders' batch
 *   contract (ag_pq_enc_page, a HOST array in both flavours), except that the input is spaced: slot i is bit i of
 *   `valid` (NULL: every slot valid) and the bytes data[offsets[i] .. offsets[i+1]); a null slot is skipped whatever
 *   its length.  pg.in is the page's first slot, pg.num_values its slots (nulls included, 0 .. 2^31-1); a slice is a
 *   page table, so there is no offset argument.  Pages may come in any order, share or skip slots, and their sections
 *   need not be contiguous.  lengths[i] (may be NULL) receives the bytes page i wrote.
 *     AG_PQ_ENC_PLAIN: PlainByteArrayEncoder.Put / PutSpaced (parquet/internal/encoding/byte_array_encoder.go:41-89):
 *       each valid value as a 4-byte little-endian length and its bytes.  Also the dictionary page of a string
 *       dictionary: with valid = NULL over the entries, or over a column's slots with valid = the `first` bitmap of
 *       ag_parquet_byte_array_dict_encode.
 *     AG_PQ_ENC_DELTA_LENGTH_BYTE_ARRAY: DeltaLengthByteArrayEncoder (delta_length_byte_array.go:44-96): the lengths as
 *       a DELTA_BINARY_PACKED INT32 stream, then the values' bytes back to back.
 *     AG_PQ_ENC_DELTA_BYTE_ARRAY: DeltaByteArrayEncoder (delta_byte_array.go:56-149): the lengths of the prefixes each
 *       valid value shares with the previous valid value of the page as a DELTA_BINARY_PACKED INT32 stream, then the
 *       suffixes as a DELTA_LENGTH_BYTE_ARRAY section.
 *     The length streams use the reference's block shape, 128 values in 4 miniblocks (delta_bit_packing.go:338-339),
 *     byte for byte as ag_parquet_delta_encode writes them.
 *   ag_parquet_byte_array_max_size: with value_bytes = offsets[in + n] - offsets[in] (0 .. 2^62), PLAIN 4n + value_bytes,
 *     DELTA_LENGTH_BYTE_ARRAY delta(n) + value_bytes, DELTA_BYTE_ARRAY 2 delta(n) + value_bytes, where delta(n) is
 *     ag_parquet_delta_max_size(4, 128, 4, n).  It needs no GPU.
 *   Checks, every one AG_ERR_INVALID before any output byte is written:
 *     on the host: an unknown encoding or offset width, a page-table error of the page encoders (negative field,
 *       num_values past 2^31-1), and NULL offsets, data or output that a page reaches;
 *     on the device, by one pass over the offsets and validity the pages reach (never `data`), naming the lowest
 *       failing page: a capacity below the page's bound; then, for the slot errors, with the page's lowest offending
 *       slot in *bad_pos: a negative offsets[in], offsets that decrease inside the page, a valid value longer than
 *       2^31-1 bytes.  A page with a slot error is reported for it rather than for its capacity.  *bad_pos is
 *       AG_NO_ERROR_POS otherwise (may be NULL).
 *   The device flavour synchronises `s` once, after the checking pass, and leaves the encode stream-ordered: no error
 *   depends on the data after it.  d_lengths and *d_bad_pos are device memory; *d_bad_pos is written once the checking
 *   pass has run.  The kernels read d_data in whole aligned 16-byte words, so they may read up to 15 bytes before
 *   the first and after the last data byte a page reaches, never outside the aligned 16-byte words holding those bytes:
 *   d_data must be readable there, as a cudaMalloc allocation (256-byte aligned) or a padded Arrow buffer (64 bytes)
 *   is.  The host flavour stages the offsets and validity the pages reach, then the data bytes they reach, and copies
 *   back each page's written bytes.  Without a usable GPU both flavours return AG_ERR_CUDA.
 *   Differences from the reference (DESIGN §2):
 *     - DELTA_BYTE_ARRAY: every page starts fresh (its first valid value has prefix 0), as parquet-cpp writes it; the
 *       reference carries the previous page's last value into the next page, which its own decoder refuses;
 *     - a valid value longer than 2^31-1 bytes is refused; the reference writes uint32(len) unchecked.
 * ================================================================================= */
ag_status ag_parquet_byte_array_max_size(int encoding, int64_t num_values, int64_t value_bytes, int64_t* size);
ag_status ag_parquet_byte_array_encode(int encoding, int offset_width, const void* offsets, const uint8_t* data,
                                       const uint8_t* valid, const ag_pq_enc_page* pages, int64_t n_pages,
                                       uint8_t* out, int64_t* lengths, int64_t* bad_pos);
ag_status ag_parquet_byte_array_encode_dev(int encoding, int offset_width, const void* d_offsets, const uint8_t* d_data,
                                           const uint8_t* d_valid, const ag_pq_enc_page* pages, int64_t n_pages,
                                           uint8_t* d_out, int64_t* d_lengths, int64_t* d_bad_pos, ag_stream_t s);

/* ================================================================================= *
 * BYTE_ARRAY dictionaries: the memo table of DictByteArrayEncoder (parquet/internal/encoding/byte_array_encoder.go:
 *   97-135, encoder.go:241-325) over a column chunk of Arrow Binary / String (offset_width 4) or LargeBinary /
 *   LargeString (offset_width 8) arrays.  Every valid value is keyed on its raw bytes, so the dictionary's entries come in
 *   order of first appearance; nulls are skipped.
 *   chunks: a HOST array of n_chunks descriptors in table order, in both flavours.  Slot i of a chunk is bit i of
 *     `valid` (NULL: every slot valid) and the bytes data[offsets[i] .. offsets[i+1]); the chunk holds slots
 *     [offset, offset + length).  The slots of all chunks are numbered in turn ("global slots"), at most 2^31-1 of
 *     them (more is AG_ERR_NOT_IMPLEMENTED), and share one dictionary.
 *   Outputs:
 *     indices      one uint32 per valid slot of all chunks, in order: entry k is the k-th distinct value.  This is the
 *                  input of ag_parquet_rle_encode with AG_PQ_RLE_IN_U32.
 *     chunk.first  bit i set iff slot i of the chunk is the first valid appearance of its value in the call, in the
 *                  chunk's own slot numbering.  Written in whole aligned 32-bit words covering [offset, offset + length),
 *                  with the bits outside those slots cleared: ceil((offset + length) / 32) * 4 bytes, 4-byte aligned.
 *                  ag_parquet_byte_array_encode(AG_PQ_ENC_PLAIN) with valid = first over the chunk's slots writes the
 *                  chunk's share of the dictionary page; over a one-chunk column, the whole page.
 *     counts[3]    the dictionary's entries, the entries' value bytes (sum of len), and the valid slots.
 *     mark_counts  for every global slot position marks[j] in [0, total slots] (a HOST array; may be NULL when n_marks
 *                  is 0): [2j] the entries first seen at a slot below marks[j], [2j + 1] their dictEncodedSize (the sum
 *                  of len + 4: the size of the PLAIN dictionary page).  The dictionary of any prefix of the slots is a
 *                  prefix of the whole dictionary and the prefix's indices are unchanged, so marks at page ends give
 *                  each page's index bit width (BitWidth() of the entries so far: 0 for none, 1 for one, else
 *                  bits.Len32(entries - 1)) and marks at the writer's batch ends give its fallback cut.
 *   Checks, every one before any output is written:
 *     on the host, before the device is touched (AG_ERR_INVALID): an unknown offset width; a negative chunk offset or
 *       length; NULL offsets, data or first of a non-empty chunk, or a first bitmap that is not 4-byte aligned; a mark
 *       outside [0, total slots]; NULL indices (with slots), counts, or mark_counts (with marks);
 *     on the device, by one pass over the offsets and validity (never `data`), as ag_parquet_byte_array_encode makes
 *       them: a negative first offset of a chunk, offsets that decrease, a valid value longer than 2^31-1 bytes.  Each
 *       is AG_ERR_INVALID naming the chunk, with the lowest offending global slot in *bad_pos (AG_NO_ERROR_POS
 *       otherwise; may be NULL).
 *   The device flavour synchronises `s` once, after that pass; the rest is stream-ordered.  d_indices, d_mark_counts,
 *   d_counts and *d_bad_pos are device memory.  `data` is read in whole aligned 16-byte words under the rule of
 *   ag_parquet_byte_array_encode.  ag_unique_set_policy applies to the table.  The host flavour stages what the chunks
 *   reach and copies back indices, every first bitmap, counts and mark_counts.  Without a usable GPU both flavours
 *   return AG_ERR_CUDA once the host checks pass.
 * ================================================================================= */
typedef struct ag_pq_ba_chunk {
  const void*    offsets;   /* offset_width bytes each; slot i uses offsets[i], offsets[i+1] */
  const uint8_t* data;
  const uint8_t* valid;     /* may be NULL */
  int64_t        offset;    /* first slot of the chunk */
  int64_t        length;    /* slots */
  uint8_t*       first;     /* out: first-appearance bitmap */
} ag_pq_ba_chunk;
ag_status ag_parquet_byte_array_dict_encode(int offset_width, const ag_pq_ba_chunk* chunks, int64_t n_chunks,
                                            const int64_t* marks, int64_t n_marks, uint32_t* indices,
                                            int64_t* mark_counts, int64_t* counts, int64_t* bad_pos);
ag_status ag_parquet_byte_array_dict_encode_dev(int offset_width, const ag_pq_ba_chunk* chunks, int64_t n_chunks,
                                                const int64_t* marks, int64_t n_marks, uint32_t* d_indices,
                                                int64_t* d_mark_counts, int64_t* d_counts, int64_t* d_bad_pos,
                                                ag_stream_t s);

/* ================================================================================= *
 * BOOLEAN, INT32 / INT64 / FLOAT / DOUBLE, INT96 and FIXED_LEN_BYTE_ARRAY pages — the same batch-of-pages contract as
 *   ag_parquet_dict_decode: a host page table, pages in any order, valid == NULL for dense output, pg.out is both the
 *   slot and the bit offset in `valid`, decoded[i] counts page i's slots, and the device flavour synchronises `s`
 *   once.  Each error is AG_ERR_INVALID "<fn>: page %lld: <message> (%lld values decoded)" naming the lowest failing
 *   page; every other page is decoded in full.  A spaced page with fewer values than valid slots cannot occur for
 *   BOOLEAN, whose value count is the page's slot count.
 *
 *   ag_parquet_bool_decode: PlainBooleanDecoder / RleBooleanDecoder .DecodeToBitmap and decodeSpacedToBitmap
 *   (parquet/internal/encoding/boolean_decoder.go:264-304,321-341,382-417), as record_reader.go:331-370 calls them:
 *   an Arrow boolean bitmap.  encoding AG_PQ_ENC_PLAIN or AG_PQ_ENC_RLE.  pg.out is the page's first bit in `valid`
 *   and in `out_bits`; a null slot gets 0.  Bits outside [pg.out, pg.out + decoded[i]) of every page are left
 *   untouched, also where two pages share a byte or a 32-bit word of out_bits.  Pages sharing a byte are decoded at
 *   the same time, so the device flavour merges a partly written word with 32-bit atomics on the aligned word: d_out_bits
 *   must be readable and writable through every aligned 4-byte word that holds a bit of a page (a cudaMalloc buffer
 *   rounded up to a multiple of 4 bytes is); the bytes of those words outside the pages keep their values.  The host
 *   flavour stages the bitmap, so out_bits needs only its own bytes.
 *     AG_PQ_ENC_PLAIN: bit-packed, LSB first.  "parquet: boolean data has %d bits available, need %d: unexpected EOF"
 *       when the page holds fewer bits than the values it needs (valid slots); nothing of the page is delivered.
 *     AG_PQ_ENC_RLE: a 4-byte little-endian length on every page (v1 and v2), then an RLE / bit-packed stream of bit
 *       width 1.  "invalid length - %d (corrupt data page?)" (page shorter than 4 bytes) and "received invalid number
 *       of bytes - %d (corrupt data page?)" (length past the page) deliver nothing.  A stream that ends before the
 *       values the page needs is "unexpected EOF" after the values delivered (DecodeToBitmap's io.ErrUnexpectedEOF;
 *       unlike a level stream's short count).  Bad run headers are the run-walk messages of ag_parquet_dict_decode.
 *
 *   ag_parquet_fixed_decode: values of width 4 (INT32, FLOAT), 8 (INT64, DOUBLE), 12 (INT96) or type_length
 *   (FIXED_LEN_BYTE_ARRAY; type_length is ignored for the other types) bytes per slot in `out`; a null slot gets zero
 *   bytes (record_reader.go:847-871 AppendNull).  Accepted encodings (typed_encoder.go:250-291,432-437,714-727):
 *   INT32 / INT64 / FLOAT / DOUBLE and FIXED_LEN_BYTE_ARRAY: PLAIN, PLAIN_DICTIONARY / RLE_DICTIONARY and
 *   BYTE_STREAM_SPLIT; INT96: PLAIN and dictionary.  Any other type, encoding or a type_length < 1 is AG_ERR_INVALID
 *   before any launch.  For widths 4 and 8, `out` and `dict` are aligned to the width; other widths have no alignment
 *   requirement.
 *     AG_PQ_ENC_PLAIN (plain_encoding_types.go:61-110, fixed_len_byte_array_decoder.go): dense or spaced, so one call
 *       replaces one copy per page.  A page with fewer values than it needs delivers nothing: widths 4 / 8 "parquet:
 *       eof exception decode plain (fewer values than valid slots)" (ag_parquet_plain_decode_spaced's message), INT96
 *       "parquet: eof exception decode plain INT96, nvals: %d, nbytes: %d, datalen: %d", FIXED_LEN_BYTE_ARRAY
 *       "parquet: eof exception".
 *     AG_PQ_ENC_PLAIN_DICTIONARY / AG_PQ_ENC_RLE_DICTIONARY: `dict` holds dict_len values of the width, which this call
 *       produces from the dictionary page with AG_PQ_ENC_PLAIN, dense (so its length is checked too).  Runs, bit
 *       widths, their messages and an out-of-range index (message, *bad_pos, a zeroed slot) are those of
 *       ag_parquet_dict_decode.
 *     AG_PQ_ENC_BYTE_STREAM_SPLIT (byte_stream_split.go:98-250, fixed_len_byte_array_decoder.go): byte j of the value
 *       of dense rank r is data[j * stride + r], stride = len / width.  "data size (%d) is too small for the number of
 *       values in in BYTE_STREAM_SPLIT (%d)" when the page holds more than num_values values (the reference's wording);
 *       "ByteStreamSplit data size %d not aligned with byte_width: %d" (FIXED_LEN_BYTE_ARRAY: "... not aligned with type
 *       FIXED_LEN_BYTE_ARRAY and byte_width: %d"); "parquet: eof exception" when the values to read take more than
 *       2^31-1 bytes; spaced, fewer values than valid slots: "parquet: number of values / definitions levels read did
 *       not match".  Each delivers nothing.  Dense, a page with fewer values than slots delivers stride slots.
 *   Differences from the reference (DESIGN §2): a boolean null slot is 0 (decodeSpacedToBitmap can leave packed bits
 *   there); an RLE boolean repeated byte other than 0 or 1 is true (value != 0, rle.go:161-165 does not mask it); a
 *   BYTE_STREAM_SPLIT page's value count is its stride, len / width (SetData replaces nvals with it).
 *   Device flavours: d_decoded (may be NULL) is device memory; *d_bad_pos (may be NULL) is overwritten
 *   (AG_NO_ERROR_POS when every index is in range, n_pages == 0 included).  Host flavours: decoded and bad_pos (may be NULL) are host
 *   memory; they stage `data`, `valid`, the dictionary and (booleans) the output bitmap's bytes up to the last page's
 *   last slot, and copy back only what the call wrote, so the rest of `out` / `out_bits` is untouched.
 * ================================================================================= */
#define AG_PQ_ENC_RLE                     3
#define AG_PQ_ENC_BYTE_STREAM_SPLIT       9
#define AG_PQ_TYPE_INT32                  1
#define AG_PQ_TYPE_INT64                  2
#define AG_PQ_TYPE_INT96                  3
#define AG_PQ_TYPE_FLOAT                  4
#define AG_PQ_TYPE_DOUBLE                 5
#define AG_PQ_TYPE_FIXED_LEN_BYTE_ARRAY   7
ag_status ag_parquet_bool_decode(int encoding, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages, const uint8_t* valid,
                                 uint8_t* out_bits, int64_t* decoded);
ag_status ag_parquet_bool_decode_dev(int encoding, const uint8_t* d_data, const ag_pq_page* pages, int64_t n_pages, const uint8_t* d_valid,
                                     uint8_t* d_out_bits, int64_t* d_decoded, ag_stream_t s);
ag_status ag_parquet_fixed_decode(int physical_type, int type_length, int encoding, const uint8_t* data, const ag_pq_page* pages,
                                  int64_t n_pages, const uint8_t* valid, const void* dict, int64_t dict_len, void* out, int64_t* decoded,
                                  int64_t* bad_pos);
ag_status ag_parquet_fixed_decode_dev(int physical_type, int type_length, int encoding, const uint8_t* d_data, const ag_pq_page* pages,
                                      int64_t n_pages, const uint8_t* d_valid, const void* d_dict, int64_t dict_len, void* d_out,
                                      int64_t* d_decoded, int64_t* d_bad_pos, ag_stream_t s);

/* ================================================================================= *
 * SNAPPY page decompression — a batch of pages in one call, so that a reader uploads a column chunk as it sits in the
 *   file and decodes it in device memory.  The output is what the page decoders above take (`ag_pq_page` offsets then
 *   point into `dst`).  serializedPageReader.decompress (parquet/file/page_reader.go:597-621) -> compress.Decode
 *   (parquet/compress/compress.go:107) -> snappyCodec.DecodeWithError (parquet/compress/snappy.go:43-45).
 *     src      byte offset of the page's compressed bytes in `src`
 *     src_len  compressed bytes
 *     dst      byte offset of the page's output in `dst` (any byte offset)
 *     dst_len  the page header's uncompressed size (a v2 page: minus its level bytes, which are never compressed)
 *   `pages` is a HOST array in both flavours; pages may come in any order.  written (may be NULL) receives the bytes
 *   each page wrote.  The device flavour synchronises `s` once, to read the per-page error codes back; d_written is a
 *   device array.  The host flavour stages `src` and `dst` through device memory and copies back only written bytes.
 *   `src` and `dst` must not overlap (not checked).
 *   Argument checks, AG_ERR_INVALID before any launch: a negative field, src_len or dst_len above 2^32-1, and dst
 *   ranges that overlap each other (empty ranges overlap nothing).
 *   Format: raw Snappy, with the checks golang/snappy's decode makes.  A preamble holds the uncompressed length as a
 *   binary.Uvarint (missing, overflowing or above 0xffffffff is corrupt), then elements by the low two tag bits:
 *     00 literal, length-1 = tag>>2, or for 60..63 the next 1..4 bytes little-endian;
 *     01 copy, length 4+((tag>>2)&7), 11-bit offset (tag>>5)<<8 | next byte;
 *     10 copy, length 1+(tag>>2), 2-byte offset;   11 copy, length 1+(tag>>2), 4-byte offset.
 *   Copies may overlap their own output (offset < length).  Corrupt: a literal or an offset cut off by the end of the
 *   stream; a copy with offset 0 or an offset greater than the bytes produced so far; an element that would produce
 *   more than the preamble's length; a stream that ends before the output is full (so trailing elements after a full
 *   output are corrupt too).
 *   Page outcomes:
 *     - src_len == 0 && dst_len == 0: success with 0 bytes (the empty v2 value region of a page with no values);
 *     - preamble != dst_len: "parquet: metadata said %d bytes uncompressed data page, got %d bytes"
 *       (page_reader.go:1094-1095); nothing of the page is written and written = 0;
 *     - a corrupt stream: "parquet: could not decompress page: snappy: corrupt input"; written = the bytes the elements
 *       before the failing one produce, and those bytes are correct;
 *     - every other page of the batch is decoded in full.  The call returns AG_ERR_INVALID naming the lowest failing
 *       page: "snappy_decompress: page %lld: <message> (%lld bytes written)".
 *   No byte outside [dst, dst + dst_len) of any page is ever written, on error paths too.
 *   Differences from the reference (DESIGN §2):
 *     - the reference calls github.com/klauspost/compress/snappy, whose source is not in the reference tree; the inner
 *       message follows golang/snappy's ErrCorrupt and is not pinned against the reference;
 *     - S2 extensions (repeat-offset copies) are corrupt here: a SNAPPY page is plain Snappy;
 *     - a size mismatch is reported from the preamble without decoding the body (the reference decodes first, so it
 *       would report a corrupt body before the mismatch);
 *     - dictionary pages get the data-page wording of the size message.
 * ================================================================================= */
typedef struct ag_pq_compressed {
  int64_t src;
  int64_t src_len;
  int64_t dst;
  int64_t dst_len;
} ag_pq_compressed;
ag_status ag_parquet_snappy_decompress(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst,
                                       int64_t* written);
ag_status ag_parquet_snappy_decompress_dev(const uint8_t* d_src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* d_dst,
                                           int64_t* d_written, ag_stream_t s);

/* ================================================================================= *
 * ZSTD page decompression — the same batch contract as SNAPPY above (`ag_pq_compressed` host table, pages in any
 *   order, `written` in bytes per page, one stream synchronisation in the device flavour, the host flavour stages
 *   `src` and `dst` and copies back only written bytes, the same argument checks before any launch).
 *   serializedPageReader.decompress (parquet/file/page_reader.go:597-621) -> zstdCodec.DecodeWithError
 *   (parquet/compress/zstd.go:115-118) with the decoder of getdecoder (:100-105): zstd.NewReader(nil), default options.
 *   Format (RFC 8878), what that decoder's DecodeAll accepts for a page body:
 *     - one or more frames back to back; skippable frames (magic 0x184D2A50..0x184D2A5F, 4-byte size) are skipped;
 *     - the frame header in full (descriptor, window descriptor, dictionary ID, content size of 0 / 1 / 2 (+256) / 4 /
 *       8 bytes); the reserved bit set is corrupt; a non-zero dictionary ID is refused (no dictionary is supplied);
 *     - Raw, RLE and Compressed zstd blocks; the reserved type is corrupt; a zstd block's stored size and output are at
 *       most min(window, 128 KiB);
 *     - Raw, RLE, Huffman (1 stream, or 4 with the jump table) and Treeless literals (the frame's previous Huffman
 *       table); Huffman descriptions with FSE-compressed or direct 4-bit weights, code lengths up to 11 bits;
 *     - every sequence-count form; Predefined, RLE, FSE_Compressed and Repeat modes, accuracy logs up to 9 / 8 / 9
 *       (LL / OF / ML); the repeat-offset rules, including the shift for a literal length of 0 and `rep0 - 1`;
 *     - the content checksum: the low 32 bits of XXH64 (seed 0) over the frame's output.
 *   Exactness checks: a Huffman stream decodes exactly its share of the literals; every backward bitstream has its
 *   padding marker and is consumed exactly; sequences never consume more literals than the zstd block has; an offset
 *   of 0, beyond the bytes the frame has produced or beyond its window is corrupt; a frame with a content size produces
 *   exactly that many bytes.  A page's sequences may not exceed dst_len / 3 (every match is at least 3 bytes).
 *   Page outcomes:
 *     - src_len == 0 && dst_len == 0: success with 0 bytes;
 *     - every frame has a content size and their sum != dst_len: "parquet: metadata said %d bytes uncompressed data
 *       page, got %d bytes" with that sum; nothing of the page is written;
 *     - the page decodes, but its frames (some without a content size) produce a total != dst_len: the same message
 *       with the real total; nothing of the page is written;
 *     - a corrupt page: "parquet: could not decompress page: zstd: <check>"; written = the bytes of the whole zstd
 *       blocks (and earlier frames) before the first failing zstd block, and those bytes are correct.  <check> is the
 *       first that fails, checked per page in this order: the frame / zstd-block header walk, then per zstd block its
 *       section headers, Huffman literals, sequences bitstream, then execution:
 *         truncated     the input ends inside a frame header, zstd block or checksum
 *         bad magic     neither a zstd nor a skippable frame
 *         frame header  the reserved bit of the frame header descriptor is set
 *         dictionary    a non-zero dictionary ID
 *         block type    the reserved zstd-block type
 *         block size    a zstd block's stored size or output above min(window, 128 KiB)
 *         literals      a literals section header that does not fit its zstd block
 *         huffman       a bad Huffman description or stream, or Treeless literals with no previous table
 *         fse           a bad FSE table description
 *         sequences     a bad sequences header or bitstream, Repeat with no previous table, a page with more than
 *                       dst_len / 3 sequences, sequences that consume more literals than the zstd block has
 *         offset        an offset of 0, beyond the frame's output so far or beyond its window
 *         content size  a frame that does not produce its content size
 *         page size     the output passes dst_len before the failing zstd block (the output stops there instead)
 *     - a checksum mismatch: "parquet: could not decompress page: zstd: checksum mismatch"; the frame's bytes are out
 *       and written counts them (with every other zstd block before the first failing one);
 *     - every other page of the batch is decoded in full.  The call returns AG_ERR_INVALID naming the lowest failing
 *       page: "zstd_decompress: page %lld: <message> (%lld bytes written)".
 *   No byte outside [dst, dst + dst_len) of any page is ever written, on error paths too.
 *   Differences from the reference (DESIGN §2):
 *     - klauspost/compress's source is not in the reference tree, so the inner messages are not pinned against it;
 *     - dictionaries are refused;
 *     - sizes are reported as above, from the frame headers or before anything is executed, not after a full decode;
 *     - dictionary pages get the data-page wording of the size message.
 * ================================================================================= */
ag_status ag_parquet_zstd_decompress(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst,
                                     int64_t* written);
ag_status ag_parquet_zstd_decompress_dev(const uint8_t* d_src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* d_dst,
                                         int64_t* d_written, ag_stream_t s);

/* ================================================================================= *
 * GZIP page decompression — the same batch contract as SNAPPY above (`ag_pq_compressed` host table, pages in any
 *   order, `written` in bytes per page, one stream synchronisation in the device flavour, the host flavour stages
 *   `src` and `dst` and copies back only written bytes, the same argument checks before any launch).
 *   serializedPageReader.decompress (parquet/file/page_reader.go:597-621) -> compress.Decode
 *   (parquet/compress/compress.go:107) -> gzipCodec.DecodeWithError (parquet/compress/gzip.go:51-79):
 *   gzip.NewReader, io.ReadFull into dst_len bytes, then one more byte must read as EOF.
 *   Format, what that reader (klauspost/compress/gzip, a fork of Go's compress/gzip and compress/flate) accepts:
 *     - one or more gzip members (RFC 1952) back to back.  After a member: no bytes left ends the stream, 1-9 bytes
 *       are a truncation, anything else that is not a gzip header (zero padding too) is a bad header;
 *     - the header: 1f 8b, CM = 8, FLG, MTIME, XFL, OS; FEXTRA (2-byte length, then that many bytes); FNAME and FCOMMENT
 *       NUL-terminated with at most 511 bytes before the NUL; FHCRC = the low 16 bits of the CRC32 of the header bytes
 *       before it.  Reserved FLG bits are ignored.  A zlib-wrapped (RFC 1950) or raw DEFLATE body is a bad header;
 *     - DEFLATE (RFC 1951) stored, fixed and dynamic blocks.  Stored: LEN == ~NLEN.  Dynamic: HLIT <= 286, HDIST <= 30;
 *       a repeat code 16 with no previous length, or any repeat past HLIT + HDIST, is corrupt.  Every code is complete
 *       except a code of one symbol of length 1; a distance code may have no symbols at all (a distance symbol is then
 *       corrupt); a literal/length code must have end-of-block (256).  Literal/length symbols 286 and 287 and distance
 *       symbols 30 and 31 are corrupt.  A distance reaches back at most to the member's first output byte (every
 *       member starts a fresh window);
 *     - the trailer: CRC32 (IEEE, reflected) and ISIZE (output mod 2^32) of the member.
 *   Page outcomes, as events in stream order (the first one wins).  Every message starts with
 *   "parquet: could not decompress page: ":
 *     - src_len == 0 && dst_len == 0: success with 0 bytes;
 *     - the input ends inside a member (a stored block cut off counts as a whole), or 1-9 bytes follow a member:
 *       "unexpected EOF";
 *     - every member decodes cleanly but the total is short of dst_len: "unexpected EOF", or "EOF" when the total is 0;
 *     - output byte dst_len + 1 is produced: "codec: gzip: decoded data exceeds destination size <dst_len>";
 *     - bad magic or CM, an FHCRC mismatch, a name or comment too long, or non-gzip bytes after a member:
 *       "gzip: invalid header";
 *     - a member's CRC32 or ISIZE does not match at its trailer: "gzip: invalid checksum";
 *     - corrupt DEFLATE: "gzip: <check>", one of
 *         block type      BTYPE 3
 *         stored length   LEN does not match NLEN
 *         code lengths    HLIT or HDIST out of range, a bad repeat, a bit sequence the code-length code does not have
 *         huffman         an over-subscribed or incomplete code, or no end-of-block code
 *         symbol          an invalid literal/length or distance symbol
 *         distance        a distance beyond the member's output so far
 *     - written counts the bytes of every element (literal, copy, stored block) decoded before the first decode event,
 *       at most dst_len, and those bytes are correct.  A checksum mismatch does not stop decoding: the member's bytes
 *       are out and counted, with those of the members after it up to the first decode event;
 *     - every other page of the batch is decoded in full.  The call returns AG_ERR_INVALID naming the lowest failing
 *       page: "gzip_decompress: page %lld: <message> (%lld bytes written)".
 *   No byte outside [dst, dst + dst_len) of any page is ever written, on error paths too.
 *   Differences from the reference (DESIGN §2):
 *     - klauspost/compress's source is not in the reference tree, so the rules above restate Go's readers; Go reports
 *       corrupt DEFLATE as "flate: corrupt input before offset N", with an N that depends on its bit reader, so the
 *       <check> names are this library's own;
 *     - src_len == 0 && dst_len == 0 is a success (the reference reports "EOF").
 * ================================================================================= */
ag_status ag_parquet_gzip_decompress(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst,
                                     int64_t* written);
ag_status ag_parquet_gzip_decompress_dev(const uint8_t* d_src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* d_dst,
                                         int64_t* d_written, ag_stream_t s);

/* ================================================================================= *
 * LZ4_RAW page decompression — the same batch contract as SNAPPY above (`ag_pq_compressed` host table, pages in any
 *   order, `written` in bytes per page, one stream synchronisation in the device flavour, the host flavour stages
 *   `src` and `dst` and copies back only written bytes, the same argument checks before any launch).
 *   serializedPageReader.decompress (parquet/file/page_reader.go:597-621) -> compress.Decode
 *   (parquet/compress/compress.go:107) -> lz4RawCodec.DecodeWithError (parquet/compress/lz4_raw.go:63-70):
 *   lz4.UncompressBlock (pierrec/lz4 v4) into dst_len bytes.
 *   Format: an LZ4 block, as pierrec/lz4 v4's block decoder accepts it.  A block is a sequence of sequences:
 *     - a token byte; the literal length token >> 4, and if that is 15 it continues with extension bytes: each is
 *       added, and the run ends at the first byte that is not 255;
 *     - that many literal bytes;
 *     - if the input ends here, the stream ends cleanly when token & 15 == 0 and is corrupt otherwise;
 *     - a 2-byte little-endian offset;
 *     - the match length (token & 15) + 4, continued with extension bytes as the literal length is when the nibble is 15;
 *     - the match copies from `offset` bytes back and may overlap its own output.  After a match the end of the input
 *       is a clean end.
 *   Page outcomes:
 *     - src_len == 0 && dst_len == 0: success with 0 bytes;
 *     - a corrupt stream: "parquet: could not decompress page: lz4: invalid source or destination buffer too short"
 *       (pierrec's ErrInvalidSourceShortBuffer).  Corrupt: an empty source with dst_len > 0; a length extension, the
 *       literals or the offset cut off by the end of the input; a non-zero match nibble at the end of the input; offset
 *       0; an offset beyond the bytes produced so far; an element that would write past dst_len.  written counts the
 *       bytes of the elements before the failing one (a sequence's literal run and its match are separate elements),
 *       and those bytes are correct;
 *     - a stream that decodes cleanly to n != dst_len bytes: "parquet: metadata said %d bytes uncompressed data page,
 *       got %d bytes" with n (page_reader.go:1094-1095); nothing of the page is written and written = 0;
 *     - every other page of the batch is decoded in full.  The call returns AG_ERR_INVALID naming the lowest failing
 *       page: "lz4_raw_decompress: page %lld: <message> (%lld bytes written)".
 *   No byte outside [dst, dst + dst_len) of any page is ever written, on error paths too.
 *   Differences (DESIGN §2):
 *     - pierrec/lz4's source is not in the reference tree, so the rules above restate its block decoder;
 *     - liblz4 (pyarrow's decoder) enforces the end-of-block rules (the last 5 bytes are literals, the last match
 *       starts at least 12 bytes before the end); pierrec does not, and neither does this library: a stream that ends
 *       in a match decodes here;
 *     - liblz4 ignores a non-zero match nibble in the final literal-only sequence, and copies a match with offset 0 from
 *       the output position itself; here both are corrupt;
 *     - src_len == 0 && dst_len == 0 is a success (the reference and liblz4 refuse an empty block).
 * ================================================================================= */
ag_status ag_parquet_lz4_raw_decompress(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst,
                                        int64_t* written);
ag_status ag_parquet_lz4_raw_decompress_dev(const uint8_t* d_src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* d_dst,
                                            int64_t* d_written, ag_stream_t s);

/* ================================================================================= *
 * SNAPPY page compression — the decompressors' batch shape read the other way round, so that pages encoded on the
 *   device are compressed there too.  serializedPageWriter.Compress (parquet/file/page_writer.go:229-233) sizes a
 *   buffer with CompressBound and calls EncodeLevel; for SNAPPY that is snappyCodec (parquet/compress/snappy.go:27-33,
 *   51-53), github.com/klauspost/compress's snappy.Encode with the bound 32 + n + n/6.
 *     src      byte offset of the page's uncompressed bytes in `src`
 *     src_len  their count, at most 2^32-1
 *     dst      byte offset of the page's stream in `dst`
 *     dst_len  the capacity there, at least ag_parquet_snappy_max_size(src_len)
 *   `pages` is a HOST array in both flavours; pages may come in any order and may share or skip input.  written (may
 *   be NULL) receives each stream's length, preamble included.  No byte outside [dst, dst + written) of any page is
 *   written.  `src` and `dst` must not overlap (not checked).
 *   Argument checks, AG_ERR_INVALID naming the page before any launch: a negative field, src_len above 2^32-1, a
 *   capacity below the bound, and dst ranges [dst, dst + dst_len) that overlap.  Once they pass no data-dependent error
 *   exists, so the device flavour does not synchronise `s`: d_written is a device array written in stream order, and
 *   the call's tables and scratch (about the input's size) are stream-ordered allocations.  The host flavour stages `src` through device
 *   memory and copies back only the written bytes.  Without a usable GPU both return AG_ERR_CUDA.
 *   Format: raw Snappy, one parse stated exactly (tests/snappy_encode_model.py):
 *     - the preamble uvarint(src_len); a page shorter than 4 bytes is the preamble and one literal (an empty page is
 *       the single byte 0x00);
 *     - 64 KiB fragments (the last may be shorter), each encoded on its own: an empty hash table, copies only within
 *       the fragment (offsets 1..65535), its trailing bytes flushed as a literal;
 *     - the candidate positions p of a fragment [s, e) are those with p + 4 <= e, walked in windows of 32 from a
 *       cursor.  For each p in order: h(p) = ((load32le(p) * 0x1E35A7BD) mod 2^32) >> 20; its candidate q is the
 *       latest position inserted with that hash (earlier positions of the window count); p is then inserted.  The
 *       first p whose q holds the same 4 bytes starts a match, and the rest of the window is neither looked up nor
 *       inserted.  The match extends while p + L < e and src[q + L] == src[p + L]; the bytes since the last match end
 *       go out as a literal, then the copy, and the cursor moves to p + L.  A window without a match moves the cursor
 *       past its last position;
 *     - golang/snappy's element forms: a literal header holds length-1 in the tag below 60, else tag 60..63 and the
 *       minimal 1..4 length bytes.  A copy of L bytes: 64-byte copies (2-byte offset) while L >= 68, a 60-byte copy
 *       if L > 64 remains, then the 1-byte-offset form when L < 12 and offset < 2048, else the 2-byte-offset form.
 *   Differences from the reference (DESIGN §2): klauspost/compress's source is not in the reference tree, so its bytes
 *   are not pinned.  The streams here are valid raw Snappy within the same bound, and their size is close to a
 *   production encoder's.
 *   ag_parquet_snappy_max_size: 32 + n + n/6; n < 0 or n > 2^32-1 is AG_ERR_INVALID.  It needs no GPU.
 * ================================================================================= */
ag_status ag_parquet_snappy_max_size(int64_t n, int64_t* size);
ag_status ag_parquet_snappy_compress(const uint8_t* src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* dst,
                                     int64_t* written);
ag_status ag_parquet_snappy_compress_dev(const uint8_t* d_src, const ag_pq_compressed* pages, int64_t n_pages, uint8_t* d_dst,
                                         int64_t* d_written, ag_stream_t s);

/* ================================================================================= *
 * Parity helpers for inputs too large to bring back to the host (SURVEY §8d):
 * order-sensitive 64-bit checksum  sum_i mix64(i) * word_i  (mod 2^64)  over a buffer
 * viewed as little-endian uint64 words (n_words = nbytes/8), and a counter-based
 * generator so 1B-row datasets are produced on the device and reproduced on the CPU.
 * ================================================================================= */
ag_status ag_checksum64_dev(const void* d_buf, size_t n_words, uint64_t* d_res, ag_stream_t s);
/* kind: 0 = splitmix64(seed + i) as u64; 1 = uniform int64 in [lo, hi] (hi-lo+1 <= 2^32, via
 * multiply-shift on the high 32 bits); 2 = uniform int32 in [lo, hi]; 3 = double(k) with k
 * uniform integer in [lo, hi]; 4 = bitmap with P(bit)=lo/hi (n = bits); 5 / 6 = sorted / reverse-sorted int32
 * ramp over [lo, hi] (the sorted index datasets of SURVEY §8d). */
ag_status ag_generate_dev(int kind, uint64_t seed, int64_t lo, int64_t hi, void* d_out, size_t n, ag_stream_t s);

#ifdef __cplusplus
}
#endif
#endif /* ARROWGPU_H */
