/* arrowgpu_cdata.h — device-resident hand-off through the Arrow C Device Data Interface.
 *
 * SURVEY.md §8(f) rank 2: batches stay in HBM between operators and cross library boundaries
 * without a copy.  The struct layouts below are the published Arrow C Data / C Device Data ABI
 * (the reference carries the same declarations in arrow/cdata/abi.h:50-140 and consumes them in
 * arrow/cdata/cdata.go:72, cdata_exports.go:533; its own producers only emit ARROW_DEVICE_CPU,
 * arrow/cdata/exports.go:316,357).  They are guarded by the standard macros so this header can
 * be included next to any other copy of the ABI.
 *
 * What a consumer does with an exported array:   wait on *sync_event (a cudaEvent_t*) on its own
 * stream, read buffers[0] (validity, may be NULL) and buffers[1] (values) as device pointers,
 * call array.release when done.  What a producer hands to ag_import_device_array: the same.
 */
#ifndef ARROWGPU_CDATA_H
#define ARROWGPU_CDATA_H

#include <stdint.h>

#include "arrowgpu.h"

#ifdef __cplusplus
extern "C" {
#endif

#ifndef ARROW_C_DATA_INTERFACE
#define ARROW_C_DATA_INTERFACE

#define ARROW_FLAG_DICTIONARY_ORDERED 1
#define ARROW_FLAG_NULLABLE 2
#define ARROW_FLAG_MAP_KEYS_SORTED 4

struct ArrowSchema {
  const char* format;   /* "c C s S i I l L f g b" for the types of this library */
  const char* name;
  const char* metadata;
  int64_t flags;
  int64_t n_children;
  struct ArrowSchema** children;
  struct ArrowSchema* dictionary;
  void (*release)(struct ArrowSchema*);
  void* private_data;
};

struct ArrowArray {
  int64_t length;
  int64_t null_count;   /* -1 = not computed */
  int64_t offset;       /* in elements (bits for bitmaps) */
  int64_t n_buffers;    /* 2 for primitive / boolean arrays: validity, values */
  int64_t n_children;
  const void** buffers;
  struct ArrowArray** children;
  struct ArrowArray* dictionary;
  void (*release)(struct ArrowArray*);
  void* private_data;
};

#endif /* ARROW_C_DATA_INTERFACE */

#ifndef ARROW_C_DEVICE_DATA_INTERFACE
#define ARROW_C_DEVICE_DATA_INTERFACE

typedef int32_t ArrowDeviceType;

/* device types this library distinguishes (the ABI assigns more ids; any other value is refused as
 * "not a CUDA device" by ag_import_device_array) */
#define ARROW_DEVICE_CPU 1
#define ARROW_DEVICE_CUDA 2
#define ARROW_DEVICE_CUDA_HOST 3
#define ARROW_DEVICE_CUDA_MANAGED 13

struct ArrowDeviceArray {
  struct ArrowArray array;   /* buffers are addresses on (device_type, device_id) */
  int64_t device_id;
  ArrowDeviceType device_type;
  void* sync_event;          /* CUDA: cudaEvent_t* to wait on before touching the buffers, or NULL */
  int64_t reserved[3];
};

#endif /* ARROW_C_DEVICE_DATA_INTERFACE */

#ifndef ARROW_C_DEVICE_STREAM_INTERFACE
#define ARROW_C_DEVICE_STREAM_INTERFACE

/* A stream of ArrowDeviceArrays on ONE device (arrow/cdata/abi.h:170-200 of the reference; the published Arrow C
 * Device Stream ABI).  Callbacks return 0 or an errno-compatible code; get_next marks the end of the stream with a
 * released array (out->array.release == NULL).  Every array must be released independently of the stream. */
struct ArrowDeviceArrayStream {
  ArrowDeviceType device_type;
  int (*get_schema)(struct ArrowDeviceArrayStream* self, struct ArrowSchema* out);
  int (*get_next)(struct ArrowDeviceArrayStream* self, struct ArrowDeviceArray* out);
  const char* (*get_last_error)(struct ArrowDeviceArrayStream* self);
  void (*release)(struct ArrowDeviceArrayStream* self);
  void* private_data;
};

#endif /* ARROW_C_DEVICE_STREAM_INTERFACE */

/* What an array looks like to the *_dev entry points of arrowgpu.h. */
typedef struct ag_array_view {
  int type;             /* AG_TYPE_* (0 when no schema / type was given) */
  int64_t length;
  int64_t null_count;
  int64_t offset;
  const uint8_t* validity;  /* may be NULL */
  const void* values;
  int32_t device_type;
  int64_t device_id;
} ag_array_view;

/* Arrow format string <-> arrow.Type id for the types on this path.  Pure host code. */
ag_status ag_schema_format_to_type(const char* format, int* type);
const char* ag_type_to_schema_format(int type); /* NULL for unsupported ids */

/* Fills `out` from a device array without touching the device (no wait, no ownership change):
 * checks the layout this library understands (2 buffers, no children, no dictionary).  `schema`
 * may be NULL (then out->type = 0).  Works on ARROW_DEVICE_CPU arrays too — it only reads the
 * struct — which is how the tests check the layout against another producer (pyarrow). */
ag_status ag_device_array_describe(const struct ArrowDeviceArray* in, const struct ArrowSchema* schema, ag_array_view* out);

/* A Dictionary<int32, T> array (one level, arrow/cdata/cdata.go importer's dictionary case): schema format "i" with
 * schema->dictionary set, array->dictionary set, the dictionary a primitive array on the same device.  Fills the view of
 * the indices and of the dictionary values; ag_device_array_describe itself keeps refusing dictionary arrays. */
ag_status ag_dictionary_device_array_describe(const struct ArrowDeviceArray* in, const struct ArrowSchema* schema,
                                              ag_array_view* indices, ag_array_view* dictionary);

/* Export device buffers as an ArrowDeviceArray{ARROW_DEVICE_CUDA, current device}.
 *   d_validity may be NULL.  An event is recorded on `produced_on` and published as sync_event so
 *   that the consumer orders itself after the kernels that produced the buffers.
 *   `release_buffers(opaque)` (may be NULL) runs once, when the consumer calls out->array.release:
 *   that is where the owner drops its reference (ag_dev_free, a Go finalizer, a shared_ptr).
 *   If `out_schema` is non-NULL it is filled with a matching schema (release frees it). */
ag_status ag_export_device_array(int type, int64_t length, int64_t null_count, int64_t offset,
                                 const void* d_validity, const void* d_values,
                                 void (*release_buffers)(void* opaque), void* opaque, ag_stream_t produced_on,
                                 struct ArrowDeviceArray* out, struct ArrowSchema* out_schema);

/* Import: validates (ARROW_DEVICE_CUDA on the current device, ARROW_DEVICE_CUDA_HOST or
 * ARROW_DEVICE_CUDA_MANAGED — pinned / managed memory is addressable by the kernels as is), makes
 * `consume_on` wait for in->sync_event, and fills `out` with pointers that can be passed straight to
 * the *_dev entry points.  Ownership stays with `in`: call in->array.release(&in->array) after the
 * last kernel that reads the buffers has completed.  ARROW_DEVICE_CPU is rejected with
 * AG_ERR_INVALID (upload it: ag_upload / ArrayData::FromHost). */
ag_status ag_import_device_array(struct ArrowDeviceArray* in, const struct ArrowSchema* schema, ag_stream_t consume_on, ag_array_view* out);

/* One level of dictionary (Dictionary<int32, T>, the layout of arrow/cdata's dictionary export: the parent is the int32
 * indices with format "i", schema->dictionary / array->dictionary the value type's primitive array).
 *   Export: the parent's release runs `release_buffers(opaque)` (which must cover the index AND the dictionary
 *   buffers) and then releases the dictionary child; the schema's release frees the child schema.  Both share the
 *   device and the sync_event of the parent.  ag_export_device_array keeps refusing AG_TYPE_DICTIONARY.
 *   Import: ag_dictionary_device_array_describe plus the device checks and the wait of ag_import_device_array.
 *   Ownership stays with `in`: releasing the parent releases the dictionary. */
ag_status ag_export_dictionary_device_array(int value_type, int64_t length, int64_t null_count, int64_t offset,
                                            const void* d_index_validity, const int32_t* d_indices,
                                            int64_t dict_length, int64_t dict_null_count, int64_t dict_offset,
                                            const void* d_dict_validity, const void* d_dict_values,
                                            void (*release_buffers)(void* opaque), void* opaque, ag_stream_t produced_on,
                                            struct ArrowDeviceArray* out, struct ArrowSchema* out_schema);
ag_status ag_import_dictionary_device_array(struct ArrowDeviceArray* in, const struct ArrowSchema* schema, ag_stream_t consume_on,
                                            ag_array_view* indices, ag_array_view* dictionary);

/* A run-end encoded array (the layout pyarrow and arrow/cdata export for arrow.RUN_END_ENCODED): the parent has format
 * "+r", no buffers, null_count 0 and carries the logical offset and length; its two children are "run_ends" (format
 * "s" / "i" / "l", non-nullable) and "values" (a primitive array).  All three live on one device.
 *   Describe: fills the parent's view (type AG_TYPE_RUN_END_ENCODED, length, offset; no buffers) and the views of the
 *   two children; ag_device_array_describe itself keeps refusing run-end encoded arrays.
 *   Export: the parent's release runs `release_buffers(opaque)` (which must cover the run-end AND the values buffers)
 *   and then releases each child a consumer has not moved out; the schema's release frees the child schemas.  The
 *   children share the device of the parent.  ag_export_device_array keeps refusing AG_TYPE_RUN_END_ENCODED.
 *   Import: describe plus the device checks and the wait of ag_import_device_array.  Ownership stays with `in`. */
ag_status ag_run_end_encoded_device_array_describe(const struct ArrowDeviceArray* in, const struct ArrowSchema* schema,
                                                   ag_array_view* parent, ag_array_view* run_ends, ag_array_view* values);
ag_status ag_export_run_end_encoded_device_array(int value_type, int run_end_type, int64_t length, int64_t offset,
                                                 int64_t n_runs, const void* d_run_ends,
                                                 int64_t values_length, int64_t values_null_count, int64_t values_offset,
                                                 const void* d_values_validity, const void* d_values,
                                                 void (*release_buffers)(void* opaque), void* opaque, ag_stream_t produced_on,
                                                 struct ArrowDeviceArray* out, struct ArrowSchema* out_schema);
ag_status ag_import_run_end_encoded_device_array(struct ArrowDeviceArray* in, const struct ArrowSchema* schema, ag_stream_t consume_on,
                                                 ag_array_view* parent, ag_array_view* run_ends, ag_array_view* values);

#ifdef __cplusplus
}
#endif
#endif /* ARROWGPU_CDATA_H */
