// Arrow C Device Data Interface hand-off (include/arrowgpu_cdata.h): export device-resident
// buffers as ArrowDeviceArray{ARROW_DEVICE_CUDA} with a cudaEvent_t* sync_event, import the same
// from any other producer.  No kernels here: the point is that record batches cross the
// boundary by pointer and stay in HBM (SURVEY §8f rank 2; the reference's own device-array
// producers are CPU-only, arrow/cdata/exports.go:316,357).
#include "common.cuh"

#include "../../include/arrowgpu_cdata.h"

#include <stdlib.h>
#include <string.h>

namespace ag {
namespace {

struct ExportState {
  const void* buffers[2];
  cudaEvent_t event;
  bool have_event;
  void (*release_buffers)(void*);
  void* opaque;
  struct ArrowArray* dictionary;   // a dictionary array's child (heap), released and freed with the parent
  struct ArrowArray* children[2];  // a run-end encoded array's run_ends and values (heap), released and freed with it
};

void release_exported_array(struct ArrowArray* a) {
  if (!a || !a->release) return;
  ExportState* st = static_cast<ExportState*>(a->private_data);
  if (st) {
    if (st->have_event) cudaEventDestroy(st->event);
    if (st->release_buffers) st->release_buffers(st->opaque);
    if (st->dictionary) {
      if (st->dictionary->release) st->dictionary->release(st->dictionary);   // unless the consumer moved it out
      free(st->dictionary);
    }
    for (struct ArrowArray* c : st->children) {
      if (!c) continue;
      if (c->release) c->release(c);   // unless the consumer moved it out
      free(c);
    }
    free(st);
  }
  a->release = nullptr;  // the ABI's "released" marker
  a->private_data = nullptr;
}

void release_exported_schema(struct ArrowSchema* s) {
  if (!s || !s->release) return;
  s->release = nullptr;  // format / name point at static strings: nothing to free
}

// a dictionary schema owns its value schema (heap)
void release_dictionary_schema(struct ArrowSchema* s) {
  if (!s || !s->release) return;
  if (s->dictionary) {
    if (s->dictionary->release) s->dictionary->release(s->dictionary);
    free(s->dictionary);
    s->dictionary = nullptr;
  }
  s->release = nullptr;
}

// a run-end encoded schema owns its two child schemas and their pointer array (heap)
void release_run_end_schema(struct ArrowSchema* s) {
  if (!s || !s->release) return;
  for (int64_t k = 0; k < s->n_children; ++k) {
    struct ArrowSchema* c = s->children[k];
    if (c->release) c->release(c);
    free(c);
  }
  free(s->children);
  s->children = nullptr;
  s->release = nullptr;
}

int run_end_type_of(const char* format) {
  if (!format) return 0;
  if (strcmp(format, "s") == 0) return AG_TYPE_INT16;
  if (strcmp(format, "i") == 0) return AG_TYPE_INT32;
  if (strcmp(format, "l") == 0) return AG_TYPE_INT64;
  return 0;
}

}  // namespace
}  // namespace ag

using namespace ag;

extern "C" const char* ag_type_to_schema_format(int type) {
  switch (type) {
    case AG_TYPE_BOOL: return "b";
    case AG_TYPE_INT8: return "c";
    case AG_TYPE_UINT8: return "C";
    case AG_TYPE_INT16: return "s";
    case AG_TYPE_UINT16: return "S";
    case AG_TYPE_INT32: return "i";
    case AG_TYPE_UINT32: return "I";
    case AG_TYPE_INT64: return "l";
    case AG_TYPE_UINT64: return "L";
    case AG_TYPE_FLOAT32: return "f";
    case AG_TYPE_FLOAT64: return "g";
    default: return nullptr;
  }
}

extern "C" ag_status ag_schema_format_to_type(const char* format, int* type) {
  if (!format || !type) AG_FAIL(AG_ERR_INVALID, "cdata: NULL format / type");
  static const int ids[] = {AG_TYPE_BOOL, AG_TYPE_INT8, AG_TYPE_UINT8, AG_TYPE_INT16, AG_TYPE_UINT16, AG_TYPE_INT32,
                            AG_TYPE_UINT32, AG_TYPE_INT64, AG_TYPE_UINT64, AG_TYPE_FLOAT32, AG_TYPE_FLOAT64};
  for (int id : ids) {
    if (strcmp(format, ag_type_to_schema_format(id)) == 0) { *type = id; return AG_OK; }
  }
  AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "cdata: format '%s' is not a boolean / numeric primitive type", format);
}

extern "C" ag_status ag_device_array_describe(const struct ArrowDeviceArray* in, const struct ArrowSchema* schema, ag_array_view* out) {
  if (!in || !out) AG_FAIL(AG_ERR_INVALID, "cdata: NULL array / view");
  const struct ArrowArray& a = in->array;
  if (!a.release) AG_FAIL(AG_ERR_INVALID, "cdata: array was already released");
  if (a.n_buffers != 2) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "cdata: expected 2 buffers (validity, values), got %lld", (long long)a.n_buffers);
  if (a.n_children != 0 || a.dictionary) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "cdata: nested / dictionary arrays are outside this path");
  if (a.length < 0 || a.offset < 0) AG_FAIL(AG_ERR_INVALID, "cdata: negative length or offset");
  if (!a.buffers) AG_FAIL(AG_ERR_INVALID, "cdata: NULL buffers");
  out->type = 0;
  if (schema) {
    if (!schema->release) AG_FAIL(AG_ERR_INVALID, "cdata: schema was already released");
    AG_TRY(ag_schema_format_to_type(schema->format, &out->type));
  }
  out->length = a.length;
  out->null_count = a.null_count;
  out->offset = a.offset;
  out->validity = static_cast<const uint8_t*>(a.buffers[0]);
  out->values = a.buffers[1];
  out->device_type = in->device_type;
  out->device_id = in->device_id;
  if (a.length > 0 && !out->values) AG_FAIL(AG_ERR_INVALID, "cdata: NULL values buffer");
  return AG_OK;
}

// One level of dictionary: the parent's buffers are the indices (format "i"), the dictionary child a primitive array on
// the parent's device.  Both are described by ag_device_array_describe on shallow copies without the dictionary link.
extern "C" ag_status ag_dictionary_device_array_describe(const struct ArrowDeviceArray* in, const struct ArrowSchema* schema,
                                                         ag_array_view* indices, ag_array_view* dictionary) {
  if (!in || !schema || !indices || !dictionary) AG_FAIL(AG_ERR_INVALID, "cdata: NULL array / schema / view");
  if (!in->array.dictionary || !schema->dictionary) AG_FAIL(AG_ERR_INVALID, "cdata: not a dictionary array");
  if (!schema->format || strcmp(schema->format, "i") != 0)
    AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "cdata: dictionary indices of format '%s' (only int32 'i')", schema->format ? schema->format : "");
  struct ArrowDeviceArray parent = *in;
  parent.array.dictionary = nullptr;
  struct ArrowSchema parent_schema = *schema;
  parent_schema.dictionary = nullptr;
  AG_TRY(ag_device_array_describe(&parent, &parent_schema, indices));
  struct ArrowDeviceArray child = *in;
  child.array = *in->array.dictionary;
  AG_TRY(ag_device_array_describe(&child, schema->dictionary, dictionary));
  return AG_OK;
}

extern "C" ag_status ag_export_device_array(int type, int64_t length, int64_t null_count, int64_t offset,
                                            const void* d_validity, const void* d_values,
                                            void (*release_buffers)(void*), void* opaque, ag_stream_t produced_on,
                                            struct ArrowDeviceArray* out, struct ArrowSchema* out_schema) {
  AG_TRY(ensure_init());
  if (!out) AG_FAIL(AG_ERR_INVALID, "cdata: NULL output");
  const char* fmt = ag_type_to_schema_format(type);
  if (!fmt) AG_FAIL(AG_ERR_TYPE, "cdata: unsupported type id %d", type);
  if (length < 0 || offset < 0) AG_FAIL(AG_ERR_INVALID, "cdata: negative length or offset");
  if (length > 0 && !d_values) AG_FAIL(AG_ERR_INVALID, "cdata: NULL values buffer");
  ExportState* st = static_cast<ExportState*>(calloc(1, sizeof(ExportState)));
  if (!st) AG_FAIL(AG_ERR_OOM, "cdata: out of host memory");
  st->buffers[0] = d_validity;
  st->buffers[1] = d_values;
  st->release_buffers = release_buffers;
  st->opaque = opaque;
  cudaError_t e = cudaEventCreateWithFlags(&st->event, cudaEventDisableTiming);
  if (e == cudaSuccess) {
    st->have_event = true;
    e = cudaEventRecord(st->event, resolve_stream(produced_on));
  }
  if (e != cudaSuccess) {
    if (st->have_event) cudaEventDestroy(st->event);
    free(st);
    AG_FAIL(AG_ERR_CUDA, "cdata: %s", cudaGetErrorString(e));
  }
  int dev = 0;
  cudaGetDevice(&dev);
  memset(out, 0, sizeof(*out));
  out->array.length = length;
  out->array.null_count = null_count;
  out->array.offset = offset;
  out->array.n_buffers = 2;
  out->array.n_children = 0;
  out->array.buffers = st->buffers;
  out->array.children = nullptr;
  out->array.dictionary = nullptr;
  out->array.release = release_exported_array;
  out->array.private_data = st;
  out->device_id = dev;
  out->device_type = ARROW_DEVICE_CUDA;
  out->sync_event = &st->event;
  if (out_schema) {
    memset(out_schema, 0, sizeof(*out_schema));
    out_schema->format = fmt;
    out_schema->name = "";
    out_schema->metadata = nullptr;
    out_schema->flags = ARROW_FLAG_NULLABLE;
    out_schema->release = release_exported_schema;
  }
  return AG_OK;
}

namespace {
// the device checks and the wait of an import
ag_status import_wait(const struct ArrowDeviceArray* in, ag_stream_t consume_on) {
  switch (in->device_type) {
    case ARROW_DEVICE_CUDA: {
      int dev = 0;
      cudaGetDevice(&dev);
      if (in->device_id != dev)
        AG_FAIL(AG_ERR_INVALID, "cdata: array lives on CUDA device %lld, the calling thread works on device %d (ag_set_device first)", (long long)in->device_id, dev);
      break;
    }
    case ARROW_DEVICE_CUDA_HOST:
    case ARROW_DEVICE_CUDA_MANAGED:
      break;  // pinned / managed memory: addressable from the kernels through unified addressing
    case ARROW_DEVICE_CPU:
      AG_FAIL(AG_ERR_INVALID, "cdata: ARROW_DEVICE_CPU array — pageable host memory is not device-addressable; upload it (ag_upload) or allocate it with ag_host_alloc and export it as ARROW_DEVICE_CUDA_HOST");
    default:
      AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "cdata: device type %d is not a CUDA device", (int)in->device_type);
  }
  if (in->sync_event) {
    cudaEvent_t ev = *static_cast<cudaEvent_t*>(in->sync_event);
    AG_CUDA_TRY(cudaStreamWaitEvent(resolve_stream(consume_on), ev, 0));
  }
  return AG_OK;
}
}  // namespace

extern "C" ag_status ag_import_device_array(struct ArrowDeviceArray* in, const struct ArrowSchema* schema, ag_stream_t consume_on, ag_array_view* out) {
  AG_TRY(ensure_init());
  AG_TRY(ag_device_array_describe(in, schema, out));
  return import_wait(in, consume_on);
}

extern "C" ag_status ag_import_dictionary_device_array(struct ArrowDeviceArray* in, const struct ArrowSchema* schema, ag_stream_t consume_on,
                                                       ag_array_view* indices, ag_array_view* dictionary) {
  AG_TRY(ensure_init());
  AG_TRY(ag_dictionary_device_array_describe(in, schema, indices, dictionary));
  return import_wait(in, consume_on);
}

extern "C" ag_status ag_export_dictionary_device_array(int value_type, int64_t length, int64_t null_count, int64_t offset,
                                                       const void* d_index_validity, const int32_t* d_indices,
                                                       int64_t dict_length, int64_t dict_null_count, int64_t dict_offset,
                                                       const void* d_dict_validity, const void* d_dict_values,
                                                       void (*release_buffers)(void*), void* opaque, ag_stream_t produced_on,
                                                       struct ArrowDeviceArray* out, struct ArrowSchema* out_schema) {
  AG_TRY(ensure_init());
  if (!out) AG_FAIL(AG_ERR_INVALID, "cdata: NULL output");
  const char* value_fmt = ag_type_to_schema_format(value_type);
  if (!value_fmt) AG_FAIL(AG_ERR_TYPE, "cdata: unsupported dictionary value type id %d", value_type);
  if (dict_length < 0 || dict_offset < 0) AG_FAIL(AG_ERR_INVALID, "cdata: negative dictionary length or offset");
  if (dict_length > 0 && !d_dict_values) AG_FAIL(AG_ERR_INVALID, "cdata: NULL dictionary values buffer");
  struct ArrowArray* child = static_cast<struct ArrowArray*>(calloc(1, sizeof(struct ArrowArray)));
  struct ArrowSchema* child_schema = out_schema ? static_cast<struct ArrowSchema*>(calloc(1, sizeof(struct ArrowSchema))) : nullptr;
  if (!child || (out_schema && !child_schema)) { free(child); free(child_schema); AG_FAIL(AG_ERR_OOM, "cdata: out of host memory"); }
  // the child: a primitive export whose buffers the parent's release_buffers covers
  struct ArrowDeviceArray tmp;
  ag_status rc = ag_export_device_array(value_type, dict_length, dict_null_count, dict_offset, d_dict_validity, d_dict_values, nullptr, nullptr,
                                        produced_on, &tmp, child_schema);
  if (rc != AG_OK) { free(child); free(child_schema); return rc; }
  *child = tmp.array;
  // the parent: the int32 indices; its release runs release_buffers and then releases the child
  rc = ag_export_device_array(AG_TYPE_INT32, length, null_count, offset, d_index_validity, d_indices, release_buffers, opaque, produced_on,
                              out, out_schema);
  if (rc != AG_OK) {
    child->release(child);
    free(child);
    if (child_schema) { child_schema->release(child_schema); free(child_schema); }
    return rc;
  }
  static_cast<ExportState*>(out->array.private_data)->dictionary = child;
  out->array.dictionary = child;
  if (out_schema) {
    out_schema->dictionary = child_schema;
    out_schema->release = release_dictionary_schema;
  }
  return AG_OK;
}

// Run-end encoded: a "+r" parent without buffers and two children, run_ends and values, each described by
// ag_device_array_describe on a shallow copy of the parent's device array.
extern "C" ag_status ag_run_end_encoded_device_array_describe(const struct ArrowDeviceArray* in, const struct ArrowSchema* schema,
                                                              ag_array_view* parent, ag_array_view* run_ends, ag_array_view* values) {
  if (!in || !schema || !parent || !run_ends || !values) AG_FAIL(AG_ERR_INVALID, "cdata: NULL array / schema / view");
  const struct ArrowArray& a = in->array;
  if (!a.release || !schema->release) AG_FAIL(AG_ERR_INVALID, "cdata: array or schema was already released");
  if (!schema->format || strcmp(schema->format, "+r") != 0) AG_FAIL(AG_ERR_INVALID, "cdata: not a run-end encoded array (format '%s')", schema->format ? schema->format : "");
  if (a.n_children != 2 || schema->n_children != 2 || !a.children || !schema->children)
    AG_FAIL(AG_ERR_INVALID, "cdata: a run-end encoded array has two children (run_ends, values)");
  if (a.n_buffers != 0 || a.dictionary) AG_FAIL(AG_ERR_INVALID, "cdata: a run-end encoded parent has no buffers and no dictionary");
  if (a.length < 0 || a.offset < 0) AG_FAIL(AG_ERR_INVALID, "cdata: negative length or offset");
  if (a.null_count > 0) AG_FAIL(AG_ERR_INVALID, "cdata: a run-end encoded parent has no nulls of its own");
  const int rt = run_end_type_of(schema->children[0]->format);
  if (!rt) AG_FAIL(AG_ERR_INVALID, "cdata: run_ends of format '%s' (int16 's', int32 'i' or int64 'l')",
                   schema->children[0]->format ? schema->children[0]->format : "");
  struct ArrowDeviceArray child = *in;
  child.array = *a.children[0];
  AG_TRY(ag_device_array_describe(&child, schema->children[0], run_ends));
  if (run_ends->null_count > 0) AG_FAIL(AG_ERR_INVALID, "cdata: run_ends must not contain nulls");
  child.array = *a.children[1];
  AG_TRY(ag_device_array_describe(&child, schema->children[1], values));
  if (values->length < run_ends->length) AG_FAIL(AG_ERR_INVALID, "cdata: the values child is shorter than run_ends");
  memset(parent, 0, sizeof(*parent));
  parent->type = AG_TYPE_RUN_END_ENCODED;
  parent->length = a.length;
  parent->offset = a.offset;
  parent->device_type = in->device_type;
  parent->device_id = in->device_id;
  return AG_OK;
}

extern "C" ag_status ag_import_run_end_encoded_device_array(struct ArrowDeviceArray* in, const struct ArrowSchema* schema, ag_stream_t consume_on,
                                                            ag_array_view* parent, ag_array_view* run_ends, ag_array_view* values) {
  AG_TRY(ensure_init());
  AG_TRY(ag_run_end_encoded_device_array_describe(in, schema, parent, run_ends, values));
  return import_wait(in, consume_on);
}

extern "C" ag_status ag_export_run_end_encoded_device_array(int value_type, int run_end_type, int64_t length, int64_t offset,
                                                            int64_t n_runs, const void* d_run_ends,
                                                            int64_t values_length, int64_t values_null_count, int64_t values_offset,
                                                            const void* d_values_validity, const void* d_values,
                                                            void (*release_buffers)(void*), void* opaque, ag_stream_t produced_on,
                                                            struct ArrowDeviceArray* out, struct ArrowSchema* out_schema) {
  AG_TRY(ensure_init());
  if (!out) AG_FAIL(AG_ERR_INVALID, "cdata: NULL output");
  if (!ag_type_to_schema_format(value_type)) AG_FAIL(AG_ERR_TYPE, "cdata: unsupported run-end encoded value type id %d", value_type);
  if (run_end_type != AG_TYPE_INT16 && run_end_type != AG_TYPE_INT32 && run_end_type != AG_TYPE_INT64)
    AG_FAIL(AG_ERR_INVALID, "cdata: bad run end type %d", run_end_type);
  if (length < 0 || offset < 0 || n_runs < 0 || values_length < 0 || values_offset < 0) AG_FAIL(AG_ERR_INVALID, "cdata: negative length or offset");
  struct ArrowArray* kids[2] = {nullptr, nullptr};
  struct ArrowSchema* kid_schemas[2] = {nullptr, nullptr};
  struct ArrowSchema** schema_children = nullptr;
  auto cleanup = [&] {
    for (int k = 0; k < 2; ++k) {
      if (kids[k]) { if (kids[k]->release) kids[k]->release(kids[k]); free(kids[k]); }
      if (kid_schemas[k]) { if (kid_schemas[k]->release) kid_schemas[k]->release(kid_schemas[k]); free(kid_schemas[k]); }
    }
    free(schema_children);
  };
  for (int k = 0; k < 2; ++k) {
    kids[k] = static_cast<struct ArrowArray*>(calloc(1, sizeof(struct ArrowArray)));
    if (out_schema) kid_schemas[k] = static_cast<struct ArrowSchema*>(calloc(1, sizeof(struct ArrowSchema)));
    if (!kids[k] || (out_schema && !kid_schemas[k])) { cleanup(); AG_FAIL(AG_ERR_OOM, "cdata: out of host memory"); }
  }
  if (out_schema) {
    schema_children = static_cast<struct ArrowSchema**>(calloc(2, sizeof(struct ArrowSchema*)));
    if (!schema_children) { cleanup(); AG_FAIL(AG_ERR_OOM, "cdata: out of host memory"); }
  }
  // the children: primitive exports whose buffers the parent's release_buffers covers
  struct ArrowDeviceArray tmp;
  ag_status rc = ag_export_device_array(run_end_type, n_runs, 0, 0, nullptr, d_run_ends, nullptr, nullptr, produced_on, &tmp, kid_schemas[0]);
  if (rc != AG_OK) { cleanup(); return rc; }
  *kids[0] = tmp.array;
  rc = ag_export_device_array(value_type, values_length, values_null_count, values_offset, d_values_validity, d_values, nullptr, nullptr,
                              produced_on, &tmp, kid_schemas[1]);
  if (rc != AG_OK) { cleanup(); return rc; }
  *kids[1] = tmp.array;
  // the parent: an empty primitive export turned into "+r" without buffers; its release runs release_buffers, then the
  // children
  rc = ag_export_device_array(value_type, 0, 0, 0, nullptr, nullptr, release_buffers, opaque, produced_on, out, out_schema);
  if (rc != AG_OK) { cleanup(); return rc; }
  ExportState* st = static_cast<ExportState*>(out->array.private_data);
  out->array.length = length;
  out->array.offset = offset;
  st->children[0] = kids[0];
  st->children[1] = kids[1];
  out->array.n_buffers = 0;
  out->array.n_children = 2;
  out->array.children = st->children;
  if (out_schema) {
    kid_schemas[0]->name = "run_ends";
    kid_schemas[0]->flags = 0;   // run ends are never null
    kid_schemas[1]->name = "values";
    schema_children[0] = kid_schemas[0];
    schema_children[1] = kid_schemas[1];
    out_schema->format = "+r";
    out_schema->n_children = 2;
    out_schema->children = schema_children;
    out_schema->release = release_run_end_schema;
  }
  return AG_OK;
}
