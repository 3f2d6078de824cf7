// compute.cc — host-side mirror of arrow-go's compute executors and function registry driving
// the device kernels of libarrowgpu.so.  See arrowgpu_compute.h for the reference map.
#include "arrowgpu_compute.h"

#include <string.h>
#include <algorithm>
#include <mutex>
#include <tuple>

namespace arrowgpu {

// ---------------------------------------------------------------- types -------------------
int BitWidth(Type t) {
  switch (t) {
    case Type::BOOL: return 1;
    case Type::UINT8: case Type::INT8: return 8;
    case Type::UINT16: case Type::INT16: case Type::FLOAT16: return 16;
    case Type::UINT32: case Type::INT32: case Type::FLOAT32: return 32;
    case Type::UINT64: case Type::INT64: case Type::FLOAT64: return 64;
    default: return 0;
  }
}
const char* TypeName(Type t) {
  if (t == Type::DICTIONARY) return "dictionary";
  if (t == Type::RUN_END_ENCODED) return "run_end_encoded";
  static const char* names[] = {"null", "bool", "uint8", "int8", "uint16", "int16", "uint32", "int32", "uint64", "int64", "float16", "float32", "float64"};
  const int i = (int)t;
  return (i >= 0 && i <= 12) ? names[i] : "unknown";
}
bool IsSignedInteger(Type t) { return t == Type::INT8 || t == Type::INT16 || t == Type::INT32 || t == Type::INT64; }
bool IsInteger(Type t) { return IsSignedInteger(t) || t == Type::UINT8 || t == Type::UINT16 || t == Type::UINT32 || t == Type::UINT64; }
bool IsFloating(Type t) { return t == Type::FLOAT32 || t == Type::FLOAT64; }
bool IsNumeric(Type t) { return IsInteger(t) || IsFloating(t); }

Status Status::FromNative(int c) {
  if (c == AG_OK) return OK();
  char buf[512];
  ag_last_error(buf, sizeof(buf));
  return Make(c, buf);
}

#define RETURN_NOT_OK(expr)                \
  do {                                     \
    ::arrowgpu::Status _st = (expr);       \
    if (!_st.ok()) return _st;             \
  } while (0)
#define NATIVE(expr)                                            \
  do {                                                          \
    int _c = (expr);                                            \
    if (_c != AG_OK) return ::arrowgpu::Status::FromNative(_c); \
  } while (0)

static inline int64_t BytesForBits(int64_t n) { return (n + 7) / 8; }
static inline int64_t DataBytes(Type t, int64_t n) { return t == Type::BOOL ? BytesForBits(n) : n * (BitWidth(t) / 8); }
// An n-bit bitmap rounded up to whole 32-bit words: what the kernels that store a word at a time write.
static inline int64_t BitmapWordBytes(int64_t nbits) { return ((nbits + 31) / 32) * 4; }
// Point a span buffer at all of `b`.
static void SetBuffer(exec::BufferSpan* s, const std::shared_ptr<Buffer>& b) { s->buf = b->data(); s->len = b->size(); s->owner = b; }

// ---------------------------------------------------------------- Buffer ------------------
Buffer::~Buffer() {
  if (foreign_) { if (on_release_) on_release_(); }
  else if (data_) ag_dev_free(data_);
}

std::shared_ptr<Buffer> Buffer::Wrap(const void* device_ptr, int64_t nbytes, std::function<void()> on_release) {
  auto b = std::shared_ptr<Buffer>(new Buffer());
  b->data_ = const_cast<uint8_t*>(static_cast<const uint8_t*>(device_ptr));
  b->size_ = nbytes;
  b->foreign_ = true;
  b->on_release_ = std::move(on_release);
  return b;
}

Status Buffer::Allocate(int64_t nbytes, std::shared_ptr<Buffer>* out) {
  auto b = std::shared_ptr<Buffer>(new Buffer());
  void* p = nullptr;
  NATIVE(ag_dev_alloc(&p, (size_t)(nbytes + 8)));  // +8: bitmap kernels address whole 32-bit words
  b->data_ = (uint8_t*)p;
  b->size_ = nbytes;
  *out = std::move(b);
  return Status::OK();
}
Status Buffer::FromHost(const void* host, int64_t nbytes, std::shared_ptr<Buffer>* out) {
  RETURN_NOT_OK(Allocate(nbytes, out));
  if (nbytes) {
    NATIVE(ag_upload((*out)->data(), host, (size_t)nbytes, nullptr));
    NATIVE(ag_stream_sync(nullptr));
  }
  return Status::OK();
}
Status Buffer::ToHost(void* host, int64_t nbytes, int64_t byte_offset) const {
  if (nbytes) {
    NATIVE(ag_download(host, data_ + byte_offset, (size_t)nbytes, nullptr));
    NATIVE(ag_stream_sync(nullptr));
  }
  return Status::OK();
}

// ---------------------------------------------------------------- ArrayData ---------------
namespace {
struct ExportedBuffers { std::shared_ptr<Buffer> b[4]; };   // [2], [3]: a dictionary array's dictionary buffers
void ReleaseExportedBuffers(void* opaque) { delete static_cast<ExportedBuffers*>(opaque); }
}  // namespace

Status ArrayData::ExportDevice(struct ArrowDeviceArray* out, struct ArrowSchema* out_schema) const {
  if (type == Type::RUN_END_ENCODED) {
    const ArrayData &r = *run_ends, &v = *values;
    auto* keep = new ExportedBuffers{{r.buffers[1], v.buffers[0], v.buffers[1]}};
    const int rc = ag_export_run_end_encoded_device_array((int)v.type, (int)r.type, length, offset, r.length,
                                                          r.buffers[1] ? r.buffers[1]->data() + r.offset * (BitWidth(r.type) / 8) : nullptr,
                                                          v.length, v.null_count, v.offset, v.buffers[0] ? v.buffers[0]->data() : nullptr,
                                                          v.buffers[1] ? v.buffers[1]->data() : nullptr, ReleaseExportedBuffers, keep, nullptr, out, out_schema);
    if (rc != AG_OK) { delete keep; return Status::FromNative(rc); }
    return Status::OK();
  }
  if (type == Type::DICTIONARY) {
    const ArrayData& d = *dictionary;
    auto* keep = new ExportedBuffers{{buffers[0], buffers[1], d.buffers[0], d.buffers[1]}};
    const int rc = ag_export_dictionary_device_array((int)d.type, length, null_count, offset, buffers[0] ? buffers[0]->data() : nullptr,
                                                     (const int32_t*)buffers[1]->data(), d.length, d.null_count, d.offset,
                                                     d.buffers[0] ? d.buffers[0]->data() : nullptr, d.buffers[1] ? d.buffers[1]->data() : nullptr,
                                                     ReleaseExportedBuffers, keep, nullptr, out, out_schema);
    if (rc != AG_OK) { delete keep; return Status::FromNative(rc); }
    return Status::OK();
  }
  auto* keep = new ExportedBuffers{{buffers[0], buffers[1]}};
  const int rc = ag_export_device_array((int)type, length, null_count, offset, buffers[0] ? buffers[0]->data() : nullptr,
                                        buffers[1] ? buffers[1]->data() : nullptr, ReleaseExportedBuffers, keep, nullptr, out, out_schema);
  if (rc != AG_OK) { delete keep; return Status::FromNative(rc); }
  return Status::OK();
}

Status ArrayData::ImportDevice(struct ArrowDeviceArray* in, const struct ArrowSchema* schema, std::shared_ptr<ArrayData>* out) {
  if (in && schema && schema->format && strcmp(schema->format, "+r") == 0) {
    ag_array_view pv, rv, vv;
    NATIVE(ag_import_run_end_encoded_device_array(in, schema, nullptr, &pv, &rv, &vv));
    // move the struct: the importer owns it now; the children keep the parent alive, its release releases them
    auto owned = std::make_shared<ArrowDeviceArray>(*in);
    in->array.release = nullptr;
    auto releaser = std::shared_ptr<void>(nullptr, [owned](void*) { if (owned->array.release) owned->array.release(&owned->array); });
    auto child = [&](const ag_array_view& v) {
      auto c = std::make_shared<ArrayData>();
      c->type = (Type)v.type; c->length = v.length; c->offset = v.offset; c->null_count = v.validity ? v.null_count : 0;
      const int64_t m = v.offset + v.length;
      if (v.validity) c->buffers[0] = Buffer::Wrap(v.validity, BytesForBits(m), [releaser] {});
      c->buffers[1] = Buffer::Wrap(v.values, DataBytes(c->type, m), [releaser] {});
      return c;
    };
    auto d = std::make_shared<ArrayData>();
    d->type = Type::RUN_END_ENCODED; d->length = pv.length; d->offset = pv.offset; d->null_count = 0;
    d->run_ends = child(rv);
    d->values = child(vv);
    *out = d;
    return Status::OK();
  }
  const bool dict = in && in->array.dictionary;
  ag_array_view v, dv{};
  if (dict) {
    if (!schema) return Status::Invalid("import: a schema is required");
    NATIVE(ag_import_dictionary_device_array(in, schema, nullptr, &v, &dv));
  } else {
    NATIVE(ag_import_device_array(in, schema, nullptr, &v));
  }
  if (v.type == 0) return Status::Invalid("import: a schema is required");
  // move the struct: the importer owns it now (C Data Interface "moving an array")
  auto owned = std::make_shared<ArrowDeviceArray>(*in);
  in->array.release = nullptr;
  auto releaser = std::shared_ptr<void>(nullptr, [owned](void*) { if (owned->array.release) owned->array.release(&owned->array); });
  auto d = std::make_shared<ArrayData>();
  d->type = (Type)v.type; d->length = v.length; d->offset = v.offset; d->null_count = v.null_count;
  const int64_t n = v.offset + v.length;
  if (v.validity) d->buffers[0] = Buffer::Wrap(v.validity, BytesForBits(n), [releaser] {});
  d->buffers[1] = Buffer::Wrap(v.values, DataBytes((Type)v.type, n), [releaser] {});
  if (!v.validity) d->null_count = 0;
  if (dict) {   // the indices and the dictionary keep the parent alive; its release releases the dictionary
    d->type = Type::DICTIONARY;
    auto c = std::make_shared<ArrayData>();
    c->type = (Type)dv.type; c->length = dv.length; c->offset = dv.offset; c->null_count = dv.validity ? dv.null_count : 0;
    const int64_t m = dv.offset + dv.length;
    if (dv.validity) c->buffers[0] = Buffer::Wrap(dv.validity, BytesForBits(m), [releaser] {});
    c->buffers[1] = Buffer::Wrap(dv.values, DataBytes(c->type, m), [releaser] {});
    d->dictionary = c;
  }
  *out = d;
  return Status::OK();
}

std::shared_ptr<ArrayData> ArrayData::Slice(int64_t off, int64_t len) const {
  auto d = std::make_shared<ArrayData>(*this);
  d->offset = offset + off;
  d->length = len;
  // array.NewSliceData: a slice of an array with nulls has an unknown null count
  if (null_count != 0 && !(off == 0 && len == length)) d->null_count = (null_count == length) ? len : kUnknownNullCount;
  return d;
}

Status ArrayData::FromHost(Type type, int64_t length, int64_t offset, const uint8_t* validity, const void* values,
                           int64_t null_count, std::shared_ptr<ArrayData>* out) {
  if (BitWidth(type) == 0) return Status::TypeError(std::string("unsupported type ") + TypeName(type));
  if (length < 0 || offset < 0) return Status::Invalid("negative length or offset");
  auto d = std::make_shared<ArrayData>();
  d->type = type; d->length = length; d->offset = offset; d->null_count = validity ? null_count : 0;
  RETURN_NOT_OK(Buffer::FromHost(values, DataBytes(type, offset + length), &d->buffers[1]));
  if (validity) RETURN_NOT_OK(Buffer::FromHost(validity, BytesForBits(offset + length), &d->buffers[0]));
  *out = std::move(d);
  return Status::OK();
}

Status ArrayData::ToHost(void* values, uint8_t* validity, int64_t* null_count_out) const {
  if (type == Type::DICTIONARY) return Status::TypeError("to_host: a dictionary array is read through its indices and dictionary");
  if (type == Type::RUN_END_ENCODED) return Status::TypeError("to_host: a run-end encoded array is read through its run ends and values");
  if (length == 0) { if (null_count_out) *null_count_out = 0; return Status::OK(); }
  const int w = BitWidth(type);
  if (values) {
    if (type == Type::BOOL) {
      // re-base to bit 0 on the device, then copy
      std::shared_ptr<Buffer> tmp;
      RETURN_NOT_OK(Buffer::Allocate(BytesForBits(length), &tmp));
      NATIVE(ag_bitmap_copy_dev(buffers[1]->data(), offset, length, tmp->data(), 0, nullptr));
      RETURN_NOT_OK(tmp->ToHost(values, BytesForBits(length)));
    } else {
      RETURN_NOT_OK(buffers[1]->ToHost(values, length * (w / 8), offset * (w / 8)));
    }
  }
  int64_t nulls = null_count;
  if (buffers[0]) {
    std::shared_ptr<Buffer> tmp;
    RETURN_NOT_OK(Buffer::Allocate(BytesForBits(length) + 8, &tmp));
    NATIVE(ag_bitmap_copy_dev(buffers[0]->data(), offset, length, tmp->data(), 0, nullptr));
    if (validity) RETURN_NOT_OK(tmp->ToHost(validity, BytesForBits(length)));
    if (nulls == kUnknownNullCount) {
      int64_t* cnt = (int64_t*)(tmp->data() + ((BytesForBits(length) + 7) & ~7ll));
      std::shared_ptr<Buffer> cbuf;
      RETURN_NOT_OK(Buffer::Allocate(8, &cbuf));
      (void)cnt;
      NATIVE(ag_bitmap_popcount_dev(buffers[0]->data(), offset, length, (int64_t*)cbuf->data(), nullptr));
      int64_t set = 0;
      RETURN_NOT_OK(cbuf->ToHost(&set, 8));
      nulls = length - set;
    }
  } else {
    if (validity) memset(validity, 0xff, (size_t)BytesForBits(length));
    nulls = 0;
  }
  if (null_count_out) *null_count_out = nulls;
  return Status::OK();
}

int64_t ChunkedArray::NullN() const {
  int64_t n = 0;
  for (auto& c : chunks) n += (c->null_count == kUnknownNullCount) ? 1 : c->null_count;  // "may have nulls"
  return n;
}

// A chunked array of type `t` over `chunks`, its length their sum.
static std::shared_ptr<ChunkedArray> MakeChunked(Type t, std::vector<std::shared_ptr<ArrayData>> chunks) {
  auto c = std::make_shared<ChunkedArray>();
  c->type = t; c->chunks = std::move(chunks);
  for (auto& a : c->chunks) c->length += a->length;
  return c;
}

Status MakeRecordBatch(int64_t num_rows, std::vector<std::shared_ptr<ArrayData>> columns, std::shared_ptr<RecordBatch>* out) {
  if (num_rows < 0) return Status::Invalid("record batch: negative row count");
  for (size_t i = 0; i < columns.size(); ++i)
    if (!columns[i] || columns[i]->length != num_rows)
      return Status::Invalid("arrow/array: mismatch number of rows in column " + std::to_string(i) + ": got=" +
                             std::to_string(columns[i] ? columns[i]->length : -1) + ", want=" + std::to_string(num_rows));
  auto r = std::make_shared<RecordBatch>();
  r->num_rows = num_rows; r->columns = std::move(columns);
  *out = r;
  return Status::OK();
}
Status MakeTable(int64_t num_rows, std::vector<std::shared_ptr<ChunkedArray>> columns, std::shared_ptr<Table>* out) {
  if (num_rows < 0) return Status::Invalid("table: negative row count");
  for (size_t i = 0; i < columns.size(); ++i)
    if (!columns[i] || columns[i]->length != num_rows)
      return Status::Invalid("arrow/array: column " + std::to_string(i) + " expected length " + std::to_string(num_rows) + " but got length " +
                             std::to_string(columns[i] ? columns[i]->length : -1));
  auto t = std::make_shared<Table>();
  t->num_rows = num_rows; t->columns = std::move(columns);
  *out = t;
  return Status::OK();
}

namespace compute {
Type Datum::type() const {
  switch (kind) {
    case DatumKind::SCALAR: return scalar->type;
    case DatumKind::ARRAY: return array->type;
    case DatumKind::CHUNKED: return chunked->type;
    default: return Type::NA;
  }
}
int64_t Datum::Len() const {
  switch (kind) {
    case DatumKind::ARRAY: return array->length;
    case DatumKind::CHUNKED: return chunked->length;
    case DatumKind::RECORD: return record->num_rows;
    case DatumKind::TABLE: return table->num_rows;
    default: return -1;
  }
}

int NumColumns(const Datum& d) {
  if (d.kind == DatumKind::RECORD) return (int)d.record->columns.size();
  if (d.kind == DatumKind::TABLE) return (int)d.table->columns.size();
  return 0;
}
Datum ColumnDatum(const Datum& d, int i) {
  return d.kind == DatumKind::RECORD ? Datum(d.record->columns[i]) : Datum(d.table->columns[i]);
}

namespace {
// The chunks of an array (the array itself) or of a chunked array.
std::vector<std::shared_ptr<ArrayData>> ArrayChunks(const Datum& d) {
  return d.kind == DatumKind::ARRAY ? std::vector<std::shared_ptr<ArrayData>>{d.array} : d.chunked->chunks;
}

// A column of a record batch or table as its type and chunks (a record batch column is one chunk).
struct Column { Type type; std::vector<std::shared_ptr<ArrayData>> chunks; };
Column GetColumn(const Datum& d, int i) {
  const Datum c = ColumnDatum(d, i);
  return Column{c.type(), ArrayChunks(c)};
}
}  // namespace
}  // namespace compute

// ======================================================================================
// exec::ArraySpan
// ======================================================================================
namespace exec {

void ArraySpan::SetMembers(const ArrayData& d) {
  type = d.type; len = d.length; nulls = d.null_count; offset = d.offset;
  for (int i = 0; i < 2; ++i) {
    buffers[i] = BufferSpan();
    if (d.buffers[i]) SetBuffer(&buffers[i], d.buffers[i]);
  }
  if (!buffers[0].buf && type != Type::NA) nulls = 0;  // no validity bitmap => no nulls
}

void ArraySpan::SetSlice(int64_t off, int64_t length) {
  if (off == offset && length == len) return;
  if (type != Type::NA) {
    if (nulls != 0) nulls = (nulls == len) ? length : kUnknownNullCount;
  } else {
    nulls = length;
  }
  offset = off; len = length;
}

Status ArraySpan::UpdateNullCount(int64_t* out) {
  if (nulls != kUnknownNullCount) { if (out) *out = nulls; return Status::OK(); }
  if (!buffers[0].buf || buffers[0].len == 0) { nulls = 0; if (out) *out = 0; return Status::OK(); }
  std::shared_ptr<Buffer> cnt;
  RETURN_NOT_OK(Buffer::Allocate(8, &cnt));
  NATIVE(ag_bitmap_popcount_dev(buffers[0].buf, offset, len, (int64_t*)cnt->data(), nullptr));
  int64_t set = 0;
  RETURN_NOT_OK(cnt->ToHost(&set, 8));
  nulls = len - set;
  if (out) *out = nulls;
  return Status::OK();
}

std::shared_ptr<ArrayData> ArraySpan::MakeData() const {
  auto d = std::make_shared<ArrayData>();
  d->type = type; d->length = len; d->null_count = nulls; d->offset = offset;
  for (int i = 0; i < 2; ++i) d->buffers[i] = buffers[i].owner;
  if (!d->buffers[0]) d->null_count = 0;
  return d;
}

}  // namespace exec

// ======================================================================================
// compute: null propagation, span iteration, executors
// ======================================================================================
namespace compute {

using exec::ArraySpan;
using exec::ExecSpan;
using exec::ExecValue;
using exec::KernelCtx;

NullGen GetNullGen(const ExecValue& v) {  // executor.go:190-214
  if (v.type() == Type::NA) return NullGen::ALL_NULL;
  if (v.IsScalar()) return v.scalar->valid ? NullGen::ALL_VALID : NullGen::ALL_NULL;
  const ArraySpan& arr = v.array;
  // do not count if they haven't been counted already
  if (arr.nulls == 0 || arr.buffers[0].buf == nullptr) return NullGen::ALL_VALID;
  if (arr.nulls == arr.len) return NullGen::ALL_NULL;
  return NullGen::PERHAPS_NULL;
}

static NullGen GetNullGenDatum(const Datum& d) {  // executor.go:216-230
  if (d.kind == DatumKind::CHUNKED) return NullGen::PERHAPS_NULL;
  ExecValue v;
  if (d.kind == DatumKind::ARRAY) v.array.SetMembers(*d.array);
  else v.scalar = d.scalar.get();
  return GetNullGen(v);
}

Status PropagateNulls(KernelCtx* ctx, const ExecSpan& batch, ArraySpan* out) {  // executor.go:237-349
  if (out->type == Type::NA) return Status::OK();
  if (out->offset != 0 && out->buffers[0].buf == nullptr)
    return Status::Invalid("can only propagate nulls into pre-allocated memory when output offset is non-zero");
  std::vector<const ArraySpan*> arrs_with_nulls;
  bool is_all_null = false;
  const bool prealloc = out->buffers[0].buf != nullptr;
  for (auto& v : batch.values) {
    const NullGen g = GetNullGen(v);
    if (g == NullGen::ALL_NULL) is_all_null = true;
    if (g != NullGen::ALL_VALID && v.IsArray()) arrs_with_nulls.push_back(&v.array);
  }
  auto alloc_bitmap = [&]() -> Status {
    std::shared_ptr<Buffer> buf;
    RETURN_NOT_OK(ctx->AllocateBitmap(out->len + out->offset, &buf));
    SetBuffer(&out->buffers[0], buf);
    return Status::OK();
  };
  if (is_all_null) {
    out->nulls = out->len;
    if (prealloc) { NATIVE(ag_bitmap_set_dev(out->buffers[0].buf, out->offset, out->len, 0, nullptr)); return Status::OK(); }
    for (auto* arr : arrs_with_nulls) {
      if (arr->nulls == arr->len && arr->buffers[0].owner) { out->buffers[0] = arr->buffers[0]; return Status::OK(); }
    }
    RETURN_NOT_OK(alloc_bitmap());
    NATIVE(ag_bitmap_set_dev(out->buffers[0].buf, out->offset, out->len, 0, nullptr));
    return Status::OK();
  }
  out->nulls = kUnknownNullCount;
  switch (arrs_with_nulls.size()) {
    case 0:
      out->nulls = 0;
      if (prealloc) NATIVE(ag_bitmap_set_dev(out->buffers[0].buf, out->offset, out->len, 1, nullptr));
      return Status::OK();
    case 1: {
      const ArraySpan* arr = arrs_with_nulls[0];
      out->nulls = arr->nulls;
      if (prealloc) {
        NATIVE(ag_bitmap_copy_dev(arr->buffers[0].buf, arr->offset, arr->len, out->buffers[0].buf, out->offset, nullptr));
        return Status::OK();
      }
      if (arr->offset == 0) { out->buffers[0] = arr->buffers[0]; return Status::OK(); }  // zero-copy share
      // (the reference also zero-copies byte-aligned offsets with SliceBuffer; a device Buffer has no
      //  sub-buffer view here, so those are copied like the unaligned case — same bits)
      RETURN_NOT_OK(alloc_bitmap());
      NATIVE(ag_bitmap_copy_dev(arr->buffers[0].buf, arr->offset, arr->len, out->buffers[0].buf, 0, nullptr));
      return Status::OK();
    }
    default: {
      if (!prealloc) RETURN_NOT_OK(alloc_bitmap());
      uint8_t* ob = out->buffers[0].buf;
      NATIVE(ag_bitmap_op_dev(AG_BITOP_AND, arrs_with_nulls[0]->buffers[0].buf, arrs_with_nulls[0]->offset,
                              arrs_with_nulls[1]->buffers[0].buf, arrs_with_nulls[1]->offset, ob, out->offset, out->len, nullptr));
      for (size_t i = 2; i < arrs_with_nulls.size(); ++i)
        NATIVE(ag_bitmap_op_dev(AG_BITOP_AND, ob, out->offset, arrs_with_nulls[i]->buffers[0].buf, arrs_with_nulls[i]->offset,
                                ob, out->offset, out->len, nullptr));
      return Status::OK();
    }
  }
}

// iterateExecSpans, executor.go:757-863, on chunk lengths only (metadata): testable without a GPU.
Status IterateExecSpans(const std::vector<std::vector<int64_t>>& lens, const std::vector<bool>& is_chunked,
                        int64_t max_chunk_size, std::vector<SpanPiece>* out) {
  out->clear();
  const size_t nargs = lens.size();
  int64_t length = -1;
  bool all_same = true;
  for (size_t i = 0; i < nargs; ++i) {
    if (lens[i].empty() && !is_chunked[i]) continue;  // scalar
    int64_t tot = 0;
    for (int64_t l : lens[i]) tot += l;
    if (length < 0) length = tot; else if (length != tot) all_same = false;
  }
  if (length < 0) length = 1;  // all scalars: a single row (checkIfAllScalar / PromoteExecSpanScalars)
  if (!all_same) return Status::Invalid("array args must all be the same length");
  max_chunk_size = std::min(length, max_chunk_size);
  std::vector<int> chunk_idx(nargs, 0);
  std::vector<int64_t> value_pos(nargs, 0);
  int64_t pos = 0;
  while (pos != length) {
    int64_t iter = std::min(length - pos, max_chunk_size);
    for (size_t i = 0; i < nargs && iter > 0; ++i) {
      if (!is_chunked[i]) continue;
      if (lens[i].empty()) { iter = 0; continue; }
      while (value_pos[i] == lens[i][chunk_idx[i]]) { chunk_idx[i]++; value_pos[i] = 0; }  // exhausted or zero-length chunk
      iter = std::min(lens[i][chunk_idx[i]] - value_pos[i], iter);
    }
    SpanPiece p;
    p.pos = pos; p.len = iter; p.chunk_index = chunk_idx; p.chunk_pos = value_pos;
    out->push_back(p);
    for (size_t i = 0; i < nargs; ++i)
      if (!(lens[i].empty() && !is_chunked[i])) value_pos[i] += iter;
    pos += iter;
    if (iter == 0) break;  // degenerate (empty chunked argument)
  }
  return Status::OK();
}

namespace {
// IterateExecSpans over the chunk lengths of each argument (no chunks for a scalar).
Status ChunkSpans(const std::vector<std::vector<std::shared_ptr<ArrayData>>>& args, const std::vector<bool>& is_chunked,
                  int64_t max_chunk_size, std::vector<SpanPiece>* out) {
  std::vector<std::vector<int64_t>> lens(args.size());
  for (size_t i = 0; i < args.size(); ++i)
    for (auto& c : args[i]) lens[i].push_back(c->length);
  return IterateExecSpans(lens, is_chunked, max_chunk_size, out);
}
}  // namespace

// ---------------------------------------------------------------- registry ----------------
Status FunctionRegistry::AddFunction(std::shared_ptr<Function> fn, bool allow_overwrite) {
  if (!allow_overwrite && fns_.count(fn->Name())) return Status::Make(AG_ERR_INVALID, "already have a function registered with name: " + fn->Name());
  fns_[fn->Name()] = std::move(fn);
  return Status::OK();
}
Status FunctionRegistry::AddAlias(const std::string& target, const std::string& source) {
  const Function* f = GetFunction(source);
  if (!f) return Status::Make(AG_ERR_INVALID, "no function registered with name: " + source);  // arrow.ErrKey
  for (auto& kv : fns_) if (kv.second.get() == f) { fns_[target] = kv.second; return Status::OK(); }
  return Status::Invalid("alias source lives in a parent registry");
}
const Function* FunctionRegistry::GetFunction(const std::string& name) const {
  auto it = fns_.find(name);
  if (it != fns_.end()) return it->second.get();
  return parent_ ? parent_->GetFunction(name) : nullptr;
}
std::vector<std::string> FunctionRegistry::GetFunctionNames() const {
  std::vector<std::string> names = parent_ ? parent_->GetFunctionNames() : std::vector<std::string>();
  for (auto& kv : fns_) names.push_back(kv.first);
  std::sort(names.begin(), names.end());
  names.erase(std::unique(names.begin(), names.end()), names.end());
  return names;
}
std::unique_ptr<FunctionRegistry> NewChildRegistry(FunctionRegistry* parent) { return std::unique_ptr<FunctionRegistry>(new FunctionRegistry(parent)); }

template <typename K>
static Status DispatchFirstMatch(const std::string& fname, const std::vector<K>& kernels, const std::vector<Type>& types, const K** out) {
  for (auto& k : kernels) {  // first match wins (functions.go:209-213)
    if (k.any_input_type) { *out = &k; return Status::OK(); }
    if (k.in_types.size() != types.size()) continue;
    bool ok = true;
    for (size_t i = 0; i < types.size(); ++i) ok = ok && (k.in_types[i] == types[i]);
    if (ok) { *out = &k; return Status::OK(); }
  }
  std::string sig;
  for (size_t i = 0; i < types.size(); ++i) sig += std::string(i ? ", " : "") + TypeName(types[i]);
  return Status::NotImplemented("function '" + fname + "' has no kernel matching input types (" + sig + ")");
}
Status ScalarFunction::AddKernel(exec::ScalarKernel k) {
  if (!k.any_input_type && (int)k.in_types.size() != Arity()) return Status::Invalid("kernel arity does not match function arity");
  kernels_.push_back(std::move(k));
  return Status::OK();
}
Status ScalarFunction::DispatchExact(const std::vector<Type>& types, const exec::ScalarKernel** out) const {
  return DispatchFirstMatch(Name(), kernels_, types, out);
}
// commonNumeric, utils.go:178-240
Type CommonNumeric(const std::vector<Type>& types) {
  for (Type t : types) if (!IsInteger(t) && !IsFloating(t)) return Type::NA;
  for (Type t : types) if (t == Type::FLOAT64) return Type::FLOAT64;
  for (Type t : types) if (t == Type::FLOAT32) return Type::FLOAT32;
  int max_signed = 0, max_unsigned = 0;
  for (Type t : types) {
    if (IsSignedInteger(t)) max_signed = std::max(max_signed, BitWidth(t));
    else max_unsigned = std::max(max_unsigned, BitWidth(t));
  }
  if (max_signed == 0) {
    if (max_unsigned >= 64) return Type::UINT64;
    if (max_unsigned == 32) return Type::UINT32;
    if (max_unsigned == 16) return Type::UINT16;
    return Type::UINT8;
  }
  if (max_signed <= max_unsigned) {  // bitutil.NextPowerOf2(maxWidthUnsigned + 1)
    int w = 1;
    while (w < max_unsigned + 1) w <<= 1;
    max_signed = w;
  }
  if (max_signed >= 64) return Type::INT64;
  if (max_signed == 32) return Type::INT32;
  if (max_signed == 16) return Type::INT16;
  return Type::INT8;
}

Status ScalarFunction::DispatchBest(std::vector<Type>* types, const exec::ScalarKernel** out) const {
  if (DispatchExact(*types, out).ok()) return Status::OK();
  if (promote_numeric && types->size() == 2) {  // "only promote types for binary funcs", arithmetic.go:127-137
    const Type common = CommonNumeric(*types);
    if (common != Type::NA) { (*types)[0] = common; (*types)[1] = common; }
  }
  return DispatchExact(*types, out);
}

Status VectorFunction::AddKernel(exec::VectorKernel k) { kernels_.push_back(std::move(k)); return Status::OK(); }
Status VectorFunction::DispatchExact(const std::vector<Type>& types, const exec::VectorKernel** out) const {
  return DispatchFirstMatch(Name(), kernels_, types, out);
}

// ---------------------------------------------------------------- scalar executor ---------
static Status CheckArgs(const Function& fn, const std::vector<Datum>& args) {
  if ((int)args.size() != fn.Arity())
    return Status::Invalid("function '" + fn.Name() + "' accepts " + std::to_string(fn.Arity()) + " arguments but " + std::to_string(args.size()) + " passed");
  for (auto& a : args) if (a.kind == DatumKind::NONE) return Status::Invalid("tried executing function with non-value type");  // checkAllIsValue
  return Status::OK();
}

namespace {
struct ErrorWord {  // device int64 "first failing row", reset per call
  std::shared_ptr<Buffer> buf;
  Status Init() { RETURN_NOT_OK(Buffer::Allocate(8, &buf)); NATIVE(ag_error_word_reset_dev((int64_t*)buf->data(), nullptr)); return Status::OK(); }
  Status Read(int64_t* v) { return buf->ToHost(v, 8); }
  int64_t* word() const { return (int64_t*)buf->data(); }
};
}  // namespace

// scalarExecutor: executor.go:487-728 (Init :435-440, setupPrealloc :658-702, executeSpans :598-623,
// executeSingleSpan :644-656, emitResult :704-728) + WrapResults :521-580.
Status ScalarFunction::Execute(const ExecCtx& ectx, const FunctionOptions* opts, const std::vector<Datum>& args_in, Datum* out) const {
  RETURN_NOT_OK(CheckArgs(*this, args_in));
  std::vector<Type> in_types;
  for (auto& a : args_in) in_types.push_back(a.type());
  const exec::ScalarKernel* kernel = nullptr;
  RETURN_NOT_OK(DispatchBest(&in_types, &kernel));
  // "cast arguments if necessary" (exec.go:101-121): implicit promotion runs the safe cast
  std::vector<Datum> cast_args;
  for (size_t i = 0; i < args_in.size(); ++i) {
    if (args_in[i].type() == in_types[i]) continue;
    if (cast_args.empty()) cast_args = args_in;
    RETURN_NOT_OK(CastDatum(ectx, args_in[i], SafeCastOptions(in_types[i]), &cast_args[i]));
  }
  const std::vector<Datum>& args = cast_args.empty() ? args_in : cast_args;
  const Type out_type = kernel->out_type(in_types);

  // span iteration metadata
  std::vector<std::vector<std::shared_ptr<ArrayData>>> chunks(args.size());
  std::vector<bool> is_chunked(args.size(), false);
  bool have_chunked = false, all_scalar = true;
  for (size_t i = 0; i < args.size(); ++i) {
    if (args[i].kind != DatumKind::ARRAY && args[i].kind != DatumKind::CHUNKED) continue;
    chunks[i] = ArrayChunks(args[i]);
    is_chunked[i] = args[i].kind == DatumKind::CHUNKED;
    have_chunked = have_chunked || is_chunked[i];
    all_scalar = false;
  }
  if (all_scalar) return Status::NotImplemented("scalar-only execution (PromoteExecSpanScalars) is not part of the accelerated path");
  std::vector<SpanPiece> pieces;
  RETURN_NOT_OK(ChunkSpans(chunks, is_chunked, ectx.ChunkSize, &pieces));
  int64_t total = 0;
  for (size_t i = 0; i < args.size(); ++i) if (args[i].kind != DatumKind::SCALAR) { total = args[i].Len(); break; }

  // setupPrealloc (executor.go:658-702)
  bool validity_prealloc = false, elide_validity = false;
  if (out_type != Type::NA) {
    if (kernel->null_handling == exec::NullHandling::COMPUTED_PREALLOC) validity_prealloc = true;
    else if (kernel->null_handling == exec::NullHandling::INTERSECTION) {
      elide_validity = true;
      for (auto& a : args) if (GetNullGenDatum(a) != NullGen::ALL_VALID) { elide_validity = false; break; }
      validity_prealloc = !elide_validity;
    }
  }
  const bool data_prealloc = kernel->mem_alloc == exec::MemAlloc::PREALLOC;
  const bool contiguous = ectx.PreallocContiguous && kernel->can_write_into_slices && data_prealloc &&
                          (validity_prealloc || elide_validity || kernel->null_handling == exec::NullHandling::OUTPUT_NOT_NULL);

  KernelCtx kctx;
  kctx.kernel = kernel;
  kctx.state = opts;
  ErrorWord err_word;
  if (kernel->can_fail) { RETURN_NOT_OK(err_word.Init()); kctx.error_word = err_word.word(); }

  auto prepare_output = [&](int64_t length, ArraySpan* o) -> Status {  // prepareOutput, executor.go:441-470
    *o = ArraySpan();
    o->type = out_type; o->len = length; o->offset = 0; o->nulls = kUnknownNullCount;
    if (validity_prealloc) {
      std::shared_ptr<Buffer> b;
      RETURN_NOT_OK(kctx.AllocateBitmap(length, &b));
      SetBuffer(&o->buffers[0], b);
    }
    if (data_prealloc) {
      std::shared_ptr<Buffer> b;
      RETURN_NOT_OK(kctx.Allocate(DataBytes(out_type, length), &b));  // allocateDataBuffer, executor.go:155-163
      SetBuffer(&o->buffers[1], b);
    }
    if (kernel->null_handling == exec::NullHandling::OUTPUT_NOT_NULL || elide_validity) o->nulls = 0;
    return Status::OK();
  };

  auto build_span = [&](const SpanPiece& p, ExecSpan* span) {
    span->len = p.len;
    span->values.assign(args.size(), ExecValue());
    for (size_t i = 0; i < args.size(); ++i) {
      ExecValue& v = span->values[i];
      if (args[i].kind == DatumKind::SCALAR) { v.scalar = args[i].scalar.get(); continue; }
      const ArrayData& d = (args[i].kind == DatumKind::ARRAY) ? *args[i].array : *args[i].chunked->chunks[p.chunk_index[i]];
      v.array.SetMembers(d);
      v.array.SetSlice(d.offset + p.chunk_pos[i], p.len);
    }
  };

  auto exec_single = [&](const ExecSpan& span, ArraySpan* o) -> Status {  // executeSingleSpan, executor.go:644-656
    if (o->type != Type::NA && kernel->null_handling == exec::NullHandling::INTERSECTION && !elide_validity)
      RETURN_NOT_OK(PropagateNulls(&kctx, span, o));
    return kernel->exec(&kctx, span, o);
  };

  std::vector<std::shared_ptr<ArrayData>> results;
  if (contiguous) {
    ArraySpan output;
    RETURN_NOT_OK(prepare_output(total, &output));
    const bool batched = static_cast<bool>(kernel->exec_batch) && pieces.size() > 1;
    std::vector<ExecSpan> all_spans;
    std::vector<ArraySpan> all_outs;
    for (auto& p : pieces) {
      if (p.len == 0) continue;
      ExecSpan span;
      build_span(p, &span);
      ArraySpan slice = output;
      slice.SetSlice(p.pos, p.len);       // out.SetSlice(resultOffset, input.Len), executor.go:609
      slice.nulls = kUnknownNullCount;
      kctx.row_base = p.pos;
      if (batched) {
        // validity still goes span by span (bitmap launches are tiny); the value kernel runs once
        if (out_type != Type::NA && kernel->null_handling == exec::NullHandling::INTERSECTION && !elide_validity)
          RETURN_NOT_OK(PropagateNulls(&kctx, span, &slice));
        all_spans.push_back(std::move(span));
        all_outs.push_back(slice);
      } else {
        RETURN_NOT_OK(exec_single(span, &slice));
      }
    }
    if (batched && !all_spans.empty()) RETURN_NOT_OK(kernel->exec_batch(&kctx, all_spans, all_outs));
    output.nulls = (elide_validity || kernel->null_handling == exec::NullHandling::OUTPUT_NOT_NULL) ? 0 : kUnknownNullCount;
    results.push_back(output.MakeData());
  } else {
    for (auto& p : pieces) {
      if (p.len == 0 && pieces.size() > 1) continue;
      ExecSpan span;
      build_span(p, &span);
      ArraySpan o;
      RETURN_NOT_OK(prepare_output(p.len, &o));
      kctx.row_base = p.pos;
      RETURN_NOT_OK(exec_single(span, &o));
      results.push_back(o.MakeData());
    }
  }
  if (results.empty()) {  // zero-length input: one empty output
    ArraySpan o;
    RETURN_NOT_OK(prepare_output(0, &o));
    o.nulls = 0;
    results.push_back(o.MakeData());
  }
  if (kernel->can_fail) {
    int64_t bad = 0;
    RETURN_NOT_OK(err_word.Read(&bad));
    if (bad != AG_NO_ERROR_POS) return Status::Invalid(kernel->fail_message);  // the output is released, exec.go:161-170
  }
  // emitResult :704-708 recounts nulls lazily; we leave them unknown (ToHost counts on demand)
  if (have_chunked) {  // WrapResults: Chunked if any input was chunked (executor.go:521-580)
    *out = Datum(MakeChunked(out_type, results));
  } else {
    *out = Datum(results.empty() ? std::make_shared<ArrayData>() : results[0]);
  }
  return Status::OK();
}

// ---------------------------------------------------------------- vector executor ---------
// vectorExecutor, executor.go:886-1154: chunk-wise kernels run once per aligned span and emit one
// output array per span; non-chunkwise kernels (array_take) need whole arrays.
Status VectorFunction::Execute(const ExecCtx& ectx, const FunctionOptions* opts, const std::vector<Datum>& args, Datum* out) const {
  (void)ectx;
  RETURN_NOT_OK(CheckArgs(*this, args));
  std::vector<Type> in_types;
  for (auto& a : args) in_types.push_back(a.type());
  const exec::VectorKernel* kernel = nullptr;
  RETURN_NOT_OK(DispatchExact(in_types, &kernel));
  const Type out_type = kernel->out_type(in_types);
  KernelCtx kctx;
  kctx.kernel = kernel;
  kctx.state = opts;
  bool have_chunked = false;
  std::vector<std::vector<std::shared_ptr<ArrayData>>> chunks(args.size());
  std::vector<bool> is_chunked(args.size(), false);
  for (size_t i = 0; i < args.size(); ++i) {
    if (args[i].kind == DatumKind::SCALAR) return Status::NotImplemented("vector kernels take array-like arguments");
    chunks[i] = ArrayChunks(args[i]);
    is_chunked[i] = args[i].kind != DatumKind::ARRAY;
    have_chunked = have_chunked || is_chunked[i];
  }
  std::vector<std::shared_ptr<ArrayData>> results;
  if (kernel->can_execute_chunkwise) {
    // exec.go:152-155: "vector kernel arguments must all be the same length"
    int64_t l0 = args[0].Len();
    for (auto& a : args) if (a.Len() != l0) return Status::Invalid("vector kernel arguments must all be the same length");
    std::vector<SpanPiece> pieces;
    RETURN_NOT_OK(ChunkSpans(chunks, is_chunked, INT64_MAX, &pieces));
    if (pieces.empty()) { SpanPiece p; p.pos = 0; p.len = 0; p.chunk_index.assign(args.size(), 0); p.chunk_pos.assign(args.size(), 0); pieces.push_back(p); }
    for (auto& p : pieces) {
      ExecSpan span;
      span.len = p.len;
      span.values.assign(args.size(), ExecValue());
      for (size_t i = 0; i < args.size(); ++i) {
        if (args[i].kind == DatumKind::CHUNKED && args[i].chunked->chunks.empty()) { span.values[i].array.type = in_types[i]; continue; }
        const ArrayData& d = (args[i].kind == DatumKind::ARRAY) ? *args[i].array : *args[i].chunked->chunks[p.chunk_index[i]];
        span.values[i].array.SetMembers(d);
        span.values[i].array.SetSlice(d.offset + p.chunk_pos[i], p.len);
      }
      ArraySpan o;
      o.type = out_type;
      RETURN_NOT_OK(kernel->exec(&kctx, span, &o));
      results.push_back(o.MakeData());
    }
  } else if (have_chunked && kernel->exec_chunked && args.size() == 1) {
    ArraySpan o;
    o.type = out_type;
    RETURN_NOT_OK(kernel->exec_chunked(&kctx, *args[0].chunked, &o));
    results.push_back(o.MakeData());
  } else {
    if (have_chunked) return Status::NotImplemented("non-chunkwise vector kernel on chunked input (resolved by the meta function)");
    ExecSpan span;
    span.values.assign(args.size(), ExecValue());
    for (size_t i = 0; i < args.size(); ++i) span.values[i].array.SetMembers(*args[i].array);
    span.len = args.empty() ? 0 : args[0].array->length;
    ArraySpan o;
    o.type = out_type;
    RETURN_NOT_OK(kernel->exec(&kctx, span, &o));
    results.push_back(o.MakeData());
  }
  if (have_chunked) {
    *out = Datum(MakeChunked(out_type, results));
  } else {
    *out = Datum(results[0]);
  }
  return Status::OK();
}

Status CallFunction(const ExecCtx& ctx, const std::string& name, const FunctionOptions* opts, const std::vector<Datum>& args, Datum* out) {
  FunctionRegistry* reg = ctx.Registry ? ctx.Registry : GetFunctionRegistry();
  const Function* fn = reg->GetFunction(name);
  if (!fn) return Status::Make(AG_ERR_INVALID, "no function registered with name: " + name);  // arrow.ErrKey
  // dictionary arrays reach the kernels only through dictionary_encode (its identity case), run-end encoded arrays only
  // through run_end_decode
  for (auto& a : args) {
    if (a.kind == DatumKind::NONE) continue;
    // only sort_indices and take take whole record batches and tables; the kernels of every other function take
    // columns.  "filter" keeps refusing them: FilterRecordBatch / FilterTable filter a record batch or table.
    if (name != "sort_indices" && name != "take" && (a.kind == DatumKind::RECORD || a.kind == DatumKind::TABLE))
      return Status::NotImplemented("function '" + name + "' has no kernel for record batch or table arguments");
    if (name != "dictionary_encode" && a.type() == Type::DICTIONARY) return Status::NotImplemented("function '" + name + "' has no kernel for dictionary arguments");
    if (name != "run_end_decode" && a.type() == Type::RUN_END_ENCODED) return Status::NotImplemented("function '" + name + "' has no kernel for run-end encoded arguments");
  }
  return fn->Execute(ctx, opts, args, out);
}

// ======================================================================================
// kernels (arrow/compute/internal/kernels) on device spans
// ======================================================================================
namespace {

using exec::ExecResult;

inline const uint8_t* ValuesPtr(const ArraySpan& a) {  // exec.GetSpanValues: Buf[1] advanced by Offset (exec/utils.go:38-44)
  return a.buffers[1].buf + a.offset * (BitWidth(a.type) / 8);
}
inline uint8_t* ValuesPtr(ExecResult* a) { return a->buffers[1].buf + a->offset * (BitWidth(a->type) / 8); }

// The validity bitmap a kernel reads, or nullptr when the array has none or no nulls.
const uint8_t* ValidityOrNull(const ArrayData& a) { return a.buffers[0] && a.null_count != 0 ? a.buffers[0]->data() : nullptr; }
bool MayHaveNulls(const ArrayData& a) { return ValidityOrNull(a) != nullptr; }
bool MayHaveNulls(const std::vector<std::shared_ptr<ArrayData>>& chunks) {
  for (auto& c : chunks) if (MayHaveNulls(*c)) return true;
  return false;
}

// Rows [pos, pos + len) of `a` as one chunk of a device chunk list.
ag_sort_chunk ChunkDesc(const ArrayData& a, int64_t pos, int64_t len) {
  return ag_sort_chunk{a.buffers[1] ? a.buffers[1]->data() : nullptr, ValidityOrNull(a), a.offset + pos, len};
}
// The chunk list of a column for ag_sort_indices_keys_dev / ag_take_columns_dev.
std::vector<ag_sort_chunk> ChunkDescs(const std::vector<std::shared_ptr<ArrayData>>& chunks) {
  std::vector<ag_sort_chunk> d;
  for (auto& a : chunks) d.push_back(ChunkDesc(*a, 0, a->length));
  return d;
}

// A new array of `n` rows of type `t` at offset 0 (preallocateData, vector_selection.go:83-93): the values (word-rounded
// for BOOL) and, exactly when `nullable`, a word-rounded validity bitmap with an unknown null count.
Status AllocateOutput(Type t, int64_t n, bool nullable, std::shared_ptr<ArrayData>* out) {
  auto d = std::make_shared<ArrayData>();
  d->type = t; d->length = n; d->offset = 0; d->null_count = nullable ? kUnknownNullCount : 0;
  RETURN_NOT_OK(Buffer::Allocate(t == Type::BOOL ? BitmapWordBytes(n) : n * (BitWidth(t) / 8), &d->buffers[1]));
  if (nullable) RETURN_NOT_OK(Buffer::Allocate(BitmapWordBytes(n), &d->buffers[0]));
  *out = std::move(d);
  return Status::OK();
}

// The IndexError naming the index at row `row` of the `type` indices starting at element `offset` of `buf` (helpers.go:951).
Status IndexOutOfBounds(const Buffer& buf, Type type, int64_t offset, int64_t row) {
  const int iw = BitWidth(type) / 8;
  uint8_t raw[8] = {0};
  RETURN_NOT_OK(buf.ToHost(raw, iw, (offset + row) * iw));
  if (IsSignedInteger(type)) {
    long long v = 0;
    switch (iw) { case 1: v = (int8_t)raw[0]; break; case 2: { int16_t t; memcpy(&t, raw, 2); v = t; break; }
                  case 4: { int32_t t; memcpy(&t, raw, 4); v = t; break; } default: memcpy(&v, raw, 8); }
    return Status::IndexError(std::to_string(v) + " out of bounds");
  }
  unsigned long long uv = 0;
  memcpy(&uv, raw, 8);
  return Status::IndexError(std::to_string(uv) + " out of bounds");
}

const std::vector<Type>& kNumericTypesForCast() {
  static const std::vector<Type> v = {Type::UINT8, Type::INT8, Type::UINT16, Type::INT16, Type::UINT32, Type::INT32,
                                      Type::UINT64, Type::INT64, Type::FLOAT32, Type::FLOAT64};
  return v;
}

int ShapeOf(const ExecSpan& b) { return b.values[0].IsArray() ? (b.values[1].IsArray() ? AG_SHAPE_AA : AG_SHAPE_AS) : AG_SHAPE_SA; }

// ScalarBinary over the native loops (helpers.go:193-236 -> base_arithmetic_amd64.go:34-37)
exec::ArrayKernelExec ArithBinaryExec(int8_t op) {
  return [op](KernelCtx*, const ExecSpan& batch, ExecResult* out) -> Status {
    const int shape = ShapeOf(batch);
    const void* l = batch.values[0].IsArray() ? (const void*)ValuesPtr(batch.values[0].array) : (const void*)batch.values[0].scalar->value;
    const void* r = batch.values[1].IsArray() ? (const void*)ValuesPtr(batch.values[1].array) : (const void*)batch.values[1].scalar->value;
    NATIVE(ag_arith_binary_dev((int)out->type, op, shape, l, r, ValuesPtr(out), batch.len, nullptr));
    return Status::OK();
  };
}

// The same kernel over every aligned span of a chunked call in ONE launch
exec::BatchKernelExec ArithBinaryBatchExec(int8_t op) {
  return [op](KernelCtx*, const std::vector<ExecSpan>& spans, std::vector<ExecResult>& outs) -> Status {
    if (spans.empty()) return Status::OK();
    const int shape = ShapeOf(spans[0]);
    std::vector<ag_span3> table(spans.size());
    for (size_t i = 0; i < spans.size(); ++i) {
      const ExecValue &a = spans[i].values[0], &b = spans[i].values[1];
      table[i].l = a.IsArray() ? (const void*)ValuesPtr(a.array) : (const void*)a.scalar->value;
      table[i].r = b.IsArray() ? (const void*)ValuesPtr(b.array) : (const void*)b.scalar->value;
      table[i].out = ValuesPtr(&outs[i]);
      table[i].n = spans[i].len;
    }
    NATIVE(ag_arith_binary_spans_dev((int)outs[0].type, op, shape, table.data(), (int64_t)table.size(), nullptr));
    return Status::OK();
  };
}

// ScalarBinaryNotNull / checked integer kernels (helpers.go:284-380, base_arithmetic.go:249-294)
exec::ArrayKernelExec ArithCheckedExec(int8_t op) {
  return [op](KernelCtx* ctx, const ExecSpan& batch, ExecResult* out) -> Status {
    const int shape = ShapeOf(batch);
    const ExecValue &a = batch.values[0], &b = batch.values[1];
    // "fast path if one side is entirely null" (helpers.go:287): nothing is written
    if ((a.IsScalar() && !a.scalar->valid) || (b.IsScalar() && !b.scalar->valid)) return Status::OK();
    const void* l = a.IsArray() ? (const void*)a.array.buffers[1].buf : (const void*)a.scalar->value;
    const void* r = b.IsArray() ? (const void*)b.array.buffers[1].buf : (const void*)b.scalar->value;
    const int w = BitWidth(out->type) / 8;
    const uint8_t* lv = (a.IsArray() && a.array.MayHaveNulls()) ? a.array.buffers[0].buf : nullptr;
    const uint8_t* rv = (b.IsArray() && b.array.MayHaveNulls()) ? b.array.buffers[0].buf : nullptr;
    const int64_t loff = a.IsArray() ? a.array.offset : 0, roff = b.IsArray() ? b.array.offset : 0;
    if (a.IsArray()) l = (const uint8_t*)l + loff * w;
    if (b.IsArray()) r = (const uint8_t*)r + roff * w;
    NATIVE(ag_arith_checked_dev((int)out->type, op, shape, l, lv, loff, r, rv, roff, ValuesPtr(out), batch.len, ctx->error_word, nullptr));
    return Status::OK();
  };
}

// AbsoluteValueChecked / NegateChecked (base_arithmetic.go:295-340): every slot, MinInt -> "overflow"
exec::ArrayKernelExec ArithUnaryCheckedExec(int8_t op) {
  return [op](KernelCtx* ctx, const ExecSpan& batch, ExecResult* out) -> Status {
    NATIVE(ag_arith_unary_checked_dev((int)out->type, op, ValuesPtr(batch.values[0].array), ValuesPtr(out), batch.len, ctx->error_word, nullptr));
    return Status::OK();
  };
}

exec::ArrayKernelExec ArithUnaryExec(int8_t op) {
  return [op](KernelCtx*, const ExecSpan& batch, ExecResult* out) -> Status {
    NATIVE(ag_arith_unary_same_dev((int)out->type, op, ValuesPtr(batch.values[0].array), ValuesPtr(out), batch.len, nullptr));
    return Status::OK();
  };
}

// compareKernel (scalar_comparisons.go:199-218): output pointer at byte Offset/8, bit prefix Offset%8
exec::ArrayKernelExec CompareExec(int cmp) {
  return [cmp](KernelCtx*, const ExecSpan& batch, ExecResult* out) -> Status {
    const int shape = ShapeOf(batch);
    const ExecValue &a = batch.values[0], &b = batch.values[1];
    const void* l = a.IsArray() ? (const void*)ValuesPtr(a.array) : (const void*)a.scalar->value;
    const void* r = b.IsArray() ? (const void*)ValuesPtr(b.array) : (const void*)b.scalar->value;
    NATIVE(ag_compare_dev((int)a.type(), cmp, shape, l, r, out->buffers[1].buf + out->offset / 8, batch.len, (int)(out->offset % 8), nullptr));
    return Status::OK();
  };
}

// and / or / xor / and_not (scalar_boolean.go:67-279) incl. the scalar-operand special cases
exec::ArrayKernelExec BoolBinaryExec(int bitop) {
  return [bitop](KernelCtx*, const ExecSpan& batch, ExecResult* out) -> Status {
    const ExecValue &a = batch.values[0], &b = batch.values[1];
    uint8_t* ob = out->buffers[1].buf;
    if (a.IsArray() && b.IsArray()) {
      NATIVE(ag_bitmap_op_dev(bitop, a.array.buffers[1].buf, a.array.offset, b.array.buffers[1].buf, b.array.offset, ob, out->offset, batch.len, nullptr));
      return Status::OK();
    }
    // commutativeBinaryKernel / AndNot CallScalarLeft / CallScalarRight
    const bool scalar_left = a.IsScalar();
    const Scalar* s = scalar_left ? a.scalar : b.scalar;
    const ArraySpan& arr = scalar_left ? b.array : a.array;
    if (!s->valid) return Status::OK();
    bool sv = s->value[0] != 0;
    int op = bitop;
    if (bitop == AG_BITOP_ANDNOT && !scalar_left) { op = AG_BITOP_AND; sv = !sv; }  // AndNot.CallScalarRight = And with inverted scalar
    enum { COPY, INVERT, SET0, SET1 } act;
    switch (op) {
      case AG_BITOP_AND: act = sv ? COPY : SET0; break;
      case AG_BITOP_OR: act = sv ? SET1 : COPY; break;
      case AG_BITOP_XOR: act = sv ? INVERT : COPY; break;
      default: /* ANDNOT, scalar left */ act = sv ? INVERT : SET0; break;
    }
    switch (act) {
      case COPY: NATIVE(ag_bitmap_copy_dev(arr.buffers[1].buf, arr.offset, arr.len, ob, out->offset, nullptr)); break;
      case INVERT: NATIVE(ag_bitmap_invert_dev(arr.buffers[1].buf, arr.offset, arr.len, ob, out->offset, nullptr)); break;
      case SET0: NATIVE(ag_bitmap_set_dev(ob, out->offset, out->len, 0, nullptr)); break;
      case SET1: NATIVE(ag_bitmap_set_dev(ob, out->offset, out->len, 1, nullptr)); break;
    }
    return Status::OK();
  };
}

// Kleene and / or / and_not (scalar_boolean.go:92-334): array ⊕ array through computeKleene
// (:29-65); scalar operands through the CallScalarLeft tables (:109-141, :186-221, :296-330) with
// CallScalarRight = commutative swap (types.go:80-83), and_not's = and_kleene with the scalar
// inverted (:332-334).
exec::ArrayKernelExec KleeneExec(int kop, int plain_bitop) {
  return [kop, plain_bitop](KernelCtx*, const ExecSpan& batch, ExecResult* out) -> Status {
    if (batch.len == 0) return Status::OK();  // SimpleBinary, types.go:91-93
    const ExecValue &a = batch.values[0], &b = batch.values[1];
    uint8_t* ov = out->buffers[0].buf;
    uint8_t* od = out->buffers[1].buf;
    const int64_t oo = out->offset, n = batch.len;
    if (a.IsArray() && b.IsArray()) {
      ArraySpan l = a.array, r = b.array;
      int64_t ln = 0, rn = 0;
      RETURN_NOT_OK(l.UpdateNullCount(&ln));
      RETURN_NOT_OK(r.UpdateNullCount(&rn));
      if (ln == 0 && rn == 0) {
        NATIVE(ag_bitmap_set_dev(ov, oo, n, 1, nullptr));
        out->nulls = 0;
        NATIVE(ag_bitmap_op_dev(plain_bitop, l.buffers[1].buf, l.offset, r.buffers[1].buf, r.offset, od, oo, n, nullptr));
        return Status::OK();
      }
      NATIVE(ag_kleene_dev(kop, ln ? l.buffers[0].buf : nullptr, l.buffers[1].buf, l.offset, rn ? r.buffers[0].buf : nullptr, r.buffers[1].buf, r.offset,
                           ov, od, oo, n, nullptr));
      out->nulls = kUnknownNullCount;
      return Status::OK();
    }
    // one scalar operand.  Reduce to "scalar on the left" of a (possibly different) kernel.
    const bool scalar_left = a.IsScalar();
    const Scalar* sc = scalar_left ? a.scalar : b.scalar;
    ArraySpan arr = scalar_left ? b.array : a.array;
    bool s_valid = sc->valid, s_val = sc->value[0] != 0;
    int op = kop;  // which CallScalarLeft table to use
    if (kop == AG_KLEENE_ANDNOT && !scalar_left) { op = AG_KLEENE_AND; s_val = !s_val; }  // :332-334 (invertScalar keeps nulls)
    int64_t an = 0;
    RETURN_NOT_OK(arr.UpdateNullCount(&an));
    const uint8_t* av = arr.buffers[0].buf;
    const uint8_t* ad = arr.buffers[1].buf;
    const int64_t ao = arr.offset;
    auto all_valid = [&]() -> Status { NATIVE(ag_bitmap_set_dev(ov, oo, n, 1, nullptr)); out->nulls = 0; return Status::OK(); };
    auto copy_valid_from_arr = [&]() -> Status {
      if (an == 0) return all_valid();
      NATIVE(ag_bitmap_copy_dev(av, ao, n, ov, oo, nullptr));
      out->nulls = kUnknownNullCount;
      return Status::OK();
    };
    out->nulls = kUnknownNullCount;
    const bool s_true = s_valid && s_val, s_false = s_valid && !s_val;
    if (op == AG_KLEENE_AND) {          // KleeneAndOpKernel.CallScalarLeft :109-141
      if (s_false) { RETURN_NOT_OK(all_valid()); NATIVE(ag_bitmap_set_dev(od, oo, n, 0, nullptr)); }
      else if (s_true) { RETURN_NOT_OK(copy_valid_from_arr()); NATIVE(ag_bitmap_copy_dev(ad, ao, n, od, oo, nullptr)); }
      else {  // null scalar: valid iff right is (valid and) false
        if (an == 0) NATIVE(ag_bitmap_invert_dev(ad, ao, n, ov, oo, nullptr));
        else NATIVE(ag_bitmap_op_dev(AG_BITOP_ANDNOT, av, ao, ad, ao, ov, oo, n, nullptr));
        NATIVE(ag_bitmap_copy_dev(ad, ao, n, od, oo, nullptr));
      }
    } else if (op == AG_KLEENE_OR) {    // KleeneOrOpKernel.CallScalarLeft :186-221
      if (s_true) { RETURN_NOT_OK(all_valid()); NATIVE(ag_bitmap_set_dev(od, oo, n, 1, nullptr)); }
      else if (s_false) { RETURN_NOT_OK(copy_valid_from_arr()); NATIVE(ag_bitmap_copy_dev(ad, ao, n, od, oo, nullptr)); }
      else {  // null scalar: valid iff right is (valid and) true
        if (an == 0) NATIVE(ag_bitmap_copy_dev(ad, ao, n, ov, oo, nullptr));
        else NATIVE(ag_bitmap_op_dev(AG_BITOP_AND, av, ao, ad, ao, ov, oo, n, nullptr));
        NATIVE(ag_bitmap_copy_dev(ad, ao, n, od, oo, nullptr));
      }
    } else {                            // KleeneAndNotOpKernel.CallScalarLeft :296-330 (scalar AND NOT array)
      if (s_false) { RETURN_NOT_OK(all_valid()); NATIVE(ag_bitmap_set_dev(od, oo, n, 0, nullptr)); }
      else if (s_true) { RETURN_NOT_OK(copy_valid_from_arr()); NATIVE(ag_bitmap_invert_dev(ad, ao, n, od, oo, nullptr)); }
      else {  // null scalar: valid iff right is (valid and) true
        if (an == 0) NATIVE(ag_bitmap_copy_dev(ad, ao, n, ov, oo, nullptr));
        else NATIVE(ag_bitmap_op_dev(AG_BITOP_AND, av, ao, ad, ao, ov, oo, n, nullptr));
        NATIVE(ag_bitmap_invert_dev(ad, ao, n, od, oo, nullptr));
      }
    }
    return Status::OK();
  };
}

// isNullExec / isNotNullExec (scalar_comparisons.go:718-745): NullComputedNoPrealloc, MemNoPrealloc,
// the output never has a validity bitmap
Status IsNullExec(KernelCtx* ctx, const ExecSpan& batch, ExecResult* out) {
  const ArraySpan& in = batch.values[0].array;
  std::shared_ptr<Buffer> b;
  RETURN_NOT_OK(ctx->AllocateBitmap(in.len, &b));  // zero-filled: "no validity buffer" means all false
  if (in.buffers[0].buf) NATIVE(ag_bitmap_invert_dev(in.buffers[0].buf, in.offset, in.len, b->data(), 0, nullptr));
  out->type = Type::BOOL; out->len = in.len; out->offset = 0; out->nulls = 0;
  out->buffers[0] = exec::BufferSpan();
  SetBuffer(&out->buffers[1], b);
  return Status::OK();
}
Status IsNotNullExec(KernelCtx* ctx, const ExecSpan& batch, ExecResult* out) {
  const ArraySpan& in = batch.values[0].array;
  std::shared_ptr<Buffer> b;
  RETURN_NOT_OK(ctx->AllocateBitmap(in.len, &b));
  if (in.buffers[0].buf) NATIVE(ag_bitmap_copy_dev(in.buffers[0].buf, in.offset, in.len, b->data(), 0, nullptr));
  else NATIVE(ag_bitmap_set_dev(b->data(), 0, in.len, 1, nullptr));  // memory.Set(0xFF)
  out->type = Type::BOOL; out->len = in.len; out->offset = 0; out->nulls = 0;
  out->buffers[0] = exec::BufferSpan();
  SetBuffer(&out->buffers[1], b);
  return Status::OK();
}
// isNanKernelExec (scalar_comparisons.go:754-765): the NE kernel with the input on both sides;
// integer inputs are ConstBoolExec(false) (:747-752)
Status IsNanExec(KernelCtx*, const ExecSpan& batch, ExecResult* out) {
  const ArraySpan& in = batch.values[0].array;
  if (!IsFloating(in.type)) { NATIVE(ag_bitmap_set_dev(out->buffers[1].buf, out->offset, batch.len, 0, nullptr)); return Status::OK(); }
  NATIVE(ag_compare_dev((int)in.type, AG_CMP_NE, AG_SHAPE_AA, ValuesPtr(in), ValuesPtr(in), out->buffers[1].buf + out->offset / 8, batch.len,
                        (int)(out->offset % 8), nullptr));
  return Status::OK();
}

// NotExecKernel (scalar_boolean.go:336-347): invert data, share the validity buffer
// ---- numeric casts (kernels/numeric_cast.go:37-71 over cast_numeric.go:101-131) ----------
// Integer bounds of intsCanFit / checkIntToFloatTrunc, only needed to word the error like the
// reference ("integer value %d not in range: %d to %d", helpers.go:591-594).
void SafeIntBounds(Type in, Type out, __int128* lo, __int128* hi) {
  auto tmin = [](Type t) -> __int128 { return IsSignedInteger(t) ? -((__int128)1 << (BitWidth(t) - 1)) : 0; };
  auto tmax = [](Type t) -> __int128 { return IsSignedInteger(t) ? ((__int128)1 << (BitWidth(t) - 1)) - 1 : ((__int128)1 << BitWidth(t)) - 1; };
  if (IsFloating(out)) {
    const int mant = out == Type::FLOAT32 ? 24 : 53;
    *hi = (__int128)1 << mant;
    *lo = IsSignedInteger(in) ? -*hi : 0;
    return;
  }
  *lo = std::max(tmin(in), tmin(out));
  *hi = std::min(tmax(in), tmax(out));
}
std::string Int128ToString(__int128 v) {
  if (v == 0) return "0";
  const bool neg = v < 0;
  unsigned __int128 u = neg ? (unsigned __int128)(-(v + 1)) + 1 : (unsigned __int128)v;
  std::string r;
  while (u) { r.insert(r.begin(), (char)('0' + (int)(u % 10))); u /= 10; }
  return neg ? "-" + r : r;
}

const char* CastFunctionName(Type t);

Status CastNumericExec(KernelCtx* ctx, const ExecSpan& batch, ExecResult* out) {
  // cast_<type> called by name carries whatever options the caller passed (functions.go:163-167 refuses none)
  const auto* fo = static_cast<const FunctionOptions*>(ctx->state);   // the executor's state is the call's options
  const auto* opts = dynamic_cast<const CastOptions*>(fo);
  if (!fo) return Status::Invalid(std::string("function '") + CastFunctionName(out->type) + "' cannot be called without options");
  if (!opts) return Status::Invalid(std::string(CastFunctionName(out->type)) + ": expected CastOptions, got " + fo->TypeName());
  const ArraySpan& in = batch.values[0].array;
  if (batch.len == 0) return Status::OK();
  NATIVE(ag_cast_numeric_checked_dev((int)in.type, (int)out->type, ValuesPtr(in), in.buffers[0].buf, in.offset, ValuesPtr(out), batch.len,
                                     opts->AllowIntOverflow ? 1 : 0, opts->AllowFloatTruncate ? 1 : 0, ctx->error_word, nullptr));
  // one 8-byte read per span: the error names the offending VALUE, like the reference's does
  int64_t bad = AG_NO_ERROR_POS;
  NATIVE(ag_download(&bad, ctx->error_word, sizeof(bad), nullptr));
  NATIVE(ag_stream_sync(nullptr));
  if (bad == AG_NO_ERROR_POS) return Status::OK();
  const int w = BitWidth(in.type) / 8;
  uint8_t raw[8] = {0};
  NATIVE(ag_download(raw, ValuesPtr(in) + bad * w, (size_t)w, nullptr));
  NATIVE(ag_stream_sync(nullptr));
  if (IsFloating(in.type)) {  // numeric_cast.go:614-617
    double v;
    if (in.type == Type::FLOAT32) { float f; memcpy(&f, raw, 4); v = f; } else memcpy(&v, raw, 8);
    char buf[128];
    snprintf(buf, sizeof(buf), "float value %f was truncated converting to %s", v, TypeName(out->type));
    return Status::Invalid(buf);
  }
  __int128 v = 0, lo, hi;
  switch (in.type) {
    case Type::INT8: v = (int8_t)raw[0]; break;
    case Type::UINT8: v = raw[0]; break;
    case Type::INT16: { int16_t t; memcpy(&t, raw, 2); v = t; break; }
    case Type::UINT16: { uint16_t t; memcpy(&t, raw, 2); v = t; break; }
    case Type::INT32: { int32_t t; memcpy(&t, raw, 4); v = t; break; }
    case Type::UINT32: { uint32_t t; memcpy(&t, raw, 4); v = t; break; }
    case Type::INT64: { int64_t t; memcpy(&t, raw, 8); v = t; break; }
    default: { uint64_t t; memcpy(&t, raw, 8); v = t; break; }
  }
  SafeIntBounds(in.type, out->type, &lo, &hi);
  return Status::Invalid("integer value " + Int128ToString(v) + " not in range: " + Int128ToString(lo) + " to " + Int128ToString(hi));
}

const char* CastFunctionName(Type t) {  // cast.go:841-880
  switch (t) {
    case Type::INT8: return "cast_int8"; case Type::INT16: return "cast_int16"; case Type::INT32: return "cast_int32";
    case Type::INT64: return "cast_int64"; case Type::UINT8: return "cast_uint8"; case Type::UINT16: return "cast_uint16";
    case Type::UINT32: return "cast_uint32"; case Type::UINT64: return "cast_uint64"; case Type::FLOAT32: return "cast_float";
    case Type::FLOAT64: return "cast_double"; default: return nullptr;
  }
}

std::shared_ptr<ScalarFunction> MakeCastTo(Type to) {  // GetCastToInteger / GetCastToFloating, numeric_cast.go:835-906
  auto fn = std::make_shared<ScalarFunction>(CastFunctionName(to), 1);
  for (Type t : kNumericTypesForCast()) {
    exec::ScalarKernel k;
    k.in_types = {t};
    k.out_type = [to](const std::vector<Type>&) { return to; };
    k.exec = CastNumericExec;
    k.expr_op = AG_EXPR_CAST;
    k.can_fail = true;  // the executor supplies the error word; CastNumericExec words the error itself
    k.fail_message = "cast failed";
    fn->AddKernel(std::move(k));
  }
  return fn;
}

Status NotExec(KernelCtx*, const ExecSpan& batch, ExecResult* out) {
  const ArraySpan& in = batch.values[0].array;
  NATIVE(ag_bitmap_invert_dev(in.buffers[1].buf, in.offset, in.len, out->buffers[1].buf, out->offset, nullptr));
  if (in.buffers[0].buf && in.nulls != 0) {
    if (in.offset == out->offset) out->buffers[0] = in.buffers[0];
    else {
      std::shared_ptr<Buffer> b;
      RETURN_NOT_OK(Buffer::Allocate((out->offset + out->len + 7) / 8, &b));
      NATIVE(ag_bitmap_copy_dev(in.buffers[0].buf, in.offset, in.len, b->data(), out->offset, nullptr));
      SetBuffer(&out->buffers[0], b);
    }
  }
  out->nulls = in.nulls;
  return Status::OK();
}

// PrimitiveFilter (vector_selection.go:449-520)
Status PrimitiveFilterExec(KernelCtx* ctx, const ExecSpan& batch, ExecResult* out) {
  ArraySpan values = batch.values[0].array, filter = batch.values[1].array;
  const FilterOptions* opts = static_cast<const FilterOptions*>(ctx->state);
  const int sel = opts ? (int)opts->NullSelection : (int)DropNulls;
  int64_t vn = 0, fn = 0;
  RETURN_NOT_OK(values.UpdateNullCount(&vn));
  RETURN_NOT_OK(filter.UpdateNullCount(&fn));
  const uint8_t* mvalid = fn != 0 ? filter.buffers[0].buf : nullptr;
  const uint8_t* vvalid = vn != 0 ? values.buffers[0].buf : nullptr;
  // getFilterOutputSize (:57-81)
  std::shared_ptr<Buffer> scal;
  RETURN_NOT_OK(Buffer::Allocate(16, &scal));
  NATIVE(ag_filter_output_size_dev(filter.buffers[1].buf, mvalid, filter.offset, filter.len, sel, (int64_t*)scal->data(), nullptr));
  int64_t out_len = 0;
  RETURN_NOT_OK(scal->ToHost(&out_len, 8));
  const bool allocate_validity = vn != 0 || fn != 0;                                  // :473
  std::shared_ptr<ArrayData> res;
  RETURN_NOT_OK(AllocateOutput(values.type, out_len, allocate_validity, &res));   // preallocateData (:83-93)
  out->SetMembers(*res);
  out->nulls = (vn == 0 && (sel == DropNulls || fn == 0)) ? 0 : kUnknownNullCount;  // :464-468
  if (values.len == 0) return Status::OK();
  NATIVE(ag_filter_primitive_dev(BitWidth(values.type), values.buffers[1].buf, vvalid, values.offset, filter.buffers[1].buf, mvalid, filter.offset,
                                 values.len, sel, out->buffers[1].buf, out->buffers[0].buf, out_len, (int64_t*)scal->data() + 1, nullptr));
  return Status::OK();
}

// ---- cumulative_sum[_checked] (kernels/vector_cumulative.go:332-410) -------------------------
// cumulativeStartValue :81-112: nil -> zero, null scalar -> error, other types -> safe cast.
Status CumulativeStart(const CumulativeOptions* opts, Type t, bool* has_start, uint8_t (&raw)[8]) {
  *has_start = false;
  memset(raw, 0, 8);
  if (!opts || !opts->Start) return Status::OK();
  if (!opts->Start->valid) return Status::Invalid("cumulative sum start value must be valid");
  std::shared_ptr<Scalar> sc = opts->Start;
  if (sc->type != t) {
    Datum casted;
    ExecCtx ectx;
    Status st = CastDatum(ectx, Datum(sc), SafeCastOptions(t), &casted);
    if (!st.ok()) return Status::Invalid(std::string("cannot cast cumulative sum start value to ") + TypeName(t) + ": " + st.msg);
    sc = casted.scalar;
  }
  memcpy(raw, sc->value, 8);
  *has_start = true;
  return Status::OK();
}

struct CumsumRun {  // device state + error word shared by the chunks of one call
  std::shared_ptr<Buffer> state;
  ErrorWord bad;
  Status Init(Type t, const CumulativeOptions* opts) {
    bool has_start; uint8_t raw[8];
    RETURN_NOT_OK(CumulativeStart(opts, t, &has_start, raw));
    RETURN_NOT_OK(Buffer::Allocate(sizeof(ag_cumsum_state), &state));
    NATIVE(ag_cumulative_sum_state_init_dev(state->data(), (int)t, has_start ? raw : nullptr, nullptr));
    return bad.Init();
  }
};

// cumulativeSumSpans: one output array for all input spans; validity only when some span may have nulls
Status CumulativeSpans(bool checked, const CumulativeOptions* opts, Type t, const std::vector<ArraySpan>& inputs, ExecResult* out) {
  if (!IsInteger(t) && !IsFloating(t)) return Status::TypeError(std::string("cumulative sum input type must be numeric, got ") + TypeName(t));
  int64_t total = 0;
  bool needs_validity = false;
  for (auto& in : inputs) { total += in.len; needs_validity = needs_validity || (in.buffers[0].buf != nullptr && in.nulls != 0); }
  out->type = t; out->len = total; out->offset = 0; out->nulls = 0;
  if (total == 0) {   // no rows, but the start value is still checked: initCumulativeSum runs for every call (:119-144)
    bool has_start;
    uint8_t raw[8];
    return CumulativeStart(opts, t, &has_start, raw);
  }
  CumsumRun run;
  RETURN_NOT_OK(run.Init(t, opts));
  std::shared_ptr<Buffer> data, validity;
  const int w = BitWidth(t) / 8;
  RETURN_NOT_OK(Buffer::Allocate(total * w, &data));
  if (needs_validity) RETURN_NOT_OK(Buffer::Allocate(BytesForBits(total), &validity));
  int64_t pos = 0;
  for (auto& in : inputs) {
    if (in.len == 0) continue;
    // a bitmap that is known to be all set (null_count == 0: Array.from_numpy(valid=all true), filter / take outputs,
    // preallocated PropagateNulls bitmaps) takes the no-nulls path like the reference (vector_cumulative.go:341-346)
    const uint8_t* in_valid = in.nulls != 0 ? in.buffers[0].buf : nullptr;
    NATIVE(ag_cumulative_sum_dev((int)t, ValuesPtr(in), in_valid, in.offset, in.len, opts && opts->SkipNulls ? 1 : 0, checked ? 1 : 0,
                                 data->data() + pos * w, validity ? validity->data() : nullptr, pos, run.state->data(), run.bad.word(), nullptr));
    pos += in.len;
  }
  if (checked) {
    int64_t bad = 0;
    RETURN_NOT_OK(run.bad.Read(&bad));
    if (bad != AG_NO_ERROR_POS) return Status::Invalid("overflow");  // errOverflow, base_arithmetic.go:137
  }
  SetBuffer(&out->buffers[1], data);
  if (validity) {
    ag_cumsum_state hs;
    RETURN_NOT_OK(run.state->ToHost(&hs, sizeof(hs)));
    SetBuffer(&out->buffers[0], validity);
    out->nulls = hs.null_count;
  }
  return Status::OK();
}

exec::ArrayKernelExec CumulativeExec(bool checked) {  // cumulativeSumExec :370-383
  return [checked](KernelCtx* ctx, const ExecSpan& batch, ExecResult* out) -> Status {
    const ArraySpan& in = batch.values[0].array;
    return CumulativeSpans(checked, static_cast<const CumulativeOptions*>(ctx->state), in.type, {in}, out);
  };
}

std::function<Status(KernelCtx*, const ChunkedArray&, ExecResult*)> CumulativeExecChunked(bool checked) {  // :385-410
  return [checked](KernelCtx* ctx, const ChunkedArray& c, ExecResult* out) -> Status {
    std::vector<ArraySpan> spans(c.chunks.size());
    for (size_t i = 0; i < c.chunks.size(); ++i) spans[i].SetMembers(*c.chunks[i]);
    return CumulativeSpans(checked, static_cast<const CumulativeOptions*>(ctx->state), c.type, spans, out);
  };
}

std::shared_ptr<VectorFunction> MakeCumulative(const std::string& name, bool checked) {
  auto fn = std::make_shared<VectorFunction>(name, 1);
  exec::VectorKernel k;
  k.any_input_type = true;  // the exec rejects non-numeric inputs with ErrType like the reference's start-value check
  k.out_type = [](const std::vector<Type>& t) { return t[0]; };
  k.exec = CumulativeExec(checked);
  k.exec_chunked = CumulativeExecChunked(checked);
  k.null_handling = exec::NullHandling::COMPUTED_NO_PREALLOC;
  k.mem_alloc = exec::MemAlloc::NO_PREALLOC;
  k.can_execute_chunkwise = false;  // vector_cumulative.go:420-421
  fn->AddKernel(std::move(k));
  return fn;
}

// PrimitiveTake (vector_selection.go:1162-1192)
Status PrimitiveTakeExec(KernelCtx* ctx, const ExecSpan& batch, ExecResult* out) {
  ArraySpan values = batch.values[0].array, indices = batch.values[1].array;
  const TakeOptions* opts = static_cast<const TakeOptions*>(ctx->state);
  const bool bounds = opts ? opts->BoundsCheck : true;
  if (!IsInteger(indices.type)) return Status::Invalid("invalid index type for bounds checking");  // helpers.go:978
  int64_t vn = 0, in_ = 0;
  RETURN_NOT_OK(values.UpdateNullCount(&vn));
  RETURN_NOT_OK(indices.UpdateNullCount(&in_));
  const bool allocate_validity = vn != 0 || in_ != 0;  // :1175
  std::shared_ptr<ArrayData> res;
  RETURN_NOT_OK(AllocateOutput(values.type, indices.len, allocate_validity, &res));
  out->SetMembers(*res);
  if (indices.len == 0) return Status::OK();
  ErrorWord word;
  RETURN_NOT_OK(word.Init());
  const int iw = BitWidth(indices.type);
  NATIVE(ag_take_primitive_dev(BitWidth(values.type), values.buffers[1].buf, vn ? values.buffers[0].buf : nullptr, values.offset, values.len, iw,
                               IsSignedInteger(indices.type), indices.buffers[1].buf + indices.offset * (iw / 8), in_ ? indices.buffers[0].buf : nullptr,
                               indices.offset, indices.len, bounds ? 1 : 0, out->buffers[1].buf, out->buffers[0].buf, word.word(), nullptr));
  if (bounds) {
    int64_t bad = 0;
    RETURN_NOT_OK(word.Read(&bad));
    if (bad != AG_NO_ERROR_POS) return IndexOutOfBounds(*indices.buffers[1].owner, indices.type, indices.offset, bad);
  }
  return Status::OK();
}

// The expression-program op of a kernel, read from the device op its exec launches: the plain loops of
// ag_arith_binary_dev / ag_arith_unary_same_dev (launch_binary, launch_unary_same_op: a *_CHECKED op there is the plain
// loop) and the checked kernels of ag_arith_checked_dev / ag_arith_unary_checked_dev (launch_checked_op).
int PlainExprOp(int8_t op) {
  switch (op) {
    case AG_OP_ADD: case AG_OP_ADD_CHECKED: return AG_EXPR_ADD;
    case AG_OP_SUB: case AG_OP_SUB_CHECKED: return AG_EXPR_SUB;
    case AG_OP_MUL: case AG_OP_MUL_CHECKED: return AG_EXPR_MUL;
    case AG_OP_BIT_AND: return AG_EXPR_BIT_AND;
    case AG_OP_BIT_OR: return AG_EXPR_BIT_OR;
    case AG_OP_BIT_XOR: return AG_EXPR_BIT_XOR;
    case AG_OP_ABS: case AG_OP_ABS_CHECKED: return AG_EXPR_ABS;
    case AG_OP_NEGATE: return AG_EXPR_NEG;
    case AG_OP_NEGATE_CHECKED: return AG_EXPR_NEG_UNSIGNED_ZERO;
    case AG_OP_SIGN: return AG_EXPR_SIGN;
    case AG_OP_BIT_NOT: return AG_EXPR_BIT_NOT;
    default: return -1;
  }
}
int CheckedExprOp(int8_t op) {
  switch (op) {
    case AG_OP_ADD_CHECKED: return AG_EXPR_ADD_CHECKED;
    case AG_OP_SUB_CHECKED: return AG_EXPR_SUB_CHECKED;
    case AG_OP_MUL_CHECKED: return AG_EXPR_MUL_CHECKED;
    case AG_OP_DIV: return AG_EXPR_DIV;
    case AG_OP_DIV_CHECKED: return AG_EXPR_DIV_CHECKED;
    case AG_OP_SHIFT_LEFT: return AG_EXPR_SHL;
    case AG_OP_SHIFT_RIGHT: return AG_EXPR_SHR;
    case AG_OP_SHIFT_LEFT_CHECKED: return AG_EXPR_SHL_CHECKED;
    case AG_OP_SHIFT_RIGHT_CHECKED: return AG_EXPR_SHR_CHECKED;
    case AG_OP_ABS_CHECKED: return AG_EXPR_ABS_CHECKED;
    case AG_OP_NEGATE_CHECKED: return AG_EXPR_NEG_CHECKED;
    default: return -1;
  }
}

Type FirstType(const std::vector<Type>& t) { return t[0]; }
Type BoolType(const std::vector<Type>&) { return Type::BOOL; }

const Type kNumericTypes[] = {Type::UINT8, Type::INT8, Type::UINT16, Type::INT16, Type::UINT32, Type::INT32, Type::UINT64, Type::INT64, Type::FLOAT32, Type::FLOAT64};

std::shared_ptr<ScalarFunction> MakeArithBinary(const std::string& name, int8_t unchecked_op, int8_t checked_op, bool checked, const char* fail_msg) {
  // GetArithmeticBinaryKernels (scalar_arithmetic.go:86-95): one [ty,ty]->ty kernel per numeric type
  auto fn = std::make_shared<ScalarFunction>(name, 2);
  fn->promote_numeric = true;  // arithmeticFunction.DispatchBest, arithmetic.go:112-140
  for (Type t : kNumericTypes) {
    exec::ScalarKernel k;
    k.in_types = {t, t};
    k.out_type = FirstType;
    if (checked && IsInteger(t)) {  // integral checked funcs use the NotNull versions (base_arithmetic_amd64.go:103-106)
      k.exec = ArithCheckedExec(checked_op);
      k.expr_op = CheckedExprOp(checked_op);
      k.can_fail = true;
      k.fail_message = fail_msg;
    } else {
      k.exec = ArithBinaryExec(checked ? checked_op : unchecked_op);
      k.expr_op = PlainExprOp(checked ? checked_op : unchecked_op);
      k.exec_batch = ArithBinaryBatchExec(checked ? checked_op : unchecked_op);
    }
    fn->AddKernel(std::move(k));
  }
  return fn;
}

// divide / divide_unchecked (arithmetic.go:782-785; kernels base_arithmetic.go:154-161,287-294,386-397): every kernel is
// ScalarBinaryNotNull.  Integers fail on a zero divisor in BOTH flavours; floats only in the checked one.
std::shared_ptr<ScalarFunction> MakeDivide(const std::string& name, bool checked) {
  auto fn = std::make_shared<ScalarFunction>(name, 2);
  fn->promote_numeric = true;
  for (Type t : kNumericTypes) {
    exec::ScalarKernel k;
    k.in_types = {t, t};
    k.out_type = FirstType;
    k.exec = ArithCheckedExec(checked ? AG_OP_DIV_CHECKED : AG_OP_DIV);
    k.expr_op = CheckedExprOp(checked ? AG_OP_DIV_CHECKED : AG_OP_DIV);
    k.can_fail = true;   // the NotNull entry point always takes an error word; the unchecked float op never raises it
    k.fail_message = "divide by zero";
    fn->AddKernel(std::move(k));
  }
  return fn;
}

const Type kIntTypes[] = {Type::UINT8, Type::INT8, Type::UINT16, Type::INT16, Type::UINT32, Type::INT32, Type::UINT64, Type::INT64};

// bit_wise_and / or / xor (arithmetic.go:944-961, GetBitwiseBinaryKernels scalar_arithmetic.go:245-255): integer types,
// every slot; validity by intersection
std::shared_ptr<ScalarFunction> MakeBitwiseBinary(const std::string& name, int8_t op) {
  auto fn = std::make_shared<ScalarFunction>(name, 2);
  fn->promote_numeric = true;
  for (Type t : kIntTypes) {
    exec::ScalarKernel k;
    k.in_types = {t, t};
    k.out_type = FirstType;
    k.exec = ArithBinaryExec(op);
    k.exec_batch = ArithBinaryBatchExec(op);
    k.expr_op = PlainExprOp(op);
    fn->AddKernel(std::move(k));
  }
  return fn;
}

// shift_left / shift_right (+ _unchecked) (arithmetic.go:970-996, GetShiftKernels scalar_arithmetic.go:401-412)
std::shared_ptr<ScalarFunction> MakeShift(const std::string& name, int8_t op, bool checked) {
  auto fn = std::make_shared<ScalarFunction>(name, 2);
  fn->promote_numeric = true;
  for (Type t : kIntTypes) {
    exec::ScalarKernel k;
    k.in_types = {t, t};
    k.out_type = FirstType;
    k.exec = ArithCheckedExec(op);
    k.expr_op = CheckedExprOp(op);
    k.can_fail = true;   // error word always supplied; only the checked ops raise it
    k.fail_message = "shift amount must be >= 0 and less than precision of type";
    fn->AddKernel(std::move(k));
  }
  return fn;
}

std::shared_ptr<ScalarFunction> MakeArithUnary(const std::string& name, int8_t op) {
  auto fn = std::make_shared<ScalarFunction>(name, 1);
  for (Type t : kNumericTypes) {
    exec::ScalarKernel k;
    k.in_types = {t};
    k.out_type = FirstType;
    k.exec = ArithUnaryExec(op);
    k.expr_op = PlainExprOp(op);
    fn->AddKernel(std::move(k));
  }
  return fn;
}

std::shared_ptr<ScalarFunction> MakeArithUnaryChecked(const std::string& name, int8_t op, bool signed_only) {
  auto fn = std::make_shared<ScalarFunction>(name, 1);
  for (Type t : kNumericTypes) {
    if (signed_only && !IsSignedInteger(t) && !IsFloating(t)) continue;  // GetArithmeticUnarySignedKernels, arithmetic.go:839-840
    exec::ScalarKernel k;
    k.in_types = {t};
    k.out_type = FirstType;
    if (IsSignedInteger(t)) { k.exec = ArithUnaryCheckedExec(op); k.expr_op = CheckedExprOp(op); k.can_fail = true; k.fail_message = "overflow"; }
    else { k.exec = ArithUnaryExec(op); k.expr_op = PlainExprOp(op); }
    fn->AddKernel(std::move(k));
  }
  return fn;
}

std::shared_ptr<ScalarFunction> MakeCompare(const std::string& name, int cmp) {  // CompareKernels, scalar_comparisons.go:654-716
  auto fn = std::make_shared<ScalarFunction>(name, 2);
  fn->promote_numeric = true;  // compareFunction.DispatchBest, scalar_compare.go:37-65
  for (Type t : kNumericTypes) {
    exec::ScalarKernel k;
    k.in_types = {t, t};
    k.out_type = BoolType;
    k.exec = CompareExec(cmp);
    k.expr_op = AG_EXPR_EQ + cmp;   // AG_CMP_EQ .. AG_CMP_LE in the order of AG_EXPR_EQ .. AG_EXPR_LE
    fn->AddKernel(std::move(k));
  }
  return fn;
}

std::shared_ptr<ScalarFunction> MakeBool(const std::string& name, exec::ArrayKernelExec ex, exec::NullHandling nh, int expr_op) {  // scalar_bool.go:123-140
  auto fn = std::make_shared<ScalarFunction>(name, 2);
  exec::ScalarKernel k;
  k.in_types = {Type::BOOL, Type::BOOL};
  k.out_type = BoolType;
  k.exec = std::move(ex);
  k.expr_op = expr_op;
  k.null_handling = nh;
  fn->AddKernel(std::move(k));
  return fn;
}

Status ConcatenateChunks(const ChunkedArray& c, std::shared_ptr<ArrayData>* out);
Status TakeRecordOrTable(const TakeOptions& opts, const Datum& values, const Datum& indices, Datum* out);

}  // namespace

// GetFunctionRegistry (registry.go:47-62): the functions of the hot path under their reference names
FunctionRegistry* GetFunctionRegistry() {
  static FunctionRegistry* reg = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    reg = new FunctionRegistry();
    // arithmetic.go:635-636,679-682,782-785: add / sub / multiply (+ "subtract" alias) and _unchecked
    reg->AddFunction(MakeArithBinary("add", AG_OP_ADD, AG_OP_ADD_CHECKED, true, "overflow"), false);
    reg->AddFunction(MakeArithBinary("add_unchecked", AG_OP_ADD, AG_OP_ADD_CHECKED, false, ""), false);
    reg->AddFunction(MakeArithBinary("sub", AG_OP_SUB, AG_OP_SUB_CHECKED, true, "overflow"), false);
    reg->AddFunction(MakeArithBinary("sub_unchecked", AG_OP_SUB, AG_OP_SUB_CHECKED, false, ""), false);
    reg->AddAlias("subtract", "sub");
    reg->AddAlias("subtract_unchecked", "sub_unchecked");
    reg->AddFunction(MakeArithBinary("multiply", AG_OP_MUL, AG_OP_MUL_CHECKED, true, "overflow"), false);
    reg->AddFunction(MakeArithBinary("multiply_unchecked", AG_OP_MUL, AG_OP_MUL_CHECKED, false, ""), false);
    reg->AddFunction(MakeArithUnary("abs_unchecked", AG_OP_ABS), false);
    reg->AddFunction(MakeArithUnary("negate_unchecked", AG_OP_NEGATE), false);
    reg->AddFunction(MakeArithUnary("sign", AG_OP_SIGN), false);
    reg->AddFunction(MakeArithUnaryChecked("abs", AG_OP_ABS_CHECKED, false), false);       // arithmetic.go:822-823
    reg->AddFunction(MakeArithUnaryChecked("negate", AG_OP_NEGATE_CHECKED, true), false);  // arithmetic.go:839-846
    reg->AddFunction(MakeDivide("divide", true), false);                                   // arithmetic.go:784-785
    reg->AddFunction(MakeDivide("divide_unchecked", false), false);
    reg->AddFunction(MakeBitwiseBinary("bit_wise_and", AG_OP_BIT_AND), false);             // arithmetic.go:949-951
    reg->AddFunction(MakeBitwiseBinary("bit_wise_or", AG_OP_BIT_OR), false);
    reg->AddFunction(MakeBitwiseBinary("bit_wise_xor", AG_OP_BIT_XOR), false);
    {
      auto fn = std::make_shared<ScalarFunction>("bit_wise_not", 1);                       // arithmetic.go:965-972
      for (Type t : kIntTypes) {
        exec::ScalarKernel k;
        k.in_types = {t};
        k.out_type = FirstType;
        k.exec = ArithUnaryExec(AG_OP_BIT_NOT);
        k.expr_op = PlainExprOp(AG_OP_BIT_NOT);
        fn->AddKernel(std::move(k));
      }
      reg->AddFunction(fn, false);
    }
    reg->AddFunction(MakeShift("shift_left", AG_OP_SHIFT_LEFT_CHECKED, true), false);      // arithmetic.go:980-983
    reg->AddFunction(MakeShift("shift_left_unchecked", AG_OP_SHIFT_LEFT, false), false);
    reg->AddFunction(MakeShift("shift_right", AG_OP_SHIFT_RIGHT_CHECKED, true), false);
    reg->AddFunction(MakeShift("shift_right_unchecked", AG_OP_SHIFT_RIGHT, false), false);
    // scalar_compare.go:102-153
    reg->AddFunction(MakeCompare("equal", AG_CMP_EQ), false);
    reg->AddFunction(MakeCompare("not_equal", AG_CMP_NE), false);
    reg->AddFunction(MakeCompare("greater", AG_CMP_GT), false);
    reg->AddFunction(MakeCompare("greater_equal", AG_CMP_GE), false);
    reg->AddFunction(MakeCompare("less", AG_CMP_LT), false);
    reg->AddFunction(MakeCompare("less_equal", AG_CMP_LE), false);
    // scalar_bool.go:123-140
    reg->AddFunction(MakeBool("and", BoolBinaryExec(AG_BITOP_AND), exec::NullHandling::INTERSECTION, AG_EXPR_AND), false);
    reg->AddFunction(MakeBool("or", BoolBinaryExec(AG_BITOP_OR), exec::NullHandling::INTERSECTION, AG_EXPR_OR), false);
    reg->AddFunction(MakeBool("xor", BoolBinaryExec(AG_BITOP_XOR), exec::NullHandling::INTERSECTION, AG_EXPR_XOR), false);
    reg->AddFunction(MakeBool("and_not", BoolBinaryExec(AG_BITOP_ANDNOT), exec::NullHandling::INTERSECTION, AG_EXPR_AND_NOT), false);
    reg->AddFunction(MakeBool("and_kleene", KleeneExec(AG_KLEENE_AND, AG_BITOP_AND), exec::NullHandling::COMPUTED_PREALLOC, AG_EXPR_KLEENE_AND), false);
    reg->AddFunction(MakeBool("or_kleene", KleeneExec(AG_KLEENE_OR, AG_BITOP_OR), exec::NullHandling::COMPUTED_PREALLOC, AG_EXPR_KLEENE_OR), false);
    reg->AddFunction(MakeBool("and_not_kleene", KleeneExec(AG_KLEENE_ANDNOT, AG_BITOP_ANDNOT), exec::NullHandling::COMPUTED_PREALLOC, AG_EXPR_KLEENE_AND_NOT), false);
    {
      auto fn = std::make_shared<ScalarFunction>("not", 1);
      exec::ScalarKernel k;
      k.in_types = {Type::BOOL};
      k.out_type = BoolType;
      k.exec = NotExec;
      k.expr_op = AG_EXPR_NOT;
      k.null_handling = exec::NullHandling::COMPUTED_NO_PREALLOC;
      k.can_write_into_slices = false;
      fn->AddKernel(std::move(k));
      reg->AddFunction(fn, false);
    }
    // scalar_compare.go / scalar_comparisons.go:718-813: is_null, is_not_null, is_nan
    for (auto& spec : std::vector<std::pair<const char*, exec::ArrayKernelExec>>{{"is_null", IsNullExec}, {"is_not_null", IsNotNullExec}}) {
      const int expr_op = spec.first == std::string("is_null") ? AG_EXPR_IS_NULL : AG_EXPR_IS_NOT_NULL;
      auto fn = std::make_shared<ScalarFunction>(spec.first, 1);
      exec::ScalarKernel k;
      k.any_input_type = true;
      k.out_type = BoolType;
      k.exec = spec.second;
      k.expr_op = expr_op;
      k.null_handling = exec::NullHandling::COMPUTED_NO_PREALLOC;
      k.mem_alloc = exec::MemAlloc::NO_PREALLOC;
      k.can_write_into_slices = false;
      fn->AddKernel(std::move(k));
      reg->AddFunction(fn, false);
    }
    {
      auto fn = std::make_shared<ScalarFunction>("is_nan", 1);
      for (Type t : kNumericTypes) {
        exec::ScalarKernel k;
        k.in_types = {t};
        k.out_type = BoolType;
        k.exec = IsNanExec;
        k.expr_op = AG_EXPR_IS_NAN;
        k.null_handling = exec::NullHandling::OUTPUT_NOT_NULL;
        fn->AddKernel(std::move(k));
      }
      reg->AddFunction(fn, false);
    }
    // cast.go:45-81,841-880: cast_<type> scalar functions for the numeric types + the "cast" meta function
    for (Type t : kNumericTypes) reg->AddFunction(MakeCastTo(t), false);
    reg->AddFunction(std::make_shared<MetaFunction>("cast", 1, [](const ExecCtx& ctx, const FunctionOptions* fo, const std::vector<Datum>& args, Datum* out) -> Status {
      const auto* co = dynamic_cast<const CastOptions*>(fo);
      if (!co || co->ToType == Type::NA) return Status::Invalid("cast requires that options be passed with a ToType");
      if (args.size() != 1 || args[0].kind == DatumKind::NONE) return Status::Invalid("cast takes one value argument");
      if (args[0].type() == co->ToType) { *out = args[0]; return Status::OK(); }
      const char* fname = CastFunctionName(co->ToType);
      FunctionRegistry* r = ctx.Registry ? ctx.Registry : GetFunctionRegistry();
      const Function* fn = fname ? r->GetFunction(fname) : nullptr;
      if (!fn) return Status::NotImplemented(std::string("unsupported cast to ") + TypeName(co->ToType) + " from " + TypeName(args[0].type()));
      if (args[0].kind != DatumKind::SCALAR) return fn->Execute(ctx, fo, args, out);
      // scalar input: a one-element array through the same kernel (the reference promotes scalars to
      // length-1 arrays for scalar-only execution too, executor.go PromoteExecSpanScalars)
      const Scalar& sc = *args[0].scalar;
      auto res = std::make_shared<Scalar>();
      res->type = co->ToType;
      if (!sc.valid) { *out = Datum(res); return Status::OK(); }
      std::shared_ptr<ArrayData> one;
      RETURN_NOT_OK(ArrayData::FromHost(sc.type, 1, 0, nullptr, sc.value, 0, &one));
      Datum casted;
      RETURN_NOT_OK(fn->Execute(ctx, fo, {Datum(one)}, &casted));
      RETURN_NOT_OK(casted.array->ToHost(res->value, nullptr, nullptr));
      res->valid = true;
      *out = Datum(res);
      return Status::OK();
    }), false);
    // vector_sort.go:383-390, vector_hash.go, scalar_set_lookup.go: registry names bound to the GPU kernels
    reg->AddFunction(std::make_shared<MetaFunction>("sort_indices", 1, [](const ExecCtx& ctx, const FunctionOptions* fo, const std::vector<Datum>& args, Datum* out) -> Status {
      const auto* so = dynamic_cast<const SortOptions*>(fo);
      if (args.size() != 1) return Status::Invalid("sort_indices takes one argument");
      if (const auto* sk = dynamic_cast<const SortKeys*>(fo)) return SortIndices(ctx, args[0], *sk, out);
      if (args[0].kind == DatumKind::RECORD || args[0].kind == DatumKind::TABLE)
        return Status::Invalid("sort_indices: record batches and tables are sorted with SortKeys options");
      return SortIndices(ctx, args[0], so ? *so : SortOptions(), out);
    }), false);
    reg->AddFunction(std::make_shared<MetaFunction>("unique", 1, [](const ExecCtx& ctx, const FunctionOptions*, const std::vector<Datum>& args, Datum* out) -> Status {
      if (args.size() != 1) return Status::Invalid("unique takes one argument");
      return Unique(ctx, args[0], out);
    }), false);
    reg->AddFunction(std::make_shared<MetaFunction>("dictionary_encode", 1, [](const ExecCtx& ctx, const FunctionOptions* fo, const std::vector<Datum>& args, Datum* out) -> Status {
      const auto* o = dynamic_cast<const DictionaryEncodeOptions*>(fo);
      if (fo && !o) return Status::Invalid(std::string("dictionary_encode: expected DictionaryEncodeOptions, got ") + fo->TypeName());
      if (args.size() != 1) return Status::Invalid("dictionary_encode takes one argument");
      return DictionaryEncode(ctx, o ? *o : DictionaryEncodeOptions(), args[0], out);
    }), false);
    // vector_run_ends.go:46-61: chunkwise, so runs never cross a chunk boundary
    reg->AddFunction(std::make_shared<MetaFunction>("run_end_encode", 1, [](const ExecCtx& ctx, const FunctionOptions* fo, const std::vector<Datum>& args, Datum* out) -> Status {
      if (!fo) return Status::Invalid("function 'run_end_encode' cannot be called without options");   // functions.go:163-167
      const auto* o = dynamic_cast<const RunEndEncodeOptions*>(fo);
      if (!o) return Status::Invalid(std::string("run_end_encode: expected RunEndEncodeOptions, got ") + fo->TypeName());
      if (args.size() != 1) return Status::Invalid("run_end_encode takes one argument");
      return RunEndEncode(ctx, *o, args[0], out);
    }), false);
    reg->AddFunction(std::make_shared<MetaFunction>("run_end_decode", 1, [](const ExecCtx& ctx, const FunctionOptions*, const std::vector<Datum>& args, Datum* out) -> Status {
      if (args.size() != 1) return Status::Invalid("run_end_decode takes one argument");
      return RunEndDecode(ctx, args[0], out);
    }), false);
    reg->AddFunction(std::make_shared<MetaFunction>("is_in", 1, [](const ExecCtx& ctx, const FunctionOptions* fo, const std::vector<Datum>& args, Datum* out) -> Status {
      const auto* so = dynamic_cast<const SetLookupOptions*>(fo);
      if (!so) return Status::Invalid("is_in requires SetLookupOptions");
      if (args.size() != 1) return Status::Invalid("is_in takes one argument");
      return IsIn(ctx, *so, args[0], out);
    }), false);
    // vector_cumulative.go:75-93
    reg->AddFunction(MakeCumulative("cumulative_sum", false), false);
    reg->AddFunction(MakeCumulative("cumulative_sum_checked", true), false);
    // selection.go:593-650: array_filter / array_take vector functions + filter / take meta functions
    {
      auto fn = std::make_shared<VectorFunction>("array_filter", 2);
      exec::VectorKernel k;
      k.any_input_type = true;
      k.out_type = FirstType;
      k.exec = PrimitiveFilterExec;
      k.null_handling = exec::NullHandling::COMPUTED_NO_PREALLOC;
      k.mem_alloc = exec::MemAlloc::NO_PREALLOC;
      k.can_execute_chunkwise = true;
      fn->AddKernel(std::move(k));
      reg->AddFunction(fn, false);
    }
    {
      auto fn = std::make_shared<VectorFunction>("array_take", 2);
      exec::VectorKernel k;
      k.any_input_type = true;
      k.out_type = FirstType;
      k.exec = PrimitiveTakeExec;
      k.null_handling = exec::NullHandling::COMPUTED_NO_PREALLOC;
      k.mem_alloc = exec::MemAlloc::NO_PREALLOC;
      k.can_execute_chunkwise = false;  // selection.go:639
      fn->AddKernel(std::move(k));
      reg->AddFunction(fn, false);
    }
    reg->AddFunction(std::make_shared<MetaFunction>("filter", 2, [](const ExecCtx& ctx, const FunctionOptions* opts, const std::vector<Datum>& args, Datum* out) -> Status {
      // filterMetaFunc, selection.go:41-85
      if (args.size() != 2) return Status::Invalid("filter takes 2 arguments");
      if (args[1].kind != DatumKind::ARRAY && args[1].kind != DatumKind::CHUNKED) return Status::NotImplemented("filter should be array-like");
      if (args[1].type() != Type::BOOL) return Status::NotImplemented("filter argument must be boolean type");
      return CallFunction(ctx, "array_filter", opts, args, out);
    }), false);
    reg->AddFunction(std::make_shared<MetaFunction>("take", 2, [](const ExecCtx& ctx, const FunctionOptions* opts, const std::vector<Datum>& args, Datum* out) -> Status {
      // takeMetaFunc, selection.go:93-114 -> takeArrayImpl :206-244 / takeChunkedImpl :246-300
      if (args.size() != 2) return Status::Invalid("take takes 2 arguments");
      if (args[1].kind != DatumKind::ARRAY && args[1].kind != DatumKind::CHUNKED) return Status::NotImplemented("unsupported types for take operation");
      if (args[0].kind == DatumKind::RECORD || args[0].kind == DatumKind::TABLE)   // takeRecordImpl / takeTableImpl
        return TakeRecordOrTable(dynamic_cast<const TakeOptions*>(opts) ? *dynamic_cast<const TakeOptions*>(opts) : TakeOptions(), args[0], args[1], out);
      Datum values = args[0];
      const bool values_chunked = values.kind == DatumKind::CHUNKED;
      if (values_chunked) {  // ChunkedPrimitiveTake resolves chunks per index; on the device we gather from one table
        std::shared_ptr<ArrayData> cat;
        RETURN_NOT_OK(ConcatenateChunks(*values.chunked, &cat));
        values = Datum(cat);
      } else if (values.kind != DatumKind::ARRAY) {
        return Status::NotImplemented("unsupported types for take operation");
      }
      if (args[1].kind == DatumKind::ARRAY) {
        Datum r;
        RETURN_NOT_OK(CallFunction(ctx, "array_take", opts, {values, args[1]}, &r));
        *out = values_chunked ? Datum(MakeChunked(r.array->type, {r.array})) : r;
        return Status::OK();
      }
      std::vector<std::shared_ptr<ArrayData>> chunks;
      for (auto& chunk : args[1].chunked->chunks) {  // one array_take per index chunk (selection.go:221-234)
        Datum r;
        RETURN_NOT_OK(CallFunction(ctx, "array_take", opts, {values, Datum(chunk)}, &r));
        chunks.push_back(r.array);
      }
      *out = Datum(MakeChunked(values.type(), std::move(chunks)));
      return Status::OK();
    }), false);
  });
  return reg;
}

namespace {
Status ConcatenateChunks(const ChunkedArray& c, std::shared_ptr<ArrayData>* out) {  // array.Concatenate on device (D2D)
  auto d = std::make_shared<ArrayData>();
  d->type = c.type; d->length = c.length; d->offset = 0;
  const int w = BitWidth(c.type) / 8;
  if (w == 0) return Status::NotImplemented("concatenate of boolean chunks");
  RETURN_NOT_OK(Buffer::Allocate(c.length * w, &d->buffers[1]));
  const bool any_nulls = MayHaveNulls(c.chunks);
  if (any_nulls) RETURN_NOT_OK(Buffer::Allocate((c.length + 7) / 8, &d->buffers[0]));
  int64_t pos = 0;
  for (auto& ch : c.chunks) {
    NATIVE(ag_copy_dev(d->buffers[1]->data() + pos * w, ch->buffers[1]->data() + ch->offset * w, (size_t)(ch->length * w), nullptr));
    if (any_nulls) {
      if (MayHaveNulls(*ch)) NATIVE(ag_bitmap_copy_dev(ch->buffers[0]->data(), ch->offset, ch->length, d->buffers[0]->data(), pos, nullptr));
      else NATIVE(ag_bitmap_set_dev(d->buffers[0]->data(), pos, ch->length, 1, nullptr));
    }
    pos += ch->length;
  }
  d->null_count = any_nulls ? kUnknownNullCount : 0;
  *out = d;
  return Status::OK();
}
}  // namespace

// arithmetic.go:1090-1142
static Status CumulativeImpl(const ExecCtx& ctx, const char* fn, const CumulativeOptions& opts, const Datum& values, Datum* out) {
  if (values.kind == DatumKind::SCALAR) {  // the vector executor promotes a scalar argument to a length-1 array
    if (!values.scalar) return Status::Invalid("cumulative sum: empty datum");
    std::shared_ptr<ArrayData> one;
    const uint8_t zero = 0;
    RETURN_NOT_OK(ArrayData::FromHost(values.scalar->type, 1, 0, values.scalar->valid ? nullptr : &zero, values.scalar->value,
                                      values.scalar->valid ? 0 : 1, &one));
    return CallFunction(ctx, fn, &opts, {Datum(one)}, out);
  }
  return CallFunction(ctx, fn, &opts, {values}, out);
}
Status CumulativeSum(const ExecCtx& ctx, const CumulativeOptions& opts, const Datum& values, Datum* out) { return CumulativeImpl(ctx, "cumulative_sum", opts, values, out); }
Status CumulativeSumChecked(const ExecCtx& ctx, const CumulativeOptions& opts, const Datum& values, Datum* out) { return CumulativeImpl(ctx, "cumulative_sum_checked", opts, values, out); }

Status CastDatum(const ExecCtx& ctx, const Datum& val, const CastOptions& opts, Datum* out) {  // cast.go:919-921
  return CallFunction(ctx, "cast", &opts, {val}, out);
}

static Status ArithImpl(const ExecCtx& ctx, const ArithmeticOptions& opts, const char* fn, const Datum& l, const Datum& r, Datum* out) {
  std::string name = fn;
  if (opts.NoCheckOverflow) name += "_unchecked";
  return CallFunction(ctx, name, nullptr, {l, r}, out);
}
Status Add(const ExecCtx& ctx, const ArithmeticOptions& o, const Datum& l, const Datum& r, Datum* out) { return ArithImpl(ctx, o, "add", l, r, out); }
Status Subtract(const ExecCtx& ctx, const ArithmeticOptions& o, const Datum& l, const Datum& r, Datum* out) { return ArithImpl(ctx, o, "sub", l, r, out); }
Status Multiply(const ExecCtx& ctx, const ArithmeticOptions& o, const Datum& l, const Datum& r, Datum* out) { return ArithImpl(ctx, o, "multiply", l, r, out); }
// ---- sort_indices / unique / is_in (SURVEY 8f rank 3): single fixed-width column, anything else is ErrNotImplemented
// like the reference's type switches (vector_sort.go:183-185, scalar_set_lookup.go:270-272) ------------------------
static Status OneArray(const Datum& d, const char* fn, std::shared_ptr<ArrayData>* out) {
  if (d.kind == DatumKind::ARRAY) { *out = d.array; return Status::OK(); }
  if (d.kind == DatumKind::CHUNKED && d.chunked->chunks.size() == 1) { *out = d.chunked->chunks[0]; return Status::OK(); }
  return Status::NotImplemented(std::string(fn) + ": the GPU kernel takes one array (a multi-chunk input is merged by the parent registry's function)");
}
static Status MakeOut(Type t, int64_t len, std::shared_ptr<Buffer> data, std::shared_ptr<Buffer> valid, int64_t nulls, Datum* out) {
  auto a = std::make_shared<ArrayData>();
  a->type = t; a->length = len; a->offset = 0; a->null_count = nulls;
  a->buffers[0] = valid; a->buffers[1] = data;
  *out = Datum(a);
  return Status::OK();
}

Status SortIndices(const ExecCtx& ctx, const Datum& input, const SortOptions& opts, Datum* out) {
  std::shared_ptr<ArrayData> a;
  RETURN_NOT_OK(OneArray(input, "sort_indices", &a));
  if (!IsInteger(a->type) && !IsFloating(a->type)) return Status::NotImplemented(std::string("unsupported type for sort_indices operation: ") + TypeName(a->type));
  std::shared_ptr<Buffer> idx;
  RETURN_NOT_OK(Buffer::Allocate(std::max<int64_t>(a->length, 1) * 8, &idx));
  int64_t nulls = 0, nans = 0;
  NATIVE(ag_sort_indices_dev((int)a->type, a->buffers[1] ? a->buffers[1]->data() : nullptr, ValidityOrNull(*a), a->offset, a->length, (int)opts.Order, (int)opts.Placement,
                             (uint64_t*)idx->data(), &nulls, &nans, nullptr));
  return MakeOut(Type::UINT64, a->length, idx, nullptr, 0, out);
}

// sortIndicesImpl (vector_sort.go:117-200) + the column checks of kernels.SortIndices (internal/kernels/vector_sort.go:390-416):
// the key columns go to the device as chunk lists, whatever their chunking.
Status SortIndices(const ExecCtx& ctx, const Datum& input, const SortKeys& opts, Datum* out) {
  if (opts.Keys.empty()) return Status::Invalid("must provide at least one sort key");
  std::vector<Column> cols;   // one per key
  std::vector<SortKey> keys = opts.Keys;
  switch (input.kind) {
    case DatumKind::ARRAY:      // one column: the first key only, ColumnIndex ignored
    case DatumKind::CHUNKED:
      cols.push_back(Column{input.type(), ArrayChunks(input)});
      keys.resize(1);
      break;
    case DatumKind::RECORD:
    case DatumKind::TABLE: {
      const int ncols = NumColumns(input);
      for (size_t i = 0; i < keys.size(); ++i) {
        const int c = keys[i].ColumnIndex;
        if (c < 0 || c >= ncols) return Status::Invalid("sort key " + std::to_string(i) + " has invalid column index " + std::to_string(c));
        cols.push_back(GetColumn(input, c));
      }
      break;
    }
    default:
      return Status::NotImplemented("unsupported type for sort_indices operation");
  }
  const int64_t n = input.Len();
  for (auto& c : cols)
    if (c.type != Type::BOOL && !IsInteger(c.type) && !IsFloating(c.type))
      return Status::NotImplemented(std::string("sorting not supported for type ") + TypeName(c.type));
  std::vector<std::vector<ag_sort_chunk>> chunks(cols.size());
  std::vector<ag_sort_key> desc(cols.size());
  for (size_t i = 0; i < cols.size(); ++i) {
    chunks[i] = ChunkDescs(cols[i].chunks);
    desc[i] = ag_sort_key{(int)cols[i].type, (int)keys[i].Order, (int)keys[i].Placement, (int)chunks[i].size(), chunks[i].data()};
  }
  std::shared_ptr<Buffer> idx;
  RETURN_NOT_OK(Buffer::Allocate(std::max<int64_t>(n, 1) * 8, &idx));
  NATIVE(ag_sort_indices_keys_dev((int)desc.size(), desc.data(), n, (uint64_t*)idx->data(), nullptr));
  return MakeOut(Type::UINT64, n, idx, nullptr, 0, out);
}

Status SortIndicesRecordBatch(const ExecCtx& ctx, const std::shared_ptr<RecordBatch>& batch, const std::vector<SortKey>& keys, Datum* out) {
  if (keys.empty()) return Status::Invalid("at least one sort key is required");
  SortKeys o; o.Keys = keys;
  return CallFunction(ctx, "sort_indices", &o, {Datum(batch)}, out);
}
Status SortIndicesTable(const ExecCtx& ctx, const std::shared_ptr<Table>& table, const std::vector<SortKey>& keys, Datum* out) {
  if (keys.empty()) return Status::Invalid("at least one sort key is required");
  SortKeys o; o.Keys = keys;
  return CallFunction(ctx, "sort_indices", &o, {Datum(table)}, out);
}

// ---- take / filter / sort on record batches and tables ---------------------------------------------------------------
// Every column of a record batch or table is gathered by one ag_take_columns_dev launch per index chunk (per filter span
// for FilterTable), never one launch per column.  Arrays and chunked arrays keep the "take" meta function's own path.
namespace {
bool SelectionType(Type t) { return t == Type::BOOL || IsNumeric(t); }

// The columns of a record batch or table; ErrNotImplemented for the first one of a type the gather does not take.
Status SelColumns(const Datum& values, std::vector<Column>* cols) {
  for (int i = 0; i < NumColumns(values); ++i) {
    cols->push_back(GetColumn(values, i));
    if (!SelectionType(cols->back().type))
      return Status::NotImplemented("take: column " + std::to_string(i) + " has unsupported type " + TypeName(cols->back().type) +
                                    " (boolean and numeric columns only)");
  }
  return Status::OK();
}

// One ag_take_columns_dev launch: rows [0, idx.length) of `idx` from every column, read from `chunks[c]` (their lengths
// sum to nrows), into a new output per column appended to (*res)[c].  An output has a validity bitmap when
// `idx_nullable` or a chunk it reads may have nulls.  `d_bad`: the error word of a bounds-checked gather, reset here;
// nullptr for no bounds check.
Status GatherColumns(const std::vector<Column>& cols, const std::vector<std::vector<ag_sort_chunk>>& chunks, int64_t nrows, const ArrayData& idx,
                     bool idx_nullable, int64_t* d_bad, std::vector<std::vector<std::shared_ptr<ArrayData>>>* res) {
  std::vector<ag_take_column> desc(cols.size());
  for (size_t c = 0; c < cols.size(); ++c) {
    bool nullable = idx_nullable;
    for (auto& ch : chunks[c]) nullable = nullable || ch.valid != nullptr;
    std::shared_ptr<ArrayData> o;
    RETURN_NOT_OK(AllocateOutput(cols[c].type, idx.length, nullable, &o));
    (*res)[c].push_back(o);
    desc[c] = ag_take_column{(int)cols[c].type, (int)chunks[c].size(), chunks[c].data(), o->buffers[1]->data(), o->buffers[0] ? o->buffers[0]->data() : nullptr};
  }
  if (d_bad) NATIVE(ag_error_word_reset_dev(d_bad, nullptr));
  const int iw = BitWidth(idx.type);
  const void* iptr = idx.buffers[1] ? idx.buffers[1]->data() + idx.offset * (iw / 8) : nullptr;
  NATIVE(ag_take_columns_dev((int)desc.size(), desc.data(), nrows, iw, IsSignedInteger(idx.type), iptr, ValidityOrNull(idx), idx.offset, idx.length,
                             d_bad ? 1 : 0, d_bad, nullptr));
  return Status::OK();
}

// The record batch (`kind` RECORD: the one output of each column) or table (each column's outputs as its chunks) of
// `num_rows` rows that GatherColumns filled `res` for.
Status MakeSelection(DatumKind kind, const std::vector<Column>& cols, const std::vector<std::vector<std::shared_ptr<ArrayData>>>& res, int64_t num_rows,
                     Datum* out) {
  if (kind == DatumKind::RECORD) {
    std::vector<std::shared_ptr<ArrayData>> arrs;
    for (auto& r : res) arrs.push_back(r[0]);
    std::shared_ptr<RecordBatch> rb;
    RETURN_NOT_OK(MakeRecordBatch(num_rows, std::move(arrs), &rb));
    *out = Datum(rb);
    return Status::OK();
  }
  std::vector<std::shared_ptr<ChunkedArray>> ccols;
  for (size_t c = 0; c < cols.size(); ++c) ccols.push_back(MakeChunked(cols[c].type, res[c]));
  std::shared_ptr<Table> tb;
  RETURN_NOT_OK(MakeTable(num_rows, std::move(ccols), &tb));
  *out = Datum(tb);
  return Status::OK();
}

// takeRecordImpl (selection.go:160-204) and takeTableImpl -> takeChunkedImpl -> ChunkedPrimitiveTake (:117-158, 246-300,
// kernels/vector_selection.go:1194-1228): a record batch takes by the concatenated indices and gives arrays of
// len(indices) rows; a table gives every column one chunk per index chunk (an array index: one chunk).
Status TakeRecordOrTable(const TakeOptions& opts, const Datum& values, const Datum& indices, Datum* out) {
  std::vector<Column> cols;
  RETURN_NOT_OK(SelColumns(values, &cols));
  const Type it = indices.type();
  if (!IsInteger(it)) return Status::Invalid("invalid index type for bounds checking");   // helpers.go:978
  std::vector<std::shared_ptr<ArrayData>> idx;
  if (indices.kind == DatumKind::CHUNKED && values.kind == DatumKind::RECORD) {   // chunked indices are concatenated first (:163-171)
    std::shared_ptr<ArrayData> cat;
    RETURN_NOT_OK(ConcatenateChunks(*indices.chunked, &cat));
    idx.push_back(cat);
  } else {
    idx = ArrayChunks(indices);
  }
  std::vector<std::vector<ag_sort_chunk>> chunks(cols.size());
  for (size_t c = 0; c < cols.size(); ++c) chunks[c] = ChunkDescs(cols[c].chunks);
  const bool idx_nullable = MayHaveNulls(idx);
  std::shared_ptr<Buffer> words;
  RETURN_NOT_OK(Buffer::Allocate(8 * std::max<int64_t>((int64_t)idx.size(), 1), &words));
  int64_t* d_bad = (int64_t*)words->data();
  std::vector<std::vector<std::shared_ptr<ArrayData>>> res(cols.size());
  // the reference takes column by column, so without columns nothing is gathered or bounds-checked
  const size_t launches = cols.empty() ? 0 : idx.size();
  for (size_t k = 0; k < launches; ++k)
    RETURN_NOT_OK(GatherColumns(cols, chunks, values.Len(), *idx[k], idx_nullable, opts.BoundsCheck ? d_bad + k : nullptr, &res));
  if (opts.BoundsCheck && launches > 0) {   // checkIndexBoundsChunked: the first offending row in index order
    std::vector<int64_t> bad(launches);
    RETURN_NOT_OK(words->ToHost(bad.data(), 8 * (int64_t)launches));
    for (size_t k = 0; k < launches; ++k)
      if (bad[k] != AG_NO_ERROR_POS) return IndexOutOfBounds(*idx[k]->buffers[1], idx[k]->type, idx[k]->offset, bad[k]);
  }
  int64_t out_rows = 0;
  for (auto& a : idx) out_rows += a->length;
  // array.NewTable(schema, cols, -1): a table without columns has no rows
  return MakeSelection(values.kind, cols, res, values.kind == DatumKind::TABLE && cols.empty() ? 0 : out_rows, out);
}

// GetTakeIndices (kernels/vector_selection.go:102-236) of each mask span, with one read-back for all their lengths:
// uint32 row indices relative to the span, validity only when EmitNulls meets a null mask slot.
Status MaskSpansToIndices(const std::vector<std::shared_ptr<ArrayData>>& masks, NullSelectionBehavior sel, std::vector<std::shared_ptr<ArrayData>>* out) {
  const size_t ns = masks.size();
  std::shared_ptr<Buffer> lens;
  RETURN_NOT_OK(Buffer::Allocate(16 * std::max<int64_t>((int64_t)ns, 1), &lens));
  int64_t* d_len = (int64_t*)lens->data();
  for (size_t k = 0; k < ns; ++k) {
    const ArrayData& m = *masks[k];
    if (m.length > (int64_t)UINT32_MAX) return Status::NotImplemented("filter: more than 2^32-1 rows in one chunk");
    NATIVE(ag_filter_output_size_dev(m.buffers[1]->data(), ValidityOrNull(m), m.offset, m.length, (int)sel,
                                     d_len + 2 * k, nullptr));
  }
  std::vector<int64_t> h(2 * std::max<size_t>(ns, 1));
  RETURN_NOT_OK(lens->ToHost(h.data(), 16 * (int64_t)ns));
  for (size_t k = 0; k < ns; ++k) {
    const ArrayData& m = *masks[k];
    const int64_t len = h[2 * k];
    const bool nullable = sel == EmitNulls && MayHaveNulls(m);
    std::shared_ptr<ArrayData> d;
    RETURN_NOT_OK(AllocateOutput(Type::UINT32, len, nullable, &d));
    if (len > 0)
      NATIVE(ag_take_indices_dev(32, m.buffers[1]->data(), ValidityOrNull(m), m.offset, m.length, (int)sel,
                                 d->buffers[1]->data(), nullable ? d->buffers[0]->data() : nullptr, len, d_len + 2 * k + 1, nullptr));
    out->push_back(d);
  }
  return Status::OK();
}
}  // namespace

// FilterRecordBatch (selection.go:679-722): the mask becomes indices once, every column is gathered without a bounds check
Status FilterRecordBatch(const ExecCtx& ctx, const std::shared_ptr<RecordBatch>& batch, const std::shared_ptr<ArrayData>& filter,
                         const FilterOptions& opts, std::shared_ptr<RecordBatch>* out) {
  if (!filter || batch->num_rows != filter->length) return Status::Invalid("filter inputs must all be the same length");
  if (filter->type != Type::BOOL) return Status::NotImplemented("filter argument must be boolean type");
  std::vector<std::shared_ptr<ArrayData>> idx;
  RETURN_NOT_OK(MaskSpansToIndices({filter}, opts.NullSelection, &idx));
  TakeOptions to; to.BoundsCheck = false;
  Datum r;
  RETURN_NOT_OK(TakeRecordOrTable(to, Datum(batch), Datum(idx[0]), &r));
  *out = r.record;
  return Status::OK();
}

// FilterTable (selection.go:724-800): columns and filter are cut at every chunk boundary of any of them (the walk of
// RechunkArraysConsistently, which IterateExecSpans does); each span's mask becomes indices once and all columns are
// gathered from that span in one launch.  A span that selects no row gives no chunk; a zero-row table comes back as it is.
Status FilterTable(const ExecCtx& ctx, const std::shared_ptr<Table>& table, const Datum& filter, const FilterOptions& opts, std::shared_ptr<Table>* out) {
  if (table->num_rows != filter.Len()) return Status::Invalid("filter inputs must all be the same length");
  if (table->num_rows == 0) { *out = table; return Status::OK(); }
  if (filter.kind != DatumKind::ARRAY && filter.kind != DatumKind::CHUNKED) return Status::NotImplemented("filter should be array-like");
  if (filter.type() != Type::BOOL) return Status::NotImplemented("filter argument must be boolean type");
  std::vector<Column> cols;
  RETURN_NOT_OK(SelColumns(Datum(table), &cols));
  const std::vector<std::shared_ptr<ArrayData>> fchunks = ArrayChunks(filter);
  std::vector<std::vector<std::shared_ptr<ArrayData>>> args;
  for (auto& c : cols) args.push_back(c.chunks);
  args.push_back(fchunks);
  std::vector<SpanPiece> pieces;
  RETURN_NOT_OK(ChunkSpans(args, std::vector<bool>(args.size(), true), INT64_MAX, &pieces));
  std::vector<std::shared_ptr<ArrayData>> masks;
  for (auto& p : pieces) masks.push_back(fchunks[p.chunk_index.back()]->Slice(p.chunk_pos.back(), p.len));
  std::vector<std::shared_ptr<ArrayData>> idx;
  RETURN_NOT_OK(MaskSpansToIndices(masks, opts.NullSelection, &idx));
  std::vector<std::vector<std::shared_ptr<ArrayData>>> res(cols.size());
  int64_t out_rows = 0;
  for (size_t k = 0; k < pieces.size(); ++k) {
    if (idx[k]->length == 0) continue;
    const SpanPiece& p = pieces[k];
    std::vector<std::vector<ag_sort_chunk>> chunks(cols.size());
    for (size_t c = 0; c < cols.size(); ++c) chunks[c] = {ChunkDesc(*cols[c].chunks[p.chunk_index[c]], p.chunk_pos[c], p.len)};
    RETURN_NOT_OK(GatherColumns(cols, chunks, p.len, *idx[k], MayHaveNulls(*idx[k]), nullptr, &res));
    out_rows += idx[k]->length;
  }
  Datum r;
  RETURN_NOT_OK(MakeSelection(DatumKind::TABLE, cols, res, out_rows, &r));
  *out = r.table;
  return Status::OK();
}

// compute.Sort (vector_sort.go:65-81): sort_indices by `keys`, then take with default TakeOptions.  A chunked array is
// taken as a one-column table (one gather over its chunks) and comes back as a one-chunk chunked array.
Status Sort(const ExecCtx& ctx, const Datum& input, const SortKeys& keys, Datum* out) {
  Datum idx;
  RETURN_NOT_OK(SortIndices(ctx, input, keys, &idx));
  if (input.kind != DatumKind::CHUNKED) return Take(ctx, TakeOptions(), input, idx, out);
  std::shared_ptr<Table> t;
  RETURN_NOT_OK(MakeTable(input.chunked->length, {input.chunked}, &t));
  Datum r;
  RETURN_NOT_OK(Take(ctx, TakeOptions(), Datum(t), idx, &r));
  *out = Datum(r.table->columns[0]);
  return Status::OK();
}

Status Unique(const ExecCtx& ctx, const Datum& values, Datum* out) {
  std::shared_ptr<ArrayData> a;
  RETURN_NOT_OK(OneArray(values, "unique", &a));
  const int bw = BitWidth(a->type);
  if (bw != 8 && bw != 16 && bw != 32 && bw != 64) return Status::NotImplemented(std::string("unique: unsupported type ") + TypeName(a->type));
  const bool has_valid = a->buffers[0] && a->null_count != 0;
  std::shared_ptr<Buffer> data, valid, len;
  RETURN_NOT_OK(Buffer::Allocate(std::max<int64_t>(a->length, 1) * (bw / 8), &data));
  if (has_valid) RETURN_NOT_OK(Buffer::Allocate(BitmapWordBytes(a->length) + 4, &valid));
  RETURN_NOT_OK(Buffer::Allocate(16, &len));
  NATIVE(ag_unique_dev(bw, a->buffers[1] ? a->buffers[1]->data() : nullptr, has_valid ? a->buffers[0]->data() : nullptr, a->offset, a->length, data->data(),
                       has_valid ? valid->data() : nullptr, a->length, (int64_t*)len->data(), nullptr));
  int64_t k = 0;
  RETURN_NOT_OK(len->ToHost(&k, 8));
  return MakeOut(a->type, k, data, valid, has_valid ? kUnknownNullCount : 0, out);
}

Status DictionaryEncode(const ExecCtx& ctx, const DictionaryEncodeOptions& opts, const Datum& values, Datum* out) {
  if (opts.NullEncoding != NullEncodingMask && opts.NullEncoding != NullEncodingEncode)
    return Status::Invalid("dictionary_encode: invalid NullEncodingBehavior " + std::to_string((int)opts.NullEncoding));
  if (values.type() == Type::DICTIONARY) { *out = values; return Status::OK(); }   // GetVectorHashKernels' identity kernel
  if (values.kind != DatumKind::ARRAY && values.kind != DatumKind::CHUNKED) return Status::NotImplemented("dictionary_encode takes an array-like argument");
  const Type t = values.type();
  const int bw = BitWidth(t);
  if (bw != 8 && bw != 16 && bw != 32 && bw != 64) return Status::NotImplemented(std::string("dictionary_encode: unsupported type ") + TypeName(t));
  const std::vector<std::shared_ptr<ArrayData>> in = ArrayChunks(values);
  const bool encode = opts.NullEncoding == NullEncodingEncode;
  int64_t total = 0;
  for (auto& a : in) total += a->length;
  if (total >= ((int64_t)1 << 31)) return Status::NotImplemented("dictionary_encode: more than 2^31-1 rows");
  bool any_valid = false;
  std::vector<ag_dict_chunk> desc(in.size());
  std::vector<std::shared_ptr<Buffer>> idx(in.size()), idx_valid(in.size());
  for (size_t c = 0; c < in.size(); ++c) {
    const ArrayData& a = *in[c];
    const bool has_valid = a.buffers[0] && a.null_count != 0;
    any_valid |= has_valid;
    RETURN_NOT_OK(Buffer::Allocate(std::max<int64_t>(a.length, 1) * 4, &idx[c]));
    if (has_valid && !encode) RETURN_NOT_OK(Buffer::Allocate(BitmapWordBytes(a.length), &idx_valid[c]));
    desc[c] = ag_dict_chunk{a.buffers[1] ? a.buffers[1]->data() : nullptr, has_valid ? a.buffers[0]->data() : nullptr, a.offset, a.length,
                            (int32_t*)idx[c]->data(), idx_valid[c] ? idx_valid[c]->data() : nullptr};
  }
  // the call's dictionary has room for every row; the result keeps a copy of its k values only
  std::shared_ptr<Buffer> scratch, scratch_valid, counts;
  RETURN_NOT_OK(Buffer::Allocate(std::max<int64_t>(total, 1) * (bw / 8), &scratch));
  if (encode && any_valid) RETURN_NOT_OK(Buffer::Allocate((total + 7) / 8, &scratch_valid));
  RETURN_NOT_OK(Buffer::Allocate(((int64_t)in.size() + 2) * 8, &counts));
  NATIVE(ag_dictionary_encode_dev(bw, desc.data(), (int64_t)desc.size(), (int)opts.NullEncoding, scratch->data(),
                                  scratch_valid ? scratch_valid->data() : nullptr, (int64_t*)counts->data(), nullptr));
  std::vector<int64_t> cnt(in.size() + 2);
  RETURN_NOT_OK(counts->ToHost(cnt.data(), (int64_t)cnt.size() * 8));
  auto dict = std::make_shared<ArrayData>();
  dict->type = t; dict->length = cnt[0]; dict->null_count = cnt[1];
  RETURN_NOT_OK(Buffer::Allocate(cnt[0] * (bw / 8), &dict->buffers[1]));
  NATIVE(ag_copy_dev(dict->buffers[1]->data(), scratch->data(), (size_t)(cnt[0] * (bw / 8)), nullptr));
  if (cnt[1] > 0) {
    RETURN_NOT_OK(Buffer::Allocate((cnt[0] + 7) / 8, &dict->buffers[0]));
    NATIVE(ag_copy_dev(dict->buffers[0]->data(), scratch_valid->data(), (size_t)((cnt[0] + 7) / 8), nullptr));
  }
  NATIVE(ag_stream_sync(nullptr));
  auto make = [&](size_t c) {
    auto d = std::make_shared<ArrayData>();
    d->type = Type::DICTIONARY; d->length = in[c]->length; d->null_count = cnt[2 + c];
    d->buffers[1] = idx[c];
    if (d->null_count > 0) d->buffers[0] = idx_valid[c];
    d->dictionary = dict;
    return d;
  };
  if (values.kind == DatumKind::ARRAY) { *out = Datum(make(0)); return Status::OK(); }
  std::vector<std::shared_ptr<ArrayData>> chunks;
  for (size_t c = 0; c < in.size(); ++c) if (in[c]->length > 0) chunks.push_back(make(c));   // WrapResults drops empty chunks
  auto res = MakeChunked(Type::DICTIONARY, std::move(chunks));
  res->value_type = t;
  *out = Datum(res);
  return Status::OK();
}

Status IsIn(const ExecCtx& ctx, const SetLookupOptions& opts, const Datum& values, Datum* out) {
  std::shared_ptr<ArrayData> a;
  RETURN_NOT_OK(OneArray(values, "is_in", &a));
  if (!opts.ValueSet) return Status::Invalid("is_in: SetLookupOptions.ValueSet is required");
  if (opts.ValueSet->type != a->type) return Status::NotImplemented("is_in: the value set must have the input's type (casts are left to the parent registry)");
  const int bw = BitWidth(a->type);
  if (bw != 8 && bw != 16 && bw != 32 && bw != 64) return Status::Invalid(std::string("unsupported type ") + TypeName(a->type) + " for is_in function");
  const ArrayData& s = *opts.ValueSet;
  std::shared_ptr<Buffer> data, valid, cnt;
  const int64_t bm = BitmapWordBytes(a->length) + 4;
  RETURN_NOT_OK(Buffer::Allocate(bm, &data));
  RETURN_NOT_OK(Buffer::Allocate(bm, &valid));
  RETURN_NOT_OK(Buffer::Allocate(8, &cnt));
  NATIVE(ag_is_in_dev(bw, a->buffers[1] ? a->buffers[1]->data() : nullptr, ValidityOrNull(*a), a->offset, a->length,
                      s.buffers[1] ? s.buffers[1]->data() : nullptr, ValidityOrNull(s), s.offset, s.length,
                      (int)opts.NullBehavior, data->data(), valid->data(), (int64_t*)cnt->data(), nullptr));
  int64_t nulls = 0;
  RETURN_NOT_OK(cnt->ToHost(&nulls, 8));
  return MakeOut(Type::BOOL, a->length, data, nulls ? valid : nullptr, nulls, out);
}

// ---- run_end_encode / run_end_decode ------------------------------------------------------------------------------
namespace {
// The arrays a chunkwise vector kernel runs on: the executor's spans of one argument (iterateExecSpans), so a chunked
// input loses its empty chunks and a chunked input without rows gives one empty span (nullptr when it has no chunks).
Status ChunkwiseSpans(const Datum& values, std::vector<std::shared_ptr<ArrayData>>* spans) {
  const std::vector<std::shared_ptr<ArrayData>> chunks = ArrayChunks(values);
  std::vector<SpanPiece> pieces;
  RETURN_NOT_OK(ChunkSpans({chunks}, {true}, INT64_MAX, &pieces));
  for (auto& p : pieces) spans->push_back(chunks[p.chunk_index[0]]->Slice(p.chunk_pos[0], p.len));
  if (pieces.empty()) spans->push_back(chunks.empty() ? nullptr : chunks[0]->Slice(0, 0));
  return Status::OK();
}
int64_t RunEndMax(Type t) { return t == Type::INT16 ? INT16_MAX : (t == Type::INT32 ? INT32_MAX : INT64_MAX); }
const void* ElementPtr(const ArrayData& a) { return a.buffers[1] ? a.buffers[1]->data() + a.offset * (BitWidth(a.type) / 8) : nullptr; }

// CountNumberOfRuns, one 16-byte read-back, exact allocation, WriteEncodedRuns (vector_run_end_encode.go:531-565)
Status EncodeOne(Type rt, const ArrayData& a, std::shared_ptr<ArrayData>* out) {
  const Type t = a.type;
  const bool has_valid = a.buffers[0] != nullptr;
  const uint8_t* valid = has_valid ? a.buffers[0]->data() : nullptr;
  const void* vals = a.buffers[1] ? a.buffers[1]->data() : nullptr;   // row 0 at a.offset, a bit offset for BOOL
  std::shared_ptr<Buffer> counts;
  RETURN_NOT_OK(Buffer::Allocate(16, &counts));
  NATIVE(ag_run_end_count_dev((int)t, vals, valid, a.offset, a.length, (int64_t*)counts->data(), nullptr));
  int64_t cnt[2] = {0, 0};
  RETURN_NOT_OK(counts->ToHost(cnt, 16));
  const int64_t runs = cnt[0];
  std::shared_ptr<ArrayData> re, v;
  RETURN_NOT_OK(AllocateOutput(rt, runs, false, &re));
  RETURN_NOT_OK(AllocateOutput(t, runs, has_valid, &v));
  v->null_count = has_valid ? cnt[1] : 0;
  NATIVE(ag_run_end_encode_dev((int)t, (int)rt, vals, valid, a.offset, a.length, re->buffers[1]->data(), v->buffers[1]->data(),
                               has_valid ? v->buffers[0]->data() : nullptr, runs, (int64_t*)counts->data(), nullptr));
  NATIVE(ag_stream_sync(nullptr));
  auto d = std::make_shared<ArrayData>();
  d->type = Type::RUN_END_ENCODED; d->length = a.length; d->null_count = 0;
  d->run_ends = re;
  d->values = v;
  *out = d;
  return Status::OK();
}

Status DecodeOne(const ArrayData& a, std::shared_ptr<ArrayData>* out) {
  const ArrayData &re = *a.run_ends, &v = *a.values;
  if (v.length < re.length) return Status::Invalid("run_end_decode: the values child is shorter than run_ends");
  const Type t = v.type;
  const bool has_valid = v.buffers[0] != nullptr;
  std::shared_ptr<ArrayData> d;
  RETURN_NOT_OK(AllocateOutput(t, a.length, has_valid, &d));
  std::shared_ptr<Buffer> words;   // [0] null count, [1] error word
  RETURN_NOT_OK(Buffer::Allocate(16, &words));
  int64_t* w = (int64_t*)words->data();
  NATIVE(ag_error_word_reset_dev(w + 1, nullptr));
  NATIVE(ag_run_end_decode_dev((int)t, (int)re.type, ElementPtr(re), re.length, v.buffers[1] ? v.buffers[1]->data() : nullptr,
                               has_valid ? v.buffers[0]->data() : nullptr, v.offset, a.offset, a.length, d->buffers[1]->data(),
                               has_valid ? d->buffers[0]->data() : nullptr, w, w + 1, nullptr));
  int64_t h[2];
  RETURN_NOT_OK(words->ToHost(h, 16));
  if (h[1] != AG_NO_ERROR_POS)
    return Status::Invalid("run_end_decode: malformed run ends at run " + std::to_string(h[1]) + " (they must increase strictly and reach offset+length)");
  d->null_count = has_valid ? h[0] : 0;
  *out = d;
  return Status::OK();
}

bool RunEndValueType(Type t) { return t == Type::BOOL || IsNumeric(t); }
}  // namespace

Status RunEndEncode(const ExecCtx& ctx, const RunEndEncodeOptions& opts, const Datum& values, Datum* out) {
  const Type rt = opts.RunEndType;
  if (rt != Type::INT16 && rt != Type::INT32 && rt != Type::INT64) return Status::Invalid(std::string("bad run end type ") + TypeName(rt));
  if (values.kind != DatumKind::ARRAY && values.kind != DatumKind::CHUNKED) return Status::NotImplemented("run_end_encode takes an array-like argument");
  const Type t = values.type();
  if (!RunEndValueType(t)) return Status::NotImplemented(std::string("run_end_encode: unsupported type ") + TypeName(t));
  std::vector<std::shared_ptr<ArrayData>> spans;
  RETURN_NOT_OK(ChunkwiseSpans(values, &spans));
  std::vector<std::shared_ptr<ArrayData>> res;
  for (auto a : spans) {
    if (!a) { a = std::make_shared<ArrayData>(); a->type = t; }   // a chunked input without chunks
    if (a->length > RunEndMax(rt))   // validateRunEndType (vector_run_end_encode.go:437-444)
      return Status::Invalid("cannot run-end encode arrays with more elements than the run end type can hold: " + std::to_string(RunEndMax(rt)));
    std::shared_ptr<ArrayData> r;
    RETURN_NOT_OK(EncodeOne(rt, *a, &r));
    res.push_back(r);
  }
  if (values.kind == DatumKind::ARRAY) { *out = Datum(res[0]); return Status::OK(); }
  auto c = MakeChunked(Type::RUN_END_ENCODED, std::move(res));
  c->value_type = t; c->run_end_type = rt;
  *out = Datum(c);
  return Status::OK();
}

Status RunEndDecode(const ExecCtx& ctx, const Datum& values, Datum* out) {
  if (values.kind != DatumKind::ARRAY && values.kind != DatumKind::CHUNKED) return Status::NotImplemented("run_end_decode takes an array-like argument");
  if (values.type() != Type::RUN_END_ENCODED)
    return Status::NotImplemented(std::string("function 'run_end_decode' has no kernel matching input types (") + TypeName(values.type()) + ")");
  std::vector<std::shared_ptr<ArrayData>> spans;
  RETURN_NOT_OK(ChunkwiseSpans(values, &spans));
  std::vector<std::shared_ptr<ArrayData>> res;
  for (auto& a : spans) {
    std::shared_ptr<ArrayData> r;
    if (!a) {   // a chunked input without chunks
      RETURN_NOT_OK(ArrayData::FromHost(values.chunked->value_type, 0, 0, nullptr, nullptr, 0, &r));
    } else {
      RETURN_NOT_OK(DecodeOne(*a, &r));
    }
    res.push_back(r);
  }
  if (values.kind == DatumKind::ARRAY) { *out = Datum(res[0]); return Status::OK(); }
  *out = Datum(MakeChunked(values.chunked->value_type, std::move(res)));
  return Status::OK();
}

Status Filter(const ExecCtx& ctx, const Datum& values, const Datum& filter, const FilterOptions& opts, Datum* out) {
  return CallFunction(ctx, "filter", &opts, {values, filter}, out);
}
Status Take(const ExecCtx& ctx, const TakeOptions& opts, const Datum& values, const Datum& indices, Datum* out) {
  return CallFunction(ctx, "take", &opts, {values, indices}, out);
}

// ---------------------------------------------------------------- scalar expressions ------
std::shared_ptr<Expression> FieldRef(int index) {
  auto e = std::make_shared<Expression>();
  e->kind = Expression::Kind::FIELD; e->field = index;
  return e;
}
std::shared_ptr<Expression> Literal(std::shared_ptr<Scalar> value) {
  auto e = std::make_shared<Expression>();
  e->kind = Expression::Kind::LITERAL; e->literal = std::move(value);
  return e;
}
std::shared_ptr<Expression> Call(std::string name, std::vector<std::shared_ptr<Expression>> args, std::shared_ptr<FunctionOptions> options) {
  auto e = std::make_shared<Expression>();
  e->kind = Expression::Kind::CALL; e->name = std::move(name); e->args = std::move(args); e->options = std::move(options);
  return e;
}
std::shared_ptr<Expression> Cast(std::shared_ptr<Expression> arg, const CastOptions& opts) {
  return Call("cast", {std::move(arg)}, std::make_shared<CastOptions>(opts));
}

namespace {

// executeScalarBatch (exprs/exec.go:542-700) over CallFunction: arguments left to right, then the call.  is_in and
// cast are meta functions here but scalar functions in the reference, so they are called like one.
Status EvalNodeByNode(const ExecCtx& ctx, const Expression& e, const Datum& input, Datum* out) {
  switch (e.kind) {
    case Expression::Kind::LITERAL:
      if (!e.literal) return Status::Invalid("literal expression without a value");
      *out = Datum(e.literal);
      return Status::OK();
    case Expression::Kind::FIELD: {
      const int n = NumColumns(input);
      if (e.field < 0 || e.field >= n)
        return Status::Invalid("field index " + std::to_string(e.field) + " out of range: the input has " + std::to_string(n) + " columns");
      *out = ColumnDatum(input, e.field);
      return Status::OK();
    }
    case Expression::Kind::CALL: {
      std::vector<Datum> args(e.args.size());
      for (size_t i = 0; i < e.args.size(); ++i) {
        if (!e.args[i]) return Status::Invalid("call '" + e.name + "': argument " + std::to_string(i) + " is not an expression");
        RETURN_NOT_OK(EvalNodeByNode(ctx, *e.args[i], input, &args[i]));
      }
      FunctionRegistry* reg = ctx.Registry ? ctx.Registry : GetFunctionRegistry();
      const Function* fn = reg->GetFunction(e.name);
      if (fn && fn->Kind() != FuncKind::SCALAR && e.name != "cast" && e.name != "is_in")   // exec.go:625-627
        return Status::Invalid("function '" + e.name + "' is not a scalar function");
      return CallFunction(ctx, e.name, e.options.get(), args, out);
    }
  }
  return Status::NotImplemented("unknown expression kind");
}

// A bound node: a column of `cols` (an input column, an is_in result or an intermediate result), a literal, or a program op
// over bound arguments.
struct BNode {
  enum Kind { COL, LIT, OP } kind = LIT;
  int col = -1;
  std::shared_ptr<Scalar> lit;
  int op = -1, flags = 0;
  Type type = Type::NA, out = Type::NA;   // operand type, result type
  std::vector<std::shared_ptr<BNode>> args;
};
using BPtr = std::shared_ptr<BNode>;

bool ValueType(Type t) { return t == Type::BOOL || IsNumeric(t); }
bool IsNullLiteral(const BPtr& n) { return n->kind == BNode::LIT && !n->lit->valid; }

struct Binder {
  const ExecCtx& ctx;
  const Datum& input;
  std::vector<Column>* cols;
  std::map<int, int> field_col;   // field index -> its column in `cols`: a field named twice is read once

  BPtr Leaf(int c) { auto n = std::make_shared<BNode>(); n->kind = BNode::COL; n->col = c; n->out = (*cols)[c].type; return n; }
  BPtr Lit(std::shared_ptr<Scalar> s) { auto n = std::make_shared<BNode>(); n->kind = BNode::LIT; n->out = s->type; n->lit = std::move(s); return n; }
  BPtr Op(int op, Type type, Type out, std::vector<BPtr> args, int flags = 0) {
    auto n = std::make_shared<BNode>();
    n->kind = BNode::OP; n->op = op; n->type = type; n->out = out; n->args = std::move(args); n->flags = flags;
    return n;
  }
  static int CastFlags(const CastOptions& o) {
    return (o.AllowIntOverflow ? AG_EXPR_ALLOW_INT_OVERFLOW : 0) | (o.AllowFloatTruncate ? AG_EXPR_ALLOW_FLOAT_TRUNCATE : 0);
  }
  // `arg` as type `to` under `o`: a literal is cast now through the cast meta function's scalar route (the node-by-node
  // path casts it the same way), a column in the program.
  bool CastTo(BPtr arg, Type to, const CastOptions& o, BPtr* out) {
    if (arg->out == to) { *out = arg; return true; }
    if (!IsNumeric(arg->out) || !IsNumeric(to)) return false;
    if (arg->kind == BNode::LIT) {
      Datum r;
      if (!CastDatum(ctx, Datum(arg->lit), o, &r).ok()) return false;
      *out = Lit(r.scalar);
      return true;
    }
    *out = Op(AG_EXPR_CAST, arg->out, to, {arg}, CastFlags(o));
    return true;
  }

  // false: the tree is not fused (it fails, or holds something the program does not run); node by node decides.
  bool Bind(const Expression& e, BPtr* out) {
    if (e.kind == Expression::Kind::LITERAL) {
      if (!e.literal || !ValueType(e.literal->type)) return false;
      *out = Lit(e.literal);
      return true;
    }
    if (e.kind == Expression::Kind::FIELD) {
      if (e.field < 0 || e.field >= NumColumns(input)) return false;
      const auto seen = field_col.find(e.field);
      if (seen != field_col.end()) { *out = Leaf(seen->second); return true; }
      Column c = GetColumn(input, e.field);
      if (!ValueType(c.type)) return false;
      cols->push_back(std::move(c));
      field_col[e.field] = (int)cols->size() - 1;
      *out = Leaf((int)cols->size() - 1);
      return true;
    }
    std::vector<BPtr> args(e.args.size());
    bool all_literal = true;
    if (e.name == "is_in") {   // a meta function here: CallFunction runs it and its result is a column of the program
      Datum r;
      if (!EvalNodeByNode(ctx, e, input, &r).ok() || (r.kind != DatumKind::ARRAY && r.kind != DatumKind::CHUNKED)) return false;
      cols->push_back(Column{r.type(), ArrayChunks(r)});
      *out = Leaf((int)cols->size() - 1);
      return true;
    }
    for (size_t i = 0; i < e.args.size(); ++i) {
      if (!e.args[i] || !Bind(*e.args[i], &args[i])) return false;
      all_literal = all_literal && args[i]->kind == BNode::LIT;
    }
    FunctionRegistry* reg = ctx.Registry ? ctx.Registry : GetFunctionRegistry();
    if (e.name == "cast" && reg->GetFunction(e.name)) {   // the cast meta function: a literal is cast here, as it takes scalars
      const auto* co = dynamic_cast<const CastOptions*>(e.options.get());
      if (!co || co->ToType == Type::NA || args.size() != 1) return false;
      return CastTo(args[0], co->ToType, *co, out);
    }
    if (all_literal) return false;   // scalar-only execution is refused by CallFunction
    const Function* fn = reg->GetFunction(e.name);
    if (!fn) return false;
    if (fn->Kind() != FuncKind::SCALAR || (int)args.size() != fn->Arity()) return false;
    const auto* sfn = static_cast<const ScalarFunction*>(fn);
    std::vector<Type> types;
    for (auto& a : args) types.push_back(a->out);
    const exec::ScalarKernel* k = nullptr;
    if (!sfn->DispatchBest(&types, &k).ok() || k->expr_op < 0) return false;
    for (size_t i = 0; i < args.size(); ++i)   // the implicit safe casts of exec.go:101-121
      if (!CastTo(args[i], types[i], SafeCastOptions(types[i]), &args[i])) return false;
    const Type res = k->out_type(types);
    int flags = 0;
    if (k->expr_op == AG_EXPR_CAST) {   // cast_<type> by name: its options are the call's
      const auto* co = dynamic_cast<const CastOptions*>(e.options.get());
      if (!co) return false;
      flags = CastFlags(*co);
    }
    // A null literal operand: the checked kernels write nothing (helpers.go:287) and the boolean kernels leave the data
    // at 0, so the result is 0 and null in every row; the other operand still runs for its failures.
    const int op = k->expr_op;
    const bool empty_on_null = op == AG_EXPR_ADD_CHECKED || op == AG_EXPR_SUB_CHECKED || op == AG_EXPR_MUL_CHECKED || op == AG_EXPR_DIV ||
                               op == AG_EXPR_DIV_CHECKED || (op >= AG_EXPR_SHL && op <= AG_EXPR_SHR_CHECKED) ||
                               (op >= AG_EXPR_AND && op <= AG_EXPR_AND_NOT);
    if (empty_on_null && args.size() == 2 && (IsNullLiteral(args[0]) || IsNullLiteral(args[1]))) {
      *out = Op(AG_EXPR_NULL_OF, res, res, {IsNullLiteral(args[0]) ? args[1] : args[0]});
      return true;
    }
    *out = Op(op, types.empty() ? res : types[0], res, args, flags);
    return true;
  }
};

// Sethi-Ullman label (registers the subtree needs), its distinct columns and its instruction count.
struct Need { int regs = 1, nodes = 1; std::vector<int> cols; };
Need Measure(const BPtr& n) {
  Need r;
  if (n->kind == BNode::COL) { r.cols = {n->col}; return r; }
  if (n->kind == BNode::LIT) return r;
  std::vector<Need> c;
  for (auto& a : n->args) c.push_back(Measure(a));
  r.nodes = 1;
  for (auto& x : c) { r.nodes += x.nodes; r.cols.insert(r.cols.end(), x.cols.begin(), x.cols.end()); }
  std::sort(r.cols.begin(), r.cols.end());
  r.cols.erase(std::unique(r.cols.begin(), r.cols.end()), r.cols.end());
  r.regs = c[0].regs;
  if (c.size() == 2) r.regs = c[0].regs == c[1].regs ? c[0].regs + 1 : std::max(c[0].regs, c[1].regs);
  return r;
}
bool Fits(const Need& n) { return n.regs <= AG_EXPR_MAX_REGS && (int)n.cols.size() <= AG_EXPR_MAX_COLS && n.nodes <= AG_EXPR_MAX_INSTR; }

struct Emitter {
  std::vector<ag_expr_instr> ins;
  std::vector<int> col_slot;    // program column -> index into the bound columns
  std::vector<int> free_regs;
  int Alloc() { int r = free_regs.back(); free_regs.pop_back(); return r; }
  int Slot(int c) {
    for (size_t i = 0; i < col_slot.size(); ++i) if (col_slot[i] == c) return (int)i;
    col_slot.push_back(c);
    return (int)col_slot.size() - 1;
  }
  // Post-order; of two arguments the one that needs more registers goes first, and the result reuses its register.
  int Gen(const BPtr& n) {
    ag_expr_instr in{};
    in.out_type = (int)n->out;
    if (n->kind != BNode::OP) {
      in.dst = Alloc();
      in.type = (int)n->out;
      if (n->kind == BNode::COL) { in.op = AG_EXPR_LOAD; in.a = Slot(n->col); }
      else { in.op = AG_EXPR_CONST; in.flags = n->lit->valid ? 1 : 0; memcpy(&in.bits, n->lit->value, 8); }
      ins.push_back(in);
      return in.dst;
    }
    in.op = n->op; in.type = (int)n->type; in.flags = n->flags;
    if (n->args.size() == 1) {
      in.a = in.dst = Gen(n->args[0]);
    } else {
      const bool left_first = Measure(n->args[0]).regs >= Measure(n->args[1]).regs;
      if (left_first) { in.a = Gen(n->args[0]); in.b = Gen(n->args[1]); }
      else { in.b = Gen(n->args[1]); in.a = Gen(n->args[0]); }
      in.dst = in.a;
      free_regs.push_back(in.b);
    }
    ins.push_back(in);
    return in.dst;
  }
};

// One program over the rows of `cols`: spans from iterateExecSpans over the chunk layouts of the columns it reads,
// one ag_eval_program_dev launch, the output as one array.  *failed: some op of the program failed.
Status RunProgram(const BPtr& root, const std::vector<Column>& cols, int64_t nrows, std::shared_ptr<ArrayData>* out, bool* failed) {
  Emitter em;
  for (int r = AG_EXPR_MAX_REGS - 1; r >= 0; --r) em.free_regs.push_back(r);
  ag_expr_program prog{};
  prog.out_reg = em.Gen(root);
  prog.n_instr = (int)em.ins.size();
  prog.instr = em.ins.data();
  std::vector<int32_t> col_types;
  std::vector<std::vector<std::shared_ptr<ArrayData>>> chunks;
  for (int c : em.col_slot) {
    col_types.push_back((int32_t)cols[c].type);
    chunks.push_back(cols[c].chunks);
  }
  prog.n_cols = (int)col_types.size();
  prog.col_types = col_types.data();
  std::vector<SpanPiece> pieces;
  RETURN_NOT_OK(ChunkSpans(chunks, std::vector<bool>(chunks.size(), true), INT64_MAX, &pieces));
  std::vector<ag_sort_chunk> spans;
  int64_t n_spans = 0;
  for (auto& p : pieces) {
    if (p.len == 0) continue;
    for (size_t j = 0; j < chunks.size(); ++j) spans.push_back(ChunkDesc(*chunks[j][p.chunk_index[j]], p.chunk_pos[j], p.len));
    ++n_spans;
  }
  std::shared_ptr<ArrayData> a;
  RETURN_NOT_OK(AllocateOutput(root->out, nrows, true, &a));
  ErrorWord word;
  RETURN_NOT_OK(word.Init());
  NATIVE(ag_eval_program_dev(&prog, n_spans, spans.data(), a->buffers[1]->data(), a->buffers[0]->data(), word.word(), nullptr));
  int64_t bad = AG_NO_ERROR_POS;
  RETURN_NOT_OK(word.Read(&bad));
  *failed = bad != AG_NO_ERROR_POS;
  *out = a;
  return Status::OK();
}

// A tree that needs more registers, columns or instructions than one program holds: its largest subtree that does not
// fit is evaluated first, as programs of its own, and enters the rest as a column.
Status RunFused(BPtr root, std::vector<Column>* cols, int64_t nrows, std::shared_ptr<ArrayData>* out, bool* failed) {
  while (!Fits(Measure(root))) {
    // descend into an argument that does not fit; below a node whose arguments all fit, take its largest argument
    BPtr* slot = &root;
    for (bool fits = false; !fits;) {
      BPtr* next = nullptr;
      Need best;
      for (auto& a : (*slot)->args) {
        if (a->kind != BNode::OP) continue;
        const Need m = Measure(a);
        const bool better = !next || (Fits(best) && !Fits(m)) ||
                            (Fits(best) == Fits(m) && std::make_tuple(m.regs, m.cols.size(), m.nodes) > std::make_tuple(best.regs, best.cols.size(), best.nodes));
        if (better) { next = &a; best = m; }
      }
      slot = next;
      fits = Fits(best);
    }
    std::shared_ptr<ArrayData> part;
    RETURN_NOT_OK(RunProgram(*slot, *cols, nrows, &part, failed));
    if (*failed) return Status::OK();
    cols->push_back(Column{part->type, {part}});
    auto leaf = std::make_shared<BNode>();
    leaf->kind = BNode::COL; leaf->col = (int)cols->size() - 1; leaf->out = part->type;
    *slot = leaf;
  }
  return RunProgram(root, *cols, nrows, out, failed);
}

}  // namespace

Status ExecuteScalarExpression(const ExecCtx& ctx, const Expression& expr, const Datum& input, Datum* out) {
  if (input.kind != DatumKind::RECORD && input.kind != DatumKind::TABLE)
    return Status::Invalid("ExecuteScalarExpression takes a record batch or a table");
  std::vector<Column> cols;
  Binder b{ctx, input, &cols, {}};
  BPtr root;
  if (!b.Bind(expr, &root) || root->kind != BNode::OP) return EvalNodeByNode(ctx, expr, input, out);
  std::shared_ptr<ArrayData> res;
  bool failed = false;
  RETURN_NOT_OK(RunFused(root, &cols, input.Len(), &res, &failed));
  if (failed) return EvalNodeByNode(ctx, expr, input, out);   // its status, message included
  *out = input.kind == DatumKind::RECORD ? Datum(res) : Datum(MakeChunked(res->type, {res}));
  return Status::OK();
}

}  // namespace compute

// ======================================================================================
// math
// ======================================================================================
namespace math {
template <typename T, typename F>
static Status SumImpl(const ArrayData& a, Type want, T* out, F&& fn) {
  if (a.type != want) return Status::TypeError(std::string("Sum: expected ") + TypeName(want) + " got " + TypeName(a.type));
  *out = T(0);
  if (a.length == 0) return Status::OK();  // float64.go:35-37
  std::shared_ptr<Buffer> res;
  RETURN_NOT_OK(Buffer::Allocate(8, &res));
  NATIVE(fn((const T*)(a.buffers[1]->data()) + a.offset, (size_t)a.length, (T*)res->data(), nullptr));
  return res->ToHost(out, 8);
}
Status SumFloat64(const ArrayData& a, double* out) { return SumImpl<double>(a, Type::FLOAT64, out, ag_sum_f64_dev); }
Status SumInt64(const ArrayData& a, int64_t* out) { return SumImpl<int64_t>(a, Type::INT64, out, ag_sum_i64_dev); }
Status SumUint64(const ArrayData& a, uint64_t* out) { return SumImpl<uint64_t>(a, Type::UINT64, out, ag_sum_u64_dev); }
Status SumFloat64ReferenceOrder(const ArrayData& a, double* out) { return SumImpl<double>(a, Type::FLOAT64, out, ag_sum_f64_reforder_dev); }
}  // namespace math

}  // namespace arrowgpu
