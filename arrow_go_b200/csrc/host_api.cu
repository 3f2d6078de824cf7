// host_api.cu — the HOST-pointer flavour of every compute entry point.
//
// This is the form a per-span exec.ArrayKernelExec binds through cgo: it receives the raw
// bytes of ArraySpan.Buffers[i].Buf exactly like the reference's asm stubs do
// (arrow/compute/internal/kernels/base_arithmetic_avx2_amd64.go:35-39) and returns when the
// output bytes are in host memory.  Each call owns pooled streams for its duration, stages its
// operands into stream-ordered device temporaries and runs the SAME kernels as the *_dev
// flavour (so results are bit-identical between the two).  The staging helpers (Temps, h2d /
// d2h / sync, upload_bitmap, OutBitmap) live in host_stage.cuh, shared with the host flavours
// of the other files.
//
// Elementwise arithmetic and comparisons are pipelined in row chunks over three streams so
// that H2D of chunk k+1, the kernel of chunk k and D2H of chunk k-1 overlap (PCIe is full
// duplex; the kernels are ~100x faster than the link).  Buffers obtained from ag_host_alloc /
// ag_host_register are DMA'd directly; pageable memory still works but the driver bounces it
// through its own pinned staging area.
#include "host_stage.cuh"

#include <string.h>
#include <vector>

namespace ag {

// Upload rows [off, off+n) of a column of w-byte values and their validity bits (validity may be NULL).  The device
// copy of the values starts at row `off`; the copy of the validity keeps the bit phase off & 7 (upload_bitmap).  The
// kernels index a value and its validity bit with the same row number, so *d_vals comes back rebased by -phase rows:
// value i of the slice is row i + *phase of *d_vals, next to validity bit i + *phase of *d_valid.
static ag_status upload_column(Temps& t, const void* vals, const uint8_t* valid, int64_t off, int64_t n, int w,
                               const void** d_vals, uint8_t** d_valid, int64_t* phase) {
  void* dv;
  AG_TRY(t.alloc(&dv, (size_t)n * w));
  AG_TRY(h2d(dv, (const char*)vals + off * w, (size_t)n * w, t.st));
  AG_TRY(upload_bitmap(t, valid, off, n, d_valid, phase));
  *d_vals = (const char*)dv - *phase * w;
  return AG_OK;
}

// Stage one chunk of a BOOL or numeric column: a BOOL bitmap keeps its bit phase (upload_bitmap), other values are
// rebased as upload_column does; d->offset addresses row 0 of the copies.  An empty chunk stages nothing.
static ag_status upload_chunk(Temps& t, int type, const ag_sort_chunk& h, ag_sort_chunk* d) {
  *d = ag_sort_chunk{nullptr, nullptr, 0, h.length};
  if (h.length <= 0) return AG_OK;
  uint8_t* dvalid;
  if (type == AG_TYPE_BOOL) {
    uint8_t* dv;
    AG_TRY(upload_bitmap(t, static_cast<const uint8_t*>(h.vals), h.offset, h.length, &dv, &d->offset));
    d->vals = dv;
    int64_t phase;
    AG_TRY(upload_bitmap(t, h.valid, h.offset, h.length, &dvalid, &phase));
  } else {
    AG_TRY(upload_column(t, h.vals, h.valid, h.offset, h.length, type_width(type), &d->vals, &dvalid, &d->offset));
  }
  d->valid = dvalid;
  return AG_OK;
}

// AG_ERR_INDEX naming the host index at the lowest offending row `bad` (helpers.go:951), also stored in *bad_index.
static ag_status index_bounds_error(const void* idx, int idx_width, int idx_signed, int64_t bad, int64_t* bad_index) {
  int64_t v = 0;
  switch (idx_width) {
    case 8: v = idx_signed ? (int64_t)((const int8_t*)idx)[bad] : (int64_t)((const uint8_t*)idx)[bad]; break;
    case 16: v = idx_signed ? (int64_t)((const int16_t*)idx)[bad] : (int64_t)((const uint16_t*)idx)[bad]; break;
    case 32: v = idx_signed ? (int64_t)((const int32_t*)idx)[bad] : (int64_t)((const uint32_t*)idx)[bad]; break;
    default: v = ((const int64_t*)idx)[bad]; break;
  }
  if (bad_index) *bad_index = v;
  if (idx_width == 64 && !idx_signed) AG_FAIL(AG_ERR_INDEX, "%llu out of bounds", (unsigned long long)v);
  AG_FAIL(AG_ERR_INDEX, "%lld out of bounds", (long long)v);
}

// Finish a call whose output has `len` rows: copy the output validity back when the caller passed a bitmap, set *nulls
// to its clear bits when asked (d_count: one device int64 of scratch), and synchronise the stream.
static ag_status fetch_validity(uint8_t* out_valid, const uint8_t* d_valid, int64_t len, int64_t* nulls, int64_t* d_count,
                                cudaStream_t st) {
  int64_t valid = 0;
  if (out_valid) {
    AG_TRY(d2h(out_valid, d_valid, (size_t)((len + 7) / 8), st));
    if (nulls) {
      AG_TRY(bitmap_popcount_dev(d_valid, 0, len, d_count, st));
      AG_TRY(d2h(&valid, d_count, sizeof(int64_t), st));
    }
  }
  AG_TRY(sync(st));
  if (out_valid && nulls) *nulls = len - valid;
  return AG_OK;
}

constexpr int kPipe = 3;
constexpr int64_t kChunkBytes = (int64_t)32 << 20;  // per operand per pipeline stage

struct Pipe {
  CallStream s[kPipe];
  ag_status acquire() { for (auto& c : s) AG_TRY(c.acquire()); return AG_OK; }
  ag_status sync_all() { for (auto& c : s) AG_CUDA_TRY(cudaStreamSynchronize(c.st)); return AG_OK; }
};

// chunked, 3-deep pipelined elementwise call.  in[k] == nullptr marks an operand that is not an array.
template <typename Launch>
static ag_status pipelined_rows(int64_t n, int n_in, const void* const* in, const int* in_width,
                                void* out, int out_width, Launch&& launch) {
  AG_TRY(ensure_init());
  if (n == 0) return AG_OK;
  Pipe pipe;
  AG_TRY(pipe.acquire());
  int wmax = out_width;
  for (int k = 0; k < n_in; ++k) if (in[k] && in_width[k] > wmax) wmax = in_width[k];
  int64_t chunk = kChunkBytes / wmax;
  chunk &= ~(int64_t)1023;
  if (chunk > n) chunk = n;
  const int slots = (n + chunk - 1) / chunk < kPipe ? (int)((n + chunk - 1) / chunk) : kPipe;
  void* d_in[kPipe][4] = {};
  void* d_out[kPipe] = {};
  ag_status rc = AG_OK;
  for (int sl = 0; sl < slots && rc == AG_OK; ++sl) {
    for (int k = 0; k < n_in && rc == AG_OK; ++k)
      if (in[k]) rc = dev_alloc_async(&d_in[sl][k], (size_t)chunk * in_width[k] + 64, pipe.s[sl]);
    if (rc == AG_OK) rc = dev_alloc_async(&d_out[sl], (size_t)chunk * out_width + 64, pipe.s[sl]);
  }
  int64_t ci = 0;
  for (int64_t r0 = 0; r0 < n && rc == AG_OK; r0 += chunk, ++ci) {
    const int sl = (int)(ci % kPipe);
    const int64_t len = (n - r0 < chunk) ? (n - r0) : chunk;
    cudaStream_t st = pipe.s[sl];
    for (int k = 0; k < n_in && rc == AG_OK; ++k)
      if (in[k]) rc = h2d(d_in[sl][k], (const char*)in[k] + r0 * in_width[k], (size_t)len * in_width[k], st);
    if (rc == AG_OK) rc = launch(d_in[sl], d_out[sl], len, st);
    if (rc == AG_OK) rc = d2h((char*)out + r0 * out_width, d_out[sl], (size_t)len * out_width, st);
  }
  for (int sl = 0; sl < slots; ++sl) {
    for (int k = 0; k < n_in; ++k) if (d_in[sl][k]) cudaFreeAsync(d_in[sl][k], pipe.s[sl]);
    if (d_out[sl]) cudaFreeAsync(d_out[sl], pipe.s[sl]);
  }
  ag_status rs = pipe.sync_all();
  return rc != AG_OK ? rc : rs;
}

// Host flavour of the batched-span call.  Spans are cut into pieces of at most one stage (32 MB per operand), pieces
// that continue each other in host memory on every operand are merged (slices of one allocation: a chunked array built
// from NewSlice views), and pieces are PACKED into stages of up to 32 MB: each piece is copied to the next 16-byte
// aligned offset of the stage's device buffers, ONE kernel runs over the packed range (the few padding rows between
// pieces compute garbage nobody reads), and each piece is copied back from the same offset.  So a chunked call with
// 8 MB chunks runs the same 3-deep H2D / kernel / D2H pipeline, with the same stage size, as one contiguous column
// (one stage per span would leave the pipeline short of bytes; scripts/e2e_probe.py times both forms).
static ag_status host_arith_binary_spans(int type, int8_t op, int shape, const ag_span3* spans, int64_t n_spans) {
  AG_TRY(ensure_init());
  const int w = type_width(type);
  if (w == 0) AG_FAIL(AG_ERR_TYPE, "arith: unsupported type id %d", type);
  if (n_spans < 0 || (n_spans > 0 && !spans)) AG_FAIL(AG_ERR_INVALID, "arith_spans: bad span table");
  const bool la = shape != AG_SHAPE_SA, ra = shape != AG_SHAPE_AS;
  const int64_t chunk = (kChunkBytes / w) & ~(int64_t)1023;   // rows per stage
  const int64_t pad = 16 / w;                                   // pieces start on 16-byte boundaries of the stage
  struct Piece { const char* l; const char* r; char* out; int64_t n; };
  std::vector<Piece> pieces;
  const void* scalar_l = nullptr; const void* scalar_r = nullptr;
  for (int64_t i = 0; i < n_spans; ++i) {
    const ag_span3& sp = spans[i];
    if (sp.n < 0) AG_FAIL(AG_ERR_INVALID, "arith_spans: negative length");
    if (sp.n == 0) continue;
    if (!sp.l || !sp.r || !sp.out) AG_FAIL(AG_ERR_INVALID, "arith_spans: NULL operand");
    if (!la) scalar_l = sp.l;
    if (!ra) scalar_r = sp.r;
    for (int64_t r0 = 0; r0 < sp.n; r0 += chunk) {
      Piece p{(const char*)sp.l + (la ? r0 * w : 0), (const char*)sp.r + (ra ? r0 * w : 0), (char*)sp.out + r0 * w, sp.n - r0 < chunk ? sp.n - r0 : chunk};
      if (!pieces.empty()) {
        Piece& q = pieces.back();
        const bool cont = (!la || q.l + q.n * w == p.l) && (!ra || q.r + q.n * w == p.r) && q.out + q.n * w == p.out;
        if (cont && q.n + p.n <= chunk) { q.n += p.n; continue; }
      }
      pieces.push_back(p);
    }
  }
  if (pieces.empty()) return AG_OK;
  Pipe pipe;
  AG_TRY(pipe.acquire());
  void* d_l[kPipe] = {}; void* d_r[kPipe] = {}; void* d_o[kPipe] = {};
  ag_status rc = AG_OK;
  const size_t stage_bytes = (size_t)(chunk + pad) * w + 64;
  for (int sl = 0; sl < kPipe && rc == AG_OK; ++sl) {
    if (la) rc = dev_alloc_async(&d_l[sl], stage_bytes, pipe.s[sl]);
    if (rc == AG_OK && ra) rc = dev_alloc_async(&d_r[sl], stage_bytes, pipe.s[sl]);
    if (rc == AG_OK) rc = dev_alloc_async(&d_o[sl], stage_bytes, pipe.s[sl]);
  }
  int64_t ci = 0;
  for (size_t first = 0; first < pieces.size() && rc == AG_OK; ++ci) {
    const int sl = (int)(ci % kPipe);
    cudaStream_t st = pipe.s[sl];
    // pieces [first, last) of this stage, each at a 16-byte aligned row offset
    size_t last = first;
    int64_t rows = 0;
    while (last < pieces.size()) {
      const int64_t at = (rows + pad - 1) / pad * pad;
      if (last > first && at + pieces[last].n > chunk) break;
      rows = at + pieces[last].n;
      ++last;
    }
    int64_t at = 0;
    for (size_t k = first; k < last && rc == AG_OK; ++k) {
      at = (at + pad - 1) / pad * pad;
      if (la) rc = h2d((char*)d_l[sl] + at * w, pieces[k].l, (size_t)pieces[k].n * w, st);
      if (rc == AG_OK && ra) rc = h2d((char*)d_r[sl] + at * w, pieces[k].r, (size_t)pieces[k].n * w, st);
      at += pieces[k].n;
    }
    if (rc == AG_OK) rc = arith_binary_dev(type, op, shape, la ? d_l[sl] : scalar_l, ra ? d_r[sl] : scalar_r, d_o[sl], rows, st);
    at = 0;
    for (size_t k = first; k < last && rc == AG_OK; ++k) {
      at = (at + pad - 1) / pad * pad;
      rc = d2h(pieces[k].out, (const char*)d_o[sl] + at * w, (size_t)pieces[k].n * w, st);
      at += pieces[k].n;
    }
    first = last;
  }
  for (int sl = 0; sl < kPipe; ++sl) {
    if (d_l[sl]) cudaFreeAsync(d_l[sl], pipe.s[sl]);
    if (d_r[sl]) cudaFreeAsync(d_r[sl], pipe.s[sl]);
    if (d_o[sl]) cudaFreeAsync(d_o[sl], pipe.s[sl]);
  }
  ag_status rs = pipe.sync_all();
  return rc != AG_OK ? rc : rs;
}

static ag_status host_arith_binary(int type, int8_t op, int shape, const void* l, const void* r, void* out, int64_t n) {
  const int w = type_width(type);
  if (w == 0) AG_FAIL(AG_ERR_TYPE, "arith: unsupported type id %d", type);
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "arith: negative length");
  if (n > 0 && (!l || !r || !out)) AG_FAIL(AG_ERR_INVALID, "arith: NULL operand");
  const void* in[2] = {shape == AG_SHAPE_SA ? nullptr : l, shape == AG_SHAPE_AS ? nullptr : r};
  const int widths[2] = {w, w};
  return pipelined_rows(n, 2, in, widths, out, w, [&](void* const* d_in, void* d_out, int64_t len, cudaStream_t st) {
    return arith_binary_dev(type, op, shape, shape == AG_SHAPE_SA ? l : d_in[0], shape == AG_SHAPE_AS ? r : d_in[1], d_out, len, st);
  });
}

}  // namespace ag

using namespace ag;

extern "C" {

// ---- arithmetic ------------------------------------------------------------------
ag_status ag_arith_binary(int type, int8_t op, const void* l, const void* r, void* out, int64_t n) {
  return host_arith_binary(type, op, AG_SHAPE_AA, l, r, out, n);
}
ag_status ag_arith_arr_scalar(int type, int8_t op, const void* l, const void* r, void* out, int64_t n) {
  return host_arith_binary(type, op, AG_SHAPE_AS, l, r, out, n);
}
ag_status ag_arith_scalar_arr(int type, int8_t op, const void* l, const void* r, void* out, int64_t n) {
  return host_arith_binary(type, op, AG_SHAPE_SA, l, r, out, n);
}
ag_status ag_arith_binary_spans(int type, int8_t op, int shape, const ag_span3* spans, int64_t n_spans) {
  return host_arith_binary_spans(type, op, shape, spans, n_spans);
}
ag_status ag_arith_unary_same(int type, int8_t op, const void* in, void* out, int64_t n) {
  const int w = type_width(type);
  if (w == 0) AG_FAIL(AG_ERR_TYPE, "arith: unsupported type id %d", type);
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "arith: negative length");
  if (n > 0 && (!in || !out)) AG_FAIL(AG_ERR_INVALID, "arith: NULL operand");
  const void* ins[1] = {in};
  const int widths[1] = {w};
  return pipelined_rows(n, 1, ins, widths, out, w, [&](void* const* d_in, void* d_out, int64_t len, cudaStream_t st) {
    return arith_unary_same_dev(type, op, d_in[0], d_out, len, st);
  });
}
ag_status ag_arith_unary_diff(int itype, int otype, int8_t op, const void* in, void* out, int64_t n) {
  const int wi = type_width(itype), wo = type_width(otype);
  if (wi == 0 || wo == 0) AG_FAIL(AG_ERR_TYPE, "arith: unsupported type id");
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "arith: negative length");
  if (n > 0 && (!in || !out)) AG_FAIL(AG_ERR_INVALID, "arith: NULL operand");
  const void* ins[1] = {in};
  const int widths[1] = {wi};
  return pipelined_rows(n, 1, ins, widths, out, wo, [&](void* const* d_in, void* d_out, int64_t len, cudaStream_t st) {
    return arith_unary_diff_dev(itype, otype, op, d_in[0], d_out, len, st);
  });
}

ag_status ag_arith_checked(int type, int8_t op, int shape, const void* l, const uint8_t* lvalid, int64_t loff,
                           const void* r, const uint8_t* rvalid, int64_t roff, void* out, int64_t n, int64_t* first_bad) {
  AG_TRY(ensure_init());
  if (first_bad) *first_bad = AG_NO_ERROR_POS;
  const int w = type_width(type);
  if (w == 0) AG_FAIL(AG_ERR_TYPE, "arith_checked: type id %d is not a numeric type", type);
  if (type_is_float(type) && op != AG_OP_DIV && op != AG_OP_DIV_CHECKED)
    AG_FAIL(AG_ERR_TYPE, "arith_checked: type id %d is not an integer type (floating point types have NotNull kernels for DIV / DIV_CHECKED only)", type);
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "arith_checked: negative length");
  if (n == 0) return AG_OK;
  if ((shape == AG_SHAPE_SA && !l) || (shape == AG_SHAPE_AS && !r)) return AG_OK;  // null scalar
  if (!l || !r || !out) AG_FAIL(AG_ERR_INVALID, "arith_checked: NULL operand");
  CallStream cs;
  AG_TRY(cs.acquire());
  Temps t(cs);
  void *dl = nullptr, *dr = nullptr, *dout = nullptr;
  uint8_t *dlv = nullptr, *drv = nullptr;
  int64_t dloff = 0, droff = 0;
  int64_t* d_bad = nullptr;
  if (shape != AG_SHAPE_SA) { AG_TRY(t.alloc(&dl, (size_t)n * w)); AG_TRY(h2d(dl, l, (size_t)n * w, cs)); AG_TRY(upload_bitmap(t, lvalid, loff, n, &dlv, &dloff)); }
  if (shape != AG_SHAPE_AS) { AG_TRY(t.alloc(&dr, (size_t)n * w)); AG_TRY(h2d(dr, r, (size_t)n * w, cs)); AG_TRY(upload_bitmap(t, rvalid, roff, n, &drv, &droff)); }
  AG_TRY(t.alloc(&dout, (size_t)n * w));
  AG_TRY(t.alloc_t(&d_bad, sizeof(int64_t)));
  AG_TRY(error_word_reset(d_bad, cs));
  AG_TRY(arith_checked_dev(type, op, shape, shape == AG_SHAPE_SA ? l : dl, dlv, dloff, shape == AG_SHAPE_AS ? r : dr, drv, droff, dout, n, d_bad, cs));
  int64_t bad = AG_NO_ERROR_POS;
  AG_TRY(d2h(&bad, d_bad, sizeof(bad), cs));
  AG_TRY(d2h(out, dout, (size_t)n * w, cs));
  AG_TRY(sync(cs));
  if (first_bad) *first_bad = bad;
  if (bad != AG_NO_ERROR_POS) {
    if (op == AG_OP_DIV || op == AG_OP_DIV_CHECKED) AG_FAIL(AG_ERR_INVALID, "divide by zero");  // errDivByZero, base_arithmetic.go:139
    if (op == AG_OP_SHIFT_LEFT_CHECKED || op == AG_OP_SHIFT_RIGHT_CHECKED)
      AG_FAIL(AG_ERR_INVALID, "shift amount must be >= 0 and less than precision of type");     // errShift, scalar_arithmetic.go:294
    AG_FAIL(AG_ERR_INVALID, "overflow");                                                        // errOverflow,  base_arithmetic.go:138
  }
  return AG_OK;
}

ag_status ag_arith_unary_checked(int type, int8_t op, const void* in, void* out, int64_t n, int64_t* first_bad) {
  AG_TRY(ensure_init());
  if (first_bad) *first_bad = AG_NO_ERROR_POS;
  const int w = type_width(type);
  if (w == 0) AG_FAIL(AG_ERR_TYPE, "arith: unsupported type id %d", type);
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "arith: negative length");
  if (n == 0) return AG_OK;
  if (!in || !out) AG_FAIL(AG_ERR_INVALID, "arith: NULL operand");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  void *din, *dout; int64_t* d_bad;
  AG_TRY(t.alloc(&din, (size_t)n * w)); AG_TRY(t.alloc(&dout, (size_t)n * w)); AG_TRY(t.alloc_t(&d_bad, sizeof(int64_t)));
  AG_TRY(h2d(din, in, (size_t)n * w, cs));
  AG_TRY(error_word_reset(d_bad, cs));
  AG_TRY(arith_unary_checked_dev(type, op, din, dout, n, d_bad, cs));
  int64_t bad = AG_NO_ERROR_POS;
  AG_TRY(d2h(&bad, d_bad, sizeof(bad), cs));
  AG_TRY(d2h(out, dout, (size_t)n * w, cs));
  AG_TRY(sync(cs));
  if (first_bad) *first_bad = bad;
  if (bad != AG_NO_ERROR_POS) AG_FAIL(AG_ERR_INVALID, "overflow");
  return AG_OK;
}

// ---- numeric casts -----------------------------------------------------------------
ag_status ag_cast_numeric(int itype, int otype, const void* in, void* out, int64_t n) {
  const int wi = type_width(itype), wo = type_width(otype);
  if (wi == 0 || wo == 0) AG_FAIL(AG_ERR_TYPE, "cast: unsupported type id");
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "cast: negative length");
  if (n > 0 && (!in || !out)) AG_FAIL(AG_ERR_INVALID, "cast: NULL operand");
  const void* ins[1] = {in};
  const int widths[1] = {wi};
  return pipelined_rows(n, 1, ins, widths, out, wo, [&](void* const* d_in, void* d_out, int64_t len, cudaStream_t st) {
    return cast_numeric_dev(itype, otype, d_in[0], nullptr, 0, d_out, len, 1, 1, nullptr, 0, st);
  });
}

ag_status ag_cast_numeric_checked(int itype, int otype, const void* in, const uint8_t* valid, int64_t valid_offset,
                                  void* out, int64_t n, int allow_int_overflow, int allow_float_truncate, int64_t* first_bad) {
  AG_TRY(ensure_init());
  if (first_bad) *first_bad = AG_NO_ERROR_POS;
  const int wi = type_width(itype), wo = type_width(otype);
  if (wi == 0 || wo == 0) AG_FAIL(AG_ERR_TYPE, "cast: unsupported type id");
  if (n < 0 || valid_offset < 0) AG_FAIL(AG_ERR_INVALID, "cast: negative length or offset");
  if (n == 0) return AG_OK;
  if (!in || !out) AG_FAIL(AG_ERR_INVALID, "cast: NULL operand");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  void *din, *dout; int64_t* d_bad; uint8_t* dvalid; int64_t dvoff;
  AG_TRY(t.alloc(&din, (size_t)n * wi)); AG_TRY(t.alloc(&dout, (size_t)n * wo)); AG_TRY(t.alloc_t(&d_bad, sizeof(int64_t)));
  AG_TRY(h2d(din, in, (size_t)n * wi, cs));
  AG_TRY(upload_bitmap(t, valid, valid_offset, n, &dvalid, &dvoff));
  AG_TRY(error_word_reset(d_bad, cs));
  AG_TRY(cast_numeric_dev(itype, otype, din, dvalid, dvoff, dout, n, allow_int_overflow, allow_float_truncate, d_bad, 0, cs));
  int64_t bad = AG_NO_ERROR_POS;
  AG_TRY(d2h(&bad, d_bad, sizeof(bad), cs));
  AG_TRY(d2h(out, dout, (size_t)n * wo, cs));
  AG_TRY(sync(cs));
  if (first_bad) *first_bad = bad;
  if (bad != AG_NO_ERROR_POS) {
    // numeric_cast.go:614-617 / helpers.go:591-594 wording; the offending element is in the caller's buffer
    if (type_is_float(itype)) {
      const double v = itype == AG_TYPE_FLOAT32 ? (double)((const float*)in)[bad] : ((const double*)in)[bad];
      AG_FAIL(AG_ERR_INVALID, "float value %f was truncated converting to type id %d", v, otype);
    }
    AG_FAIL(AG_ERR_INVALID, "integer value not in range (row %lld)", (long long)bad);
  }
  return AG_OK;
}

// ---- cumulative sum ----------------------------------------------------------------
ag_status ag_cumulative_sum(int type, const void* in, const uint8_t* valid, int64_t valid_offset, int64_t n,
                            const void* start, int skip_nulls, int checked,
                            void* out, uint8_t* out_valid, int64_t* null_count, int64_t* first_bad) {
  AG_TRY(ensure_init());
  if (first_bad) *first_bad = AG_NO_ERROR_POS;
  if (null_count) *null_count = 0;
  const int w = type_width(type);
  if (w == 0) AG_FAIL(AG_ERR_TYPE, "cumulative_sum: input type must be numeric, got type id %d", type);
  if (n < 0 || valid_offset < 0) AG_FAIL(AG_ERR_INVALID, "cumulative_sum: negative length or offset");
  if (n == 0) return AG_OK;
  if (!in || !out) AG_FAIL(AG_ERR_INVALID, "cumulative_sum: NULL operand");
  if (valid && !out_valid) AG_FAIL(AG_ERR_INVALID, "cumulative_sum: an input with a validity bitmap needs an output validity bitmap");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  void *din, *dout; int64_t* d_bad; uint8_t *dvalid, *dovalid = nullptr; int64_t dvoff; ag_cumsum_state* dstate;
  AG_TRY(t.alloc(&din, (size_t)n * w)); AG_TRY(t.alloc(&dout, (size_t)n * w)); AG_TRY(t.alloc_t(&d_bad, sizeof(int64_t)));
  AG_TRY(t.alloc_t(&dstate, sizeof(ag_cumsum_state)));
  AG_TRY(h2d(din, in, (size_t)n * w, cs));
  const size_t obytes = (size_t)bytes_for_bits(n);
  AG_TRY(upload_bitmap(t, valid, valid_offset, n, &dvalid, &dvoff));
  if (out_valid) {
    AG_TRY(t.alloc_t(&dovalid, obytes + 4));
    AG_CUDA_TRY(cudaMemsetAsync(dovalid, 0, obytes + 4, cs));
  }
  AG_TRY(error_word_reset(d_bad, cs));
  AG_TRY(cumulative_sum_state_init(dstate, type, start, cs));
  AG_TRY(cumulative_sum_dev(type, din, dvalid, dvoff, n, skip_nulls, checked, dout, dovalid, 0, dstate, d_bad, cs));
  int64_t bad = AG_NO_ERROR_POS;
  ag_cumsum_state hs;
  AG_TRY(d2h(&bad, d_bad, sizeof(bad), cs));
  AG_TRY(d2h(&hs, dstate, sizeof(hs), cs));
  AG_TRY(d2h(out, dout, (size_t)n * w, cs));
  if (out_valid) {
    // whole bytes except the last, whose bits past n keep the caller's values
    AG_TRY(sync(cs));
    std::vector<uint8_t> tmp(obytes);
    AG_TRY(d2h(tmp.data(), dovalid, obytes, cs));
    AG_TRY(sync(cs));
    const int tail = (int)(n & 7);
    if (tail) { const uint8_t m = (uint8_t)((1u << tail) - 1u); tmp[obytes - 1] = (uint8_t)((tmp[obytes - 1] & m) | (out_valid[obytes - 1] & ~m)); }
    memcpy(out_valid, tmp.data(), obytes);
  }
  AG_TRY(sync(cs));
  if (first_bad) *first_bad = bad;
  if (null_count) *null_count = hs.null_count;
  if (checked && bad != AG_NO_ERROR_POS) AG_FAIL(AG_ERR_INVALID, "overflow");
  return AG_OK;
}

// ---- comparisons -------------------------------------------------------------------
ag_status ag_compare(int type, int cmp, int shape, const void* l, const void* r, uint8_t* out_bits, int64_t n, int bit_offset) {
  AG_TRY(ensure_init());
  const int w = type_width(type);
  if (w == 0) AG_FAIL(AG_ERR_TYPE, "compare: unsupported type id %d", type);
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "compare: negative length");
  if (n == 0) return AG_OK;
  if (!l || !r || !out_bits) AG_FAIL(AG_ERR_INVALID, "compare: NULL operand");
  const int phase = bit_offset & 7;  // the reference uses offset % 8 relative to `out` (scalar_comparison.cc:72)
  Pipe pipe;
  AG_TRY(pipe.acquire());
  cudaStream_t s0 = pipe.s[0];
  Temps t(s0);
  OutBitmap ob;
  AG_TRY(ob.stage(t, out_bits, phase, n));
  AG_TRY(sync(s0));  // the edge bytes are on the device before the kernels of the other streams write next to them
  ag_status rc = AG_OK;
  // chunk boundaries fall on multiples of 1024 output bits, so chunks never share an output word
  int64_t chunk = (kChunkBytes / w) & ~(int64_t)1023;
  const bool la = shape != AG_SHAPE_SA, ra = shape != AG_SHAPE_AS;
  void* d_l[kPipe] = {};
  void* d_r[kPipe] = {};
  for (int sl = 0; sl < kPipe && rc == AG_OK; ++sl) {
    if (la) rc = dev_alloc_async(&d_l[sl], (size_t)chunk * w + 64, pipe.s[sl]);
    if (rc == AG_OK && ra) rc = dev_alloc_async(&d_r[sl], (size_t)chunk * w + 64, pipe.s[sl]);
  }
  int64_t r0 = 0, ci = 0;
  while (r0 < n && rc == AG_OK) {
    int64_t len = (ci == 0) ? (chunk - phase) : chunk;  // (phase + r0) % 1024 == 0 from the second chunk on
    if (len > n - r0) len = n - r0;
    const int sl = (int)(ci % kPipe);
    cudaStream_t st = pipe.s[sl];
    if (la) rc = h2d(d_l[sl], (const char*)l + r0 * w, (size_t)len * w, st);
    if (rc == AG_OK && ra) rc = h2d(d_r[sl], (const char*)r + r0 * w, (size_t)len * w, st);
    const int64_t obit = phase + r0;
    if (rc == AG_OK) rc = compare_dev(type, cmp, shape, la ? d_l[sl] : l, ra ? d_r[sl] : r, ob.d + (obit >> 3), len, (int)(obit & 7), st);
    r0 += len; ++ci;
  }
  for (int sl = 0; sl < kPipe; ++sl) {
    if (d_l[sl]) cudaFreeAsync(d_l[sl], pipe.s[sl]);
    if (d_r[sl]) cudaFreeAsync(d_r[sl], pipe.s[sl]);
  }
  const ag_status rs = pipe.sync_all();
  AG_TRY(rc);
  AG_TRY(rs);
  AG_TRY(ob.fetch(s0));
  return sync(s0);
}

#define AG_CMP_NAMED(NAME, CMP, SHAPE)                                                                        \
  ag_status NAME(int type, const void* l, const void* r, void* out, int64_t n, int offset) {                  \
    return ag_compare(type, CMP, SHAPE, l, r, (uint8_t*)out, n, offset);                                      \
  }
AG_CMP_NAMED(ag_cmp_eq_aa, AG_CMP_EQ, AG_SHAPE_AA) AG_CMP_NAMED(ag_cmp_eq_as, AG_CMP_EQ, AG_SHAPE_AS) AG_CMP_NAMED(ag_cmp_eq_sa, AG_CMP_EQ, AG_SHAPE_SA)
AG_CMP_NAMED(ag_cmp_ne_aa, AG_CMP_NE, AG_SHAPE_AA) AG_CMP_NAMED(ag_cmp_ne_as, AG_CMP_NE, AG_SHAPE_AS) AG_CMP_NAMED(ag_cmp_ne_sa, AG_CMP_NE, AG_SHAPE_SA)
AG_CMP_NAMED(ag_cmp_gt_aa, AG_CMP_GT, AG_SHAPE_AA) AG_CMP_NAMED(ag_cmp_gt_as, AG_CMP_GT, AG_SHAPE_AS) AG_CMP_NAMED(ag_cmp_gt_sa, AG_CMP_GT, AG_SHAPE_SA)
AG_CMP_NAMED(ag_cmp_ge_aa, AG_CMP_GE, AG_SHAPE_AA) AG_CMP_NAMED(ag_cmp_ge_as, AG_CMP_GE, AG_SHAPE_AS) AG_CMP_NAMED(ag_cmp_ge_sa, AG_CMP_GE, AG_SHAPE_SA)
#undef AG_CMP_NAMED

// ---- bitmaps -----------------------------------------------------------------------
ag_status ag_bitmap_op(int bitop, const uint8_t* l, int64_t loff, const uint8_t* r, int64_t roff, uint8_t* out, int64_t ooff, int64_t n) {
  AG_TRY(ensure_init());
  if (n < 0 || loff < 0 || roff < 0 || ooff < 0) AG_FAIL(AG_ERR_INVALID, "bitmap_op: negative length or offset");
  if (n == 0) return AG_OK;
  if (!l || !r || !out) AG_FAIL(AG_ERR_INVALID, "bitmap_op: NULL bitmap");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  uint8_t *dl, *dr; int64_t dlo, dro;
  AG_TRY(upload_bitmap(t, l, loff, n, &dl, &dlo));
  AG_TRY(upload_bitmap(t, r, roff, n, &dr, &dro));
  OutBitmap ob; AG_TRY(ob.stage(t, out, ooff, n));
  AG_TRY(bitmap_op_dev(bitop, dl, dlo, dr, dro, ob.d, ob.doff, n, cs));
  AG_TRY(ob.fetch(cs));
  return sync(cs);
}
static ag_status host_bitmap_copy(const uint8_t* src, int64_t soff, int64_t n, uint8_t* dst, int64_t doff, bool invert) {
  AG_TRY(ensure_init());
  if (n < 0 || soff < 0 || doff < 0) AG_FAIL(AG_ERR_INVALID, "bitmap_copy: negative length or offset");
  if (n == 0) return AG_OK;
  if (!src || !dst) AG_FAIL(AG_ERR_INVALID, "bitmap_copy: NULL bitmap");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  uint8_t* ds; int64_t dso;
  AG_TRY(upload_bitmap(t, src, soff, n, &ds, &dso));
  OutBitmap ob; AG_TRY(ob.stage(t, dst, doff, n));
  AG_TRY(bitmap_copy_dev(ds, dso, n, ob.d, ob.doff, invert, cs));
  AG_TRY(ob.fetch(cs));
  return sync(cs);
}
ag_status ag_bitmap_copy(const uint8_t* src, int64_t soff, int64_t n, uint8_t* dst, int64_t doff) { return host_bitmap_copy(src, soff, n, dst, doff, false); }
ag_status ag_bitmap_invert(const uint8_t* src, int64_t soff, int64_t n, uint8_t* dst, int64_t doff) { return host_bitmap_copy(src, soff, n, dst, doff, true); }
ag_status ag_bitmap_set(uint8_t* bits, int64_t off, int64_t n, int value) {
  AG_TRY(ensure_init());
  if (n < 0 || off < 0) AG_FAIL(AG_ERR_INVALID, "bitmap_set: negative length or offset");
  if (n == 0) return AG_OK;
  if (!bits) AG_FAIL(AG_ERR_INVALID, "bitmap_set: NULL bitmap");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  OutBitmap ob; AG_TRY(ob.stage(t, bits, off, n));
  AG_TRY(bitmap_set_dev(ob.d, ob.doff, n, value, cs));
  AG_TRY(ob.fetch(cs));
  return sync(cs);
}
ag_status ag_bitmap_popcount(const uint8_t* bits, int64_t off, int64_t n, int64_t* count) {
  AG_TRY(ensure_init());
  if (!count) AG_FAIL(AG_ERR_INVALID, "popcount: NULL result");
  *count = 0;
  if (n < 0 || off < 0) AG_FAIL(AG_ERR_INVALID, "popcount: negative length or offset");
  if (n == 0) return AG_OK;
  if (!bits) AG_FAIL(AG_ERR_INVALID, "popcount: NULL bitmap");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  uint8_t* d; int64_t doff; int64_t* d_count;
  AG_TRY(upload_bitmap(t, bits, off, n, &d, &doff));
  AG_TRY(t.alloc_t(&d_count, sizeof(int64_t)));
  AG_TRY(bitmap_popcount_dev(d, doff, n, d_count, cs));
  AG_TRY(d2h(count, d_count, sizeof(int64_t), cs));
  return sync(cs);
}
ag_status ag_kleene(int kop, const uint8_t* lvalid, const uint8_t* ldata, int64_t loff, const uint8_t* rvalid, const uint8_t* rdata, int64_t roff,
                    uint8_t* out_valid, uint8_t* out_data, int64_t ooff, int64_t n) {
  AG_TRY(ensure_init());
  if (n < 0 || loff < 0 || roff < 0 || ooff < 0) AG_FAIL(AG_ERR_INVALID, "kleene: negative length or offset");
  if (n == 0) return AG_OK;
  if (!ldata || !rdata || !out_valid || !out_data) AG_FAIL(AG_ERR_INVALID, "kleene: NULL bitmap");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  uint8_t *dlv, *dld, *drv, *drd; int64_t o1, o2, o3, o4;
  AG_TRY(upload_bitmap(t, lvalid, loff, n, &dlv, &o1));
  AG_TRY(upload_bitmap(t, ldata, loff, n, &dld, &o2));
  AG_TRY(upload_bitmap(t, rvalid, roff, n, &drv, &o3));
  AG_TRY(upload_bitmap(t, rdata, roff, n, &drd, &o4));
  OutBitmap ov, od;
  AG_TRY(ov.stage(t, out_valid, ooff, n));
  AG_TRY(od.stage(t, out_data, ooff, n));
  AG_TRY(kleene_dev(kop, dlv, dld, o2, drv, drd, o4, ov.d, od.d, ov.doff, n, cs));
  AG_TRY(ov.fetch(cs));
  AG_TRY(od.fetch(cs));
  return sync(cs);
}

// ---- filter / take -----------------------------------------------------------------
ag_status ag_filter_output_size(const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n, int null_selection, int64_t* out_len) {
  AG_TRY(ensure_init());
  if (!out_len) AG_FAIL(AG_ERR_INVALID, "filter_output_size: NULL result");
  *out_len = 0;
  if (n < 0 || moff < 0) AG_FAIL(AG_ERR_INVALID, "filter_output_size: negative length or offset");
  if (n == 0) return AG_OK;
  if (!mask) AG_FAIL(AG_ERR_INVALID, "filter_output_size: NULL mask");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  uint8_t *dm, *dmv; int64_t o1, o2; int64_t* d_len;
  AG_TRY(upload_bitmap(t, mask, moff, n, &dm, &o1));
  AG_TRY(upload_bitmap(t, mvalid, moff, n, &dmv, &o2));
  AG_TRY(t.alloc_t(&d_len, sizeof(int64_t)));
  AG_TRY(filter_output_size_dev(dm, dmv, o1, n, null_selection, d_len, cs));
  AG_TRY(d2h(out_len, d_len, sizeof(int64_t), cs));
  return sync(cs);
}

ag_status ag_filter_primitive(int bit_width, const void* vals, const uint8_t* vvalid, int64_t voff,
                              const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n, int null_selection,
                              void* out, uint8_t* out_valid, int64_t* out_len, int64_t* out_nulls) {
  AG_TRY(ensure_init());
  if (!out_len) AG_FAIL(AG_ERR_INVALID, "filter: NULL out_len");
  *out_len = 0;
  if (out_nulls) *out_nulls = 0;
  if (n < 0 || moff < 0 || voff < 0) AG_FAIL(AG_ERR_INVALID, "filter: negative length or offset");
  if (bit_width != 1 && bit_width != 8 && bit_width != 16 && bit_width != 32 && bit_width != 64) AG_FAIL(AG_ERR_TYPE, "filter: invalid values bit width %d", bit_width);
  if (n == 0) return AG_OK;
  if (!vals || !mask) AG_FAIL(AG_ERR_INVALID, "filter: NULL values/mask");
  if (bit_width == 1) {  // boolean values: bitmap in, bitmap out
    CallStream cs; AG_TRY(cs.acquire());
    Temps t(cs);
    uint8_t *dm, *dmv, *dvv, *dvd; int64_t om, omv, ovv, ovd; int64_t* d_len;
    AG_TRY(upload_bitmap(t, mask, moff, n, &dm, &om));
    AG_TRY(upload_bitmap(t, mvalid, moff, n, &dmv, &omv));
    AG_TRY(upload_bitmap(t, (const uint8_t*)vals, voff, n, &dvd, &ovd));
    AG_TRY(upload_bitmap(t, vvalid, voff, n, &dvv, &ovv));
    AG_TRY(t.alloc_t(&d_len, 2 * sizeof(int64_t)));
    AG_TRY(filter_output_size_dev(dm, dmv, om, n, null_selection, d_len, cs));
    int64_t len = 0;
    AG_TRY(d2h(&len, d_len, sizeof(int64_t), cs));
    AG_TRY(sync(cs));
    uint8_t *dout, *dov = nullptr;
    AG_TRY(t.alloc_t(&dout, (size_t)((len + 31) / 32) * 4));
    if (out_valid) AG_TRY(t.alloc_t(&dov, (size_t)((len + 31) / 32) * 4));
    // values bitmap and its validity share the row numbering: both copies keep phase voff & 7
    AG_TRY(filter_primitive_dev(1, dvd, dvv, ovd, dm, dmv, om, n, null_selection, dout, dov, len, d_len + 1, cs));
    AG_TRY(d2h(out, dout, (size_t)((len + 7) / 8), cs));
    AG_TRY(fetch_validity(out_valid, dov, len, out_nulls, d_len, cs));
    *out_len = len;
    return AG_OK;
  }
  const int w = bit_width / 8;
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  uint8_t *dm, *dmv, *dvv; int64_t om, omv, ovv; int64_t* d_len;
  AG_TRY(upload_bitmap(t, mask, moff, n, &dm, &om));
  AG_TRY(upload_bitmap(t, mvalid, moff, n, &dmv, &omv));
  AG_TRY(t.alloc_t(&d_len, 2 * sizeof(int64_t)));
  // pass 1 over the mask (getFilterOutputSize) while the values are still in flight
  AG_TRY(filter_output_size_dev(dm, dmv, om, n, null_selection, d_len, cs));
  int64_t len = 0;
  AG_TRY(d2h(&len, d_len, sizeof(int64_t), cs));
  const void* dv;
  AG_TRY(upload_column(t, vals, vvalid, voff, n, w, &dv, &dvv, &ovv));
  AG_TRY(sync(cs));
  void* dout; AG_TRY(t.alloc(&dout, (size_t)len * w));
  uint8_t* dov = nullptr;
  if (out_valid) AG_TRY(t.alloc_t(&dov, (size_t)((len + 31) / 32) * 4));
  AG_TRY(filter_primitive_dev(bit_width, dv, dvv, ovv, dm, dmv, om, n, null_selection, dout, dov, len, d_len + 1, cs));
  AG_TRY(d2h(out, dout, (size_t)len * w, cs));
  AG_TRY(fetch_validity(out_valid, dov, len, out_nulls, d_len, cs));
  *out_len = len;
  return AG_OK;
}

ag_status ag_take_indices(int index_width, const uint8_t* mask, const uint8_t* mvalid, int64_t moff, int64_t n,
                          int null_selection, void* out_idx, uint8_t* out_valid, int64_t* out_len) {
  AG_TRY(ensure_init());
  if (!out_len) AG_FAIL(AG_ERR_INVALID, "take_indices: NULL out_len");
  *out_len = 0;
  if (n < 0 || moff < 0) AG_FAIL(AG_ERR_INVALID, "take_indices: negative length or offset");
  if (index_width != 16 && index_width != 32) AG_FAIL(AG_ERR_TYPE, "take_indices: index width must be 16 or 32");
  if (n == 0) return AG_OK;
  if (!mask) AG_FAIL(AG_ERR_INVALID, "take_indices: NULL mask");
  const int w = index_width / 8;
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  uint8_t *dm, *dmv; int64_t om, omv; int64_t* d_len;
  AG_TRY(upload_bitmap(t, mask, moff, n, &dm, &om));
  AG_TRY(upload_bitmap(t, mvalid, moff, n, &dmv, &omv));
  AG_TRY(t.alloc_t(&d_len, 2 * sizeof(int64_t)));
  AG_TRY(filter_output_size_dev(dm, dmv, om, n, null_selection, d_len, cs));
  int64_t len = 0;
  AG_TRY(d2h(&len, d_len, sizeof(int64_t), cs));
  AG_TRY(sync(cs));
  void* dout; AG_TRY(t.alloc(&dout, (size_t)len * w));
  uint8_t* dov = nullptr;
  if (out_valid) AG_TRY(t.alloc_t(&dov, (size_t)((len + 31) / 32) * 4));
  AG_TRY(take_indices_dev(index_width, dm, dmv, om, n, null_selection, dout, dov, len, d_len + 1, cs));
  AG_TRY(d2h(out_idx, dout, (size_t)len * w, cs));
  if (out_valid) AG_TRY(d2h(out_valid, dov, (size_t)((len + 7) / 8), cs));
  AG_TRY(sync(cs));
  *out_len = len;
  return AG_OK;
}

ag_status ag_take_primitive(int bit_width, const void* vals, const uint8_t* vvalid, int64_t voff, int64_t vlen,
                            int idx_width, int idx_signed, const void* idx, const uint8_t* ivalid, int64_t ioff,
                            int64_t n, int bounds_check, void* out, uint8_t* out_valid,
                            int64_t* out_nulls, int64_t* bad_pos, int64_t* bad_index) {
  AG_TRY(ensure_init());
  if (bad_pos) *bad_pos = AG_NO_ERROR_POS;
  if (out_nulls) *out_nulls = 0;
  if (n < 0 || voff < 0 || ioff < 0 || vlen < 0) AG_FAIL(AG_ERR_INVALID, "take: negative length or offset");
  if (bit_width != 1 && bit_width != 8 && bit_width != 16 && bit_width != 32 && bit_width != 64) AG_FAIL(AG_ERR_INVALID, "take: invalid values byte width for take");
  if (idx_width != 8 && idx_width != 16 && idx_width != 32 && idx_width != 64) AG_FAIL(AG_ERR_INDEX, "take: invalid indices byte width");
  if (n == 0) return AG_OK;
  if (!idx || !out) AG_FAIL(AG_ERR_INVALID, "take: NULL indices/output");
  const bool is_bool = bit_width == 1;
  const int w = is_bool ? 0 : bit_width / 8, iw = idx_width / 8;
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  const void* dv; void *di, *dout; uint8_t *dvv, *div; int64_t ovv, oiv; int64_t* d_word;
  if (is_bool) {
    // the values bitmap keeps its phase voff & 7 and is not rebased; the kernel takes that phase from ovv
    uint8_t* dvb; int64_t ovb;
    AG_TRY(upload_bitmap(t, (const uint8_t*)vals, voff, vlen, &dvb, &ovb));
    AG_TRY(upload_bitmap(t, vvalid, voff, vlen, &dvv, &ovv));
    if (!vvalid) ovv = voff & 7;
    dv = dvb;
  } else {
    AG_TRY(upload_column(t, vals, vvalid, voff, vlen, w, &dv, &dvv, &ovv));
  }
  AG_TRY(t.alloc(&di, (size_t)n * iw));
  AG_TRY(h2d(di, idx, (size_t)n * iw, cs));
  AG_TRY(upload_bitmap(t, ivalid, ioff, n, &div, &oiv));
  AG_TRY(t.alloc(&dout, is_bool ? (size_t)((n + 31) / 32) * 4 : (size_t)n * w));
  uint8_t* dov = nullptr;
  if (out_valid) AG_TRY(t.alloc_t(&dov, (size_t)((n + 31) / 32) * 4));
  AG_TRY(t.alloc_t(&d_word, 2 * sizeof(int64_t)));
  AG_TRY(error_word_reset(d_word, cs));
  AG_TRY(take_primitive_dev(bit_width, dv, dvv, ovv, vlen, idx_width, idx_signed, di, div, oiv, n,
                            bounds_check, dout, dov, d_word, cs));
  int64_t bad = AG_NO_ERROR_POS;
  AG_TRY(d2h(&bad, d_word, sizeof(int64_t), cs));
  AG_TRY(sync(cs));
  if (bad != AG_NO_ERROR_POS) {
    if (bad_pos) *bad_pos = bad;
    return index_bounds_error(idx, idx_width, idx_signed, bad, bad_index);
  }
  AG_TRY(d2h(out, dout, is_bool ? (size_t)((n + 7) / 8) : (size_t)n * w, cs));
  return fetch_validity(out_valid, dov, n, out_nulls, d_word + 1, cs);
}

ag_status ag_sort_indices(int type, const void* vals, const uint8_t* valid, int64_t offset, int64_t n, int order,
                          int null_placement, uint64_t* out, int64_t* null_count, int64_t* nan_count) {
  AG_TRY(ensure_init());
  if (null_count) *null_count = 0;
  if (nan_count) *nan_count = 0;
  const int w = type_width(type);
  if (w == 0) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "sort_indices: unsupported type id %d (fixed-width numeric columns only)", type);
  if (n < 0 || offset < 0) AG_FAIL(AG_ERR_INVALID, "sort_indices: negative length or offset");
  if (n == 0) return AG_OK;
  if (!vals || !out) AG_FAIL(AG_ERR_INVALID, "sort_indices: NULL values/output");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  const void* dv; uint8_t* dvalid; int64_t ov; uint64_t* dout;
  AG_TRY(upload_column(t, vals, valid, offset, n, w, &dv, &dvalid, &ov));
  AG_TRY(t.alloc_t(&dout, (size_t)n * 8));
  AG_TRY(sort_indices_dev(type, dv, dvalid, ov, n, order, null_placement, dout, null_count, nan_count, cs));
  AG_TRY(d2h(out, dout, (size_t)n * 8, cs));
  return sync(cs);
}

ag_status ag_sort_indices_keys(int nkeys, const ag_sort_key* keys, int64_t n, uint64_t* out) {
  AG_TRY(ensure_init());
  AG_TRY(sort_indices_keys_check(nkeys, keys, n));
  if (n == 0) return AG_OK;
  if (!out) AG_FAIL(AG_ERR_INVALID, "sort_indices: NULL output");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  std::vector<ag_sort_key> dkeys(keys, keys + nkeys);
  std::vector<std::vector<ag_sort_chunk>> dchunks(nkeys);
  for (int j = 0; j < nkeys; ++j) {
    dchunks[j].resize(keys[j].nchunks);
    for (int c = 0; c < keys[j].nchunks; ++c) AG_TRY(upload_chunk(t, keys[j].type, keys[j].chunks[c], &dchunks[j][c]));
    dkeys[j].chunks = dchunks[j].data();
  }
  uint64_t* dout;
  AG_TRY(t.alloc_t(&dout, (size_t)n * 8));
  AG_TRY(sort_indices_keys_dev(nkeys, dkeys.data(), n, dout, cs));
  AG_TRY(d2h(out, dout, (size_t)n * 8, cs));
  return sync(cs);
}

ag_status ag_take_columns(int ncols, const ag_take_column* cols, int64_t nrows, int idx_width, int idx_signed, const void* idx,
                          const uint8_t* idx_valid, int64_t idx_offset, int64_t n, int bounds_check, int64_t* bad_pos, int64_t* bad_index) {
  AG_TRY(ensure_init());
  if (bad_pos) *bad_pos = AG_NO_ERROR_POS;
  AG_TRY(take_columns_check(ncols, cols, nrows, idx_width, idx_offset, n));
  if (n == 0) return AG_OK;
  if (!idx) AG_FAIL(AG_ERR_INVALID, "take_columns: NULL indices");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  const size_t words = (size_t)((n + 31) / 32) * 4;
  std::vector<ag_take_column> dcols(cols, cols + ncols);
  std::vector<std::vector<ag_sort_chunk>> dchunks(ncols);
  for (int j = 0; j < ncols; ++j) {
    dchunks[j].resize(cols[j].nchunks);
    for (int c = 0; c < cols[j].nchunks; ++c) AG_TRY(upload_chunk(t, cols[j].type, cols[j].chunks[c], &dchunks[j][c]));
    dcols[j].chunks = dchunks[j].data();
    AG_TRY(t.alloc(&dcols[j].out, cols[j].type == AG_TYPE_BOOL ? words : (size_t)n * type_width(cols[j].type)));
    dcols[j].out_valid = nullptr;
    if (cols[j].out_valid) AG_TRY(t.alloc_t(&dcols[j].out_valid, words));
  }
  const int iw = idx_width / 8;
  void* di;
  uint8_t* div;
  int64_t oiv;
  int64_t* d_word;
  AG_TRY(t.alloc(&di, (size_t)n * iw));
  AG_TRY(h2d(di, idx, (size_t)n * iw, cs));
  AG_TRY(upload_bitmap(t, idx_valid, idx_offset, n, &div, &oiv));
  AG_TRY(t.alloc_t(&d_word, sizeof(int64_t)));
  AG_TRY(error_word_reset(d_word, cs));
  AG_TRY(take_columns_dev(ncols, dcols.data(), nrows, idx_width, idx_signed, di, div, oiv, n, bounds_check, d_word, cs));
  int64_t bad = AG_NO_ERROR_POS;
  AG_TRY(d2h(&bad, d_word, sizeof(int64_t), cs));
  AG_TRY(sync(cs));
  if (bad != AG_NO_ERROR_POS) {
    if (bad_pos) *bad_pos = bad;
    return index_bounds_error(idx, idx_width, idx_signed, bad, bad_index);
  }
  for (int j = 0; j < ncols; ++j) {
    const bool is_bool = cols[j].type == AG_TYPE_BOOL;
    AG_TRY(d2h(cols[j].out, dcols[j].out, is_bool ? (size_t)((n + 7) / 8) : (size_t)n * type_width(cols[j].type), cs));
    if (cols[j].out_valid) AG_TRY(d2h(cols[j].out_valid, dcols[j].out_valid, (size_t)((n + 7) / 8), cs));
  }
  return sync(cs);
}

// The program's spans staged chunk by chunk (upload_chunk); the output is fetched only when no row failed.
ag_status ag_eval_program(const ag_expr_program* prog, int64_t n_spans, const ag_sort_chunk* spans, void* out, uint8_t* out_valid,
                          int64_t* first_bad) {
  AG_TRY(ensure_init());
  if (first_bad) *first_bad = AG_NO_ERROR_POS;
  AG_TRY(eval_program_check(prog, n_spans, spans));
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  const int nc = prog->n_cols;
  std::vector<ag_sort_chunk> dspans((size_t)(n_spans * nc));
  int64_t rows = 0;
  for (int64_t i = 0; i < n_spans && nc > 0; ++i) {
    rows += spans[i * nc].length > 0 ? spans[i * nc].length : 0;
    for (int j = 0; j < nc; ++j) {
      AG_TRY(upload_chunk(t, prog->col_types[j], spans[i * nc + j], &dspans[i * nc + j]));
    }
  }
  const size_t words = (size_t)((rows + 31) / 32) * 4;
  void* dout = nullptr;
  uint8_t* dvalid = nullptr;
  int64_t* d_word;
  AG_TRY(t.alloc(&dout, (size_t)rows * 8));   // room for any output type
  if (out_valid) AG_TRY(t.alloc_t(&dvalid, words));
  AG_TRY(t.alloc_t(&d_word, sizeof(int64_t)));
  AG_TRY(error_word_reset(d_word, cs));
  AG_TRY(eval_program_dev(prog, n_spans, dspans.data(), dout, dvalid, d_word, cs));
  if (rows == 0) return sync(cs);
  int64_t bad = AG_NO_ERROR_POS;
  AG_TRY(d2h(&bad, d_word, sizeof(int64_t), cs));
  AG_TRY(sync(cs));
  if (bad != AG_NO_ERROR_POS) {
    if (first_bad) *first_bad = bad;
    AG_FAIL(AG_ERR_INVALID, "expression failed at row %lld", (long long)bad);
  }
  int out_type = AG_TYPE_NULL;   // a checked program's result type: out_type of the last instruction that wrote out_reg
  for (int i = 0; i < prog->n_instr; ++i) if (prog->instr[i].dst == prog->out_reg) out_type = prog->instr[i].out_type;
  AG_TRY(d2h(out, dout, out_type == AG_TYPE_BOOL ? (size_t)((rows + 7) / 8) : (size_t)rows * type_width(out_type), cs));
  if (out_valid) AG_TRY(d2h(out_valid, dvalid, (size_t)((rows + 7) / 8), cs));
  return sync(cs);
}

ag_status ag_is_in(int bit_width, const void* vals, const uint8_t* valid, int64_t offset, int64_t n, const void* set_vals,
                   const uint8_t* set_valid, int64_t set_offset, int64_t set_n, int null_behavior, uint8_t* out_data, uint8_t* out_valid,
                   int64_t* out_nulls) {
  AG_TRY(ensure_init());
  if (out_nulls) *out_nulls = 0;
  if (bit_width != 8 && bit_width != 16 && bit_width != 32 && bit_width != 64) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "is_in: fixed-width values of 1/2/4/8 bytes only");
  if (n < 0 || set_n < 0 || offset < 0 || set_offset < 0) AG_FAIL(AG_ERR_INVALID, "is_in: negative length or offset");
  if (n == 0) return AG_OK;
  if (!vals || !out_data || (set_n > 0 && !set_vals)) AG_FAIL(AG_ERR_INVALID, "is_in: NULL values / value set / output");
  const int w = bit_width / 8;
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  const void *dv, *ds = nullptr; uint8_t *dvv, *dsv = nullptr, *dod, *dov; int64_t ov, os = 0; int64_t* d_nulls;
  AG_TRY(upload_column(t, vals, valid, offset, n, w, &dv, &dvv, &ov));
  if (set_n > 0) AG_TRY(upload_column(t, set_vals, set_valid, set_offset, set_n, w, &ds, &dsv, &os));
  const size_t bm = (size_t)((n + 31) / 32) * 4;
  AG_TRY(t.alloc_t(&dod, bm));
  AG_TRY(t.alloc_t(&dov, bm));
  AG_TRY(t.alloc_t(&d_nulls, 8));
  AG_TRY(is_in_dev(bit_width, dv, dvv, ov, n, ds, dsv, os, set_n, null_behavior, dod,
                   out_valid ? dov : nullptr, d_nulls, cs));
  AG_TRY(d2h(out_data, dod, (size_t)((n + 7) / 8), cs));
  if (out_valid) AG_TRY(d2h(out_valid, dov, (size_t)((n + 7) / 8), cs));
  int64_t nulls = 0;
  AG_TRY(d2h(&nulls, d_nulls, 8, cs));
  AG_TRY(sync(cs));
  if (out_nulls) *out_nulls = nulls;
  return AG_OK;
}

ag_status ag_unique(int bit_width, const void* vals, const uint8_t* valid, int64_t offset, int64_t n, void* out, uint8_t* out_valid,
                    int64_t* out_len, int64_t* out_nulls) {
  AG_TRY(ensure_init());
  if (!out_len) AG_FAIL(AG_ERR_INVALID, "unique: NULL out_len");
  *out_len = 0;
  if (out_nulls) *out_nulls = 0;
  if (bit_width != 8 && bit_width != 16 && bit_width != 32 && bit_width != 64) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "unique: fixed-width values of 1/2/4/8 bytes only");
  if (n < 0 || offset < 0) AG_FAIL(AG_ERR_INVALID, "unique: negative length or offset");
  if (n == 0) return AG_OK;
  if (!vals || !out) AG_FAIL(AG_ERR_INVALID, "unique: NULL values/output");
  if (valid && !out_valid) AG_FAIL(AG_ERR_INVALID, "unique: an input with a validity bitmap needs an output validity bitmap");
  const int w = bit_width / 8;
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  const void* dv; void* dout; uint8_t *dvv, *dov = nullptr; int64_t ov; int64_t* d_len;
  AG_TRY(upload_column(t, vals, valid, offset, n, w, &dv, &dvv, &ov));
  AG_TRY(t.alloc(&dout, (size_t)n * w));
  if (valid) AG_TRY(t.alloc_t(&dov, (size_t)((n + 31) / 32) * 4));
  AG_TRY(t.alloc_t(&d_len, 16));
  AG_TRY(unique_dev(bit_width, dv, dvv, ov, n, dout, dov, n, d_len, cs));
  int64_t len = 0;
  AG_TRY(d2h(&len, d_len, 8, cs));
  AG_TRY(sync(cs));
  AG_TRY(d2h(out, dout, (size_t)len * w, cs));
  AG_TRY(fetch_validity(dov ? out_valid : nullptr, dov, len, out_nulls, d_len + 1, cs));
  *out_len = len;
  return AG_OK;
}

ag_status ag_dictionary_encode(int bit_width, const ag_dict_chunk* chunks, int64_t n_chunks, int null_encoding, void* dict,
                               uint8_t* dict_valid, int64_t* counts) {
  AG_TRY(ensure_init());
  if (!counts) AG_FAIL(AG_ERR_INVALID, "dictionary_encode: NULL counts");
  if (n_chunks < 0 || (n_chunks > 0 && !chunks)) AG_FAIL(AG_ERR_INVALID, "dictionary_encode: bad chunk table");
  if (bit_width != 8 && bit_width != 16 && bit_width != 32 && bit_width != 64)
    AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "dictionary_encode: fixed-width values of 1/2/4/8 bytes only (got %d bits)", bit_width);
  for (int64_t c = 0; c < n_chunks; ++c)
    if (chunks[c].length < 0 || chunks[c].offset < 0) AG_FAIL(AG_ERR_INVALID, "dictionary_encode: chunk %lld: negative length or offset", (long long)c);
  const int w = bit_width / 8;
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  // device copies of the chunks: values rebased to the validity's bit phase, outputs at offset 0
  std::vector<ag_dict_chunk> dc((size_t)n_chunks);
  int64_t total = 0;
  for (int64_t c = 0; c < n_chunks; ++c) {
    const ag_dict_chunk& h = chunks[c];
    ag_dict_chunk& d = dc[(size_t)c];
    d = ag_dict_chunk{nullptr, nullptr, 0, h.length, nullptr, nullptr};
    total += h.length;
    if (h.length == 0) continue;
    if (!h.values || !h.indices) AG_FAIL(AG_ERR_INVALID, "dictionary_encode: chunk %lld: NULL values or indices", (long long)c);
    uint8_t* dvalid;
    AG_TRY(upload_column(t, h.values, h.validity, h.offset, h.length, w, &d.values, &dvalid, &d.offset));
    d.validity = dvalid;
    AG_TRY(t.alloc_t(&d.indices, (size_t)h.length * 4));
    if (h.indices_validity) AG_TRY(t.alloc_t(&d.indices_validity, (size_t)((h.length + 31) / 32) * 4));
  }
  if (total > 0 && !dict) AG_FAIL(AG_ERR_INVALID, "dictionary_encode: NULL dictionary");
  void* ddict = nullptr; uint8_t* ddv = nullptr; int64_t* dcounts;
  if (total > 0) AG_TRY(t.alloc(&ddict, (size_t)total * w));
  if (dict_valid && total > 0) AG_TRY(t.alloc_t(&ddv, (size_t)((total + 7) / 8)));
  AG_TRY(t.alloc_t(&dcounts, (size_t)(n_chunks + 2) * 8));
  AG_TRY(dictionary_encode_dev(bit_width, dc.data(), n_chunks, null_encoding, ddict, ddv, dcounts, cs));
  AG_TRY(d2h(counts, dcounts, (size_t)(n_chunks + 2) * 8, cs));
  AG_TRY(sync(cs));
  const int64_t k = counts[0];
  AG_TRY(d2h(dict, ddict, (size_t)k * w, cs));
  if (ddv && null_encoding == AG_NULL_ENCODING_ENCODE) AG_TRY(d2h(dict_valid, ddv, (size_t)((k + 7) / 8), cs));
  for (int64_t c = 0; c < n_chunks; ++c) {
    const ag_dict_chunk& h = chunks[c];
    const ag_dict_chunk& d = dc[(size_t)c];
    if (h.length == 0) continue;
    AG_TRY(d2h(h.indices, d.indices, (size_t)h.length * 4, cs));
    if (null_encoding == AG_NULL_ENCODING_MASK && h.validity && h.indices_validity)
      AG_TRY(d2h(h.indices_validity, d.indices_validity, (size_t)((h.length + 7) / 8), cs));
  }
  return sync(cs);
}

// Stage a values column for the run-end kernels: rows [off, off+n) of `vals` (a bitmap for BOOL) and `valid`
// (upload_chunk).
static ag_status upload_values(Temps& t, int type, const void* vals, const uint8_t* valid, int64_t off, int64_t n, ag_sort_chunk* d) {
  if (type != AG_TYPE_BOOL && type_width(type) == 0) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "run_end: type id %d (boolean and the 10 numeric types only)", type);
  return upload_chunk(t, type, ag_sort_chunk{vals, valid, off, n}, d);
}
static int run_end_width(int run_end_type) {
  return run_end_type == AG_TYPE_INT16 ? 2 : (run_end_type == AG_TYPE_INT32 ? 4 : (run_end_type == AG_TYPE_INT64 ? 8 : 0));
}
static size_t value_bytes(int type, int64_t n) { return (size_t)(type == AG_TYPE_BOOL ? (n + 7) / 8 : n * type_width(type)); }
static size_t word_bytes(int64_t nbits) { return (size_t)((nbits + 31) / 32) * 4; }

ag_status ag_run_end_count(int type, const void* vals, const uint8_t* valid, int64_t offset, int64_t n, int64_t* counts) {
  AG_TRY(ensure_init());
  if (!counts) AG_FAIL(AG_ERR_INVALID, "run_end_count: NULL counts");
  counts[0] = counts[1] = 0;
  if (n < 0 || offset < 0) AG_FAIL(AG_ERR_INVALID, "run_end_count: negative length or offset");
  if (n == 0) return AG_OK;
  if (!vals) AG_FAIL(AG_ERR_INVALID, "run_end_count: NULL values");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  ag_sort_chunk v; int64_t* dc;
  AG_TRY(upload_values(t, type, vals, valid, offset, n, &v));
  AG_TRY(t.alloc_t(&dc, 16));
  AG_TRY(run_end_count_dev(type, v.vals, v.valid, v.offset, n, dc, cs));
  AG_TRY(d2h(counts, dc, 16, cs));
  return sync(cs);
}

ag_status ag_run_end_encode(int type, int run_end_type, const void* vals, const uint8_t* valid, int64_t offset, int64_t n,
                            void* run_ends, void* out, uint8_t* out_valid, int64_t capacity, int64_t* counts) {
  AG_TRY(ensure_init());
  if (!counts) AG_FAIL(AG_ERR_INVALID, "run_end_encode: NULL counts");
  counts[0] = counts[1] = 0;
  const int rw = run_end_width(run_end_type);
  if (rw == 0) AG_FAIL(AG_ERR_INVALID, "run_end_encode: bad run end type %d", run_end_type);
  if (n < 0 || offset < 0 || capacity < 0) AG_FAIL(AG_ERR_INVALID, "run_end_encode: negative length, offset or capacity");
  if (capacity > 0 && (!run_ends || !out)) AG_FAIL(AG_ERR_INVALID, "run_end_encode: NULL run_ends / values output");
  if (valid && capacity > 0 && !out_valid) AG_FAIL(AG_ERR_INVALID, "run_end_encode: an input with a validity bitmap needs an output validity bitmap");
  if (n > 0 && !vals) AG_FAIL(AG_ERR_INVALID, "run_end_encode: NULL values");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  ag_sort_chunk v{}; int64_t* dc;
  void *dre, *dout; uint8_t* dov = nullptr;
  if (n > 0) AG_TRY(upload_values(t, type, vals, valid, offset, n, &v));
  AG_TRY(t.alloc(&dre, (size_t)capacity * rw));
  AG_TRY(t.alloc(&dout, type == AG_TYPE_BOOL ? word_bytes(capacity) : value_bytes(type, capacity)));
  if (valid) AG_TRY(t.alloc_t(&dov, word_bytes(capacity)));
  AG_TRY(t.alloc_t(&dc, 16));
  AG_TRY(run_end_encode_dev(type, run_end_type, v.vals, v.valid, v.offset, n, dre, dout, dov, capacity, dc, cs));
  AG_TRY(d2h(counts, dc, 16, cs));
  AG_TRY(sync(cs));
  const int64_t runs = counts[0] < capacity ? counts[0] : capacity;
  AG_TRY(d2h(run_ends, dre, (size_t)runs * rw, cs));
  AG_TRY(d2h(out, dout, value_bytes(type, runs), cs));
  if (dov) AG_TRY(d2h(out_valid, dov, (size_t)((runs + 7) / 8), cs));
  return sync(cs);
}

ag_status ag_run_end_decode(int type, int run_end_type, const void* run_ends, int64_t n_runs, const void* vals, const uint8_t* valid,
                            int64_t values_offset, int64_t offset, int64_t length, void* out, uint8_t* out_valid, int64_t* null_count) {
  AG_TRY(ensure_init());
  if (null_count) *null_count = 0;
  const int rw = run_end_width(run_end_type);
  if (rw == 0) AG_FAIL(AG_ERR_INVALID, "run_end_decode: bad run end type %d", run_end_type);
  if (n_runs < 0 || values_offset < 0 || offset < 0 || length < 0) AG_FAIL(AG_ERR_INVALID, "run_end_decode: negative length or offset");
  if (length == 0) return AG_OK;
  if (!run_ends && n_runs > 0) AG_FAIL(AG_ERR_INVALID, "run_end_decode: NULL run_ends");
  if (!vals || !out) AG_FAIL(AG_ERR_INVALID, "run_end_decode: NULL values / output");
  if (valid && !out_valid) AG_FAIL(AG_ERR_INVALID, "run_end_decode: a values child with a validity bitmap needs an output validity bitmap");
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  void *dre, *dout, *z; ag_sort_chunk v{}; uint8_t *zv, *dov = nullptr; int64_t* dw;
  AG_TRY(t.alloc(&dre, (size_t)n_runs * rw));
  AG_TRY(h2d(dre, run_ends, (size_t)n_runs * rw, cs));
  if (n_runs > 0) AG_TRY(upload_values(t, type, vals, valid, values_offset, n_runs, &v));
  else { AG_TRY(t.alloc(&z, 8)); v.vals = z; }
  if (valid && !v.valid) { AG_TRY(t.alloc_t(&zv, 8)); v.valid = zv; }
  AG_TRY(t.alloc(&dout, type == AG_TYPE_BOOL ? word_bytes(length) : value_bytes(type, length)));
  if (valid) AG_TRY(t.alloc_t(&dov, word_bytes(length)));
  AG_TRY(t.alloc_t(&dw, 16));
  AG_TRY(error_word_reset(dw + 1, cs));
  AG_TRY(run_end_decode_dev(type, run_end_type, dre, n_runs, v.vals, v.valid, v.offset, offset, length, dout, dov, dw, dw + 1, cs));
  int64_t h[2];
  AG_TRY(d2h(h, dw, 16, cs));
  AG_TRY(sync(cs));
  if (h[1] != AG_NO_ERROR_POS)
    AG_FAIL(AG_ERR_INVALID, "run_end_decode: malformed run ends at run %lld (they must increase strictly and reach offset+length)", (long long)h[1]);
  AG_TRY(d2h(out, dout, value_bytes(type, length), cs));
  if (dov) AG_TRY(d2h(out_valid, dov, (size_t)((length + 7) / 8), cs));
  AG_TRY(sync(cs));
  if (null_count) *null_count = h[0];
  return AG_OK;
}

}  // extern "C"
