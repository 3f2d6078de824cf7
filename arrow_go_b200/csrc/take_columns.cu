// take_columns.cu — gather many chunked columns by one index vector in one launch (take on record batches and tables).
//
// Replaces the per-column loops of takeRecordImpl / takeTableImpl / FilterRecordBatch / FilterTable
// (arrow/compute/selection.go:117-204, 679-800), each column being ChunkedPrimitiveTake / PrimitiveTake
// (kernels/vector_selection.go:1162-1228) with the semantics of take_kernel (take.cu):
//     out[c][i]       = column c's row idx[i], rows numbered across its chunks
//     out_valid[c][i] = idxValid[i] ∧ columnValid[c][idx[i]]          (value 0 where it is clear)
// Only valid index slots are bounds-checked; an index is out of bounds when it is negative (signed types) or >= nrows
// once read as unsigned; the lowest offending row is lowered into *d_bad_pos with atomicMin.
//
// Layout: a block iteration covers 1024 consecutive rows, thread t handles rows t, t+256, t+512, t+768 (as in
// take_kernel), so a warp's rows of one step are 32 consecutive rows starting at a multiple of 32 and every output
// validity word (and BOOL value word) is one __ballot_sync.  Each thread loads its 4 indices once and checks them once.
// Columns are visited grouped by chunk layout (the lengths of their non-empty chunks): the chunk of each index is found
// once per distinct layout by a binary search over the layout's chunk starts (in shared memory when every layout's
// starts fit), then every column of the layout gathers with 4 loads in flight per thread.
//
// Bytes per output row: the index (1-8 B) once, then per column one gathered value (a 32 B sector for random indices
// into a column larger than L2), one value write and one validity bit.
#include "host_stage.cuh"

#include <algorithm>
#include <vector>

namespace ag {

constexpr int kTcThreads = 256;
constexpr int kTcUnroll = 4;
constexpr int kTcSmemStarts = 6144;   // 48 KB of int64 chunk starts: the dynamic shared memory a launch gets without opting in

struct TcChunk { const void* vals; const uint8_t* valid; int64_t offset; };
// One column: value width in bits (1 = BOOL), its layout, its first chunk in the chunk table.
struct TcColumn { int bits; int layout; int chunk0; void* out; uint32_t* out_valid; };
// One layout: nchunks non-empty chunks whose starts are starts[first .. first + nchunks] (the last one = nrows).
struct TcLayout { int first; int nchunks; };

struct TcParams {
  const TcColumn* cols;     // grouped by layout
  int ncols;
  const TcLayout* layouts;
  const TcChunk* chunks;
  const int64_t* starts;
  int nstarts;
  int starts_in_smem;
  unsigned long long nrows;
  const void* idx;
  const uint8_t* ivalid;
  int64_t ioff;
  int64_t n;
  int idx_signed;
  int bounds_check;
  long long* bad_pos;
};

// largest c in [0, nchunks) with starts[c] <= r  (chunks are non-empty, r < starts[nchunks])
__device__ __forceinline__ int tc_find_chunk(const int64_t* starts, int nchunks, int64_t r) {
  int lo = 0, hi = nchunks;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (starts[mid] <= r) lo = mid; else hi = mid;
  }
  return lo;
}

template <typename V>
__device__ __forceinline__ void tc_gather(const TcParams& p, const TcColumn& col, int64_t base, const int (&ch)[kTcUnroll],
                                          const int64_t (&loc)[kTcUnroll], const bool (&live)[kTcUnroll], int lane) {
  V v[kTcUnroll];
  bool ok[kTcUnroll];
#pragma unroll
  for (int k = 0; k < kTcUnroll; ++k) {
    v[k] = V(0);
    ok[k] = live[k];
    if (ok[k]) {
      const TcChunk c = p.chunks[col.chunk0 + ch[k]];
      const int64_t e = c.offset + loc[k];
      if (c.valid) ok[k] = bit_is_set(c.valid, e);
      if (ok[k]) v[k] = reinterpret_cast<const V*>(c.vals)[e];
    }
  }
  V* __restrict__ out = reinterpret_cast<V*>(col.out);
#pragma unroll
  for (int k = 0; k < kTcUnroll; ++k) {
    const int64_t i = base + k * kTcThreads + threadIdx.x;
    if (i < p.n) __stcs(out + i, v[k]);
    if (col.out_valid) {
      const int64_t w = (base + k * kTcThreads + (threadIdx.x & ~31)) >> 5;   // warp-uniform
      store_valid_word(col.out_valid, w, __ballot_sync(0xffffffffu, ok[k]), p.n, lane);
    }
  }
}

__device__ __forceinline__ void tc_gather_bool(const TcParams& p, const TcColumn& col, int64_t base, const int (&ch)[kTcUnroll],
                                               const int64_t (&loc)[kTcUnroll], const bool (&live)[kTcUnroll], int lane) {
  bool bit[kTcUnroll], ok[kTcUnroll];
#pragma unroll
  for (int k = 0; k < kTcUnroll; ++k) {
    bit[k] = false;
    ok[k] = live[k];
    if (ok[k]) {
      const TcChunk c = p.chunks[col.chunk0 + ch[k]];
      const int64_t e = c.offset + loc[k];
      if (c.valid) ok[k] = bit_is_set(c.valid, e);
      if (ok[k]) bit[k] = bit_is_set(reinterpret_cast<const uint8_t*>(c.vals), e);
    }
  }
  uint32_t* out = reinterpret_cast<uint32_t*>(col.out);
#pragma unroll
  for (int k = 0; k < kTcUnroll; ++k) {
    const int64_t w = (base + k * kTcThreads + (threadIdx.x & ~31)) >> 5;
    const uint32_t dbits = __ballot_sync(0xffffffffu, bit[k]);
    const uint32_t vbits = __ballot_sync(0xffffffffu, ok[k]);
    store_bool_words(out, col.out_valid, w, dbits, vbits, p.n, lane);
  }
}

template <typename I>
__global__ void __launch_bounds__(kTcThreads, 3)
take_columns_kernel(const TcParams p) {
  extern __shared__ int64_t s_starts[];
  const I* __restrict__ idx = reinterpret_cast<const I*>(p.idx);
  constexpr I kSignBit = (I)((I)1 << (sizeof(I) * 8 - 1));
  const int lane = threadIdx.x & 31;
  const int64_t* starts = p.starts;
  if (p.starts_in_smem) {
    for (int j = threadIdx.x; j < p.nstarts; j += kTcThreads) s_starts[j] = p.starts[j];
    __syncthreads();
    starts = s_starts;
  }
  const int64_t step = (int64_t)gridDim.x * kTcThreads * kTcUnroll;
  long long my_bad = AG_NO_ERROR_POS;
  for (int64_t base = (int64_t)blockIdx.x * kTcThreads * kTcUnroll; base < p.n; base += step) {
    int64_t row[kTcUnroll];
    bool live[kTcUnroll];   // the row exists, its index slot is valid and in bounds
#pragma unroll
    for (int k = 0; k < kTcUnroll; ++k) {
      const int64_t i = base + k * kTcThreads + threadIdx.x;
      live[k] = false;
      row[k] = 0;
      if (i < p.n) {
        const I ix = __ldcs(idx + i);
        live[k] = !p.ivalid || bit_is_set(p.ivalid, p.ioff + i);
        if (live[k]) {
          const bool oob = (p.idx_signed && (ix & kSignBit)) || (unsigned long long)ix >= p.nrows;   // take_index_oob
          if (oob) {
            live[k] = false;   // never dereferenced; with bounds_check the whole call fails anyway
            if (p.bounds_check && i < my_bad) my_bad = i;
          } else {
            row[k] = (int64_t)ix;
          }
        }
      }
    }
    int layout = -1;
    int ch[kTcUnroll] = {0, 0, 0, 0};
    int64_t loc[kTcUnroll] = {0, 0, 0, 0};
    for (int c = 0; c < p.ncols; ++c) {
      const TcColumn col = p.cols[c];
      if (col.layout != layout) {   // columns come grouped by layout: one search per distinct layout
        layout = col.layout;
        const TcLayout L = p.layouts[layout];
        const int64_t* st = starts + L.first;
#pragma unroll
        for (int k = 0; k < kTcUnroll; ++k) {
          ch[k] = live[k] ? tc_find_chunk(st, L.nchunks, row[k]) : 0;
          loc[k] = live[k] ? row[k] - st[ch[k]] : 0;
        }
      }
      switch (col.bits) {
        case 1: tc_gather_bool(p, col, base, ch, loc, live, lane); break;
        case 8: tc_gather<uint8_t>(p, col, base, ch, loc, live, lane); break;
        case 16: tc_gather<uint16_t>(p, col, base, ch, loc, live, lane); break;
        case 32: tc_gather<uint32_t>(p, col, base, ch, loc, live, lane); break;
        default: tc_gather<unsigned long long>(p, col, base, ch, loc, live, lane); break;
      }
    }
  }
  if (p.bounds_check) lower_error_row(my_bad, p.bad_pos);
}

static int tc_bits(int type) { return type == AG_TYPE_BOOL ? 1 : type_width(type) * 8; }

ag_status take_columns_check(int ncols, const ag_take_column* cols, int64_t nrows, int idx_width, int64_t idx_offset, int64_t n) {
  if (ncols < 0 || (ncols > 0 && !cols)) AG_FAIL(AG_ERR_INVALID, "take_columns: bad column list");
  if (nrows < 0 || n < 0 || idx_offset < 0) AG_FAIL(AG_ERR_INVALID, "take_columns: negative length or offset");
  if (idx_width != 8 && idx_width != 16 && idx_width != 32 && idx_width != 64) AG_FAIL(AG_ERR_INDEX, "take_columns: invalid indices byte width");
  for (int j = 0; j < ncols; ++j) {
    const ag_take_column& c = cols[j];
    if (c.type != AG_TYPE_BOOL && type_width(c.type) == 0)
      AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "take_columns: column %d: unsupported type id %d (boolean and numeric columns only)", j, c.type);
    AG_TRY(check_chunk_list("take_columns: column", j, c.nchunks, c.chunks, nrows, "row count"));
    if (n > 0 && !c.out) AG_FAIL(AG_ERR_INVALID, "take_columns: column %d: NULL output", j);
  }
  return AG_OK;
}

ag_status take_columns_dev(int ncols, const ag_take_column* cols, int64_t nrows, int idx_width, int idx_signed, const void* idx,
                           const uint8_t* idx_valid, int64_t idx_offset, int64_t n, int bounds_check, int64_t* d_bad_pos, cudaStream_t st) {
  AG_TRY(take_columns_check(ncols, cols, nrows, idx_width, idx_offset, n));
  if (n == 0 || (ncols == 0 && !bounds_check)) return AG_OK;
  if (!idx) AG_FAIL(AG_ERR_INVALID, "take_columns: NULL indices");
  if (bounds_check && !d_bad_pos) AG_FAIL(AG_ERR_INVALID, "take_columns: bounds_check needs an error word");
  for (int j = 0; j < ncols; ++j) {
    const ag_take_column& c = cols[j];
    bool nullable = idx_valid != nullptr;
    for (int k = 0; k < c.nchunks; ++k) nullable = nullable || (c.chunks[k].valid && c.chunks[k].length > 0);
    if (nullable && !c.out_valid) AG_FAIL(AG_ERR_INVALID, "take_columns: column %d may have nulls but no output validity buffer was given", j);
    if (c.out_valid && (reinterpret_cast<uintptr_t>(c.out_valid) & 3)) AG_FAIL(AG_ERR_INVALID, "take_columns: column %d: out_valid must be 4-byte aligned", j);
    if (c.type == AG_TYPE_BOOL && (reinterpret_cast<uintptr_t>(c.out) & 3)) AG_FAIL(AG_ERR_INVALID, "take_columns: column %d: boolean output bitmap must be 4-byte aligned", j);
  }
  // layouts (lengths of the non-empty chunks), chunk table and the column order grouped by layout (host only)
  std::vector<std::vector<int64_t>> lay_lens;
  std::vector<TcLayout> layouts;
  std::vector<int64_t> starts;
  std::vector<TcChunk> chunks;
  std::vector<TcColumn> tcols;
  for (int j = 0; j < ncols; ++j) {
    const ag_take_column& c = cols[j];
    std::vector<int64_t> lens;
    TcColumn tc{tc_bits(c.type), 0, (int)chunks.size(), c.out, reinterpret_cast<uint32_t*>(c.out_valid)};
    for (int k = 0; k < c.nchunks; ++k) {
      const ag_sort_chunk& ch = c.chunks[k];
      if (ch.length == 0) continue;
      lens.push_back(ch.length);
      chunks.push_back(TcChunk{ch.vals, ch.valid, ch.offset});
    }
    const auto it = std::find(lay_lens.begin(), lay_lens.end(), lens);
    if (it != lay_lens.end()) {
      tc.layout = (int)(it - lay_lens.begin());
    } else {
      tc.layout = (int)lay_lens.size();
      layouts.push_back(TcLayout{(int)starts.size(), (int)lens.size()});
      int64_t s = 0;
      for (int64_t l : lens) { starts.push_back(s); s += l; }
      starts.push_back(s);
      lay_lens.push_back(std::move(lens));
    }
    tcols.push_back(tc);
  }
  std::stable_sort(tcols.begin(), tcols.end(), [](const TcColumn& a, const TcColumn& b) { return a.layout < b.layout; });
  if (starts.size() > (size_t)INT32_MAX || chunks.size() > (size_t)INT32_MAX) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "take_columns: too many chunks");
  TableImage img(st);
  const size_t o_col = img.add(tcols), o_lay = img.add(layouts), o_ch = img.add(chunks), o_st = img.add(starts);
  AG_TRY(img.upload("take_columns tables"));
  TcParams p{};
  p.cols = img.at<const TcColumn>(o_col);
  p.ncols = (int)tcols.size();
  p.layouts = img.at<const TcLayout>(o_lay);
  p.chunks = img.at<const TcChunk>(o_ch);
  p.starts = img.at<const int64_t>(o_st);
  p.nstarts = (int)starts.size();
  p.starts_in_smem = p.nstarts <= kTcSmemStarts;
  p.nrows = (unsigned long long)nrows;
  p.idx = idx; p.ivalid = idx_valid; p.ioff = idx_offset; p.n = n;
  p.idx_signed = idx_signed; p.bounds_check = bounds_check;
  p.bad_pos = reinterpret_cast<long long*>(d_bad_pos);
  const size_t smem = p.starts_in_smem ? (size_t)p.nstarts * sizeof(int64_t) : 0;
  const int64_t need = (n + kTcThreads * kTcUnroll - 1) / (kTcThreads * kTcUnroll);
  return visit_width(idx_width, [&](auto tag) {
    const auto kernel = take_columns_kernel<typename decltype(tag)::type>;
    kernel<<<grid_one_wave(kernel, kTcThreads, need), kTcThreads, smem, st>>>(p);
    return check_launch("take_columns_kernel");
  }, [&] { AG_FAIL(AG_ERR_INDEX, "take_columns: invalid indices byte width"); });
}

}  // namespace ag

using namespace ag;

extern "C" ag_status ag_take_columns_dev(int ncols, const ag_take_column* cols, int64_t nrows, int idx_width, int idx_signed,
                                         const void* d_idx, const uint8_t* d_idx_valid, int64_t idx_offset, int64_t n,
                                         int bounds_check, int64_t* d_bad_pos, ag_stream_t s) {
  AG_TRY(ensure_init());
  return take_columns_dev(ncols, cols, nrows, idx_width, idx_signed, d_idx, d_idx_valid, idx_offset, n, bounds_check, d_bad_pos,
                          resolve_stream(s));
}
