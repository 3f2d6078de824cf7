// byte_array.cu — BYTE_ARRAY Parquet pages decoded on the device into an Arrow Binary / LargeBinary array (offsets plus
// one data buffer), for the four encodings a string column chunk uses:
//   PLAIN                     PlainByteArrayDecoder.Decode / DecodeSpaced (parquet/internal/encoding/byte_array_decoder.go:144-189)
//   PLAIN_ / RLE_DICTIONARY   dictDecoder over the RLE/bit-packed indices (decoder.go:125-160), as ag_parquet_dict_decode
//   DELTA_LENGTH_BYTE_ARRAY   DeltaLengthByteArrayDecoder.SetData / Decode (delta_length_byte_array.go:113-188)
//   DELTA_BYTE_ARRAY          DeltaByteArrayDecoder.SetData / Decode (delta_byte_array.go:166-303)
//
// Every value lives in a dense per-page array indexed d = tile_base[p] * 1024 + rank (so a page's values start on a
// 1024-value boundary).  Three stages:
//   1. Lengths per dense value (vlen, int64) and where its bytes start (vsrc):
//      - PLAIN: ba_plain_parse_kernel, one block per page, streams the page through the shared-memory window of
//        pq_window.cuh in spans of 1024 candidate starts.  Every candidate reads the 4-byte length it would have and its
//        next start; the chain of real values through the span is found by span_chain's pointer doubling (as
//        snappy_parse_kernel finds Snappy elements), and a block scan of the chain ranks the values.  A value longer
//        than the window moves the next span past it without loading it.
//      - dictionary: pq_runs_kernel + pq_expand_kernel<kIndex> write one int32 index per slot; the length is
//        dict_off[i+1] - dict_off[i].
//      - DELTA_LENGTH / DELTA: delta_walk_kernel and delta_values_kernel (pq_decode.cuh) decode every length of the
//        stream (DELTA: the prefix stream, then the suffix stream from its bytesRead()); ba_len_tiles_kernel (tile
//        sums) and ba_len_page_kernel check them, tile_sum_scan_kernel scans the tile sums per page, and
//        ba_len_write_kernel scans each tile into payload offsets and writes vlen / vsrc.
//   2. Offsets: ba_slot_kernel maps slots to dense ranks (spaced_rank, null slots get 0) and writes every slot's
//      length and source; ba_sum_kernel / ba_scan_kernel (segment_excl_scan) / ba_offsets_kernel scan the lengths over
//      all slots, decide on the device whether the int32 offsets overflow and whether the bytes fit `out_cap`, and
//      write the offsets at their width.
//   3. Bytes: ba_gather_kernel, a grid over 16-byte pieces of the output; each piece finds its slot by binary search
//      in the offsets.  DELTA_BYTE_ARRAY byte j of value k comes from the suffix of the last value m <= k with
//      prefix[m] <= j: ba_psv_kernel finds every value's previous smaller prefix through a tree of group minima, and
//      the gather follows that chain.
// Roofline.  encoded bytes read + offsets written + data written (+ dictionary bytes read).  This design also writes
// and reads 16 B per value (vlen, vsrc) and 24 B per slot of scratch.
#include <string.h>

#include <algorithm>
#include <vector>

#include "pq_decode.cuh"

namespace ag {

namespace {

constexpr int kBaThreads = kPqThreads;
constexpr int kPsvLevels = 7;               // group minima of 32^1 .. 32^7 values (pages hold < 2^31 values)

enum BaErr : int {
  kBaNone = 0,
  kBaEof = 1,              // PLAIN: a length prefix or a value cut off
  kBaNegPlain = 2,         // PLAIN: negative length
  kBaLenStream = 3,        // DELTA_LENGTH lengths / DELTA suffix lengths: a DELTA_BINARY_PACKED error (DeltaPage)
  kBaPrefixStream = 4,     // DELTA prefix lengths: a DELTA_BINARY_PACKED error (DeltaPage)
  kBaNegLen = 5,           // arg = the length
  kBaExceed = 6,
  kBaCount = 7,            // prefix and suffix counts differ
  kBaFirstPrefix = 8,
  kBaBadPrefix = 9,        // arg = the prefix length
  kBaShort = 10,           // spaced: fewer values than valid slots
  kBaDict = 11,            // the index stream (PageState err)
};

struct BaPage {
  int64_t produced;        // dense values delivered
  int64_t slots;           // output slots written
  int64_t arg;
  int64_t first_neg;       // DELTA: lowest rank with a negative length (atomicMin); INT64_MAX if none
  int64_t first_badp;      // DELTA_BYTE_ARRAY: lowest rank whose prefix is invalid (atomicMin)
  int64_t payload;         // DELTA: absolute offset of the suffix / value bytes
  int32_t err;
  int32_t pad;
};

struct BaCtl {             // stage 2's decision, read by the gather and the host
  long long total;
  int write_offsets;       // 0: int32 offsets overflow
  int fits;                // 1: the bytes fit out_cap
  int decoded;             // 1: the pages were decoded (0: an argument check failed first)
  int pad;
};

struct BaArgs {
  const ag_pq_page* pages;
  const int64_t* tile_base;   // [n_pages + 1]
  int64_t n_pages, n_tiles, n_slots;
  const uint8_t* data;
  const uint8_t* valid;
  int64_t* tile_cnt;          // spaced: first dense rank of every tile
  BaPage* st;
  int64_t* vlen;              // dense
  int64_t* vsrc;              // dense: absolute source byte offset (data, or dict_data for a dictionary)
  const int32_t* pre;         // DELTA: prefix lengths (dense)
  const int32_t* suf;         // DELTA_LENGTH / DELTA: (suffix) lengths (dense)
  int64_t* psv;               // DELTA: previous value with a smaller prefix (dense index)
  int32_t* lv[kPsvLevels];    // DELTA: group minima of the prefix lengths
  int nlev;
  const DeltaPage* dps;       // DELTA: prefix stream pages
  const DeltaPage* dls;       // DELTA_LENGTH lengths / DELTA suffix stream pages
  const PageState* pqs;       // dictionary
  const int32_t* idx;         // dictionary: index per slot (-1: out of range)
  const void* doff;           // dictionary offsets, offset_width each
  int64_t* slen;              // per slot: length
  int64_t* ssrc;              // per slot: source offset (DELTA: dense index)
  int64_t* soff;              // per slot: exclusive offset, n_slots + 1
  int64_t* csum;              // per 1024-slot chunk of all slots: length sum, then its first offset
  BaCtl* ctl;
  int64_t* d_decoded;
  int kind;                   // AG_PQ_ENC_*
  int ow;
  int64_t offset_base, cap_rel;   // cap_rel: bytes of out_data usable from offset_base
  void* offsets;
  uint8_t* out;               // out_data + offset_base
  const uint8_t* src_base;    // data, or dict_data
};

__device__ __forceinline__ int64_t page_slots(const BaArgs& a, int64_t p, const ag_pq_page& pg, int64_t need, int64_t produced, int err) {
  return slots_written(a.valid, pg, a.tile_cnt, a.tile_base[p], a.tile_base[p + 1], need, produced, err == kBaShort);
}

__device__ __forceinline__ void finish_page(const BaArgs& a, int64_t p, int64_t produced, int64_t slots, int err, int64_t arg) {
  BaPage& s = a.st[p];
  s.produced = produced; s.slots = slots; s.err = err; s.arg = arg;
  if (a.d_decoded) a.d_decoded[p] = slots;
}

// ---------------------------------------------------------------- PLAIN ----
// one block per page: the length-prefixed chain, window by window
__global__ void __launch_bounds__(kBaThreads)
ba_plain_parse_kernel(BaArgs a) {
  __shared__ uint4 win[kWinVec];
  __shared__ uint16_t jmp[2][kSpan];
  __shared__ uint32_t reach[kSpan / 32];
  __shared__ int warp_tot[kBaThreads / 32];
  __shared__ int64_t s_pos, s_nval, s_fail, s_next;
  __shared__ int s_err, s_done;
  const int64_t p = blockIdx.x;
  const ag_pq_page pg = a.pages[p];
  const int tid = threadIdx.x;
  const int64_t need = a.valid ? scan_tile_ranks(a.tile_cnt, a.tile_base[p], a.tile_base[p + 1], warp_tot) : pg.num_values;
  const uint8_t* in = a.data + pg.data;
  const int64_t len = pg.len;
  const int64_t d0 = a.tile_base[p] * kTile;
  if (tid == 0) { s_pos = 0; s_nval = 0; s_next = len; s_err = kBaNone; s_done = need == 0; }
  const uint8_t* wb = reinterpret_cast<const uint8_t*>(win);
  const uintptr_t sbeg = reinterpret_cast<uintptr_t>(in);
  int64_t wlo = INT64_MIN / 2;
  while (true) {
    __syncthreads();
    if (s_done) break;
    const int64_t cur = s_pos;
    if ((cur + kSpan + 4 < len ? cur + kSpan + 4 : len) > wlo + kWinBytes) {
      const uintptr_t a0 = (sbeg + cur) & ~(uintptr_t)15;
      load_window(win, sbeg, sbeg + len, a0);
      wlo = (int64_t)a0 - (int64_t)sbeg;
    }
    // ---- the value that would start at each of this thread's positions ----
    uint32_t J[kPer];
    int64_t vl[kPer], nx[kPer];
    int bad[kPer];
    bool last[kPer];                                             // no next value inside the span
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const int q = tid * kPer + k;
      const int64_t i = cur + q;
      J[k] = kSpan; vl[k] = 0; nx[k] = len; bad[k] = kBaEof;
      if (i + 4 <= len) {
        const int64_t o = i - wlo;
        const int32_t L = (int32_t)((uint32_t)wb[o] | (uint32_t)wb[o + 1] << 8 | (uint32_t)wb[o + 2] << 16 | (uint32_t)wb[o + 3] << 24);
        vl[k] = L;
        if (L < 0) bad[k] = kBaNegPlain;
        else if ((int64_t)L > len - i - 4) bad[k] = kBaEof;
        else {
          bad[k] = kBaNone;
          nx[k] = i + 4 + L;
          if (q + 4 + (int64_t)L < kSpan && nx[k] < len) J[k] = (uint32_t)(q + 4 + L);
        }
      }
      last[k] = J[k] == kSpan;
      jmp[0][q] = (uint16_t)J[k];
    }
    if (tid == 0) s_fail = INT64_MAX;
    span_chain(J, jmp, reach);
    // ---- ranks, values, the first failing value, the next span ----
    int cnt = 0;
#pragma unroll
    for (int k = 0; k < kPer; ++k) cnt += (cur + tid * kPer + k < len && bit_on(reach, tid * kPer + k)) ? 1 : 0;
    int tot;
    const int ex = block_excl_scan(cnt, warp_tot, &tot);
    const int64_t n0 = s_nval;
    int rk = ex;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const int q = tid * kPer + k;
      if (cur + q >= len || !bit_on(reach, q)) continue;
      const int64_t rank = n0 + rk++;
      if (rank >= need) continue;
      if (bad[k] != kBaNone) {
        atomicMin((unsigned long long*)&s_fail, (unsigned long long)rank);   // its error is resolved below
        continue;
      }
      a.vlen[d0 + rank] = vl[k];
      a.vsrc[d0 + rank] = pg.data + cur + q + 4;
      if (last[k]) s_next = nx[k];                              // the chain's last value in the span
    }
    __syncthreads();
    if (tid == 0) {
      if (s_fail != INT64_MAX) {
        s_nval = s_fail; s_done = 1;
      } else {
        s_nval = n0 + tot;
        if (s_nval >= need) { s_nval = need; s_done = 1; }
        else if (s_next >= len) { s_fail = s_nval; s_done = 1; }  // the next length prefix is missing
        else s_pos = s_next;
      }
    }
    // the error of the failing value (every thread that saw it agrees on the rank)
    __syncthreads();
    if (s_fail != INT64_MAX) {
      rk = ex;
#pragma unroll
      for (int k = 0; k < kPer; ++k) {
        const int q = tid * kPer + k;
        if (cur + q >= len || !bit_on(reach, q)) continue;
        if (n0 + rk++ == s_fail) s_err = bad[k];
      }
      if (s_fail == n0 + tot && tid == 0) s_err = kBaEof;
    }
  }
  __syncthreads();
  if (tid == 0) {
    const int64_t produced = s_nval;
    const int err = produced < need ? (s_err != kBaNone ? s_err : kBaEof) : kBaNone;
    finish_page(a, p, produced, page_slots(a, p, pg, need, produced, err), err, 0);
  }
}

// ---------------------------------------------------------------- DELTA_LENGTH / DELTA ----
// One block per page: the page's stream errors, then (after the length tiles) its payload checks.  Runs twice:
// PHASE 0 before the tiles (stream errors, counts, payload start), PHASE 1 after them (negative / exceed, delivered).
struct LenTile { long long before_neg; long long neg; };   // per dense tile: the length sum before its first negative, that rank

template <int PHASE>
__global__ void __launch_bounds__(kBaThreads)
ba_len_page_kernel(BaArgs a, const LenTile* lt, const long long* tile_sum) {
  __shared__ int warp_tot[kBaThreads / 32];
  __shared__ long long warp_sum[kBaThreads / 32];
  const int64_t p = blockIdx.x;
  const ag_pq_page pg = a.pages[p];
  const int tid = threadIdx.x;
  const int64_t t0 = a.tile_base[p], t1 = a.tile_base[p + 1];
  BaPage& s = a.st[p];
  const DeltaPage dl = a.dls[p];
  const bool dba = a.kind == AG_PQ_ENC_DELTA_BYTE_ARRAY;
  if (PHASE == 0) {
    const int64_t need = a.valid ? scan_tile_ranks(a.tile_cnt, t0, t1, warp_tot) : pg.num_values;
    if (tid == 0) {
      int err = kBaNone;
      int64_t pre_end = 0;
      if (dba) {
        const DeltaPage dp = a.dps[p];
        if (dp.err != kDErrNone) err = kBaPrefixStream;
        pre_end = dp.end;
      }
      if (!err && dl.err != kDErrNone) err = kBaLenStream;
      s.produced = 0; s.slots = 0; s.arg = need;                 // arg: need, until phase 1
      s.first_neg = INT64_MAX; s.first_badp = INT64_MAX;
      s.payload = pg.data + pre_end + dl.end;
      s.err = err;
    }
    return;
  }
  // PHASE 1: the first failing length in order: lengths exceeding the payload before the first negative one, else
  // the first negative one
  long long run = 0, before = -1, negrank = INT64_MAX;
  for (int64_t t = t0; t < t1; t += kBaThreads) {
    const int64_t i = t + tid;
    const LenTile x = i < t1 ? lt[i] : LenTile{0, INT64_MAX};
    const long long sum = i < t1 ? tile_sum[i] : 0;
    const bool has = x.neg != INT64_MAX;
    // exclusive sum of the tile sums before each tile
    long long tot;
    const long long incl = block_incl_scan(sum, warp_sum, &tot);
    int any;
    block_excl_scan(has ? 1 : 0, warp_tot, &any);
    if (negrank == INT64_MAX && any) {
      // the first tile (in this chunk) with a negative length
      __shared__ long long s_neg, s_before;
      if (tid == 0) s_neg = INT64_MAX;
      __syncthreads();
      if (has) atomicMin((unsigned long long*)&s_neg, (unsigned long long)x.neg);
      __syncthreads();
      if (has && x.neg == s_neg) s_before = run + incl - sum + x.before_neg;
      __syncthreads();
      negrank = s_neg; before = s_before;
    }
    run += tot;
  }
  if (tid == 0 && s.err == kBaNone) {
    const int64_t total = (int64_t)dl.produced;                  // every length of the stream
    const long long payload_len = pg.data + pg.len - s.payload;
    const long long upto = negrank == INT64_MAX ? run : before;  // sum of the lengths before the first negative one
    int err = kBaNone;
    int64_t arg = 0;
    if (upto > payload_len) err = kBaExceed;
    else if (negrank != INT64_MAX) { err = kBaNegLen; arg = a.suf[t0 * kTile + negrank]; }
    else if (dba && (int64_t)a.dps[p].produced != total) err = kBaCount;
    const int64_t need = s.arg;
    int64_t produced = 0;
    if (!err) {
      // Decode's prefix checks come before DecodeSpaced's count check
      produced = need < total ? need : total;
      const int64_t bp = dba ? s.first_badp : INT64_MAX;
      if (bp < produced) { err = bp == 0 ? kBaFirstPrefix : kBaBadPrefix; arg = a.pre[t0 * kTile + bp]; produced = bp; }
      else if (a.valid && total < need) { err = kBaShort; produced = 0; }
    }
    s.err = err;
    finish_page(a, p, produced, page_slots(a, p, pg, need, produced, err), err, arg);
  } else if (tid == 0) {
    finish_page(a, p, 0, page_slots(a, p, pg, s.arg, 0, s.err), s.err, 0);
  }
}

// one block per dense tile: the tile's length sum (into tile_sum), its first negative length, the sum before it;
// DELTA: the first invalid prefix length (value k needs 0 <= prefix[k] <= length[k-1], and prefix[0] == 0)
__global__ void __launch_bounds__(kBaThreads)
ba_len_tiles_kernel(BaArgs a, LenTile* lt, long long* tile_sum) {
  __shared__ long long warp_sum[kBaThreads / 32];
  __shared__ unsigned long long s_neg;
  const int64_t tile = blockIdx.x;
  const int64_t p = find_page(a.tile_base, a.n_pages, tile);
  const int64_t r0 = (tile - a.tile_base[p]) * kTile, d0 = a.tile_base[p] * kTile;
  const int64_t total = (int64_t)a.dls[p].produced;
  const bool ok = a.st[p].err == kBaNone;
  const int tid = threadIdx.x;
  if (tid == 0) s_neg = INT64_MAX;
  __syncthreads();
  long long sum = 0;
  int64_t bp = INT64_MAX;
  const bool dba = a.kind == AG_PQ_ENC_DELTA_BYTE_ARRAY;
#pragma unroll
  for (int q = 0; q < kTile / kBaThreads; ++q) {
    const int64_t r = r0 + q * kBaThreads + tid;
    if (!ok || r >= total) continue;
    const int32_t L = a.suf[d0 + r];
    sum += L;
    if (L < 0) atomicMin(&s_neg, (unsigned long long)r);
    if (dba && r < (int64_t)a.dps[p].produced) {
      const int32_t P = a.pre[d0 + r];
      bool badp;
      if (r == 0) badp = P != 0;
      else badp = P < 0 || (long long)P > (long long)a.pre[d0 + r - 1] + a.suf[d0 + r - 1];
      if (badp && bp == INT64_MAX) bp = r;
    }
  }
  if (bp != INT64_MAX) atomicMin((unsigned long long*)&a.st[p].first_badp, (unsigned long long)bp);
  long long tot;
  block_incl_scan(sum, warp_sum, &tot);
  // the sum before the tile's first negative length (a second pass over the tile, only when it has one)
  const unsigned long long neg = s_neg;
  long long before = 0;
  if (neg != INT64_MAX) {
    long long b = 0;
#pragma unroll
    for (int q = 0; q < kTile / kBaThreads; ++q) {
      const int64_t r = r0 + q * kBaThreads + tid;
      if (r < (int64_t)neg) b += a.suf[d0 + r];
    }
    long long bt;
    block_incl_scan(b, warp_sum, &bt);
    before = bt;
  }
  if (tid == 0) { lt[tile] = LenTile{before, (long long)neg}; tile_sum[tile] = tot; }
}

// one block per dense tile of a delivered page: the value lengths and where each value's (suffix) bytes start
__global__ void __launch_bounds__(kBaThreads)
ba_len_write_kernel(BaArgs a, const long long* tile_before) {
  __shared__ long long warp_sum[kBaThreads / 32];
  const int64_t tile = blockIdx.x;
  const int64_t p = find_page(a.tile_base, a.n_pages, tile);
  const BaPage s = a.st[p];
  const int64_t r0 = (tile - a.tile_base[p]) * kTile, d0 = a.tile_base[p] * kTile;
  if (r0 >= s.produced) return;                                  // block-uniform
  const int tid = threadIdx.x;
  const bool dba = a.kind == AG_PQ_ENC_DELTA_BYTE_ARRAY;
  long long carry = s.payload + tile_before[tile];
#pragma unroll
  for (int q = 0; q < kTile / kBaThreads; ++q) {
    const int64_t r = r0 + q * kBaThreads + tid;
    const long long L = r < s.produced ? a.suf[d0 + r] : 0;
    long long tot;
    const long long incl = block_incl_scan(L, warp_sum, &tot);
    if (r < s.produced) {
      a.vsrc[d0 + r] = carry + incl - L;
      a.vlen[d0 + r] = dba ? L + a.pre[d0 + r] : L;
    }
    carry += tot;
  }
}

// DELTA_BYTE_ARRAY: minima of the prefix lengths over groups of 32^(l+1) values; level 0 reads the prefixes
__global__ void __launch_bounds__(kBaThreads)
ba_min_kernel(const int32_t* in, int32_t* out, int64_t n_out) {
  const int64_t g = ((int64_t)blockIdx.x * kBaThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (g >= n_out) return;                                        // warp-uniform
  int32_t v = in[g * 32 + lane];
#pragma unroll
  for (int o = 16; o; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (lane == 0) out[g] = v;
}

// the minimum over entry e of level l (level -1 = the prefixes themselves)
__device__ __forceinline__ int32_t lvl_min(const BaArgs& a, int l, int64_t e) { return l < 0 ? a.pre[e] : a.lv[l][e]; }

// last m in [lo, k) with pre[m] < thr, or -1.  Entries at level l cover 32^(l+1) values; only groups that end before
// k are looked at, so no value at or after k (possibly never decoded) is read.
__device__ int64_t last_less(const BaArgs& a, int64_t lo, int64_t k, int32_t thr) {
  for (int l = -1; l < a.nlev; ++l) {
    const int sh = 5 * (l + 1);
    const int64_t e_hi = (k >> sh) - 1;
    const int64_t stop = l + 1 < a.nlev ? ((k >> sh) & ~(int64_t)31) : 0;
    for (int64_t e = e_hi; e >= stop; --e) {
      const int64_t start = e << sh, end = start + ((int64_t)1 << sh);
      if (end <= lo) return -1;
      if (lvl_min(a, l, e) >= thr) continue;
      // descend: the last child holding a value below thr and reaching past lo
      int ll = l;
      int64_t ee = e;
      while (ll >= 0) {
        int64_t c = ee * 32 + 31;
        const int csh = 5 * ll;
        for (; c >= ee * 32; --c) {
          if (((c + 1) << csh) <= lo) { c = -1; break; }
          if (lvl_min(a, ll - 1, c) < thr) break;
        }
        if (c < ee * 32) return -1;                             // only values before lo are below thr
        ee = c; --ll;
      }
      return ee >= lo ? ee : -1;
    }
  }
  return -1;
}

// one thread per delivered value with a non-zero prefix: its previous value with a smaller prefix
__global__ void __launch_bounds__(kBaThreads)
ba_psv_kernel(BaArgs a) {
  const int64_t tile = blockIdx.x;
  const int64_t p = find_page(a.tile_base, a.n_pages, tile);
  const int64_t produced = a.st[p].produced, d0 = a.tile_base[p] * kTile;
  for (int q = threadIdx.x; q < kTile; q += kBaThreads) {
    const int64_t r = (tile - a.tile_base[p]) * kTile + q;
    if (r == 0 || r >= produced) continue;
    const int32_t P = a.pre[d0 + r];
    if (P > 0) a.psv[d0 + r] = last_less(a, d0, d0 + r, P);
  }
}

// ---------------------------------------------------------------- slots, offsets, bytes ----
// dictionary pages: their PageState (runs kernel) becomes a BaPage
__global__ void ba_from_dict_kernel(BaArgs a) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.n_pages) return;
  const PageState s = a.pqs[p];
  BaPage& b = a.st[p];
  b.produced = s.produced; b.err = s.err != kErrNone ? kBaDict : kBaNone; b.arg = s.err;
  finish_page(a, p, s.produced, s.slots, b.err, s.err);
}

// one block per slot tile of a page: every written slot's length and source
template <bool SPACED, bool DICT>
__global__ void __launch_bounds__(kBaThreads)
ba_slot_kernel(BaArgs a) {
  __shared__ int warp_tot[kBaThreads / 32];
  const int64_t tile = blockIdx.x;
  const int64_t p = find_page(a.tile_base, a.n_pages, tile);
  const ag_pq_page pg = a.pages[p];
  const BaPage ps = a.st[p];
  const int64_t s0 = (tile - a.tile_base[p]) * kTile, d0 = a.tile_base[p] * kTile;
  if (s0 >= ps.slots) return;                                    // block-uniform
  const int tid = threadIdx.x;
  int64_t rank_base = SPACED ? a.tile_cnt[tile] : s0;
#pragma unroll
  for (int q = 0; q < kTile / kBaThreads; ++q) {
    const int64_t s = s0 + q * kBaThreads + tid;
    const bool in = s < ps.slots;
    bool v = in;
    int64_t rank = s;
    if (SPACED) rank = spaced_rank(in, a.valid, pg.out + s, warp_tot, rank_base, v);
    if (!in) continue;
    int64_t L = 0, src = 0;
    if (v) {
      if (DICT) {
        const int32_t i = a.idx[pg.out + s];
        if (i >= 0) {
          int64_t o0, o1;
          if (a.ow == 4) { o0 = reinterpret_cast<const int32_t*>(a.doff)[i]; o1 = reinterpret_cast<const int32_t*>(a.doff)[i + 1]; }
          else { o0 = reinterpret_cast<const int64_t*>(a.doff)[i]; o1 = reinterpret_cast<const int64_t*>(a.doff)[i + 1]; }
          L = o1 > o0 ? o1 - o0 : 0;
          src = o0;
        }
      } else {
        L = a.vlen[d0 + rank];
        src = a.kind == AG_PQ_ENC_DELTA_BYTE_ARRAY ? d0 + rank : a.vsrc[d0 + rank];
      }
    }
    a.slen[pg.out + s] = L;
    a.ssrc[pg.out + s] = src;
  }
}

// one block per 1024-slot chunk of all slots: the chunk's length sum
__global__ void __launch_bounds__(kBaThreads)
ba_sum_kernel(BaArgs a) {
  __shared__ long long warp_sum[kBaThreads / 32];
  const int64_t c = blockIdx.x;
  long long sum = 0;
#pragma unroll
  for (int q = 0; q < kTile / kBaThreads; ++q) {
    const int64_t i = c * kTile + q * kBaThreads + threadIdx.x;
    if (i < a.n_slots) sum += a.slen[i];
  }
  long long tot;
  block_incl_scan(sum, warp_sum, &tot);
  if (threadIdx.x == 0) a.csum[c] = tot;
}

// one block: chunk sums -> first offsets, the total, and the decisions
__global__ void __launch_bounds__(kBaThreads)
ba_scan_kernel(BaArgs a, int64_t n_chunks) {
  __shared__ long long warp_sum[kBaThreads / 32];
  const long long run = segment_excl_scan(a.csum, 0, n_chunks, warp_sum);
  if (threadIdx.x == 0) {
    BaCtl c;
    c.total = run;
    c.write_offsets = !(a.ow == 4 && a.offset_base + run > 0x7fffffffLL);
    c.fits = c.write_offsets && run <= a.cap_rel;
    c.decoded = 1;
    c.pad = 0;
    *a.ctl = c;
  }
}

// one block per chunk: the offsets at their width, and the int64 offsets the gather searches
__global__ void __launch_bounds__(kBaThreads)
ba_offsets_kernel(BaArgs a) {
  __shared__ long long warp_sum[kBaThreads / 32];
  const int64_t c = blockIdx.x;
  const BaCtl ctl = *a.ctl;
  long long carry = a.csum[c];
#pragma unroll
  for (int q = 0; q < kTile / kBaThreads; ++q) {
    const int64_t i = c * kTile + q * kBaThreads + threadIdx.x;
    const long long L = i < a.n_slots ? a.slen[i] : 0;
    long long tot;
    const long long incl = block_incl_scan(L, warp_sum, &tot);
    if (i < a.n_slots) {
      const long long o = carry + incl - L;
      a.soff[i] = o;
      if (ctl.write_offsets) {
        if (a.ow == 4) reinterpret_cast<int32_t*>(a.offsets)[i] = (int32_t)(a.offset_base + o);
        else reinterpret_cast<int64_t*>(a.offsets)[i] = a.offset_base + o;
      }
    }
    carry += tot;
  }
  if (c == 0 && threadIdx.x == 0) {
    a.soff[a.n_slots] = ctl.total;
    if (ctl.write_offsets) {
      if (a.ow == 4) reinterpret_cast<int32_t*>(a.offsets)[a.n_slots] = (int32_t)(a.offset_base + ctl.total);
      else reinterpret_cast<int64_t*>(a.offsets)[a.n_slots] = a.offset_base + ctl.total;
    }
  }
}

// the slot holding output byte `rel` (rel < total): the last slot i with soff[i] <= rel, which holds a value.  The
// search runs over the chunks' first offsets (csum, small and L2-resident) first, then inside one 1024-slot chunk.
__device__ __forceinline__ int64_t slot_of_byte(const int64_t* soff, const int64_t* csum, int64_t n_slots, int64_t rel) {
  int64_t lo = 0, hi = (n_slots + kTile - 1) / kTile - 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (csum[mid] <= rel) lo = mid; else hi = mid - 1;
  }
  hi = min(lo * kTile + kTile, n_slots) - 1;
  lo = lo * kTile;
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (soff[mid] <= rel) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// a grid over 16-byte pieces of out_data (aligned to its address); only when every byte fits
template <bool DBA>
__global__ void __launch_bounds__(kBaThreads)
ba_gather_kernel(BaArgs a) {
  const BaCtl ctl = *a.ctl;
  if (!ctl.fits || ctl.total == 0) return;
  const uintptr_t beg = reinterpret_cast<uintptr_t>(a.out), endp = beg + (uintptr_t)ctl.total;
  const uintptr_t a0 = beg & ~(uintptr_t)15;
  const int64_t n_pieces = (int64_t)((endp - a0 + 15) >> 4);
  for (int64_t q = (int64_t)blockIdx.x * kBaThreads + threadIdx.x; q < n_pieces; q += (int64_t)gridDim.x * kBaThreads) {
    const uintptr_t pa = a0 + (uintptr_t)q * 16;
    const int64_t lo = pa < beg ? 0 : (int64_t)(pa - beg);
    const int64_t hi = min((int64_t)(pa + 16 - beg), (int64_t)ctl.total);
    // bytes from the last down: a byte before its slot's start finds its slot by binary search (never a walk over a
    // run of empty slots), and for DELTA_BYTE_ARRAY the source value of byte j is reached from that of byte j+1 of the
    // same value, since the chain from value k passes every last-value-with-prefix-at-most-j in decreasing order
    uint8_t b[16];
    int64_t slot = slot_of_byte(a.soff, a.csum, a.n_slots, hi - 1), m = -1;
    for (int64_t rel = hi - 1; rel >= lo; --rel) {
      if (rel < a.soff[slot]) { slot = slot_of_byte(a.soff, a.csum, a.n_slots, rel); m = -1; }
      const int64_t j = rel - a.soff[slot];
      uint8_t v;
      if (DBA) {
        if (m < 0) m = a.ssrc[slot];
        while (a.pre[m] > j) m = a.psv[m];
        v = __ldg(a.data + a.vsrc[m] + (j - a.pre[m]));
      } else {
        v = __ldg(a.src_base + a.ssrc[slot] + j);
      }
      b[(int)(rel + beg - pa)] = v;
    }
    if (pa >= beg && pa + 16 <= endp) {
      uint4 w;
      memcpy(&w, b, 16);
      *reinterpret_cast<uint4*>(pa) = w;
    } else {
      for (int64_t rel = lo; rel < hi; ++rel) a.out[rel] = b[(int)(rel + beg - pa)];
    }
  }
}

// DELTA_BYTE_ARRAY: the suffix stream starts at the prefix stream's bytesRead()
__global__ void ba_skip_kernel(const DeltaPage* ps, int64_t* skip, int64_t n) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) skip[p] = ps[p].end;
}

void ba_err_text(const BaPage& s, const DeltaPage& dp, const DeltaPage& dl, char* buf, size_t n) {
  switch (s.err) {
    case kBaEof: snprintf(buf, n, "parquet: eof reading bytearray"); break;
    case kBaNegPlain: snprintf(buf, n, "parquet: invalid BYTE_ARRAY value"); break;
    case kBaLenStream: delta_err_text(dl, buf, n); break;
    case kBaPrefixStream: delta_err_text(dp, buf, n); break;
    case kBaNegLen: snprintf(buf, n, "parquet: negative delta byte array length %lld", (long long)s.arg); break;
    case kBaExceed: snprintf(buf, n, "parquet: delta byte array lengths exceed payload size"); break;
    case kBaCount: snprintf(buf, n, "parquet: delta prefix and suffix length counts do not match"); break;
    case kBaFirstPrefix: snprintf(buf, n, "parquet: first delta byte array prefix length must be zero"); break;
    case kBaBadPrefix: snprintf(buf, n, "parquet: invalid delta byte array prefix length %lld", (long long)s.arg); break;
    case kBaShort: snprintf(buf, n, "parquet: number of values / definition levels read did not match"); break;
    case kBaDict: snprintf(buf, n, "%s", err_text((int)s.arg)); break;
    default: snprintf(buf, n, "unknown error"); break;
  }
}

}  // namespace

// The device flavour's work.  out_at_base = out_data + offset_base (may be NULL when cap_rel == 0).  *h_total and
// h_decoded (may be NULL) are host memory; d_decoded and d_bad_pos (may be NULL) device memory.  Synchronises `st` once.
static ag_status byte_array_dev(int enc, int ow, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages, int64_t n_slots,
                                const uint8_t* valid, const void* doff, const uint8_t* ddata, int64_t dict_len, int64_t offset_base,
                                void* offsets, uint8_t* out_at_base, int64_t cap_rel, int64_t* h_total, int64_t* d_decoded,
                                int64_t* h_decoded, int64_t* d_bad_pos, BaCtl* h_ctl, cudaStream_t st) {
  const char* fn = "byte_array_decode";
  if (h_ctl) *h_ctl = BaCtl{0, 0, 0, 0, 0};
  const bool dict = enc == AG_PQ_ENC_PLAIN_DICTIONARY || enc == AG_PQ_ENC_RLE_DICTIONARY;
  const bool delta = enc == AG_PQ_ENC_DELTA_LENGTH_BYTE_ARRAY || enc == AG_PQ_ENC_DELTA_BYTE_ARRAY;
  const bool dba = enc == AG_PQ_ENC_DELTA_BYTE_ARRAY;
  if (!dict && !delta && enc != AG_PQ_ENC_PLAIN) AG_FAIL(AG_ERR_INVALID, "%s: encoding %d is not a BYTE_ARRAY encoding", fn, enc);
  if (ow != 4 && ow != 8) AG_FAIL(AG_ERR_INVALID, "%s: offset_width must be 4 or 8", fn);
  if (n_pages < 0 || n_slots < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative page or slot count", fn);
  if (n_pages > 0 && !pages) AG_FAIL(AG_ERR_INVALID, "%s: NULL page table", fn);
  if (!offsets) AG_FAIL(AG_ERR_INVALID, "%s: NULL offsets", fn);
  if (offset_base < 0 || (ow == 4 && offset_base > 0x7fffffffLL)) AG_FAIL(AG_ERR_INVALID, "%s: offset_base out of range for the offset width", fn);
  if (reinterpret_cast<uintptr_t>(offsets) & (ow - 1)) AG_FAIL(AG_ERR_INVALID, "%s: offsets not aligned to offset_width", fn);
  if (dict && dict_len < 0) AG_FAIL(AG_ERR_INVALID, "%s: negative dictionary length", fn);
  if (dict && !doff) AG_FAIL(AG_ERR_INVALID, "%s: NULL dictionary offsets", fn);
  if (dict && (reinterpret_cast<uintptr_t>(doff) & (ow - 1))) AG_FAIL(AG_ERR_INVALID, "%s: dictionary offsets not aligned to offset_width", fn);
  // plan: pages | run_base[n+1] | tile_base[n+1] | delta pages (out = first dense index)
  PagePlan plan;
  AG_TRY(plan_pages(fn, pages, n_pages, [&](const ag_pq_page& g) { return dict ? std::min(g.num_values, g.len) : (int64_t)0; }, &plan));
  const size_t o_dpages = plan.bytes.size();
  plan.bytes.resize(o_dpages + (size_t)n_pages * sizeof(ag_pq_page));
  const int64_t* tile_base = plan.tile_base();
  ag_pq_page* dpages = reinterpret_cast<ag_pq_page*>(plan.bytes.data() + o_dpages);
  std::vector<std::pair<int64_t, int64_t>> ranges;
  for (int64_t i = 0; i < n_pages; ++i) {
    const ag_pq_page& g = pages[i];
    if (g.out + g.num_values > n_slots) AG_FAIL(AG_ERR_INVALID, "%s: page %lld: slots past n_slots", fn, (long long)i);
    if (g.num_values) ranges.emplace_back(g.out, g.out + g.num_values);
    dpages[i] = g;
    dpages[i].out = tile_base[i] * kTile;
  }
  std::sort(ranges.begin(), ranges.end());
  for (size_t i = 1; i < ranges.size(); ++i)
    if (ranges[i].first < ranges[i - 1].second) AG_FAIL(AG_ERR_INVALID, "%s: page slot ranges overlap", fn);
  if (plan.any_data && !data) AG_FAIL(AG_ERR_INVALID, "%s: NULL page data", fn);
  const int64_t n_tiles = plan.n_tiles, n_runs = plan.n_desc, n_dense = n_tiles * kTile;
  const int64_t n_chunks = (n_slots + kTile - 1) / kTile;

  // psv levels: 32^(l+1) values per entry, until one entry covers everything
  int nlev = 0;
  int64_t lev_n[kPsvLevels] = {0};
  if (dba) for (int64_t m = n_dense / 32; nlev < kPsvLevels; m = (m + 31) / 32) { lev_n[nlev++] = m; if (m <= 1) break; }

  // scratch
  Carve sc;
  const size_t o_plan = sc.take(plan.bytes.size());
  const size_t o_st = sc.take((size_t)n_pages * sizeof(BaPage));
  const size_t o_tc = sc.take(valid ? (size_t)n_tiles * 8 : 0);
  const size_t o_vlen = sc.take(dict ? 0 : (size_t)n_dense * 8);
  const size_t o_vsrc = sc.take(dict ? 0 : (size_t)n_dense * 8);
  const size_t o_slen = sc.take((size_t)n_slots * 8);
  const size_t o_ssrc = sc.take((size_t)n_slots * 8);
  const size_t o_soff = sc.take((size_t)(n_slots + 1) * 8);
  const size_t o_csum = sc.take((size_t)n_chunks * 8);
  const size_t o_ctl = sc.take(sizeof(BaCtl));
  const size_t o_bad = sc.take(8);
  // dictionary
  const size_t o_pqs = sc.take(dict ? (size_t)n_pages * sizeof(PageState) : 0);
  const size_t o_ti = sc.take(dict ? (size_t)n_tiles * 8 : 0);
  const size_t o_runs = sc.take(dict ? (size_t)n_runs * 8 : 0);
  const size_t o_idx = sc.take(dict ? (size_t)n_slots * 4 : 0);
  // delta
  const size_t o_dls = sc.take(delta ? (size_t)n_pages * sizeof(DeltaPage) : 0);
  const size_t o_dps = sc.take(dba ? (size_t)n_pages * sizeof(DeltaPage) : 0);
  const size_t o_mbl = sc.take(delta ? (size_t)tile_base[n_pages] * (kTile / 32) * sizeof(DeltaMini) : 0);
  const size_t o_mbp = sc.take(dba ? (size_t)tile_base[n_pages] * (kTile / 32) * sizeof(DeltaMini) : 0);
  const size_t o_mbb = sc.take(delta ? (size_t)(n_pages + 1) * 8 : 0);
  const size_t o_tsum = sc.take(delta ? (size_t)n_tiles * 8 : 0);
  const size_t o_suf = sc.take(delta ? (size_t)n_dense * 4 : 0);
  const size_t o_pre = sc.take(dba ? (size_t)n_dense * 4 : 0);
  const size_t o_skip = sc.take(dba ? (size_t)n_pages * 8 : 0);
  const size_t o_lt = sc.take(delta ? (size_t)n_tiles * sizeof(LenTile) : 0);
  const size_t o_tb = sc.take(delta ? (size_t)n_tiles * 8 : 0);
  const size_t o_psv = sc.take(dba ? (size_t)n_dense * 8 : 0);
  size_t o_lv[kPsvLevels];
  for (int l = 0; l < nlev; ++l) o_lv[l] = sc.take((size_t)lev_n[l] * 4 + 128);

  Temps t(st);
  uint8_t* d;
  AG_TRY(t.alloc_t(&d, sc.size));
  PqPlan pl;
  AG_TRY(upload_plan(plan, d + o_plan, st, &pl));
  BaArgs a{};
  a.pages = pl.pages;
  a.tile_base = pl.tile_base;
  a.n_pages = n_pages; a.n_tiles = n_tiles; a.n_slots = n_slots;
  a.data = data; a.valid = valid;
  a.tile_cnt = valid ? reinterpret_cast<int64_t*>(d + o_tc) : nullptr;
  a.st = reinterpret_cast<BaPage*>(d + o_st);
  a.vlen = reinterpret_cast<int64_t*>(d + o_vlen);
  a.vsrc = reinterpret_cast<int64_t*>(d + o_vsrc);
  a.slen = reinterpret_cast<int64_t*>(d + o_slen);
  a.ssrc = reinterpret_cast<int64_t*>(d + o_ssrc);
  a.soff = reinterpret_cast<int64_t*>(d + o_soff);
  a.csum = reinterpret_cast<int64_t*>(d + o_csum);
  a.ctl = reinterpret_cast<BaCtl*>(d + o_ctl);
  a.d_decoded = d_decoded;
  a.kind = enc; a.ow = ow; a.offset_base = offset_base; a.cap_rel = cap_rel;
  a.offsets = offsets; a.out = out_at_base;
  a.src_base = dict ? ddata : data;
  a.doff = doff;
  a.pqs = reinterpret_cast<const PageState*>(d + o_pqs);
  a.idx = reinterpret_cast<const int32_t*>(d + o_idx);
  a.dls = reinterpret_cast<const DeltaPage*>(d + o_dls);
  a.dps = reinterpret_cast<const DeltaPage*>(d + o_dps);
  a.suf = reinterpret_cast<const int32_t*>(d + o_suf);
  a.pre = reinterpret_cast<const int32_t*>(d + o_pre);
  a.psv = reinterpret_cast<int64_t*>(d + o_psv);
  a.nlev = nlev;
  for (int l = 0; l < nlev; ++l) a.lv[l] = reinterpret_cast<int32_t*>(d + o_lv[l]);
  unsigned long long* bad = reinterpret_cast<unsigned long long*>(d_bad_pos ? (void*)d_bad_pos : (void*)(d + o_bad));
  if (n_slots) AG_CUDA_TRY(cudaMemsetAsync(a.slen, 0, (size_t)n_slots * 8, st));

  // ---- stage 1: values ----
  AG_TRY(launch_tile_counts(pl, valid, a.tile_cnt, st));
  if (n_pages && enc == AG_PQ_ENC_PLAIN) {
    ba_plain_parse_kernel<<<(unsigned)n_pages, kBaThreads, 0, st>>>(a);
    AG_TRY(check_launch("ba_plain_parse_kernel"));
  } else if (n_pages && dict) {
    PqArgs c{};
    c.plan = pl;
    c.data = data; c.valid = valid;
    c.st = reinterpret_cast<PageState*>(d + o_pqs);
    c.runs = n_runs ? reinterpret_cast<uint2*>(d + o_runs) : nullptr;
    c.tile_cnt = a.tile_cnt;
    c.tile_info = reinterpret_cast<int2*>(d + o_ti);
    c.d_decoded = nullptr;
    c.bad = bad;
    c.kind = kIndex; c.width = 4; c.dict_len = dict_len; c.out = d + o_idx;
    pq_runs_kernel<<<(unsigned)n_pages, kRleThreads, 0, st>>>(c);
    AG_TRY(check_launch("pq_runs_kernel"));
    AG_TRY((valid ? launch_expand<kIndex, int32_t, true>(c, st) : launch_expand<kIndex, int32_t, false>(c, st)));
    ba_from_dict_kernel<<<(unsigned)((n_pages + 127) / 128), 128, 0, st>>>(a);
    AG_TRY(check_launch("ba_from_dict_kernel"));
  } else if (n_pages) {
    // every length of the (prefix, then suffix) stream, dense, from the DELTA_BINARY_PACKED passes
    int64_t* mbb = reinterpret_cast<int64_t*>(d + o_mbb);
    std::vector<int64_t> hm((size_t)n_pages + 1);
    for (int64_t i = 0; i <= n_pages; ++i) hm[i] = tile_base[i] * (kTile / 32);
    AG_TRY(h2d(mbb, hm.data(), hm.size() * 8, st));
    DeltaArgs da{};
    da.pages = reinterpret_cast<const ag_pq_page*>(d + o_plan + o_dpages);
    da.mb_base = mbb; da.tile_base = a.tile_base; da.n_pages = n_pages; da.data = data; da.valid = nullptr;
    da.tile_sum = reinterpret_cast<unsigned long long*>(d + o_tsum);
    da.d_decoded = nullptr; da.width = 4;
    auto run_stream = [&](DeltaPage* ps, DeltaMini* mb, const int64_t* skip, void* out) -> ag_status {
      da.st = ps; da.mb = mb; da.skip = skip; da.out = out;
      delta_walk_kernel<<<(unsigned)n_pages, kRleThreads, 0, st>>>(da);
      AG_TRY(check_launch("delta_walk_kernel"));
      if (n_tiles) AG_TRY((launch_delta_values<uint32_t, false>(da, n_tiles, st)));
      return AG_OK;
    };
    int64_t* skip = nullptr;
    if (dba) {
      AG_TRY(run_stream(const_cast<DeltaPage*>(a.dps), reinterpret_cast<DeltaMini*>(d + o_mbp), nullptr, d + o_pre));
      skip = reinterpret_cast<int64_t*>(d + o_skip);
      ba_skip_kernel<<<(unsigned)((n_pages + 127) / 128), 128, 0, st>>>(a.dps, skip, n_pages);
      AG_TRY(check_launch("ba_skip_kernel"));
    }
    AG_TRY(run_stream(const_cast<DeltaPage*>(a.dls), reinterpret_cast<DeltaMini*>(d + o_mbl), skip, d + o_suf));
    LenTile* lt = reinterpret_cast<LenTile*>(d + o_lt);
    long long* tb = reinterpret_cast<long long*>(d + o_tb);   // per tile: length sum, then the page's sum before it
    ba_len_page_kernel<0><<<(unsigned)n_pages, kBaThreads, 0, st>>>(a, lt, tb);
    AG_TRY(check_launch("ba_len_page_kernel"));
    if (n_tiles) {
      ba_len_tiles_kernel<<<(unsigned)n_tiles, kBaThreads, 0, st>>>(a, lt, tb);
      AG_TRY(check_launch("ba_len_tiles_kernel"));
    }
    ba_len_page_kernel<1><<<(unsigned)n_pages, kBaThreads, 0, st>>>(a, lt, tb);
    AG_TRY(check_launch("ba_len_page_kernel"));
    if (n_tiles) {
      tile_sum_scan_kernel<<<(unsigned)n_pages, kBaThreads, 0, st>>>(a.tile_base, reinterpret_cast<unsigned long long*>(tb));
      AG_TRY(check_launch("tile_sum_scan_kernel"));
      ba_len_write_kernel<<<(unsigned)n_tiles, kBaThreads, 0, st>>>(a, tb);
      AG_TRY(check_launch("ba_len_write_kernel"));
    }
    if (dba && n_tiles) {
      const int32_t* in = a.pre;
      for (int l = 0; l < nlev; ++l) {
        ba_min_kernel<<<(unsigned)((lev_n[l] * 32 + kBaThreads - 1) / kBaThreads), kBaThreads, 0, st>>>(in, a.lv[l], lev_n[l]);
        AG_TRY(check_launch("ba_min_kernel"));
        in = a.lv[l];
      }
      ba_psv_kernel<<<(unsigned)n_tiles, kBaThreads, 0, st>>>(a);
      AG_TRY(check_launch("ba_psv_kernel"));
    }
  }

  // ---- stage 2: slots and offsets ----
  if (n_tiles) {
    if (dict) valid ? ba_slot_kernel<true, true><<<(unsigned)n_tiles, kBaThreads, 0, st>>>(a) : ba_slot_kernel<false, true><<<(unsigned)n_tiles, kBaThreads, 0, st>>>(a);
    else valid ? ba_slot_kernel<true, false><<<(unsigned)n_tiles, kBaThreads, 0, st>>>(a) : ba_slot_kernel<false, false><<<(unsigned)n_tiles, kBaThreads, 0, st>>>(a);
    AG_TRY(check_launch("ba_slot_kernel"));
  }
  if (n_chunks) {
    ba_sum_kernel<<<(unsigned)n_chunks, kBaThreads, 0, st>>>(a);
    AG_TRY(check_launch("ba_sum_kernel"));
  }
  ba_scan_kernel<<<1, kBaThreads, 0, st>>>(a, n_chunks);
  AG_TRY(check_launch("ba_scan_kernel"));
  ba_offsets_kernel<<<(unsigned)(n_chunks ? n_chunks : 1), kBaThreads, 0, st>>>(a);
  AG_TRY(check_launch("ba_offsets_kernel"));

  // ---- stage 3: bytes ----
  if (cap_rel > 0 && out_at_base) {
    const int64_t max_pieces = cap_rel / 16 + 2;
    const unsigned grid = grid_for(max_pieces, kBaThreads, 8);
    if (dba) ba_gather_kernel<true><<<grid, kBaThreads, 0, st>>>(a);
    else ba_gather_kernel<false><<<grid, kBaThreads, 0, st>>>(a);
    AG_TRY(check_launch("ba_gather_kernel"));
  }

  // ---- one synchronisation: pages, decisions, bad index ----
  std::vector<BaPage> hs((size_t)n_pages);
  std::vector<DeltaPage> hdl(delta ? (size_t)n_pages : 0), hdp(dba ? (size_t)n_pages : 0);
  BaCtl ctl;
  int64_t hbad = AG_NO_ERROR_POS;
  AG_TRY(d2h(hs.data(), a.st, (size_t)n_pages * sizeof(BaPage), st));
  if (delta) AG_TRY(d2h(hdl.data(), a.dls, (size_t)n_pages * sizeof(DeltaPage), st));
  if (dba) AG_TRY(d2h(hdp.data(), a.dps, (size_t)n_pages * sizeof(DeltaPage), st));
  AG_TRY(d2h(&ctl, a.ctl, sizeof ctl, st));
  if (dict && n_pages) AG_TRY(d2h(&hbad, bad, 8, st));
  AG_TRY(sync(st));
  if (h_ctl) *h_ctl = ctl;
  if (d_bad_pos && (!dict || n_pages == 0)) {
    // no index was looked at (not a dictionary call, or no page): *d_bad_pos is still overwritten
    static const int64_t none = AG_NO_ERROR_POS;
    AG_TRY(h2d(d_bad_pos, &none, 8, st));
    AG_TRY(sync(st));
  }
  if (h_decoded)
    for (int64_t i = 0; i < n_pages; ++i) h_decoded[i] = hs[i].slots;
  if (!ctl.write_offsets)
    AG_FAIL(AG_ERR_INVALID, "%s: offset_base + total = %lld does not fit int32 offsets", fn, (long long)(offset_base + ctl.total));
  if (h_total) *h_total = ctl.total;
  for (int64_t i = 0; i < n_pages; ++i)
    if (hs[i].err != kBaNone) {
      char msg[200];
      ba_err_text(hs[i], dba ? hdp[i] : DeltaPage{}, delta ? hdl[i] : DeltaPage{}, msg, sizeof msg);
      AG_FAIL(AG_ERR_INVALID, "%s: page %lld: %s (%lld values decoded)", fn, (long long)i, msg, (long long)hs[i].slots);
    }
  if (dict && hbad != AG_NO_ERROR_POS)
    AG_FAIL(AG_ERR_INVALID, "%s: invalid index values found for dictionary converter (output slot %lld)", fn, (long long)hbad);
  return AG_OK;
}

}  // namespace ag

using namespace ag;

extern "C" {

ag_status ag_parquet_byte_array_decode_dev(int encoding, int offset_width, const uint8_t* d_data, const ag_pq_page* pages, int64_t n_pages,
                                           int64_t n_slots, const uint8_t* d_valid, const void* d_dict_offsets, const uint8_t* d_dict_data,
                                           int64_t dict_len, int64_t offset_base, void* d_offsets, uint8_t* d_out_data, int64_t out_cap,
                                           int64_t* total, int64_t* d_decoded, int64_t* d_bad_pos, ag_stream_t s) {
  AG_TRY(ensure_init());
  if (out_cap < 0) AG_FAIL(AG_ERR_INVALID, "byte_array_decode: negative out_cap");
  const int64_t cap_rel = d_out_data && out_cap > offset_base ? out_cap - offset_base : 0;
  return byte_array_dev(encoding, offset_width, d_data, pages, n_pages, n_slots, d_valid, d_dict_offsets, d_dict_data, dict_len, offset_base,
                        d_offsets, cap_rel ? d_out_data + offset_base : nullptr, cap_rel, total, d_decoded, nullptr, d_bad_pos, nullptr,
                        resolve_stream(s));
}

ag_status ag_parquet_byte_array_decode(int encoding, int offset_width, const uint8_t* data, const ag_pq_page* pages, int64_t n_pages,
                                       int64_t n_slots, const uint8_t* valid, const void* dict_offsets, const uint8_t* dict_data,
                                       int64_t dict_len, int64_t offset_base, void* offsets, uint8_t* out_data, int64_t out_cap,
                                       int64_t* total, int64_t* decoded, int64_t* bad_pos) {
  AG_TRY(ensure_init());
  if (bad_pos) *bad_pos = AG_NO_ERROR_POS;
  if (out_cap < 0) AG_FAIL(AG_ERR_INVALID, "byte_array_decode: negative out_cap");
  if (offset_width != 4 && offset_width != 8) AG_FAIL(AG_ERR_INVALID, "byte_array_decode: offset_width must be 4 or 8");
  if (n_pages < 0 || n_slots < 0) AG_FAIL(AG_ERR_INVALID, "byte_array_decode: negative page or slot count");
  if (n_pages > 0 && !pages) AG_FAIL(AG_ERR_INVALID, "byte_array_decode: NULL page table");
  if (!offsets) AG_FAIL(AG_ERR_INVALID, "byte_array_decode: NULL offsets");
  const bool dict = encoding == AG_PQ_ENC_PLAIN_DICTIONARY || encoding == AG_PQ_ENC_RLE_DICTIONARY;
  if (dict && dict_len < 0) AG_FAIL(AG_ERR_INVALID, "byte_array_decode: negative dictionary length");
  int64_t data_end = 0, bound = 0;
  for (int64_t i = 0; i < n_pages; ++i) {
    if (pages[i].data < 0 || pages[i].len < 0) AG_FAIL(AG_ERR_INVALID, "byte_array_decode: page %lld: negative field", (long long)i);
    data_end = std::max(data_end, pages[i].data + pages[i].len);
    bound += pages[i].len;
  }
  if (data_end > 0 && !data) AG_FAIL(AG_ERR_INVALID, "byte_array_decode: NULL page data");
  int64_t dict_bytes = 0;
  if (dict && dict_len > 0) {
    if (!dict_offsets) AG_FAIL(AG_ERR_INVALID, "byte_array_decode: NULL dictionary offsets");
    int64_t lo = 0, hi = 0, maxlen = 0;
    for (int64_t i = 0; i <= dict_len; ++i) {
      const int64_t v = offset_width == 4 ? reinterpret_cast<const int32_t*>(dict_offsets)[i] : reinterpret_cast<const int64_t*>(dict_offsets)[i];
      if (i == 0) lo = v;
      else maxlen = std::max(maxlen, v - hi);
      hi = v;
    }
    dict_bytes = std::max<int64_t>(hi, 0);
    if (dict_bytes > 0 && !dict_data) AG_FAIL(AG_ERR_INVALID, "byte_array_decode: NULL dictionary data");
    (void)lo;
    bound = maxlen > 0 && n_slots > INT64_MAX / maxlen ? INT64_MAX : n_slots * maxlen;
  } else if (dict) {
    bound = 0;
  }
  CallStream cs; AG_TRY(cs.acquire());
  Temps t(cs);
  const size_t vbytes = valid ? (size_t)((n_slots + 7) >> 3) : 0;
  const size_t obytes = (size_t)(n_slots + 1) * offset_width;
  const size_t doff_bytes = dict ? (size_t)(dict_len + 1) * offset_width : 0;
  uint8_t *dd = nullptr, *dv = nullptr, *doff = nullptr, *ddata = nullptr, *dofs = nullptr, *dout = nullptr;
  AG_TRY(t.alloc_t(&dd, (size_t)data_end));
  AG_TRY(h2d(dd, data, (size_t)data_end, cs));
  if (vbytes) { AG_TRY(t.alloc_t(&dv, vbytes)); AG_TRY(h2d(dv, valid, vbytes, cs)); }
  if (dict) {
    AG_TRY(t.alloc_t(&doff, doff_bytes));
    if (dict_len >= 0 && dict_offsets) AG_TRY(h2d(doff, dict_offsets, doff_bytes, cs));
    AG_TRY(t.alloc_t(&ddata, (size_t)dict_bytes));
    AG_TRY(h2d(ddata, dict_data, (size_t)dict_bytes, cs));
  }
  AG_TRY(t.alloc_t(&dofs, obytes));
  const int64_t room = out_data && out_cap > offset_base ? out_cap - offset_base : 0;
  int64_t* dbad = nullptr;
  AG_TRY(t.alloc_t(&dbad, 8));
  if (encoding == AG_PQ_ENC_DELTA_BYTE_ARRAY) bound = room;        // nothing but the caller's capacity bounds it
  // the device buffer holds min(room, bound) bytes; a room below the bound is passed as is, so the device makes the
  // decision it would make for out_cap (and then writes nothing)
  const int64_t cap_rel = std::min(room, bound);
  if (cap_rel > 0) AG_TRY(t.alloc_t(&dout, (size_t)cap_rel));
  std::vector<int64_t> dec((size_t)n_pages, 0);
  BaCtl ctl;
  const ag_status rc = byte_array_dev(encoding, offset_width, dd, pages, n_pages, n_slots, dv, doff, ddata, dict_len, offset_base, dofs,
                                      cap_rel > 0 ? dout : nullptr, room, nullptr, nullptr, dec.data(), dict ? dbad : nullptr, &ctl, cs);
  if (rc != AG_OK && rc != AG_ERR_INVALID) return rc;
  if (decoded && ctl.decoded) memcpy(decoded, dec.data(), (size_t)n_pages * 8);
  if (ctl.write_offsets) {
    if (total) *total = ctl.total;
    AG_TRY(d2h(offsets, dofs, obytes, cs));
    if (ctl.fits && ctl.total > 0) AG_TRY(d2h(out_data + offset_base, dout, (size_t)ctl.total, cs));
  }
  if (dict && bad_pos) AG_TRY(d2h(bad_pos, dbad, 8, cs));
  const ag_status rs = sync(cs);
  return rc != AG_OK ? rc : rs;
}

}  // extern "C"
