// hash.cu — is_in, unique and dictionary_encode for fixed-width columns on sm_90a (SURVEY §8f rank 3).
//
// Replaces, for 1/2/4/8-byte values, the memo-table kernels of the reference:
//   is_in   arrow/compute/internal/kernels/scalar_set_lookup.go:112-413 (SetLookupState.Init builds a memo table of
//           the value set keyed by the RAW BYTES of a value — floats compare by bit pattern: NaN == NaN of the same
//           payload, -0.0 != +0.0; isInKernelExec :373-413 writes a data bit and a validity bit per row by the
//           NullMatchingBehavior table restated in is_in_kernel below);
//   unique  arrow/compute/internal/kernels/vector_hash.go (the distinct values in order of FIRST appearance, a null
//           kept once at the position of its first appearance);
//   dictionary_encode  kernels/vector_hash.go:144-241 (int32 indices into the distinct values in order of first
//           appearance over every chunk of a column; a null masked, or encoded as one entry where it first appears).
// Both sit on the same open-addressing table: 16-byte slots {64-bit key = the value's bytes zero-extended, lowest row
// that carried the key}, linear probing from an even slot (so a probe can always look at an aligned pair), load factor
// <= 0.5, keys inserted with atomicCAS, first rows with atomicMin.  The first row is all `unique` needs: a row is
// emitted iff it is the first row of its key, and the emitted rows are compacted in row order by the filter kernel
// (filter.cu) — so the output order is the reference's and does not depend on the order in which threads reached the
// table.
//   is_in : value sets up to 4096 entries are probed in shared memory (at most 8192 key slots = 64 KB, load factor <= 1/4
//           for sets up to 2048 values, two slots per 128-bit read); 1- and 2-byte values skip hashing altogether:
//           the set becomes a 256 / 65536-bit membership bitmap.  Larger sets are probed in HBM / L2.
//   unique: a column of more than 2M rows first runs against a 2M-slot table that stays L2-resident (32 MB); only when
//           more than 1M distinct values turn up does the insert raise an overflow word, and the full-size table
//           (2n slots) is cleared and filled by kernels that test that word first — the choice is made on the device,
//           the call stays stream-ordered.  Each warp also keeps the last keys it met in a small shared-memory cache:
//           a key met at a lower row of the same warp cannot be a first appearance, so low-cardinality columns
//           (the usual dictionary-encoding case) hardly touch the table at all.
// Roofline: HBM, 8 B/row read once per pass (is_in: one pass; unique: insert + mark + compaction).
#include "host_stage.cuh"

namespace ag {

constexpr int kHThreads = 256;
constexpr int kHWarps = kHThreads / 32;
constexpr int kHUnroll = 4;                 // 32-row groups a warp has in flight
constexpr unsigned long long kEmptyKey = 0xffffffffffffffffull;
constexpr unsigned kNoRow = 0xffffffffu;
constexpr unsigned kNoCap = 0xffffffffu;

struct alignas(16) Slot { unsigned long long key; unsigned first; unsigned pad; };

struct HashTable {
  Slot* slots;                // cleared to all-ones: key = kEmptyKey (free), first = kNoRow
  unsigned long long mask;    // slots - 1
  int shift;                  // 64 - log2(slots)
  unsigned cap;               // distinct keys after which an insert raises special[3] and stops (kNoCap: never)
  unsigned* special;          // [0] lowest row whose key is the all-ones pattern (cannot live in `slots`), [1] lowest NULL row,
                              // [2] distinct keys inserted, [3] overflow word (0xffffffff after the clear = not raised)
};

// multiplicative (Fibonacci) hash of the folded key, forced even: every probe sequence starts on an aligned slot pair
__device__ __forceinline__ unsigned long long hash_slot(unsigned long long key, int shift) {
  const unsigned long long x = key ^ (key >> 32);
  return ((x * 0x9E3779B97F4A7C15ull) >> shift) & ~1ull;
}
__device__ __forceinline__ bool overflowed(const HashTable& t) { return *reinterpret_cast<volatile unsigned*>(&t.special[3]) == 1u; }

template <typename V>
__device__ __forceinline__ unsigned long long raw_key(const V* __restrict__ vals, int64_t i) {
  return (unsigned long long)vals[i];
}

// lower `*p` to `row` (rows arrive roughly in increasing order, so after the first few rows of a key the word already
// holds a lower row and a plain load replaces the atomic: 100M rows over 100 keys would otherwise serialise 100M atomics
// on 100 addresses)
__device__ __forceinline__ void lower_row(unsigned* p, unsigned seen, unsigned row) {
  if (seen > row) atomicMin(p, row);
}

// after each probe step of an insert: true when the insert should give up.  A capped table can fill up completely
// while the inserts that were in flight when the cap was crossed finish.
__device__ __forceinline__ bool probe_gives_up(const HashTable& t, unsigned& probes) {
  if (t.cap == kNoCap || ((++probes & 7u) != 0u)) return false;
  if (overflowed(t)) return true;
  // a probe this long at load factor <= 1/2 means the table has filled up behind the counter (the lanes that
  // created the last keys report them only after their warp step, and a lane spinning here would keep its own
  // warp from ever reporting): raise the word from here
  if (probes >= 1024u) { *reinterpret_cast<volatile unsigned*>(&t.special[3]) = 1u; return true; }
  return false;
}

// distinct keys so far, one atomic per warp step (a column of all-distinct values would otherwise put 2M atomics on
// one word before the cap stops it: 2.9 ms); raises the overflow word past the cap.  special[2] is cleared to
// 0xffffffff = count - 1.  Every lane of the warp calls it.
__device__ __forceinline__ void count_made(const HashTable& t, bool made, int lane) {
  if (t.cap == kNoCap) return;
  const unsigned m = __ballot_sync(0xffffffffu, made);
  if (lane == 0 && m) {
    const unsigned c = (unsigned)__popc(m);
    if (atomicAdd(&t.special[2], c) + 1u + c > t.cap) *reinterpret_cast<volatile unsigned*>(&t.special[3]) = 1u;
  }
}

// returns true when this call created the key's slot
__device__ __forceinline__ bool table_insert(const HashTable& t, unsigned long long key, unsigned row) {
  unsigned long long h = hash_slot(key, t.shift);
  unsigned probes = 0;
  while (true) {
    Slot* s = t.slots + h;
    const ulonglong2 raw = __ldcg(reinterpret_cast<const ulonglong2*>(s));   // key and first row in one L2 request
    unsigned long long cur = raw.x;
    unsigned seen = (unsigned)raw.y;
    bool made = false;
    if (cur == kEmptyKey) {
      cur = atomicCAS(&s->key, kEmptyKey, key);
      if (cur == kEmptyKey) { made = true; seen = kNoRow; cur = key; }
      else if (cur == key) seen = kNoRow;     // somebody else created it just now: its first row is not in `raw`
    }
    if (cur == key) { lower_row(&s->first, seen, row); return made; }
    h = (h + 1) & t.mask;
    if (probe_gives_up(t, probes)) return false;
  }
}
// lowest row that carried `key`, kNoRow when absent (the table is complete: plain cached loads)
__device__ __forceinline__ unsigned table_first_row(const HashTable& t, unsigned long long key) {
  unsigned long long h = hash_slot(key, t.shift);
  while (true) {
    const ulonglong2 raw = *reinterpret_cast<const ulonglong2*>(t.slots + h);
    if (raw.x == key) return (unsigned)raw.y;
    if (raw.x == kEmptyKey) return kNoRow;
    h = (h + 1) & t.mask;
  }
}

// Per-warp cache of keys already met (direct-mapped, 256 entries).  A warp walks its rows in increasing order, so a hit
// means: this key sits at a lower row that this warp has already sent to the table.
constexpr int kWarpCacheSlots = 256;
__device__ __forceinline__ int warp_cache_slot(unsigned long long key) {
  return (int)(((key ^ (key >> 32)) * 0x9E3779B97F4A7C15ull) >> 56);
}

// `run_if`: NULL, or a device word the kernel tests first (the full-size pass of `unique` runs only after an overflow).
// `row_base`: the row number of the first value (dictionary_encode numbers the rows of all chunks of a column in turn)
template <typename V>
__global__ void __launch_bounds__(kHThreads)
hash_insert_kernel(const V* __restrict__ vals, const uint8_t* __restrict__ valid, int64_t off, int64_t n, const HashTable t,
                   const unsigned* __restrict__ run_if, unsigned row_base) {
  __shared__ unsigned long long s_cache[kHWarps][kWarpCacheSlots];
  if (run_if && *run_if != 1u) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long* cache = s_cache[warp];
  for (int i = lane; i < kWarpCacheSlots; i += 32) cache[i] = kEmptyKey;
  __syncwarp();
  const int64_t n_words = (n + 31) >> 5;
  const int64_t warp0 = ((int64_t)blockIdx.x * kHThreads + threadIdx.x) >> 5;
  const int64_t warps = ((int64_t)gridDim.x * kHThreads) >> 5;
  for (int64_t w0 = warp0 * kHUnroll; w0 < n_words; w0 += warps * kHUnroll) {
    if (__any_sync(0xffffffffu, t.cap != kNoCap && overflowed(t))) return;   // the small table is being abandoned (warp-uniform exit)
    V x[kHUnroll];
    int kind[kHUnroll];                                  // 0 nothing, 1 value, 2 null
    if (!valid && ((w0 + kHUnroll) << 5) <= n) {         // interior, no nulls: unconditional loads
      const V* __restrict__ p = vals + off + (w0 << 5) + lane;
#pragma unroll
      for (int k = 0; k < kHUnroll; ++k) { x[k] = __ldcs(p + 32 * k); kind[k] = 1; }
    } else {
#pragma unroll
      for (int k = 0; k < kHUnroll; ++k) {
        const int64_t i = ((w0 + k) << 5) + lane;
        kind[k] = i < n ? ((valid && !bit_is_set(valid, off + i)) ? 2 : 1) : 0;
        x[k] = kind[k] == 1 ? __ldcs(vals + off + i) : V(0);
      }
    }
#pragma unroll
    for (int k = 0; k < kHUnroll; ++k) {
      const unsigned row = row_base + (unsigned)(((w0 + k) << 5) + lane);
      const unsigned long long key = (unsigned long long)x[k];
      const int cs = warp_cache_slot(key);
      const bool ones = sizeof(V) == 8 && key == kEmptyKey;     // narrower values zero-extend: never all ones
      if (kind[k] == 2) lower_row(&t.special[1], *reinterpret_cast<volatile unsigned*>(&t.special[1]), row);
      else if (kind[k] == 1 && ones) lower_row(&t.special[0], *reinterpret_cast<volatile unsigned*>(&t.special[0]), row);
      const bool go = kind[k] == 1 && !ones && cache[cs] != key;
      __syncwarp();
      bool made = false;
      if (go) { made = table_insert(t, key, row); atomicExch(&cache[cs], key); }   // several lanes may share a slot: one whole key wins
      __syncwarp();
      count_made(t, made, lane);
    }
  }
}

__global__ void __launch_bounds__(kHThreads)
table_clear_kernel(uint4* __restrict__ p, int64_t n16, const unsigned* __restrict__ run_if) {
  if (run_if && *run_if != 1u) return;
  const uint4 ones = make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu);
  for (int64_t i = (int64_t)blockIdx.x * kHThreads + threadIdx.x; i < n16; i += (int64_t)gridDim.x * kHThreads) p[i] = ones;
}

// isInKernelExec (scalar_set_lookup.go:373-413), per row:
//   valid value : in the set -> (true, valid); else INCONCLUSIVE with a null in the set -> (false, null); else (false, valid)
//   null        : MATCH with a null in the set -> (true, valid); SKIP, or MATCH without one -> (false, valid); else (false, null)
constexpr int kIsInSmemSlots = 8192;   // 64 KB of keys
enum { kMemberTable = 0, kMemberSmem = 1, kMemberBitmap = 2 };

// membership bitmap of a 1- or 2-byte value set: bit v of `bits`; a null in the set lowers special[1]
template <typename V>
__global__ void __launch_bounds__(kHThreads)
set_bitmap_kernel(const V* __restrict__ set, const uint8_t* __restrict__ valid, int64_t off, int64_t n, unsigned* __restrict__ bits,
                  unsigned* __restrict__ special) {
  for (int64_t i = (int64_t)blockIdx.x * kHThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kHThreads) {
    if (valid && !bit_is_set(valid, off + i)) atomicMin(&special[1], (unsigned)i);
    else { const unsigned v = (unsigned)set[off + i]; atomicOr(&bits[v >> 5], 1u << (v & 31)); }
  }
}

template <typename V, int kMember>
__global__ void __launch_bounds__(kHThreads)
is_in_kernel(const V* __restrict__ vals, const uint8_t* __restrict__ valid, int64_t off, int64_t n, const HashTable t,
             const unsigned* __restrict__ set_bits, int null_behavior, uint32_t* __restrict__ out_data, uint32_t* __restrict__ out_valid,
             unsigned long long* __restrict__ null_count) {
  extern __shared__ __align__(16) unsigned long long s_keys[];   // kMemberSmem: the table's keys; kMemberBitmap: the bitmap words
  constexpr int kBitWords = sizeof(V) == 1 ? 8 : 2048;
  if (kMember == kMemberSmem) {
    // the column streams through L1 and would keep evicting a table that lives in global memory
    for (unsigned i = threadIdx.x; i <= (unsigned)t.mask; i += kHThreads) s_keys[i] = t.slots[i].key;
    __syncthreads();
  } else if (kMember == kMemberBitmap) {
    unsigned* sb = reinterpret_cast<unsigned*>(s_keys);
    for (int i = threadIdx.x; i < kBitWords; i += kHThreads) sb[i] = set_bits[i];
    __syncthreads();
  }
  const bool set_has_null = t.special[1] != kNoRow;
  const bool set_has_ones = t.special[0] != kNoRow;
  auto member = [&](unsigned long long key) -> bool {
    if (kMember == kMemberBitmap) {
      const unsigned* sb = reinterpret_cast<const unsigned*>(s_keys);
      return (sb[(unsigned)key >> 5] >> ((unsigned)key & 31)) & 1u;
    }
    if (sizeof(V) == 8 && key == kEmptyKey) return set_has_ones;      // narrower values zero-extend: never all ones
    unsigned long long h = hash_slot(key, t.shift);
    while (true) {
      unsigned long long k0, k1;
      if (kMember == kMemberSmem) {
        const ulonglong2 pr = *reinterpret_cast<const ulonglong2*>(s_keys + h);   // h is even: one aligned pair
        k0 = pr.x; k1 = pr.y;
      } else {
        k0 = t.slots[h].key; k1 = t.slots[h + 1].key;                             // same 32-byte sector
      }
      if (k0 == key || k1 == key) return true;
      if (k0 == kEmptyKey || k1 == kEmptyKey) return false;
      h = (h + 2) & t.mask;
    }
  };
  const int lane = threadIdx.x & 31;
  const int64_t n_words = (n + 31) >> 5;
  const int64_t warp0 = ((int64_t)blockIdx.x * kHThreads + threadIdx.x) >> 5;
  const int64_t warps = ((int64_t)gridDim.x * kHThreads) >> 5;
  unsigned long long nulls = 0;
  const bool miss_is_null = null_behavior == AG_NULL_INCONCLUSIVE && set_has_null;
  for (int64_t w0 = warp0 * kHUnroll; w0 < n_words; w0 += warps * kHUnroll) {
    if (!valid && ((w0 + kHUnroll) << 5) <= n) {
      // interior, no input nulls: no range tests, no masks; word k of the step is stored by lane k
      // (profile: the edge handling below was half of the 112 instructions per row of this kernel)
      const V* __restrict__ p = vals + off + (w0 << 5) + lane;
      V x[kHUnroll];
#pragma unroll
      for (int k = 0; k < kHUnroll; ++k) x[k] = __ldcs(p + 32 * k);
      uint32_t mine = 0;
#pragma unroll
      for (int k = 0; k < kHUnroll; ++k) {
        const uint32_t dbits = __ballot_sync(0xffffffffu, member((unsigned long long)x[k]));
        if (lane == k) mine = dbits;
      }
      if (lane < kHUnroll) {
        out_data[w0 + lane] = mine;
        if (out_valid) out_valid[w0 + lane] = miss_is_null ? mine : 0xffffffffu;
        if (miss_is_null) nulls += __popc(~mine);
      }
      continue;
    }
    V x[kHUnroll];
    bool have[kHUnroll], isnull[kHUnroll];
#pragma unroll
    for (int k = 0; k < kHUnroll; ++k) {   // independent loads first: 4 rows in flight per lane
      const int64_t i = ((w0 + k) << 5) + lane;
      have[k] = i < n;
      isnull[k] = have[k] && valid && !bit_is_set(valid, off + i);
      x[k] = (have[k] && !isnull[k]) ? __ldcs(vals + off + i) : V(0);
    }
#pragma unroll
    for (int k = 0; k < kHUnroll; ++k) {
      const int64_t w = w0 + k;
      if (w >= n_words) break;   // warp-uniform
      bool d = false, v = true;
      if (have[k]) {
        if (isnull[k]) {
          if (null_behavior == AG_NULL_MATCH && set_has_null) d = true;
          else if (null_behavior == AG_NULL_SKIP || (null_behavior == AG_NULL_MATCH && !set_has_null)) d = false;
          else v = false;
        } else if (member((unsigned long long)x[k])) {
          d = true;
        } else if (null_behavior == AG_NULL_INCONCLUSIVE && set_has_null) {
          v = false;
        }
      }
      const uint32_t dbits = __ballot_sync(0xffffffffu, d);
      const uint32_t vbits = __ballot_sync(0xffffffffu, v);
      if (lane == 0) {
        const int64_t rem = n - (w << 5);
        const uint32_t m = rem >= 32 ? 0xffffffffu : bit_range_mask(0, (int)rem);
        bitmap_store32_masked(out_data + w, dbits, m);
        if (out_valid) bitmap_store32_masked(out_valid + w, vbits, m);
        nulls += __popc(~vbits & m);
      }
    }
  }
  if (lane < kHUnroll && nulls && null_count) atomicAdd(null_count, nulls);
}

// The complete table of a call: `big` (the full-size table; slots == NULL when the call has only one table) when the
// small one overflowed, else the small one.
__device__ __forceinline__ HashTable live_table(const HashTable& small_t, const HashTable& big_t) {
  const bool use_big = big_t.slots && overflowed(small_t);
  HashTable t = use_big ? big_t : small_t;
  t.cap = kNoCap;
  return t;
}

// unique: row i is kept iff it is the first row of its key (or the first null row).
template <typename V>
__global__ void __launch_bounds__(kHThreads)
unique_mark_kernel(const V* __restrict__ vals, const uint8_t* __restrict__ valid, int64_t off, int64_t n, const HashTable small_t,
                   const HashTable big_t, uint32_t* __restrict__ keep) {
  __shared__ unsigned long long s_cache[kHWarps][kWarpCacheSlots];
  const HashTable t = live_table(small_t, big_t);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long* cache = s_cache[warp];
  for (int i = lane; i < kWarpCacheSlots; i += 32) cache[i] = kEmptyKey;
  __syncwarp();
  const unsigned first_ones = t.special[0], first_null = t.special[1];
  const int64_t n_words = (n + 31) >> 5;
  const int64_t warp0 = ((int64_t)blockIdx.x * kHThreads + threadIdx.x) >> 5;
  const int64_t warps = ((int64_t)gridDim.x * kHThreads) >> 5;
  for (int64_t w0 = warp0 * kHUnroll; w0 < n_words; w0 += warps * kHUnroll) {
    V x[kHUnroll];
    int kind[kHUnroll];
    if (!valid && ((w0 + kHUnroll) << 5) <= n) {         // interior, no nulls: unconditional loads
      const V* __restrict__ p = vals + off + (w0 << 5) + lane;
#pragma unroll
      for (int k = 0; k < kHUnroll; ++k) { x[k] = __ldcs(p + 32 * k); kind[k] = 1; }
    } else {
#pragma unroll
      for (int k = 0; k < kHUnroll; ++k) {
        const int64_t i = ((w0 + k) << 5) + lane;
        kind[k] = i < n ? ((valid && !bit_is_set(valid, off + i)) ? 2 : 1) : 0;
        x[k] = kind[k] == 1 ? __ldcs(vals + off + i) : V(0);
      }
    }
#pragma unroll
    for (int k = 0; k < kHUnroll; ++k) {
      const int64_t w = w0 + k;
      if (w >= n_words) break;   // warp-uniform
      const unsigned row = (unsigned)((w << 5) + lane);
      const unsigned long long key = (unsigned long long)x[k];
      const int cs = warp_cache_slot(key);
      const bool ones = sizeof(V) == 8 && key == kEmptyKey;
      bool kp = false;
      if (kind[k] == 2) kp = first_null == row;
      else if (kind[k] == 1 && ones) kp = first_ones == row;
      const bool go = kind[k] == 1 && !ones && cache[cs] != key;   // a cached key sits at a lower row: not first
      __syncwarp();
      if (go) { kp = table_first_row(t, key) == row; atomicExch(&cache[cs], key); }
      __syncwarp();
      const uint32_t bits = __ballot_sync(0xffffffffu, kp);
      if (lane == 0) keep[w] = bits;
    }
  }
}

struct TableMem {
  void* block = nullptr;
  size_t bytes = 0;
  HashTable t{};
  // slots = the power of two >= max(2 * entries, min_slots)
  ag_status alloc(int64_t entries, unsigned long long min_slots, unsigned cap, cudaStream_t st) {
    unsigned long long slots = 1024;
    while (slots < (unsigned long long)entries * 2 || slots < min_slots) slots <<= 1;
    int bits = 0;
    while ((1ull << bits) < slots) ++bits;
    bytes = slots * sizeof(Slot) + 64;
    AG_TRY(dev_alloc_async(&block, bytes, st));
    t.slots = reinterpret_cast<Slot*>(block);
    t.special = reinterpret_cast<unsigned*>(reinterpret_cast<char*>(block) + slots * sizeof(Slot));
    t.mask = slots - 1;
    t.shift = 64 - bits;
    t.cap = cap;
    return AG_OK;
  }
  // every key free, every first row = none, special = {none, none, 0xffffffff (the counter: +1 per key wraps to 0 first), not raised}
  ag_status clear(cudaStream_t st, const unsigned* run_if = nullptr) {
    if (!run_if) { AG_CUDA_TRY(cudaMemsetAsync(block, 0xff, bytes, st)); return AG_OK; }
    table_clear_kernel<<<grid_for((int64_t)(bytes / 16), kHThreads * 8, 8), kHThreads, 0, st>>>(reinterpret_cast<uint4*>(block), (int64_t)(bytes / 16), run_if);
    return check_launch("table_clear_kernel");
  }
  void release(cudaStream_t st) { if (block) cudaFreeAsync(block, st); block = nullptr; }
};

template <typename V>
static ag_status is_in_t(const void* vals, const uint8_t* valid, int64_t off, int64_t n, const void* set, const uint8_t* set_valid, int64_t set_off,
                         int64_t set_n, int null_behavior, uint8_t* out_data, uint8_t* out_valid, int64_t* d_null_count, cudaStream_t st) {
  constexpr bool kSmall = sizeof(V) <= 2;
  TableMem tm;
  // 1-/2-byte values: a 1024-slot block whose first 8 KB hold the membership bitmap (zeroed), `special` behind it as usual
  // others: load factor <= 1/4 while the table still fits the shared-memory copy (a 1000-value set: 4096 slots = 32 KB,
  // six blocks per SM), <= 1/2 beyond
  unsigned long long min_slots = 1024;
  if (!kSmall) { while (min_slots < (unsigned long long)set_n * 4 && min_slots < (unsigned long long)kIsInSmemSlots) min_slots <<= 1; }
  AG_TRY(tm.alloc(kSmall ? 0 : set_n, min_slots, kNoCap, st));
  ag_status rc = tm.clear(st);
  unsigned* bits = reinterpret_cast<unsigned*>(tm.block);
  do {
    if (rc != AG_OK) break;
    if (kSmall && cudaMemsetAsync(bits, 0, 8192, st) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "memset", __FILE__, __LINE__); break; }
    if (set_n > 0) {
      if constexpr (kSmall) set_bitmap_kernel<V><<<grid_for(set_n, kHThreads, 8), kHThreads, 0, st>>>(reinterpret_cast<const V*>(set), set_valid, set_off, set_n, bits, tm.t.special);
      else hash_insert_kernel<V><<<grid_for(set_n, kHThreads * kHUnroll, 8), kHThreads, 0, st>>>(reinterpret_cast<const V*>(set), set_valid, set_off, set_n, tm.t, nullptr, 0u);
      if ((rc = check_launch("is_in set kernel")) != AG_OK) break;
    }
    if (d_null_count && cudaMemsetAsync(d_null_count, 0, 8, st) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "memset", __FILE__, __LINE__); break; }
    uint32_t* od = reinterpret_cast<uint32_t*>(out_data);
    uint32_t* ov = reinterpret_cast<uint32_t*>(out_valid);
    unsigned long long* nc = reinterpret_cast<unsigned long long*>(d_null_count);
    const V* v = reinterpret_cast<const V*>(vals);
    if constexpr (kSmall) {
      is_in_kernel<V, kMemberBitmap><<<grid_for(n, kHThreads * kHUnroll, 8), kHThreads, 8192, st>>>(v, valid, off, n, tm.t, bits, null_behavior, od, ov, nc);
    } else if (tm.t.mask < (unsigned long long)kIsInSmemSlots) {
      const int smem = (int)((tm.t.mask + 1) * 8);
      static std::atomic<unsigned> attr_set{0u};   // per V, one bit per device
      if ((rc = ensure_dynamic_smem((const void*)is_in_kernel<V, kMemberSmem>, kIsInSmemSlots * 8, &attr_set)) != AG_OK) break;
      const int per_sm = smem > 32768 ? 3 : (smem > 16384 ? 6 : 8);
      is_in_kernel<V, kMemberSmem><<<grid_for(n, kHThreads * kHUnroll, per_sm), kHThreads, smem, st>>>(v, valid, off, n, tm.t, nullptr, null_behavior, od, ov, nc);
    } else {
      is_in_kernel<V, kMemberTable><<<grid_for(n, kHThreads * kHUnroll, 8), kHThreads, 0, st>>>(v, valid, off, n, tm.t, nullptr, null_behavior, od, ov, nc);
    }
    rc = check_launch("is_in_kernel");
  } while (0);
  tm.release(st);
  return rc;
}

ag_status is_in_dev(int bit_width, const void* vals, const uint8_t* valid, int64_t off, int64_t n, const void* set, const uint8_t* set_valid,
                    int64_t set_off, int64_t set_n, int null_behavior, uint8_t* out_data, uint8_t* out_valid, int64_t* d_null_count, cudaStream_t st) {
  if (n < 0 || set_n < 0 || off < 0 || set_off < 0) AG_FAIL(AG_ERR_INVALID, "is_in: negative length or offset");
  if (null_behavior < 0 || null_behavior > 3) AG_FAIL(AG_ERR_INVALID, "is_in: bad null matching behaviour %d", null_behavior);
  if (n == 0) return AG_OK;
  if (!vals || !out_data || (set_n > 0 && !set)) AG_FAIL(AG_ERR_INVALID, "is_in: NULL values / value set / output");
  if ((reinterpret_cast<uintptr_t>(out_data) & 3) || (reinterpret_cast<uintptr_t>(out_valid) & 3)) AG_FAIL(AG_ERR_INVALID, "is_in: output bitmaps must be 4-byte aligned");
  if (set_n >= (1ll << 31)) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "is_in: value set too large");
  return visit_width(bit_width, [&](auto tag) {
    return is_in_t<typename decltype(tag)::type>(vals, valid, off, n, set, set_valid, set_off, set_n, null_behavior, out_data, out_valid,
                                                 d_null_count, st);
  }, [&] { AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "is_in: fixed-width values of 1/2/4/8 bytes only (got %d bits)", bit_width); });
}

// columns above `small_rows` try a table of `small_slots` slots (2M x 16 B = 32 MB: resident in H100's 50 MB L2) first
static std::atomic<long long> g_unique_small_rows{1ll << 21};
static std::atomic<long long> g_unique_small_slots{1ll << 21};

template <typename V>
static ag_status unique_t(int bit_width, const void* vals, const uint8_t* valid, int64_t off, int64_t n, void* out, uint8_t* out_valid,
                          int64_t capacity, int64_t* d_out_len, cudaStream_t st) {
  const bool two = n > g_unique_small_rows.load(std::memory_order_relaxed);
  const unsigned long long small_slots = (unsigned long long)g_unique_small_slots.load(std::memory_order_relaxed);
  TableMem small_t, big_t;
  uint32_t* keep = nullptr;
  ag_status rc = AG_OK;
  do {
    if (two) rc = small_t.alloc(0, small_slots, (unsigned)(small_slots / 2), st);
    else rc = small_t.alloc(n, 1024, kNoCap, st);
    if (rc != AG_OK) break;
    if ((rc = small_t.clear(st)) != AG_OK) break;
    if (two && (rc = big_t.alloc(n, 1024, kNoCap, st)) != AG_OK) break;
    if ((rc = dev_alloc_async((void**)&keep, (size_t)((n + 31) / 32) * 4 + 64, st)) != AG_OK) break;
    const V* v = reinterpret_cast<const V*>(vals);
    const int grid = grid_for(n, kHThreads * kHUnroll, 8);
    hash_insert_kernel<V><<<grid, kHThreads, 0, st>>>(v, valid, off, n, small_t.t, nullptr, 0u);
    if ((rc = check_launch("hash_insert_kernel")) != AG_OK) break;
    if (two) {
      const unsigned* raised = small_t.t.special + 3;
      if ((rc = big_t.clear(st, raised)) != AG_OK) break;
      hash_insert_kernel<V><<<grid, kHThreads, 0, st>>>(v, valid, off, n, big_t.t, raised, 0u);
      if ((rc = check_launch("hash_insert_kernel")) != AG_OK) break;
    }
    unique_mark_kernel<V><<<grid, kHThreads, 0, st>>>(v, valid, off, n, small_t.t, big_t.t, keep);
    if ((rc = check_launch("unique_mark_kernel")) != AG_OK) break;
    if (out_valid) {
      if (cudaMemsetAsync(out_valid, 0, (size_t)((capacity + 31) / 32) * 4, st) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "memset", __FILE__, __LINE__); break; }
    }
    rc = filter_primitive_dev(bit_width, vals, valid, off, reinterpret_cast<const uint8_t*>(keep), nullptr, 0, n, AG_DROP_NULLS, out, out_valid,
                              capacity, d_out_len, st);
  } while (0);
  if (keep) cudaFreeAsync(keep, st);
  small_t.release(st);
  big_t.release(st);
  return rc;
}

ag_status unique_dev(int bit_width, const void* vals, const uint8_t* valid, int64_t off, int64_t n, void* out, uint8_t* out_valid, int64_t capacity,
                     int64_t* d_out_len, cudaStream_t st) {
  if (n < 0 || off < 0 || capacity < 0) AG_FAIL(AG_ERR_INVALID, "unique: negative length or offset");
  if (!d_out_len) AG_FAIL(AG_ERR_INVALID, "unique: NULL length word");
  if (n == 0) { AG_CUDA_TRY(cudaMemsetAsync(d_out_len, 0, sizeof(int64_t), st)); return AG_OK; }
  if (!vals || (!out && capacity > 0)) AG_FAIL(AG_ERR_INVALID, "unique: NULL values/output");
  if (valid && !out_valid && capacity > 0) AG_FAIL(AG_ERR_INVALID, "unique: an input with a validity bitmap needs an output validity bitmap");
  if (n >= (1ll << 31)) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "unique: more than 2^31-1 rows per call");
  return visit_width(bit_width, [&](auto tag) {
    return unique_t<typename decltype(tag)::type>(bit_width, vals, valid, off, n, out, out_valid, capacity, d_out_len, st);
  }, [&] { AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "unique: fixed-width values of 1/2/4/8 bytes only (got %d bits)", bit_width); });
}

// ---- dictionary_encode ----------------------------------------------------------------------------------------------
// After `unique`'s inserts over every chunk (rows numbered across chunks), a key's dictionary index is the number of
// first rows below its own first row: the rank of its bit in an n-bit bitmap of first rows.
//   dict_first_bits_kernel  sets bit `first` of every live slot, of the all-ones key and (Encode) of the null;
//   popcounts of the bitmap words -> cumulative_sum (scan.cu) -> inclusive word counts;
//   dict_rank_kernel        writes each slot's rank into Slot::pad and the key into dict[rank], the ranks of the
//                           all-ones key and of the null into special[4] / special[5], and the dictionary length;
//   dict_index_kernel       probes the table for every row of a chunk: coalesced int32 indices, ballot validity.
// special[4] / special[5] keep the clear's all-ones until the rank pass writes them.

__global__ void __launch_bounds__(kHThreads)
dict_first_bits_kernel(const HashTable small_t, const HashTable big_t, int encode_null, uint32_t* __restrict__ bits) {
  const HashTable t = live_table(small_t, big_t);
  const int64_t slots = (int64_t)t.mask + 1;
  for (int64_t i = (int64_t)blockIdx.x * kHThreads + threadIdx.x; i < slots; i += (int64_t)gridDim.x * kHThreads) {
    const ulonglong2 raw = __ldcs(reinterpret_cast<const ulonglong2*>(t.slots + i));
    if (raw.x != kEmptyKey) { const unsigned f = (unsigned)raw.y; atomicOr(&bits[f >> 5], 1u << (f & 31)); }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const unsigned ones = t.special[0], null_row = t.special[1];
    if (ones != kNoRow) atomicOr(&bits[ones >> 5], 1u << (ones & 31));
    if (encode_null && null_row != kNoRow) atomicOr(&bits[null_row >> 5], 1u << (null_row & 31));
  }
}

__global__ void __launch_bounds__(kHThreads)
bit_word_popc_kernel(const uint32_t* __restrict__ bits, int64_t n_words, int* __restrict__ counts) {
  for (int64_t i = (int64_t)blockIdx.x * kHThreads + threadIdx.x; i < n_words; i += (int64_t)gridDim.x * kHThreads) counts[i] = __popc(bits[i]);
}

// rank of row f (a set bit): the set bits below it
__device__ __forceinline__ unsigned first_row_rank(const uint32_t* __restrict__ bits, const int* __restrict__ incl, unsigned f) {
  return (unsigned)incl[f >> 5] - (unsigned)__popc(bits[f >> 5] >> (f & 31));
}

template <typename V>
__global__ void __launch_bounds__(kHThreads)
dict_rank_kernel(const HashTable small_t, const HashTable big_t, int encode_null, const uint32_t* __restrict__ bits,
                 const int* __restrict__ incl, int64_t n_words, V* __restrict__ dict, uint8_t* __restrict__ dict_valid,
                 int64_t* __restrict__ dict_len) {   // dict_len: {dictionary length, dictionary null count}, cleared
  const HashTable t = live_table(small_t, big_t);
  const int64_t slots = (int64_t)t.mask + 1;
  for (int64_t i = (int64_t)blockIdx.x * kHThreads + threadIdx.x; i < slots; i += (int64_t)gridDim.x * kHThreads) {
    const ulonglong2 raw = *reinterpret_cast<const ulonglong2*>(t.slots + i);
    if (raw.x == kEmptyKey) continue;
    const unsigned r = first_row_rank(bits, incl, (unsigned)raw.y);
    t.slots[i].pad = r;
    if (dict) dict[r] = (V)raw.x;   // NULL: ranks only (byte-array keys are hashes)
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const unsigned ones = t.special[0], null_row = t.special[1];
    if (ones != kNoRow) { const unsigned r = first_row_rank(bits, incl, ones); t.special[4] = r; dict[r] = (V)kEmptyKey; }
    if (encode_null && null_row != kNoRow) {
      const unsigned r = first_row_rank(bits, incl, null_row);
      t.special[5] = r;
      dict[r] = V(0);
      if (dict_valid) dict_valid[r >> 3] &= (uint8_t)~(1u << (r & 7));
      dict_len[1] = 1;   // the dictionary's null count
    }
    dict_len[0] = incl[n_words - 1];
  }
}

// the dictionary index of a key of the complete table
__device__ __forceinline__ unsigned table_index(const HashTable& t, unsigned long long key) {
  unsigned long long h = hash_slot(key, t.shift);
  while (true) {
    const ulonglong2 raw = *reinterpret_cast<const ulonglong2*>(t.slots + h);
    if (raw.x == key) return (unsigned)(raw.y >> 32);   // Slot::pad
    h = (h + 1) & t.mask;
  }
}

// indices of one chunk; `out_valid` (Mask mode, chunk with a validity bitmap) gets one ballot word per 32 rows
template <typename V>
__global__ void __launch_bounds__(kHThreads)
dict_index_kernel(const V* __restrict__ vals, const uint8_t* __restrict__ valid, int64_t off, int64_t n, const HashTable small_t,
                  const HashTable big_t, int encode_null, int32_t* __restrict__ out, uint32_t* __restrict__ out_valid,
                  unsigned long long* __restrict__ null_count) {
  const HashTable t = live_table(small_t, big_t);
  const unsigned ones_index = t.special[4];
  const unsigned null_index = encode_null ? t.special[5] : 0u;
  const int lane = threadIdx.x & 31;
  const int64_t n_words = (n + 31) >> 5;
  const int64_t warp0 = ((int64_t)blockIdx.x * kHThreads + threadIdx.x) >> 5;
  const int64_t warps = ((int64_t)gridDim.x * kHThreads) >> 5;
  unsigned long long nulls = 0;
  for (int64_t w0 = warp0 * kHUnroll; w0 < n_words; w0 += warps * kHUnroll) {
    V x[kHUnroll];
    int kind[kHUnroll];                                  // 0 nothing, 1 value, 2 null
    if (!valid && ((w0 + kHUnroll) << 5) <= n) {         // interior, no nulls: unconditional loads
      const V* __restrict__ p = vals + off + (w0 << 5) + lane;
#pragma unroll
      for (int k = 0; k < kHUnroll; ++k) { x[k] = __ldcs(p + 32 * k); kind[k] = 1; }
    } else {
#pragma unroll
      for (int k = 0; k < kHUnroll; ++k) {
        const int64_t i = ((w0 + k) << 5) + lane;
        kind[k] = i < n ? ((valid && !bit_is_set(valid, off + i)) ? 2 : 1) : 0;
        x[k] = kind[k] == 1 ? __ldcs(vals + off + i) : V(0);
      }
    }
#pragma unroll
    for (int k = 0; k < kHUnroll; ++k) {
      const int64_t w = w0 + k;
      if (w >= n_words) break;   // warp-uniform
      const int64_t i = (w << 5) + lane;
      const unsigned long long key = (unsigned long long)x[k];
      unsigned idx = null_index;
      if (kind[k] == 1) idx = (sizeof(V) == 8 && key == kEmptyKey) ? ones_index : table_index(t, key);
      if (kind[k]) __stcs(out + i, (int32_t)idx);
      if (out_valid) {
        const uint32_t vbits = __ballot_sync(0xffffffffu, kind[k] == 1);
        if (lane == 0) {
          const int64_t rem = n - (w << 5);
          const uint32_t m = rem >= 32 ? 0xffffffffu : bit_range_mask(0, (int)rem);
          out_valid[w] = vbits;
          nulls += __popc(~vbits & m);
        }
      }
    }
  }
  if (lane == 0 && nulls) atomicAdd(null_count, nulls);
}

template <typename V>
static ag_status dictionary_encode_t(const ag_dict_chunk* chunks, int64_t n_chunks, int64_t total, int null_encoding, void* dict,
                                     uint8_t* dict_valid, int64_t* d_counts, cudaStream_t st) {
  const bool two = total > g_unique_small_rows.load(std::memory_order_relaxed);
  const unsigned long long small_slots = (unsigned long long)g_unique_small_slots.load(std::memory_order_relaxed);
  const int encode = null_encoding == AG_NULL_ENCODING_ENCODE;
  const int64_t n_words = (total + 31) / 32;
  TableMem small_t, big_t;
  void* scratch = nullptr;
  ag_status rc = AG_OK;
  do {
    if (two) rc = small_t.alloc(0, small_slots, (unsigned)(small_slots / 2), st);
    else rc = small_t.alloc(total, 1024, kNoCap, st);
    if (rc != AG_OK) break;
    if ((rc = small_t.clear(st)) != AG_OK) break;
    if (two && (rc = big_t.alloc(total, 1024, kNoCap, st)) != AG_OK) break;
    // first-row bitmap | word popcounts | their inclusive scan | scan state, each region 256-byte aligned (the scan
    // reads and writes whole vectors)
    const size_t words_b = ((size_t)n_words * 4 + 255) & ~(size_t)255;
    if ((rc = dev_alloc_async(&scratch, 3 * words_b + 64, st)) != AG_OK) break;
    uint32_t* bits = static_cast<uint32_t*>(scratch);
    int* counts = reinterpret_cast<int*>(static_cast<char*>(scratch) + words_b);
    int* incl = reinterpret_cast<int*>(static_cast<char*>(scratch) + 2 * words_b);
    void* scan_state = static_cast<char*>(scratch) + 3 * words_b;
    if (cudaMemsetAsync(bits, 0, words_b, st) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "memset", __FILE__, __LINE__); break; }
    if (encode && dict_valid && cudaMemsetAsync(dict_valid, 0xff, (size_t)((total + 7) / 8), st) != cudaSuccess) {
      rc = cuda_fail(cudaGetLastError(), "memset", __FILE__, __LINE__); break;
    }
    // inserts: every chunk into the small table, then (only when it overflowed) every chunk into the full-size one
    for (int pass = 0; pass < (two ? 2 : 1) && rc == AG_OK; ++pass) {
      const unsigned* raised = pass ? small_t.t.special + 3 : nullptr;
      if (pass && (rc = big_t.clear(st, raised)) != AG_OK) break;
      int64_t row = 0;
      for (int64_t c = 0; c < n_chunks; ++c) {
        const ag_dict_chunk& ch = chunks[c];
        if (ch.length == 0) continue;
        hash_insert_kernel<V><<<grid_for(ch.length, kHThreads * kHUnroll, 8), kHThreads, 0, st>>>(
            reinterpret_cast<const V*>(ch.values), ch.validity, ch.offset, ch.length, pass ? big_t.t : small_t.t, raised, (unsigned)row);
        if ((rc = check_launch("hash_insert_kernel")) != AG_OK) break;
        row += ch.length;
      }
    }
    if (rc != AG_OK) break;
    // ranks; grids cover the largest table the call may have ended on
    const int64_t max_slots = (int64_t)((two ? big_t.t.mask : small_t.t.mask) + 1);
    const int slot_grid = grid_for(max_slots, kHThreads * 4, 8);
    dict_first_bits_kernel<<<slot_grid, kHThreads, 0, st>>>(small_t.t, big_t.t, encode, bits);
    if ((rc = check_launch("dict_first_bits_kernel")) != AG_OK) break;
    bit_word_popc_kernel<<<grid_for(n_words, kHThreads * 4, 8), kHThreads, 0, st>>>(bits, n_words, counts);
    if ((rc = check_launch("bit_word_popc_kernel")) != AG_OK) break;
    if ((rc = cumulative_sum_state_init(scan_state, AG_TYPE_INT32, nullptr, st)) != AG_OK) break;
    if ((rc = cumulative_sum_dev(AG_TYPE_INT32, counts, nullptr, 0, n_words, 0, 0, incl, nullptr, 0, scan_state, nullptr, st)) != AG_OK) break;
    dict_rank_kernel<V><<<slot_grid, kHThreads, 0, st>>>(small_t.t, big_t.t, encode, bits, incl, n_words, reinterpret_cast<V*>(dict),
                                                        encode ? dict_valid : nullptr, d_counts);
    if ((rc = check_launch("dict_rank_kernel")) != AG_OK) break;
    // indices
    for (int64_t c = 0; c < n_chunks; ++c) {
      const ag_dict_chunk& ch = chunks[c];
      if (ch.length == 0) continue;
      uint32_t* ov = (!encode && ch.validity) ? reinterpret_cast<uint32_t*>(ch.indices_validity) : nullptr;
      dict_index_kernel<V><<<grid_for(ch.length, kHThreads * kHUnroll, 8), kHThreads, 0, st>>>(
          reinterpret_cast<const V*>(ch.values), ch.validity, ch.offset, ch.length, small_t.t, big_t.t, encode, ch.indices, ov,
          reinterpret_cast<unsigned long long*>(d_counts + 2 + c));
      if ((rc = check_launch("dict_index_kernel")) != AG_OK) break;
    }
  } while (0);
  if (scratch) cudaFreeAsync(scratch, st);
  small_t.release(st);
  big_t.release(st);
  return rc;
}

ag_status dictionary_encode_dev(int bit_width, const ag_dict_chunk* chunks, int64_t n_chunks, int null_encoding, void* dict,
                                uint8_t* dict_valid, int64_t* d_counts, cudaStream_t st) {
  if (null_encoding != AG_NULL_ENCODING_MASK && null_encoding != AG_NULL_ENCODING_ENCODE)
    AG_FAIL(AG_ERR_INVALID, "dictionary_encode: invalid null encoding %d", null_encoding);
  if (n_chunks < 0 || (n_chunks > 0 && !chunks)) AG_FAIL(AG_ERR_INVALID, "dictionary_encode: bad chunk table");
  if (!d_counts) AG_FAIL(AG_ERR_INVALID, "dictionary_encode: NULL counts");
  if (bit_width != 8 && bit_width != 16 && bit_width != 32 && bit_width != 64)
    AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "dictionary_encode: fixed-width values of 1/2/4/8 bytes only (got %d bits)", bit_width);
  int64_t total = 0;
  bool any_valid = false;
  for (int64_t c = 0; c < n_chunks; ++c) {
    const ag_dict_chunk& ch = chunks[c];
    if (ch.length < 0 || ch.offset < 0) AG_FAIL(AG_ERR_INVALID, "dictionary_encode: chunk %lld: negative length or offset", (long long)c);
    if (ch.length == 0) continue;
    if (!ch.values || !ch.indices) AG_FAIL(AG_ERR_INVALID, "dictionary_encode: chunk %lld: NULL values or indices", (long long)c);
    if (null_encoding == AG_NULL_ENCODING_MASK && ch.validity && !ch.indices_validity)
      AG_FAIL(AG_ERR_INVALID, "dictionary_encode: chunk %lld: a chunk with a validity bitmap needs an index validity bitmap", (long long)c);
    if (reinterpret_cast<uintptr_t>(ch.indices_validity) & 3)
      AG_FAIL(AG_ERR_INVALID, "dictionary_encode: chunk %lld: the index validity bitmap must be 4-byte aligned", (long long)c);
    any_valid |= ch.validity != nullptr;
    total += ch.length;
    if (total >= (1ll << 31)) AG_FAIL(AG_ERR_NOT_IMPLEMENTED, "dictionary_encode: more than 2^31-1 rows per call");
  }
  if (total > 0 && !dict) AG_FAIL(AG_ERR_INVALID, "dictionary_encode: NULL dictionary");
  if (null_encoding == AG_NULL_ENCODING_ENCODE && any_valid && !dict_valid)
    AG_FAIL(AG_ERR_INVALID, "dictionary_encode: encoding the nulls of an input with validity bitmaps needs a dictionary validity bitmap");
  AG_CUDA_TRY(cudaMemsetAsync(d_counts, 0, (size_t)(n_chunks + 2) * sizeof(int64_t), st));
  if (total == 0) return AG_OK;
  return visit_width(bit_width, [&](auto tag) {
    return dictionary_encode_t<typename decltype(tag)::type>(chunks, n_chunks, total, null_encoding, dict, dict_valid, d_counts, st);
  }, [] { return AG_OK; });   // the width was checked above
}


// ---- BYTE_ARRAY dictionaries (DictByteArrayEncoder) -----------------------------------------------------------------
// The same table, ranks and two-table policy as dictionary_encode, over slots numbered across the chunks of a column
// chunk.  A slot's key is a 64-bit hash of the value's bytes (never the all-ones pattern), and a key match counts only
// once the bytes compare equal to the row in Slot::first: that field is only ever lowered to rows whose bytes matched,
// so it always holds a row carrying the value.  Unequal values with equal hashes probe on.  The creator of a slot
// publishes its row right after its key CAS, and a lane that finds the key before the row waits for it.
//   ba_dict_insert_kernel   one 1024-slot tile of a chunk per block step (the checking pass's tiles, whose valid
//                           counts give every valid slot its dense position); each warp walks 4 steps of 32 slots in
//                           slot order.  Values up to kBaWarpLen bytes are hashed and compared by their lane, longer ones
//                           by the whole warp, one at a time.  The hash sums one mix per 16-byte piece, so both ways
//                           give the same key.  A per-warp cache of values met at lower slots {hash, bytes, table slot}
//                           answers repeats without touching the table (hits are confirmed by comparing bytes).  Every
//                           valid slot records its table slot at its dense position (4 B per valid value), so the index
//                           pass does not hash again.
//   dict_first_bits_kernel, bit_word_popc_kernel, cumulative_sum, dict_rank_kernel (ranks only): as dictionary_encode.
//   ba_dict_word_bytes_kernel  len + 4 of the first rows of every bitmap word; its scan and the word-count scan
//                           answer the marks (ba_dict_marks_kernel: the scans at the mark's word, plus the partial word).
//                           Scanning per word keeps the scan's length known on the host (the entry count is not).
//   ba_dict_index_kernel    the rank of every valid slot's table slot, coalesced uint32 at its dense position.
//   ba_dict_first_kernel    per chunk: the first-row bitmap rebased to the chunk's slot numbering, whole words.
// Bytes: offsets and validity read by the checking pass and again by the insert pass, data read once (repeats from the
// cache, L1 or L2), 4 B per valid slot written and read back, indices written, bitmaps ~1 bit per slot.

constexpr int kBaWarpLen = 256;        // longer values are hashed and compared by a whole warp
constexpr int kBaCacheSlots = 128;     // per warp
static_assert(kBaTile == kHThreads * kHUnroll, "a warp's 4 steps of 32 slots cover its share of a tile");

struct BaCache {
  unsigned long long key[kBaCacheSlots];   // kEmptyKey: free
  const uint8_t* ptr[kBaCacheSlots];
  uint2 len_slot[kBaCacheSlots];           // {value length, table slot}
};

// the bytes of global slot `row`
template <typename O>
__device__ __forceinline__ const uint8_t* ba_value(const BaDictPlan& p, unsigned row, int64_t& len) {
  const int64_t c = find_page(p.row_base, p.n_chunks, row);
  const ag_pq_ba_chunk& ch = p.chunks[c];
  const O* o = static_cast<const O*>(ch.offsets) + ch.offset + ((int64_t)row - p.row_base[c]);
  const int64_t o0 = (int64_t)o[0];
  len = (int64_t)o[1] - o0;
  return ch.data + o0;
}

// piece k of a value: its bytes [16k, 16k + 16), zero-padded past the value's end
__device__ __forceinline__ unsigned long long piece_mix(const uint8_t* p, int64_t len, int64_t k) {
  const u128 w = window(p + 16 * k, len - 16 * k < 16 ? (int)(len - 16 * k) : 16);
  return mix64((unsigned long long)w ^ mix64((unsigned long long)(w >> 64) + (unsigned long long)k * 0x9E3779B97F4A7C15ull));
}
__device__ __forceinline__ unsigned long long finish_hash(unsigned long long sum, int64_t len) {
  const unsigned long long h = mix64(sum ^ (unsigned long long)len);
  return h == kEmptyKey ? 0ull : h;
}
__device__ __forceinline__ unsigned long long thread_hash(const uint8_t* p, int64_t len) {
  unsigned long long s = 0;
  for (int64_t k = 0; 16 * k < len; ++k) s += piece_mix(p, len, k);
  return finish_hash(s, len);
}
__device__ __forceinline__ unsigned long long warp_hash(const uint8_t* p, int64_t len, int lane) {
  unsigned long long s = 0;
  for (int64_t k = lane; 16 * k < len; k += 32) s += piece_mix(p, len, k);
#pragma unroll
  for (int m = 16; m; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
  return finish_hash(s, len);
}
__device__ __forceinline__ bool thread_equal(const uint8_t* x, const uint8_t* y, int64_t len) {
  if (x == y) return true;
  for (int64_t k = 0; k < len; k += 16) {
    const int c = len - k < 16 ? (int)(len - k) : 16;
    if (window(x + k, c) != window(y + k, c)) return false;
  }
  return true;
}
__device__ __forceinline__ bool warp_equal(const uint8_t* x, const uint8_t* y, int64_t len, int lane) {
  bool ne = false;
  if (x != y)
    for (int64_t k = 16 * lane; k < len && !ne; k += 512) {
      const int c = len - k < 16 ? (int)(len - k) : 16;
      ne = window(x + k, c) != window(y + k, c);
    }
  return !__any_sync(0xffffffffu, ne);
}

// The table slot of value v (len bytes) at global slot `row`, -1 when a capped table gives up.  WARP: every lane of
// the warp calls it with the same arguments; lane 0 makes the atomic updates.
template <bool WARP, typename O>
__device__ __forceinline__ long long ba_table_insert(const HashTable& t, const BaDictPlan& p, unsigned long long key, unsigned row,
                                                    const uint8_t* v, int64_t len, bool& made, int lane) {
  unsigned long long h = hash_slot(key, t.shift);
  unsigned probes = 0;
  made = false;
  while (true) {
    Slot* s = t.slots + h;
    const ulonglong2 raw = __ldcg(reinterpret_cast<const ulonglong2*>(s));
    unsigned long long cur = raw.x;
    unsigned seen = (unsigned)raw.y;
    if (cur == kEmptyKey) {
      if (!WARP || lane == 0) {
        cur = atomicCAS(&s->key, kEmptyKey, key);
        if (cur == kEmptyKey) atomicExch(&s->first, row);   // publish the row before anything else
      }
      if (WARP) cur = __shfl_sync(0xffffffffu, cur, 0);
      if (cur == kEmptyKey) { made = true; return (long long)h; }
      seen = kNoRow;
    }
    if (cur == key) {
      while (seen == kNoRow) seen = *reinterpret_cast<volatile unsigned*>(&s->first);   // its creator is publishing it
      if (WARP) seen = __shfl_sync(0xffffffffu, seen, 0);
      int64_t flen;
      const uint8_t* f = ba_value<O>(p, seen, flen);
      if (flen == len && (WARP ? warp_equal(f, v, len, lane) : thread_equal(f, v, len))) {
        if (!WARP || lane == 0) lower_row(&s->first, seen, row);
        return (long long)h;
      }
    }
    h = (h + 1) & t.mask;
    bool stop = probe_gives_up(t, probes);
    if (WARP) stop = __shfl_sync(0xffffffffu, stop, 0);
    if (stop) return -1;
  }
}

// `run_if`: NULL, or the small table's overflow word (the full-size pass)
template <typename O>
__global__ void __launch_bounds__(kHThreads, 3)
ba_dict_insert_kernel(const BaDictPlan p, uint32_t* __restrict__ ref, const HashTable t, const unsigned* __restrict__ run_if) {
  __shared__ BaCache s_cache[kHWarps];
  __shared__ unsigned s_cnt[kHWarps];
  if (run_if && *run_if != 1u) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt = (1u << lane) - 1u;
  BaCache& cache = s_cache[warp];
  for (int i = lane; i < kBaCacheSlots; i += 32) cache.key[i] = kEmptyKey;
  __syncwarp();
  for (int64_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    if (__syncthreads_or(t.cap != kNoCap && overflowed(t))) return;   // the small table is being abandoned
    const int64_t c = find_page(p.tile_base, p.n_chunks, tile);
    const ag_pq_ba_chunk ch = p.chunks[c];
    const O* offs = static_cast<const O*>(ch.offsets) + ch.offset;
    const int64_t j0 = (tile - p.tile_base[c]) * kBaTile + warp * (32 * kHUnroll);   // the warp's first slot in the chunk
    auto valid_at = [&](int64_t j) { return j < ch.length && (!ch.valid || bit_is_set(ch.valid, ch.offset + j)); };
    unsigned cnt = 0;
#pragma unroll
    for (int k = 0; k < kHUnroll; ++k) cnt += __popc(__ballot_sync(0xffffffffu, valid_at(j0 + 32 * k + lane)));
    if (lane == 0) s_cnt[warp] = cnt;
    __syncthreads();   // s_cnt is written again only after the next step's barrier
    int64_t d = p.dense[c] + (int64_t)p.tile_cnt[tile + c];
    for (int w = 0; w < warp; ++w) d += s_cnt[w];
    const unsigned row0 = (unsigned)(p.row_base[c] + j0);
#pragma unroll 1
    for (int k = 0; k < kHUnroll; ++k) {
      const int64_t j = j0 + 32 * k + lane;
      const bool v = valid_at(j);
      const unsigned vb = __ballot_sync(0xffffffffu, v);
      const unsigned row = row0 + 32 * k + lane;
      const int64_t o0 = v ? (int64_t)offs[j] : 0;
      const uint8_t* ptr = ch.data + o0;
      const int64_t len = v ? (int64_t)offs[j + 1] - o0 : 0;
      unsigned long long key = 0;
      long long slot = -1;
      bool hit = false, made = false;
      int cs = 0;
      if (v && len <= kBaWarpLen) {
        key = thread_hash(ptr, len);
        cs = warp_cache_slot(key) & (kBaCacheSlots - 1);
        hit = cache.key[cs] == key && cache.len_slot[cs].x == (unsigned)len && thread_equal(cache.ptr[cs], ptr, len);
        if (hit) slot = cache.len_slot[cs].y;
      }
      for (unsigned m = __ballot_sync(0xffffffffu, v && len > kBaWarpLen); m; m &= m - 1) {   // long values, one at a time
        const int src = __ffs(m) - 1;
        const uint8_t* q = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(ptr), src));
        const int64_t ql = __shfl_sync(0xffffffffu, len, src);
        const unsigned long long qk = warp_hash(q, ql, lane);
        const int qs = warp_cache_slot(qk) & (kBaCacheSlots - 1);
        long long qslot = -1;
        bool qmade = false;
        const bool qhit = cache.key[qs] == qk && cache.len_slot[qs].x == (unsigned)ql && warp_equal(cache.ptr[qs], q, ql, lane);
        if (qhit) qslot = cache.len_slot[qs].y;
        else qslot = ba_table_insert<true, O>(t, p, qk, row0 + 32 * k + src, q, ql, qmade, lane);
        if (lane == src) { key = qk; cs = qs; hit = qhit; slot = qslot; made = qmade; }
      }
      __syncwarp();
      if (v && len <= kBaWarpLen && !hit) slot = ba_table_insert<false, O>(t, p, key, row, ptr, len, made, lane);
      __syncwarp();
      // the cache keeps one of the values that went to the table per cache slot (lanes may share a slot)
      const bool go = v && !hit && slot >= 0;
      const unsigned same = __match_any_sync(0xffffffffu, go ? cs : kBaCacheSlots + lane);
      if (go && lane == __ffs(same) - 1) {
        cache.key[cs] = key;
        cache.ptr[cs] = ptr;
        cache.len_slot[cs] = make_uint2((unsigned)len, (unsigned)slot);
      }
      if (v && slot >= 0) ref[d + __popc(vb & lt)] = (uint32_t)slot;
      d += __popc(vb);
      __syncwarp();   // the cache writes are seen by the next step
      count_made(t, made, lane);
    }
  }
}

// len + 4 of the first rows of every word of the first-row bitmap
template <typename O>
__global__ void __launch_bounds__(kHThreads)
ba_dict_word_bytes_kernel(const BaDictPlan p, const uint32_t* __restrict__ bits, int64_t n_words, long long* __restrict__ wbytes) {
  for (int64_t i = (int64_t)blockIdx.x * kHThreads + threadIdx.x; i < n_words; i += (int64_t)gridDim.x * kHThreads) {
    long long s = 0;
    for (uint32_t b = bits[i]; b; b &= b - 1) {
      int64_t len;
      ba_value<O>(p, (unsigned)(i * 32 + __ffs(b) - 1), len);
      s += len + 4;
    }
    wbytes[i] = s;
  }
}

// incl / wscan: inclusive scans of the bitmap words' entries and bytes
template <typename O>
__global__ void __launch_bounds__(kHThreads)
ba_dict_marks_kernel(const BaDictPlan p, const uint32_t* __restrict__ bits, const int* __restrict__ incl,
                     const long long* __restrict__ wscan, int64_t n_words, const int64_t* __restrict__ marks, int64_t n_marks,
                     int64_t* __restrict__ mark_counts, int64_t* __restrict__ counts) {
  for (int64_t j = (int64_t)blockIdx.x * kHThreads + threadIdx.x; j < n_marks; j += (int64_t)gridDim.x * kHThreads) {
    const int64_t m = marks[j], w = m >> 5;
    long long e = w ? incl[w - 1] : 0, s = w ? wscan[w - 1] : 0;
    if (m & 31) {
      for (uint32_t b = bits[w] & ((1u << (m & 31)) - 1u); b; b &= b - 1) {
        int64_t len;
        ba_value<O>(p, (unsigned)(w * 32 + __ffs(b) - 1), len);
        ++e;
        s += len + 4;
      }
    }
    mark_counts[2 * j] = e;
    mark_counts[2 * j + 1] = s;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    counts[0] = incl[n_words - 1];
    counts[1] = wscan[n_words - 1] - 4ll * incl[n_words - 1];
    counts[2] = p.valid;
  }
}

__global__ void __launch_bounds__(kHThreads)
ba_dict_index_kernel(const HashTable small_t, const HashTable big_t, const uint32_t* __restrict__ ref, int64_t n, uint32_t* __restrict__ out) {
  const HashTable t = live_table(small_t, big_t);
  for (int64_t i = (int64_t)blockIdx.x * kHThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kHThreads)
    __stcs(out + i, t.slots[__ldcs(ref + i)].pad);
}

// words [offset / 32, ceil((offset + length) / 32)) of a chunk's `first`: global bit row + i - offset at chunk slot i
__global__ void __launch_bounds__(kHThreads)
ba_dict_first_kernel(const uint32_t* __restrict__ bits, int64_t n_words, int64_t row, int64_t offset, int64_t length, uint32_t* __restrict__ first) {
  const int64_t w0 = offset >> 5, w1 = (offset + length + 31) >> 5;
  auto word = [&](int64_t i) { return i >= 0 && i < n_words ? bits[i] : 0u; };
  for (int64_t w = w0 + (int64_t)blockIdx.x * kHThreads + threadIdx.x; w < w1; w += (int64_t)gridDim.x * kHThreads) {
    const int64_t g = row + (w << 5) - offset;        // global slot of the word's bit 0 (negative before the chunk)
    const uint32_t x = __funnelshift_r(word(g >> 5), word((g >> 5) + 1), (int)(g & 31));
    const int64_t a = offset - (w << 5), b = offset + length - (w << 5);
    first[w] = x & bit_range_mask(a > 0 ? (int)a : 0, b < 32 ? (int)b : 32);
  }
}

template <typename O>
static ag_status ba_dict_encode_t(BaDictPlan p, const ag_pq_ba_chunk* h_chunks, const int64_t* marks, int64_t n_marks, uint32_t* indices,
                                  int64_t* mark_counts, int64_t* counts, cudaStream_t st) {
  const int64_t total = p.slots;
  const bool two = total > g_unique_small_rows.load(std::memory_order_relaxed);
  const unsigned long long small_slots = (unsigned long long)g_unique_small_slots.load(std::memory_order_relaxed);
  const int64_t n_words = (total + 31) / 32;
  TableMem small_t, big_t;
  TableImage img(st);
  void* scratch = nullptr;
  ag_status rc = AG_OK;
  do {
    std::vector<int64_t> rb((size_t)p.n_chunks + 1, 0);
    for (int64_t c = 0; c < p.n_chunks; ++c) rb[(size_t)c + 1] = rb[(size_t)c] + h_chunks[c].length;
    const size_t o_rb = img.add(rb), o_marks = img.add(std::vector<int64_t>(marks, marks + n_marks));
    const size_t o_ch = img.add(std::vector<ag_pq_ba_chunk>(h_chunks, h_chunks + p.n_chunks));
    if ((rc = img.upload("byte_array_dict_encode")) != AG_OK) break;
    p.row_base = img.at<int64_t>(o_rb);
    p.chunks = img.at<ag_pq_ba_chunk>(o_ch);
    if (two) rc = small_t.alloc(0, small_slots, (unsigned)(small_slots / 2), st);
    else rc = small_t.alloc(p.valid, 1024, kNoCap, st);
    if (rc != AG_OK) break;
    if ((rc = small_t.clear(st)) != AG_OK) break;
    if (two && (rc = big_t.alloc(p.valid, 1024, kNoCap, st)) != AG_OK) break;
    // first-row bitmap | word popcounts | their scan | scan state | word bytes | their scan | scan state | table slots
    Carve sc;
    const size_t o_bits = sc.take((size_t)n_words * 4), o_cnt = sc.take((size_t)n_words * 4), o_incl = sc.take((size_t)n_words * 4);
    const size_t o_st = sc.take(64), o_wb = sc.take((size_t)n_words * 8), o_ws = sc.take((size_t)n_words * 8), o_st2 = sc.take(64);
    const size_t o_ref = sc.take((size_t)p.valid * 4);
    if ((rc = dev_alloc_async(&scratch, sc.size, st)) != AG_OK) break;
    char* d = static_cast<char*>(scratch);
    uint32_t* bits = reinterpret_cast<uint32_t*>(d + o_bits);
    int* wcnt = reinterpret_cast<int*>(d + o_cnt);
    int* incl = reinterpret_cast<int*>(d + o_incl);
    long long* wb = reinterpret_cast<long long*>(d + o_wb);
    long long* ws = reinterpret_cast<long long*>(d + o_ws);
    uint32_t* ref = reinterpret_cast<uint32_t*>(d + o_ref);
    if (cudaMemsetAsync(bits, 0, (size_t)n_words * 4, st) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "memset", __FILE__, __LINE__); break; }
    // inserts: every chunk into the small table, then (only when it overflowed) every chunk into the full-size one
    const int grid = grid_one_wave(ba_dict_insert_kernel<O>, kHThreads, p.n_tiles);
    for (int pass = 0; pass < (two ? 2 : 1) && rc == AG_OK; ++pass) {
      const unsigned* raised = pass ? small_t.t.special + 3 : nullptr;
      if (pass && (rc = big_t.clear(st, raised)) != AG_OK) break;
      ba_dict_insert_kernel<O><<<grid, kHThreads, 0, st>>>(p, ref, pass ? big_t.t : small_t.t, raised);
      rc = check_launch("ba_dict_insert_kernel");
    }
    if (rc != AG_OK) break;
    const int64_t max_slots = (int64_t)((two ? big_t.t.mask : small_t.t.mask) + 1);
    const int slot_grid = grid_for(max_slots, kHThreads * 4, 8), word_grid = grid_for(n_words, kHThreads * 4, 8);
    dict_first_bits_kernel<<<slot_grid, kHThreads, 0, st>>>(small_t.t, big_t.t, 0, bits);
    if ((rc = check_launch("dict_first_bits_kernel")) != AG_OK) break;
    bit_word_popc_kernel<<<word_grid, kHThreads, 0, st>>>(bits, n_words, wcnt);
    if ((rc = check_launch("bit_word_popc_kernel")) != AG_OK) break;
    if ((rc = cumulative_sum_state_init(d + o_st, AG_TYPE_INT32, nullptr, st)) != AG_OK) break;
    if ((rc = cumulative_sum_dev(AG_TYPE_INT32, wcnt, nullptr, 0, n_words, 0, 0, incl, nullptr, 0, d + o_st, nullptr, st)) != AG_OK) break;
    dict_rank_kernel<unsigned long long><<<slot_grid, kHThreads, 0, st>>>(small_t.t, big_t.t, 0, bits, incl, n_words, nullptr, nullptr, counts);
    if ((rc = check_launch("dict_rank_kernel")) != AG_OK) break;
    ba_dict_word_bytes_kernel<O><<<word_grid, kHThreads, 0, st>>>(p, bits, n_words, wb);
    if ((rc = check_launch("ba_dict_word_bytes_kernel")) != AG_OK) break;
    if ((rc = cumulative_sum_state_init(d + o_st2, AG_TYPE_INT64, nullptr, st)) != AG_OK) break;
    if ((rc = cumulative_sum_dev(AG_TYPE_INT64, wb, nullptr, 0, n_words, 0, 0, ws, nullptr, 0, d + o_st2, nullptr, st)) != AG_OK) break;
    ba_dict_marks_kernel<O><<<grid_for(n_marks, kHThreads, 8), kHThreads, 0, st>>>(p, bits, incl, ws, n_words, img.at<int64_t>(o_marks),
                                                                                   n_marks, mark_counts, counts);
    if ((rc = check_launch("ba_dict_marks_kernel")) != AG_OK) break;
    if (p.valid > 0) {
      ba_dict_index_kernel<<<grid_for(p.valid, kHThreads * 4, 8), kHThreads, 0, st>>>(small_t.t, big_t.t, ref, p.valid, indices);
      if ((rc = check_launch("ba_dict_index_kernel")) != AG_OK) break;
    }
    for (int64_t c = 0; c < p.n_chunks && rc == AG_OK; ++c) {
      const ag_pq_ba_chunk& ch = h_chunks[c];
      if (ch.length == 0) continue;
      const int64_t words = (ch.offset + ch.length + 31) / 32 - ch.offset / 32;
      ba_dict_first_kernel<<<grid_for(words, kHThreads, 8), kHThreads, 0, st>>>(bits, n_words, rb[(size_t)c], ch.offset, ch.length,
                                                                                reinterpret_cast<uint32_t*>(ch.first));
      rc = check_launch("ba_dict_first_kernel");
    }
  } while (0);
  if (scratch) cudaFreeAsync(scratch, st);
  small_t.release(st);
  big_t.release(st);
  return rc;
}

ag_status ba_dict_encode_dev(BaDictPlan p, const ag_pq_ba_chunk* h_chunks, const int64_t* marks, int64_t n_marks, uint32_t* indices,
                             int64_t* mark_counts, int64_t* counts, cudaStream_t st) {
  if (p.slots == 0) {   // every mark is 0
    AG_CUDA_TRY(cudaMemsetAsync(counts, 0, 3 * sizeof(int64_t), st));
    if (n_marks) AG_CUDA_TRY(cudaMemsetAsync(mark_counts, 0, (size_t)n_marks * 2 * sizeof(int64_t), st));
    return AG_OK;
  }
  return p.ow == 4 ? ba_dict_encode_t<int32_t>(p, h_chunks, marks, n_marks, indices, mark_counts, counts, st)
                   : ba_dict_encode_t<int64_t>(p, h_chunks, marks, n_marks, indices, mark_counts, counts, st);
}

}  // namespace ag

using namespace ag;

extern "C" ag_status ag_is_in_dev(int bit_width, const void* d_vals, const uint8_t* d_valid, int64_t offset, int64_t n, const void* d_set,
                                  const uint8_t* d_set_valid, int64_t set_offset, int64_t set_n, int null_behavior, uint8_t* d_out_data,
                                  uint8_t* d_out_valid, int64_t* d_null_count, ag_stream_t s) {
  AG_TRY(ensure_init());
  return is_in_dev(bit_width, d_vals, d_valid, offset, n, d_set, d_set_valid, set_offset, set_n, null_behavior, d_out_data, d_out_valid, d_null_count,
                   resolve_stream(s));
}

extern "C" ag_status ag_unique_set_policy(int64_t small_rows, int64_t small_slots) {
  if (small_rows < 0 || small_slots < 0) AG_FAIL(AG_ERR_INVALID, "ag_unique_set_policy: negative argument");
  if (small_slots && (small_slots < 1024 || small_slots > (1ll << 31) || (small_slots & (small_slots - 1))))
    AG_FAIL(AG_ERR_INVALID, "ag_unique_set_policy: small_slots must be a power of two in [1024, 2^31]");
  g_unique_small_rows.store(small_rows ? small_rows : (1ll << 21), std::memory_order_relaxed);
  g_unique_small_slots.store(small_slots ? small_slots : (1ll << 21), std::memory_order_relaxed);
  return AG_OK;
}

extern "C" ag_status ag_unique_dev(int bit_width, const void* d_vals, const uint8_t* d_valid, int64_t offset, int64_t n, void* d_out,
                                   uint8_t* d_out_valid, int64_t capacity, int64_t* d_out_len, ag_stream_t s) {
  AG_TRY(ensure_init());
  return unique_dev(bit_width, d_vals, d_valid, offset, n, d_out, d_out_valid, capacity, d_out_len, resolve_stream(s));
}

extern "C" ag_status ag_dictionary_encode_dev(int bit_width, const ag_dict_chunk* chunks, int64_t n_chunks, int null_encoding, void* d_dict,
                                              uint8_t* d_dict_valid, int64_t* d_counts, ag_stream_t s) {
  AG_TRY(ensure_init());
  return dictionary_encode_dev(bit_width, chunks, n_chunks, null_encoding, d_dict, d_dict_valid, d_counts, resolve_stream(s));
}
