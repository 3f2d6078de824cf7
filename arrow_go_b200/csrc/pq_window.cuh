// pq_window.cuh — the device protocols the Parquet page kernels that stream a page through shared memory share
// (pq_runs_kernel and delta_walk_kernel in pq_decode.cuh, ba_plain_parse_kernel in byte_array.cu, snappy_parse_kernel in
// snappy.cu, lz4_parse_kernel in lz4.cu).  Internal, not part of the ABI; device helpers only, no kernels.
//   load_window       one 16 KB window of a stream, 16-byte aligned to the absolute address
//   span_chain        the chain of elements through a span of 1024 candidate starts, by pointer doubling
//   block_incl_scan / block_excl_scan   one value per thread over a kPqThreads block
//   read_uvarint      binary.Uvarint
#pragma once

#include "common.cuh"

namespace ag {

namespace {

constexpr int kPqThreads = 256;             // threads per block of every page kernel
constexpr int kWinVec = 1024;               // 16-byte vectors per shared-memory window (16 KB)
constexpr int kWinBytes = kWinVec * 16;
constexpr int kSpan = 1024;                 // candidate element starts per parse step
constexpr int kPer = kSpan / kPqThreads;    // 4 consecutive positions per thread

// The window [a0, a0 + 16 KB) over absolute addresses of the stream [sbeg, send), a0 16-byte aligned, then a block
// barrier.  Only vectors that hold at least one byte of the stream are loaded: an aligned vector never straddles a
// mapping boundary, so no load touches memory past the stream's own pages.
__device__ __forceinline__ void load_window(uint4* win, uintptr_t sbeg, uintptr_t send, uintptr_t a0) {
#pragma unroll 4
  for (int v = threadIdx.x; v < kWinVec; v += kPqThreads) {
    const uintptr_t ad = a0 + (uintptr_t)v * 16;
    if (ad < send && ad + 16 > sbeg) win[v] = __ldcs(reinterpret_cast<const uint4*>(ad));
  }
  __syncthreads();
}

__device__ __forceinline__ bool bit_on(const uint32_t* m, int q) { return (m[q >> 5] >> (q & 31)) & 1u; }

// The chain through a span that starts on an element.  J[k] is the span position of the element after the one that
// would start at this thread's position q = tid * kPer + k (kSpan: none inside the span), and the caller has already
// stored it in jmp[0][q] (storing it where it is computed keeps the parse kernels free of spills).  On return, bit q of
// `reach` is set for every position on the chain, and J is spent.  Round r adds the positions 2^r elements after every
// position already on the chain; a round that adds none proves it closed, so a span of e elements takes about log2(e)
// rounds.
__device__ __forceinline__ void span_chain(uint32_t (&J)[kPer], uint16_t (&jmp)[2][kSpan], uint32_t (&reach)[kSpan / 32]) {
  const int tid = threadIdx.x;
  if (tid < kSpan / 32) reach[tid] = tid == 0 ? 1u : 0u;
  __syncthreads();
  for (int r = 0;; ++r) {
    bool grew = false;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const int q = tid * kPer + k;
      const uint32_t j = J[k];
      if (j < kSpan && bit_on(reach, q) && !bit_on(reach, (int)j)) {
        atomicOr(&reach[j >> 5], 1u << (j & 31));
        grew = true;
      }
    }
    if (!__syncthreads_or(grew)) break;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      J[k] = J[k] < kSpan ? jmp[r & 1][J[k]] : kSpan;
      jmp[(r + 1) & 1][tid * kPer + k] = (uint16_t)J[k];
    }
  }
}

// inclusive block scan of one value per thread (int ranks, or unsigned sums that wrap at their width)
template <typename V>
__device__ __forceinline__ V block_incl_scan(V v, V* warp_tot, V* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  V x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const V y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_tot[wid] = x;
  __syncthreads();
  V off = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kPqThreads / 32; ++w) {
    const V t = warp_tot[w];
    off += (w < wid) ? t : (V)0;
    tot += t;
  }
  __syncthreads();
  *total = tot;
  return off + x;
}

template <typename V>
__device__ __forceinline__ V block_excl_scan(V v, V* warp_tot, V* total) {
  return block_incl_scan(v, warp_tot, total) - v;
}

// binary.ReadUvarint: at most 10 bytes, the 10th at most 1
template <typename B>
__device__ __forceinline__ bool read_uvarint(B byte_at, int64_t& pos, int64_t len, unsigned long long* v) {
  unsigned long long x = 0;
  for (int i = 0; i < 10; ++i) {
    if (pos >= len) return false;
    const uint32_t c = byte_at(pos++);
    if (c < 0x80) {
      if (i == 9 && c > 1) return false;
      *v = x | (unsigned long long)c << (7 * i);
      return true;
    }
    x |= (unsigned long long)(c & 0x7f) << (7 * i);
  }
  return false;
}

}  // namespace

}  // namespace ag
