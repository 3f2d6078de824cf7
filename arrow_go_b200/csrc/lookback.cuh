// lookback.cuh — the decoupled look-back of the single-pass compaction kernels (filter.cu, run_end.cu).
// Internal, not part of the ABI.
#pragma once

#include "common.cuh"

namespace ag {

// Tile status word: 2 flag bits + a 62-bit count, written with one store, so a reader never sees a flag
// without its value.  0 = not yet published.
constexpr unsigned long long kFlagShift = 62;
constexpr unsigned long long kFlagAgg = 1ull << kFlagShift;
constexpr unsigned long long kFlagIncl = 2ull << kFlagShift;
constexpr unsigned long long kValMask = (1ull << kFlagShift) - 1;

__device__ __forceinline__ unsigned long long ld_status(const unsigned long long* p) {
  return *reinterpret_cast<const volatile unsigned long long*>(p);
}
__device__ __forceinline__ void st_status(unsigned long long* p, unsigned long long v) {
  *reinterpret_cast<volatile unsigned long long*>(p) = v;
}

// One warp.  Returns the exclusive prefix of `tile` (rows emitted by all earlier tiles).
//
// Two levels, so the number of DEPENDENT L2 round trips does not grow with the number of tiles in
// flight.  (A flat 32-wide look-back needs about q/64 hops for the q-th tile of a wave: with 450-740
// resident blocks in lockstep the last tiles of a wave waited 7-10 hops while HBM idled.)
//   level 1: tiles form groups of 32.  A tile publishes its AGGREGATE in st[tile] (written once) and
//            reads the aggregates of the earlier tiles of its own group: one batch of <= 31 polls;
//   level 2: the last tile of a group publishes the GROUP aggregate in gst[g] and, after its own
//            look-back, the group's INCLUSIVE prefix in the same word; every tile looks back over the
//            groups before its own, 32 at a time, until it meets an inclusive prefix.  Fewer than 32
//            groups (1024 tiles) are ever in flight, so that is one hop.
// One 64-bit word carries flag + count, so a reader never sees a flag without its value.  A tile waits
// only on lower tiles, which the static tile order + one resident wave guarantee are running or done.
template <bool kPublish = true>   // false: the caller has already published the tile's aggregate
__device__ __forceinline__ unsigned long long lookback(unsigned long long* st, unsigned long long* gst, int64_t tile,
                                                       unsigned long long total, int lane) {
  const int64_t g = tile >> 5;
  const int q = (int)(tile & 31);
  if (kPublish && lane == 0) st_status(st + tile, kFlagAgg | total);
  // level 1
  unsigned long long s = (lane < q) ? 0ull : kFlagAgg;  // lanes >= q: nothing to wait for
  do {
    if ((s >> kFlagShift) == 0) s = ld_status(st + (g << 5) + lane);
  } while (__any_sync(0xffffffffu, (s >> kFlagShift) == 0));
  unsigned long long part = (lane < q) ? (s & kValMask) : 0ull;
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) part += __shfl_xor_sync(0xffffffffu, part, m);
  const bool leader = q == 31;
  if (leader && lane == 0) st_status(gst + g, kFlagAgg | (part + total));
  // level 2
  unsigned long long running = 0;
  int64_t look = g - 1;
  while (look >= 0) {
    const int64_t idx = look - lane;
    unsigned flag;
    do {
      s = (idx >= 0) ? ld_status(gst + idx) : kFlagIncl;  // before group 0: inclusive prefix 0
      flag = (unsigned)(s >> kFlagShift);
    } while (__any_sync(0xffffffffu, flag == 0));
    const unsigned incl = __ballot_sync(0xffffffffu, flag == 2);
    unsigned long long v = s & kValMask;
    if (incl) {
      const int first = __ffs(incl) - 1;  // closest group that already knows its inclusive prefix
      if (lane > first) v = 0;
    }
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    running += v;
    if (incl) break;
    look -= 32;
  }
  if (leader && lane == 0) st_status(gst + g, kFlagIncl | (running + part + total));
  return running + part;
}

}  // namespace ag
