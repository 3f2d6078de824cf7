// lz_exec.cu — the executor every Parquet page decompressor (snappy.cu, zstd.cu, gzip.cu, lz4.cu) ends with: a page's
// output from element descriptors {first output byte, literal source / copy offset, kind}, in 2048-byte batches with
// pointer jumping over in-batch sources.
#include "lz_exec.cuh"

namespace ag {

namespace {

// One block (kLzThreads) writes page p's output in batches of kLzBatch bytes, in order.  Each element produces at
// least one byte.  Byte j of a copy at `pos` with offset r is dst[pos - r + (j mod r)], so every output byte names
// one source byte: a literal byte, an output byte before the batch (read back from dst, written by this block), or
// an earlier byte of the same batch, which pointer jumping in shared memory resolves.
__device__ __forceinline__ void lz_exec_page(const LzExec& a, int64_t p) {
  __shared__ uint32_t s_out[kLzBatch + 1], s_ref[kLzBatch + 1];
  __shared__ uint8_t s_lit[kLzBatch + 1];
  __shared__ unsigned long long s_src[kLzBatch];
  const int64_t written = a.done[p * a.stride], nelem = a.done[p * a.stride + 1];
  if (written <= 0 || nelem <= 0) return;                        // block-uniform
  const ag_pq_compressed pg = a.pages[p];
  const uint8_t* in = a.src + pg.src;
  const uint8_t* lit = a.lit ? a.lit + a.lit_base[p] : nullptr;
  uint8_t* out = a.dst + pg.dst;
  const int64_t eb = a.elem_base[p];
  const int tid = threadIdx.x;
  int64_t e0 = 0;                                                // the element holding the batch's first byte
  for (int64_t B = 0; B < written; B += kLzBatch) {
    const int nb = (int)(written - B < kLzBatch ? written - B : kLzBatch);
    // elements e0 .. e0 + nl - 1 hold every byte of [B, B + kLzBatch] (each element produces at least one byte)
    const int nl = (int)(nelem - e0 < kLzBatch + 1 ? nelem - e0 : kLzBatch + 1);
    for (int k = tid; k < nl; k += kLzThreads) {
      s_out[k] = a.e_out[eb + e0 + k];
      s_ref[k] = a.e_ref[eb + e0 + k];
      s_lit[k] = a.e_lit[eb + e0 + k];
    }
    __syncthreads();
    auto holder = [&](uint32_t pos) {                            // last loaded element starting at or before pos
      int lo = 0, hi = nl - 1;
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (s_out[mid] <= pos) lo = mid; else hi = mid - 1;
      }
      return lo;
    };
    for (int b = tid; b < nb; b += kLzThreads) {
      const uint32_t pos = (uint32_t)(B + b);
      const int e = holder(pos);
      const uint32_t j = pos - s_out[e], r = s_ref[e];
      unsigned long long s;
      if (s_lit[e]) {
        s = (s_lit[e] == kLzSrc ? kFromSrc : kFromLit) | (unsigned long long)(r + j);
      } else {
        const uint32_t q = s_out[e] - r + (j < r ? j : j % r);
        s = (int64_t)q < B ? kFromDst | q : (unsigned long long)((int64_t)q - B);
      }
      s_src[b] = s;
    }
    __syncthreads();
    while (true) {                                               // pointer jumping to a byte outside the batch
      bool pend = false;
      for (int b = tid; b < nb; b += kLzThreads) {
        const unsigned long long v = s_src[b];
        if (v < kFromLit) {
          const unsigned long long w = s_src[v];
          s_src[b] = w;
          pend |= w < kFromLit;
        }
      }
      if (!__syncthreads_or(pend)) break;
    }
    for (int b = tid; b < nb; b += kLzThreads) {
      const unsigned long long v = s_src[b];
      // dst bytes before the batch were written by this block before the last barrier: a plain (coherent) load
      out[B + b] = (v & kFromSrc) ? __ldg(in + (v & kLzPosMask)) : (v & kFromLit) ? lit[v & kLzPosMask] : out[v & kLzPosMask];
    }
    e0 += holder((uint32_t)(B + kLzBatch < written ? B + kLzBatch : written - 1));
    __syncthreads();
  }
}

// one block per page: the page's output from its element descriptors
__global__ void __launch_bounds__(kLzThreads)
lz_exec_kernel(LzExec a) {
  lz_exec_page(a, blockIdx.x);
}

}  // namespace

ag_status lz_exec_launch(const LzExec& x, int64_t n_pages, cudaStream_t st) {
  lz_exec_kernel<<<(unsigned)n_pages, kLzThreads, 0, st>>>(x);
  return check_launch("lz_exec_kernel");
}

}  // namespace ag
