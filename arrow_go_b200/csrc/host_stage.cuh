// host_stage.cuh — how a synchronous host-pointer entry point stages memory.  Internal, not part of the ABI.
//
// The host flavour of an entry point owns a pooled stream for its duration, uploads its operands into stream-ordered
// device temporaries, runs the same *_dev code as the device flavour and copies the results back:
//
//   CallStream cs; AG_TRY(cs.acquire());
//   Temps t(cs);
//   AG_TRY(t.alloc(&d, nbytes));
//   AG_TRY(h2d(d, host_in, nbytes, cs));
//   AG_TRY(something_dev(d, ..., cs));
//   AG_TRY(d2h(host_out, d_out, nbytes, cs));
//   return sync(cs);
//
// Errors are early returns: on every path Temps waits for the stream and then frees the temporaries, so no copy of
// caller memory is still in flight when the call returns.  Only calls that end synchronised may use Temps; the
// asynchronous *_dev paths keep their scratch stream-ordered.
#pragma once

#include <string.h>
#include <type_traits>
#include <vector>

#include "common.cuh"

namespace ag {

// Stream-ordered temporaries of one host call; freed (async) when the call returns.
struct Temps {
  cudaStream_t st;
  std::vector<void*> ptrs;
  explicit Temps(cudaStream_t s) : st(s) {}
  ag_status alloc(void** p, size_t nbytes) {
    AG_TRY(dev_alloc_async(p, nbytes + 64, st));  // +64: kernels may read/write whole aligned words at the edges
    ptrs.push_back(*p);
    return AG_OK;
  }
  template <typename T> ag_status alloc_t(T** p, size_t nbytes) { return alloc(reinterpret_cast<void**>(p), nbytes); }
  ~Temps() {
    // An early (error) return may leave H2D / D2H copies of CALLER memory in flight on this pooled stream: wait for
    // them before the function returns and before the stream goes back to the pool.  On the success paths the
    // stream is already idle and this costs a few microseconds.
    cudaStreamSynchronize(st);
    for (void* p : ptrs) cudaFreeAsync(p, st);
  }
};

static inline ag_status h2d(void* d, const void* h, size_t nbytes, cudaStream_t st) {
  if (nbytes) AG_CUDA_TRY(cudaMemcpyAsync(d, h, nbytes, cudaMemcpyHostToDevice, st));
  return AG_OK;
}
static inline ag_status d2h(void* h, const void* d, size_t nbytes, cudaStream_t st) {
  if (nbytes) AG_CUDA_TRY(cudaMemcpyAsync(h, d, nbytes, cudaMemcpyDeviceToHost, st));
  return AG_OK;
}
static inline ag_status sync(cudaStream_t st) { AG_CUDA_TRY(cudaStreamSynchronize(st)); return AG_OK; }

static inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }

// Carves one scratch allocation into 256-byte aligned regions: take(n) returns the offset of the next n bytes, and
// `size` is what to allocate once every region is taken.
struct Carve {
  size_t size = 0;
  size_t take(size_t nbytes) { const size_t r = size; size = align256(size + nbytes); return r; }
};

// Host tables of a *_dev call packed into one device image: add() copies a table into the next 256-byte aligned region
// and returns its offset, upload() makes one allocation and one H2D copy, at<T>(offset) is the table on the device.
// The image is freed (stream-ordered, after the work that reads it) when it goes out of scope.
struct TableImage {
  cudaStream_t st;
  Carve carve;
  std::vector<unsigned char> host;
  void* dev = nullptr;
  explicit TableImage(cudaStream_t s) : st(s) {}
  ~TableImage() { dev_free_async(dev, st); }
  template <typename T> size_t add(const std::vector<T>& v) {
    static_assert(std::is_trivially_copyable<T>::value, "tables are copied as bytes");
    const size_t off = carve.take(v.size() * sizeof(T));
    host.resize(carve.size);
    if (!v.empty()) memcpy(host.data() + off, v.data(), v.size() * sizeof(T));
    return off;
  }
  ag_status upload(const char* what) {
    AG_TRY(dev_alloc_async(&dev, carve.size, st));
    const cudaError_t e = cudaMemcpyAsync(dev, host.data(), carve.size, cudaMemcpyHostToDevice, st);
    return e == cudaSuccess ? AG_OK : cuda_fail(e, what, __FILE__, __LINE__);
  }
  template <typename T> T* at(size_t off) const { return reinterpret_cast<T*>(static_cast<char*>(dev) + off); }
};

// Upload the bytes of a bitmap range [off, off+n) to a device temp; the device copy keeps the
// same bit phase (off % 8) so kernels address it with bit offset (off & 7).
static inline ag_status upload_bitmap(Temps& t, const uint8_t* h, int64_t off, int64_t n, uint8_t** d, int64_t* doff) {
  *d = nullptr; *doff = 0;
  if (!h) return AG_OK;
  const int64_t b0 = off >> 3, b1 = (off + n + 7) >> 3;
  AG_TRY(t.alloc_t(d, (size_t)(b1 - b0)));
  AG_TRY(h2d(*d, h + b0, (size_t)(b1 - b0), t.st));
  *doff = off & 7;
  return AG_OK;
}

// An output bitmap range is staged with its existing first/last bytes so that bits outside
// [off, off+n) survive the round trip; only the bytes of the range are written back.
struct OutBitmap {
  uint8_t* h = nullptr; uint8_t* d = nullptr; int64_t b0 = 0, nbytes = 0, doff = 0;
  ag_status stage(Temps& t, uint8_t* host, int64_t off, int64_t n) {
    h = host; b0 = off >> 3; nbytes = ((off + n + 7) >> 3) - b0; doff = off & 7;
    AG_TRY(t.alloc_t(&d, (size_t)nbytes));
    AG_TRY(h2d(d, h + b0, 1, t.st));
    if (nbytes > 1) AG_TRY(h2d(d + nbytes - 1, h + b0 + nbytes - 1, 1, t.st));
    return AG_OK;
  }
  ag_status fetch(cudaStream_t st) { return d2h(h + b0, d, (size_t)nbytes, st); }
};

}  // namespace ag
