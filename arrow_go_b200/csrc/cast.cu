// Numeric casts — the data movement under implicit type promotion (compute/exec.go:101-121:
// DispatchBest + CastDatum with SafeCastOptions) and the explicit `cast` function for the 10
// numeric types.  Replaces cast_type_numeric_{avx2,sse4} (_lib/cast_numeric.cc:22-101; Go
// dispatch cast_numeric.go:101-131) and the safety checks that frame it in numeric_cast.go:
//   CastIntToInt        :37-46   intsCanFit -> intsInRange (helpers.go:545-653) then the loop
//   CastFloatingToInteger :53-60 loop, then checkFloatTrunc  (numeric_cast.go:613-660)
//   CastIntegerToFloating :62-71 checkIntToFloatTrunc (:698-729) then the loop
//   CastFloatingToFloating :48-51 loop only
// One kernel does the conversion for EVERY slot (castNumberToNumberUnsafe casts nulls too) and,
// in the checked flavours, evaluates the reference's predicate on the valid slots in the same
// pass; the lowest failing row goes to the error word with atomicMin (the reference reports the
// first failing element in row order).
//
// float -> integer follows the conversion the reference's pure-Go loop performs on amd64 (and
// the scalar tail of its assembly): truncate toward zero through a 64-bit signed conversion
// whose out-of-range / NaN result is INT64_MIN, then keep the low bits; uint64 uses the
// "subtract 2^63" sequence.  For inputs whose truncated value is representable in the output
// type — the only inputs the reference's AVX2 body, SSE4 body and scalar tail agree on, and
// the only ones a safe cast accepts — this is bit-exact with cast_type_numeric_*.
#include "common.cuh"
#include "elem_ops.cuh"

namespace ag {

namespace {

constexpr int kCastThreads = 256;
constexpr int kCastUnroll = 8;

template <int kBytes> struct RawVec;
template <> struct RawVec<1> { using type = uint8_t; };
template <> struct RawVec<2> { using type = uint16_t; };
template <> struct RawVec<4> { using type = uint32_t; };
template <> struct RawVec<8> { using type = uint2; };
template <> struct RawVec<16> { using type = uint4; };

// E consecutive elements of T moved with the widest accesses <= 16 bytes.
template <typename T, int E>
struct Pack {
  static constexpr int kBytes = E * (int)sizeof(T);
  static constexpr int kAccess = kBytes >= 16 ? 16 : kBytes;
  static constexpr int kN = kBytes / kAccess;
  using Raw = typename RawVec<kAccess>::type;
  union { Raw raw[kN]; T v[E]; };
  __device__ __forceinline__ void load(const T* p) {
    const Raw* rp = reinterpret_cast<const Raw*>(p);
#pragma unroll
    for (int j = 0; j < kN; ++j) {
      if constexpr (kAccess == 16) raw[j] = __ldcs(rp + j);
      else if constexpr (kAccess == 8) raw[j] = __ldcs(rp + j);
      else raw[j] = rp[j];
    }
  }
  __device__ __forceinline__ void store(T* p) const {
    Raw* rp = reinterpret_cast<Raw*>(p);
#pragma unroll
    for (int j = 0; j < kN; ++j) {
      if constexpr (kAccess == 16) __stcs(rp + j, raw[j]);
      else if constexpr (kAccess == 8) __stcs(rp + j, raw[j]);
      else rp[j] = raw[j];
    }
  }
};

template <typename I, typename O>
struct CastGeom {
  static constexpr int kWide = sizeof(I) > sizeof(O) ? sizeof(I) : sizeof(O);
  // one 16-byte vector per lane on the wide side, the matching 2..16 bytes on the narrow side: every
  // warp access is one contiguous run (a 32-byte-per-lane layout left half-written sectors behind
  // each store instruction and ran the widening casts at 0.58 of the HBM roofline)
  static constexpr int E = 16 / kWide;
  static constexpr int kTile = kCastThreads * E * kCastUnroll;  // rows per block tile
  static constexpr int kInAlign = Pack<I, E>::kAccess;
  static constexpr int kOutAlign = Pack<O, E>::kAccess;
};

template <typename I, typename O, int kCheck>
__global__ void __launch_bounds__(kCastThreads)
cast_vec_kernel(const I* __restrict__ in, O* __restrict__ out, int64_t n,
                const uint8_t* __restrict__ valid, int64_t voff, I lo, I hi, long long* first_bad, long long row_base) {
  using G = CastGeom<I, O>;
  constexpr int E = G::E;
  const int64_t n_tiles = (n + G::kTile - 1) / G::kTile;
  long long my_bad = AG_NO_ERROR_POS;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t e0 = tile * G::kTile;
    const int len = (int)((n - e0 < G::kTile) ? (n - e0) : G::kTile);
    const I* ip = in + e0;
    O* op = out + e0;
    const int npack = len / E;
    Pack<I, E> a[kCastUnroll];
#pragma unroll
    for (int k = 0; k < kCastUnroll; ++k) {
      const int pi = k * kCastThreads + threadIdx.x;
      if (pi < npack) a[k].load(ip + (int64_t)pi * E);
    }
#pragma unroll
    for (int k = 0; k < kCastUnroll; ++k) {
      const int pi = k * kCastThreads + threadIdx.x;
      if (pi < npack) {
        Pack<O, E> o;
#pragma unroll
        for (int e = 0; e < E; ++e) {
          o.v[e] = cast_one<I, O>(a[k].v[e]);
          if constexpr (kCheck != 0) {
            if (cast_fails<I, O, kCheck>(a[k].v[e], o.v[e], lo, hi)) {
              const int64_t row = e0 + (int64_t)pi * E + e;
              if ((!valid || bit_is_set(valid, voff + row)) && row_base + row < my_bad) my_bad = row_base + row;
            }
          }
        }
        o.store(op + (int64_t)pi * E);
      }
    }
    const int i = npack * E + threadIdx.x;  // ragged end of the last tile
    if (i < len) {
      const I v = ip[i];
      const O o = cast_one<I, O>(v);
      op[i] = o;
      if constexpr (kCheck != 0) {
        if (cast_fails<I, O, kCheck>(v, o, lo, hi)) {
          const int64_t row = e0 + i;
          if ((!valid || bit_is_set(valid, voff + row)) && row_base + row < my_bad) my_bad = row_base + row;
        }
      }
    }
  }
  if constexpr (kCheck != 0) lower_error_row(my_bad, first_bad);
}

// Element-aligned operands (odd element offsets): one element per thread, still coalesced.
template <typename I, typename O, int kCheck>
__global__ void __launch_bounds__(kCastThreads)
cast_scalar_kernel(const I* __restrict__ in, O* __restrict__ out, int64_t n,
                   const uint8_t* __restrict__ valid, int64_t voff, I lo, I hi, long long* first_bad, long long row_base) {
  const int64_t stride = (int64_t)gridDim.x * kCastThreads;
  long long my_bad = AG_NO_ERROR_POS;
  for (int64_t i = (int64_t)blockIdx.x * kCastThreads + threadIdx.x; i < n; i += stride) {
    const I v = in[i];
    const O o = cast_one<I, O>(v);
    out[i] = o;
    if constexpr (kCheck != 0) {
      if (cast_fails<I, O, kCheck>(v, o, lo, hi) && (!valid || bit_is_set(valid, voff + i)) && row_base + i < my_bad) my_bad = row_base + i;
    }
  }
  if constexpr (kCheck != 0) lower_error_row(my_bad, first_bad);
}

template <typename I, typename O, int kCheck>
ag_status launch_cast(const void* in, void* out, int64_t n, const uint8_t* valid, int64_t voff,
                      I lo, I hi, int64_t* first_bad, int64_t row_base, cudaStream_t st) {
  using G = CastGeom<I, O>;
  const bool vec = (reinterpret_cast<uintptr_t>(in) % G::kInAlign) == 0 && (reinterpret_cast<uintptr_t>(out) % G::kOutAlign) == 0;
  if (vec) {
    const int grid = grid_one_wave(cast_vec_kernel<I, O, kCheck>, kCastThreads, (n + G::kTile - 1) / G::kTile);
    cast_vec_kernel<I, O, kCheck><<<grid, kCastThreads, 0, st>>>((const I*)in, (O*)out, n, valid, voff, lo, hi, (long long*)first_bad, row_base);
  } else {
    const int grid = grid_for(n, kCastThreads * 4, 8);
    cast_scalar_kernel<I, O, kCheck><<<grid, kCastThreads, 0, st>>>((const I*)in, (O*)out, n, valid, voff, lo, hi, (long long*)first_bad, row_base);
  }
  return check_launch("cast_kernel");
}

template <typename I, typename O>
ag_status cast_io(const void* in, void* out, int64_t n, const uint8_t* valid, int64_t voff,
                  int allow_int_overflow, int allow_float_truncate, int64_t* first_bad, int64_t row_base, cudaStream_t st) {
  if constexpr (!IsFloat<I>::v) {
    const bool want = first_bad && (IsFloat<O>::v ? !allow_float_truncate : !allow_int_overflow);
    I lo = 0, hi = 0;
    if (want && safe_bounds<I, O>(&lo, &hi)) return launch_cast<I, O, 1>(in, out, n, valid, voff, lo, hi, first_bad, row_base, st);
    return launch_cast<I, O, 0>(in, out, n, nullptr, 0, I(0), I(0), nullptr, 0, st);
  } else if constexpr (!IsFloat<O>::v) {
    if (first_bad && !allow_float_truncate) return launch_cast<I, O, 2>(in, out, n, valid, voff, I(0), I(0), first_bad, row_base, st);
    return launch_cast<I, O, 0>(in, out, n, nullptr, 0, I(0), I(0), nullptr, 0, st);
  } else {
    return launch_cast<I, O, 0>(in, out, n, nullptr, 0, I(0), I(0), nullptr, 0, st);
  }
}

}  // namespace

ag_status cast_numeric_dev(int itype, int otype, const void* in, const uint8_t* valid, int64_t voff, void* out, int64_t n,
                           int allow_int_overflow, int allow_float_truncate, int64_t* first_bad, int64_t row_base, cudaStream_t st) {
  if (n < 0) AG_FAIL(AG_ERR_INVALID, "cast: negative length");
  if (type_width(itype) == 0) AG_FAIL(AG_ERR_TYPE, "cast: unsupported input type id %d", itype);
  if (type_width(otype) == 0) AG_FAIL(AG_ERR_TYPE, "cast: unsupported output type id %d", otype);
  if (n == 0) return AG_OK;
  if (!in || !out) AG_FAIL(AG_ERR_INVALID, "cast: NULL operand");
  if (itype == otype) {  // castNumberMemCpy, helpers.go:659-688
    AG_CUDA_TRY(cudaMemcpyAsync(out, in, (size_t)n * type_width(itype), cudaMemcpyDeviceToDevice, st));
    return AG_OK;
  }
  return visit_type(itype, [&](auto itag) {
    return visit_type(otype, [&](auto otag) {
      return cast_io<typename decltype(itag)::type, typename decltype(otag)::type>(in, out, n, valid, voff, allow_int_overflow,
                                                                                 allow_float_truncate, first_bad, row_base, st);
    }, [&] { AG_FAIL(AG_ERR_TYPE, "cast: unsupported output type id %d", otype); });
  }, [&] { AG_FAIL(AG_ERR_TYPE, "cast: unsupported input type id %d", itype); });
}

}  // namespace ag

using namespace ag;

extern "C" ag_status ag_cast_numeric_dev(int itype, int otype, const void* d_in, void* d_out, int64_t n, ag_stream_t s) {
  AG_TRY(ensure_init());
  return cast_numeric_dev(itype, otype, d_in, nullptr, 0, d_out, n, 1, 1, nullptr, 0, resolve_stream(s));
}

extern "C" ag_status ag_cast_numeric_checked_dev(int itype, int otype, const void* d_in, const uint8_t* d_valid, int64_t valid_offset,
                                                 void* d_out, int64_t n, int allow_int_overflow, int allow_float_truncate,
                                                 int64_t* d_first_bad, ag_stream_t s) {
  AG_TRY(ensure_init());
  if (!d_first_bad) AG_FAIL(AG_ERR_INVALID, "cast: checked flavour needs an error word");
  return cast_numeric_dev(itype, otype, d_in, d_valid, valid_offset, d_out, n, allow_int_overflow, allow_float_truncate, d_first_bad, 0, resolve_stream(s));
}
