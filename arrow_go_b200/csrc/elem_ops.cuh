// elem_ops.cuh — the per-element and per-word operations of the scalar kernels, shared by the single-op kernels
// (elementwise.cu, compare.cu, cast.cu, bitmap.cu) and the expression program (expr.cu), so that a fused expression
// computes every slot with the same code as the node-by-node calls.  Internal, not part of the ABI.
#pragma once

#include <type_traits>

#include "common.cuh"

namespace ag {

// ---- arithmetic (elementwise.cu) ----
// Integers run on their storage type (visit_storage_type), so int8/uint8 ... int64/uint64 share kernels.
struct OpAdd { template <typename T> static __device__ __forceinline__ T apply(T a, T b) { return (T)(a + b); } };
struct OpSub { template <typename T> static __device__ __forceinline__ T apply(T a, T b) { return (T)(a - b); } };
struct OpMul {
  template <typename T> static __device__ __forceinline__ T apply(T a, T b) {
    if constexpr (std::is_floating_point<T>::value) return a * b;
    else if constexpr (sizeof(T) == 8) return (T)(a * b);
    else return (T)((uint32_t)a * (uint32_t)b);
  }
};
// explicit round-to-nearest intrinsics: no FMA contraction, no reassociation
// bitwiseKernelOp (scalar_arithmetic.go:191-243): the reference runs BitmapAnd/Or/Xor over the value buffers, i.e. the
// plain bitwise op on every slot; integer types only (the float instantiations are never dispatched).
struct OpBitAnd { template <typename T> static __device__ __forceinline__ T apply(T a, T b) { if constexpr (std::is_integral<T>::value) return (T)(a & b); else return a; } };
struct OpBitOr { template <typename T> static __device__ __forceinline__ T apply(T a, T b) { if constexpr (std::is_integral<T>::value) return (T)(a | b); else return a; } };
struct OpBitXor { template <typename T> static __device__ __forceinline__ T apply(T a, T b) { if constexpr (std::is_integral<T>::value) return (T)(a ^ b); else return a; } };
template <> __device__ __forceinline__ double OpAdd::apply<double>(double a, double b) { return __dadd_rn(a, b); }
template <> __device__ __forceinline__ float OpAdd::apply<float>(float a, float b) { return __fadd_rn(a, b); }
template <> __device__ __forceinline__ double OpSub::apply<double>(double a, double b) { return __dsub_rn(a, b); }
template <> __device__ __forceinline__ float OpSub::apply<float>(float a, float b) { return __fsub_rn(a, b); }
template <> __device__ __forceinline__ double OpMul::apply<double>(double a, double b) { return __dmul_rn(a, b); }
template <> __device__ __forceinline__ float OpMul::apply<float>(float a, float b) { return __fmul_rn(a, b); }

// AbsoluteValue base_arithmetic.cc:160-176 (floats: clear the sign bit; signed ints:
// (x + mask) ^ mask), Negate :194-205, NegateChecked :207-219 (unsigned -> 0), Sign :221-234.
struct UAbs {
  template <typename TO, typename T> static __device__ __forceinline__ TO apply(T x) {
    if constexpr (std::is_same<T, float>::value) return __uint_as_float(__float_as_uint(x) & 0x7fffffffu);
    else if constexpr (std::is_same<T, double>::value) return __longlong_as_double(__double_as_longlong(x) & 0x7fffffffffffffffll);
    else if constexpr (std::is_unsigned<T>::value) return x;
    else {
      using U = typename std::make_unsigned<T>::type;
      const U mask = (U)(x >> (sizeof(T) * 8 - 1));
      return (T)(((U)x + mask) ^ mask);
    }
  }
};
struct UNeg {
  template <typename TO, typename T> static __device__ __forceinline__ TO apply(T x) {
    if constexpr (std::is_same<T, float>::value) return __uint_as_float(__float_as_uint(x) ^ 0x80000000u);
    else if constexpr (std::is_same<T, double>::value) return __longlong_as_double(__double_as_longlong(x) ^ (long long)0x8000000000000000ull);
    else { using U = typename std::make_unsigned<T>::type; return (T)((U)0 - (U)x); }
  }
};
struct UNegChecked {  // identical to UNeg except unsigned -> 0 (base_arithmetic.cc:213-214)
  template <typename TO, typename T> static __device__ __forceinline__ TO apply(T x) {
    if constexpr (std::is_unsigned<T>::value) return 0;
    else return UNeg::apply<TO, T>(x);
  }
};
struct UBitNot {  // bitwiseNot, scalar_arithmetic.go:257-259 (integer types; floats are refused before the launch)
  template <typename TO, typename T> static __device__ __forceinline__ TO apply(T x) {
    if constexpr (std::is_integral<T>::value) return (TO)(T)~x; else return (TO)x;
  }
};
struct USign {
  template <typename TO, typename T> static __device__ __forceinline__ TO apply(T x) {
    // NaN: the reference's shipped AVX2/SSE4 objects lost the isnan() test of base_arithmetic.cc:224
    // to -funsafe-math-optimizations (kernels/Makefile:23-27): sign(NaN) = +-1 by sign bit.
    if constexpr (std::is_floating_point<T>::value) return (TO)((x == 0) ? T(0) : (signbit(x) ? T(-1) : T(1)));
    else if constexpr (std::is_unsigned<T>::value) return (TO)(x > 0 ? 1 : 0);
    else return (TO)(x > 0 ? 1 : (x ? -1 : 0));
  }
};

// base_arithmetic.go:249-278: carry = ((a&b) | ((a|b) &^ out)) >> shiftBy, "carry > 0", with
// shiftBy = bits-1 (unsigned) or bits-2 (signed) evaluated in the operand type (arithmetic
// shift for signed).  We restate the formula bit for bit, including what it does for signed
// operands (it flags a carry into the sign bit that is not carried out).
template <typename ST> struct ChkAdd {
  static __device__ __forceinline__ ST apply(ST a, ST b, bool& bad) {
    using U = typename std::make_unsigned<ST>::type;
    constexpr int shift_by = (int)sizeof(ST) * 8 - 1 - (std::is_signed<ST>::value ? 1 : 0);
    const ST o = (ST)((U)a + (U)b);
    const ST c = (ST)((ST)((ST)(a & b) | ((ST)(a | b) & (ST)~o)) >> shift_by);
    bad = c > 0;
    return o;
  }
};
template <typename ST> struct ChkSub {
  static __device__ __forceinline__ ST apply(ST a, ST b, bool& bad) {
    using U = typename std::make_unsigned<ST>::type;
    constexpr int shift_by = (int)sizeof(ST) * 8 - 1 - (std::is_signed<ST>::value ? 1 : 0);
    const ST o = (ST)((U)a - (U)b);
    const ST c = (ST)((ST)((ST)((ST)~a & b) | ((ST)~(ST)(a ^ b) & o)) >> shift_by);
    bad = c > 0;
    return o;
  }
};
// mulWithOverflow base_arithmetic.go:84-108 (division-based test; an overflowing slot yields 0)
template <typename ST> struct ChkMul {
  static __device__ __forceinline__ ST apply(ST a, ST b, bool& bad) {
    using U = typename std::make_unsigned<ST>::type;
    constexpr ST tmax = std::is_signed<ST>::value ? (ST)(((U)1 << (sizeof(ST) * 8 - 1)) - 1) : (ST)~(U)0;
    constexpr ST tmin = std::is_signed<ST>::value ? (ST)((U)1 << (sizeof(ST) * 8 - 1)) : (ST)0;
    bool ovf = false;
    if (a > 0) { if (b > 0) { ovf = a > (ST)(tmax / b); } else { ovf = b < (ST)(tmin / a); } }
    else if (b > 0) { ovf = a < (ST)(tmin / b); }
    else { ovf = (a != 0) && (b < (ST)(tmax / a)); }
    bad = ovf;
    return ovf ? (ST)0 : (ST)((U)a * (U)b);
  }
};
// Div / DivChecked base_arithmetic.go:154-161,287-294: b == 0 -> error (value 0); Go's
// MinInt / -1 wraps to MinInt.
template <typename ST> struct ChkDiv {
  static __device__ __forceinline__ ST apply(ST a, ST b, bool& bad) {
    using U = typename std::make_unsigned<ST>::type;
    bad = (b == 0);
    if (b == 0) return 0;
    if constexpr (std::is_signed<ST>::value) {
      constexpr ST tmin = (ST)((U)1 << (sizeof(ST) * 8 - 1));
      if (a == tmin && b == (ST)-1) return a;
    }
    return (ST)(a / b);
  }
};

// shiftKernelSignedImpl / UnsignedImpl (scalar_arithmetic.go:293-379): an amount outside [0, maxShift) leaves lhs as it
// is and, in the checked flavour, fails the call; maxShift = bits - 1 for SIGNED types, bits for unsigned.
template <typename ST, bool kLeft, bool kChecked> struct ChkShift {
  static __device__ __forceinline__ ST apply(ST a, ST b, bool& bad) {
    using U = typename std::make_unsigned<ST>::type;
    constexpr int max_shift = (int)sizeof(ST) * 8 - (std::is_signed<ST>::value ? 1 : 0);
    const bool invalid = (std::is_signed<ST>::value && b < 0) || (unsigned long long)b >= (unsigned long long)max_shift;
    bad = kChecked && invalid;
    if (invalid) return a;
    if (kLeft) return (ST)((U)a << (int)b);
    return (ST)(a >> (int)b);
  }
};
// floating point Div / DivChecked (base_arithmetic.go:386-397): IEEE quotient; the checked op fails on a zero divisor
template <typename FT, bool kChecked> struct ChkFDiv {
  static __device__ __forceinline__ FT apply(FT a, FT b, bool& bad) {
    bad = kChecked && b == FT(0);
    if (bad) return FT(0);
    if constexpr (sizeof(FT) == 8) return __ddiv_rn(a, b); else return __fdiv_rn(a, b);
  }
};

// ---- comparisons (compare.cu) ----
struct CmpEq { template <typename T> static __device__ __forceinline__ bool apply(T a, T b) { return a == b; } };
struct CmpNe { template <typename T> static __device__ __forceinline__ bool apply(T a, T b) { return a != b; } };
struct CmpGt { template <typename T> static __device__ __forceinline__ bool apply(T a, T b) { return a > b; } };
struct CmpGe { template <typename T> static __device__ __forceinline__ bool apply(T a, T b) { return a >= b; } };


// ---- numeric casts (cast.cu) ----
template <typename T> struct IsFloat { static constexpr bool v = false; };
template <> struct IsFloat<float> { static constexpr bool v = true; };
template <> struct IsFloat<double> { static constexpr bool v = true; };
template <typename T> struct IsSigned { static constexpr bool v = T(-1) < T(0); };

__device__ __forceinline__ long long x86_cvtt(double v) {
  // CVTTSD2SI r64: NaN and out-of-range give the "integer indefinite" value
  if (!(v >= -9223372036854775808.0 && v < 9223372036854775808.0)) return (long long)0x8000000000000000ull;
  return __double2ll_rz(v);
}

template <typename I, typename O>
__device__ __forceinline__ O cast_one(I v) {
  if constexpr (IsFloat<I>::v && !IsFloat<O>::v) {
    const double d = (double)v;  // float -> double is exact
    if constexpr (sizeof(O) == 8 && !IsSigned<O>::v) {
      // Go / clang uint64 conversion: values >= 2^63 go through (x - 2^63) with the top bit set
      if (d >= 9223372036854775808.0) return (O)((unsigned long long)x86_cvtt(d - 9223372036854775808.0) ^ 0x8000000000000000ull);
      return (O)(unsigned long long)x86_cvtt(d);
    } else {
      return (O)x86_cvtt(d);  // wrap-truncation to the output width
    }
  } else if constexpr (!IsFloat<I>::v && IsFloat<O>::v) {
    if constexpr (sizeof(O) == 4) {
      if constexpr (IsSigned<I>::v) return __ll2float_rn((long long)v);
      else return __ull2float_rn((unsigned long long)v);
    } else {
      if constexpr (IsSigned<I>::v) return __ll2double_rn((long long)v);
      else return __ull2double_rn((unsigned long long)v);
    }
  } else if constexpr (IsFloat<I>::v && IsFloat<O>::v) {
    if constexpr (sizeof(I) == 8 && sizeof(O) == 4) return __double2float_rn(v);
    else return (O)v;
  } else {
    return (O)v;  // integer -> integer: sign/zero extension or truncation
  }
}

// kCheck: 0 none, 1 integer input in [lo, hi] (intsInRange), 2 float -> int round trip
// (wasTrunc: OutT -> InT conversion of the result differs from the input; NaN always differs).
template <typename I, typename O, int kCheck>
__device__ __forceinline__ bool cast_fails(I in, O out, I lo, I hi) {
  if constexpr (kCheck == 1) return in < lo || in > hi;
  else if constexpr (kCheck == 2) return cast_one<O, I>(out) != in;
  else return false;
}

template <typename T> struct Lim;
#define AG_LIM(T, LO, HI) template <> struct Lim<T> { static constexpr T lo = LO; static constexpr T hi = HI; };
AG_LIM(uint8_t, 0, 0xff) AG_LIM(int8_t, -128, 127) AG_LIM(uint16_t, 0, 0xffff) AG_LIM(int16_t, -32768, 32767)
AG_LIM(uint32_t, 0, 0xffffffffu) AG_LIM(int32_t, (-2147483647 - 1), 2147483647)
AG_LIM(unsigned long long, 0, 0xffffffffffffffffull) AG_LIM(long long, (-9223372036854775807ll - 1), 9223372036854775807ll)
#undef AG_LIM

// Safe bounds of an integer input type I for target O, in I's own domain
// (getSafeMinMaxSigned / Unsigned, helpers.go:496-543) and for float targets
// (checkIntToFloatTrunc, numeric_cast.go:698-729).  Returns false when every I fits.
template <typename I, typename O>
bool safe_bounds(I* lo, I* hi) {
  if constexpr (IsFloat<O>::v) {
    constexpr int mant = sizeof(O) == 4 ? 24 : 53;
    if (sizeof(I) * 8 <= (size_t)mant) return false;  // int8/16 always; int32/uint32 -> float64
    const I lim = (I)((unsigned long long)1 << mant);
    *hi = lim;
    *lo = IsSigned<I>::v ? (I)(0 - lim) : (I)0;
    return true;
  } else {
    I l = Lim<I>::lo, h = Lim<I>::hi;
    if constexpr (IsSigned<I>::v) {
      if constexpr (IsSigned<O>::v) { if (sizeof(I) > sizeof(O)) { l = (I)Lim<O>::lo; h = (I)Lim<O>::hi; } }
      else { l = 0; if (sizeof(I) > sizeof(O)) h = (I)Lim<O>::hi; }
    } else {
      if constexpr (IsSigned<O>::v) { if (sizeof(I) >= sizeof(O)) h = (I)Lim<O>::hi; }
      else { if (sizeof(I) > sizeof(O)) h = (I)Lim<O>::hi; }
    }
    *lo = l; *hi = h;
    return !(l == Lim<I>::lo && h == Lim<I>::hi);  // intsInRange's early return, helpers.go:581-583
  }
}

// ---- bitmap and Kleene words (bitmap.cu) ----
enum WordOp {
  W_AND = 0, W_OR, W_XOR, W_ANDNOT, W_XNOR,   // == AG_BITOP_*
  W_COPY, W_INVERT, W_SET0, W_SET1,
  // Kleene: inputs (lvalid, ldata, rvalid, rdata)
  W_KAND_V, W_KAND_D, W_KOR_V, W_KOR_D, W_KANDNOT_V, W_KANDNOT_D,
};

template <int kOp>
__device__ __forceinline__ uint32_t word_op(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  switch (kOp) {
    case W_AND: return a & b;
    case W_OR: return a | b;
    case W_XOR: return a ^ b;
    case W_ANDNOT: return a & ~b;
    case W_XNOR: return ~(a ^ b);
    case W_COPY: return a;
    case W_INVERT: return ~a;
    case W_SET0: return 0u;
    case W_SET1: return 0xffffffffu;
    default: break;
  }
  // Kleene (scalar_boolean.go:42-46): a=lvalid b=ldata c=rvalid d=rdata
  const uint32_t lt = a & b, lf = a & ~b, rt = c & d, rf = c & ~d;
  switch (kOp) {
    case W_KAND_V: return lf | rf | (lt & rt);
    case W_KAND_D: return lt & rt;
    case W_KOR_V: return lt | rt | (lf & rf);
    case W_KOR_D: return lt | rt;
    case W_KANDNOT_V: return lf | rt | (lt & rf);
    case W_KANDNOT_D: return lt & rf;
    default: return 0;
  }
}

}  // namespace ag
