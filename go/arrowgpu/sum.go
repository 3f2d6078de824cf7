package arrowgpu

/*
#include "arrowgpu.h"
*/
import "C"

import (
	"unsafe"

	"github.com/apache/arrow-go/v18/arrow/array"
)

// arrow/math.Float64Funcs.Sum has no plugin point (the function pointer is an unexported field set in init,
// arrow/math/float64.go:25-31), so the GPU reductions are siblings with the same semantics: validity is ignored,
// values[offset:offset+len] are summed, an empty array gives 0 (float64.go:34-39).

// SumFloat64 returns a compensated sum: |res - S| <= 2 eps |S| + gamma_n^2 sum|x|, so within 1 ULP of the correctly
// rounded sum on well-conditioned data (the reference's AVX2 / SSE4 / pure-Go builds give three different last bits
// on general data; when every partial sum is exact all agree with this one).  A NaN, or +inf and -inf together, give
// NaN; infinities or an overflow of one sign give that infinity.
func SumFloat64(a *array.Float64) float64 {
	v := a.Float64Values()
	if len(v) == 0 {
		return 0
	}
	var r C.double
	if err := check(C.ag_sum_f64((*C.double)(unsafe.Pointer(&v[0])), C.size_t(len(v)), &r)); err != nil {
		panic(err)
	}
	return float64(r)
}

// SumFloat64ReferenceOrder reproduces sum_float64_avx2 (float64_avx2_amd64.s) bit for bit on any input.
func SumFloat64ReferenceOrder(a *array.Float64) float64 {
	v := a.Float64Values()
	if len(v) == 0 {
		return 0
	}
	var r C.double
	if err := check(C.ag_sum_f64_reforder((*C.double)(unsafe.Pointer(&v[0])), C.size_t(len(v)), &r)); err != nil {
		panic(err)
	}
	return float64(r)
}

func SumInt64(a *array.Int64) int64 {
	v := a.Int64Values()
	if len(v) == 0 {
		return 0
	}
	var r C.int64_t
	if err := check(C.ag_sum_i64((*C.int64_t)(unsafe.Pointer(&v[0])), C.size_t(len(v)), &r)); err != nil {
		panic(err)
	}
	return int64(r)
}

func SumUint64(a *array.Uint64) uint64 {
	v := a.Uint64Values()
	if len(v) == 0 {
		return 0
	}
	var r C.uint64_t
	if err := check(C.ag_sum_u64((*C.uint64_t)(unsafe.Pointer(&v[0])), C.size_t(len(v)), &r)); err != nil {
		panic(err)
	}
	return uint64(r)
}
