package arrowgpu

/*
#include "arrowgpu.h"
*/
import "C"

import (
	"fmt"

	"github.com/apache/arrow-go/v18/arrow"
	"github.com/apache/arrow-go/v18/arrow/compute"
	"github.com/apache/arrow-go/v18/arrow/compute/exec"
	"github.com/apache/arrow-go/v18/arrow/compute/internal/kernels"
)

// ---- run_end_encode / run_end_decode (vector_run_ends.go:46-85, kernels/vector_run_end_encode.go) -------------------
//
// Chunk-wise vector kernels for BOOL and the numeric types; every other value type (strings, binary, fixed-size binary)
// keeps the parent registry's kernels through vectorDelegating.  Encode is the reference's CountNumberOfRuns then
// WriteEncodedRuns (:531-565): ag_run_end_count sizes the children exactly, ag_run_end_encode fills them.  Decode
// clips the last run at offset+length and refuses malformed run ends with ErrInvalid (see DESIGN.md §8).

var runEndTypes = []arrow.DataType{arrow.PrimitiveTypes.Int16, arrow.PrimitiveTypes.Int32, arrow.PrimitiveTypes.Int64}

// byteOrBit is the element width in bits of a value type (1 for BOOL).
func byteOrBit(dt arrow.DataType) int {
	if dt.ID() == arrow.BOOL {
		return 1
	}
	return int(byteWidth(dt) * 8)
}

func runEndEncodeExec(ctx *exec.KernelCtx, batch *exec.ExecSpan, out *exec.ExecResult) error {
	opts, ok := ctx.State.(kernels.RunEndEncodeState)
	if !ok {
		return fmt.Errorf("%w: function 'run_end_encode' cannot be called without options", arrow.ErrInvalid)
	}
	rt := opts.RunEndType
	switch rt.ID() {
	case arrow.INT16, arrow.INT32, arrow.INT64:
	default:
		return fmt.Errorf("%w: bad run end type %s", arrow.ErrInvalid, rt)
	}
	in := &batch.Values[0].Array
	vt := in.Type
	var counts [2]C.int64_t
	if err := check(C.ag_run_end_count(C.int(vt.ID()), base0(in.Buffers[1].Buf), bitmap(in.Buffers[0].Buf), C.int64_t(in.Offset),
		C.int64_t(in.Len), &counts[0])); err != nil {
		return err
	}
	runs := int64(counts[0])
	out.Type = arrow.RunEndEncodedOf(rt, vt)
	out.Len = in.Len
	out.Nulls = 0
	out.Children = make([]exec.ArraySpan, 2)
	ends, values := &out.Children[0], &out.Children[1]
	ends.Type, values.Type = rt, vt
	preallocate(ctx, runs, int(byteWidth(rt)*8), false, ends)
	// the values child has a validity bitmap iff the input has one (PreallocOutput, :143-180)
	preallocate(ctx, runs, byteOrBit(vt), in.Buffers[0].Buf != nil, values)
	if err := check(C.ag_run_end_encode(C.int(vt.ID()), C.int(rt.ID()), base0(in.Buffers[1].Buf), bitmap(in.Buffers[0].Buf),
		C.int64_t(in.Offset), C.int64_t(in.Len), base0(ends.Buffers[1].Buf), base0(values.Buffers[1].Buf),
		bitmap(values.Buffers[0].Buf), C.int64_t(runs), &counts[0])); err != nil {
		return err
	}
	values.Nulls = int64(counts[1])
	return nil
}

func runEndDecodeExec(ctx *exec.KernelCtx, batch *exec.ExecSpan, out *exec.ExecResult) error {
	in := &batch.Values[0].Array
	ends, values := &in.Children[0], &in.Children[1]
	if values.Len < ends.Len {
		return fmt.Errorf("%w: run_end_decode: the values child is shorter than run_ends", arrow.ErrInvalid)
	}
	vt := values.Type
	preallocate(ctx, in.Len, byteOrBit(vt), values.Buffers[0].Buf != nil, out)
	var nulls C.int64_t
	if err := check(C.ag_run_end_decode(C.int(vt.ID()), C.int(ends.Type.ID()), valuesAt(ends), C.int64_t(ends.Len),
		base0(values.Buffers[1].Buf), bitmap(values.Buffers[0].Buf), C.int64_t(values.Offset), C.int64_t(in.Offset),
		C.int64_t(in.Len), base0(out.Buffers[1].Buf), bitmap(out.Buffers[0].Buf), &nulls)); err != nil {
		return err
	}
	out.Nulls = int64(nulls)
	if values.Buffers[0].Buf == nil {
		out.Nulls = 0
	}
	return nil
}

func runEndFunctions() (enc, dec *compute.VectorFunction) {
	enc = compute.NewVectorFunction("run_end_encode", compute.Unary(), compute.EmptyFuncDoc)
	dec = compute.NewVectorFunction("run_end_decode", compute.Unary(), compute.EmptyFuncDoc)
	valueTypes := append(append([]arrow.DataType{}, numericTypes...), arrow.FixedWidthTypes.Boolean)
	for _, vt := range valueTypes {
		vt := vt
		k := exec.NewVectorKernel([]exec.InputType{exec.NewExactInput(vt)},
			exec.NewComputedOutputType(func(ctx *exec.KernelCtx, _ []arrow.DataType) (arrow.DataType, error) {
				opts, ok := ctx.State.(kernels.RunEndEncodeState)
				if !ok {
					return nil, fmt.Errorf("%w: function 'run_end_encode' cannot be called without options", arrow.ErrInvalid)
				}
				return arrow.RunEndEncodedOf(opts.RunEndType, vt), nil
			}), runEndEncodeExec, exec.OptionsInit[kernels.RunEndEncodeState])
		k.NullHandling = exec.NullComputedNoPrealloc
		k.MemAlloc = exec.MemNoPrealloc
		if err := enc.AddKernel(k); err != nil {
			panic(err)
		}
		for _, rt := range runEndTypes {
			dk := exec.NewVectorKernel([]exec.InputType{exec.NewExactInput(arrow.RunEndEncodedOf(rt, vt))}, exec.NewOutputType(vt),
				runEndDecodeExec, nil)
			dk.NullHandling = exec.NullComputedNoPrealloc
			dk.MemAlloc = exec.MemNoPrealloc
			if err := dec.AddKernel(dk); err != nil {
				panic(err)
			}
		}
	}
	return enc, dec
}

// registerRunEnds adds run_end_encode and run_end_decode to a registry built by NewRegistry.
func registerRunEnds(reg, parent compute.FunctionRegistry) {
	enc, dec := runEndFunctions()
	addVector(reg, parent, enc) // other value types go to the parent's kernels
	addVector(reg, parent, dec)
}
