package arrowgpu

/*
#include <stdlib.h>
#include "arrowgpu.h"
*/
import "C"

import (
	"context"
	"fmt"
	"runtime"
	"unsafe"

	"github.com/apache/arrow-go/v18/arrow"
	"github.com/apache/arrow-go/v18/arrow/array"
	"github.com/apache/arrow-go/v18/arrow/compute"
	"github.com/apache/arrow-go/v18/arrow/compute/exec"
	"github.com/apache/arrow-go/v18/arrow/compute/internal/kernels"
	"github.com/apache/arrow-go/v18/arrow/memory"
)

// ---- is_in (scalar_set_lookup.go:70-171, kernels/scalar_set_lookup.go:112-413) ---------------------------------
//
// The reference's kernel state is a memo table of the value set; here it is the value set itself as ONE array of the
// argument's type (cast with SafeCastOptions and concatenated exactly where initSetLookup does it), and the table is
// built on the device inside ag_is_in.  Values are compared by their raw bytes on both sides, like the memo tables.

type setState struct {
	set      arrow.Array
	behavior C.int // NullMatchingBehavior: MATCH 0, SKIP 1, EMIT_NULL 2, INCONCLUSIVE 3 (= AG_NULL_*)
}

func initIsIn(ctx *exec.KernelCtx, args exec.KernelInitArgs) (exec.KernelState, error) {
	if args.Options == nil {
		return nil, fmt.Errorf("%w: calling a set lookup function without SetOptions", compute.ErrInvalid)
	}
	opts, ok := args.Options.(*compute.SetOptions)
	if !ok {
		return nil, fmt.Errorf("%w: expected SetOptions, got %T", compute.ErrInvalid, args.Options)
	}
	valueset, ok := opts.ValueSet.(compute.ArrayLikeDatum)
	if !ok {
		return nil, fmt.Errorf("%w: expected array-like datum, got %T", compute.ErrInvalid, opts.ValueSet)
	}
	argType := args.Inputs[0]
	var owned compute.Datum
	if !arrow.TypeEqual(valueset.Type(), argType) { // scalar_set_lookup.go:94-112: the set is cast to the argument's type
		result, err := compute.CastDatum(ctx.Ctx, valueset, compute.SafeCastOptions(argType))
		if err != nil {
			return nil, fmt.Errorf("%w: array type doesn't match type of values set: %s vs %s", compute.ErrInvalid, argType, valueset.Type())
		}
		owned = result
		valueset = result.(compute.ArrayLikeDatum)
	}
	if owned != nil {
		defer owned.Release()
	}
	var set arrow.Array
	switch valueset.Kind() {
	case compute.KindArray:
		set = valueset.(*compute.ArrayDatum).MakeArray()
	case compute.KindChunked:
		var err error
		if set, err = array.Concatenate(valueset.(*compute.ChunkedDatum).Value.Chunks(), exec.GetAllocator(ctx.Ctx)); err != nil {
			return nil, err
		}
	default:
		return nil, fmt.Errorf("%w: expected array or chunked array, got %s", compute.ErrInvalid, opts.ValueSet.Kind())
	}
	return &setState{set: set, behavior: C.int(opts.NullBehavior)}, nil
}

// isInExec writes the data and validity bitmaps of one batch (isInKernelExec :373-413).  The kernel is registered with
// CanWriteIntoSlices = false, so `out` is a fresh allocation at bit offset 0 — what the C entry point expects.
func isInExec(ctx *exec.KernelCtx, batch *exec.ExecSpan, out *exec.ExecResult) error {
	st := ctx.State.(*setState)
	in := &batch.Values[0].Array
	if out.Offset != 0 {
		return fmt.Errorf("%w: arrowgpu: is_in into a sliced output", arrow.ErrNotImplemented)
	}
	set := st.set.Data()
	var setValid *C.uint8_t
	if set.NullN() != 0 && set.Buffers()[0] != nil {
		setValid = bitmap(set.Buffers()[0].Bytes())
	}
	var setVals []byte
	if set.Len() > 0 {
		setVals = set.Buffers()[1].Bytes()
	}
	bw := in.Type.(arrow.FixedWidthDataType).BitWidth()
	var nulls C.int64_t
	err := check(C.ag_is_in(C.int(bw), base0(in.Buffers[1].Buf), validityOf(in), C.int64_t(in.Offset), C.int64_t(in.Len),
		base0(setVals), setValid, C.int64_t(set.Offset()), C.int64_t(set.Len()), st.behavior,
		bitmap(out.Buffers[1].Buf), bitmap(out.Buffers[0].Buf), &nulls))
	if err != nil {
		return err
	}
	out.Nulls = int64(nulls)
	return nil
}

func isInFunction() *compute.ScalarFunction {
	fn := compute.NewScalarFunction("is_in", compute.Unary(), compute.EmptyFuncDoc)
	for _, ty := range numericTypes {
		kn := exec.NewScalarKernel([]exec.InputType{exec.NewExactInput(ty)}, exec.NewOutputType(arrow.FixedWidthTypes.Boolean), isInExec, initIsIn)
		kn.MemAlloc = exec.MemPrealloc                 // scalar_set_lookup.go:190-191
		kn.NullHandling = exec.NullComputedPrealloc
		kn.CanWriteIntoSlices = false
		kn.CleanupFn = func(state exec.KernelState) error {
			if s, ok := state.(*setState); ok && s.set != nil {
				s.set.Release()
				s.set = nil
			}
			return nil
		}
		if err := fn.AddKernel(kn); err != nil {
			panic(err)
		}
	}
	return fn
}

// ---- unique (vector_hash.go:105-113, kernels/vector_hash.go) -------------------------------------------------------
//
// The reference hashes chunk by chunk into one memo table and materialises it in Finalize; ag_unique needs the whole
// column at once (the first row of every key is a global minimum), so the kernel is not chunk-wise: a chunked input is
// concatenated first.  Output: the distinct values in order of first appearance, one null where it first appears.

func uniqueExec(ctx *exec.KernelCtx, batch *exec.ExecSpan, out *exec.ExecResult) error {
	in := &batch.Values[0].Array
	bw := in.Type.(arrow.FixedWidthDataType).BitWidth()
	preallocate(ctx, in.Len, bw, in.MayHaveNulls(), out) // n slots are always enough; Len is trimmed below
	var outLen, outNulls C.int64_t
	err := check(C.ag_unique(C.int(bw), base0(in.Buffers[1].Buf), validityOf(in), C.int64_t(in.Offset), C.int64_t(in.Len),
		base0(out.Buffers[1].Buf), bitmap(out.Buffers[0].Buf), &outLen, &outNulls))
	if err != nil {
		return err
	}
	out.Len, out.Nulls = int64(outLen), int64(outNulls)
	return nil
}

func uniqueChunked(ctx *exec.KernelCtx, cols []*arrow.Chunked, out *exec.ExecResult) ([]*exec.ExecResult, error) {
	arr, err := array.Concatenate(cols[0].Chunks(), exec.GetAllocator(ctx.Ctx))
	if err != nil {
		return nil, err
	}
	defer arr.Release()
	span := exec.ExecSpan{Len: int64(arr.Len()), Values: make([]exec.ExecValue, 1)}
	span.Values[0].Array.SetMembers(arr.Data())
	if err := uniqueExec(ctx, &span, out); err != nil {
		return nil, err
	}
	return []*exec.ExecResult{out}, nil
}

func uniqueFunction() *compute.VectorFunction {
	fn := compute.NewVectorFunction("unique", compute.Unary(), compute.EmptyFuncDoc)
	for _, ty := range numericTypes {
		k := exec.NewVectorKernel([]exec.InputType{exec.NewExactInput(ty)}, kernels.OutputFirstType, uniqueExec, nil)
		k.CanExecuteChunkWise = false
		k.ExecChunked = uniqueChunked
		k.NullHandling = exec.NullComputedNoPrealloc
		k.MemAlloc = exec.MemNoPrealloc
		if err := fn.AddKernel(k); err != nil {
			panic(err)
		}
	}
	return fn
}

// ---- dictionary_encode (vector_hash.go:105-121, kernels/vector_hash.go:144-241) --------------------------------------
//
// Not chunk-wise: the dictionary is shared by every chunk and built over the whole column, so ExecChunked hands all
// chunks to ONE ag_dictionary_encode call (rows numbered across chunks) instead of concatenating them.  Output:
// Dictionary<int32, T>; empty chunks are dropped by the executor's WrapResults as in the reference.

func dictEncodeNulls(ctx *exec.KernelCtx) (C.int, error) {
	opts, ok := ctx.State.(kernels.DictionaryEncodeOptions)
	if !ok {
		return C.AG_NULL_ENCODING_MASK, nil // no options: Mask, the reference's default
	}
	switch opts.NullEncoding {
	case kernels.NullEncodingMask:
		return C.AG_NULL_ENCODING_MASK, nil
	case kernels.NullEncodingEncode:
		return C.AG_NULL_ENCODING_ENCODE, nil
	}
	return 0, fmt.Errorf("%w: invalid NullEncodingBehavior %d", arrow.ErrInvalid, opts.NullEncoding)
}

func dictEncodeSpans(ctx *exec.KernelCtx, ins []*exec.ArraySpan) ([]*exec.ExecResult, error) {
	ne, err := dictEncodeNulls(ctx)
	if err != nil {
		return nil, err
	}
	valueType := ins[0].Type
	bw := valueType.(arrow.FixedWidthDataType).BitWidth()
	total := int64(0)
	outs := make([]*exec.ExecResult, len(ins))
	descs := make([]C.ag_dict_chunk, len(ins))
	for i, in := range ins {
		out := &exec.ExecResult{Type: &arrow.DictionaryType{IndexType: arrow.PrimitiveTypes.Int32, ValueType: valueType}}
		preallocate(ctx, in.Len, 32, in.MayHaveNulls() && ne == C.AG_NULL_ENCODING_MASK, out)
		descs[i] = C.ag_dict_chunk{values: base0(in.Buffers[1].Buf), validity: validityOf(in), offset: C.int64_t(in.Offset),
			length: C.int64_t(in.Len), indices: (*C.int32_t)(base0(out.Buffers[1].Buf)), indices_validity: bitmap(out.Buffers[0].Buf)}
		outs[i] = out
		total += in.Len
	}
	// the call writes into scratch room for every row; the result keeps a copy of the dictionary's k values only
	scratch := make([]byte, total*int64(bw/8)+8)
	var scratchValid []byte
	if ne == C.AG_NULL_ENCODING_ENCODE {
		scratchValid = make([]byte, total/8+8)
	}
	counts := make([]C.int64_t, len(ins)+2)
	var descPtr *C.ag_dict_chunk
	if len(descs) > 0 {
		descPtr = &descs[0]
	}
	if err := check(C.ag_dictionary_encode(C.int(bw), descPtr, C.int64_t(len(descs)), ne, base0(scratch),
		bitmap(scratchValid), &counts[0])); err != nil {
		return nil, err
	}
	k := int64(counts[0])
	dict := &exec.ArraySpan{Type: valueType}
	preallocate(ctx, k, bw, counts[1] != 0, dict)
	copy(dict.Buffers[1].Buf, scratch[:k*int64(bw/8)])
	if counts[1] != 0 {
		copy(dict.Buffers[0].Buf, scratchValid[:(k+7)/8])
	}
	dict.Nulls = int64(counts[1])
	for i, out := range outs {
		out.Nulls = int64(counts[2+i])
		if out.Nulls == 0 {
			out.Buffers[0] = exec.BufferSpan{} // the indices' validity is present only when they hold nulls
		}
		out.SetDictionary(dict)
	}
	return outs, nil
}

func dictEncodeExec(ctx *exec.KernelCtx, batch *exec.ExecSpan, out *exec.ExecResult) error {
	res, err := dictEncodeSpans(ctx, []*exec.ArraySpan{&batch.Values[0].Array})
	if err != nil {
		return err
	}
	*out = *res[0]
	return nil
}

func dictEncodeChunked(ctx *exec.KernelCtx, cols []*arrow.Chunked, _ *exec.ExecResult) ([]*exec.ExecResult, error) {
	chunks := cols[0].Chunks()
	ins := make([]*exec.ArraySpan, len(chunks))
	for i, c := range chunks {
		ins[i] = &exec.ArraySpan{}
		ins[i].SetMembers(c.Data())
	}
	if len(ins) == 0 {
		return nil, nil
	}
	return dictEncodeSpans(ctx, ins)
}

func dictionaryEncodeFunction() *compute.VectorFunction {
	fn := compute.NewVectorFunction("dictionary_encode", compute.Unary(), compute.EmptyFuncDoc)
	for _, ty := range numericTypes {
		outType := &arrow.DictionaryType{IndexType: arrow.PrimitiveTypes.Int32, ValueType: ty}
		k := exec.NewVectorKernel([]exec.InputType{exec.NewExactInput(ty)}, exec.NewOutputType(outType), dictEncodeExec,
			func(_ *exec.KernelCtx, args exec.KernelInitArgs) (exec.KernelState, error) {
				if o, ok := args.Options.(*kernels.DictionaryEncodeOptions); ok {
					return *o, nil
				}
				return nil, nil
			})
		k.CanExecuteChunkWise = false
		k.ExecChunked = dictEncodeChunked
		k.NullHandling = exec.NullComputedNoPrealloc
		k.MemAlloc = exec.MemNoPrealloc
		if err := fn.AddKernel(k); err != nil {
			panic(err)
		}
	}
	return fn
}

// ---- sort_indices (vector_sort.go:42-204, kernels.SortIndices vector_sort.go:385-481) -------------------------------
//
// A MetaFunction in the reference.  Every input whose key columns are numeric or boolean goes to ag_sort_indices_keys:
// an array or chunked array by its first key (ColumnIndex ignored, vector_sort.go:130-152), a record batch or table by
// every key, whatever the chunking of its columns.  The device order places NaN next to the nulls on every path
// (DESIGN §2).  Other key types, invalid column indices (so the parent reports them) and calls without SortOptions go
// to the parent's implementation.

func sortIndicesFunction(parent compute.Function) *compute.MetaFunction {
	return compute.NewMetaFunction("sort_indices", compute.Unary(), compute.EmptyFuncDoc,
		func(ctx context.Context, opts compute.FunctionOptions, args ...compute.Datum) (compute.Datum, error) {
			keys, isKeys := opts.(compute.SortOptions)
			if isKeys && len(keys) >= 1 {
				if cols, ks, n, ok := sortKeyColumns(args[0], keys); ok {
					return sortKeyed(ctx, cols, ks, n)
				}
			}
			if parent == nil {
				return nil, fmt.Errorf("%w: unsupported type for sort_indices operation: %s", arrow.ErrNotImplemented, args[0])
			}
			return parent.Execute(ctx, opts, args...)
		})
}

func isNumeric(dt arrow.DataType) bool {
	for _, ty := range numericTypes {
		if arrow.TypeEqual(ty, dt) {
			return true
		}
	}
	return false
}

func isSortable(dt arrow.DataType) bool { return dt.ID() == arrow.BOOL || isNumeric(dt) }

// sortColumn is one key column: its type and the data of its chunks.
type sortColumn struct {
	dt     arrow.DataType
	chunks []arrow.ArrayData
}

// sortKeyColumns resolves the chunks of every key column; ok is false when the device cannot take the call.  Only
// arrow.ArrayData is kept: the datum owns it for the duration of the call.
func sortKeyColumns(d compute.Datum, keys compute.SortOptions) (cols []sortColumn, ks []compute.SortKey, n int64, ok bool) {
	chunksOf := func(c *arrow.Chunked) sortColumn {
		col := sortColumn{dt: c.DataType()}
		for _, ch := range c.Chunks() {
			col.chunks = append(col.chunks, ch.Data())
		}
		return col
	}
	switch in := d.(type) {
	case *compute.ArrayDatum:
		return []sortColumn{{in.Value.DataType(), []arrow.ArrayData{in.Value}}}, keys[:1], int64(in.Value.Len()), isSortable(in.Value.DataType())
	case *compute.ChunkedDatum:
		return []sortColumn{chunksOf(in.Value)}, keys[:1], int64(in.Value.Len()), isSortable(in.Value.DataType())
	case *compute.RecordDatum:
		batch := in.Value
		for _, k := range keys {
			if k.ColumnIndex < 0 || int64(k.ColumnIndex) >= batch.NumCols() || !isSortable(batch.Column(k.ColumnIndex).DataType()) {
				return nil, nil, 0, false
			}
			col := batch.Column(k.ColumnIndex)
			cols = append(cols, sortColumn{col.DataType(), []arrow.ArrayData{col.Data()}})
		}
		return cols, keys, batch.NumRows(), true
	case *compute.TableDatum:
		tbl := in.Value
		for _, k := range keys {
			if k.ColumnIndex < 0 || int64(k.ColumnIndex) >= tbl.NumCols() || !isSortable(tbl.Column(k.ColumnIndex).DataType()) {
				return nil, nil, 0, false
			}
			cols = append(cols, chunksOf(tbl.Column(k.ColumnIndex).Data()))
		}
		return cols, keys, tbl.NumRows(), true
	}
	return nil, nil, 0, false
}

func sortKeyed(ctx context.Context, cols []sortColumn, keys []compute.SortKey, n int64) (compute.Datum, error) {
	// The key and chunk descriptors live in C memory.  The buffers they point at may be Go memory (a Go allocator's
	// arrays), so they stay pinned until the call returns (cgo pointer rules); Pin does nothing for C memory.
	var pin runtime.Pinner
	defer pin.Unpin()
	total := 0
	for _, col := range cols {
		total += len(col.chunks)
	}
	descs := unsafe.Slice((*C.ag_sort_key)(C.malloc(C.size_t(len(cols))*C.size_t(unsafe.Sizeof(C.ag_sort_key{})))), len(cols))
	defer C.free(unsafe.Pointer(&descs[0]))
	chunkMem := (*C.ag_sort_chunk)(C.malloc(C.size_t(max(total, 1)) * C.size_t(unsafe.Sizeof(C.ag_sort_chunk{}))))
	defer C.free(unsafe.Pointer(chunkMem))
	chunks := unsafe.Slice(chunkMem, max(total, 1))
	next := 0
	for i, col := range cols {
		first := next
		for _, data := range col.chunks {
			var vals []byte
			if data.Len() > 0 {
				vals = data.Buffers()[1].Bytes()
			}
			var valid *C.uint8_t
			if data.NullN() != 0 && data.Buffers()[0] != nil {
				valid = bitmap(data.Buffers()[0].Bytes())
			}
			if p := base0(vals); p != nil {
				pin.Pin(p)
			}
			if valid != nil {
				pin.Pin(valid)
			}
			chunks[next] = C.ag_sort_chunk{vals: base0(vals), valid: valid, offset: C.int64_t(data.Offset()), length: C.int64_t(data.Len())}
			next++
		}
		var firstChunk *C.ag_sort_chunk // a column without chunks (no rows) has none to point at
		if next > first {
			firstChunk = &chunks[first]
		}
		// arrow.Type ids are the AG_TYPE_* ids; SortOrder / NullPlacement are 0 / 1 on both sides (kernels/vector_sort.go:34-46)
		descs[i] = C.ag_sort_key{_type: C.int(col.dt.ID()), order: C.int(keys[i].Order), null_placement: C.int(keys[i].NullPlacement),
			nchunks: C.int(next - first), chunks: firstChunk}
	}
	buf := memory.NewResizableBuffer(exec.GetAllocator(ctx))
	buf.Resize(int(n) * 8)
	err := check(C.ag_sort_indices_keys(C.int(len(descs)), &descs[0], C.int64_t(n), (*C.uint64_t)(base0(buf.Bytes()))))
	if err != nil {
		buf.Release()
		return nil, err
	}
	out := array.NewData(arrow.PrimitiveTypes.Uint64, int(n), []*memory.Buffer{nil, buf}, nil, 0, 0)
	buf.Release() // NewData retained it
	return &compute.ArrayDatum{Value: out}, nil
}

// registerLookupSort adds is_in, unique, dictionary_encode and sort_indices to a registry built by NewRegistry.
func registerLookupSort(reg, parent compute.FunctionRegistry) {
	addScalar(reg, parent, isInFunction())
	addVector(reg, parent, uniqueFunction())
	addVector(reg, parent, dictionaryEncodeFunction()) // other types (and dictionary inputs) go to the parent's kernels
	p, _ := parent.GetFunction("sort_indices")
	reg.AddFunction(sortIndicesFunction(p), true)
}
