package arrowgpu

/*
#include <stdlib.h>
#include "arrowgpu.h"
*/
import "C"

import (
	"context"
	"runtime"
	"unsafe"

	"github.com/apache/arrow-go/v18/arrow"
	"github.com/apache/arrow-go/v18/arrow/array"
	"github.com/apache/arrow-go/v18/arrow/bitutil"
	"github.com/apache/arrow-go/v18/arrow/compute"
	"github.com/apache/arrow-go/v18/arrow/compute/exec"
	"github.com/apache/arrow-go/v18/arrow/memory"
)

// ---- take on record batches and tables (selection.go:93-204) -----------------------------------------------------
//
// A MetaFunction in the reference, which takes a record batch or table column by column.  Here every column of a
// record batch or table whose columns are all boolean or numeric, with integer indices, is gathered by one
// ag_take_columns call per index chunk: a record batch by the concatenated indices (takeRecordImpl), a table with one
// output chunk per index chunk (takeTableImpl).  Arrays, chunked arrays and every other input go to the parent's take.
// arrow-go's Sort calls "take" through the registry, so it reaches this path too; FilterRecordBatch and FilterTable
// already reach the device per column through array_take.

func takeFunction(parent compute.Function) *compute.MetaFunction {
	return compute.NewMetaFunction("take", compute.Binary(), compute.EmptyFuncDoc,
		func(ctx context.Context, opts compute.FunctionOptions, args ...compute.Datum) (compute.Datum, error) {
			if cols, nrows, ok := selectionColumns(args[0]); ok && integerIndices(args[1]) {
				bounds := true
				if o, isTake := opts.(*compute.TakeOptions); isTake {
					bounds = o.BoundsCheck
				}
				return takeColumnsDatum(ctx, args[0], cols, nrows, args[1], bounds)
			}
			return parent.Execute(ctx, opts, args...)
		})
}

func integerIndices(d compute.Datum) bool {
	if a, ok := d.(compute.ArrayLikeDatum); ok && (d.Kind() == compute.KindArray || d.Kind() == compute.KindChunked) {
		return arrow.IsInteger(a.Type().ID())
	}
	return false
}

// selectionColumns: the columns of a record batch or table as chunk lists; ok is false for any other input or when a
// column is neither boolean nor numeric.
func selectionColumns(d compute.Datum) (cols []sortColumn, nrows int64, ok bool) {
	switch in := d.(type) {
	case *compute.RecordDatum:
		for _, c := range in.Value.Columns() {
			if !isSortable(c.DataType()) {
				return nil, 0, false
			}
			cols = append(cols, sortColumn{c.DataType(), []arrow.ArrayData{c.Data()}})
		}
		return cols, in.Value.NumRows(), true
	case *compute.TableDatum:
		for i := 0; i < int(in.Value.NumCols()); i++ {
			c := in.Value.Column(i).Data()
			if !isSortable(c.DataType()) {
				return nil, 0, false
			}
			col := sortColumn{dt: c.DataType()}
			for _, ch := range c.Chunks() {
				col.chunks = append(col.chunks, ch.Data())
			}
			cols = append(cols, col)
		}
		return cols, in.Value.NumRows(), true
	}
	return nil, 0, false
}

func takeColumnsDatum(ctx context.Context, values compute.Datum, cols []sortColumn, nrows int64, indices compute.Datum, bounds bool) (compute.Datum, error) {
	mem := exec.GetAllocator(ctx)
	var idx []arrow.Array
	switch in := indices.(type) {
	case *compute.ArrayDatum:
		a := in.MakeArray()
		defer a.Release()
		idx = []arrow.Array{a}
	case *compute.ChunkedDatum:
		idx = in.Value.Chunks()
		if values.Kind() == compute.KindRecord { // takeRecordImpl concatenates chunked indices first
			cat, err := array.Concatenate(idx, mem)
			if err != nil {
				return nil, err
			}
			defer cat.Release()
			idx = []arrow.Array{cat}
		}
	}
	idxNulls := false
	for _, a := range idx {
		idxNulls = idxNulls || a.NullN() != 0
	}
	out := make([][]arrow.Array, len(cols))
	release := func() {
		for _, c := range out {
			for _, a := range c {
				a.Release()
			}
		}
	}
	if len(cols) > 0 { // the reference takes column by column: without columns nothing is gathered or checked
		for _, ix := range idx {
			res, err := takeColumns(mem, cols, nrows, ix, idxNulls, bounds)
			if err != nil {
				release()
				return nil, err
			}
			for c := range cols {
				out[c] = append(out[c], res[c])
			}
		}
	}
	defer release()
	if rec, ok := values.(*compute.RecordDatum); ok {
		arrs := make([]arrow.Array, len(cols))
		for c := range cols {
			arrs[c] = out[c][0]
		}
		return &compute.RecordDatum{Value: array.NewRecordBatch(rec.Value.Schema(), arrs, int64(idx[0].Len()))}, nil
	}
	tbl := values.(*compute.TableDatum).Value
	columns := make([]arrow.Column, len(cols))
	for c := range cols {
		chk := arrow.NewChunked(cols[c].dt, out[c])
		columns[c] = *arrow.NewColumn(tbl.Schema().Field(c), chk)
		chk.Release()
	}
	defer func() {
		for i := range columns {
			columns[i].Release()
		}
	}()
	return &compute.TableDatum{Value: array.NewTable(tbl.Schema(), columns, -1)}, nil
}

// takeColumns gathers every column by one index array in one ag_take_columns call.  The descriptors live in C memory
// and the Go buffers they point at stay pinned for the call (cgo pointer rules).
func takeColumns(mem memory.Allocator, cols []sortColumn, nrows int64, idx arrow.Array, idxNulls, bounds bool) ([]arrow.Array, error) {
	var pin runtime.Pinner
	defer pin.Unpin()
	n := idx.Len()
	total := 0
	for _, col := range cols {
		total += len(col.chunks)
	}
	descs := unsafe.Slice((*C.ag_take_column)(C.malloc(C.size_t(len(cols))*C.size_t(unsafe.Sizeof(C.ag_take_column{})))), len(cols))
	defer C.free(unsafe.Pointer(&descs[0]))
	chunkMem := (*C.ag_sort_chunk)(C.malloc(C.size_t(max(total, 1)) * C.size_t(unsafe.Sizeof(C.ag_sort_chunk{}))))
	defer C.free(unsafe.Pointer(chunkMem))
	chunks := unsafe.Slice(chunkMem, max(total, 1))
	pinned := func(b []byte) *C.uint8_t {
		if p := base0(b); p != nil {
			pin.Pin(p)
			return (*C.uint8_t)(p)
		}
		return nil
	}
	vals := make([]*memory.Buffer, len(cols))
	valid := make([]*memory.Buffer, len(cols))
	next := 0
	for i, col := range cols {
		first := next
		nullable := idxNulls
		for _, data := range col.chunks {
			var v []byte
			if data.Len() > 0 {
				v = data.Buffers()[1].Bytes()
			}
			var ok *C.uint8_t
			if data.NullN() != 0 && data.Buffers()[0] != nil {
				ok = pinned(data.Buffers()[0].Bytes())
				nullable = true
			}
			chunks[next] = C.ag_sort_chunk{vals: unsafe.Pointer(pinned(v)), valid: ok, offset: C.int64_t(data.Offset()), length: C.int64_t(data.Len())}
			next++
		}
		var firstChunk *C.ag_sort_chunk
		if next > first {
			firstChunk = &chunks[first]
		}
		nbytes := int(bitutil.BytesForBits(int64(n)))
		if col.dt.ID() != arrow.BOOL {
			nbytes = n * col.dt.(arrow.FixedWidthDataType).BitWidth() / 8
		}
		vals[i] = memory.NewResizableBuffer(mem)
		vals[i].Resize(nbytes)
		var outValid *C.uint8_t
		if nullable { // allocValidity (vector_selection.go:1175)
			valid[i] = memory.NewResizableBuffer(mem)
			valid[i].Resize(int(bitutil.BytesForBits(int64(n))))
			outValid = pinned(valid[i].Bytes())
		}
		descs[i] = C.ag_take_column{_type: C.int(col.dt.ID()), nchunks: C.int(next - first), chunks: firstChunk,
			out: unsafe.Pointer(pinned(vals[i].Bytes())), out_valid: outValid}
	}
	data := idx.Data()
	iw := data.DataType().(arrow.FixedWidthDataType).BitWidth()
	var ivalid *C.uint8_t
	if idx.NullN() != 0 && data.Buffers()[0] != nil {
		ivalid = pinned(data.Buffers()[0].Bytes())
	}
	var iptr unsafe.Pointer
	if n > 0 {
		iptr = unsafe.Pointer(&data.Buffers()[1].Bytes()[data.Offset()*iw/8])
		pin.Pin(iptr)
	}
	signed := C.int(0)
	if arrow.IsSignedInteger(data.DataType().ID()) {
		signed = 1
	}
	check0 := C.int(0)
	if bounds {
		check0 = 1
	}
	var badPos, badIdx C.int64_t
	err := check(C.ag_take_columns(C.int(len(cols)), &descs[0], C.int64_t(nrows), C.int(iw), signed, iptr, ivalid,
		C.int64_t(data.Offset()), C.int64_t(n), check0, &badPos, &badIdx))
	out := make([]arrow.Array, len(cols))
	for i, col := range cols {
		if err == nil {
			nulls := 0
			if valid[i] != nil {
				nulls = array.UnknownNullCount
			}
			d := array.NewData(col.dt, n, []*memory.Buffer{valid[i], vals[i]}, nil, nulls, 0)
			out[i] = array.MakeFromData(d)
			d.Release()
		}
		vals[i].Release()
		if valid[i] != nil {
			valid[i].Release()
		}
	}
	if err != nil {
		return nil, err
	}
	return out, nil
}

// registerSelection adds the take meta function to a registry built by NewRegistry.
func registerSelection(reg, parent compute.FunctionRegistry) {
	p, _ := parent.GetFunction("take")
	reg.AddFunction(takeFunction(p), true)
}
