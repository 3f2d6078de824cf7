package arrowgpu_test

import (
	"strings"
	"testing"

	"github.com/apache/arrow-go/v18/arrow"
	"github.com/apache/arrow-go/v18/arrow/array"
	"github.com/apache/arrow-go/v18/arrow/compute"
	"github.com/apache/arrow-go/v18/arrow/memory"
)

// sort_indices through ag_sort_indices_keys for a plain array, a record batch and a two-batch table, with Go-allocated
// buffers (pinned for the call) — vector_sort_test.go:1374-1395,1641-1665.
func TestSortIndicesKeys(t *testing.T) {
	ctx := gpuCtx()
	mem := memory.NewCheckedAllocator(memory.NewGoAllocator())
	defer mem.AssertSize(t, 0)
	schema := arrow.NewSchema([]arrow.Field{
		{Name: "a", Type: arrow.PrimitiveTypes.Uint8, Nullable: true},
		{Name: "b", Type: arrow.PrimitiveTypes.Uint32, Nullable: true},
	}, nil)
	b1, _, err := array.RecordFromJSON(mem, schema, strings.NewReader(`[{"a": null, "b": 5}, {"a": 1, "b": 3}, {"a": 3, "b": null}]`))
	if err != nil {
		t.Fatal(err)
	}
	defer b1.Release()
	b2, _, err := array.RecordFromJSON(mem, schema, strings.NewReader(
		`[{"a": null, "b": null}, {"a": 2, "b": 5}, {"a": 1, "b": 5}, {"a": 3, "b": 5}]`))
	if err != nil {
		t.Fatal(err)
	}
	defer b2.Release()
	tbl := array.NewTableFromRecords(schema, []arrow.RecordBatch{b1, b2})
	defer tbl.Release()

	keys := func(atStart bool) compute.SortOptions { // (a ascending, b descending), one placement for both
		k0, k1 := compute.DefaultSortKey(), compute.DefaultSortKey()
		k1.ColumnIndex, k1.Order = 1, compute.SortOrderDescending
		if atStart {
			k0.NullPlacement, k1.NullPlacement = compute.SortNullsAtStart, compute.SortNullsAtStart
		}
		return compute.SortOptions{k0, k1}
	}
	check := func(name string, d compute.Datum, opts compute.SortOptions, want string) {
		t.Helper()
		got, err := compute.CallFunction(ctx, "sort_indices", opts, d)
		if err != nil {
			t.Fatalf("%s: %v", name, err)
		}
		defer got.Release()
		w, _, _ := array.FromJSON(mem, arrow.PrimitiveTypes.Uint64, strings.NewReader(want))
		defer w.Release()
		arr := got.(*compute.ArrayDatum).MakeArray()
		defer arr.Release()
		if !array.Equal(arr, w) {
			t.Fatalf("%s: got %v want %v", name, arr, w)
		}
	}
	check("table, nulls at end", compute.NewDatumWithoutOwning(tbl), keys(false), `[5, 1, 4, 6, 2, 0, 3]`)
	check("table, nulls at start", compute.NewDatumWithoutOwning(tbl), keys(true), `[3, 0, 5, 1, 4, 2, 6]`)
	check("record batch", compute.NewDatumWithoutOwning(b1), keys(false), `[1, 2, 0]`)
	check("array, first key only", compute.NewDatumWithoutOwning(b2.Column(1)), keys(true), `[0, 1, 2, 3]`)
	check("chunked", compute.NewDatumWithoutOwning(tbl.Column(0).Data()), keys(false), `[1, 5, 4, 2, 6, 0, 3]`)
}
