"""Take on record batches and tables, FilterRecordBatch, FilterTable and Sort on the device (one ag_take_columns_dev
launch per index chunk or filter span), against the NumPy model of tests/table_select_model.py: values, every validity
bit, row counts and output chunk lengths; plus the C ABI of ag_take_columns in both flavours."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pyarrow.compute as pac
import pytest

import table_select_model as M
from arrow_go_b200 import _native as N
from arrow_go_b200 import compute as pc
from exec_model import NAME, Col, Fail, Layout, np_of, random_cuts
from helpers import Dev

pytestmark = pytest.mark.gpu

TYPES = [pc.BOOL, pc.UINT8, pc.INT8, pc.UINT16, pc.INT16, pc.UINT32, pc.INT32, pc.UINT64, pc.INT64, pc.FLOAT32, pc.FLOAT64]
IDX = [pc.INT8, pc.UINT8, pc.INT16, pc.UINT16, pc.INT32, pc.UINT32, pc.INT64, pc.UINT64]
VALIDITY = ("none", "zero_nulls", "nulls")


# ---------------------------------------------------------------------------------------------------------------
# fixtures: logical columns in random physical layouts

def _values(rng, t, n):
    dt = np_of(t)
    if t == pc.BOOL:
        return rng.random(n) < 0.5
    if dt in (np.float32, np.float64):
        return rng.standard_normal(n).astype(dt)
    return rng.integers(0, 256, n * np.dtype(dt).itemsize, dtype=np.uint8).view(dt)


def _layout(rng, n, max_chunks=8):
    cuts = random_cuts(rng, n, int(rng.integers(1, max_chunks + 1)))
    offs = [int(rng.integers(1, 18)) if rng.random() < 0.5 else 0 for _ in cuts[1:]]   # misaligned bitmap offsets
    return Layout("chunked", cuts=cuts, offsets=offs, pad=int(rng.integers(0, 9)), seed=int(rng.integers(0, 1 << 31)))


def _upload(p, t):
    m = p.offset + p.length
    return pc.Array.from_numpy(p.values[:m], None if p.valid is None else p.valid[:m], t, offset=p.offset)


class Column:
    """A logical column, its model chunks and its device form (a chunked array, or one array for a record batch)."""

    def __init__(self, rng, t, n, validity, layout=None):
        self.type = t
        valid = rng.random(n) >= 0.3 if validity == "nulls" else None
        self.col = Col(t, _values(rng, t, n), valid)
        self.layout = layout or _layout(rng, n)
        self.pieces = self.layout.pieces(self.col, bitmap=validity != "none")
        self.model = [(p.values[p.offset:p.offset + p.length], None if p.valid is None else p.valid[p.offset:p.offset + p.length])
                      for p in self.pieces]
        self.arrays = [_upload(p, t) for p in self.pieces]
        self.chunked = pc.Chunked(self.arrays, t)


def _indices(rng, t, nrows, m, nulls, chunks, oob=False):
    """(model indices, device datum): m indices of type t, valid ones in [0, nrows) unless `oob` plants offenders."""
    dt = np_of(t)
    hi = max(min(nrows, int(np.iinfo(dt).max) + 1), 1)
    v = rng.integers(0, hi, m).astype(dt)
    ok = rng.random(m) >= 0.25 if nulls else None
    if nrows == 0 and m and ok is None:
        ok = np.zeros(m, dtype=bool)
    if oob and m:
        bad = rng.integers(0, m, 3)
        v[bad] = np.array(-1 if np.issubdtype(dt, np.signedinteger) else np.iinfo(dt).max).astype(dt)
    if chunks:
        cuts = random_cuts(rng, m, chunks)
        parts = [(v[a:b], None if ok is None else ok[a:b]) for a, b in zip(cuts, cuts[1:])]
        dev = pc.Chunked([pc.Array.from_numpy(pv, pok, t) for pv, pok in parts], t)
        return (parts, True), dev
    return ([(v, ok)], False), pc.Array.from_numpy(v, ok, t)


def _check_array(got, want):
    vals, valid = want
    gv, gok, _ = got.to_numpy()
    assert len(got) == vals.size
    assert np.array_equal(gok, valid)
    assert np.array_equal(gv.view(np.uint8) if gv.dtype != bool else gv, np.asarray(vals, dtype=gv.dtype).view(np.uint8) if gv.dtype != bool else vals)


def _check_table(got, want, types):
    cols, rows = want
    assert got.kind == pc.KIND_TABLE and len(got) == rows
    gcols = got.columns()
    assert len(gcols) == len(cols)
    for gc, wc, t in zip(gcols, cols, types):
        assert gc.kind == pc.KIND_CHUNKED and gc.type == t
        chunks = gc.chunks()
        assert [len(c) for c in chunks] == [v.size for v, _ in wc]
        for c, w in zip(chunks, wc):
            _check_array(c, w)


def _check_record(got, want, types):
    cols, rows = want
    assert got.kind == pc.KIND_RECORD and len(got) == rows
    gcols = got.columns()
    assert len(gcols) == len(cols) and [c.type for c in gcols] == list(types)
    for gc, w in zip(gcols, cols):
        assert gc.kind == pc.KIND_ARRAY
        _check_array(gc, w)


def _snapshot(columns):
    return [[a.to_numpy() for a in c.arrays] for c in columns]


def _same_snapshot(a, b):
    for ca, cb in zip(a, b):
        for (va, oa, na), (vb, ob, nb) in zip(ca, cb):
            assert np.array_equal(va, vb) and np.array_equal(oa, ob) and na == nb


def _random_columns(rng, n, ncols):
    return [Column(rng, TYPES[int(rng.integers(0, len(TYPES)))], n, VALIDITY[int(rng.integers(0, 3))]) for _ in range(ncols)]


# ---------------------------------------------------------------------------------------------------------------
# take

@pytest.mark.parametrize("seed", range(24))
def test_take_table_and_record_batch(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(0, 3000))
    cols = _random_columns(rng, n, int(rng.integers(1, 7)))
    if seed % 4 == 0:   # shared chunk layouts: one chunk search for several columns
        shared = _layout(rng, n)
        cols += [Column(rng, t, n, v, shared) for t, v in ((pc.INT64, "nulls"), (pc.BOOL, "zero_nulls"), (pc.FLOAT32, "none"))]
    types = [c.type for c in cols]
    it = IDX[seed % len(IDX)]
    bounds = seed % 3 != 2
    model_idx, dev_idx = _indices(rng, it, n, int(rng.integers(0, 2500)), seed % 2 == 0, [0, 1, 3, 6][seed % 4], oob=not bounds)
    before = _snapshot(cols)
    table = pc.Table([c.chunked for c in cols], n)
    got = pc.Take(table, dev_idx, bounds_check=bounds)
    _check_table(got, M.take_table([c.model for c in cols], n, model_idx, bounds), types)
    # a record batch of the same rows: each column one (sliced) array
    recs = [Column(rng, c.type, n, VALIDITY[int(rng.integers(0, 3))], Layout("slice", offsets=[int(rng.integers(1, 18))], pad=3, seed=seed))
            for c in cols]
    batch = pc.RecordBatch([r.arrays[0] for r in recs], n)
    got = pc.Take(batch, dev_idx, bounds_check=bounds)
    _check_record(got, M.take_record([r.model for r in recs], n, model_idx, bounds), types)
    _same_snapshot(before, _snapshot(cols))


@pytest.mark.parametrize("it", IDX, ids=[NAME[t] for t in IDX])
def test_take_bounds_error_names_lowest_row_across_index_chunks(it):
    rng = np.random.default_rng(it)
    n = 100
    cols = [Column(rng, pc.INT32, n, "nulls"), Column(rng, pc.BOOL, n, "none")]
    table = pc.Table([c.chunked for c in cols], n)
    dt = np_of(it)
    bad = np.array(-5 if np.issubdtype(dt, np.signedinteger) else 101).astype(dt)
    v = rng.integers(0, n, 50).astype(dt)
    ok = np.ones(50, dtype=bool)
    v[7], ok[7] = bad, False          # a null slot is never checked
    v[31] = bad                       # the lowest offending row: in the second index chunk
    v[44] = np.array(n + 3).astype(dt) if np.iinfo(dt).max > n else bad
    parts = [(v[:20], ok[:20]), (v[20:20], ok[20:20]), (v[20:], ok[20:])]
    idx = pc.Chunked([pc.Array.from_numpy(pv, pok, it) for pv, pok in parts], it)
    want = M.take_table([c.model for c in cols], n, (parts, True))
    assert isinstance(want, Fail)
    for values in (table, pc.RecordBatch([pc.Array.from_numpy(*M._flat(c.model), c.type) for c in cols], n)):
        with pytest.raises(pc.ArrowError) as e:
            pc.Take(values, idx)
        assert e.value.sentinel == "ErrIndex" and e.value.msg == want.msg


def test_take_empty_and_zero_column_inputs():
    rng = np.random.default_rng(7)
    empty = Column(rng, pc.INT64, 0, "nulls", Layout("chunked", cuts=[0, 0, 0], offsets=[0, 3], seed=1))
    table = pc.Table([empty.chunked], 0)
    out = pc.Take(table, pc.Array.from_numpy(np.zeros(0, np.int32)))
    assert len(out) == 0 and [len(c) for c in out.columns()[0].chunks()] == [0]
    # indices into a zero-row table: every valid index is out of bounds, null ones are not checked
    with pytest.raises(pc.ArrowError) as e:
        pc.Take(table, pc.Array.from_numpy(np.array([0], np.int32)))
    assert e.value.msg == "0 out of bounds"
    out = pc.Take(table, pc.Array.from_numpy(np.array([3, 4], np.int32), np.array([False, False])))
    vals, valid, nulls = out.columns()[0].to_numpy()
    assert len(out) == 2 and not valid.any() and nulls == 2
    # zero columns: a record batch keeps the index count, a table has no rows, nothing is bounds-checked
    idx = pc.Array.from_numpy(np.array([5, 9], np.int64))
    rb = pc.Take(pc.RecordBatch([], 3), idx)
    assert rb.kind == pc.KIND_RECORD and len(rb) == 2 and rb.columns() == []
    tb = pc.Take(pc.Table([], 3), idx)
    assert tb.kind == pc.KIND_TABLE and len(tb) == 0
    # an empty chunked index gives columns without chunks
    tb = pc.Take(pc.Table([Column(rng, pc.UINT16, 10, "none").chunked], 10), pc.Chunked([], pc.INT32))
    assert len(tb) == 0 and tb.columns()[0].chunks() == []


def test_take_other_column_types_not_implemented():
    d = pc.DictionaryEncode(pc.Array.from_numpy(np.array([1, 2, 1], np.int32)))
    rb = pc.RecordBatch([pc.Array.from_numpy(np.arange(3, dtype=np.int8)), d], 3)
    with pytest.raises(pc.ArrowError) as e:
        pc.Take(rb, pc.Array.from_numpy(np.array([0], np.int32)))
    assert e.value.sentinel == "ErrNotImplemented" and "column 1" in e.value.msg
    with pytest.raises(pc.ArrowError) as e:
        pc.Take(pc.RecordBatch([pc.Array.from_numpy(np.arange(3, dtype=np.int8))], 3), pc.Array.from_numpy(np.array([0.5])))
    assert e.value.sentinel == "ErrInvalid"


# ---------------------------------------------------------------------------------------------------------------
# filter

@pytest.mark.parametrize("sel", [pc.DROP_NULLS, pc.EMIT_NULLS], ids=["drop", "emit"])
@pytest.mark.parametrize("seed", range(10))
def test_filter_table_and_record_batch(seed, sel):
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.integers(1, 4000))
    cols = _random_columns(rng, n, int(rng.integers(0, 6)))
    types = [c.type for c in cols]
    mask = Column(rng, pc.BOOL, n, VALIDITY[seed % 3])
    before = _snapshot(cols + [mask])
    mdev = mask.chunked if seed % 2 else mask.arrays[0] if len(mask.arrays) == 1 else mask.chunked
    mmodel = (mask.model, seed % 2 == 1)
    got = pc.FilterTable(pc.Table([c.chunked for c in cols], n), mdev, sel)
    _check_table(got, M.filter_table([c.model for c in cols], n, mmodel, sel), types)
    flat_mask = M._flat(mask.model)
    m = pc.Array.from_numpy(flat_mask[0], None if mask.model and all(ok is None for _, ok in mask.model) else flat_mask[1], pc.BOOL)
    recs = [pc.Array.from_numpy(*M._flat(c.model), c.type) for c in cols]
    got = pc.FilterRecordBatch(pc.RecordBatch(recs, n), m, sel)
    _check_record(got, M.filter_record_batch([c.model for c in cols], n, ([flat_mask], False), sel), types)
    _same_snapshot(before, _snapshot(cols + [mask]))


def test_filter_errors_and_zero_rows():
    rng = np.random.default_rng(3)
    col = Column(rng, pc.FLOAT64, 10, "nulls")
    table = pc.Table([col.chunked], 10)
    short = pc.Array.from_numpy(np.ones(9, bool))
    for fn, values in ((pc.FilterTable, table), (pc.FilterRecordBatch, pc.RecordBatch([pc.Array.from_numpy(np.zeros(10))], 10))):
        with pytest.raises(pc.ArrowError) as e:
            fn(values, short)
        assert e.value.sentinel == "ErrInvalid" and e.value.msg == "filter inputs must all be the same length"
    # a zero-row table comes back with its columns unchanged
    empty = Column(rng, pc.INT8, 0, "none", Layout("chunked", cuts=[0, 0, 0], offsets=[0, 0], seed=2))
    out = pc.FilterTable(pc.Table([empty.chunked], 0), pc.Array.from_numpy(np.zeros(0, bool)))
    assert len(out) == 0 and [len(c) for c in out.columns()[0].chunks()] == [0, 0]
    # CallFunction("filter") keeps refusing record batches and tables
    with pytest.raises(pc.ArrowError) as e:
        pc.CallFunction("filter", [table, pc.Array.from_numpy(np.ones(10, bool))], ("filter", 0))
    assert e.value.sentinel == "ErrNotImplemented"


# ---------------------------------------------------------------------------------------------------------------
# sort

def test_sort_against_pyarrow():
    rng = np.random.default_rng(11)
    n = 5000
    k0 = rng.integers(0, 20, n).astype(np.int32)
    k1 = rng.standard_normal(n)
    pay = rng.random(n) < 0.5
    v1 = rng.random(n) >= 0.1
    cuts = random_cuts(rng, n, 5)
    def chunked(v, ok, t):
        return pc.Chunked([pc.Array.from_numpy(v[a:b], None if ok is None else ok[a:b], t) for a, b in zip(cuts, cuts[1:])], t)
    table = pc.Table([chunked(k0, None, pc.INT32), chunked(k1, v1, pc.FLOAT64), chunked(pay, None, pc.BOOL)], n)
    keys = [(0, pc.DESCENDING, pc.NULLS_AT_END), (1, pc.ASCENDING, pc.NULLS_AT_START)]
    want_idx = pac.sort_indices(pa.table({"a": k0, "b": pa.array(k1, mask=~v1), "c": pay}),
                                sort_keys=[("a", "descending"), ("b", "ascending")], null_placement="at_start").to_numpy()
    # pyarrow places nulls per call, not per key: with one nullable key the orders agree
    got = pc.Sort(table, keys)
    assert got.kind == pc.KIND_TABLE and len(got) == n
    c0, c1, c2 = [c.to_numpy() for c in got.columns()]
    assert np.array_equal(c0[0], k0[want_idx])
    assert np.array_equal(c1[1], v1[want_idx]) and np.array_equal(c1[0][c1[1]], k1[want_idx][v1[want_idx]])
    assert np.array_equal(c2[0], pay[want_idx])
    rb = pc.Sort(pc.RecordBatch([pc.Array.from_numpy(k0), pc.Array.from_numpy(k1, v1), pc.Array.from_numpy(pay)], n), keys)
    assert rb.kind == pc.KIND_RECORD and np.array_equal(rb.columns()[2].to_numpy()[0], pay[want_idx])
    # arrays and chunked arrays by their first key, with np.lexsort as the model (stable, ascending)
    order = np.lexsort((np.arange(n), k0))
    assert np.array_equal(pc.Sort(pc.Array.from_numpy(k0), [(0, pc.ASCENDING, pc.NULLS_AT_END)]).to_numpy()[0], k0[order])
    out = pc.Sort(chunked(pay, None, pc.BOOL), [(0, pc.ASCENDING, pc.NULLS_AT_END)])
    assert out.kind == pc.KIND_CHUNKED and len(out.chunks()) == 1
    assert np.array_equal(out.to_numpy()[0], np.sort(pay, kind="stable"))
    assert "sort" not in pc.function_names()


# ---------------------------------------------------------------------------------------------------------------
# the C ABI

def _bits(v, off=0):
    return np.concatenate([np.packbits(np.concatenate([np.zeros(off, bool), v]), bitorder="little"), np.zeros(8, np.uint8)])


def test_host_flavour_matches_device_flavour():
    rng = np.random.default_rng(5)
    n, m = 700, 900
    a = rng.integers(-1000, 1000, n).astype(np.int16)
    b = rng.random(n) < 0.5
    bv = rng.random(n) >= 0.2
    idx = rng.integers(0, n, m).astype(np.uint32)
    iv = rng.random(m) >= 0.1
    want_a = M.gather((a, np.ones(n, bool)), idx, iv)
    want_b = M.gather((b, bv), idx, iv)
    # host: column a in two chunks (the second at element offset 5), b in one chunk at bit offset 3
    a2 = np.concatenate([np.zeros(5, np.int16), a[300:]])
    bb, bvb, ivb = _bits(b, 3), _bits(bv, 3), _bits(iv, 6)
    out_a, out_av = np.zeros(m, np.int16), np.zeros(m // 8 + 1, np.uint8)
    out_b, out_bv = np.zeros(m // 8 + 1, np.uint8), np.zeros(m // 8 + 1, np.uint8)
    cols = N.take_column_table([(N.INT16, [(a.ctypes.data, None, 0, 300), (a2.ctypes.data, None, 5, n - 300)], out_a.ctypes.data, out_av.ctypes.data),
                                (N.BOOL, [(bb.ctypes.data, bvb.ctypes.data, 3, n)], out_b.ctypes.data, out_bv.ctypes.data)])
    bad, bad_idx = C.c_int64(), C.c_int64()
    N.call("ag_take_columns", 2, cols, n, 32, 0, idx.ctypes.data, ivb.ctypes.data, 6, m, 1, C.byref(bad), C.byref(bad_idx))
    assert bad.value == N.NO_ERROR_POS
    unpack = lambda x: np.unpackbits(x, bitorder="little")[:m].astype(bool)   # noqa: E731
    assert np.array_equal(out_a, want_a[0]) and np.array_equal(unpack(out_av), want_a[1])
    assert np.array_equal(unpack(out_b), want_b[0]) and np.array_equal(unpack(out_bv), want_b[1])
    # device: same call on device buffers
    da, da2, db, dbv, di, div = Dev(a), Dev(a2), Dev(bb), Dev(bvb), Dev(idx), Dev(ivb)
    oa, oav, ob, obv = Dev(nbytes=2 * m), Dev(nbytes=m // 8 + 8), Dev(nbytes=m // 8 + 8), Dev(nbytes=m // 8 + 8)
    word = Dev(np.array([N.NO_ERROR_POS], np.int64))
    dcols = N.take_column_table([(N.INT16, [(da.ptr, None, 0, 300), (da2.ptr, None, 5, n - 300)], oa.ptr, oav.ptr),
                                 (N.BOOL, [(db.ptr, dbv.ptr, 3, n)], ob.ptr, obv.ptr)])
    N.call("ag_take_columns_dev", 2, dcols, n, 32, 0, di.ptr, div.ptr, 6, m, 1, word.ptr, None)
    N.call("ag_stream_sync", None)
    assert word.get()[0] == N.NO_ERROR_POS
    assert np.array_equal(oa.get(np.int16, m), want_a[0]) and np.array_equal(unpack(oav.get(np.uint8)), want_a[1])
    assert np.array_equal(unpack(ob.get(np.uint8)), want_b[0]) and np.array_equal(unpack(obv.get(np.uint8)), want_b[1])
    # an offending row: both flavours name the lowest one
    idx[[600, 200]] = [n, n + 1]
    iv[[600, 200]] = True
    ivb = _bits(iv, 6)
    st, msg = N.call_status("ag_take_columns", 2, cols, n, 32, 0, idx.ctypes.data, ivb.ctypes.data, 6, m, 1, C.byref(bad), C.byref(bad_idx))
    assert st == N.AG_ERR_INDEX and msg == f"{n + 1} out of bounds" and bad.value == 200 and bad_idx.value == n + 1
    di, div = Dev(idx), Dev(ivb)
    N.call("ag_take_columns_dev", 2, dcols, n, 32, 0, di.ptr, div.ptr, 6, m, 1, word.ptr, None)
    N.call("ag_stream_sync", None)
    assert word.get()[0] == 200


@pytest.mark.parametrize("flavour", ["ag_take_columns", "ag_take_columns_dev"])
def test_descriptor_errors(flavour):
    vals = np.arange(10, dtype=np.int64)
    out = np.zeros(10, np.int64)
    idx = np.arange(4, dtype=np.int32)
    def call(cols, nrows):
        tail = (C.byref(C.c_int64()), C.byref(C.c_int64())) if flavour == "ag_take_columns" else (None, None)
        return N.call_status(flavour, len(cols), N.take_column_table(cols), nrows, 32, 1, idx.ctypes.data, None, 0, 4, 0, *tail)
    st, msg = call([(N.INT64, [(vals.ctypes.data, None, 0, 4), (vals.ctypes.data, None, 4, 5)], out.ctypes.data, None)], 10)
    assert st == N.AG_ERR_INVALID and "column 0" in msg and "does not match" in msg
    st, msg = call([(N.INT64, [(vals.ctypes.data, None, -1, 10)], out.ctypes.data, None)], 10)
    assert st == N.AG_ERR_INVALID and "negative" in msg
    st, msg = call([(N.INT64, [(vals.ctypes.data, None, 0, 10)], out.ctypes.data, None), (N.FLOAT16, [(vals.ctypes.data, None, 0, 10)], out.ctypes.data, None)], 10)
    assert st == N.AG_ERR_NOT_IMPLEMENTED and "column 1" in msg
    st, msg = call([(N.INT64, [(vals.ctypes.data, None, 0, -2), (vals.ctypes.data, None, 0, 12)], out.ctypes.data, None)], 10)
    assert st == N.AG_ERR_INVALID


# ---------------------------------------------------------------------------------------------------------------
# past 2^31 output rows, with a boolean column whose bit positions pass 2^32

def test_past_2_31_output_rows_and_2_32_bits():
    torch = pytest.importorskip("torch")
    nrows = (1 << 32) + 4099
    n = (1 << 31) + 1000
    nbytes = (nrows + 7) // 8
    dev = torch.device("cuda:0")
    pat = torch.arange(nbytes + 8, dtype=torch.int32, device=dev).mul_(131).add_(7).bitwise_and_(0xFF).to(torch.uint8)
    idx = torch.arange(n, dtype=torch.int64, device=dev).mul_(3).add_(5).remainder_(nrows)
    out = torch.zeros((n + 31) // 32 * 4 + 64, dtype=torch.uint8, device=dev)
    # the column in two chunks: the second starts at bit 3 of its bitmap, past 2^32 rows of the first
    first = (1 << 32) + 17
    cols = N.take_column_table([(N.BOOL, [(pat.data_ptr(), None, 0, first), (pat.data_ptr(), None, first + 3, nrows - first)], out.data_ptr(), None)])
    # the second chunk reads bits [first + 3, first + 3 + (nrows - first)) of the same bitmap: row r >= first maps to bit r + 3
    word = torch.full((1,), N.NO_ERROR_POS, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    N.call("ag_take_columns_dev", 1, cols, nrows, 64, 1, idx.data_ptr(), None, 0, n, 1, word.data_ptr(), None)
    N.call("ag_stream_sync", None)
    assert int(word.item()) == N.NO_ERROR_POS
    for lo in (0, (1 << 31) - 4096, n - 4096):   # the last window crosses output row 2^31
        hi = lo + 4096
        i = np.arange(lo, hi, dtype=np.int64)
        r = (i * 3 + 5) % nrows
        bit = np.where(r >= first, r + 3, r)
        byte = bit >> 3
        want = ((((byte * 131 + 7) & 0xFF).astype(np.uint8) >> (bit & 7).astype(np.uint8)) & 1).astype(bool)
        got = np.unpackbits(out[lo // 8:hi // 8].cpu().numpy(), bitorder="little").astype(bool)
        assert np.array_equal(got, want), lo
    del pat, idx, out
    torch.cuda.empty_cache()
