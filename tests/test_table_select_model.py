"""The NumPy model of take / filter on record batches and tables (tests/table_select_model.py) against pyarrow, on
values, validity and row counts, plus the output chunk lengths the reference's code gives (pyarrow chunks differently,
so those are pinned by hand).  Runs without a GPU."""
import numpy as np
import pyarrow as pa
import pytest

import table_select_model as M
from exec_model import Fail, random_cuts

TYPES = [np.bool_, np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32, np.uint64, np.int64, np.float32, np.float64]
IDX = [np.int8, np.uint8, np.int16, np.uint16, np.int32, np.uint32, np.int64, np.uint64]


def _values(rng, dt, n):
    if dt == np.bool_:
        return rng.random(n) < 0.5
    if np.issubdtype(dt, np.floating):
        return rng.standard_normal(n).astype(dt)
    return rng.integers(0, 256, n * np.dtype(dt).itemsize, dtype=np.uint8).view(dt)


def _column(rng, dt, n, nulls):
    vals = _values(rng, dt, n)
    valid = rng.random(n) >= 0.3 if nulls else None
    cuts = random_cuts(rng, n, int(rng.integers(1, 6)))
    return [(vals[a:b], None if valid is None else valid[a:b]) for a, b in zip(cuts, cuts[1:])]


def _pa_chunked(chunks, dt):
    arrs = [pa.array(v, mask=None if ok is None else ~ok, type=pa.from_numpy_dtype(dt)) for v, ok in chunks]
    return pa.chunked_array(arrs, type=pa.from_numpy_dtype(dt))


def _check_flat(model_chunks, pa_col):
    vals, valid = M._flat(model_chunks)
    want = pa_col.combine_chunks() if isinstance(pa_col, pa.ChunkedArray) else pa_col
    wvalid = np.asarray(want.is_valid())
    assert np.array_equal(valid, wvalid)
    wv = want.fill_null(pa.scalar(False if pa.types.is_boolean(want.type) else 0, want.type)).to_numpy(zero_copy_only=False)
    assert np.array_equal(vals[valid], np.asarray(wv)[wvalid].astype(vals.dtype))
    assert not vals[~valid].any()


def _indices(rng, n_rows, m, dt, nulls, chunks):
    hi = max(min(n_rows, int(np.iinfo(dt).max) + 1), 1)
    v = rng.integers(0, hi, m).astype(dt) if n_rows else np.zeros(m, dtype=dt)
    ok = rng.random(m) >= 0.2 if nulls or not n_rows else None
    if not n_rows:
        ok = np.zeros(m, dtype=bool)
    cuts = random_cuts(rng, m, chunks) if chunks else [0, m]
    return [(v[a:b], None if ok is None else ok[a:b]) for a, b in zip(cuts, cuts[1:])], bool(chunks)


@pytest.mark.parametrize("seed", range(12))
def test_take_matches_pyarrow(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(0, 300))
    types = [TYPES[int(rng.integers(0, len(TYPES)))] for _ in range(int(rng.integers(1, 5)))]
    cols = [_column(rng, dt, n, rng.random() < 0.5) for dt in types]
    idt = IDX[seed % len(IDX)]
    indices = _indices(rng, n, int(rng.integers(0, 200)), idt, seed % 2 == 0, int(rng.integers(1, 5)) if seed % 3 else 0)
    pa_idx = _pa_chunked(indices[0], idt) if indices[1] else pa.array(indices[0][0][0], mask=None if indices[0][0][1] is None else ~indices[0][0][1], type=pa.from_numpy_dtype(idt))
    table = pa.table({f"c{i}": _pa_chunked(c, dt) for i, (c, dt) in enumerate(zip(cols, types))})
    want = table.take(pa_idx)
    got, rows = M.take_table(cols, n, indices)
    assert rows == want.num_rows
    for c, chunks in enumerate(got):
        assert [len(v) for v, _ in chunks] == [len(v) for v, _ in indices[0]]   # one chunk per index chunk
        _check_flat(chunks, want.column(c))
    rec, rows = M.take_record(cols, n, indices)
    assert rows == want.num_rows
    for c, col in enumerate(rec):
        _check_flat([col], want.column(c))


def test_take_bounds_error_matches_pyarrow():
    cols = [[(np.arange(5, dtype=np.int64), None)]]
    for bad in ([1, 7, 2, 9], [0, -3, 8]):
        idx = np.array(bad, dtype=np.int32)
        with pytest.raises(IndexError):
            pa.table({"a": np.arange(5)}).take(pa.array(idx))
        r = M.take_table(cols, 5, ([(idx[:1], None), (idx[1:], None)], True))
        assert isinstance(r, Fail) and r.sentinel == "ErrIndex" and r.msg == f"{bad[1]} out of bounds"
    # a null index slot is never bounds-checked
    _, rows = M.take_record(cols, 5, ([(np.array([9, 1], np.int32), np.array([False, True]))], False))
    assert rows == 2
    # without columns nothing is taken or checked; a table without columns has no rows
    assert M.take_record([], 0, ([(np.array([4], np.int32), None)], False)) == ([], 1)
    assert M.take_table([], 0, ([(np.array([4], np.int32), None)], False)) == ([], 0)


@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("sel", [M.DROP_NULLS, M.EMIT_NULLS])
def test_filter_matches_pyarrow(seed, sel):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(0, 300))
    types = [TYPES[int(rng.integers(0, len(TYPES)))] for _ in range(int(rng.integers(1, 4)))]
    cols = [_column(rng, dt, n, rng.random() < 0.5) for dt in types]
    mask = _column(rng, np.bool_, n, seed % 2 == 0)
    behaviour = "drop" if sel == M.DROP_NULLS else "emit_null"
    table = pa.table({f"c{i}": _pa_chunked(c, dt) for i, (c, dt) in enumerate(zip(cols, types))})
    pmask = _pa_chunked(mask, np.bool_)
    want = table.filter(pmask, null_selection_behavior=behaviour)
    got = M.filter_table(cols, n, (mask, True), sel)
    if n == 0:
        assert got is None
    else:
        out, rows = got
        assert rows == want.num_rows
        for c, chunks in enumerate(out):
            assert all(len(v) for v, _ in chunks)   # a span that selects nothing gives no chunk
            _check_flat(chunks, want.column(c))
    flat_cols = [[M._flat(c)] for c in cols]
    rb = pa.RecordBatch.from_arrays([table.column(i).combine_chunks() for i in range(len(cols))], names=table.column_names)
    want_rb = rb.filter(pmask.combine_chunks(), null_selection_behavior=behaviour)
    out, rows = M.filter_record_batch(flat_cols, n, ([M._flat(mask)], False), sel)
    assert rows == want_rb.num_rows
    for c, col in enumerate(out):
        _check_flat([col], want_rb.column(c))


def test_filter_table_chunks_follow_every_boundary():
    a = [(np.arange(3), None), (np.arange(3, 5), None)]
    b = [(np.arange(5).astype(np.float64), None)]
    mask = [(np.array([True, True]), None), (np.array([True, False, True]), None)]
    out, rows = M.filter_table([a, b], 5, (mask, True), M.DROP_NULLS)
    assert rows == 4
    # spans [0,2) [2,3) [3,5): the mask cut at 2 and the column cut at 3
    assert [[len(v) for v, _ in c] for c in out] == [[2, 1, 1], [2, 1, 1]]
    assert M.spans([[3, 0, 2], [5], [2, 3]]) == [(0, 2), (2, 1), (3, 2)]
    # a span that selects nothing gives no chunk
    mask = [(np.array([False, False]), None), (np.array([True, False, True]), None)]
    out, rows = M.filter_table([a], 5, (mask, True), M.DROP_NULLS)
    assert [len(v) for v, _ in out[0]] == [1, 1] and rows == 2
    assert M.filter_table([a], 5, ([(np.ones(4, bool), None)], False), M.DROP_NULLS).msg == "filter inputs must all be the same length"
