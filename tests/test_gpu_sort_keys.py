"""sort_indices over several keys and chunked key columns on the device, against the model of tests/sort_keys_ref.py
(and the reference's literal vectors), through compute.SortIndices(keys=...) and both C flavours."""
import io
import json
import os

import numpy as np
import pytest

from arrow_go_b200 import _native as N
from arrow_go_b200 import compute as pc
from sort_keys_ref import (ASC, AT_END, AT_START, DESC, golden_columns, random_column, reference_sort_indices,
                           sort_keys_model)

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "sort_indices_keys.json")))
TYPES = ["bool", "uint8", "int8", "uint16", "int16", "uint32", "int32", "uint64", "int64", "float32", "float64"]
TYPE_ID = {"bool": N.BOOL, "uint8": N.UINT8, "int8": N.INT8, "uint16": N.UINT16, "int16": N.INT16, "uint32": N.UINT32,
           "int32": N.INT32, "uint64": N.UINT64, "int64": N.INT64, "float32": N.FLOAT32, "float64": N.FLOAT64}


def _chunked(col, ty):
    return pc.Chunked([pc.Array.from_numpy(v, ok, TYPE_ID[ty]) for v, ok in col], TYPE_ID[ty])


def _table(cols, types, n):
    return pc.Table([_chunked(c, t) for c, t in zip(cols, types)], n)


def _sort_table(cols, types, keys, n):
    out = pc.SortIndices(_table(cols, types, n), keys=keys)
    assert out.type == pc.UINT64 and len(out) == n
    vals, valid, nulls = out.to_numpy()
    assert nulls == 0
    return vals


def _bits(v):
    return np.concatenate([np.packbits(np.asarray(v, dtype=bool), bitorder="little"), np.zeros(8, np.uint8)])


def _host_flavour(cols, types, keys, n):
    """ag_sort_indices_keys with host pointers (chunks carry a leading pad element so offsets are exercised)."""
    keep, table = [], []
    for c, o, p in keys:
        chunks = []
        for v, ok in cols[c]:
            if types[c] == "bool":
                vb = _bits(np.concatenate([[False], v]))
            else:
                vb = np.concatenate([np.zeros(1, v.dtype), v])
            okb = None if ok is None else _bits(np.concatenate([[False], ok]))
            keep += [vb, okb]
            chunks.append((vb.ctypes.data, None if okb is None else okb.ctypes.data, 1, len(v)))
        table.append((TYPE_ID[types[c]], o, p, chunks))
    arr = N.sort_key_table(table)
    out = np.full(max(n, 1), 7, dtype=np.uint64)
    N.call("ag_sort_indices_keys", len(keys), arr, n, out.ctypes.data)
    return out[:n]


def _dev_flavour(cols, types, keys, n):
    import torch
    keep, table = [], []
    for c, o, p in keys:
        chunks = []
        for v, ok in cols[c]:
            host = _bits(v) if types[c] == "bool" else np.ascontiguousarray(v).view(np.uint8)
            dv = torch.from_numpy(host.copy()).cuda()
            dok = None if ok is None else torch.from_numpy(_bits(ok)).cuda()
            keep += [dv, dok]
            chunks.append((dv.data_ptr() if len(v) else None, None if dok is None else dok.data_ptr(), 0, len(v)))
        table.append((TYPE_ID[types[c]], o, p, chunks))
    arr = N.sort_key_table(table)
    out = torch.zeros(max(n, 1), dtype=torch.int64, device="cuda")
    N.call("ag_sort_indices_keys_dev", len(keys), arr, n, out.data_ptr(), None)
    torch.cuda.synchronize()
    return out[:n].cpu().numpy().view(np.uint64)


@pytest.mark.parametrize("case", GOLDEN["cases"], ids=[c["name"] for c in GOLDEN["cases"]])
def test_golden(case):
    cols = golden_columns(case)
    keys = [tuple(k) for k in case["keys"]]
    n = len(case["want"])
    types = case["types"]
    assert _sort_table(cols, types, keys, n).tolist() == case["want"]
    assert _host_flavour(cols, types, keys, n).tolist() == case["want"]
    assert _dev_flavour(cols, types, keys, n).tolist() == case["want"]
    if case["kind"] in ("array", "chunked"):   # one column: the first key, its column index ignored
        one = _chunked(cols[0], types[0])
        if case["kind"] == "array":
            one = pc.Array.from_numpy(cols[0][0][0], cols[0][0][1], TYPE_ID[types[0]])
        assert pc.SortIndices(one, keys=[(7,) + tuple(keys[0][1:])]).to_numpy()[0].tolist() == case["want"]
    if case["kind"] == "record" and n:
        rb = pc.RecordBatch([pc.Array.from_numpy(c[0][0], c[0][1], TYPE_ID[t]) for c, t in zip(cols, types)])
        got = pc.SortIndices(rb, keys=keys).to_numpy()[0]
        assert got.tolist() == case["want"]


def _random(rng, n, nkeys, layout, types=None, small=None):
    ncols = max(1, nkeys - int(rng.integers(0, 2)))
    types = types or [TYPES[int(rng.integers(0, len(TYPES)))] for _ in range(ncols)]
    cols = []
    for ty in types:
        if layout == "one" or (layout == "aligned" and cols):
            lens = [n] if layout == "one" else [len(ch[0]) for ch in cols[0]]
        else:
            cuts = sorted(rng.integers(0, n + 1, int(rng.integers(0, 6))).tolist())
            lens = np.diff([0] + cuts + [n]).tolist()
        cols.append(random_column(rng, ty, lens, null_p=float(rng.choice([0, 0.05, 0.3])), nan_p=0.1,
                                  small=bool(rng.integers(0, 2)) if small is None else small))
    keys = [(int(rng.integers(0, len(types))), int(rng.integers(0, 2)), int(rng.integers(0, 2))) for _ in range(nkeys)]
    return cols, types, keys


@pytest.mark.parametrize("seed", range(24))
def test_random_against_model(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.choice([1, 2, 100, 5000, 70000]))
    cols, types, keys = _random(rng, n, [1, 2, 3, 4, 8, 9, 12][seed % 7], ["one", "aligned", "misaligned"][seed % 3])
    want = sort_keys_model(cols, keys)
    assert np.array_equal(_sort_table(cols, types, keys, n), want)
    if seed % 4 == 0:
        assert np.array_equal(_dev_flavour(cols, types, keys, n), want)


@pytest.mark.parametrize("shape", ["b0", "b32", "b64", "b_wide", "twice"])
def test_packed_key_widths(shape):
    """B = 0 (every row ties), B <= 32 (one uint32 word), 33..64 (one uint64 word), > 64 (three full-range int64 keys
    plus class bits: gather passes), and one column used twice with opposite orders."""
    rng = np.random.default_rng(7)
    n = 50000
    if shape == "b0":
        cols = [[(np.full(n, 3, np.int32), None)], [(np.full(n, 1.5), None)]]
        types, keys = ["int32", "float64"], [(0, ASC, AT_END), (1, DESC, AT_START)]
    elif shape == "b32":
        cols = [random_column(rng, "int16", [n], small=True), random_column(rng, "uint8", [n // 2, n - n // 2], null_p=0)]
        types, keys = ["int16", "uint8"], [(0, ASC, AT_START), (1, DESC, AT_END)]
    elif shape == "b64":
        cols = [random_column(rng, "int32", [n], null_p=0), random_column(rng, "int16", [n])]
        types, keys = ["int32", "int16"], [(0, DESC, AT_END), (1, ASC, AT_START)]
    elif shape == "b_wide":
        cols = [random_column(rng, "int64", [n // 3, n - n // 3]) for _ in range(3)]
        types, keys = ["int64"] * 3, [(0, ASC, AT_END), (1, DESC, AT_START), (2, ASC, AT_START)]
        cols[0] = [(np.where(v > 0, np.iinfo(np.int64).max, np.iinfo(np.int64).min), ok) for v, ok in cols[0]]
    else:
        cols = [random_column(rng, "float32", [n], small=True)]
        types, keys = ["float32"], [(0, ASC, AT_END), (0, DESC, AT_START)]
    want = sort_keys_model(cols, keys)
    assert np.array_equal(_sort_table(cols, types, keys, n), want)
    assert np.array_equal(_dev_flavour(cols, types, keys, n), want)


def test_one_row_and_empty():
    one = [[(np.array([5], np.int32), None)], [(np.array([np.nan]), None)]]
    assert _sort_table(one, ["int32", "float64"], [(0, ASC, AT_END), (1, DESC, AT_START)], 1).tolist() == [0]
    empty = [[(np.zeros(0, np.uint8), None)], [(np.zeros(0, np.uint32), None)]]
    assert _sort_table(empty, ["uint8", "uint32"], [(0, ASC, AT_END)], 0).tolist() == []
    none = pc.Table([pc.Chunked([], pc.INT32)], 0)
    assert len(pc.SortIndices(none, keys=[(0, ASC, AT_END)])) == 0


def test_chunked_array_uses_first_key():
    rng = np.random.default_rng(3)
    col = random_column(rng, "float64", [100, 0, 57, 300], small=True)
    keys = [(0, DESC, AT_START)]
    got = pc.SortIndices(_chunked(col, "float64"), keys=[(5, DESC, AT_START), (1, ASC, AT_END)]).to_numpy()[0]
    assert np.array_equal(got, sort_keys_model([col], keys))


def test_thirty_million_rows():
    rng = np.random.default_rng(30)
    n = 30_000_000
    cols = [random_column(rng, "int64", [n // 2, n - n // 2], null_p=0.05, small=False),
            random_column(rng, "float32", [n // 3, n // 3, n - 2 * (n // 3)], null_p=0.05, nan_p=0.05),
            random_column(rng, "bool", [n], null_p=0)]
    cols[0] = [(v % 1000, ok) for v, ok in cols[0]]
    types, keys = ["int64", "float32", "bool"], [(0, ASC, AT_END), (1, DESC, AT_START), (2, ASC, AT_END)]
    assert np.array_equal(_dev_flavour(cols, types, keys, n), sort_keys_model(cols, keys))


def test_ipc_record_batch_matches_pyarrow():
    pa = pytest.importorskip("pyarrow")
    pac = pytest.importorskip("pyarrow.compute")
    from arrow_go_b200 import ipc
    rng = np.random.default_rng(11)
    n = 20000
    a = pa.array(rng.integers(0, 50, n).astype(np.int32), mask=rng.random(n) < 0.1)
    b = rng.standard_normal(n)
    b[rng.random(n) < 0.05] = np.nan
    b = pa.array(b, mask=rng.random(n) < 0.1)
    c = pa.array(rng.integers(0, 2, n).astype(bool))
    batch = pa.record_batch([a, b, c], names=["a", "b", "c"])
    sink = io.BytesIO()
    with pa.ipc.new_file(sink, batch.schema) as w:
        w.write_batch(batch)
    reader = ipc.FileReader(np.frombuffer(sink.getvalue(), dtype=np.uint8).copy())
    rows, cols = reader.record_batch(0)
    rb = pc.RecordBatch(cols, rows)
    for placement in (AT_END, AT_START):
        keys = [(2, DESC, placement), (0, ASC, placement), (1, DESC, placement)]
        want = pac.sort_indices(batch, sort_keys=[("c", "descending"), ("a", "ascending"), ("b", "descending")],
                                null_placement="at_start" if placement else "at_end").to_numpy()
        assert pc.SortIndices(rb, keys=keys).to_numpy()[0].tolist() == want.tolist()


def test_errors():
    i32 = pc.Array.from_numpy(np.arange(4, dtype=np.int32))
    rb = pc.RecordBatch([i32, pc.Array.from_numpy(np.arange(4, dtype=np.float64))])
    for keys, sentinel in (([], "ErrInvalid"), ([(2, ASC, AT_END)], "ErrInvalid"), ([(-1, ASC, AT_END)], "ErrInvalid"),
                           ([(0, 2, AT_END)], "ErrInvalid"), ([(0, ASC, 5)], "ErrInvalid")):
        with pytest.raises(pc.ArrowError) as e:
            pc.SortIndices(rb, keys=keys)
        assert e.value.sentinel == sentinel, keys
    with pytest.raises(pc.ArrowError) as e:
        pc.SortIndices(rb, keys=[(2, ASC, AT_END)])
    assert "sort key 0 has invalid column index 2" in e.value.msg
    with pytest.raises(pc.ArrowError) as e:   # record batches and tables need SortKeys
        pc.SortIndices(rb)
    assert e.value.sentinel == "ErrInvalid"
    with pytest.raises(pc.ArrowError) as e:
        pc.SortIndices(pc.RecordBatch([i32, pc.DictionaryEncode(i32)]), keys=[(1, ASC, AT_END)])
    assert e.value.sentinel == "ErrNotImplemented"
    with pytest.raises(pc.ArrowError) as e:   # building checks the row counts
        pc.RecordBatch([i32, pc.Array.from_numpy(np.arange(3, dtype=np.int32))], 4)
    assert e.value.sentinel == "ErrInvalid"
    # other functions refuse record batches and tables instead of crashing
    tb = pc.Table([i32])
    for fn, args in (("add", [rb, rb]), ("filter", [tb, pc.Array.from_pylist([True] * 4, pc.BOOL)]), ("unique", [rb])):
        with pytest.raises(pc.ArrowError) as e:
            pc.CallFunction(fn, args)
        assert e.value.sentinel == "ErrNotImplemented"
    # the datum accessors answer errors for record batches and tables
    for d in (rb, tb):
        assert d.kind in (pc.KIND_RECORD, pc.KIND_TABLE) and len(d) == 4 and d.chunks() == []
        for accessor in (d.indices, d.dictionary, d.run_ends, d.values, lambda: d.slice(0, 1)):
            with pytest.raises(pc.ArrowError):
                accessor()
    # the C ABI
    v = np.arange(4, dtype=np.int32)
    out = np.zeros(4, np.uint64)
    ok = (N.INT32, 0, 0, [(v.ctypes.data, None, 0, 4)])
    for table, n, status in (([], 4, N.AG_ERR_INVALID), ([(N.INT32, 3, 0, ok[3])], 4, N.AG_ERR_INVALID),
                             ([(N.INT32, 0, 2, ok[3])], 4, N.AG_ERR_INVALID), ([ok], 5, N.AG_ERR_INVALID),
                             ([ok, (N.INT32, 0, 0, [(v.ctypes.data, None, 0, 3)])], 4, N.AG_ERR_INVALID),
                             ([(N.FLOAT16, 0, 0, ok[3])], 4, N.AG_ERR_NOT_IMPLEMENTED),
                             ([(29, 0, 0, ok[3])], 4, N.AG_ERR_NOT_IMPLEMENTED)):
        st, _ = N.call_status("ag_sort_indices_keys", len(table), N.sort_key_table(table), n, out.ctypes.data)
        assert st == status, (table, n)
    huge = (N.INT32, 0, 0, [(v.ctypes.data, None, 0, 1 << 32)])   # refused before any device work
    st, _ = N.call_status("ag_sort_indices_keys_dev", 1, N.sort_key_table([huge]), 1 << 32, None, None)
    assert st == N.AG_ERR_NOT_IMPLEMENTED


def test_inputs_unchanged():
    rng = np.random.default_rng(5)
    cols, types, keys = _random(rng, 9000, 3, "misaligned", types=["float64", "int8", "bool"])
    snap = [[(v.copy(), None if ok is None else ok.copy()) for v, ok in c] for c in cols]
    dcols = [_chunked(c, t) for c, t in zip(cols, types)]
    before = [d.to_numpy() for d in dcols]
    pc.SortIndices(pc.Table(dcols, 9000), keys=keys)
    _host_flavour(cols, types, keys, 9000)
    for d, (bv, bok, bn) in zip(dcols, before):
        av, aok, an = d.to_numpy()
        assert np.array_equal(av, bv, equal_nan=av.dtype.kind == "f") and np.array_equal(aok, bok) and an == bn
    for c, s in zip(cols, snap):
        for (v, ok), (sv, sok) in zip(c, s):
            assert np.array_equal(v, sv, equal_nan=v.dtype.kind == "f") and (ok is None or np.array_equal(ok, sok))


def test_reference_restatement_agrees_on_device_inputs():
    """The restatement and the device agree on an input of every type outside the NaN quirk."""
    rng = np.random.default_rng(21)
    cols, types, keys = _random(rng, 1500, 4, "one", types=TYPES[:4])
    assert np.array_equal(_sort_table(cols, types, keys, 1500), reference_sort_indices(cols, keys))
