"""CPU checks of dictionary_encode's NumPy restatement (tests/dictionary_encode_ref.py) against the reference's literal
cases (tests/golden/dictionary_encode.json) and pyarrow, plus the C Data Interface view of a pyarrow dictionary array."""
import ctypes as C
import json
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from dictionary_encode_ref import ENCODE, MASK, dictionary_encode_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dictionary_encode.json")


def _chunks_from_lists(ty, lists):
    out = []
    for lst in lists:
        valid = np.array([x is not None for x in lst], bool)
        vals = np.array([0 if x is None else x for x in lst], dtype=ty)
        out.append((vals, None if valid.all() else valid))
    return out


def _decoded(res):
    chunks, dictionary, dvalid = res
    idx = [[None if (v is not None and not v[i]) else int(ix[i]) for i in range(len(ix))] for ix, v, _ in chunks]
    d = [None if (dvalid is not None and not dvalid[i]) else x.item() for i, x in enumerate(dictionary)]
    return idx, d


@pytest.mark.parametrize("case", json.load(open(GOLDEN))["cases"], ids=lambda c: c["name"])
def test_oracle_matches_golden(case):
    res = dictionary_encode_ref(_chunks_from_lists(case["type"], case["chunks"]), case["null_encoding"])
    assert _decoded(res) == (case["indices"], case["dictionary"])


@pytest.mark.parametrize("ne", [MASK, ENCODE])
@pytest.mark.parametrize("ty", ["int8", "uint16", "int32", "uint64", "int64"])
@pytest.mark.parametrize("card", [5, 3000])
def test_oracle_matches_pyarrow(ty, card, ne):
    rng = np.random.default_rng(card * 7 + ne)
    info = np.iinfo(ty)
    pool = rng.integers(max(info.min, -(1 << 40)), min(info.max, 1 << 40), card, endpoint=True).astype(ty)
    chunks = []
    for n in (0, 1000, 37, 0, 2500):
        vals = pool[rng.integers(0, card, n)]
        valid = rng.random(n) >= 0.25
        chunks.append((vals, valid))
    got = _decoded(dictionary_encode_ref(chunks, ne))
    col = pa.chunked_array([pa.array(v, mask=~m) for v, m in chunks], type=pa.from_numpy_dtype(np.dtype(ty)))
    out = pc.dictionary_encode(col, null_encoding="encode" if ne else "mask")
    want_idx = [c.indices.to_pylist() for c in out.chunks]
    want_dict = out.chunk(0).dictionary.to_pylist()
    got_idx = [c for c, (v, _) in zip(got[0], chunks) if len(v)]   # pyarrow drops the empty chunks, like the reference
    assert (got_idx, got[1]) == (want_idx, want_dict)


def test_oracle_floats_compare_raw_bytes():
    nan2 = np.array([0x7ff8000000000001], np.uint64).view(np.float64)[0]
    vals = np.array([0.0, -0.0, np.nan, nan2, 0.0, np.nan, -0.0], np.float64)
    (ci, _, _), = dictionary_encode_ref([(vals, None)])[0]
    assert ci.tolist() == [0, 1, 2, 3, 0, 2, 1]


def test_describe_reads_pyarrow_dictionary_array():
    """ag_dictionary_device_array_describe on pyarrow's exported dictionary<int32, int64> (CPU device)."""
    from arrow_go_b200 import _native as N
    arr = pa.DictionaryArray.from_arrays(pa.array([2, 0, None, 1, 2], pa.int32()), pa.array([10, 20, 30], pa.int64()))
    da, sc = N.ArrowDeviceArray(), N.ArrowSchema()
    arr._export_to_c_device(C.addressof(da), C.addressof(sc))
    try:
        idx, dic = N.ArrayView(), N.ArrayView()
        N.call("ag_dictionary_device_array_describe", C.byref(da), C.byref(sc), C.byref(idx), C.byref(dic))
        assert (idx.type, idx.length, idx.null_count, idx.device_type) == (N.INT32, 5, 1, N.DEVICE_CPU)
        assert (dic.type, dic.length, dic.null_count) == (N.INT64, 3, 0)
        assert C.cast(dic.values, C.POINTER(C.c_int64))[0:3] == [10, 20, 30]
        assert C.cast(idx.values, C.POINTER(C.c_int32))[0:5][:2] == [2, 0]
    finally:
        da.array.release(C.byref(da.array))
        sc.release(C.byref(sc))
