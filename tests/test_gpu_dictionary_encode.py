"""dictionary_encode on the device: the C ABI (host flavour) and the host mirror / Python API, compared with the NumPy
restatement in tests/dictionary_encode_ref.py."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from arrow_go_b200 import _native as N
from arrow_go_b200 import compute as pc
from dictionary_encode_ref import ENCODE, MASK, dictionary_encode_ref
from helpers import ALL_TYPES, NP_OF, pack_bits

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dictionary_encode.json")
W = {np.dtype(t).itemsize for t in NP_OF.values()}


def abi_encode(chunks, ne, offsets=None):
    """chunks: [(values, valid or None)] -> the ABI's ([(indices, valid or None, nulls)], dictionary, dict valid or None)."""
    dtype = chunks[0][0].dtype
    offsets = offsets or [0] * len(chunks)
    keep, desc = [], []
    total = sum(len(v) for v, _ in chunks)
    for (v, m), off in zip(chunks, offsets):
        n = len(v)
        buf = np.concatenate([np.zeros(off, dtype), v])
        vb = pack_bits(np.concatenate([np.zeros(off, bool), m]), 0) if m is not None else None
        idx = np.full(max(n, 1), -7, np.int32)
        iv = np.zeros(((n + 31) // 32) * 4 + 4, np.uint8)
        keep += [buf, vb, idx, iv]
        desc.append((buf.ctypes.data, None if vb is None else vb.ctypes.data, off, n, idx.ctypes.data, iv.ctypes.data))
    table = N.dict_chunk_table(desc)
    dictionary = np.zeros(max(total, 1), dtype)
    dvalid = np.zeros(total // 8 + 2, np.uint8)
    counts = np.zeros(len(chunks) + 2, np.int64)
    N.call("ag_dictionary_encode", dtype.itemsize * 8, table, len(chunks), ne, dictionary.ctypes.data, dvalid.ctypes.data, counts.ctypes.data)
    k, dnulls = int(counts[0]), int(counts[1])
    out = []
    for c, (v, m) in enumerate(chunks):
        n, idx, iv = len(v), keep[4 * c + 2], keep[4 * c + 3]
        valid = np.unpackbits(iv, bitorder="little")[:n].astype(bool) if (ne == MASK and m is not None) else None
        if valid is not None and valid.all():
            valid = None
        out.append((idx[:n], valid, int(counts[2 + c])))
    dv = np.unpackbits(dvalid, bitorder="little")[:k].astype(bool) if dnulls else None
    return out, dictionary[:k], dv


def check(chunks, ne, offsets=None):
    got_chunks, got_dict, got_dv = abi_encode(chunks, ne, offsets)
    want_chunks, want_dict, want_dv = dictionary_encode_ref(chunks, ne)
    assert got_dict.tobytes() == want_dict.tobytes()
    assert (got_dv is None) == (want_dv is None) and (got_dv is None or (got_dv == want_dv).all())
    for (gi, gv, gn), (wi, wv, wn) in zip(got_chunks, want_chunks):
        assert gn == wn
        assert (gv is None) == (wv is None)
        if wv is not None:
            assert (gv == wv).all()
            assert (gi[wv] == wi[wv]).all() and (gi[~wv] == 0).all()
        else:
            assert (gi == wi).all()


def column(rng, type_id, n, card, null_frac):
    dt = np.dtype(NP_OF[type_id])
    pool = rng.integers(0, 1 << (8 * dt.itemsize - 1), card, dtype=np.uint64).astype(f"u{dt.itemsize}").view(dt)
    vals = pool[rng.integers(0, card, n)]
    valid = (rng.random(n) >= null_frac) if null_frac else None
    return vals, valid


@pytest.mark.parametrize("type_id", ALL_TYPES)
@pytest.mark.parametrize("n", [1, 31, 33, 1000, 70001])
@pytest.mark.parametrize("card", [5, 3000])
def test_types_sizes_cardinality(type_id, n, card):
    rng = np.random.default_rng(n * 31 + card + type_id)
    for ne in (MASK, ENCODE):
        check([column(rng, type_id, n, card, 0.0)], ne)


@pytest.mark.parametrize("type_id", [N.INT8, N.UINT16, N.INT32, N.INT64, N.FLOAT64])
@pytest.mark.parametrize("ne", [MASK, ENCODE])
def test_nulls_and_offsets(type_id, ne):
    rng = np.random.default_rng(type_id + 100 * ne)
    for off in range(9):
        check([column(rng, type_id, 1000 + off, 40, 0.25)], ne, [off])


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_float_bits(dt):
    bits = np.dtype(f"u{np.dtype(dt).itemsize}")
    qnan = np.array([0x7fc00001 if bits.itemsize == 4 else 0x7ff8000000000001], bits).view(dt)[0]
    vals = np.array([0.0, -0.0, np.nan, qnan, -np.nan, 1.5, 0.0, np.nan, -0.0] * 300, dt)
    check([(vals, None)], MASK)


def test_all_ones_64bit_key():
    vals = np.array([5, -1, 5, 7, -1, 0, -1], np.int64)
    valid = np.array([1, 1, 1, 0, 1, 1, 1], bool)
    for ne in (MASK, ENCODE):
        check([(vals, valid)], ne)
        check([(vals.view(np.uint64), None)], ne)
        check([(vals.view(np.float64), valid)], ne)


@pytest.mark.parametrize("ne", [MASK, ENCODE])
def test_chunked_with_empty_chunks(ne):
    rng = np.random.default_rng(9)
    parts = [column(rng, N.INT64, n, 50, 0.2) for n in (0, 33, 0, 1000, 1, 0, 4096)]
    check(parts, ne, [0, 3, 0, 5, 1, 0, 7])


@pytest.mark.parametrize("ne", [MASK, ENCODE])
def test_overflow_path(ne):
    rng = np.random.default_rng(11)
    N.call("ag_unique_set_policy", 1000, 1024)
    try:
        check([(rng.permutation(20000).astype(np.int64), rng.random(20000) > 0.1), column(rng, N.INT64, 5000, 800, 0.1)], ne)
        check([column(rng, N.INT32, 3000, 5, 0.0)], ne)   # stays in the small table
    finally:
        N.call("ag_unique_set_policy", 0, 0)


def test_golden_cases_through_python():
    for case in json.load(open(GOLDEN))["cases"]:
        ty = {"int64": pc.INT64, "int32": pc.INT32, "uint8": pc.UINT8}[case["type"]]
        arrays = [pc.Array.from_pylist(c, ty) for c in case["chunks"]]
        values = arrays[0] if len(arrays) == 1 else pc.Chunked(arrays, ty)
        out = pc.DictionaryEncode(values, case["null_encoding"])
        assert out.type == pc.DICTIONARY and out.value_type == ty
        assert out.dictionary().to_pylist() == case["dictionary"], case["name"]
        if len(arrays) == 1:
            assert out.indices().to_pylist() == case["indices"][0], case["name"]
        else:
            assert [c.indices().to_pylist() for c in out.chunks()] == case["indices"], case["name"]
        decoded = [x for c in case["chunks"] for x in c]
        assert out.to_pylist() == decoded


def test_python_chunked_shapes():
    a = pc.Array.from_pylist([1, 2, 1], pc.INT64)
    e = pc.Array.from_pylist([], pc.INT64)
    b = pc.Array.from_pylist([2, 3, None], pc.INT64)
    out = pc.DictionaryEncode(pc.Chunked([e, a, e, b], pc.INT64))
    assert out.kind == pc.KIND_CHUNKED and len(out.chunks()) == 2
    assert [c.indices().to_pylist() for c in out.chunks()] == [[0, 1, 0], [1, 2, None]]
    assert out.chunks()[0].has_validity is False and out.chunks()[1].has_validity is True
    zero = pc.DictionaryEncode(pc.Chunked([], pc.FLOAT32))
    assert zero.type == pc.DICTIONARY and zero.value_type == pc.FLOAT32 and len(zero.chunks()) == 0
    assert zero.dictionary().to_pylist() == []
    # a slice encodes at offset 0; slicing a dictionary array keeps its dictionary
    s = pc.DictionaryEncode(pc.Array.from_pylist([9, 8, 9, 7, 8], pc.INT16).slice(1, 4))
    assert s.indices().to_pylist() == [0, 1, 2, 0] and s.offset == 0
    assert s.slice(2, 2).to_pylist() == [7, 8]


def test_identity_errors_and_options():
    enc = pc.DictionaryEncode(pc.Array.from_pylist([4, 4, 5], pc.INT32))
    again = pc.DictionaryEncode(enc)
    assert again.type == pc.DICTIONARY and again.to_pylist() == [4, 4, 5]
    chunked = pc.DictionaryEncode(pc.Chunked([pc.Array.from_pylist([1], pc.INT32)], pc.INT32))
    assert pc.DictionaryEncode(chunked).to_pylist() == [1]
    with pytest.raises(pc.ArrowError) as e:
        pc.DictionaryEncode(pc.Array.from_pylist([1], pc.INT32), 99)
    assert e.value.sentinel == "ErrInvalid"
    with pytest.raises(pc.ArrowError) as e:
        pc.DictionaryEncode(pc.Array.from_pylist([True], pc.BOOL))
    assert e.value.sentinel == "ErrNotImplemented"
    with pytest.raises(pc.ArrowError) as e:
        pc.Add(enc, enc)
    assert e.value.sentinel == "ErrNotImplemented"
    with pytest.raises(pc.ArrowError):
        pc.Unique(enc)
    st, _ = N.call_status("ag_dictionary_encode", 64, N.dict_chunk_table([]), 0, 2, None, None, np.zeros(2, np.int64).ctypes.data)
    assert st == N.AG_ERR_INVALID
    st, _ = N.call_status("ag_dictionary_encode", 1, N.dict_chunk_table([]), 0, 0, None, None, np.zeros(2, np.int64).ctypes.data)
    assert st == N.AG_ERR_NOT_IMPLEMENTED
    huge = N.dict_chunk_table([(1, None, 0, 1 << 30, 1, None)] * 2)
    st, _ = N.call_status("ag_dictionary_encode_dev", 64, huge, 2, 0, 1, None, 8, None)
    assert st == N.AG_ERR_NOT_IMPLEMENTED


def test_100m_rows_100_values():
    n = 100_000_000
    rng = np.random.default_rng(5)
    pool = rng.integers(-(1 << 62), 1 << 62, 100)
    vals = pool[rng.integers(0, 100, n)]
    out = pc.DictionaryEncode(pc.Array.from_numpy(vals))
    d, _, _ = out.dictionary().to_numpy()
    idx, valid, nulls = out.indices().to_numpy()
    assert len(d) == 100 and nulls == 0 and valid.all()
    _, first = np.unique(vals, return_index=True)
    assert (d == vals[np.sort(first)]).all()
    assert (d[idx] == vals).all()


@pytest.mark.parametrize("ne", [MASK, ENCODE])
def test_export_import_round_trip(ne):
    import pyarrow as pa
    src = pc.Array.from_pylist([7, None, 3, 7, 3, None, 9], pc.INT64)
    enc = pc.DictionaryEncode(src, ne)
    da, sc = pc.export_device(enc)
    assert sc.format == b"i" and sc.dictionary and da.array.dictionary
    assert da.device_type == N.DEVICE_CUDA
    idx, dic = N.ArrayView(), N.ArrayView()
    N.call("ag_dictionary_device_array_describe", C.byref(da), C.byref(sc), C.byref(idx), C.byref(dic))
    assert (idx.type, idx.length, dic.type, dic.length) == (N.INT32, 7, N.INT64, 3 if ne == MASK else 4)
    # the exported plain export still refuses a dictionary array
    assert N.call_status("ag_device_array_describe", C.byref(da), C.byref(sc), C.byref(idx))[0] == N.AG_ERR_NOT_IMPLEMENTED
    back = pc.import_device(da, sc)   # takes the array; the schema stays ours
    assert not da.array.release
    assert back.type == pc.DICTIONARY and back.value_type == pc.INT64
    assert back.to_pylist() == [7, None, 3, 7, 3, None, 9]
    assert back.dictionary().to_pylist() == enc.dictionary().to_pylist()
    t = pa.DataType._import_from_c(C.addressof(sc))   # pyarrow reads the exported schema and releases it
    assert t == pa.dictionary(pa.int32(), pa.int64())
    del back, enc   # the last reference runs the parent's release, which releases the dictionary child


def test_export_release_chain_and_moved_child():
    enc = pc.DictionaryEncode(pc.Array.from_pylist([1.5, 2.5, 1.5], pc.FLOAT64))
    da, sc = pc.export_device(enc)
    child = C.cast(da.array.dictionary, C.POINTER(N.ArrowArray)).contents
    # a consumer may move the child out before releasing the parent
    moved = N.ArrowArray()
    C.memmove(C.byref(moved), C.byref(child), C.sizeof(N.ArrowArray))
    child.release = type(child.release)()   # NULL: moved
    da.array.release(C.byref(da.array))
    assert moved.length == 2 and moved.release
    moved.release(C.byref(moved))
    assert not moved.release
    sc.release(C.byref(sc))
    assert not sc.release


def test_chunked_of_dictionary_chunks_knows_value_type():
    a = pc.DictionaryEncode(pc.Array.from_pylist([1, 2], pc.UINT16))
    c = pc.Chunked([a, a.slice(1, 1)], pc.DICTIONARY)
    assert c.value_type == pc.UINT16 and c.to_pylist() == [1, 2, 2]
    with pytest.raises(pc.ArrowError):
        pc.Chunked([], pc.DICTIONARY)
    with pytest.raises(pc.ArrowError):
        pc.Chunked([a, pc.DictionaryEncode(pc.Array.from_pylist([1], pc.INT8))], pc.DICTIONARY)
