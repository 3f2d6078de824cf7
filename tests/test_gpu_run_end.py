"""run_end_encode / run_end_decode on the device: the C ABI (host and device flavours), the host mirror / Python API and
the C Device Data Interface, compared with the NumPy restatement in tests/run_end_ref.py."""
import ctypes as C

import numpy as np
import pytest

import run_end_ref as ref
from arrow_go_b200 import _native as N
from arrow_go_b200 import compute as pc
from helpers import ALL_TYPES, NP_OF, Dev, checksum64, pack_bits

pytestmark = pytest.mark.gpu

VALUE_TYPES = [N.BOOL] + ALL_TYPES
RUN_END_TYPES = [N.INT16, N.INT32, N.INT64]
RT_NAME = {N.INT16: "int16", N.INT32: "int32", N.INT64: "int64"}
RT_NP = {N.INT16: np.int16, N.INT32: np.int32, N.INT64: np.int64}
RT_MAX = {N.INT16: (1 << 15) - 1, N.INT32: (1 << 31) - 1, N.INT64: (1 << 63) - 1}
GUARD = 64


def np_of(type_id):
    return np.bool_ if type_id == N.BOOL else NP_OF[type_id]


def tile_rows(type_id):
    """Rows of one encode tile: 2048 groups of one 16-byte load (a 32-bit word for BOOL)."""
    return 2048 * (32 if type_id == N.BOOL else 16 // np.dtype(NP_OF[type_id]).itemsize)


def runs_column(type_id, lengths):
    """A column whose k-th run has lengths[k] rows; neighbouring runs differ."""
    k = np.repeat(np.arange(len(lengths)), lengths)
    if type_id == N.BOOL:
        return (k % 2).astype(bool)
    return ((k % 5) + 1).astype(NP_OF[type_id])


def value_buffer(type_id, vals, offset):
    """Host buffer holding `vals` from element (bit) `offset`."""
    if type_id == N.BOOL:
        return pack_bits(vals, offset, fill=0x5A, pad_bytes=8)
    return np.concatenate([np.full(offset, 7, vals.dtype), vals, np.zeros(4, vals.dtype)])


def abi_encode(type_id, rt, vals, valid, offset=0, capacity=None):
    """The host flavour: (runs, null runs, run_ends, run values, run validity or None, guard bytes of every output)."""
    n = len(vals)
    buf = value_buffer(type_id, vals, offset)
    vb = pack_bits(valid, offset, pad_bytes=8) if valid is not None else None
    counts = np.zeros(2, np.int64)
    N.call("ag_run_end_count", type_id, buf.ctypes.data, None if vb is None else vb.ctypes.data, offset, n, counts.ctypes.data)
    cap = int(counts[0]) if capacity is None else capacity
    ends = np.full(cap + GUARD, -3, RT_NP[rt])
    if type_id == N.BOOL:
        out = np.full((cap + 7) // 8 + GUARD, 0xEE, np.uint8)
    else:
        out = np.full(cap + GUARD, 99, NP_OF[type_id])
    ov = np.full((cap + 7) // 8 + GUARD, 0xEE, np.uint8)
    c2 = np.zeros(2, np.int64)
    N.call("ag_run_end_encode", type_id, rt, buf.ctypes.data, None if vb is None else vb.ctypes.data, offset, n,
           ends.ctypes.data, out.ctypes.data, ov.ctypes.data if vb is not None else None, cap, c2.ctypes.data)
    assert (c2 == counts).all()
    runs = int(counts[0])
    w = min(runs, cap)
    if type_id == N.BOOL:
        rvals = np.unpackbits(out, bitorder="little")[:w].astype(bool)
        guard_out = out[(w + 7) // 8:]
    else:
        rvals = out[:w]
        guard_out = out[w:]
    rvalid = np.unpackbits(ov, bitorder="little")[:w].astype(bool) if vb is not None else None
    assert (ends[w:] == -3).all() and (guard_out == (0xEE if type_id == N.BOOL else 99)).all()
    if vb is not None:
        assert (ov[(w + 7) // 8:] == 0xEE).all()
    return runs, int(counts[1]), ends[:w].astype(np.int64), rvals, rvalid


def check_encode(type_id, rt, vals, valid, offset=0, capacity=None):
    runs, nulls, ends, rvals, rvalid = abi_encode(type_id, rt, vals, valid, offset, capacity)
    w_ends, w_vals, w_valid, w_nulls = ref.encode(vals, valid, RT_NAME[rt])
    assert runs == len(w_ends) and nulls == w_nulls
    k = len(ends)
    assert (ends == w_ends[:k]).all()
    assert rvals.tobytes() == np.ascontiguousarray(w_vals[:k]).tobytes()   # bits of each run's first row
    assert (rvalid is None) == (w_valid is None)
    if w_valid is not None:
        assert (rvalid == w_valid[:k]).all()
    return runs


@pytest.mark.parametrize("type_id", VALUE_TYPES)
@pytest.mark.parametrize("rt", RUN_END_TYPES)
def test_encode_run_lengths(type_id, rt):
    rng = np.random.default_rng(type_id * 7 + rt)
    t = tile_rows(type_id)
    for L in [1, 2, 31, 32, 33, t - 1, t, t + 1]:
        n = min(3 * t + 17, RT_MAX[rt])
        lengths = np.full(n // L + 1, L)
        vals = runs_column(type_id, lengths)[:n]
        if len(vals) > RT_MAX[rt]:
            continue
        check_encode(type_id, rt, vals, None)
        valid = rng.random(len(vals)) >= 0.1
        check_encode(type_id, rt, vals, valid)


@pytest.mark.parametrize("type_id", VALUE_TYPES)
def test_encode_long_runs_one_run_all_null(type_id):
    rt = N.INT64
    t = tile_rows(type_id)
    n = 5 * t + 3
    rng = np.random.default_rng(type_id)
    lengths = rng.integers(t // 2, 3 * t, 8)            # runs that span many tiles
    vals = runs_column(type_id, lengths)[:n]
    check_encode(type_id, rt, vals, None)
    one = np.zeros(n, np_of(type_id))
    assert check_encode(type_id, rt, one, None) == 1    # one run
    runs, nulls, ends, _, rvalid = abi_encode(type_id, rt, one, np.zeros(n, bool))
    assert (runs, nulls, ends.tolist(), rvalid.tolist()) == (1, 1, [n], [False])   # all null
    # no bitmap and a bitmap with zero nulls give the same runs; only the second has a validity child
    a = abi_encode(type_id, rt, vals, None)
    b = abi_encode(type_id, rt, vals, np.ones(len(vals), bool))
    assert a[0] == b[0] and (a[2] == b[2]).all() and a[3].tobytes() == b[3].tobytes() and a[4] is None and b[4].all()


@pytest.mark.parametrize("type_id", VALUE_TYPES)
@pytest.mark.parametrize("offset", range(9))
def test_encode_bitmap_offsets(type_id, offset):
    rng = np.random.default_rng(offset * 13 + type_id)
    lengths = rng.integers(1, 6, 3000)
    vals = runs_column(type_id, lengths)
    valid = np.repeat(rng.random(len(lengths)) >= 0.3, lengths)
    valid[rng.integers(0, len(valid), 50)] ^= True
    check_encode(type_id, N.INT32, vals, valid, offset)
    check_encode(type_id, N.INT16, vals[:5000], valid[:5000], offset)


@pytest.mark.parametrize("type_id", [N.FLOAT32, N.FLOAT64])
def test_encode_nan_and_signed_zero(type_id):
    dt = NP_OF[type_id]
    base = np.array([np.nan, np.nan, 0.0, -0.0, -0.0, 0.0, 1.0, 1.0], dtype=dt)
    payload = base.copy()
    payload.view(f"u{payload.itemsize}")[1] += 1            # a second NaN payload
    vals = np.tile(payload, 600)
    runs = check_encode(type_id, N.INT32, vals, None)
    assert runs == 600 * 4   # each period: NaN | NaN | 0.0 -0.0 -0.0 0.0 | 1.0 1.0


@pytest.mark.parametrize("type_id", VALUE_TYPES)
def test_encode_null_rows_with_different_payloads(type_id):
    rng = np.random.default_rng(type_id + 100)
    vals = rng.integers(0, 2, 5000).astype(np_of(type_id))
    valid = np.zeros(5000, bool)
    valid[::7] = True
    check_encode(type_id, N.INT32, vals, valid)   # null rows with different payloads are different runs


@pytest.mark.parametrize("type_id", VALUE_TYPES)
@pytest.mark.parametrize("rt", RUN_END_TYPES)
def test_encode_capacity_smaller_than_runs(type_id, rt):
    rng = np.random.default_rng(type_id * 3 + rt)
    lengths = rng.integers(1, 4, 9000)
    vals = runs_column(type_id, lengths)[:30000]
    valid = rng.random(len(vals)) >= 0.2
    runs = len(ref.encode(vals, valid, "int64")[0])
    for cap in (0, 1, 31, runs // 2, runs - 1):
        assert check_encode(type_id, rt, vals, valid, 3, cap) == runs


# ---------------------------------------------------------------- decode -------------------
def abi_decode(type_id, rt, ends, rvals, rvalid, offset, length, values_offset=0):
    n_runs = len(ends)
    e = np.ascontiguousarray(ends, dtype=RT_NP[rt])
    vbuf = value_buffer(type_id, np.asarray(rvals, dtype=np_of(type_id)), values_offset)
    vb = pack_bits(rvalid, values_offset, pad_bytes=8) if rvalid is not None else None
    out = np.zeros(max(length, 1) + GUARD, np.uint8 if type_id == N.BOOL else NP_OF[type_id])
    ov = np.zeros((length + 7) // 8 + GUARD, np.uint8)
    nulls = C.c_int64(-1)
    st, msg = N.call_status("ag_run_end_decode", type_id, rt, e.ctypes.data, n_runs, vbuf.ctypes.data,
                            None if vb is None else vb.ctypes.data, values_offset, offset, length, out.ctypes.data,
                            ov.ctypes.data if vb is not None else None, C.byref(nulls))
    if st != N.AG_OK:
        return st, msg
    vals = np.unpackbits(out.view(np.uint8), bitorder="little")[:length].astype(bool) if type_id == N.BOOL else out[:length]
    valid = np.unpackbits(ov, bitorder="little")[:length].astype(bool) if vb is not None else None
    return vals, valid, nulls.value


@pytest.mark.parametrize("type_id", VALUE_TYPES)
@pytest.mark.parametrize("rt", RUN_END_TYPES)
def test_decode_slices(type_id, rt):
    rng = np.random.default_rng(type_id * 11 + rt)
    lengths = rng.integers(1, 40, 700)
    vals = runs_column(type_id, lengths)
    valid = np.repeat(rng.random(len(lengths)) >= 0.25, lengths)
    n = min(len(vals), RT_MAX[rt])
    ends, rvals, rvalid, _ = ref.encode(vals[:n], valid[:n], RT_NAME[rt])
    cases = [(0, n), (1, n - 2), (int(ends[3]) - 1, 5000), (5, 1), (n - 1, 1), (17, 4096), (17, 4097), (0, 8191)]
    for off, ln in cases:
        ln = min(ln, n - off)
        got_v, got_m, nulls = abi_decode(type_id, rt, ends, rvals, rvalid, off, ln, values_offset=100 if off % 2 else 0)
        want_v, want_m = ref.decode(ends, rvals, rvalid, off, ln)
        assert got_v.tobytes() == np.ascontiguousarray(want_v).tobytes()
        assert (got_m == want_m).all() and nulls == int((~want_m).sum())
    # no validity child: no output bitmap
    got_v, got_m, nulls = abi_decode(type_id, rt, ends, rvals, None, 3, n - 5)
    assert got_m is None and nulls == 0 and got_v.tobytes() == np.ascontiguousarray(ref.decode(ends, rvals, None, 3, n - 5)[0]).tobytes()


def test_decode_with_child_offset():
    # the reference's TestDecodeWithChildOffset: the values child starts 100 elements into its buffer
    ends = np.array([2, 5, 6], np.int32)
    rvals = np.array([10, 20, 30], np.int64)
    got_v, got_m, _ = abi_decode(N.INT64, N.INT32, ends, rvals, np.array([True, False, True]), 0, 6, values_offset=100)
    assert got_v.tolist()[:2] + got_v.tolist()[5:] == [10, 10, 30] and got_m.tolist() == [True, True, False, False, False, True]


MALFORMED = [
    ("repeated run end", [2, 4, 4, 9], 0, 9),
    ("decreasing run end", [2, 6, 5, 9], 0, 9),
    ("last run end short", [2, 4, 6, 8], 1, 8),
    ("no runs", [], 0, 3),
]


@pytest.mark.parametrize("type_id", [N.BOOL, N.UINT8, N.INT32, N.FLOAT64])
@pytest.mark.parametrize("case", MALFORMED, ids=lambda c: c[0])
def test_decode_malformed_run_ends(type_id, case):
    _, ends, off, ln = case
    rvals = np.ones(max(len(ends), 1), np_of(type_id))
    st, msg = abi_decode(type_id, N.INT32, np.array(ends, np.int64), rvals[:len(ends)] if ends else rvals, None, off, ln)
    assert st == N.AG_ERR_INVALID and "malformed run ends" in msg
    # the device flavour lowers the error word and writes nothing outside [0, length)
    d_ends = Dev(np.array(ends + [0], np.int32))
    d_vals = Dev(np.ones(16, np.uint8 if type_id == N.BOOL else NP_OF[type_id]))
    nbytes = ((ln + 31) // 32) * 4 if type_id == N.BOOL else ln * np.dtype(NP_OF[type_id]).itemsize
    out = Dev(np.full(nbytes + GUARD, 0xAB, np.uint8))
    words = Dev(np.zeros(2, np.int64))
    N.call("ag_error_word_reset_dev", words.ptr + 8, None)
    N.call("ag_run_end_decode_dev", type_id, N.INT32, d_ends.ptr, len(ends), d_vals.ptr, None, 0, off, ln, out.ptr, None,
           words.ptr, words.ptr + 8, None)
    N.call("ag_stream_sync", None)
    assert words.get()[1] != N.NO_ERROR_POS
    assert (out.get()[nbytes:] == 0xAB).all()


def test_decode_malformed_large_segment_stays_in_bounds():
    # run ends that jump back inside a long slice: many tiles, every block checks its share
    ends = np.arange(1, 50001, dtype=np.int64)
    ends[30000] = 5
    st, _ = abi_decode(N.INT64, N.INT64, ends, np.arange(50000, dtype=np.int64), None, 0, 50000)
    assert st == N.AG_ERR_INVALID


def test_abi_errors():
    x = np.arange(10, dtype=np.int32)
    counts = np.zeros(2, np.int64)
    st, msg = N.call_status("ag_run_end_encode", N.INT32, N.UINT8, x.ctypes.data, None, 0, 10, None, None, None, 0, counts.ctypes.data)
    assert st == N.AG_ERR_INVALID and "bad run end type" in msg
    st, msg = N.call_status("ag_run_end_encode_dev", N.INT32, N.INT16, 64, None, 0, 32768, None, None, None, 0, 64, None)
    assert st == N.AG_ERR_INVALID and "can hold: 32767" in msg
    st, _ = N.call_status("ag_run_end_count", N.FLOAT16, x.ctypes.data, None, 0, 10, counts.ctypes.data)
    assert st == N.AG_ERR_NOT_IMPLEMENTED
    # n == 0 is an empty result, even for int16
    N.call("ag_run_end_encode", N.INT32, N.INT16, None, None, 0, 0, None, None, None, 0, counts.ctypes.data)
    assert counts.tolist() == [0, 0]


# ---------------------------------------------------------------- host API -----------------
def host_array(type_id, vals, valid, offset=0):
    pad = np.zeros(offset, np_of(type_id))
    v = None if valid is None else np.concatenate([np.ones(offset, bool), valid])
    return pc.Array.from_numpy(np.concatenate([pad, vals]), v, type_id, offset)


@pytest.mark.parametrize("type_id", VALUE_TYPES)
@pytest.mark.parametrize("rt", RUN_END_TYPES)
def test_host_api_encode_decode(type_id, rt):
    rng = np.random.default_rng(type_id * 5 + rt)
    lengths = rng.integers(1, 50, 500)
    vals = runs_column(type_id, lengths)[:20000]
    valid = np.repeat(rng.random(len(lengths)) >= 0.2, lengths)[:len(vals)]
    for m, off in ((None, 0), (valid, 3)):
        arr = host_array(type_id, vals, m, off)
        enc = pc.RunEndEncode(arr, rt)
        assert enc.type == pc.RUN_END_ENCODED and enc.value_type == type_id and enc.run_end_type == rt and len(enc) == len(vals)
        w_ends, w_vals, w_valid, w_nulls = ref.encode(vals, m, RT_NAME[rt])
        ends, _, _ = enc.run_ends().to_numpy()
        rv, rm, rn = enc.values().to_numpy()
        assert (ends.astype(np.int64) == w_ends).all() and rv.tobytes() == np.ascontiguousarray(w_vals).tobytes()
        assert enc.values().has_validity == (m is not None) and rn == w_nulls
        if m is not None:
            assert (rm == w_valid).all()
        dec = pc.RunEndDecode(enc)
        dv, dm, dn = dec.to_numpy()
        assert dv.tobytes() == vals.tobytes() and dec.has_validity == (m is not None)
        if m is not None:
            assert (dm == m).all() and dn == int((~m).sum())
        # a slice of the encoded array changes only its offset / length
        s = enc.slice(7, 1000)
        sv, sm, _ = pc.RunEndDecode(s).to_numpy()
        assert sv.tobytes() == vals[7:1007].tobytes()
        assert s.to_pylist() == [(x.item() if ok else None) for x, ok in zip(vals[7:1007], (m if m is not None else np.ones(len(vals), bool))[7:1007])]


def test_host_api_errors():
    x = pc.Array.from_numpy(np.arange(32768, dtype=np.int32) // 3)
    with pytest.raises(pc.ArrowError, match="cannot be called without options") as e:
        pc.CallFunction("run_end_encode", [x])
    assert e.value.code == N.AG_ERR_INVALID
    with pytest.raises(pc.ArrowError, match="bad run end type") as e:
        pc.RunEndEncode(x, pc.UINT8)
    assert e.value.code == N.AG_ERR_INVALID
    with pytest.raises(pc.ArrowError, match="can hold: 32767") as e:
        pc.RunEndEncode(x, pc.INT16)
    assert e.value.code == N.AG_ERR_INVALID
    assert len(pc.RunEndEncode(x.slice(0, 32767), pc.INT16)) == 32767
    enc = pc.RunEndEncode(x, pc.INT32)
    with pytest.raises(pc.ArrowError) as e:
        pc.Add(enc, enc)
    assert e.value.code == N.AG_ERR_NOT_IMPLEMENTED
    with pytest.raises(pc.ArrowError) as e:
        pc.RunEndDecode(x)
    assert e.value.code == N.AG_ERR_NOT_IMPLEMENTED


def test_host_api_chunked():
    chunks = [pc.Array.from_numpy(np.array([1, 1, 2], np.int64)), pc.Array.from_numpy(np.zeros(0, np.int64)),
              pc.Array.from_numpy(np.array([2, 2, 3, 3], np.int64))]
    col = pc.Chunked(chunks, pc.INT64)
    enc = pc.RunEndEncode(col, pc.INT32)
    assert enc.kind == pc.KIND_CHUNKED and enc.type == pc.RUN_END_ENCODED and enc.value_type == pc.INT64
    got = [(c.run_ends().to_numpy()[0].tolist(), c.values().to_numpy()[0].tolist()) for c in enc.chunks()]
    assert got == [([2, 3], [1, 2]), ([2, 4], [2, 3])]   # runs never cross a chunk boundary; the empty chunk is dropped
    assert enc.to_pylist() == [1, 1, 2, 2, 2, 3, 3]
    dec = pc.RunEndDecode(enc)
    assert dec.kind == pc.KIND_CHUNKED and dec.type == pc.INT64 and dec.to_pylist() == [1, 1, 2, 2, 2, 3, 3]
    empty = pc.RunEndEncode(pc.Chunked([], pc.BOOL), pc.INT16)
    assert empty.kind == pc.KIND_CHUNKED and len(empty) == 0 and empty.value_type == pc.BOOL
    assert len(pc.RunEndDecode(empty)) == 0
    all_empty = pc.RunEndEncode(pc.Chunked([pc.Array.from_numpy(np.zeros(0, np.float32))] * 3, pc.FLOAT32), pc.INT64)
    assert len(all_empty.chunks()) == 1 and len(all_empty) == 0


def test_100m_rows_round_trip_checksum():
    n = 100_000_000
    rng = np.random.default_rng(7)
    lengths = rng.integers(1, 32, n // 16 + 1000)
    k = np.repeat(np.arange(len(lengths), dtype=np.uint64), lengths)[:n]
    vals = ((k * np.uint64(0x9E3779B97F4A7C15)) % np.uint64(1000)).astype(np.int64)
    want = checksum64(vals.view(np.uint64))
    d_in = Dev(vals)
    counts = Dev(np.zeros(2, np.int64))
    N.call("ag_run_end_count_dev", N.INT64, d_in.ptr, None, 0, n, counts.ptr, None)
    N.call("ag_stream_sync", None)
    runs = int(counts.get()[0])
    assert runs == int(np.count_nonzero(np.diff(vals))) + 1
    d_ends, d_vals = Dev(nbytes=runs * 4), Dev(nbytes=runs * 8)
    N.call("ag_run_end_encode_dev", N.INT64, N.INT32, d_in.ptr, None, 0, n, d_ends.ptr, d_vals.ptr, None, runs, counts.ptr, None)
    d_out = Dev(nbytes=n * 8)
    words = Dev(np.zeros(2, np.int64))
    N.call("ag_error_word_reset_dev", words.ptr + 8, None)
    N.call("ag_run_end_decode_dev", N.INT64, N.INT32, d_ends.ptr, runs, d_vals.ptr, None, 0, 0, n, d_out.ptr, None,
           words.ptr, words.ptr + 8, None)
    res = Dev(np.zeros(1, np.uint64))
    N.call("ag_checksum64_dev", d_out.ptr, n, res.ptr, None)
    N.call("ag_stream_sync", None)
    assert words.get()[1] == N.NO_ERROR_POS
    assert int(res.get()[0]) == want


# ---------------------------------------------------------------- C Device Data Interface ----
def test_export_import_round_trip():
    import pyarrow as pa
    src = pc.Array.from_numpy(np.array([7, 7, 0, 3, 3, 3, 9], np.int64), np.array([1, 1, 0, 1, 1, 1, 1], bool))
    enc = pc.RunEndEncode(src, pc.INT32).slice(1, 5)
    da, sc = pc.export_device(enc)
    assert sc.format == b"+r" and sc.n_children == 2 and da.array.n_children == 2 and da.array.n_buffers == 0
    assert da.device_type == N.DEVICE_CUDA and (da.array.offset, da.array.length, da.array.null_count) == (1, 5, 0)
    p, r, v = N.ArrayView(), N.ArrayView(), N.ArrayView()
    N.call("ag_run_end_encoded_device_array_describe", C.byref(da), C.byref(sc), C.byref(p), C.byref(r), C.byref(v))
    assert (p.type, p.offset, p.length) == (N.TYPE_RUN_END_ENCODED, 1, 5)
    assert (r.type, r.length, v.type, v.length, v.null_count) == (N.INT32, 4, N.INT64, 4, 1)
    assert N.call_status("ag_device_array_describe", C.byref(da), C.byref(sc), C.byref(p))[0] != N.AG_OK
    back = pc.import_device(da, sc)
    assert not da.array.release
    assert back.type == pc.RUN_END_ENCODED and back.value_type == pc.INT64 and back.run_end_type == pc.INT32
    assert back.to_pylist() == [7, None, 3, 3, 3]
    assert pc.RunEndDecode(back).to_pylist() == [7, None, 3, 3, 3]
    t = pa.DataType._import_from_c(C.addressof(sc))   # pyarrow reads the exported schema and releases it
    assert t == pa.run_end_encoded(pa.int32(), pa.int64())
    del back, enc


def test_describe_pyarrow_export():
    import pyarrow as pa
    import pyarrow.compute as pac
    arr = pac.run_end_encode(pa.array([1.5, 1.5, None, 2.5, 2.5, 2.5], pa.float64()), run_end_type=pa.int16()).slice(1, 4)
    da, sc = N.ArrowDeviceArray(), N.ArrowSchema()
    arr._export_to_c_device(C.addressof(da), C.addressof(sc))
    try:
        p, r, v = N.ArrayView(), N.ArrayView(), N.ArrayView()
        N.call("ag_run_end_encoded_device_array_describe", C.byref(da), C.byref(sc), C.byref(p), C.byref(r), C.byref(v))
        assert (p.type, p.offset, p.length, p.device_type) == (N.TYPE_RUN_END_ENCODED, 1, 4, N.DEVICE_CPU)
        assert (r.type, r.length, r.null_count) == (N.INT16, 3, 0)
        assert (v.type, v.length, v.null_count) == (N.FLOAT64, 3, 1)
        assert np.ctypeslib.as_array(C.cast(r.values, C.POINTER(C.c_int16)), (3,)).tolist() == [2, 3, 6]
        # a CPU array is described but not imported
        assert N.call_status("ag_import_run_end_encoded_device_array", C.byref(da), C.byref(sc), None,
                             C.byref(p), C.byref(r), C.byref(v))[0] == N.AG_ERR_INVALID
    finally:
        da.array.release(C.byref(da.array))
        sc.release(C.byref(sc))


def test_export_release_chain_and_moved_child():
    enc = pc.RunEndEncode(pc.Array.from_numpy(np.array([True, True, False])), pc.INT64)
    da, sc = pc.export_device(enc)
    kids = C.cast(da.array.children, C.POINTER(C.POINTER(N.ArrowArray)))
    child = kids[1].contents
    moved = N.ArrowArray()
    C.memmove(C.byref(moved), C.byref(child), C.sizeof(N.ArrowArray))
    child.release = type(child.release)()   # NULL: moved out by the consumer
    da.array.release(C.byref(da.array))
    assert not da.array.release
    assert moved.length == 2 and moved.release
    moved.release(C.byref(moved))
    assert not moved.release
    sc.release(C.byref(sc))
    assert not sc.release


# ---------------------------------------------------------------- past 2^31 rows ------------
def test_large_rows_int64_run_ends():
    """A uint8 column of 2^31+2^20+7 rows in runs of mixed length: encode with int64 run ends and decode, compared by
    checksums with the host's; int32 run ends refuse the column and leave their outputs untouched."""
    n = (1 << 31) + (1 << 20) + 7
    rng = np.random.default_rng(31)
    lengths = rng.integers(1, 32, n // 16 + (1 << 20))
    lengths[rng.integers(0, len(lengths), 64)] = rng.integers(1 << 16, 1 << 22, 64)   # a few long runs
    ends = np.cumsum(lengths)
    R = int(np.searchsorted(ends, n)) + 1
    ends = ends[:R]
    ends[-1] = n
    base = (np.cumsum(rng.integers(1, 256, R)) % 256).astype(np.uint8)   # neighbouring runs differ
    vals = np.repeat(base, np.diff(ends, prepend=0))
    assert len(vals) == n
    d_in = Dev(vals)
    n8 = n // 8
    want_in = checksum64(vals[:n8 * 8].view(np.uint64))
    tail = vals[n8 * 8:].copy()
    del vals
    counts = Dev(np.zeros(2, np.int64))
    # int32 run ends: refused, nothing written
    sentinel = Dev(np.full(16, 0x7E, np.uint8))
    st, msg = N.call_status("ag_run_end_encode_dev", N.UINT8, N.INT32, d_in.ptr, None, 0, n, sentinel.ptr, sentinel.ptr, None, 4,
                            counts.ptr, None)
    assert st == N.AG_ERR_INVALID and "can hold: 2147483647" in msg
    N.call("ag_stream_sync", None)
    assert (sentinel.get() == 0x7E).all()
    N.call("ag_run_end_count_dev", N.UINT8, d_in.ptr, None, 0, n, counts.ptr, None)
    N.call("ag_stream_sync", None)
    assert counts.get().tolist() == [R, 0]
    d_ends, d_vals = Dev(nbytes=R * 8), Dev(nbytes=R)
    N.call("ag_run_end_encode_dev", N.UINT8, N.INT64, d_in.ptr, None, 0, n, d_ends.ptr, d_vals.ptr, None, R, counts.ptr, None)
    res = Dev(np.zeros(1, np.uint64))
    N.call("ag_checksum64_dev", d_ends.ptr, R, res.ptr, None)
    N.call("ag_stream_sync", None)
    assert int(res.get()[0]) == checksum64(ends.astype(np.uint64))
    assert d_vals.get(np.uint8, R).tobytes() == base.tobytes()
    del d_in
    d_out = Dev(nbytes=n + 8)
    words = Dev(np.zeros(2, np.int64))
    N.call("ag_error_word_reset_dev", words.ptr + 8, None)
    N.call("ag_run_end_decode_dev", N.UINT8, N.INT64, d_ends.ptr, R, d_vals.ptr, None, 0, 0, n, d_out.ptr, None,
           words.ptr, words.ptr + 8, None)
    N.call("ag_checksum64_dev", d_out.ptr, n8, res.ptr, None)
    N.call("ag_stream_sync", None)
    assert words.get()[1] == N.NO_ERROR_POS
    assert int(res.get()[0]) == want_in
    assert d_out.buf.to_numpy(np.uint8, n - n8 * 8, n8 * 8).tobytes() == tail.tobytes()
    # a slice past 2^31 that cuts runs at both ends
    off, ln = (1 << 31) + 12345, 1 << 19
    N.call("ag_run_end_decode_dev", N.UINT8, N.INT64, d_ends.ptr, R, d_vals.ptr, None, 0, off, ln, d_out.ptr, None,
           words.ptr, words.ptr + 8, None)
    N.call("ag_stream_sync", None)
    p = np.searchsorted(ends, np.arange(off, off + ln), side="right")
    assert d_out.get(np.uint8, ln).tobytes() == base[p].tobytes()
