"""Take and sort_indices error messages byte for byte (chunk-list checks; out of bounds with bad_pos / bad_index), and a
boolean chunk at bit offset 3 through the host and device flavours of ag_sort_indices_keys and ag_take_columns."""
import ctypes as C

import numpy as np
import pytest

from arrow_go_b200 import _native as N
from arrow_go_b200 import compute as pc
from helpers import Dev, pack_bits, unpack_bits

pytestmark = pytest.mark.gpu

ROWS = 10
VALS = np.arange(ROWS, dtype=np.int64)
P = VALS.ctypes.data
# the chunks of the second column / key, an nchunks override, the message after "<column or key> 1: "
CHUNK_ERRORS = {
    "bad_list": ([(P, None, 0, ROWS)], -1, "bad chunk list"),
    "negative_offset": ([(P, None, -1, ROWS)], None, "negative chunk offset or length"),
    "negative_length": ([(P, None, 0, -2), (P, None, 0, ROWS + 2)], None, "negative chunk offset or length"),
    "null_values": ([(P, None, 0, 4), (None, None, 0, ROWS - 4)], None, "NULL chunk values"),
    "row_count": ([(P, None, 0, 4), (P, None, 4, 5)], None, "chunk row count 9 does not match {} 10"),
}


@pytest.mark.parametrize("flavour", ["ag_sort_indices_keys", "ag_sort_indices_keys_dev", "ag_take_columns", "ag_take_columns_dev"])
@pytest.mark.parametrize("case", list(CHUNK_ERRORS))
def test_chunk_list_messages(flavour, case):
    chunks, nchunks, tail = CHUNK_ERRORS[case]
    out, idx = np.zeros(ROWS, np.int64), np.arange(4, dtype=np.int32)
    host = not flavour.endswith("_dev")
    if flavour.startswith("ag_sort"):
        table = N.sort_key_table([(N.INT64, 0, 0, [(P, None, 0, ROWS)]), (N.INT64, 0, 0, chunks)])
        args = (out.ctypes.data,) if host else (None, None)
        want = "sort_indices: sort key 1: " + tail.format("column length")
    else:
        table = N.take_column_table([(N.INT64, [(P, None, 0, ROWS)], out.ctypes.data, None), (N.INT64, chunks, out.ctypes.data, None)])
        args = (32, 1, idx.ctypes.data, None, 0, 4, 0) + ((C.byref(C.c_int64()), C.byref(C.c_int64())) if host else (None, None))
        want = "take_columns: column 1: " + tail.format("row count")
    if nchunks is not None:
        table[1].nchunks = nchunks
    assert N.call_status(flavour, 2, table, ROWS, *args) == (N.AG_ERR_INVALID, want)


# a negative signed index, an index equal to the row count, a uint64 index past 2^63 (printed unsigned); rows 3 and 6
OOB = {"signed_negative": (pc.INT32, np.int32, -5), "equal_to_rows": (pc.UINT16, np.uint16, ROWS),
       "uint64_past_2_63": (pc.UINT64, np.uint64, (1 << 63) + 5)}


@pytest.mark.parametrize("path", ["ag_take_primitive", "ag_take_columns", "mirror_array", "mirror_table"])
@pytest.mark.parametrize("case", list(OOB))
def test_out_of_bounds_message(path, case):
    t, dt, bad = OOB[case]
    idx = (np.arange(8) % ROWS).astype(dt)
    idx[[3, 6]] = np.array(bad).astype(dt)
    msg, signed, width = f"{bad} out of bounds", int(np.issubdtype(dt, np.signedinteger)), idx.itemsize * 8
    pos, val, out = C.c_int64(), C.c_int64(), np.zeros(idx.size, np.int64)
    if path == "ag_take_primitive":
        got = N.call_status(path, 64, P, None, 0, ROWS, width, signed, idx.ctypes.data, None, 0, idx.size, 1, out.ctypes.data, None, None,
                            C.byref(pos), C.byref(val))
    elif path == "ag_take_columns":
        cols = N.take_column_table([(N.INT64, [(P, None, 0, 4), (P, None, 4, ROWS - 4)], out.ctypes.data, None)])
        got = N.call_status(path, 1, cols, ROWS, width, signed, idx.ctypes.data, None, 0, idx.size, 1, C.byref(pos), C.byref(val))
    else:
        values = pc.Array.from_numpy(VALS, None, pc.INT64) if path == "mirror_array" else pc.Table(
            [pc.Chunked([pc.Array.from_numpy(VALS[:4], None, pc.INT64), pc.Array.from_numpy(VALS[4:], None, pc.INT64)], pc.INT64)], ROWS)
        with pytest.raises(pc.ArrowError) as e:
            pc.Take(values, pc.Array.from_numpy(idx, None, t))
        assert e.value.sentinel == "ErrIndex" and e.value.msg == msg
        return
    assert got == (N.AG_ERR_INDEX, msg)
    assert pos.value == 3 and val.value == int(np.array(bad).astype(dt).astype(np.int64))


def test_bool_chunk_at_bit_offset_3_host_and_device_flavours():
    rng = np.random.default_rng(3)
    n, m = 300, 400
    b, bv = rng.random(n) < 0.5, rng.random(n) >= 0.2
    hb, hbv = pack_bits(b, 3), pack_bits(bv, 3)
    db, dbv = Dev(hb), Dev(hbv)
    want = np.argsort(np.where(bv, b.astype(np.int64), 2), kind="stable").astype(np.uint64)   # [false | true | null]
    got, dout = np.zeros(n, np.uint64), Dev(nbytes=8 * n)
    N.call("ag_sort_indices_keys", 1, N.sort_key_table([(N.BOOL, 0, 0, [(hb.ctypes.data, hbv.ctypes.data, 3, n)])]), n, got.ctypes.data)
    N.call("ag_sort_indices_keys_dev", 1, N.sort_key_table([(N.BOOL, 0, 0, [(db.ptr, dbv.ptr, 3, n)])]), n, dout.ptr, None)
    N.call("ag_stream_sync", None)
    assert np.array_equal(got, want) and np.array_equal(dout.get(np.uint64, n), want)
    idx = rng.integers(0, n, m).astype(np.int64)
    out, outv = np.zeros(m // 8 + 8, np.uint8), np.zeros(m // 8 + 8, np.uint8)
    cols = N.take_column_table([(N.BOOL, [(hb.ctypes.data, hbv.ctypes.data, 3, n)], out.ctypes.data, outv.ctypes.data)])
    N.call("ag_take_columns", 1, cols, n, 64, 1, idx.ctypes.data, None, 0, m, 1, C.byref(C.c_int64()), C.byref(C.c_int64()))
    assert np.array_equal(unpack_bits(out, 0, m), b[idx] & bv[idx]) and np.array_equal(unpack_bits(outv, 0, m), bv[idx])
    di, dv, dvv, word = Dev(idx), Dev(nbytes=m // 8 + 8), Dev(nbytes=m // 8 + 8), Dev(np.array([N.NO_ERROR_POS], np.int64))
    dcols = N.take_column_table([(N.BOOL, [(db.ptr, dbv.ptr, 3, n)], dv.ptr, dvv.ptr)])
    N.call("ag_take_columns_dev", 1, dcols, n, 64, 1, di.ptr, None, 0, m, 1, word.ptr, None)
    N.call("ag_stream_sync", None)
    assert word.get()[0] == N.NO_ERROR_POS
    assert np.array_equal(unpack_bits(dv.get(np.uint8), 0, m), unpack_bits(out, 0, m))
    assert np.array_equal(unpack_bits(dvv.get(np.uint8), 0, m), unpack_bits(outv, 0, m))
