#!/usr/bin/env python
"""Moderate run_end_encode / run_end_decode calls that reach every kernel of run_end.cu (count, encode over several
tiles with and without validity, with a capacity below the run count, the decode bounds and expansion kernels, BOOL and
every value width, and a malformed decode), for compute-sanitizer memcheck and racecheck:

    compute-sanitizer --tool memcheck --error-exitcode 9 python scripts/lab/san_run_end.py 20011
    compute-sanitizer --tool racecheck --error-exitcode 9 python scripts/lab/san_run_end.py 9001

The encode's output validity and BOOL value words are written by several warps of a block (shared-memory atomics) and
by neighbouring blocks (global atomicOr on a tile's edge words).  Results are compared with the NumPy restatement, so a
sanitizer-clean run is also a correct one."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import run_end_ref as ref  # noqa: E402
from arrow_go_b200 import _native as N  # noqa: E402

TYPE_OF = {np.dtype(np.bool_): N.BOOL, np.dtype(np.uint8): N.UINT8, np.dtype(np.int16): N.INT16, np.dtype(np.int32): N.INT32,
           np.dtype(np.float32): N.FLOAT32, np.dtype(np.int64): N.INT64, np.dtype(np.float64): N.FLOAT64}


def host_bits(bools):
    return np.concatenate([np.packbits(bools, bitorder="little"), np.zeros(8, np.uint8)])


def encode_decode(v, m, capacity=None):
    t = TYPE_OF[v.dtype]
    n = len(v)
    buf = host_bits(v) if t == N.BOOL else v
    vb = host_bits(m) if m is not None else None
    counts = np.zeros(2, np.int64)
    N.call("ag_run_end_count", t, buf.ctypes.data, None if vb is None else vb.ctypes.data, 0, n, counts.ctypes.data)
    runs = int(counts[0])
    cap = runs if capacity is None else capacity
    ends = np.zeros(cap + 1, np.int32)
    out = np.zeros(cap // 8 + 8, np.uint8) if t == N.BOOL else np.zeros(cap + 1, v.dtype)
    ov = np.zeros(cap // 8 + 8, np.uint8)
    N.call("ag_run_end_encode", t, N.INT32, buf.ctypes.data, None if vb is None else vb.ctypes.data, 0, n, ends.ctypes.data,
           out.ctypes.data, ov.ctypes.data if vb is not None else None, cap, counts.ctypes.data)
    w_ends, w_vals, w_valid, _ = ref.encode(v, m, "int32")
    k = min(runs, cap)
    assert runs == len(w_ends) and (ends[:k] == w_ends[:k]).all()
    rv = np.unpackbits(out, bitorder="little")[:k].astype(bool) if t == N.BOOL else out[:k]
    assert rv.tobytes() == np.ascontiguousarray(w_vals[:k]).tobytes()
    if m is not None:
        assert (np.unpackbits(ov, bitorder="little")[:k].astype(bool) == w_valid[:k]).all()
    if capacity is not None:
        return
    # decode a slice that cuts runs at both ends
    off, ln = 3, n - 5
    dout = np.zeros(ln // 8 + 8, np.uint8) if t == N.BOOL else np.zeros(ln, v.dtype)
    dov = np.zeros(ln // 8 + 8, np.uint8)
    nulls = C.c_int64()
    N.call("ag_run_end_decode", t, N.INT32, ends.ctypes.data, runs, out.ctypes.data, ov.ctypes.data if vb is not None else None,
           0, off, ln, dout.ctypes.data, dov.ctypes.data if vb is not None else None, C.byref(nulls))
    got = np.unpackbits(dout, bitorder="little")[:ln].astype(bool) if t == N.BOOL else dout
    assert got.tobytes() == np.ascontiguousarray(v[off:off + ln]).tobytes()


N.call("ag_init", 0)
n = int(sys.argv[1]) if len(sys.argv) > 1 else 20011
rng = np.random.default_rng(5)
for dt in (np.bool_, np.uint8, np.int16, np.int32, np.float32, np.int64, np.float64):
    for mean in (1, 3, 300):
        lengths = rng.integers(1, 2 * mean, n // mean + 2)
        k = np.repeat(np.arange(len(lengths)), lengths)[:n]
        v = (k % 2).astype(bool) if dt == np.bool_ else (k % 7).astype(dt)
        m = np.repeat(rng.random(len(lengths)) > 0.2, lengths)[:n]
        encode_decode(v, None)
        encode_decode(v, m)
        encode_decode(v, m, capacity=len(ref.encode(v, m)[0]) // 2)
# malformed run ends: the decode reads and writes only inside its buffers
ends = np.array([2, 4, 4, 9], np.int32)
vals = np.arange(4, dtype=np.int64)
out = np.zeros(9, np.int64)
st, _ = N.call_status("ag_run_end_decode", N.INT64, N.INT32, ends.ctypes.data, 4, vals.ctypes.data, None, 0, 0, 9,
                      out.ctypes.data, None, None)
assert st == N.AG_ERR_INVALID
print("run_end sanitizer calls ok")
