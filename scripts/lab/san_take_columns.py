#!/usr/bin/env python
"""Moderate ag_take_columns calls that reach every path of take_columns.cu (every value width and BOOL, chunk starts in
shared memory and in global memory, shared and distinct chunk layouts, empty and sliced chunks, null and out-of-range
indices with and without the bounds check, a tail shorter than a warp), for compute-sanitizer memcheck and racecheck:

    compute-sanitizer --tool memcheck --error-exitcode 9 python scripts/lab/san_take_columns.py 20011
    compute-sanitizer --tool racecheck --error-exitcode 9 python scripts/lab/san_take_columns.py 9001

Results are compared with the NumPy model of tests/table_select_model.py, so a sanitizer-clean run is also a correct
one."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import table_select_model as M  # noqa: E402
from arrow_go_b200 import _native as N  # noqa: E402

TYPES = [(N.BOOL, np.bool_), (N.UINT8, np.uint8), (N.INT16, np.int16), (N.FLOAT32, np.float32), (N.INT64, np.int64)]


def bits(v, off=0):
    return np.concatenate([np.packbits(np.concatenate([np.zeros(off, bool), v]), bitorder="little"), np.zeros(8, np.uint8)])


def unpack(b, n):
    return np.unpackbits(b, bitorder="little")[:n].astype(bool)


def run(n, m, nchunks, rng, bounds):
    cuts = sorted(set([0, n] + rng.integers(0, n + 1, nchunks - 1).tolist())) if n else [0, 0]
    cuts.insert(1, cuts[0])   # an empty chunk
    keep, table, want, outs = [], [], [], []
    idx = rng.integers(0, n + 2, m).astype(np.int64)   # a few out of range
    iv = rng.random(m) >= 0.2
    if bounds:
        idx[iv] %= max(n, 1)
        if n == 0:
            iv[:] = False
    for k, (t, dt) in enumerate(TYPES):
        v = rng.random(n) < 0.5 if t == N.BOOL else rng.integers(0, 100, n).astype(dt)
        ok = rng.random(n) >= 0.3
        my_cuts = cuts if k % 2 == 0 else [0, n]   # two layouts
        chunks = []
        for a, b in zip(my_cuts, my_cuts[1:]):
            off = int(rng.integers(0, 13))
            vb = bits(v[a:b], off) if t == N.BOOL else np.concatenate([np.zeros(off, dt), v[a:b], np.zeros(1, dt)])
            okb = bits(ok[a:b], off)
            keep += [vb, okb]
            chunks.append((vb.ctypes.data, okb.ctypes.data, off, b - a))
        out = np.zeros(m // 8 + 8, np.uint8) if t == N.BOOL else np.zeros(m, dt)
        ov = np.zeros(m // 8 + 8, np.uint8)
        outs.append((t, out, ov))
        table.append((t, chunks, out.ctypes.data, ov.ctypes.data))
        want.append(M.gather((v, ok), idx, iv))
    ivb = bits(iv, 5)
    bad, bad_idx = C.c_int64(), C.c_int64()
    st, msg = N.call_status("ag_take_columns", len(table), N.take_column_table(table), n, 64, 1, idx.ctypes.data, ivb.ctypes.data,
                            5, m, 1 if bounds else 0, C.byref(bad), C.byref(bad_idx))
    assert st == N.AG_OK, msg
    for (t, out, ov), (wv, wok) in zip(outs, want):
        assert (unpack(ov, m) == wok).all()
        got = unpack(out, m) if t == N.BOOL else out
        assert (got == wv).all()


def main():
    m = int(sys.argv[1]) if len(sys.argv) > 1 else 20011
    N.call("ag_init", 0)
    rng = np.random.default_rng(m)
    run(3000, m, 5, rng, True)
    run(20000, m, 9000, rng, True)   # more chunk starts than shared memory holds
    run(1000, m, 3, rng, False)      # out-of-range valid indices without the bounds check
    run(0, 31, 1, rng, True)         # no rows: every index null
    print("san_take_columns ok")


if __name__ == "__main__":
    main()
