#!/usr/bin/env python
"""Moderate dictionary_encode calls that reach every kernel of hash.cu's dictionary path (inserts into one table and
into both tables, the rank passes, the index pass with and without validity, Mask and Encode, every value width), for
compute-sanitizer memcheck and racecheck:

    compute-sanitizer --tool memcheck --error-exitcode 9 python scripts/lab/san_dictionary_encode.py 20011
    compute-sanitizer --tool racecheck --error-exitcode 9 python scripts/lab/san_dictionary_encode.py 9001

Results are compared with the NumPy restatement, so a sanitizer-clean run is also a correct one."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from arrow_go_b200 import _native as N  # noqa: E402
from dictionary_encode_ref import dictionary_encode_ref  # noqa: E402


def encode(chunks, ne):
    dtype = chunks[0][0].dtype
    keep, desc = [], []
    for v, m in chunks:
        vb = np.packbits(m, bitorder="little") if m is not None else None
        idx = np.zeros(max(len(v), 1), np.int32)
        iv = np.zeros(((len(v) + 31) // 32) * 4 + 4, np.uint8)
        keep += [v, vb, idx, iv]
        desc.append((v.ctypes.data, None if vb is None else vb.ctypes.data, 0, len(v), idx.ctypes.data, iv.ctypes.data))
    total = sum(len(v) for v, _ in chunks)
    dictionary = np.zeros(max(total, 1), dtype)
    dvalid = np.zeros(total // 8 + 2, np.uint8)
    counts = np.zeros(len(chunks) + 2, np.int64)
    N.call("ag_dictionary_encode", 8 * dtype.itemsize, N.dict_chunk_table(desc), len(chunks), ne, dictionary.ctypes.data,
           dvalid.ctypes.data, counts.ctypes.data)
    return [keep[4 * c + 2][:len(v)] for c, (v, _) in enumerate(chunks)], dictionary[:counts[0]]


def check(chunks, ne):
    got_idx, got_dict = encode(chunks, ne)
    want, want_dict, _ = dictionary_encode_ref(chunks, ne)
    assert got_dict.tobytes() == want_dict.tobytes()
    for g, (w, valid, _) in zip(got_idx, want):
        assert (g[valid] == w[valid]).all() if valid is not None else (g == w).all()


N.call("ag_init", 0)
n = int(sys.argv[1]) if len(sys.argv) > 1 else 20011
rng = np.random.default_rng(5)
for dt in (np.uint8, np.int16, np.int32, np.int64, np.float64):
    for card in (5, 3000):
        v = rng.integers(0, card, n).astype(dt)
        for ne in (0, 1):
            check([(v, None)], ne)
            check([(v[: n // 3], rng.random(n // 3) > 0.25), (v[n // 3:], rng.random(n - n // 3) > 0.25)], ne)
N.call("ag_unique_set_policy", 1000, 1024)   # the small table overflows: the full-size table and its gated launches
try:
    for ne in (0, 1):
        check([(rng.permutation(n).astype(np.int64), rng.random(n) > 0.1)], ne)
finally:
    N.call("ag_unique_set_policy", 0, 0)
print("dictionary_encode sanitizer calls ok")
