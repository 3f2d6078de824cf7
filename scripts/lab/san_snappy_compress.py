#!/usr/bin/env python
"""A small batch through both kernels of snappy_encode.cu (the match kernel over several fragments per page, literal-
and copy-heavy bodies, pages of 0..3 bytes, pages ending on and around 64 KiB, a partly filled last match block) in both
flavours, for compute-sanitizer memcheck and racecheck:

    compute-sanitizer --tool memcheck --error-exitcode 9 python scripts/lab/san_snappy_compress.py
    compute-sanitizer --tool racecheck --error-exitcode 9 python scripts/lab/san_snappy_compress.py

Each warp of the match kernel owns one hash table in shared memory; its lanes read the table, then write it after a
__syncwarp.  Results are compared with tests/snappy_encode_model.py, so a sanitizer-clean run is also a correct one."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import snappy_encode_model as M  # noqa: E402
from arrow_go_b200 import _native as N  # noqa: E402
from arrow_go_b200.device import DeviceBuffer  # noqa: E402


def main():
    N.call("ag_init", 0)
    rng = np.random.default_rng(int(sys.argv[1]) if len(sys.argv) > 1 else 7)
    c = M.corpora(rng, 3 * 65536 + 11)
    bodies = [b"", b"a", b"abc", c["timestamps"][:65536], c["emails"][:65537], c["indices_17bit"], c["zeros"][:131072],
              rng.integers(0, 256, 70_000, dtype=np.uint8).tobytes()]
    src = np.frombuffer(b"".join(bodies) + bytes(8), np.uint8).copy()
    pages, s, d = [], 0, 5
    for b in bodies:
        pages.append((s, len(b), d, M.max_size(len(b))))
        s += len(b)
        d += M.max_size(len(b)) + 3
    tbl = N.compressed_table(pages)
    want = [M.compress(b) for b in bodies]
    out, w = np.zeros(d, np.uint8), np.zeros(len(pages), np.int64)
    N.call("ag_parquet_snappy_compress", src.ctypes.data, tbl, len(pages), out.ctypes.data, w.ctypes.data)
    for (_, _, o, _), k, x in zip(pages, w, want):
        assert out[o:o + k].tobytes() == x
    ds, dd, dw = DeviceBuffer(src.nbytes + 64), DeviceBuffer(d + 64), DeviceBuffer(8 * len(pages) + 64)
    N.call("ag_upload", ds.ptr, src.ctypes.data, src.nbytes, None)
    N.call("ag_parquet_snappy_compress_dev", ds.ptr, tbl, len(pages), dd.ptr, dw.ptr, None)
    N.call("ag_stream_sync", None)
    got, gw = dd.to_numpy(np.uint8, d, 0), dw.to_numpy(np.int64, len(pages), 0)
    for (_, _, o, _), k, x in zip(pages, gw, want):
        assert got[o:o + k].tobytes() == x
    print("ok", len(pages), "pages", int(gw.sum()), "bytes")


if __name__ == "__main__":
    main()
