"""dictionary_encode at 100M rows, timed with CUDA events on device-resident columns, alternated with `unique` on the
same column.  Every workload's output is decoded and checked against its input in the same run.

    python scripts/dictionary_encode_bench.py [--rows N] [--reps R] [--profile]

--profile adds, per workload, the device time of each kernel of one dictionary_encode call (torch.profiler with CUDA
activities, a separate pass after the timed one, averaged over `reps` calls).

Algorithmic bytes: the values read once, the int32 indices written, plus the index validity and the dictionary; the
floor is those bytes over 3.35 TB/s (H100 SXM HBM3 data sheet)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from arrow_go_b200 import _native as N  # noqa: E402

HBM = 3.35e12


def card_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


class Dev:
    def __init__(self, nbytes):
        self.p = C.c_void_p()
        N.call("ag_dev_alloc", C.byref(self.p), max(nbytes, 8))

    def __del__(self):
        N.raw().ag_dev_free(self.p)


def upload(a):
    d = Dev(a.nbytes)
    N.call("ag_upload", d.p, a.ctypes.data, a.nbytes, None)
    return d


def download(d, dtype, n):
    a = np.empty(n, dtype)
    N.call("ag_download", a.ctypes.data, d.p, a.nbytes, None)
    N.call("ag_stream_sync", None)
    return a


def timed(fn, reps):
    e0, e1 = C.c_void_p(), C.c_void_p()
    N.call("ag_event_create", C.byref(e0))
    N.call("ag_event_create", C.byref(e1))
    ms = []
    for _ in range(reps):
        N.call("ag_event_record", e0, None)
        fn()
        N.call("ag_event_record", e1, None)
        N.call("ag_event_sync", e1)
        t = C.c_float()
        N.call("ag_event_elapsed_ms", e0, e1, C.byref(t))
        ms.append(t.value)
    N.call("ag_event_destroy", e0)
    N.call("ag_event_destroy", e1)
    return float(np.median(ms))


def kernel_split(fn, reps):
    """{kernel name: mean device ms per call} over `reps` calls of fn, from torch.profiler's CUDA activity."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        N.call("ag_stream_sync", None)
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if t > 0 and e.key != "ProfilerStep*":
            out[e.key.split("(")[0][:60]] = round(t / reps / 1e3, 3)
    del torch
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def run(name, vals, valid, ne, reps, profile=False):
    n, w = len(vals), vals.dtype.itemsize
    dv = upload(vals)
    dvalid = upload(np.packbits(valid, bitorder="little")) if valid is not None else None
    idx, ival = Dev(n * 4), Dev(((n + 31) // 32) * 4)
    dic, dicv, counts = Dev(n * w), Dev(n // 8 + 8), Dev(3 * 8)
    uout, ulen = Dev(n * w), Dev(16)
    uvalid = Dev(n // 8 + 8)
    table = N.dict_chunk_table([(dv.p.value, dvalid.p.value if dvalid else None, 0, n, idx.p.value, ival.p.value)])

    def enc():
        N.call("ag_dictionary_encode_dev", 8 * w, table, 1, ne, dic.p, dicv.p, counts.p, None)

    def uniq():
        N.call("ag_unique_dev", 8 * w, dv.p, dvalid.p if dvalid else None, 0, n, uout.p, uvalid.p if dvalid else None, n, ulen.p, None)

    for _ in range(3):
        enc()
        uniq()
    t_enc, t_uniq = [], []
    for _ in range(3):   # alternate the two so that drift hits both alike
        t_enc.append(timed(enc, reps))
        t_uniq.append(timed(uniq, reps))
    k, dnull, nulls = (int(x) for x in download(counts, np.int64, 3))
    d = download(dic, vals.dtype, k)
    ix = download(idx, np.int32, n)
    ok = valid if valid is not None else np.ones(n, bool)
    if ne == 1 and valid is not None and not valid.all():
        assert dnull == 1
    assert (d[ix[ok]] == vals[ok]).all(), name
    _, first = np.unique(vals[ok], return_index=True)
    assert k - dnull == len(first), name
    nbytes = n * w + n * 4 + k * w + (((n + 7) // 8) * 2 if valid is not None else 0)
    t = float(np.median(t_enc))
    split = {"kernels_ms": kernel_split(enc, reps)} if profile else {}
    return {**split, "workload": name, "rows": n, "dict_len": k, "index_nulls": nulls, "dictionary_encode_ms": round(t, 3),
            "unique_ms": round(float(np.median(t_uniq)), 3), "alg_bytes": nbytes, "floor_ms": round(nbytes / HBM * 1e3, 3),
            "floor_share": round(nbytes / HBM * 1e3 / t, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    N.call("ag_init", 0)
    n = a.rows
    rng = np.random.default_rng(42)
    pool = rng.integers(-(1 << 62), 1 << 62, 100)
    low = pool[rng.integers(0, 100, n)]
    nulls = rng.random(n) >= 0.10
    rows = []
    rows.append(run("int64 100 distinct", low, None, 0, a.reps, a.profile))
    rows.append(run("int64 100 distinct 10% nulls Mask", low, nulls, 0, a.reps, a.profile))
    rows.append(run("int64 100 distinct 10% nulls Encode", low, nulls, 1, a.reps, a.profile))
    del nulls
    rows.append(run("int64 4M distinct", rng.integers(0, 4_000_000, n).astype(np.int64), None, 0, a.reps, a.profile))
    rows.append(run("int64 all distinct", rng.permutation(n).astype(np.int64), None, 0, a.reps, a.profile))
    rows.append(run("int32 100 distinct", low.astype(np.int32), None, 0, a.reps, a.profile))
    res = {"card": card_info(), "results": rows}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
