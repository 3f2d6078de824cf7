"""run_end_encode and run_end_decode at 100M rows with int32 run ends, timed with CUDA events on device-resident
columns.  Every workload's runs are checked against a NumPy encode of its input, and its decode against the input, in
the same run.

    python scripts/run_end_bench.py [--rows N] [--reps R] [--profile] [--out FILE]

Encode is the full host-mirror sequence on the device: count, one 16-byte read-back, encode with an exact capacity.
Decode expands the encoded array back to n rows.  Modelled bytes:
  encode: two reads of the input (count + encode) + runs x (value width + run-end width) written;
  decode: runs x (value width + run-end width) read + n x value width written.
Validity adds n/8 bytes per read of the input and runs/8 (encode) or n/8 (decode) bytes written.  A BOOL column's
value width is 1/8 byte.  The floor is those bytes over 3.35 TB/s (H100 SXM HBM3 data sheet).

--profile adds, per workload, the device time of each kernel (torch.profiler with CUDA activities, a separate pass)."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from arrow_go_b200 import _native as N  # noqa: E402
from dictionary_encode_bench import HBM, Dev, card_info, download, kernel_split, timed, upload  # noqa: E402


def column(rng, n, mean_run, dtype):
    """n rows in runs of mean length `mean_run` (uniform in [1, 2*mean_run-1]); neighbouring runs differ."""
    if mean_run == 1:
        k = np.arange(n, dtype=np.int64)
    else:
        lengths = rng.integers(1, 2 * mean_run, n // mean_run + 64)
        k = np.repeat(np.arange(len(lengths), dtype=np.int64), lengths)[:n]
    if dtype == np.bool_:
        return (k & 1).astype(bool)
    return (k % 1000 + 1).astype(dtype)


def run(name, vals, valid, reps, profile=False):
    n = len(vals)
    is_bool = vals.dtype == np.bool_
    type_id = N.BOOL if is_bool else {np.dtype(np.int64): N.INT64, np.dtype(np.int32): N.INT32}[vals.dtype]
    host = np.packbits(vals, bitorder="little") if is_bool else vals
    dv = upload(host)
    dvalid = upload(np.packbits(valid, bitorder="little")) if valid is not None else None
    counts = Dev(16)
    N.call("ag_run_end_count_dev", type_id, dv.p, dvalid.p if dvalid else None, 0, n, counts.p, None)
    runs, null_runs = (int(x) for x in download(counts, np.int64, 2))
    w = 0.125 if is_bool else vals.dtype.itemsize
    ends = Dev(runs * 4)
    rvals = Dev(((runs + 31) // 32) * 4 if is_bool else runs * int(w))
    rvalid = Dev(((runs + 31) // 32) * 4) if valid is not None else None
    out = Dev(((n + 31) // 32) * 4 if is_bool else n * int(w))
    out_valid = Dev(((n + 31) // 32) * 4) if valid is not None else None
    c_h = np.zeros(2, np.int64)
    words = Dev(16)

    def enc():   # the host mirror's sequence: count, read back, encode with the exact capacity
        N.call("ag_run_end_count_dev", type_id, dv.p, dvalid.p if dvalid else None, 0, n, counts.p, None)
        N.call("ag_download", c_h.ctypes.data, counts.p, 16, None)
        N.call("ag_stream_sync", None)
        N.call("ag_run_end_encode_dev", type_id, N.INT32, dv.p, dvalid.p if dvalid else None, 0, n, ends.p, rvals.p,
               rvalid.p if rvalid else None, int(c_h[0]), counts.p, None)

    def dec():
        N.call("ag_run_end_decode_dev", type_id, N.INT32, ends.p, runs, rvals.p, rvalid.p if rvalid else None, 0, 0, n, out.p,
               out_valid.p if out_valid else None, words.p, C.c_void_p(words.p.value + 8), None)

    N.call("ag_error_word_reset_dev", C.c_void_p(words.p.value + 8), None)
    for _ in range(3):
        enc()
        dec()
    t_enc, t_dec = [], []
    for _ in range(3):   # alternate the two so that drift hits both alike
        t_enc.append(timed(enc, reps))
        t_dec.append(timed(dec, reps))
    # checks: the runs against NumPy, the decode against the input
    e = download(ends, np.int32, runs).astype(np.int64)
    b = np.ones(n, bool)
    b[1:] = vals[1:] != vals[:-1]
    if valid is not None:
        b[1:] |= valid[1:] != valid[:-1]
    starts = np.flatnonzero(b)
    assert runs == len(starts) and (e == np.append(starts[1:], n)).all(), name
    if is_bool:
        got = np.unpackbits(download(out, np.uint8, (n + 7) // 8), bitorder="little")[:n].astype(bool)
    else:
        got = download(out, vals.dtype, n)
    assert (got == vals).all(), name
    assert download(words, np.int64, 2)[1] == N.NO_ERROR_POS
    rw = 4
    vbits = n / 8 if valid is not None else 0
    enc_bytes = 2 * (n * w + vbits) + runs * (w + rw) + (runs / 8 if valid is not None else 0)
    dec_bytes = runs * (w + rw) + (runs / 8 if valid is not None else 0) + n * w + vbits
    te, td = float(np.median(t_enc)), float(np.median(t_dec))
    split = {"kernels_ms": {"encode": kernel_split(enc, reps), "decode": kernel_split(dec, reps)}} if profile else {}
    return {**split, "workload": name, "rows": n, "runs": runs, "null_runs": null_runs,
            "encode_ms": round(te, 3), "encode_bytes": int(enc_bytes), "encode_hbm_share": round(enc_bytes / HBM * 1e3 / te, 3),
            "decode_ms": round(td, 3), "decode_bytes": int(dec_bytes), "decode_hbm_share": round(dec_bytes / HBM * 1e3 / td, 3)}


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
    rows = []
    for mean in (1, 16, 1024):
        rows.append(run(f"int64 runs of {mean}", column(rng, n, mean, np.int64), None, a.reps, a.profile))
    nulls = np.repeat(rng.random(n // 16 + 64) >= 0.10, 16)[:n]   # 10% of the runs null, in runs of 16
    rows.append(run("int64 runs of 16, 10% nulls", column(rng, n, 16, np.int64), nulls, a.reps, a.profile))
    del nulls
    rows.append(run("int32 runs of 16", column(rng, n, 16, np.int32), None, a.reps, a.profile))
    rows.append(run("bool runs of 16", column(rng, n, 16, np.bool_), None, a.reps, a.profile))
    res = {"card": card_info(), "results": rows}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
