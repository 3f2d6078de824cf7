"""cumulative_sum on the inputs that are not the aligned unchecked case: checked integers, outputs that are not 16-byte
aligned and narrow slices, at 100M rows, timed with CUDA events on device-resident columns.

    python scripts/cumsum_paths_bench.py [--rows N] [--reps R] [--lib PATH] [--out FILE]

--lib loads another build of libarrowgpu.so (the same C ABI), so that two builds can be compared on the same inputs
from separate processes.  Each case prints one JSON line with its median time and a SHA-256 digest of everything the
call produced (values, validity bitmap, null count, first failing row): two builds that compute the same thing print
the same digests.  Every timed call re-initialises the carried state, as bench.py's cumulative_sum rows do.

Modelled bytes: n x width read + n x width written (+ n/8 read and n/8 written with a validity bitmap); the floor is
those bytes over 3.35 TB/s (H100 SXM HBM3 data sheet)."""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from arrow_go_b200 import _native as N  # noqa: E402
from dictionary_encode_bench import HBM, Dev, card_info, download, timed, upload  # noqa: E402

NO_POS = (1 << 63) - 1

# (name, type, dtype, checked, null fraction, input offset in elements, output offset in bytes)
CASES = [
    ("checked_i64", N.INT64, np.int64, 1, 0.0, 0, 0),
    ("checked_i64_nulls", N.INT64, np.int64, 1, 0.1, 0, 0),
    ("checked_i32", N.INT32, np.int32, 1, 0.0, 0, 0),
    ("checked_i32_nulls", N.INT32, np.int32, 1, 0.1, 0, 0),
    ("checked_i8", N.INT8, np.int8, 1, 0.0, 0, 0),
    ("checked_i8_nulls", N.INT8, np.int8, 1, 0.1, 0, 0),
    ("i64_out_plus8", N.INT64, np.int64, 0, 0.0, 0, 8),
    ("f64_out_plus8", N.FLOAT64, np.float64, 0, 0.0, 0, 8),
    ("i8_slice_odd", N.INT8, np.int8, 0, 0.0, 1, 0),
    ("i16_slice_odd", N.INT16, np.int16, 0, 0.0, 1, 0),
]


def column(rng, n, dtype):
    if dtype == np.float64:
        return rng.standard_normal(n)
    return rng.integers(-3, 4, n).astype(dtype)  # checked int8 leaves its range early; the kernel still runs every row


def run(case, n, reps, rng):
    name, t, dtype, checked, p_null, in_off, out_off = case
    w = np.dtype(dtype).itemsize
    x = column(rng, n + in_off, dtype)
    dx = upload(x)
    valid = rng.random(n) >= p_null if p_null else None
    dvalid = upload(np.packbits(valid, bitorder="little")) if valid is not None else None
    dout = Dev(n * w + out_off)
    ovalid = Dev((n + 7) // 8) if valid is not None else None
    state, bad = Dev(32), Dev(8)
    out_p = dout.p.value + out_off

    def call():
        N.call("ag_cumulative_sum_state_init_dev", state.p, t, None, None)
        if checked:
            N.call("ag_error_word_reset_dev", bad.p, None)
        N.call("ag_cumulative_sum_dev", t, dx.p.value + in_off * w, dvalid.p if dvalid else None, 0, n, 1, checked,
               out_p, ovalid.p if ovalid else None, 0, state.p, bad.p, None)

    call()  # warm-up, and the result the digest is taken from
    N.call("ag_stream_sync", None)
    h = hashlib.sha256()
    out = download(dout, np.uint8, n * w + out_off)[out_off:]
    h.update(out.tobytes())
    if ovalid is not None:
        h.update(download(ovalid, np.uint8, (n + 7) // 8).tobytes())
    st = download(state, np.int64, 4)
    first_bad = int(download(bad, np.int64, 1)[0]) if checked else NO_POS
    h.update(np.array([st[3], first_bad], dtype=np.int64).tobytes())
    ms = timed(call, reps)
    nbytes = 2 * n * w + (2 * n / 8 if valid is not None else 0)
    return {"case": name, "ms": round(ms, 4), "frac_of_hbm": round(nbytes / (ms * 1e-3) / HBM, 3), "null_count": int(st[3]),
            "first_bad": first_bad, "digest": h.hexdigest()[:16]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--lib", help="path of the libarrowgpu.so to load (default: the in-tree build)")
    ap.add_argument("--out", help="append the JSON lines to this file too")
    args = ap.parse_args()
    if args.lib:
        N.LIB_PATH = os.path.abspath(args.lib)
    N.call("ag_init", 0)
    lines = [{"card": card_info(), "lib": N.LIB_PATH, "rows": args.rows}]
    rng = np.random.default_rng(20261017)
    for case in CASES:
        lines.append(run(case, args.rows, args.reps, rng))
    for line in lines:
        print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
