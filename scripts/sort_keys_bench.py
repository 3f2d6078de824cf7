"""sort_indices over several keys (ag_sort_indices_keys_dev) at 100M rows, timed with CUDA events on device-resident
columns, with ag_sort_indices_dev on the first column alone for comparison.  Each workload's permutation is checked
against the model of tests/sort_keys_ref.py on its first --check-rows rows (a separate call of the same kernels).

    python scripts/sort_keys_bench.py [--rows N] [--reps R] [--check-rows M] [--profile] [--out FILE]

Workloads:
  narrow   (int32 with <= 2^16 distinct values, int64 small range): one packed word, no gather;
  wide     (int64 full range, float64): two words, so one gather pass;
  wide_nn  the same with 10 % nulls in both and 10 % NaN in the float64;
  chunked  (bool, int16, int32) in 4 chunks per column, chunk boundaries differing between the columns.
Modelled bytes (`model_bytes`): statistics and pack each read every key column (values + validity bits), pack writes
W words of 8 bytes (4 when the key fits 32 bits); a digit pass reads the key word in its histogram and (key, row) in its
scatter and writes (key, row), the last one writes 8-byte indices; the first pass of a word after the first reads the
row (4 bytes) and gathers the key word (8 bytes, random).  The floor is those bytes over 3.35 TB/s (H100 SXM HBM3 data
sheet); random gathers do not reach it.  --profile adds the device time of each kernel (torch.profiler, a separate
pass)."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from arrow_go_b200 import _native as N  # noqa: E402
from dictionary_encode_bench import HBM, Dev, card_info, download, kernel_split, timed, upload  # noqa: E402
from sort_keys_ref import _key_ranks, sort_keys_model  # noqa: E402

TYPE = {np.dtype(np.bool_): N.BOOL, np.dtype(np.int16): N.INT16, np.dtype(np.int32): N.INT32, np.dtype(np.int64): N.INT64,
        np.dtype(np.float64): N.FLOAT64}


def workload(name, n, rng):
    """[(values, valid or None, chunk lengths)], keys [(column, order, placement)]."""
    if name == "narrow":
        cols = [(rng.integers(0, 1 << 16, n).astype(np.int32), None, [n]),
                (rng.integers(-1000, 1000, n).astype(np.int64), None, [n])]
        return cols, [(0, 0, 0), (1, 1, 0)]
    if name in ("wide", "wide_nn"):
        a = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, dtype=np.int64, endpoint=True)
        b = rng.standard_normal(n)
        va = vb = None
        if name == "wide_nn":
            b[rng.random(n) < 0.1] = np.nan
            va, vb = rng.random(n) >= 0.1, rng.random(n) >= 0.1
        return [(a, va, [n]), (b, vb, [n])], [(0, 0, 0), (1, 1, 1)]
    q = n // 4
    cols = [(rng.integers(0, 2, n).astype(bool), None, [q, q, q, n - 3 * q]),
            (rng.integers(-30000, 30000, n).astype(np.int16), None, [q + 7, q, q - 7, n - 3 * q]),
            (rng.integers(-10**9, 10**9, n).astype(np.int32), None, [q - 5, q + 5, q, n - 3 * q])]
    return cols, [(0, 0, 0), (1, 1, 0), (2, 0, 0)]


def bits(v):
    return np.concatenate([np.packbits(np.asarray(v, dtype=bool), bitorder="little"), np.zeros(8, np.uint8)])


def device_keys(cols, keys):
    """Upload every chunk of every column; (ag_sort_key table, device buffers to keep alive)."""
    keep, dcols = [], []
    for vals, valid, lens in cols:
        chunks, lo = [], 0
        for ln in lens:
            v = vals[lo:lo + ln]
            dv = upload(bits(v) if v.dtype == np.bool_ else np.ascontiguousarray(v))
            dok = upload(bits(valid[lo:lo + ln])) if valid is not None else None
            keep += [dv, dok]
            chunks.append((dv.p.value, dok.p.value if dok else None, 0, ln))
            lo += ln
        dcols.append((TYPE[vals.dtype], chunks))
    return N.sort_key_table([(t, o, p, dcols[c][1]) for c, o, p in keys for t in [dcols[c][0]]]), keep


def model_bytes(cols, keys, n, bits_total):
    read = sum(cols[c][0].dtype.itemsize * n if cols[c][0].dtype != np.bool_ else n / 8 for c, _, _ in keys)
    read += sum(n / 8 for c, _, _ in keys if cols[c][1] is not None)
    kw = 4 if bits_total <= 32 else 8
    words = 1 if bits_total <= 32 else (bits_total + 63) // 64
    total = 2 * read + words * kw * n
    passes = 0
    for w in range(words):
        nd = (min(bits_total - 64 * w, 8 * kw) + 7) // 8
        for d in range(nd):
            first_of_word = d == 0 and w > 0
            hist = (4 + kw) * n if first_of_word else kw * n
            scatter = (4 + kw) * n * 2 if (w, d) != (0, 0) else (kw * n + (kw + 4) * n)
            total += hist + scatter
            passes += 1
    total += (8 - (kw + 4)) * n   # the last pass writes 8-byte indices instead of (key, row)
    return total, passes


def key_image(v, order):
    """The device's order-preserving unsigned image key' (sort_key in csrc/sort.cu), as uint64."""
    if v.dtype == np.bool_:
        k, width = v.astype(np.uint64), 1
    elif v.dtype.kind == "f":
        u = v.astype(np.float64).view(np.uint64) if v.dtype == np.float64 else v.view(np.uint32).astype(np.uint64)
        width = 8 * v.dtype.itemsize
        sign, mag = u >> np.uint64(width - 1), u & np.uint64((1 << (width - 1)) - 1)
        top = np.uint64(1 << (width - 1))
        k = np.where(sign == 1, top - mag, top | mag).astype(np.uint64)
    else:
        width = 8 * v.dtype.itemsize
        k = v.astype(np.int64).view(np.uint64) + np.uint64(1 << (width - 1)) if v.dtype.kind == "i" else v.astype(np.uint64)
        k = k & np.uint64((1 << width) - 1) if width < 64 else k
    if order == 1:
        k = ~k if width == 64 else k ^ np.uint64((1 << width) - 1)
    return k


def packed_bits(cols, keys, n):
    """B of the device plan (class bits + value bits per key), computed on the host for the byte model."""
    b = 0
    for c, o, p in keys:
        vals, valid, lens = cols[c]
        col = [(vals, valid)]
        code, _ = _key_ranks(col, o, p)
        classes = len(np.unique(code))
        b += {1: 0, 2: 1, 3: 2}[classes]
        nan = np.isnan(vals) if vals.dtype.kind == "f" else np.zeros(n, bool)
        fin = (valid if valid is not None else np.ones(n, bool)) & ~nan
        if fin.sum() > 1:
            k = key_image(vals[fin], o)
            mn, mx = int(k.min()), int(k.max())
            varying = int(np.bitwise_or.reduce(k)) ^ int(np.bitwise_and.reduce(k))
            tz = (varying & -varying).bit_length() - 1 if varying else 0
            b += ((mx - mn) >> tz).bit_length() if mx > mn else 0
    return b


def run(name, n, reps, check_rows, profile):
    rng = np.random.default_rng(sum(map(ord, name)))
    cols, keys = workload(name, n, rng)
    table, keep = device_keys(cols, keys)
    out = Dev(n * 8)
    call = lambda: N.call("ag_sort_indices_keys_dev", len(keys), table, n, out.p, None)  # noqa: E731
    call()
    ms = timed(call, reps)
    idx = download(out, np.uint64, n)
    assert idx.max() < n
    # one column, the single-key kernel, on a contiguous copy of the first key's column
    v0, ok0, _ = cols[keys[0][0]]
    single = None
    if v0.dtype != np.bool_:
        d0 = upload(np.ascontiguousarray(v0))
        dok0 = upload(bits(ok0)) if ok0 is not None else None
        out1 = Dev(n * 8)
        one = lambda: N.call("ag_sort_indices_dev", TYPE[v0.dtype], d0.p, dok0.p if dok0 else None, 0, n, keys[0][1],  # noqa: E731
                             keys[0][2], out1.p, None, None, None)
        one()
        single = timed(one, reps)
    # correctness on a prefix, same kernels
    m = min(n, check_rows)
    sub = [(v[:m], None if ok is None else ok[:m], [m]) for v, ok, _ in cols]
    t2, keep2 = device_keys(sub, keys)
    out2 = Dev(m * 8)
    N.call("ag_sort_indices_keys_dev", len(keys), t2, m, out2.p, None)
    got = download(out2, np.uint64, m)
    want = sort_keys_model([[(v, ok)] for v, ok, _ in sub], keys)
    assert np.array_equal(got, want), f"{name}: mismatch against the model"
    bits_total = packed_bits(cols, keys, n)
    mbytes, passes = model_bytes(cols, keys, n, bits_total)
    res = {"workload": name, "rows": n, "keys": len(keys), "packed_bits": bits_total, "digit_passes": passes,
           "ms": round(ms, 3), "single_key_ms": None if single is None else round(single, 3),
           "model_bytes": int(mbytes), "floor_ms": round(mbytes / HBM * 1e3, 3), "checked_rows": m}
    if profile:
        res["kernels_ms"] = kernel_split(call, 3)
    del keep, keep2
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--check-rows", type=int, default=4_000_000)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    N.call("ag_init", 0)
    results = {"card": card_info(), "cases": [run(w, a.rows, a.reps, a.check_rows, a.profile)
                                               for w in ("narrow", "wide", "wide_nn", "chunked")]}
    text = json.dumps(results, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
