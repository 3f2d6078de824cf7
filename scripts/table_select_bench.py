"""Take, FilterTable and Sort on a 100M-row table (int64, float64 with 10 % nulls, int32, bool) in 1, 16 and 1000 chunks,
through the table path (one ag_take_columns_dev launch per index chunk or filter span) and through the per-column route
(pc.Take / pc.Filter on each column), alternating the two in the same run.  Times are CUDA events on the stream both
routes run on (the median of --reps calls each).  The outputs of the two routes are compared column by column on the
same seeded inputs.

    python scripts/table_select_bench.py [--rows N] [--reps R] [--chunks 1,16,1000] [--out FILE]

Workloads:
  take_random   a random permutation of the rows (int64 indices);
  take_sorted   the sort_indices output of a clustered int32 key (runs of ~1000 rows, shuffled);
  filter_10 / filter_90   FilterTable with a mask selecting about 10 % / 90 % of the rows;
  sort_2keys    Sort by (int32 key, int64) end to end; the per-column route is SortIndices then pc.Take per column.
The per-column take of a chunked boolean column is refused (take concatenates a chunked column first, and the
concatenation does not take boolean chunks), so the per-column take and sort skip that column: their time covers three
columns, and `per_column_skipped` says so.
Modelled bytes of a take (`model_bytes`): the indices once, and per column one 32-byte sector per gathered row (random
rows of a column larger than L2; sorted indices need less), one value write and one validity bit per nullable column."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from arrow_go_b200 import _native as N  # noqa: E402
from arrow_go_b200 import compute as pc  # noqa: E402
from dictionary_encode_bench import HBM, card_info, timed  # noqa: E402

TYPES = [pc.INT64, pc.FLOAT64, pc.INT32, pc.BOOL]


def make_columns(n, rng):
    a = rng.integers(-10**12, 10**12, n, dtype=np.int64)
    b = rng.standard_normal(n)
    bv = rng.random(n) >= 0.1
    runs = np.arange(n, dtype=np.int64) // 1000
    perm = rng.permutation(runs[-1] + 1 if n else 0).astype(np.int32)
    c = perm[runs] if n else np.zeros(0, np.int32)
    d = rng.random(n) < 0.5
    return [(a, None), (b, bv), (c, None), (d, None)]


def chunked(v, ok, t, nchunks):
    cuts = np.linspace(0, v.size, nchunks + 1).astype(np.int64)
    return pc.Chunked([pc.Array.from_numpy(v[x:y], None if ok is None else ok[x:y], t) for x, y in zip(cuts, cuts[1:])], t)


def same(x, y):
    xv, xo, _ = x.to_numpy()
    yv, yo, _ = y.to_numpy()
    return bool(np.array_equal(xo, yo) and np.array_equal(xv[xo], yv[yo]))


def run_shape(n, nchunks, reps, host_cols, rng):
    cols = [chunked(v, ok, t, nchunks) for (v, ok), t in zip(host_cols, TYPES)]
    table = pc.Table(cols, n)
    usable = [i for i, t in enumerate(TYPES) if t != pc.BOOL]
    perm = pc.Array.from_numpy(rng.permutation(n).astype(np.int64))
    sorted_idx = pc.SortIndices(table, keys=[(2, pc.ASCENDING, pc.NULLS_AT_END)])
    mask10 = chunked(rng.random(n) < 0.1, None, pc.BOOL, nchunks)
    mask90 = chunked(rng.random(n) < 0.9, None, pc.BOOL, nchunks)
    keys = [(2, pc.ASCENDING, pc.NULLS_AT_END), (0, pc.DESCENDING, pc.NULLS_AT_END)]

    def per_column_sort():
        idx = pc.SortIndices(table, keys=keys)
        return [pc.Take(cols[i], idx) for i in usable]

    work = {
        "take_random": (lambda: pc.Take(table, perm), lambda: [pc.Take(cols[i], perm) for i in usable], n),
        "take_sorted": (lambda: pc.Take(table, sorted_idx), lambda: [pc.Take(cols[i], sorted_idx) for i in usable], n),
        "filter_10": (lambda: pc.FilterTable(table, mask10), lambda: [pc.Filter(cols[i], mask10) for i in range(4)], None),
        "filter_90": (lambda: pc.FilterTable(table, mask90), lambda: [pc.Filter(cols[i], mask90) for i in range(4)], None),
        "sort_2keys": (lambda: pc.Sort(table, keys), per_column_sort, n),
    }
    out = []
    for name, (new, old, rows) in work.items():
        a, b = new(), old()   # warm-up, and the outputs that are compared
        acols = a.columns()
        filt = name.startswith("filter")
        match = all(same(acols[i], b[k]) for k, i in enumerate(usable if not filt else range(4)))
        t_new, t_old = [], []
        for _ in range(reps):
            t_new.append(timed(new, 1))
            t_old.append(timed(old, 1))
        rows = len(a)
        mbytes = rows * 8 + sum(rows * 32 + rows * (4 if t == pc.INT32 else 8 if t != pc.BOOL else 0.125) for t in TYPES) + rows / 8
        out.append({"workload": name, "chunks": nchunks, "rows": n, "out_rows": rows, "table_ms": round(float(np.median(t_new)), 3),
                    "per_column_ms": round(float(np.median(t_old)), 3), "outputs_match": match,
                    "per_column_skipped": [] if filt else ["bool"],
                    "model_bytes": int(mbytes), "floor_ms": round(mbytes / HBM * 1e3, 3)})
        print(json.dumps(out[-1]), flush=True)
        del a, b
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--chunks", default="1,16,1000")
    ap.add_argument("--out")
    a = ap.parse_args()
    N.call("ag_init", 0)
    rng = np.random.default_rng(20261017)
    host_cols = make_columns(a.rows, rng)
    results = {"card": card_info(), "cases": []}
    for c in [int(x) for x in a.chunks.split(",")]:
        results["cases"] += run_shape(a.rows, c, a.reps, host_cols, rng)
    faster = [f"{r['workload']}/{r['chunks']}" for r in results["cases"] if r["per_column_ms"] < r["table_ms"]]
    results["per_column_faster"] = faster
    text = json.dumps(results, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
