"""Fused expression evaluation against the node-by-node CallFunction chain, at 100M rows on one GPU.

    python scripts/expr_bench.py [--rows N] [--repeats R] [--profile]

Workloads (the same trees for both routes, timed alternately in one run, median of R repeats):
  E0  negate_unchecked(a)                                   float64: one op, the interpreter's own overhead against
                                                            the single-op kernel (which is the node-by-node route)
  E1  greater(add(multiply(a, b), c), d)                    float64
  E2  and_kleene(greater(x, 0), less(y, z))                 int32, 10 % nulls
  E3  add(multiply(cast(i32, float64), 1.5), f64)           promotion and a literal
  E4  add(multiply(a, 3), b)                                checked int64
  E2 on a table of 16 and of 1000 chunks
The modelled bytes are every referenced column read once plus the output (values or bits, and validity bits); the
share is those bytes over the fused time, against 3.35 TB/s.  --profile adds, per workload, the device time of
every kernel of one fused call and one node-by-node chain (torch.profiler, a separate pass after the timing).  The
card and its power limit are read in the same run.
Writes scripts/results/expr_bench_h100_<power>.json.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from arrow_go_b200 import compute as pc  # noqa: E402

PEAK = 3.35e12
W = {pc.INT32: 4, pc.INT64: 8, pc.FLOAT64: 8}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if out.returncode != 0:
        raise SystemExit("no GPU: this benchmark measures on the device only")
    name, power = [x.strip() for x in out.stdout.splitlines()[0].split(",")]
    return name, power


def col(rng, t, n, nulls, chunks=1):
    if t == pc.FLOAT64:
        v = rng.standard_normal(n)
    elif t == pc.INT64:
        v = rng.integers(-1000, 1000, n).astype(np.int64)
    else:
        v = rng.integers(-1000, 1000, n).astype(np.int32)
    valid = rng.random(n) >= nulls if nulls else None
    arr = pc.Array.from_numpy(v, valid=valid, type_id=t)
    if chunks == 1:
        return arr
    cuts = np.linspace(0, n, chunks + 1).astype(np.int64)
    return pc.Chunked([arr.slice(int(a), int(b - a)) for a, b in zip(cuts[:-1], cuts[1:])], t)


def workloads(rng, n):
    f = [col(rng, pc.FLOAT64, n, 0) for _ in range(4)]
    i = [col(rng, pc.INT32, n, 0.1) for _ in range(3)]
    e1 = (("greater", [("add", [("multiply", [0, 1]), 2]), 3]), f, [pc.FLOAT64] * 4, pc.BOOL)
    e2 = (("and_kleene", [("greater", [0, ("lit", 0, pc.INT32)]), ("less", [1, 2])]), i, [pc.INT32] * 3, pc.BOOL)
    mix = [col(rng, pc.INT32, n, 0), col(rng, pc.FLOAT64, n, 0)]
    e3 = (("add", [("multiply", [("cast", 0, pc.FLOAT64), ("lit", 1.5, pc.FLOAT64)]), 1]), mix, [pc.INT32, pc.FLOAT64], pc.FLOAT64)
    g = [col(rng, pc.INT64, n, 0) for _ in range(2)]
    e4 = (("add", [("multiply", [0, ("lit", 3, pc.INT64)]), 1]), g, [pc.INT64] * 2, pc.INT64)
    e0 = (("negate_unchecked", [0]), f[:1], [pc.FLOAT64], pc.FLOAT64)
    out = {"E0": e0, "E1": e1, "E2": e2, "E3": e3, "E4": e4}
    for k in (16, 1000):
        out[f"E2_table_{k}"] = (e2[0], [col(rng, pc.INT32, n, 0.1, k) for _ in range(3)], e2[2], pc.BOOL)
    return out


def to_expr(t):
    if isinstance(t, int):
        return pc.Field(t)
    if t[0] == "lit":
        return pc.Literal(t[1], t[2])
    if t[0] == "cast":
        return pc.CastExpr(to_expr(t[1]), t[2])
    return pc.Call(t[0], [to_expr(a) for a in t[1]])


def chain(t, cols):
    if isinstance(t, int):
        return cols[t]
    if t[0] == "lit":
        return pc.Scalar(t[1], t[2])
    if t[0] == "cast":
        return pc.Cast(chain(t[1], cols), t[2])
    return pc.CallFunction(t[0], [chain(a, cols) for a in t[1]])


def has_validity(c):
    return any(ch.has_validity for ch in c.chunks()) if c.kind == pc.KIND_CHUNKED else c.has_validity


def device_split(fn, sync):
    """Seconds of device time per kernel (and copy / memset) of one call."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        sync()
    split = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = e.name.replace("(anonymous namespace)::", "").split("(")[0].split("<")[0].split("::")[-1].strip()
            split[name] = split.get(name, 0.0) + e.device_time_total / 1e6
    return split


def timed(fn, sync):
    sync()
    t0 = time.perf_counter()
    r = fn()
    sync()
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    name, power = card()
    sync = torch.cuda.synchronize
    rng = np.random.default_rng(7)
    n = a.rows
    res = {"card": name, "power_limit": power, "rows": n, "peak_bytes_per_s": PEAK, "workloads": {}}
    for key, (tree, cols, types, out_t) in workloads(rng, n).items():
        data = pc.Table(cols) if isinstance(cols[0], pc.Datum) and cols[0].kind == pc.KIND_CHUNKED else pc.RecordBatch(cols)
        expr = to_expr(tree)
        fused_fn = lambda: pc.ExecuteScalarExpression(expr, data)  # noqa: E731
        chain_fn = lambda: chain(tree, cols)  # noqa: E731
        timed(fused_fn, sync), timed(chain_fn, sync)   # warm both routes
        tf, tc = [], []
        for _ in range(a.repeats):
            tf.append(timed(fused_fn, sync)[0])
            tc.append(timed(chain_fn, sync)[0])
        out_bytes = n / 8 if out_t == pc.BOOL else n * W[out_t]
        model = sum(W[t] for t in types) * n + out_bytes + n / 8 + sum(n / 8 for c in cols if has_validity(c))
        fm, cm = statistics.median(tf), statistics.median(tc)
        row = {"fused_s": fm, "node_by_node_s": cm, "speedup": cm / fm, "modelled_bytes": model,
               "fused_share_of_hbm": model / fm / PEAK}
        if a.profile:
            row["fused_profile_s"] = device_split(fused_fn, sync)
            row["node_by_node_profile_s"] = device_split(chain_fn, sync)
            k = row["fused_profile_s"].get("expr_eval_kernel", 0.0)
            row["expr_eval_kernel_share_of_hbm"] = model / k / PEAK if k else None
        res["workloads"][key] = row
        print(key, json.dumps(row), flush=True)
    watts = power.split()[0].split(".")[0]
    path = a.out or os.path.join(ROOT, "scripts", "results", f"expr_bench_h100_{watts}w.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"card": name, "power_limit": power, "written": os.path.relpath(path, ROOT)}))


if __name__ == "__main__":
    main()
