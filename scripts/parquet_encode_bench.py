"""Device Parquet page encoders on 100M values in pages of 2^19 values: call time from device events, the split by
kernel from torch.profiler (a separate run), and the share of 3.35 TB/s on the modelled bytes (input read once plus
encoded bytes written once).  Prints one JSON document and writes it to --out.

  python scripts/parquet_encode_bench.py --out scripts/results/parquet_encode_bench_h100_<power>.json
"""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from arrow_go_b200 import _native as N  # noqa: E402

HBM = 3.35e12
N_VALUES = 100_000_000
PAGE = 1 << 19


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return name, power


def pages_of(n, bound):
    pages, o = [], 0
    for i0 in range(0, n, PAGE):
        k = min(PAGE, n - i0)
        cap = bound(k)
        pages.append((i0, k, o, cap))
        o += cap
    return pages, o


def rle_bound(bw, form, n):
    s = C.c_int64()
    N.call("ag_parquet_rle_max_size", bw, form, n, C.byref(s))
    return s.value


def delta_bound(w, block, mini, n):
    s = C.c_int64()
    N.call("ag_parquet_delta_max_size", w, block, mini, n, C.byref(s))
    return s.value


def workloads(g):
    n = N_VALUES
    u17 = torch.randint(0, 1 << 17, (n,), device="cuda", dtype=torch.int32, generator=g)
    lens = torch.randint(1, 65, (n // 16,), device="cuda", generator=g)
    reps = torch.repeat_interleave(torch.randint(0, 1 << 17, (lens.numel(),), device="cuda", dtype=torch.int32, generator=g), lens)[:n]
    nulls = torch.rand(n, device="cuda", generator=g) >= 0.1
    runs = torch.repeat_interleave(torch.rand(n // 1000, device="cuda", generator=g) >= 0.3, 1000)[:n]
    bools = torch.rand(n, device="cuda", generator=g) < 0.5

    def bitmap(b):
        w = b.view(-1, 8).to(torch.uint8) << torch.arange(8, device="cuda", dtype=torch.uint8)
        return w.sum(1, dtype=torch.uint8).contiguous()

    ts = (1_700_000_000_000_000_000 + torch.cumsum(torch.randint(0, 5_000_000, (n,), device="cuda", generator=g), 0)).contiguous()
    i32 = torch.randint(-(1 << 31), 1 << 31, (n,), device="cuda", dtype=torch.int64, generator=g).to(torch.int32)
    W = N.PQ_RLE_WIDTH
    return [
        ("dict_indices_17bit_uniform", "rle", (17, W, N.PQ_RLE_IN_U32), u17, 4 * n),
        ("dict_indices_17bit_clustered", "rle", (17, W, N.PQ_RLE_IN_U32), reps.contiguous(), 4 * n),
        ("def_levels_bitmap_10pct_nulls", "rle", (1, N.PQ_RLE_BARE, N.PQ_RLE_IN_BITMAP), bitmap(nulls), n / 8),
        ("def_levels_bitmap_null_runs", "rle", (1, N.PQ_RLE_BARE, N.PQ_RLE_IN_BITMAP), bitmap(runs), n / 8),
        ("booleans_rle", "rle", (1, N.PQ_RLE_LEN4, N.PQ_RLE_IN_BITMAP), bitmap(bools), n / 8),
        ("delta_int64_timestamps_128_4", "delta", (8, 128, 4), ts, 8 * n),
        ("delta_int64_timestamps_256_4", "delta", (8, 256, 4), ts, 8 * n),
        ("delta_int32_uniform_128_4", "delta", (4, 128, 4), i32, 4 * n),
    ]


def setup(kind, head, n):
    bound = (lambda k: rle_bound(head[0], head[1], k)) if kind == "rle" else (lambda k: delta_bound(*head, k))
    pages, total = pages_of(n, bound)
    tbl = N.enc_page_table(pages)
    out = torch.empty(total + 64, device="cuda", dtype=torch.uint8)
    lens = torch.zeros(len(pages), device="cuda", dtype=torch.int64)
    return pages, tbl, out, lens


def call(kind, head, vals, tbl, npages, out, lens):
    if kind == "rle":
        N.call("ag_parquet_rle_encode_dev", *head, vals.data_ptr(), tbl, npages, out.data_ptr(), lens.data_ptr(), None, None)
    else:
        N.call("ag_parquet_delta_encode_dev", *head, vals.data_ptr(), tbl, npages, out.data_ptr(), lens.data_ptr(), None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    N.call("ag_init", 0)
    name, power = card()
    g = torch.Generator(device="cuda")
    g.manual_seed(20261018)
    results = []
    for label, kind, head, vals, in_bytes in workloads(g):
        pages, tbl, out, lens = setup(kind, head, N_VALUES)
        call(kind, head, vals, tbl, len(pages), out, lens)             # warm-up
        times = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call(kind, head, vals, tbl, len(pages), out, lens)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3)
        enc = int(lens.sum().item())
        t = float(np.median(times))
        modelled = in_bytes + enc
        # the split by kernel, in a run of its own
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            call(kind, head, vals, tbl, len(pages), out, lens)
            torch.cuda.synchronize()
        kernels = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                m = re.search(r"(\w+_kernel)", ev.name)
                key = m.group(1) if m else ev.name.strip()
                kernels[key] = kernels.get(key, 0.0) + ev.device_time_total / 1e6
        results.append({"workload": label, "pages": len(pages), "values": N_VALUES, "input_bytes": int(in_bytes),
                        "encoded_bytes": enc, "call_s_median": t, "call_s_min": float(min(times)),
                        "modelled_bytes": int(modelled), "hbm_share": modelled / t / HBM,
                        "kernel_s": {k: round(v, 7) for k, v in kernels.items()}})
        print(json.dumps(results[-1]), flush=True)
        del out, lens
    doc = {"card": name, "power_limit": power, "hbm_peak_bytes_per_s": HBM, "page_values": PAGE, "results": results}
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")


if __name__ == "__main__":
    main()
