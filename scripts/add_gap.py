#!/usr/bin/env python
"""Where a step of the chunked Add goes: the benchmark's workload (bench.py: 100M float64 rows, left chunks of 1M rows,
right chunks of 999,983 rows -> 200 spans, one ag_arith_binary_spans_dev call per step) on the same seeds, split into
kernel time, work between kernels and the spread of block finish times, next to bounds measured in the same run.

  python scripts/add_gap.py --out results.json [--label NAME] [--steps 20]

Writes one JSON file:
  headline      ms per step of `steps` back-to-back calls between two CUDA events, as bench.py times them
  trace         the same steps in a separate pass under torch.profiler (CUDA activities): time of each
                binary_spans_kernel, of each host-to-device copy, and the gap from one kernel's end to the next
                kernel's start; fixed_us_per_step = headline step time - mean kernel time
  bounds        measured on the same card in the same run, each as GB/s and as a share of the data sheet's 3.35 TB/s:
                the contiguous call (ag_arith_binary_dev over the 100M rows, 24 B/row), ag_copy_dev of 800 MB (one read
                and one write per byte) and ag_sum_i64_dev over 800 MB (reads only)
  block_finish  scripts/lab/add_spans_lab.cu, a copy of the kernel's tile loop that stamps %globaltimer at each block's
                start and end: spread of block finish times (last - first) as a share of the kernel's time, with tiles
                taken in grid-stride order and with tiles claimed from a counter (the kernel's schedule)
  gpu           name, power limit and max SM clock from nvidia-smi, read in the same run
"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import L_CHUNK, R_CHUNK, ROWS, spans_for  # noqa: E402

DATASHEET_GBS = 3350.0


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30)
    name, power, clock = [x.strip() for x in out.stdout.strip().split(",")]
    return {"name": name, "power_limit": power, "clocks_max_sm": clock}


def build_lab(tmp):
    nvcc = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    so = os.path.join(tmp, "add_spans_lab.so")
    subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC",
                    "-o", so, os.path.join(ROOT, "scripts", "lab", "add_spans_lab.cu")], check=True)
    lib = C.CDLL(so)
    lib.add_spans_lab_grid.restype = C.c_int
    lib.add_spans_lab_grid.argtypes = [C.c_longlong]
    lib.add_spans_lab_run.restype = C.c_int
    lib.add_spans_lab_run.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_int, C.c_void_p]
    return lib


def trace_steps(step, steps, tmp):
    """Kernel, copy and gap times (µs) of `steps` calls of `step` from a torch.profiler trace."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    path = os.path.join(tmp, "trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        events = json.load(f)["traceEvents"]
    kernels = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    copies = [e for e in events if e.get("cat") == "gpu_memcpy" and "HtoD" in e.get("name", "")]
    runtime = [e.get("name", "") for e in events if e.get("cat") == "cuda_runtime"]
    spans_k = [e for e in kernels if "binary_spans_kernel" in e["name"]]
    gaps = [b["ts"] - (a["ts"] + a["dur"]) for a, b in zip(spans_k, spans_k[1:])]
    return {
        "kernels_per_step": len(kernels) / steps,
        "kernel_names": sorted({e["name"] for e in kernels}),
        "kernel_us": [e["dur"] for e in spans_k],
        "kernel_us_mean": float(np.mean([e["dur"] for e in spans_k])),
        "htod_copies_per_step": len(copies) / steps,
        "htod_copy_bytes": sorted({int(e.get("args", {}).get("bytes", -1)) for e in copies}),
        "htod_copy_us_mean": float(np.mean([e["dur"] for e in copies])) if copies else 0.0,
        "gap_us": gaps,
        "gap_us_mean": float(np.mean(gaps)) if gaps else 0.0,
        "gap_us_median": float(np.median(gaps)) if gaps else 0.0,
        "runtime_calls_per_step": {n: runtime.count(n) / steps for n in sorted(set(runtime))},
        "first_start_to_last_end_us_per_step": (spans_k[-1]["ts"] + spans_k[-1]["dur"] - spans_k[0]["ts"]) / steps,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--label", default="")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--lab-reps", type=int, default=20)
    args = ap.parse_args()

    import torch
    torch.cuda.init()
    from arrow_go_b200 import _native as N
    from arrow_go_b200.device import DeviceBuffer, Event

    result = {"label": args.label, "gpu": gpu_info(), "rows": ROWS, "bytes_per_step": 24 * ROWS}
    N.call("ag_init", 0)
    rows = ROWS
    dl, dr, dout = DeviceBuffer(rows * 8), DeviceBuffer(rows * 8), DeviceBuffer(rows * 8)
    N.call("ag_generate_dev", 3, 0x94378165, -(1 << 20), 1 << 20, dl.ptr, rows, None)
    N.call("ag_generate_dev", 3, 0x94378166, -(1 << 20), 1 << 20, dr.ptr, rows, None)
    spans = spans_for(rows, L_CHUNK, R_CHUNK)
    table = N.span_table([(dl.ptr + 8 * pos, dr.ptr + 8 * pos, dout.ptr + 8 * pos, ln) for pos, ln in spans])
    result["spans"] = len(spans)

    def add_step():
        N.call("ag_arith_binary_spans_dev", N.FLOAT64, N.OP_ADD_CHECKED, N.SHAPE_AA, table, len(spans), None)

    def timed(fn, warm, steps):
        for _ in range(warm):
            fn()
        N.call("ag_stream_sync", None)
        e0, e1 = Event(), Event()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        e1.sync()
        N.call("ag_stream_sync", None)
        return e0.elapsed_ms(e1) / steps

    K, W = args.steps, args.warmup
    ms = timed(add_step, W, K)
    result["headline"] = {"ms_per_step": ms, "gbs": 24.0 * rows / ms / 1e6, "frac_of_datasheet": 24.0 * rows / ms / 1e6 / DATASHEET_GBS,
                          "how": f"{K} back-to-back ag_arith_binary_spans_dev calls between two CUDA events after {W} warm-up calls"}

    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(W):
            add_step()
        tr = trace_steps(add_step, K, tmp)
        tr["fixed_us_per_step"] = ms * 1e3 - tr["kernel_us_mean"]
        tr["fixed_share_of_step"] = tr["fixed_us_per_step"] / (ms * 1e3)
        result["trace"] = tr

        bounds = {}
        ms_c = timed(lambda: N.call("ag_arith_binary_dev", N.FLOAT64, N.OP_ADD_CHECKED, N.SHAPE_AA, dl.ptr, dr.ptr, dout.ptr, rows, None), W, K)
        bounds["contiguous_add"] = {"ms": ms_c, "bytes": 24 * rows}
        ms_cp = timed(lambda: N.call("ag_copy_dev", dout.ptr, dl.ptr, rows * 8, None), W, K)
        bounds["copy_800mb"] = {"ms": ms_cp, "bytes": 16 * rows}
        scal = DeviceBuffer(64)
        ms_s = timed(lambda: N.call("ag_sum_i64_dev", dl.ptr, rows, scal.ptr, None), W, K)
        bounds["sum_i64_800mb"] = {"ms": ms_s, "bytes": 8 * rows}
        for b in bounds.values():
            b["gbs"] = b["bytes"] / b["ms"] / 1e6
            b["frac_of_datasheet"] = b["gbs"] / DATASHEET_GBS
        result["bounds"] = {"note": "measured bounds on this card in this run, not the kernel's peak", **bounds}

        lab = build_lab(tmp)
        ls = (C.c_void_p * len(spans))(*[dl.ptr + 8 * pos for pos, _ in spans])
        rs = (C.c_void_p * len(spans))(*[dr.ptr + 8 * pos for pos, _ in spans])
        os_ = (C.c_void_p * len(spans))(*[dout.ptr + 8 * pos for pos, _ in spans])
        ns = (C.c_longlong * len(spans))(*[ln for _, ln in spans])
        tiles = sum(max(1, -(-ln // 2048)) for _, ln in spans)   # 2048-row tiles (16 KB of float64); every span here starts 16-byte aligned: no head row
        grid = lab.add_spans_lab_grid(tiles)
        result["block_finish"] = {"grid": grid, "tiles": tiles, "tiles_per_block_grid_stride": [tiles // grid, -(-tiles // grid)],
                                  "how": "globaltimer at each block's start and after its last tile; spread = (last finish - first finish) / "
                                         "(last finish - first start); median over the launches after the first"}
        for name, claimed in (("grid_stride", 0), ("claimed", 1)):
            stamps = np.zeros(args.lab_reps * grid * 2, dtype=np.uint64)
            rc = lab.add_spans_lab_run(ls, rs, os_, ns, len(spans), args.lab_reps, claimed, stamps.ctypes.data)
            if rc != 0:
                raise RuntimeError(f"add_spans_lab_run: CUDA error {rc}")
            st = stamps.reshape(args.lab_reps, grid, 2).astype(np.int64)
            spread, kern = [], []
            for rep in st[1:]:   # the first launch loads the module
                t0, t1 = rep[:, 0].min(), rep[:, 1].max()
                kern.append((t1 - t0) / 1e3)
                spread.append((t1 - rep[:, 1].min()) / (t1 - t0))
            result["block_finish"][name] = {"kernel_us_median": float(np.median(kern)), "finish_spread_share_median": float(np.median(spread)),
                                            "finish_spread_share": spread}
        N.call("ag_stream_sync", None)

    result["checkpoint"] = {"fixed_plus_grid_stride_spread_share": result["trace"]["fixed_share_of_step"] +
                            result["block_finish"]["grid_stride"]["finish_spread_share_median"]}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({k: result[k] for k in ("label", "gpu", "headline", "checkpoint")}))
    print(json.dumps({k: v for k, v in result["trace"].items() if k not in ("kernel_us", "gap_us")}))
    print(json.dumps(result["bounds"]))
    print(json.dumps({k: ({kk: vv for kk, vv in v.items() if kk != "finish_spread_share"} if isinstance(v, dict) else v)
                      for k, v in result["block_finish"].items()}))


if __name__ == "__main__":
    main()
