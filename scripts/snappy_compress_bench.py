#!/usr/bin/env python
"""SNAPPY page compression on the device (ag_parquet_snappy_compress_dev, csrc/snappy_encode.cu) over 190 pages of 2^19
values, the page bodies of the decode bench: (a) PLAIN int64 timestamps (increments in [0, 1000)), (b) 17-bit
dictionary indices in literal runs.

  python scripts/snappy_compress_bench.py [--pages 190] [--steps K] [--warmup W]

Prints one JSON line: for each case the device time per call (CUDA events around K calls after W warm-up calls; the
call does not synchronise), input GB/s, the output size against pyarrow's C++ Snappy of the same pages, pyarrow's
single-thread host compression time of the same pages in the same run (CPU context, not a baseline), the modelled bytes
(input read + output written + fragment scratch written and read back) over the HBM peak, and a torch.profiler split
between the match and assembly kernels.  Four distinct page bodies are reused round-robin; every page writes its own
output range.  Each case asserts that the device decompressor returns the input.  Writes nothing to disk."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=190)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import pyarrow as pa
    import torch
    from torch.profiler import ProfilerActivity, profile

    from arrow_go_b200 import _native as N
    from arrow_go_b200.device import DeviceBuffer, Event
    from bench import peaks
    from parquet_pages_bench import card, kernel_ms, rle_literal_page
    from snappy_ref import put_uvarint

    N.call("ag_init", 0)
    peak, peak_kind = peaks()
    rng = np.random.default_rng(0xC0DEC)
    per_page, n_pages = 1 << 19, args.pages
    res = {"pages": n_pages, "values_per_page": per_page, "peak_gbs": peak, "peak_kind": peak_kind, **card(),
           "timing": f"CUDA events around {args.steps} calls after {args.warmup} warm-up calls"}
    cases = {
        "snappy_compress_i64_timestamps": [(np.cumsum(rng.integers(0, 1000, per_page)) + (k << 40)).astype(np.int64).tobytes() for k in range(4)],
        "snappy_compress_dict_indices_17bit": [bytes([17]) + rle_literal_page(rng.integers(0, 100_000, per_page), 17) for _ in range(4)],
    }

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        N.call("ag_stream_sync", None)
        e0, e1 = Event(), Event()
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        e1.sync()
        return e0.elapsed_ms(e1) / args.steps

    for name, bodies in cases.items():
        blob = b"".join(bodies) + bytes(16)
        offs = np.cumsum([0] + [len(b) for b in bodies])
        pages, back, d, pos = [], [], 0, 0
        for p in range(n_pages):
            n = len(bodies[p % 4])
            pages.append((int(offs[p % 4]), n, d, 32 + n + n // 6))
            d += 32 + n + n // 6
        src = DeviceBuffer(len(blob) + 64)
        N.call("ag_upload", src.ptr, np.frombuffer(blob, np.uint8).ctypes.data, len(blob), None)
        dst, dw = DeviceBuffer(d + 64), DeviceBuffer(8 * n_pages + 64)
        tbl = N.compressed_table(pages)
        call = lambda: N.call("ag_parquet_snappy_compress_dev", src.ptr, tbl, n_pages, dst.ptr, dw.ptr, None)
        ms = timed(call)
        w = dw.to_numpy(np.int64, n_pages, 0)
        for p, k in zip(pages, w):
            back.append((p[2], int(k), pos, p[1]))
            pos += p[1]
        # the device decompressor returns the input
        dec = DeviceBuffer(pos + 64)
        N.call("ag_parquet_snappy_decompress_dev", dst.ptr, N.compressed_table(back), n_pages, dec.ptr, None, None)
        N.call("ag_stream_sync", None)
        assert dec.to_numpy(np.uint8, pos, 0).tobytes() == b"".join(bodies[p % 4] for p in range(n_pages)), name
        t0 = time.perf_counter()                                   # pyarrow, one thread, host memory
        py = [pa.compress(bodies[p % 4], codec="snappy", asbytes=False) for p in range(n_pages)]
        cpu_ms = (time.perf_counter() - t0) * 1e3
        inp, out, py_out = pos, int(w.sum()), sum(b.size for b in py)
        scratch = 2 * (out - sum(len(put_uvarint(p[1])) for p in pages))   # fragments: written, then read back
        modelled = inp + out + scratch
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                call()
            torch.cuda.synchronize()
        res[name] = {"ms": ms, "input_bytes": inp, "output_bytes": out, "input_gbs": inp / ms / 1e6,
                     "pyarrow_output_bytes": py_out, "output_over_pyarrow": out / py_out, "compression_ratio": inp / out,
                     "modelled_bytes": modelled, "modelled_gbs": modelled / ms / 1e6, "frac_of_peak": modelled / ms / 1e6 / peak,
                     "kernels_ms_per_call": kernel_ms(prof, args.steps),
                     "cpu_context_pyarrow_1_thread_ms": cpu_ms,
                     "cpu_context_note": "pyarrow pa.compress of the same pages, one thread, host memory, the GPU host's CPU; context, not a baseline"}
        for b in (src, dst, dw, dec):
            b.free()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
