#!/usr/bin/env python
"""BYTE_ARRAY page encoding on the device (ag_parquet_byte_array_encode_dev, csrc/pq_encode.cu) from LargeBinary columns
(int64 offsets) in pages of about 1 MiB of value bytes, page boundaries chosen from the offsets as a writer would:
  short        random strings of 0-32 bytes                    PLAIN, DELTA_LENGTH_BYTE_ARRAY
  short_null   the same with 10 % nulls                        PLAIN, DELTA_LENGTH_BYTE_ARRAY
  keys         sorted 48-byte keys behind a 36-byte prefix     DELTA_BYTE_ARRAY
  kib          ~1 KiB random values                            PLAIN

  python scripts/parquet_bytearray_encode_bench.py [--values 20000000] [--steps K] [--warmup W] [--out FILE]

Prints one JSON line: per case the time per call (CUDA events around K calls after W warm-up calls; the call
synchronises once, after its checking pass), the modelled HBM bytes (offsets, validity and data read once, output
written once: the single-pass floor; and the design's own traffic: offsets and validity read by every pass, DELTA's
dense length scratch written and read, DELTA_BYTE_ARRAY's data read twice) over the HBM peak, a device-to-device copy
of the same data bytes timed in the same run (the floor for moving them), a torch.profiler split of the device time per
kernel (a run of its own after the timed one), and pyarrow's single-thread host encode of
the same column (CPU context, not a baseline).  Every case checks three pages against the Python restatement.  The
card name and power limit are read in the same run."""
import argparse
import io
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

PAGE_BYTES = 1 << 20


def corpus(rng, kind, n):
    """-> (offsets int64, data uint8, valid bool or None)"""
    if kind == "keys":
        nums = np.sort(rng.integers(0, 10 ** 12, n))
        digits = np.zeros((n, 12), np.uint8)
        x = nums.copy()
        for k in range(11, -1, -1):
            digits[:, k] = 48 + x % 10
            x //= 10
        prefix = np.frombuffer(b"warehouse/orders/region=emea/custom-", np.uint8)
        data = np.concatenate([np.broadcast_to(prefix, (n, 36)), digits], axis=1).ravel()
        return np.arange(n + 1, dtype=np.int64) * 48, np.ascontiguousarray(data), None
    lens = rng.integers(0, 33, n) if kind.startswith("short") else rng.integers(768, 1281, n)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    data = rng.integers(0, 256, int(offsets[-1]), dtype=np.uint8)
    valid = rng.random(n) >= 0.1 if kind == "short_null" else None
    return offsets, data, valid


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--values", type=int, default=20_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import ctypes as C

    import pyarrow as pa
    import pyarrow.parquet as pq
    import torch
    from torch.profiler import ProfilerActivity, profile

    import pq_bytearray_ref as B
    from arrow_go_b200 import _native as N
    from arrow_go_b200.device import DeviceBuffer, Event
    from bench import peaks
    from parquet_pages_bench import card, kernel_ms

    N.call("ag_init", 0)
    peak, peak_kind = peaks()
    rng = np.random.default_rng(0xBA)
    res = {"values": args.values, "page_value_bytes": PAGE_BYTES, "offsets": "int64", "peak_gbs": peak, "peak_kind": peak_kind,
           **card(), "timing": f"CUDA events around {args.steps} calls after {args.warmup} warm-up calls"}
    names = {B.PLAIN: "PLAIN", B.DELTA_LENGTH_BYTE_ARRAY: "DELTA_LENGTH_BYTE_ARRAY", B.DELTA_BYTE_ARRAY: "DELTA_BYTE_ARRAY"}
    expect = {B.PLAIN: B.plain_encode, B.DELTA_LENGTH_BYTE_ARRAY: B.dlba_encode, B.DELTA_BYTE_ARRAY: B.dba_encode}
    cases = [("short", [B.PLAIN, B.DELTA_LENGTH_BYTE_ARRAY], args.values), ("short_null", [B.PLAIN, B.DELTA_LENGTH_BYTE_ARRAY], args.values),
             ("keys", [B.DELTA_BYTE_ARRAY], args.values), ("kib", [B.PLAIN], args.values // 10)]

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

    for kind, encs, n in cases:
        offsets, data, valid = corpus(rng, kind, n)
        cuts = np.unique(np.concatenate([[0], np.searchsorted(offsets, np.arange(PAGE_BYTES, int(offsets[-1]), PAGE_BYTES)), [n]]))
        spans = [(int(a), int(b - a)) for a, b in zip(cuts[:-1], cuts[1:]) if b > a]
        vb = None if valid is None else np.packbits(valid, bitorder="little")
        d_off, d_data = DeviceBuffer(offsets.nbytes + 64), DeviceBuffer(data.nbytes + 64)
        N.call("ag_upload", d_off.ptr, offsets.ctypes.data, offsets.nbytes, None)
        N.call("ag_upload", d_data.ptr, data.ctypes.data, data.nbytes, None)
        d_valid = None
        if vb is not None:
            d_valid = DeviceBuffer(vb.nbytes + 64)
            N.call("ag_upload", d_valid.ptr, vb.ctypes.data, vb.nbytes, None)
        nvalid = n if valid is None else int(valid.sum())
        vbytes = int(offsets[-1]) if valid is None else int(((offsets[1:] - offsets[:-1]) * valid).sum())

        # the floor: a device-to-device copy of the same data bytes
        src = torch.empty(data.nbytes, dtype=torch.uint8, device="cuda")
        dst = torch.empty_like(src)
        for _ in range(args.warmup):
            dst.copy_(src)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.steps):
            dst.copy_(src)
        t1.record()
        torch.cuda.synchronize()
        copy_ms = t0.elapsed_time(t1) / args.steps
        del src, dst
        torch.cuda.empty_cache()

        for enc in encs:
            caps = []
            for i0, k in spans:
                s = C.c_int64()
                N.call("ag_parquet_byte_array_max_size", enc, k, int(offsets[i0 + k] - offsets[i0]), C.byref(s))
                caps.append(s.value)
            outs = np.concatenate([[0], np.cumsum(caps)])
            pages = [(i0, k, int(o), c) for (i0, k), o, c in zip(spans, outs, caps)]
            tbl = N.enc_page_table(pages)
            d_out, d_len = DeviceBuffer(int(outs[-1]) + 64), DeviceBuffer(8 * len(pages) + 64)
            call = lambda: N.call("ag_parquet_byte_array_encode_dev", enc, 8, d_off.ptr, d_data.ptr,   # noqa: E731
                                  None if d_valid is None else d_valid.ptr, tbl, len(pages), d_out.ptr, d_len.ptr, None, None)
            ms = timed(call)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:        # a separate run: tracing slows the host
                for _ in range(args.steps):
                    call()
                torch.cuda.synchronize()
            kern = kernel_ms(prof, args.steps)
            lens = d_len.to_numpy(np.int64, len(pages), 0)
            for p in (0, len(pages) // 2, len(pages) - 1):           # three pages against the restatement
                i0, k, o, _ = pages[p]
                vals = [data[offsets[s]:offsets[s + 1]].tobytes() for s in range(i0, i0 + k) if valid is None or valid[s]]
                assert d_out.to_numpy(np.uint8, int(lens[p]), o).tobytes() == expect[enc](vals), (kind, enc, p)
            out_bytes = int(lens.sum())
            floor = 8 * (n + 1) + (0 if vb is None else vb.nbytes) + vbytes + out_bytes
            passes = 2 if enc == B.PLAIN else 3
            design = passes * (8 * (n + 1) + (0 if vb is None else vb.nbytes)) + vbytes + out_bytes
            if enc != B.PLAIN:
                design += (8 if enc == B.DELTA_BYTE_ARRAY else 4) * nvalid * 2   # dense lengths: written, then read
            if enc == B.DELTA_BYTE_ARRAY:
                design += vbytes + 4 * nvalid                                 # prefix compares; prefixes re-read
            # pyarrow, one host thread, the same column
            arr = pa.LargeBinaryArray.from_buffers(pa.large_binary(), n, [None if vb is None else pa.py_buffer(vb),
                                                                         pa.py_buffer(offsets), pa.py_buffer(data)])
            tbl_pa = pa.table({"c": arr})
            t = time.perf_counter()
            pq.write_table(tbl_pa, io.BytesIO(), use_dictionary=False, column_encoding={"c": names[enc]}, compression="NONE",
                           data_page_size=PAGE_BYTES, data_page_version="2.0")
            cpu_ms = (time.perf_counter() - t) * 1e3
            res[f"{kind}_{names[enc]}"] = {
                "ms": ms, "pages": len(pages), "values": n, "valid_values": nvalid, "value_bytes": vbytes, "output_bytes": out_bytes,
                "floor_bytes": floor, "floor_gbs": floor / ms / 1e6, "floor_frac_of_peak": floor / ms / 1e6 / peak,
                "design_bytes": design, "design_gbs": design / ms / 1e6, "design_frac_of_peak": design / ms / 1e6 / peak,
                "kernels_ms_per_call": kern, "kernels_total_ms": sum(kern.values()),
                "d2d_copy_of_data_ms": copy_ms, "ms_over_d2d_copy": ms / copy_ms,
                "cpu_context_pyarrow_1_thread_write_ms": cpu_ms,
                "cpu_context_note": "pyarrow pq.write_table of the same column (NONE, v2 pages, includes levels, headers and footer), one thread, the GPU host's CPU; context, not a baseline"}
            for b in (d_out, d_len):
                b.free()
        for b in (d_off, d_data, d_valid):
            if b is not None:
                b.free()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
