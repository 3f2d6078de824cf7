#!/usr/bin/env python
"""Parquet page decode on the device (include/arrowgpu.h, csrc/fixed.cu and csrc/rle.cu) at ~100M values over 2^19-value (~1 MB) pages.

  python scripts/parquet_pages_bench.py [--values N] [--steps K] [--warmup W] [--profile]

Prints one JSON line: for each case the time per call (CUDA events around K device-resident calls after W warm-up
calls), the algorithmic bytes (encoded bytes read + values written + validity bits read: what a single pass has to
move) and their share of the HBM peak, with the card's name and power limit.  Each call ends in one stream
synchronisation (per-page error codes), which the times include.  Four distinct page bodies are reused round-robin;
every page writes its own output range.  Writes nothing to disk.

--bytearray runs only the BYTE_ARRAY cases (ag_parquet_byte_array_decode_dev, csrc/byte_array.cu): time, share of the HBM
peak, and a torch.profiler split of the device time over the three stages (values, offsets, bytes).

--fixed runs only the BOOLEAN and fixed-width cases (ag_parquet_bool_decode_dev / ag_parquet_fixed_decode_dev,
csrc/fixed.cu): time, share of the HBM peak and a torch.profiler split per kernel.

--profile runs only the DELTA_BINARY_PACKED, SNAPPY, ZSTD, GZIP and LZ4_RAW cases, under torch.profiler, and reports the
device time per call of each kernel (the delta block walk against the value passes, the Snappy parse against the
execute, the ZSTD walk / literals / sequences / resolve / execute / checksum kernels, the GZIP inflate / execute / CRC32
kernels, the LZ4 parse against the execute) instead.

The SNAPPY, ZSTD, GZIP and LZ4_RAW cases also print pyarrow's single-thread host decompression of the same pages on this machine's CPU: a CPU
context line, not a baseline of the kernel.
"""
import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # pq_delta_ref.delta_encode: the DELTA_BINARY_PACKED encoder, numpy per block


def rle_literal_page(idx, bw):
    """canonical literal-only hybrid stream of `idx` (a multiple of 8 values): runs of 63 groups, header byte 127"""
    bits = ((idx[:, None] >> np.arange(bw)) & 1).astype(np.uint8).ravel()
    payload = np.packbits(bits, bitorder="little").tobytes()
    out = bytearray()
    for r in range(0, idx.size, 504):
        groups = min(504, idx.size - r) // 8
        out.append(groups << 1 | 1)
        out += payload[r * bw // 8:r * bw // 8 + groups * bw]
    return bytes(out)


def rle_repeated_page(rng, n, bw, hi):
    """repeated runs only (clustered indices): run lengths 8..200, values uniform in [0, hi)"""
    out, left = bytearray(), n
    while left:
        k = min(left, int(rng.integers(8, 201)))
        v = int(rng.integers(0, hi))
        h = k << 1
        while h >= 0x80:
            out.append(h & 0x7F | 0x80)
            h >>= 7
        out.append(h)
        out += v.to_bytes((bw + 7) // 8, "little")
        left -= k
    return bytes(out)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip().split(", ")
        return {"card": out[0], "power_limit": out[1]}
    except Exception:
        return {"card": None, "power_limit": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--values", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--bytearray", action="store_true")
    ap.add_argument("--fixed", action="store_true")
    args = ap.parse_args()

    from arrow_go_b200 import _native as N
    from arrow_go_b200.device import DeviceBuffer, Event
    from bench import peaks

    N.call("ag_init", 0)
    peak, peak_kind = peaks()
    rng = np.random.default_rng(0xDEC0DE)
    per_page = 1 << 19
    n_pages = max(1, args.values // per_page)
    n = n_pages * per_page
    res = {"values": n, "pages": n_pages, "values_per_page": per_page, "peak_gbs": peak, "peak_kind": peak_kind, **card(),
           "timing": f"CUDA events around {args.steps} calls after {args.warmup} warm-up calls, one stream synchronisation per call included"}

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

    def upload(arr):
        arr = np.ascontiguousarray(arr)
        b = DeviceBuffer(arr.nbytes + 64)
        N.call("ag_upload", b.ptr, arr.ctypes.data, arr.nbytes, None)
        return b

    def page_set(bodies):
        blob = b"".join(bodies) + bytes(16)
        offs = np.cumsum([0] + [len(x) for x in bodies])
        pages = [(int(offs[p % 4]), len(bodies[p % 4]), per_page, p * per_page) for p in range(n_pages)]
        enc = sum(len(bodies[p % 4]) for p in range(n_pages))
        return upload(np.frombuffer(blob, np.uint8)), N.page_table(pages), enc

    def line(ms, ab, enc, note):
        return {"ms": ms, "values_per_s": n / ms * 1e3, "algorithmic_bytes": ab, "encoded_bytes": enc,
                "gbs": ab / ms / 1e6, "frac": ab / ms / 1e6 / peak, "note": note}

    if args.bytearray:
        res = {"peak_gbs": peak, "peak_kind": peak_kind, **card(), "timing": res["timing"]}
        res.update(bytearray_cases(args, N, np.random.default_rng(0xB17E), timed, upload, DeviceBuffer))
        print(json.dumps(res), flush=True)
        return
    if args.fixed:
        res = {"peak_gbs": peak, "peak_kind": peak_kind, **card(), "timing": res["timing"]}
        res.update(fixed_cases(args, N, np.random.default_rng(0xF1ED), timed, upload, DeviceBuffer, peak, n_pages, per_page))
        print(json.dumps(res), flush=True)
        return
    dout = DeviceBuffer(8 * n + 64)
    if args.profile:
        res.update(delta_cases(args, N, rng, n, n_pages, per_page, timed, upload, page_set, line, dout, DeviceBuffer, profile=True))
        res.update(snappy_cases(args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer, profile=True))
        res.update(zstd_cases(args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer, profile=True))
        res.update(gzip_cases(args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer, profile=True))
        res.update(lz4_raw_cases(args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer, profile=True))
        print(json.dumps(res), flush=True)
        return
    dictionary = rng.integers(-(1 << 62), 1 << 62, 100_000)
    ddict = upload(dictionary)
    valid = rng.random(n) >= 0.1
    dvalid = upload(np.packbits(valid, bitorder="little"))
    dec, bad = DeviceBuffer(8 * n_pages + 64), DeviceBuffer(64)

    # dictionary indices, bit width 17, literal runs
    lit = [bytes([17]) + rle_literal_page(rng.integers(0, 100_000, per_page), 17) for _ in range(4)]
    dblob, tbl, enc = page_set(lit)
    for label, vp, nbits in (("required", None, 0), ("10pct_nulls", dvalid.ptr, n)):
        ms = timed(lambda: N.call("ag_parquet_dict_decode_dev", 8, ddict.ptr, 100_000, dblob.ptr, tbl, n_pages, vp, dout.ptr, dec.ptr, bad.ptr, None))
        res[f"parquet_dict_decode_i64_{label}"] = line(ms, enc + 8.0 * n + nbits / 8.0, enc,
                                                       "100K-entry int64 dictionary, 17-bit indices in literal runs of 504; dictionary gather from L2")
    dblob.free()
    # clustered indices: repeated runs of 8..200 values
    rep = [bytes([17]) + rle_repeated_page(rng, per_page, 17, 100_000) for _ in range(4)]
    dblob, tbl, enc = page_set(rep)
    ms = timed(lambda: N.call("ag_parquet_dict_decode_dev", 8, ddict.ptr, 100_000, dblob.ptr, tbl, n_pages, None, dout.ptr, dec.ptr, bad.ptr, None))
    res["parquet_dict_decode_i64_runs"] = line(ms, enc + 8.0 * n, enc, "required column, repeated runs only (mean ~104 values)")
    dblob.free()
    # definition levels, bit width 1, 10 % nulls (literal runs: 1 bit per level)
    lv = [rle_literal_page((rng.random(per_page) >= 0.1).astype(np.int64), 1) for _ in range(4)]
    dblob, tbl, enc = page_set(lv)
    ms = timed(lambda: N.call("ag_parquet_levels_decode_dev", 1, N.PQ_LEVELS_V2_RLE, dblob.ptr, tbl, n_pages, dout.ptr, dec.ptr, None))
    res["parquet_levels_decode"] = line(ms, enc + 2.0 * n, enc, "max_level 1 (bit width 1), 10 % nulls, literal runs; int16 levels out")
    dblob.free(); ddict.free(); dvalid.free(); dec.free(); bad.free()
    res.update(delta_cases(args, N, rng, n, n_pages, per_page, timed, upload, page_set, line, dout, DeviceBuffer))
    res.update(snappy_cases(args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer))
    res.update(zstd_cases(args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer))
    res.update(gzip_cases(args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer))
    res.update(lz4_raw_cases(args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer))
    dout.free()
    print(json.dumps(res), flush=True)


def kernel_ms(prof, steps):
    """device ms per call of each project kernel in a torch.profiler capture"""
    import torch
    kern = {}
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            m = re.search(r"(delta_\w+_kernel|pq_\w+_kernel|snappy_\w+_kernel|zstd_\w+_kernel|gz_\w+_kernel|lz4_\w+_kernel|lz_exec_kernel|ba_\w+_kernel|fx_\w+_kernel)(<[^>]*>)?", ev.key)
            short = (m.group(1) + (m.group(2) or "")) if m else ev.key.strip()
            us = getattr(ev, "device_time_total", None) or ev.cuda_time_total
            kern[short] = kern.get(short, 0.0) + us / 1e3 / steps
    return kern


def delta_cases(args, N, rng, n, n_pages, per_page, timed, upload, page_set, line, dout, DeviceBuffer, profile=False):
    """DELTA_BINARY_PACKED: (a) int64 timestamps (sorted, increments uniform in [0, 1000), 256/4 blocks), required;
    (b) the same with 10 % nulls; (c) int32 uniform random values (128/4 blocks, every miniblock 32 bits wide);
    (d) ag_parquet_plain_decode_spaced_dev writing the output of (b), the floor for writing it."""
    import pq_delta_ref as R
    out = {}
    valid = rng.random(n) >= 0.1
    dvalid = upload(np.packbits(valid, bitorder="little"))
    dec = DeviceBuffer(8 * n_pages + 64)
    ts = [R.delta_encode(np.cumsum(rng.integers(0, 1000, per_page)) + (k << 40), 8, 256, 4) for k in range(4)]
    rnd = [R.delta_encode(rng.integers(-(1 << 31), 1 << 31, per_page), 4, 128, 4) for _ in range(4)]
    plain = [rng.integers(-(1 << 62), 1 << 62, per_page).tobytes() for _ in range(4)]
    runs = []
    dblob, tbl, enc = page_set(ts)
    runs.append(("parquet_delta_decode_i64_timestamps_required", 8, dblob, tbl, None, enc + 8.0 * n, enc,
                 "int64 sorted, increments uniform in [0, 1000): 256/4 blocks, ~10-bit miniblocks; dense output"))
    runs.append(("parquet_delta_decode_i64_timestamps_10pct_nulls", 8, dblob, tbl, dvalid.ptr, enc + 8.0 * n + n / 8.0, enc,
                 "the same pages, 10 % nulls: each page's first ~90 % of values spaced out"))
    rblob, rtbl, renc = page_set(rnd)
    runs.append(("parquet_delta_decode_i32_random", 4, rblob, rtbl, None, renc + 4.0 * n, renc,
                 "int32 uniform random: 128/4 blocks, every miniblock 32 bits wide (the most encoded bytes)"))
    if profile:
        import torch
        from torch.profiler import ProfilerActivity, profile as tprofile
        for name, w, b, t, vp, ab, e, note in runs:
            fn = (lambda w=w, b=b, t=t, vp=vp: N.call("ag_parquet_delta_decode_dev", w, b.ptr, t, n_pages, vp, dout.ptr, dec.ptr, None))
            for _ in range(args.warmup):
                fn()
            with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    fn()
                torch.cuda.synchronize()
            kern = kernel_ms(prof, args.steps)
            walk = sum(v for k, v in kern.items() if "walk" in k)
            out[name + "_profile"] = {"kernels_ms_per_call": kern, "walk_ms": walk,
                                      "value_passes_ms": sum(v for k, v in kern.items() if "delta_values" in k or "delta_scan" in k)}
    else:
        for name, w, b, t, vp, ab, e, note in runs:
            ms = timed(lambda w=w, b=b, t=t, vp=vp: N.call("ag_parquet_delta_decode_dev", w, b.ptr, t, n_pages, vp, dout.ptr, dec.ptr, None))
            out[name] = line(ms, ab, e, note)
        pblob, ptbl, _ = page_set(plain)
        penc = 8.0 * int(valid.sum())
        ms = timed(lambda: N.call("ag_parquet_plain_decode_spaced_dev", 8, pblob.ptr, ptbl, n_pages, dvalid.ptr, dout.ptr, None))
        out["parquet_plain_decode_spaced_i64_10pct_nulls"] = line(ms, penc + 8.0 * n + n / 8.0, penc,
                                                                  "PLAIN int64 pages, same slots and validity as the timestamps case: the floor for its output")
        out["delta_10pct_nulls_over_plain"] = out["parquet_delta_decode_i64_timestamps_10pct_nulls"]["ms"] / ms
        pblob.free()
    dblob.free(); rblob.free(); dvalid.free(); dec.free()
    return out


def snappy_cases(args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer, profile=False):
    """SNAPPY (ag_parquet_snappy_decompress_dev), pages compressed by pyarrow's C++ Snappy: (a) PLAIN int64 timestamp
    page bodies (copy-heavy); (b) the 17-bit dictionary-index page bodies of the dictionary case (nearly incompressible,
    literal-heavy); (c) (b) decompressed then dictionary-decoded, against the dictionary decode alone on the same pages
    uncompressed; (d) a device-to-device copy of (a)'s decompressed bytes, the floor for writing them."""
    import time

    import pyarrow as pa
    out = {}
    ts = [(np.cumsum(rng.integers(0, 1000, per_page)) + (k << 40)).astype(np.int64).tobytes() for k in range(4)]
    idx = [bytes([17]) + rle_literal_page(rng.integers(0, 100_000, per_page), 17) for _ in range(4)]

    def comp_set(bodies):
        encs = [pa.compress(b, codec="snappy", asbytes=True) for b in bodies]
        blob = b"".join(encs) + bytes(16)
        offs = np.cumsum([0] + [len(e) for e in encs])
        pages, d = [], 0
        for p in range(n_pages):
            pages.append((int(offs[p % 4]), len(encs[p % 4]), d, len(bodies[p % 4])))
            d += len(bodies[p % 4])
        t0 = time.perf_counter()                                  # pyarrow, one thread, host memory
        for p in range(n_pages):
            pa.decompress(encs[p % 4], decompressed_size=len(bodies[p % 4]), codec="snappy", asbytes=False)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        comp = sum(len(encs[p % 4]) for p in range(n_pages))
        return upload(np.frombuffer(blob, np.uint8)), N.compressed_table(pages), comp, d, cpu_ms, encs

    def snap_line(ms, comp, dec, cpu_ms, note):
        r = line(ms, comp + dec, comp, note)
        r.update({"compressed_bytes": comp, "decompressed_bytes": dec, "compression_ratio": dec / comp,
                  "cpu_context_pyarrow_1_thread_ms": cpu_ms,
                  "cpu_context_note": "pyarrow pa.decompress of the same pages, one thread, host memory, this machine's CPU; context, not a baseline"})
        return r

    tsrc, ttbl, tcomp, tdec, tcpu, _ = comp_set(ts)
    isrc, itbl, icomp, idec, icpu, _ = comp_set(idx)
    ddst = DeviceBuffer(idec + 64)
    dec = DeviceBuffer(8 * n_pages + 64)
    dictionary = rng.integers(-(1 << 62), 1 << 62, 100_000)
    ddict, bad = upload(dictionary), DeviceBuffer(64)
    dpages = N.page_table([(p * len(idx[0]), len(idx[p % 4]), per_page, p * per_page) for p in range(n_pages)])
    assert all(len(b) == len(idx[0]) for b in idx)
    snap_t = lambda: N.call("ag_parquet_snappy_decompress_dev", tsrc.ptr, ttbl, n_pages, dout.ptr, dec.ptr, None)
    snap_i = lambda: N.call("ag_parquet_snappy_decompress_dev", isrc.ptr, itbl, n_pages, ddst.ptr, dec.ptr, None)
    dict_i = lambda: N.call("ag_parquet_dict_decode_dev", 8, ddict.ptr, 100_000, ddst.ptr, dpages, n_pages, None, dout.ptr, dec.ptr, bad.ptr, None)
    if profile:
        import torch
        from torch.profiler import ProfilerActivity, profile as tprofile
        for name, fn in (("parquet_snappy_i64_timestamps", snap_t), ("parquet_snappy_dict_indices_17bit", snap_i)):
            for _ in range(args.warmup):
                fn()
            with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    fn()
                torch.cuda.synchronize()
            kern = kernel_ms(prof, args.steps)
            out[name + "_profile"] = {"kernels_ms_per_call": kern,
                                      "parse_ms": sum(v for k, v in kern.items() if "snappy_parse" in k),
                                      "execute_ms": kern.get("lz_exec_kernel", 0.0)}
    else:
        ms = timed(snap_t)
        out["parquet_snappy_i64_timestamps"] = snap_line(ms, tcomp, tdec, tcpu, "PLAIN int64 timestamp page bodies (increments in [0, 1000)): copy-heavy")
        ms = timed(snap_i)
        out["parquet_snappy_dict_indices_17bit"] = snap_line(ms, icomp, idec, icpu, "17-bit dictionary-index page bodies in literal runs: nearly incompressible, literal-heavy")
        ms_chain = timed(lambda: (snap_i(), dict_i()))
        ms_dict = timed(dict_i)
        out["parquet_snappy_then_dict_decode"] = {"ms": ms_chain, "dict_decode_alone_ms": ms_dict, "chain_over_dict_alone": ms_chain / ms_dict,
                                                  "note": "the index pages decompressed, then ag_parquet_dict_decode_dev (required, int64) from the decompressed buffer; against the dictionary decode alone"}
        cp = DeviceBuffer(tdec + 64)
        ms = timed(lambda: N.call("ag_copy_dev", cp.ptr, dout.ptr, tdec, None))
        out["device_copy_of_decompressed_timestamps"] = line(ms, 2.0 * tdec, tdec, "ag_copy_dev of (a)'s decompressed bytes: read + write, the floor for writing them")
        out["snappy_timestamps_over_copy"] = out["parquet_snappy_i64_timestamps"]["ms"] / ms
        cp.free()
    tsrc.free(); isrc.free(); ddst.free(); dec.free(); ddict.free(); bad.free()
    return out


def zstd_cases(args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer, profile=False):
    return codec_cases("zstd", args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer, profile)


def gzip_cases(args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer, profile=False):
    return codec_cases("gzip", args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer, profile)


def lz4_raw_cases(args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer, profile=False):
    return codec_cases("lz4_raw", args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer, profile)


# a codec's own kernels; every codec's execute is lz_exec_kernel, and a profile captures one codec
KERNEL_PREFIX = {"zstd": "zstd_", "gzip": "gz_", "lz4_raw": "lz4_"}


def codec_cases(codec, args, N, rng, n, n_pages, per_page, timed, upload, line, dout, DeviceBuffer, profile=False):
    """ZSTD, GZIP or LZ4_RAW (ag_parquet_<codec>_decompress_dev), the page bodies of the SNAPPY cases compressed by pyarrow at its
    default level: (a) PLAIN int64 timestamps; (b) 17-bit dictionary indices; (c) (b) decompressed then dictionary-decoded,
    against the dictionary decode alone; (d) a device-to-device copy of (a)'s decompressed bytes, the floor."""
    import time

    import pyarrow as pa
    out = {}
    ts = [(np.cumsum(rng.integers(0, 1000, per_page)) + (k << 40)).astype(np.int64).tobytes() for k in range(4)]
    idx = [bytes([17]) + rle_literal_page(rng.integers(0, 100_000, per_page), 17) for _ in range(4)]

    def comp_set(bodies):
        encs = [pa.compress(b, codec=codec, asbytes=True) for b in bodies]
        blob = b"".join(encs) + bytes(16)
        offs = np.cumsum([0] + [len(e) for e in encs])
        pages, d = [], 0
        for p in range(n_pages):
            pages.append((int(offs[p % 4]), len(encs[p % 4]), d, len(bodies[p % 4])))
            d += len(bodies[p % 4])
        t0 = time.perf_counter()                                  # pyarrow, one thread, host memory
        for p in range(n_pages):
            pa.decompress(encs[p % 4], decompressed_size=len(bodies[p % 4]), codec=codec, asbytes=False)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        comp = sum(len(encs[p % 4]) for p in range(n_pages))
        return upload(np.frombuffer(blob, np.uint8)), N.compressed_table(pages), comp, d, cpu_ms

    def z_line(ms, comp, dec, cpu_ms, note):
        r = line(ms, comp + dec, comp, note)
        r.update({"compressed_bytes": comp, "decompressed_bytes": dec, "compression_ratio": dec / comp,
                  "cpu_context_pyarrow_1_thread_ms": cpu_ms,
                  "cpu_context_note": "pyarrow pa.decompress of the same pages, one thread, host memory, this machine's CPU; context, not a baseline"})
        return r

    tsrc, ttbl, tcomp, tdec, tcpu = comp_set(ts)
    isrc, itbl, icomp, idec, icpu = comp_set(idx)
    ddst = DeviceBuffer(idec + 64)
    dec = DeviceBuffer(8 * n_pages + 64)
    dictionary = rng.integers(-(1 << 62), 1 << 62, 100_000)
    ddict, bad = upload(dictionary), DeviceBuffer(64)
    dpages = N.page_table([(p * len(idx[0]), len(idx[p % 4]), per_page, p * per_page) for p in range(n_pages)])
    assert all(len(b) == len(idx[0]) for b in idx)
    z_t = lambda: N.call(f"ag_parquet_{codec}_decompress_dev", tsrc.ptr, ttbl, n_pages, dout.ptr, dec.ptr, None)
    z_i = lambda: N.call(f"ag_parquet_{codec}_decompress_dev", isrc.ptr, itbl, n_pages, ddst.ptr, dec.ptr, None)
    dict_i = lambda: N.call("ag_parquet_dict_decode_dev", 8, ddict.ptr, 100_000, ddst.ptr, dpages, n_pages, None, dout.ptr, dec.ptr, bad.ptr, None)
    if profile:
        import torch
        from torch.profiler import ProfilerActivity, profile as tprofile
        for name, fn in ((f"parquet_{codec}_i64_timestamps", z_t), (f"parquet_{codec}_dict_indices_17bit", z_i)):
            for _ in range(args.warmup):
                fn()
            with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    fn()
                torch.cuda.synchronize()
            out[name + "_profile"] = {"kernels_ms_per_call": {k: v for k, v in kernel_ms(prof, args.steps).items() if k.startswith(KERNEL_PREFIX[codec]) or k == "lz_exec_kernel"}}
    else:
        ms = timed(z_t)
        out[f"parquet_{codec}_i64_timestamps"] = z_line(ms, tcomp, tdec, tcpu, "PLAIN int64 timestamp page bodies (increments in [0, 1000)), pyarrow's default level")
        ms = timed(z_i)
        out[f"parquet_{codec}_dict_indices_17bit"] = z_line(ms, icomp, idec, icpu, "17-bit dictionary-index page bodies in literal runs, pyarrow's default level")
        ms_chain = timed(lambda: (z_i(), dict_i()))
        ms_dict = timed(dict_i)
        out[f"parquet_{codec}_then_dict_decode"] = {"ms": ms_chain, "dict_decode_alone_ms": ms_dict, "chain_over_dict_alone": ms_chain / ms_dict,
                                                "note": "the index pages decompressed, then ag_parquet_dict_decode_dev (required, int64) from the decompressed buffer; against the dictionary decode alone"}
        cp = DeviceBuffer(tdec + 64)
        ms = timed(lambda: N.call("ag_copy_dev", cp.ptr, dout.ptr, tdec, None))
        out[f"{codec}_device_copy_of_decompressed_timestamps"] = line(ms, 2.0 * tdec, tdec, "ag_copy_dev of (a)'s decompressed bytes: read + write, the floor for writing them")
        out[f"{codec}_timestamps_over_copy"] = out[f"parquet_{codec}_i64_timestamps"]["ms"] / ms
        cp.free()
    tsrc.free(); isrc.free(); ddst.free(); dec.free(); ddict.free(); bad.free()
    return out



def bytearray_cases(args, N, rng, timed, upload, DeviceBuffer, values=20_000_000):
    """BYTE_ARRAY pages of ~1 MiB (pyarrow's default page size) into int64 offsets + data, dense, ~20M values:
    (a) RLE_DICTIONARY, 14-bit indices into 10K short strings (3..20 bytes); (b) PLAIN random lengths (0..70 bytes,
    mean ~14); (c) DELTA_LENGTH_BYTE_ARRAY of the same values; (d) DELTA_BYTE_ARRAY on sorted keys ("key_" + 9
    digits); (e) the PLAIN pages of (b) compressed with SNAPPY: decompression, then decode.  Algorithmic bytes: encoded
    bytes read + offsets written (8 per slot) + data written (+ the dictionary bytes read for (a)).  Four distinct page
    bodies are reused round-robin; every page writes its own slots."""
    import ctypes as C

    import pyarrow as pa
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile

    import pq_bytearray_ref as B
    import pq_files as F
    out = {}

    def make(bodies, per_page):
        n_pages = max(1, values // per_page)
        blob = b"".join(bodies) + bytes(16)
        offs = np.cumsum([0] + [len(x) for x in bodies])
        pages = [(int(offs[p % 4]), len(bodies[p % 4]), per_page, p * per_page) for p in range(n_pages)]
        enc = sum(len(bodies[p % 4]) for p in range(n_pages))
        return upload(np.frombuffer(blob, np.uint8)), pages, enc, n_pages

    def stages(kern):
        s = {"values": 0.0, "offsets": 0.0, "bytes": 0.0}
        for k, v in kern.items():
            if "ba_gather" in k:
                s["bytes"] += v
            elif any(x in k for x in ("ba_slot", "ba_sum", "ba_scan", "ba_offsets")):
                s["offsets"] += v
            else:
                s["values"] += v
        return s

    def run(name, enc_id, dblob, pages, enc, n_pages, per_page, data_bytes, note, dict_args=None, extra_read=0, pre=None):
        n = n_pages * per_page
        tbl = N.page_table(pages)
        doffs, dout = DeviceBuffer(8 * (n + 1) + 64), DeviceBuffer(data_bytes + 64)
        dec = DeviceBuffer(8 * n_pages + 64)
        tot = C.c_int64(0)
        do, dd, dl = dict_args or (None, None, 0)
        call = lambda: N.call("ag_parquet_byte_array_decode_dev", enc_id, 8, dblob.ptr, tbl, n_pages, n, None, do, dd, dl, 0,
                              doffs.ptr, dout.ptr, data_bytes, C.byref(tot), dec.ptr, None, None)
        fn = (lambda: (pre(), call())) if pre else call
        fn()
        assert tot.value == data_bytes, (name, tot.value, data_bytes)
        ms = timed(fn)
        ab = enc + 8.0 * (n + 1) + data_bytes + extra_read
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                fn()
            torch.cuda.synchronize()
        kern = kernel_ms(prof, args.steps)
        out[name] = {"ms": ms, "values": n, "pages": n_pages, "values_per_page": per_page, "encoded_bytes": enc,
                     "data_bytes": data_bytes, "algorithmic_bytes": ab, "gbs": ab / ms / 1e6, "frac": ab / ms / 1e6 / peak_of(),
                     "stage_ms_per_call": stages(kern), "kernels_ms_per_call": kern, "note": note}
        doffs.free(); dout.free(); dec.free()

    from bench import peaks
    peak_of = lambda: peaks()[0]

    # (a) dictionary
    dictionary = [bytes(rng.integers(97, 123, int(k), dtype=np.uint8)) for k in rng.integers(3, 21, 10_000)]
    dl = np.array([len(v) for v in dictionary], np.int64)
    ddoff, dddata = upload(np.concatenate([[0], np.cumsum(dl)]).astype(np.int64)), upload(np.frombuffer(b"".join(dictionary), np.uint8))
    per = 1 << 19
    idx = [rng.integers(0, 10_000, per) for _ in range(4)]
    bodies = [bytes([14]) + rle_literal_page(i, 14) for i in idx]
    dblob, pages, enc, n_pages = make(bodies, per)
    data = sum(int(dl[idx[p % 4]].sum()) for p in range(n_pages))
    run("bytearray_dict_short_strings", B.RLE_DICTIONARY, dblob, pages, enc, n_pages, per, data,
        "RLE_DICTIONARY pages of 2^19 14-bit indices (0.9 MiB), 10K strings of 3..20 bytes", (ddoff.ptr, dddata.ptr, 10_000), extra_read=data)
    dblob.free(); ddoff.free(); dddata.free()

    # (b) PLAIN, (c) DELTA_LENGTH, (e) SNAPPY + PLAIN: ~1 MiB pages of random-length strings
    per = 58_000
    vals = [F.random_strings(rng, per) for _ in range(4)]
    vbytes = [sum(len(v) for v in vs) for vs in vals]
    plain = [B.plain_encode(vs) for vs in vals]
    dblob, pages, enc, n_pages = make(plain, per)
    data = sum(vbytes[p % 4] for p in range(n_pages))
    run("bytearray_plain_random_lengths", B.PLAIN, dblob, pages, enc, n_pages, per, data,
        f"PLAIN pages of {per} strings of 0..70 bytes (~{len(plain[0]) >> 10} KiB)")
    # (e) the same pages compressed: decompress into dblob's layout, then decode
    comp = [pa.compress(b, codec="snappy", asbytes=True) for b in plain]
    cblob = upload(np.frombuffer(b"".join(comp) + bytes(16), np.uint8))
    coffs = np.cumsum([0] + [len(c) for c in comp])
    dst = DeviceBuffer(enc + 64)
    ctab, d = [], 0
    ppages = []
    for p in range(n_pages):
        ctab.append((int(coffs[p % 4]), len(comp[p % 4]), d, len(plain[p % 4])))
        ppages.append((d, len(plain[p % 4]), per, p * per))
        d += len(plain[p % 4])
    ctbl = N.compressed_table(ctab)
    snap = lambda: N.call("ag_parquet_snappy_decompress_dev", cblob.ptr, ctbl, n_pages, dst.ptr, None, None)
    csize = sum(len(comp[p % 4]) for p in range(n_pages))
    run("bytearray_snappy_then_plain", B.PLAIN, dst, ppages, csize, n_pages, per, data,
        "(b)'s pages compressed with SNAPPY, decompressed on the device, then decoded; algorithmic bytes count the compressed bytes",
        pre=snap)
    dblob.free(); cblob.free(); dst.free()
    dlba = [B.dlba_encode(vs) for vs in vals]
    dblob, pages, enc, n_pages = make(dlba, per)
    run("bytearray_delta_length", B.DELTA_LENGTH_BYTE_ARRAY, dblob, pages, enc, n_pages, per, data,
        f"DELTA_LENGTH_BYTE_ARRAY pages of the same {per} strings")
    dblob.free()

    # (d) DELTA_BYTE_ARRAY on sorted keys
    per = 1 << 18
    keys = [F.random_strings(rng, per, sorted_keys=True) for _ in range(4)]
    dba = [B.dba_encode(k) for k in keys]
    dblob, pages, enc, n_pages = make(dba, per)
    data = sum(sum(len(v) for v in keys[p % 4]) for p in range(n_pages))
    run("bytearray_delta_sorted_keys", B.DELTA_BYTE_ARRAY, dblob, pages, enc, n_pages, per, data,
        f"DELTA_BYTE_ARRAY pages of {per} sorted 13-byte keys (~{len(dba[0]) >> 10} KiB; prefix ~7 bytes)")
    dblob.free()
    return out


def fixed_cases(args, N, rng, timed, upload, DeviceBuffer, peak, n_pages, per):
    """BOOLEAN and fixed-width pages (ag_parquet_fixed_decode_dev / ag_parquet_bool_decode_dev), n_pages pages of `per`
    values.  Algorithmic bytes: encoded bytes read + output written (+ 1/8 B per slot of validity when spaced, + the
    dictionary for (d)).  Four distinct page bodies are reused round-robin; every page writes its own slots."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    out = {}
    n = n_pages * per
    valid = rng.random(n) >= 0.1
    dvalid = upload(np.packbits(valid, bitorder="little"))
    dec = DeviceBuffer(8 * n_pages + 64)

    def pages_of(bodies):
        blob = b"".join(bodies) + bytes(16)
        offs = np.cumsum([0] + [len(x) for x in bodies])
        pages = [(int(offs[p % 4]), len(bodies[p % 4]), per, p * per) for p in range(n_pages)]
        return upload(np.frombuffer(blob, np.uint8)), N.page_table(pages), sum(len(bodies[p % 4]) for p in range(n_pages))

    def run(name, fn, ab, note):
        fn()
        N.call("ag_stream_sync", None)
        ms = timed(fn)
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                fn()
            torch.cuda.synchronize()
        out[name] = {"ms": ms, "values": n, "pages": n_pages, "values_per_page": per, "algorithmic_bytes": ab, "gbs": ab / ms / 1e6,
                     "frac": ab / ms / 1e6 / peak, "kernels_ms_per_call": kernel_ms(prof, args.steps), "note": note}

    # (a) DOUBLE BYTE_STREAM_SPLIT, dense and 10 % nulls
    bodies = [np.ascontiguousarray(rng.standard_normal(per).view(np.uint8).reshape(per, 8).T).tobytes() for _ in range(4)]
    dblob, tbl, enc = pages_of(bodies)
    dout = DeviceBuffer(8 * n + 64)
    for label, vp, vb in (("required", None, 0.0), ("10pct_nulls", dvalid.ptr, n / 8)):
        run(f"fixed_bss_double_{label}", lambda: N.call("ag_parquet_fixed_decode_dev", N.PQ_TYPE_DOUBLE, 0, N.PQ_ENC_BYTE_STREAM_SPLIT, dblob.ptr, tbl,
                                                       n_pages, vp, None, 0, dout.ptr, dec.ptr, None, None),
            enc + 8.0 * n + vb, "DOUBLE BYTE_STREAM_SPLIT pages of 2^19 values (4 MiB)")
    dblob.free(); dout.free()
    # (b) FLBA(16) BYTE_STREAM_SPLIT
    bodies = [np.ascontiguousarray(rng.integers(0, 256, (per, 16), dtype=np.uint8).T).tobytes() for _ in range(4)]
    dblob, tbl, enc = pages_of(bodies)
    dout = DeviceBuffer(16 * n + 64)
    run("fixed_bss_flba16", lambda: N.call("ag_parquet_fixed_decode_dev", N.PQ_TYPE_FIXED_LEN_BYTE_ARRAY, 16, N.PQ_ENC_BYTE_STREAM_SPLIT, dblob.ptr,
                                           tbl, n_pages, None, None, 0, dout.ptr, dec.ptr, None, None),
        enc + 16.0 * n, "FIXED_LEN_BYTE_ARRAY(16) BYTE_STREAM_SPLIT pages, dense")
    dblob.free()
    # (c) FLBA(16) dictionary, 64K entries, 16-bit indices in literal runs
    ddict = upload(rng.integers(0, 256, (1 << 16, 16), dtype=np.uint8))
    bodies = [bytes([16]) + rle_literal_page(rng.integers(0, 1 << 16, per), 16) for _ in range(4)]
    dblob, tbl, enc = pages_of(bodies)
    bad = DeviceBuffer(64)
    run("fixed_dict_flba16", lambda: N.call("ag_parquet_fixed_decode_dev", N.PQ_TYPE_FIXED_LEN_BYTE_ARRAY, 16, N.PQ_ENC_RLE_DICTIONARY, dblob.ptr,
                                            tbl, n_pages, None, ddict.ptr, 1 << 16, dout.ptr, dec.ptr, bad.ptr, None),
        enc + 16.0 * n, "FIXED_LEN_BYTE_ARRAY(16), 64K-entry dictionary (1 MiB, L2-resident), 16-bit indices in literal runs, dense")
    dblob.free(); ddict.free(); bad.free(); dout.free()
    # (d) INT96 PLAIN spaced, 10 % nulls
    bodies = [rng.integers(0, 256, 12 * per, dtype=np.uint8).tobytes() for _ in range(4)]
    dblob, tbl, enc = pages_of(bodies)
    dout = DeviceBuffer(12 * n + 64)
    run("fixed_plain_int96_10pct_nulls", lambda: N.call("ag_parquet_fixed_decode_dev", N.PQ_TYPE_INT96, 0, N.PQ_ENC_PLAIN, dblob.ptr, tbl, n_pages,
                                                        dvalid.ptr, None, 0, dout.ptr, dec.ptr, None, None),
        12.0 * valid.sum() + 12.0 * n + n / 8, "INT96 PLAIN pages of 2^19 values, 10 % nulls (the valid slots' values are read)")
    dblob.free(); dout.free()
    # (e) BOOLEAN PLAIN dense and spaced, (f) BOOLEAN RLE of random bits
    dout = DeviceBuffer(n // 8 + 64)
    bodies = [np.packbits(rng.random(per) < 0.5, bitorder="little").tobytes() for _ in range(4)]
    dblob, tbl, enc = pages_of(bodies)
    for label, vp, vb in (("required", None, 0.0), ("10pct_nulls", dvalid.ptr, n / 8)):
        run(f"bool_plain_{label}", lambda: N.call("ag_parquet_bool_decode_dev", N.PQ_ENC_PLAIN, dblob.ptr, tbl, n_pages, vp, dout.ptr, dec.ptr, None),
            enc + n / 8 + vb, "BOOLEAN PLAIN pages of 2^19 bits")
    dblob.free()
    bodies = []
    for _ in range(4):
        s = rle_literal_page((rng.random(per) < 0.5).astype(np.int64), 1)
        bodies.append(len(s).to_bytes(4, "little") + s)
    dblob, tbl, enc = pages_of(bodies)
    run("bool_rle_random", lambda: N.call("ag_parquet_bool_decode_dev", N.PQ_ENC_RLE, dblob.ptr, tbl, n_pages, None, dout.ptr, dec.ptr, None),
        enc + n / 8, "BOOLEAN RLE pages of 2^19 random bits (literal runs of 504), dense")
    dblob.free(); dout.free(); dvalid.free(); dec.free()
    return out


if __name__ == "__main__":
    main()
