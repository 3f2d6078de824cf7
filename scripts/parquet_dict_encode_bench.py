#!/usr/bin/env python
"""BYTE_ARRAY dictionaries on the device (ag_parquet_byte_array_dict_encode_dev, csrc/hash.cu) from LargeBinary columns
(int64 offsets):
  short_10k         20M random strings of 0-32 bytes drawn from 10K values
  short_10k_null    the same with 10 % nulls
  short_500k        20M over 500K values (the small, L2-sized table)
  short_4m          20M over 4M values (the full-size table)
  keys              20M sorted 48-byte keys, all distinct
  kib_1000          2M values of 768-1280 bytes over 1000 values

  python scripts/parquet_dict_encode_bench.py [--values 20000000] [--steps K] [--warmup W] [--out FILE]

Prints one JSON line: per case the time per dictionary call (CUDA events around K calls after W warm-up calls; the
call synchronises once, after its checking pass), with marks at the ends of data pages of 2^20 slots; the modelled HBM
bytes (offsets, validity and data read once, uint32 indices and the first-appearance bitmap written) over the HBM
peak; a torch.profiler split of the device time per kernel (a run of its own); in the same run, a PLAIN page encode of
the same column (ag_parquet_byte_array_encode_dev, pages of about 1 MiB) and the whole device route to the dictionary
page and index pages (dict encode, mark counts to the host, PLAIN with `first`, one RLE call per bit width); and
pyarrow's one-thread dictionary write of the same column (context, not a baseline).  Every case checks its indices and
counts against a host dictionary of the column.  The card name and power limit are read in the same run."""
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

PAGE_SLOTS = 1 << 20
PAGE_BYTES = 1 << 20


def corpus(rng, kind, n):
    """-> (offsets int64, data uint8, valid bool or None)"""
    if kind == "keys":
        nums = np.sort(rng.integers(0, 10 ** 11, n)) + np.arange(n)       # strictly increasing: all distinct
        digits = np.zeros((n, 12), np.uint8)
        x = nums.copy()
        for k in range(11, -1, -1):
            digits[:, k] = 48 + x % 10
            x //= 10
        prefix = np.frombuffer(b"warehouse/orders/region=emea/custom-", np.uint8)
        data = np.concatenate([np.broadcast_to(prefix, (n, 36)), digits], axis=1).ravel()
        return np.arange(n + 1, dtype=np.int64) * 48, np.ascontiguousarray(data), None
    distinct = {"short_10k": 10_000, "short_10k_null": 10_000, "short_500k": 500_000, "short_4m": 4_000_000, "kib_1000": 1000}[kind]
    plens = rng.integers(0, 33, distinct) if kind.startswith("short") else rng.integers(768, 1281, distinct)
    poff = np.concatenate([[0], np.cumsum(plens)]).astype(np.int64)
    pdata = rng.integers(0, 256, int(poff[-1]), dtype=np.uint8)
    idx = rng.integers(0, distinct, n)
    lens = plens[idx]
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    src = np.repeat(poff[idx] - offsets[:-1], lens) + np.arange(int(offsets[-1]), dtype=np.int64)
    valid = rng.random(n) >= 0.1 if kind.endswith("_null") else None
    return offsets, pdata[src], valid


def host_dictionary(offsets, data, valid):
    """(entries, entry bytes, indices of the valid slots) by a host memo table keyed on the bytes"""
    n = offsets.size - 1
    raw = data.tobytes()
    index_of, indices, ebytes = {}, np.empty(n, np.uint32), 0
    m = 0
    for i in range(n):
        if valid is not None and not valid[i]:
            continue
        v = raw[offsets[i]:offsets[i + 1]]
        k = index_of.get(v)
        if k is None:
            k = index_of[v] = len(index_of)
            ebytes += len(v)
        indices[m] = k
        m += 1
    return len(index_of), ebytes, indices[:m]


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

    from arrow_go_b200 import _native as N
    from arrow_go_b200.device import DeviceBuffer, Event
    from bench import peaks
    from parquet_pages_bench import card, kernel_ms

    N.call("ag_init", 0)
    peak, peak_kind = peaks()
    rng = np.random.default_rng(0xD1C7)
    res = {"values": args.values, "page_slots": PAGE_SLOTS, "offsets": "int64", "peak_gbs": peak, "peak_kind": peak_kind,
           **card(), "timing": f"CUDA events around {args.steps} calls after {args.warmup} warm-up calls"}
    cases = [("short_10k", args.values), ("short_10k_null", args.values), ("short_500k", args.values), ("short_4m", args.values),
             ("keys", args.values), ("kib_1000", args.values // 10)]

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
        b = DeviceBuffer(arr.nbytes + 64)
        N.call("ag_upload", b.ptr, arr.ctypes.data, arr.nbytes, None)
        return b

    def rle_bound(bw, k):
        s = C.c_int64()
        N.call("ag_parquet_rle_max_size", bw, N.PQ_RLE_WIDTH, k, C.byref(s))
        return s.value

    for kind, n in cases:
        offsets, data, valid = corpus(rng, kind, n)
        vb = None if valid is None else np.packbits(valid, bitorder="little")
        d_off, d_data = upload(offsets), upload(data)
        d_valid = None if vb is None else upload(vb)
        nvalid = n if valid is None else int(valid.sum())
        dense = np.arange(n + 1) if valid is None else np.concatenate([[0], np.cumsum(valid)])
        vbytes = int(offsets[-1]) if valid is None else int(((offsets[1:] - offsets[:-1]) * valid).sum())
        marks = np.append(np.arange(PAGE_SLOTS, n, PAGE_SLOTS), n).astype(np.int64)
        n_first = ((n + 31) // 32) * 4
        d_idx, d_mc, d_cnt, d_first = DeviceBuffer(4 * nvalid + 64), DeviceBuffer(16 * marks.size + 64), DeviceBuffer(64), DeviceBuffer(n_first + 64)
        tbl = N.ba_chunk_table([(d_off.ptr, d_data.ptr, None if d_valid is None else d_valid.ptr, 0, n, d_first.ptr)])
        dict_call = lambda: N.call("ag_parquet_byte_array_dict_encode_dev", 8, tbl, 1, marks.ctypes.data, marks.size,  # noqa: E731
                                   d_idx.ptr, d_mc.ptr, d_cnt.ptr, None, None)
        ms = timed(dict_call)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:        # a separate run: tracing slows the host
            for _ in range(args.steps):
                dict_call()
            torch.cuda.synchronize()
        kern = kernel_ms(prof, args.steps)
        entries, ebytes, indices = host_dictionary(offsets, data, valid)
        cnt = d_cnt.to_numpy(np.int64, 3, 0)
        assert cnt.tolist() == [entries, ebytes, nvalid], (kind, cnt, entries, ebytes)
        assert np.array_equal(d_idx.to_numpy(np.uint32, nvalid, 0), indices), kind
        model = 8 * (n + 1) + (0 if vb is None else vb.nbytes) + vbytes + 4 * nvalid + n_first

        # PLAIN pages of the same column, about 1 MiB of value bytes each
        cuts = np.unique(np.concatenate([[0], np.searchsorted(offsets, np.arange(PAGE_BYTES, int(offsets[-1]), PAGE_BYTES)), [n]]))
        spans = [(int(a), int(b - a)) for a, b in zip(cuts[:-1], cuts[1:]) if b > a]
        caps = []
        for i0, k in spans:
            s = C.c_int64()
            N.call("ag_parquet_byte_array_max_size", N.PQ_ENC_PLAIN, k, int(offsets[i0 + k] - offsets[i0]), C.byref(s))
            caps.append(s.value)
        outs = np.concatenate([[0], np.cumsum(caps)])
        ptbl = N.enc_page_table([(i0, k, int(o), c) for (i0, k), o, c in zip(spans, outs, caps)])
        d_plain, d_plen = DeviceBuffer(int(outs[-1]) + 64), DeviceBuffer(8 * len(spans) + 64)
        plain_ms = timed(lambda: N.call("ag_parquet_byte_array_encode_dev", N.PQ_ENC_PLAIN, 8, d_off.ptr, d_data.ptr,
                                        None if d_valid is None else d_valid.ptr, ptbl, len(spans), d_plain.ptr, d_plen.ptr, None, None))
        d_plain.free()
        d_plen.free()

        # the whole device route: dictionary page and index pages of PAGE_SLOTS slots each
        s = C.c_int64()
        N.call("ag_parquet_byte_array_max_size", N.PQ_ENC_PLAIN, n, int(offsets[-1]), C.byref(s))
        dcap = s.value
        d_dpage, d_dlen = DeviceBuffer(dcap + 64), DeviceBuffer(64)
        page_dense = [(int(dense[a]), int(dense[min(a + PAGE_SLOTS, n)] - dense[a])) for a in range(0, n, PAGE_SLOTS)]
        icaps = [rle_bound(32, k) for _, k in page_dense]
        iouts = np.concatenate([[0], np.cumsum(icaps)])
        d_ipages, d_ilen = DeviceBuffer(int(iouts[-1]) + 64), DeviceBuffer(8 * len(page_dense) + 64)
        dtbl = N.enc_page_table([(0, n, 0, dcap)])
        mc = np.zeros(2 * marks.size, np.int64)

        def route():
            dict_call()
            N.call("ag_download", mc.ctypes.data, d_mc.ptr, mc.nbytes, None)
            N.call("ag_stream_sync", None)
            N.call("ag_parquet_byte_array_encode_dev", N.PQ_ENC_PLAIN, 8, d_off.ptr, d_data.ptr, d_first.ptr, dtbl, 1, d_dpage.ptr,
                   d_dlen.ptr, None, None)
            widths = {}
            for p, (d0, k) in enumerate(page_dense):
                e = int(mc[2 * p])
                bw = 0 if e == 0 else 1 if e == 1 else (e - 1).bit_length()
                widths.setdefault(bw, []).append((d0, k, int(iouts[p]), rle_bound(bw, k)))
            for bw, pages in widths.items():
                N.call("ag_parquet_rle_encode_dev", bw, N.PQ_RLE_WIDTH, N.PQ_RLE_IN_U32, d_idx.ptr, N.enc_page_table(pages), len(pages),
                       d_ipages.ptr, d_ilen.ptr, None, None)
        route_ms = timed(route)
        dict_page_bytes = int(d_dlen.to_numpy(np.int64, 1, 0)[0])
        assert dict_page_bytes == 4 * entries + ebytes, kind
        for b in (d_dpage, d_dlen, d_ipages, d_ilen):
            b.free()

        arr = pa.LargeBinaryArray.from_buffers(pa.large_binary(), n, [None if vb is None else pa.py_buffer(vb), pa.py_buffer(offsets),
                                                                     pa.py_buffer(data)])
        t = time.perf_counter()
        pq.write_table(pa.table({"c": arr}), io.BytesIO(), use_dictionary=True, compression="NONE", data_page_version="2.0")
        cpu_ms = (time.perf_counter() - t) * 1e3
        res[kind] = {
            "ms": ms, "values": n, "valid_values": nvalid, "entries": entries, "entry_bytes": ebytes, "value_bytes": vbytes,
            "marks": int(marks.size), "model_bytes": model, "model_gbs": model / ms / 1e6, "model_frac_of_peak": model / ms / 1e6 / peak,
            "kernels_ms_per_call": kern, "kernels_total_ms": sum(kern.values()),
            "plain_pages_ms": plain_ms, "plain_pages": len(spans), "route_to_dictionary_and_index_pages_ms": route_ms,
            "dictionary_page_bytes": dict_page_bytes,
            "cpu_context_pyarrow_1_thread_write_ms": cpu_ms,
            "cpu_context_note": "pyarrow pq.write_table of the same column with a dictionary (NONE, v2 pages, includes levels, headers, "
                                "footer and its own fallback), one thread, the GPU host's CPU; context, not a baseline"}
        print(kind, json.dumps(res[kind]), file=sys.stderr, flush=True)
        for b in (d_off, d_data, d_valid, d_idx, d_mc, d_cnt, d_first):
            if b is not None:
                b.free()
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
