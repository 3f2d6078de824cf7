"""Test helper: read one planned column chunk (pq_pages.chunk_plan) into a column's values and validity, once through the
device entry points in the order INTEGRATION.md §6 documents for a column reader, and once through the Python
restatements.  Both return (values, validity) in the form pq_files.expected gives.  Not product code."""
import ctypes as C

import numpy as np

import pq_bytearray_ref as B
import pq_delta_ref as D
import pq_fixed_ref as X
import pq_pages as P
import pq_ref as R
from arrow_go_b200 import _native as N
from helpers import Dev, ptr

CANARY = 0xA7
NUMERIC = {P.INT32: np.int32, P.INT64: np.int64, P.FLOAT: np.float32, P.DOUBLE: np.float64}
DICT_ENCODINGS = (P.PLAIN_DICTIONARY, P.RLE_DICTIONARY)


def _groups(pages):
    """{encoding: [values descriptor]}, the two dictionary encodings as one, in the order the encodings first occur"""
    out = {}
    for enc, desc in pages:
        out.setdefault(P.RLE_DICTIONARY if enc in DICT_ENCODINGS else enc, []).append(desc)
    return out


def read_chunk_dev(ag, plan, offset_width=8, host_values=False):
    """The column reader flow on the device -> (values, validity):
       1. upload the chunk as it sits in the file;
       2. one ag_parquet_{snappy,zstd,gzip,lz4_raw}_decompress_dev call, or device copies of the pages that are not compressed,
          every page body at its 8-byte aligned offset of one buffer `dst` (checked against host_decompress);
       3. an optional column's levels -> ag_parquet_def_levels_to_bitmap_dev -> the validity bitmap;
       4. the values, by physical type, width and encoding.
    BYTE_ARRAY values go to an Arrow array of `offset_width`; host_values runs their decode through the host entry
    point on host copies of `dst` and the validity."""
    n = plan["n_slots"]
    dchunk = Dev(P.as_array(plan["chunk"]))
    ddst = Dev(nbytes=plan["n_dst"])
    if plan["comp"]:
        fn = {"SNAPPY": "ag_parquet_snappy_decompress_dev", "ZSTD": "ag_parquet_zstd_decompress_dev",
              "GZIP": "ag_parquet_gzip_decompress_dev", "LZ4": "ag_parquet_lz4_raw_decompress_dev"}[plan["codec"]]
        dw = Dev(np.full(len(plan["comp"]), -1, np.int64))
        ag.call(fn, dchunk.ptr, N.compressed_table(plan["comp"]), len(plan["comp"]), ddst.ptr, dw.ptr, None)
    for s, d, k in plan["copies"]:
        ag.call("ag_copy_dev", ddst.ptr + d, dchunk.ptr + s, k, None)
    ag.call("ag_stream_sync", None)
    if plan["comp"]:
        assert dw.get().tolist() == [c[3] for c in plan["comp"]]
    dst = ddst.get(np.uint8, plan["n_dst"])
    assert dst.tobytes() == P.host_decompress(plan)

    dvalid = None
    if plan["max_def"]:
        levels = [lv for _, lv, _ in plan["pages"]]
        enc, src = (N.PQ_LEVELS_V1_RLE, ddst) if plan["v1"] else (N.PQ_LEVELS_V2_RLE, dchunk)
        dlv, dldec = Dev(nbytes=2 * n), Dev(np.full(len(levels), -1, np.int64))
        ag.call("ag_parquet_levels_decode_dev", plan["max_def"], enc, src.ptr, N.page_table(levels), len(levels), dlv.ptr, dldec.ptr, None)
        dvalid, dcounts = Dev(nbytes=n // 8 + 8), Dev(np.zeros(2, np.int64))
        ag.call("ag_parquet_def_levels_to_bitmap_dev", dlv.ptr, n, plan["max_def"], -1, dvalid.ptr, 0, n, dcounts.ptr, None)
        ag.call("ag_stream_sync", None)
        assert dldec.get().tolist() == [lv[2] for lv in levels]
    valid = np.unpackbits(dvalid.get(np.uint8, n // 8 + 1), bitorder="little")[:n].astype(bool) if dvalid else np.ones(n, bool)

    pages = P.value_sections(plan, dst)
    if plan["ptype"] == P.BYTE_ARRAY:
        return _byte_array_dev(ag, plan, pages, dst, ddst, valid, dvalid, offset_width, host_values), valid
    vp = dvalid.ptr if dvalid else None
    ptype, tl = plan["ptype"], plan["type_length"]
    decoded = []                                                # (device counts, pages) of every call that counts
    if ptype == P.BOOLEAN:
        dout = Dev(np.zeros(n // 8 + 8, np.uint8))
        for enc, group in _groups(pages).items():
            decoded.append((Dev(np.full(len(group), -1, np.int64)), group))
            ag.call("ag_parquet_bool_decode_dev", enc, ddst.ptr, N.page_table(group), len(group), vp, dout.ptr, decoded[-1][0].ptr, None)
        values = np.unpackbits(dout.get(), bitorder="little")[:n]
    else:
        width = X.width_of(ptype, tl)
        dout = Dev(np.full(n * width, CANARY, np.uint8))
        ddict = None
        if plan["dict"] and ptype not in NUMERIC:               # the fixed decoder takes the dictionary as values
            b, ln, nv = plan["dict"]
            ddict = Dev(nbytes=nv * width)
            ag.call("ag_parquet_fixed_decode_dev", ptype, tl, P.PLAIN, ddst.ptr + b, N.page_table([(0, ln, nv, 0)]), 1, None, None,
                    0, ddict.ptr, None, None, None)
        for enc, group in _groups(pages).items():
            tbl, k = N.page_table(group), len(group)
            if ptype in NUMERIC and enc == P.PLAIN:             # no counts, no index to go wrong
                ag.call("ag_parquet_plain_decode_spaced_dev", width, ddst.ptr, tbl, k, vp, dout.ptr, None)
                continue
            ddec, dbad = Dev(np.full(k, -1, np.int64)), Dev(np.full(1, -1, np.int64))
            if ptype in NUMERIC and enc == P.RLE_DICTIONARY:
                b, _, nv = plan["dict"]
                ag.call("ag_parquet_dict_decode_dev", width, ddst.ptr + b, nv, ddst.ptr, tbl, k, vp, dout.ptr, ddec.ptr, dbad.ptr, None)
            elif ptype in NUMERIC and enc == P.DELTA_BINARY_PACKED:
                ag.call("ag_parquet_delta_decode_dev", width, ddst.ptr, tbl, k, vp, dout.ptr, ddec.ptr, None)
                dbad = None
            else:
                dic = ddict if enc == P.RLE_DICTIONARY else None
                ag.call("ag_parquet_fixed_decode_dev", ptype, tl, enc, ddst.ptr, tbl, k, vp, dic.ptr if dic else None,
                        plan["dict"][2] if dic else 0, dout.ptr, ddec.ptr, dbad.ptr, None)
            assert dbad is None or dbad.get()[0] == N.NO_ERROR_POS
            decoded.append((ddec, group))
        values = dout.get()
    ag.call("ag_stream_sync", None)
    for ddec, group in decoded:
        assert ddec.get().tolist() == [p[2] for p in group]
    return values.tobytes(), valid


def _byte_array_dev(ag, plan, pages, dst, ddst, valid, dvalid, ow, host):
    """INTEGRATION.md §6 item 3, BYTE_ARRAY steps 1-5: the dictionary page as PLAIN, dense, into the dictionary's
    offsets and data; then one call per encoding in slot order (the dictionary-encoded pages, then the PLAIN pages a
    writer fell back to), chained with offset_base into one offsets buffer and one data buffer"""
    n = plan["n_slots"]
    odt = np.int32 if ow == 4 else np.int64
    if host:
        fn, tail, mem, addr, back = "ag_parquet_byte_array_decode", (), (lambda a: a), ptr, (lambda a: a)
        src = dst
        vbits = np.packbits(valid, bitorder="little") if dvalid else None
    else:
        fn, tail, mem, back = "ag_parquet_byte_array_decode_dev", (None,), Dev, (lambda d: d.get())
        addr = lambda d: None if d is None else d.ptr                     # noqa: E731
        src, vbits = ddst, dvalid

    def decode(enc, group, first, end, offsets, out, cap, vbits=None, dictionary=(None, None, 0), base=0):
        """one call over the pages `group`, which fill slots [first, end) -> its total"""
        total = C.c_int64(-1)
        group = [(d, ln, nv, o - first) for d, ln, nv, o in group]
        ag.call(fn, enc, ow, addr(src), N.page_table(group), len(group), end - first,
                None if vbits is None else addr(vbits) + first // 8, addr(dictionary[0]), addr(dictionary[1]), dictionary[2],
                base, addr(offsets) + first * ow, addr(out), cap, C.byref(total), None, None, *tail)
        return total.value

    dictionary = (None, None, 0)
    if plan["dict"]:
        b, ln, nv = plan["dict"]
        dictionary = (mem(np.zeros(nv + 1, odt)), mem(np.zeros(ln + 1, np.uint8)), nv)
        decode(P.PLAIN, [(b, ln, nv, 0)], 0, nv, dictionary[0], dictionary[1], ln)
    groups = []
    for enc, group in _groups(pages).items():
        first, end = min(p[3] for p in group), max(p[3] + p[2] for p in group)
        assert first == (groups[-1][3] if groups else 0), "pages of different encodings interleave"
        # the validity advances with the offsets in whole bytes: pyarrow starts pages at multiples of its write batch
        assert first % 8 == 0 or vbits is None, first
        groups.append((enc, group, first, end))
    offsets = mem(np.zeros(n + 1, odt))
    cap = 0
    for enc, group, first, end in groups:                       # PLAIN / DELTA_LENGTH totals are bounded by the page bytes
        if enc in (P.PLAIN, P.DELTA_LENGTH_BYTE_ARRAY):
            cap += sum(p[1] for p in group)
        else:
            cap += decode(enc, group, first, end, offsets, None, 0, vbits, dictionary)
    out, base = mem(np.zeros(cap + 1, np.uint8)), 0
    for enc, group, first, end in groups:
        base += decode(enc, group, first, end, offsets, out, cap, vbits, dictionary, base)
    ag.call("ag_stream_sync", None)
    offs, data = back(offsets).astype(np.int64), back(out).tobytes()
    assert offs[0] == 0 and offs[n] == base
    return [data[offs[s]:offs[s + 1]] for s in range(n)]


def read_chunk_oracle(plan, dst):
    """the same chunk through the Python restatements (pq_ref, pq_delta_ref, pq_fixed_ref, pq_bytearray_ref), page by
    page, over the decompressed buffer `dst` -> (values, validity)"""
    n, ptype, max_def = plan["n_slots"], plan["ptype"], plan["max_def"]
    dst = bytes(dst)
    valid = np.ones(n, bool)
    if max_def:
        src = dst if plan["v1"] else bytes(plan["chunk"])
        for _, (b, ln, nv, o), _ in plan["pages"]:
            levels, err = R.levels_decode_page(src[b:b + ln], max_def, plan["v1"], nv)
            assert err == R.ERR_NONE and levels.size == nv
            valid[o:o + nv] = levels >= max_def
    if ptype == P.BYTE_ARRAY:
        out, width = [b""] * n, None
    elif ptype == P.BOOLEAN:
        out, width = np.zeros(n, np.uint8), 0
    else:
        width = X.width_of(ptype, plan["type_length"])
        out = np.zeros((n, width), np.uint8)
    dictionary = None
    if plan["dict"]:
        b, ln, nv = plan["dict"]
        if ptype == P.BYTE_ARRAY:
            dictionary, slots, msg = B.plain_decode(dst[b:b + ln], nv)
        elif ptype in NUMERIC:
            dictionary, slots, msg = np.frombuffer(dst[b:b + nv * width], NUMERIC[ptype]), nv, None
        else:
            dictionary, slots, msg, _ = X.fixed_decode(ptype, width, P.PLAIN, dst[b:b + ln], nv)
        assert msg is None and slots == nv
    for enc, (b, ln, nv, o) in P.value_sections(plan, dst):
        page, v = dst[b:b + ln], valid[o:o + nv].copy() if max_def else nv
        bad = msg = None
        if ptype == P.BYTE_ARRAY:
            vals, slots, msg, bad = B.decode(enc, page, v, dictionary)
        elif ptype == P.BOOLEAN:
            vals, slots, msg = X.bool_decode(enc, page, v)
        elif ptype in NUMERIC and enc in DICT_ENCODINGS:
            vals, slots, err, bad = R.dict_decode(page, dictionary, v)
            assert err == R.ERR_NONE
        elif ptype in NUMERIC and enc == P.PLAIN:
            vals, err = R.plain_decode_spaced(page, NUMERIC[ptype], valid[o:o + nv])
            assert err == R.ERR_NONE
            slots = nv
        elif ptype in NUMERIC and enc == P.DELTA_BINARY_PACKED:
            vals, slots, err, msg = D.delta_decode(page, width, v)
            msg = msg if err != D.DERR_NONE else None
        else:
            vals, slots, msg, bad = X.fixed_decode(ptype, width, enc, page, v, dictionary)
        assert msg is None and bad is None and slots == nv, (enc, msg, bad, slots, nv)
        if ptype in NUMERIC and enc in (*DICT_ENCODINGS, P.PLAIN, P.DELTA_BINARY_PACKED):
            vals = np.asarray(vals, NUMERIC[ptype]).view(np.uint8).reshape(-1, width)
        out[o:o + nv] = vals
    return (out if ptype == P.BYTE_ARRAY else out.tobytes()), valid
