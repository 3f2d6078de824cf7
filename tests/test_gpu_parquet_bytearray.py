"""Device BYTE_ARRAY page decode (PLAIN, dictionary, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY) into Arrow offsets + data
against the Python restatement in tests/pq_bytearray_ref.py, host and _dev flavours, offset widths 4 and 8; pyarrow
files end to end against pq.read_table."""
import ctypes as C
import json
import os
import zlib

import numpy as np
import pytest

import pq_bytearray_ref as B
import pq_delta_ref as D
import pq_files as F
import pq_pages as P
from arrow_go_b200 import _native as N
from helpers import Dev, checksum64, ptr
from pq_chunk import read_chunk_dev
from pq_pages import batch

gpu = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
WIDTHS = pytest.mark.parametrize("ow", [4, 8], ids=["off32", "off64"])
ENCODERS = {B.PLAIN: B.plain_encode, B.DELTA_LENGTH_BYTE_ARRAY: B.dlba_encode, B.DELTA_BYTE_ARRAY: B.dba_encode}
CANARY = 0xA7
# 300 tiles of 1024 slots, the last one partial: the one-block scans over a page's tiles take a full 256-tile step and
# a partial one, and two such pages take the all-slot chunk scan past its first 256 chunks
SEAM_SLOTS = 307_195
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "parquet_bytearray.json")))


def run_ba(ag, enc, ow, blob, pages, n_slots, vbits=None, dict_off=None, dict_data=None, offset_base=0, out_cap=None, dev=False):
    """-> (status, message, offsets int64, data bytes (out_cap of them, canary elsewhere), decoded, total, bad_pos)"""
    odt = np.int32 if ow == 4 else np.int64
    tbl = N.page_table(pages)
    cap = (sum(p[1] for p in pages) + 64) * 4 + offset_base if out_cap is None else out_cap
    if dict_off is not None and out_cap is None:
        cap = offset_base + n_slots * int(max(np.diff(dict_off).max(initial=0), 0)) + 64
    offs = np.full(n_slots + 1, -9, odt)
    out = np.full(max(cap, 1), CANARY, np.uint8)
    dec = np.full(len(pages), -1, np.int64)
    total = C.c_int64(-1)
    dlen = 0 if dict_off is None else dict_off.size - 1
    if not dev:
        bad = C.c_int64(-1)
        st, msg = ag.call_status("ag_parquet_byte_array_decode", enc, ow, ptr(blob), tbl, len(pages), n_slots, ptr(vbits),
                                 ptr(dict_off), ptr(dict_data), dlen, offset_base, ptr(offs), ptr(out) if cap else None, cap,
                                 C.byref(total), ptr(dec), C.byref(bad))
        return st, msg, offs.astype(np.int64), out, dec, total.value, bad.value
    db, do, dout, ddec, dbad = Dev(blob), Dev(offs), Dev(out), Dev(dec), Dev(np.array([-1], np.int64))
    dv = Dev(vbits) if vbits is not None else None
    ddo = Dev(dict_off) if dict_off is not None else None
    ddd = Dev(dict_data) if dict_data is not None else None
    st, msg = ag.call_status("ag_parquet_byte_array_decode_dev", enc, ow, db.ptr, tbl, len(pages), n_slots, dv.ptr if dv else None,
                             ddo.ptr if ddo else None, ddd.ptr if ddd else None, dlen, offset_base, do.ptr,
                             dout.ptr if cap else None, cap, C.byref(total), ddec.ptr, dbad.ptr, None)
    ag.call("ag_stream_sync", None)
    return st, msg, do.get().astype(np.int64), dout.get(), ddec.get(), total.value, int(dbad.get()[0])


def expect(enc, blob, pages, n_slots, valid=None, dictionary=None, offset_base=0):
    """oracle: (offsets, data, decoded, [(page index, message)], bad slot)"""
    placed, dec, errs, bad = [], [], [], None
    for k, (b, ln, nv, o) in enumerate(pages):
        v = nv if valid is None else valid[o:o + nv].copy()
        vals, slots, msg, bd = B.decode(enc, bytes(blob[b:b + ln]), v, dictionary)
        placed.append((o, vals))
        dec.append(slots)
        if msg:
            errs.append((k, msg))
        if bd is not None and (bad is None or o + bd < bad):
            bad = o + bd
    offs, data = B.arrow_buffers(n_slots, placed, offset_base)
    return offs, data, dec, errs, bad


def dict_buffers(dictionary, ow):
    lens = np.array([len(v) for v in dictionary], np.int64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32 if ow == 4 else np.int64)
    return off, np.frombuffer(b"".join(dictionary) + b"\0", np.uint8).copy()


def compare(ag, enc, ow, streams, rng, dev, frac=None, gap=True, dictionary=None):
    blob, pages, n_slots = batch(streams, rng, gap=gap)
    valid = vbits = None
    if frac is not None:
        valid = rng.random(n_slots + 64) >= frac
        vbits = np.packbits(valid, bitorder="little")
    doff = ddata = None
    if dictionary is not None:
        doff, ddata = dict_buffers(dictionary, ow)
    st, msg, offs, out, dec, total, bad = run_ba(ag, enc, ow, blob, pages, n_slots, vbits, doff, ddata, dev=dev)
    woffs, wdata, wdec, errs, wbad = expect(enc, blob, pages, n_slots, valid, dictionary)
    assert dec.tolist() == wdec, (msg, errs)
    assert offs.tolist() == woffs.tolist(), (msg, errs)
    assert total == len(wdata)
    assert out[:len(wdata)].tobytes() == wdata and (out[len(wdata):] == CANARY).all()
    return st, msg, errs, bad, wbad


def random_streams(rng, enc, long_values=False):
    streams = []
    for n in (1, 7, 1000, 5000):
        vals = F.random_strings(rng, n, sorted_keys=bool(rng.integers(0, 2)))
        streams.append((ENCODERS[enc](vals), n))
    streams.append((ENCODERS[enc]([b""] * 300), 300))                        # empty values only
    streams.append((ENCODERS[enc]([]), 0))
    if long_values:
        big = [bytes(rng.integers(0, 256, 20_000, dtype=np.uint8)), b"ab", bytes(rng.integers(0, 256, (1 << 20) + 77, dtype=np.uint8)), b""]
        streams.append((ENCODERS[enc](big + F.random_strings(rng, 50)), 54))
    return streams


@gpu
@FLAVOURS
@WIDTHS
@pytest.mark.parametrize("enc", [B.PLAIN, B.DELTA_LENGTH_BYTE_ARRAY, B.DELTA_BYTE_ARRAY], ids=["plain", "dlba", "dba"])
def test_random_pages(ag, enc, ow, dev):
    rng = np.random.default_rng(40 + enc + ow)
    streams = random_streams(rng, enc, long_values=True)
    for frac in (None, 0.3, 1.0):
        st, msg, errs, _, _ = compare(ag, enc, ow, streams, rng, dev, frac)
        if frac is not None and enc != B.PLAIN:
            continue                                                          # spaced pages with more valid slots than values
        assert st == N.AG_OK and not errs, msg
    seam = ENCODERS[enc](F.random_strings(rng, SEAM_SLOTS))
    st, msg, errs, _, _ = compare(ag, enc, ow, [(seam, SEAM_SLOTS)] * 2, rng, dev, 0.1)
    assert st == N.AG_OK and not errs, msg


@gpu
@FLAVOURS
@WIDTHS
def test_dictionary_pages(ag, ow, dev):
    rng = np.random.default_rng(41 + ow)
    import pq_ref as R
    dictionary = F.random_strings(rng, 400) + [b"", b"z" * 5000]
    streams = []
    for n in (1, 100, 3000, 20000):
        idx = rng.integers(0, len(dictionary), n)
        streams.append((bytes([9]) + R.rle_encode(idx, 9), n))
    seam = [(bytes([9]) + R.rle_encode(rng.integers(0, len(dictionary), SEAM_SLOTS), 9), SEAM_SLOTS)] * 2
    for frac, ss in ((None, streams), (0.25, streams), (0.1, seam)):
        st, msg, errs, bad, wbad = compare(ag, B.RLE_DICTIONARY, ow, ss, rng, dev, frac, dictionary=dictionary)
        assert st == N.AG_OK and not errs and bad == 2 ** 63 - 1 and wbad is None, msg
    bad_stream = bytes([9]) + R.rle_encode(np.array([1, 2, len(dictionary) + 3, 4]), 9)
    st, msg, errs, bad, wbad = compare(ag, B.RLE_DICTIONARY, ow, streams[:2] + [(bad_stream, 4)], rng, dev, gap=False, dictionary=dictionary)
    assert st == N.AG_ERR_INVALID and "invalid index values found for dictionary converter" in msg and bad == wbad


def error_cases():
    """(name, encoding, page bytes, num_values, null fraction)"""
    dl = B.dlba_encode([b"abc", b"de"])
    return [
        ("plain_empty_page", B.PLAIN, b"", 3, None),
        ("plain_empty_page_spaced", B.PLAIN, b"", 40, 0.2),
        ("plain_cut_length", B.PLAIN, B.plain_encode([b"a", b"bc"]) + b"\x01\x00", 3, None),
        ("plain_cut_value", B.PLAIN, B.plain_encode([b"a"] * 2000) + b"\x09\0\0\0abc", 2001, None),
        ("plain_negative", B.PLAIN, B.plain_encode([b"xy"] * 10) + b"\xfe\xff\xff\xff", 11, None),
        ("plain_cut_spaced", B.PLAIN, B.plain_encode([b"q"] * 50), 80, 0.1),
        ("dlba_negative", B.DELTA_LENGTH_BYTE_ARRAY, D.delta_encode([3, -1, 2], 4) + b"abcde", 3, None),
        ("dlba_exceed", B.DELTA_LENGTH_BYTE_ARRAY, dl[:-1], 2, None),
        ("dlba_header", B.DELTA_LENGTH_BYTE_ARRAY, b"\x80", 2, None),
        ("dlba_count", B.DELTA_LENGTH_BYTE_ARRAY, dl, 1, None),
        ("dlba_short_spaced", B.DELTA_LENGTH_BYTE_ARRAY, dl, 40, 0.0),
        ("dba_first_prefix", B.DELTA_BYTE_ARRAY, D.delta_encode([1, 0], 4) + B.dlba_encode([b"a", b"b"]), 2, None),
        ("dba_bad_prefix", B.DELTA_BYTE_ARRAY, D.delta_encode([0, 1, 1, 9, 0], 4) + B.dlba_encode([b"ab", b"c", b"d", b"e", b"f"]), 5, None),
        ("dba_bad_prefix_spaced", B.DELTA_BYTE_ARRAY, D.delta_encode([0, 1, 1, 9, 0], 4) + B.dlba_encode([b"ab", b"c", b"d", b"e", b"f"]), 9, 0.4),
        ("dba_negative_prefix", B.DELTA_BYTE_ARRAY, D.delta_encode([0, -1], 4) + B.dlba_encode([b"ab", b"c"]), 2, None),
        ("dba_count", B.DELTA_BYTE_ARRAY, D.delta_encode([0], 4) + B.dlba_encode([b"ab", b"c"]), 2, None),
        ("dba_suffix_exceed", B.DELTA_BYTE_ARRAY, D.delta_encode([0, 1], 4) + B.dlba_encode([b"ab", b"c"])[:-1], 2, None),
    ]


@gpu
@FLAVOURS
@pytest.mark.parametrize("case", error_cases(), ids=lambda c: c[0])
def test_error_cases(ag, case, dev):
    name, enc, stream, nv, frac = case
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    good = ENCODERS[enc](F.random_strings(rng, 500))
    for ow in (4, 8):
        st, msg, errs, _, _ = compare(ag, enc, ow, [(good, 500), (stream, nv), (stream, nv)], rng, dev, frac, gap=False)
        assert errs and errs[0][0] in (1, 2), errs                           # spaced: the validity decides what a page needs
        assert st == N.AG_ERR_INVALID and f"byte_array_decode: page {errs[0][0]}: {errs[0][1]} (" in msg, (msg, errs)


@gpu
@FLAVOURS
@pytest.mark.parametrize("enc", [B.PLAIN, B.DELTA_BYTE_ARRAY], ids=["plain", "dba"])
def test_capacity_and_size_query(ag, enc, dev):
    rng = np.random.default_rng(43)
    vals = F.random_strings(rng, 3000, sorted_keys=enc == B.DELTA_BYTE_ARRAY)
    blob, pages, n_slots = batch([(ENCODERS[enc](vals), 3000)], rng, gap=False)
    woffs, wdata, _, _, _ = expect(enc, blob, pages, n_slots, offset_base=5)
    for cap in (5 + len(wdata) - 1, 0):
        st, msg, offs, out, dec, total, _ = run_ba(ag, enc, 4, blob, pages, n_slots, offset_base=5, out_cap=cap, dev=dev)
        assert st == N.AG_OK, msg
        assert total == len(wdata) and offs.tolist() == woffs.tolist()
        assert (out == CANARY).all()
    st, msg, offs, out, dec, total, _ = run_ba(ag, enc, 8, blob, pages, n_slots, offset_base=5, out_cap=5 + len(wdata), dev=dev)
    assert st == N.AG_OK and out[5:].tobytes() == wdata and (out[:5] == CANARY).all()


@gpu
@FLAVOURS
def test_int32_overflow_writes_nothing(ag, dev):
    vals = [b"x" * 7] * 3
    blob = np.frombuffer(B.plain_encode(vals) + bytes(8), np.uint8).copy()
    base = 2 ** 31 - 10
    st, msg, offs, out, dec, total, _ = run_ba(ag, B.PLAIN, 4, blob, [(0, len(blob) - 8, 3, 0)], 3, offset_base=base, out_cap=base + 64 if not dev else 0, dev=dev)
    assert st == N.AG_ERR_INVALID and "int32" in msg
    assert (offs == -9).all() and (out == CANARY).all()
    st, msg, offs, out, dec, total, _ = run_ba(ag, B.PLAIN, 8, blob, [(0, len(blob) - 8, 3, 0)], 3, offset_base=base, out_cap=0, dev=dev)
    assert st == N.AG_OK and offs.tolist() == [base, base + 7, base + 14, base + 21] and total == 21


@gpu
def test_invalid_arguments(ag):
    blob = np.frombuffer(B.plain_encode([b"ab"]) + bytes(8), np.uint8).copy()
    offs = np.zeros(8, np.int64)
    for enc, ow in ((1, 4), (5, 8), (0, 2), (0, 16)):
        st, msg = ag.call_status("ag_parquet_byte_array_decode", enc, ow, ptr(blob), N.page_table([(0, 6, 1, 0)]), 1, 1, None, None,
                                 None, 0, 0, ptr(offs), None, 0, None, None, None)
        assert st == N.AG_ERR_INVALID, (enc, ow)
    st, msg = ag.call_status("ag_parquet_byte_array_decode", 0, 8, ptr(blob), N.page_table([(0, 6, 2, 0), (0, 6, 2, 1)]), 2, 4, None,
                             None, None, 0, 0, ptr(offs), None, 0, None, None, None)
    assert st == N.AG_ERR_INVALID and "overlap" in msg


def write_and_plan(path, rng, enc, nf, version, n, **kw):
    tbl = F.write_column(path, F.make_string_column(rng, enc, n, nf), nullable=nf is not None, encoding=enc, version=version, **kw)
    return tbl, P.chunk_plan(path)


def check_chunk(ag, tbl, plan, flavours=((4, True), (8, False))):
    """read the chunk with each (offset width, values through the host entry point) against pyarrow"""
    want, wvalid = F.expected(tbl, plan)
    for ow, host in flavours:
        values, valid = read_chunk_dev(ag, plan, offset_width=ow, host_values=host)
        assert np.array_equal(valid, wvalid)
        assert values == want, (ow, host)


@gpu
@pytest.mark.parametrize("case", F.ba_cases(), ids=F.case_id)
def test_pyarrow_files_end_to_end(ag, case, tmp_path):
    enc, nf, ver, ps = case
    rng = np.random.default_rng(zlib.crc32(F.case_id(case).encode()))
    check_chunk(ag, *write_and_plan(str(tmp_path / "c.parquet"), rng, enc, nf, ver, 8000, data_page_size=ps))


@gpu
def test_dictionary_fallback_chunk_chained(ag, tmp_path):
    rng = np.random.default_rng(44)
    tbl, plan = write_and_plan(str(tmp_path / "c.parquet"), rng, "RLE_DICTIONARY", 0.1, "1.0", 30_000, dictionary_pagesize_limit=2048)
    assert B.PLAIN in P.encodings(plan)
    check_chunk(ag, tbl, plan)


@gpu
@pytest.mark.parametrize("codec", ["snappy", "zstd"])
def test_compressed_string_chunks(ag, codec, tmp_path):
    rng = np.random.default_rng(45)
    for enc in F.BA_ENCODINGS:
        tbl, plan = write_and_plan(str(tmp_path / f"{enc}.parquet"), rng, enc, 0.1, "2.0", 20_000, compression=codec.upper())
        assert plan["codec"] == codec.upper()
        check_chunk(ag, tbl, plan, flavours=((8, False),))


@gpu
def test_large_batch_checksum(ag):
    """32M short strings in 2^19-value PLAIN pages, dense: the data buffer through the device checksum"""
    rng = np.random.default_rng(46)
    per_page, n_pages = 1 << 19, 64
    bodies = [F.random_strings(rng, per_page) for _ in range(2)]
    encs = [B.plain_encode(v) for v in bodies]
    blob, offs = bytearray(), []
    for e in encs:
        offs.append(len(blob))
        blob += e
    blob += bytes(16)
    pages = [(offs[p % 2], len(encs[p % 2]), per_page, p * per_page) for p in range(n_pages)]
    n = per_page * n_pages
    lens = [sum(len(v) for v in b) for b in bodies]
    total = sum(lens[p % 2] for p in range(n_pages))
    db, do, dout = Dev(np.frombuffer(bytes(blob), np.uint8).copy()), Dev(nbytes=8 * (n + 1)), Dev(nbytes=total + 64)
    t = C.c_int64(0)
    ag.call("ag_parquet_byte_array_decode_dev", B.PLAIN, 8, db.ptr, N.page_table(pages), n_pages, n, None, None, None, 0, 0,
            do.ptr, dout.ptr, total, C.byref(t), None, None, None)
    ag.call("ag_stream_sync", None)
    assert t.value == total
    data = b"".join(b"".join(bodies[p % 2]) for p in range(n_pages))
    words = np.frombuffer(data[:total // 8 * 8], np.uint64)
    res = Dev(np.zeros(1, np.uint64))
    ag.call("ag_checksum64_dev", dout.ptr, total // 8, res.ptr, None)
    ag.call("ag_stream_sync", None)
    assert int(res.get()[0]) == checksum64(words)
    got_off = do.get(np.int64, n + 1)
    assert got_off[-1] == total and got_off[per_page] == lens[0]


@gpu
@FLAVOURS
@pytest.mark.parametrize("case", GOLD["cases"], ids=lambda c: c["name"])
def test_reference_vectors(ag, case, dev):
    """the reference's test vectors, each page after a good one: the oracle's outcome, byte for byte"""
    rng = np.random.default_rng(zlib.crc32(case["name"].encode()))
    enc = case["encoding"]
    good = ENCODERS[enc](F.random_strings(rng, 300))
    for ow in (4, 8):
        st, msg, errs, _, _ = compare(ag, enc, ow, [(good, 300), (bytes(case["bytes"]), case["num_values"])], rng, dev, gap=False)
        if case["error"] is None:
            assert st == N.AG_OK and not errs, msg
        else:
            assert errs == [(1, case["error"])] and st == N.AG_ERR_INVALID and f"page 1: {case['error']} (" in msg, (msg, errs)
