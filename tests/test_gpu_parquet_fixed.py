"""Device BOOLEAN and fixed-width page decode (PLAIN, dictionary, BYTE_STREAM_SPLIT; INT32 / INT64 / FLOAT / DOUBLE /
INT96 / FIXED_LEN_BYTE_ARRAY) against the Python restatement in tests/pq_fixed_ref.py, host and _dev flavours; pyarrow
files and the golden fixtures end to end against pq.read_table."""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

import pq_files as F
import pq_fixed_ref as X
import pq_pages as P
import pq_ref as R
from arrow_go_b200 import _native as N
from helpers import Dev, ptr
from pq_chunk import read_chunk_dev
from pq_pages import batch

gpu = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
CANARY = 0xA7
NO_ERROR_POS = (1 << 63) - 1
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TYPES = [(X.INT32, 4), (X.INT64, 8), (X.FLOAT, 4), (X.DOUBLE, 8), (X.INT96, 12)] + [(X.FLBA, w) for w in list(range(1, 41)) + [96, 3072]]


def run_fixed(ag, ptype, width, enc, blob, pages, n_out, vbits=None, dictionary=None, dev=False):
    """-> (status, message, out bytes (n_out * width), decoded, bad_pos).  The _dev flavour's output and dictionary
    sit at an odd byte offset when the width has no alignment requirement."""
    tl = width if ptype == X.FLBA else 0
    tbl = N.page_table(pages)
    out = np.full(n_out * width, CANARY, np.uint8)
    dec = np.full(len(pages), -1, np.int64)
    dd = None if dictionary is None else np.ascontiguousarray(dictionary, np.uint8).reshape(-1)
    dlen = 0 if dictionary is None else len(dictionary)
    if not dev:
        bad = C.c_int64(-1)
        st, msg = ag.call_status("ag_parquet_fixed_decode", ptype, tl, enc, ptr(blob), tbl, len(pages), ptr(vbits), ptr(dd), dlen,
                                 ptr(out), ptr(dec), C.byref(bad))
        return st, msg, out, dec, bad.value
    off = 0 if width in (4, 8) else 3
    db, do, ddec, dbad = Dev(blob), Dev(out, byte_offset=off), Dev(dec), Dev(np.array([-1], np.int64))
    dv = Dev(vbits) if vbits is not None else None
    ddict = Dev(dd, byte_offset=off) if dd is not None else None
    st, msg = ag.call_status("ag_parquet_fixed_decode_dev", ptype, tl, enc, db.ptr, tbl, len(pages), dv.ptr if dv else None,
                             ddict.ptr if ddict else None, dlen, do.ptr, ddec.ptr, dbad.ptr, None)
    ag.call("ag_stream_sync", None)
    return st, msg, do.get(), ddec.get(), int(dbad.get()[0])


def expect_fixed(ptype, width, enc, blob, pages, n_out, valid=None, dictionary=None):
    want = np.full(n_out * width, CANARY, np.uint8)
    dec, errs, bad = [], [], None
    for k, (b, ln, nv, o) in enumerate(pages):
        v = nv if valid is None else valid[o:o + nv].copy()
        rows, slots, msg, bd = X.fixed_decode(ptype, width, enc, bytes(blob[b:b + ln]), v, dictionary)
        want[o * width:(o + slots) * width] = np.asarray(rows, np.uint8).reshape(-1)
        dec.append(slots)
        if msg:
            errs.append((k, msg))
        if bd is not None and (bad is None or o + bd < bad):
            bad = o + bd
    return want, dec, errs, bad


def check_status(st, msg, fn, dec, errs):
    """the lowest failing page is named with its message and decoded count"""
    if errs:
        k, m = errs[0]
        assert st == N.AG_ERR_INVALID and f"{fn}: page {k}: {m} ({dec[k]} values decoded)" in msg, (msg, errs)
    else:
        assert st == N.AG_OK, msg


def compare_fixed(ag, ptype, width, enc, streams, rng, dev, frac=None, dictionary=None, gap=True):
    blob, pages, n_out = batch(streams, rng, gap=gap)
    valid = vbits = None
    if frac is not None:
        valid = rng.random(n_out + 64) >= frac
        vbits = np.packbits(valid, bitorder="little")
    st, msg, out, dec, bad = run_fixed(ag, ptype, width, enc, blob, pages, n_out, vbits, dictionary, dev)
    want, wdec, errs, wbad = expect_fixed(ptype, width, enc, blob, pages, n_out, valid, dictionary)
    assert dec.tolist() == wdec, (ptype, width, enc, msg, errs)
    assert out.tobytes() == want.tobytes(), (ptype, width, enc)
    if wbad is None:
        check_status(st, msg, "fixed_decode", wdec, errs)
        assert bad == NO_ERROR_POS, msg
    else:                                                        # a page error is reported before a bad index
        assert bad == wbad and st == N.AG_ERR_INVALID, msg
        if errs:
            check_status(st, msg, "fixed_decode", wdec, errs)
        else:
            assert f"fixed_decode: invalid index values found for dictionary converter (output slot {wbad})" in msg
    return st, msg


def fixed_streams(rng, width, enc, dict_len, counts=(1, 7, 1000, 2500)):
    streams = []
    for n in counts:
        if enc == X.PLAIN:
            streams.append((rng.integers(0, 256, n * width, dtype=np.uint8).tobytes(), n))
        elif enc == X.BYTE_STREAM_SPLIT:
            streams.append((X.bss_encode(rng.integers(0, 256, (n, width), dtype=np.uint8)), n))
        else:
            idx = np.repeat(rng.integers(0, dict_len, n), rng.integers(1, 12, n))[:n]
            streams.append((X.dict_encode(idx, bw=int(rng.integers(max(dict_len - 1, 1).bit_length(), 21))), n))
    streams.append((b"", 0))
    return streams


@gpu
@FLAVOURS
@pytest.mark.parametrize("enc", [X.PLAIN, X.RLE_DICTIONARY, X.BYTE_STREAM_SPLIT], ids=["plain", "dict", "bss"])
def test_random_pages_every_width(ag, enc, dev):
    rng = np.random.default_rng(60 + enc + dev)
    for ptype, width in TYPES:
        if enc == X.BYTE_STREAM_SPLIT and ptype == X.INT96:
            continue
        counts = (1, 7, 300) if width > 100 else (1, 7, 1000, 2500)
        dictionary = rng.integers(0, 256, (300, width), dtype=np.uint8) if enc == X.RLE_DICTIONARY else None
        streams = fixed_streams(rng, width, enc, 300, counts)
        for frac in (None, 0.3, 1.0):
            st, msg = compare_fixed(ag, ptype, width, enc, streams, rng, dev, frac, dictionary)
            assert st == N.AG_OK, (ptype, width, frac, msg)


@gpu
@FLAVOURS
def test_fixed_errors_and_bad_indices(ag, dev):
    rng = np.random.default_rng(70 + dev)
    cases = [
        (X.INT32, 4, X.BYTE_STREAM_SPLIT, (bytes(16), 1)),                  # data size too small
        (X.DOUBLE, 8, X.BYTE_STREAM_SPLIT, (bytes(12), 2)),                 # not aligned
        (X.FLBA, 5, X.BYTE_STREAM_SPLIT, (bytes(12), 3)),                   # not aligned, FLBA wording
        (X.INT32, 4, X.PLAIN, (bytes(10), 3)),
        (X.INT96, 12, X.PLAIN, (bytes(30), 3)),
        (X.FLBA, 7, X.PLAIN, (bytes(30), 5)),
        (X.FLBA, 7, X.RLE_DICTIONARY, (bytes([40]) + bytes(3), 5)),         # bit width > 32
        (X.INT64, 8, X.RLE_DICTIONARY, (bytes([3]) + b"\x00", 5)),          # zero run
        (X.FLBA, 3, X.RLE_DICTIONARY, (bytes([2]) + R.literal_run(list(range(4)) * 16, 2)[:5], 64)),   # truncated literal
    ]
    for ptype, width, enc, bad_stream in cases:
        dictionary = rng.integers(0, 256, (4, width), dtype=np.uint8) if enc == X.RLE_DICTIONARY else None
        if enc == X.RLE_DICTIONARY:
            streams = [(X.dict_encode([1, 2, 3, 0, 1]), 5), bad_stream, (X.dict_encode([3] * 40), 40)]
        elif enc == X.BYTE_STREAM_SPLIT:
            streams = [(X.bss_encode(rng.integers(0, 256, (10, width), dtype=np.uint8)), 10), bad_stream] + [(X.bss_encode(rng.integers(0, 256, (3, width), dtype=np.uint8)), 3)]
        else:
            streams = [(rng.integers(0, 256, 10 * width, dtype=np.uint8).tobytes(), 10), bad_stream]
        for frac in (None, 0.2):
            st, msg = compare_fixed(ag, ptype, width, enc, streams + [bad_stream], rng, dev, frac, dictionary)
            assert frac is not None or st == N.AG_ERR_INVALID, (ptype, width, enc, msg)
    # spaced BYTE_STREAM_SPLIT with fewer values than valid slots
    st, msg = compare_fixed(ag, X.FLOAT, 4, X.BYTE_STREAM_SPLIT, [(bytes(8), 6)], rng, dev, 0.0, gap=False)
    assert st == N.AG_ERR_INVALID and X.MSG_BSS_SHORT in msg
    # out-of-range indices: message, lowest slot, zeroed slot, for 4/8-byte and other widths
    for ptype, width in ((X.INT64, 8), (X.INT96, 12), (X.FLBA, 33)):
        dictionary = rng.integers(0, 256, (10, width), dtype=np.uint8)
        streams = [(X.dict_encode([1, 2, 3, 4]), 4), (X.dict_encode([9, 12, 1, 15]), 4), (X.dict_encode([0, 11]), 2)]
        for frac in (None, 0.3):
            st, msg = compare_fixed(ag, ptype, width, X.RLE_DICTIONARY, streams, rng, dev, frac, dictionary)


@gpu
def test_fixed_argument_checks(ag):
    blob = np.zeros(64, np.uint8)
    out = np.zeros(64, np.uint8)
    tbl = N.page_table([(0, 8, 2, 0)])
    for ptype, tl, enc in ((X.INT96, 0, X.BYTE_STREAM_SPLIT), (X.INT32, 0, 5), (X.INT64, 0, X.RLE), (X.FLBA, 0, X.PLAIN),
                           (X.FLBA, -3, X.PLAIN), (0, 0, X.PLAIN), (6, 0, X.PLAIN), (X.DOUBLE, 0, 7)):
        st, msg = ag.call_status("ag_parquet_fixed_decode", ptype, tl, enc, ptr(blob), tbl, 1, None, None, 0, ptr(out), None, None)
        assert st == N.AG_ERR_INVALID and "fixed_decode" in msg, (ptype, tl, enc, msg)
    for enc in (X.RLE_DICTIONARY, X.BYTE_STREAM_SPLIT, 5):
        st, msg = ag.call_status("ag_parquet_bool_decode", enc, ptr(blob), tbl, 1, None, ptr(out), None)
        assert st == N.AG_ERR_INVALID and "bool_decode" in msg, msg
    assert (out == 0).all()


# ------------------------------------------------------------------------------------------------------ BOOLEAN ----
def run_bool(ag, enc, blob, pages, init, vbits=None, dev=False, byte_offset=0):
    tbl = N.page_table(pages)
    dec = np.full(len(pages), -1, np.int64)
    if not dev:
        out = init.copy()
        st, msg = ag.call_status("ag_parquet_bool_decode", enc, ptr(blob), tbl, len(pages), ptr(vbits), ptr(out), ptr(dec))
        return st, msg, out, dec
    db, do, ddec = Dev(blob), Dev(init, byte_offset=byte_offset), Dev(dec)
    dv = Dev(vbits) if vbits is not None else None
    st, msg = ag.call_status("ag_parquet_bool_decode_dev", enc, db.ptr, tbl, len(pages), dv.ptr if dv else None, do.ptr, ddec.ptr, None)
    ag.call("ag_stream_sync", None)
    return st, msg, do.get(), ddec.get()


def expect_bool(enc, blob, pages, init, valid=None):
    bits = np.unpackbits(init, bitorder="little")
    dec, errs = [], []
    for k, (b, ln, nv, o) in enumerate(pages):
        v = nv if valid is None else valid[o:o + nv].copy()
        vals, slots, msg = X.bool_decode(enc, bytes(blob[b:b + ln]), v)
        bits[o:o + slots] = vals
        dec.append(slots)
        if msg:
            errs.append((k, msg))
    return np.packbits(bits, bitorder="little"), dec, errs


def compare_bool(ag, enc, streams, rng, dev, frac=None, gap=True):
    blob, pages, n_out = batch(streams, rng, gap=gap)
    init = rng.integers(0, 256, (n_out + 7) // 8 + 8, dtype=np.uint8)          # sentinel bits around and between pages
    valid = vbits = None
    if frac is not None:
        valid = rng.random(init.size * 8) >= frac
        vbits = np.packbits(valid, bitorder="little")
    for off in ((0, 1, 2, 3) if dev else (0,)):
        st, msg, out, dec = run_bool(ag, enc, blob, pages, init, vbits, dev, byte_offset=off)
        want, wdec, errs = expect_bool(enc, blob, pages, init, valid)
        assert dec.tolist() == wdec, (msg, errs)
        assert out.tobytes() == want.tobytes(), (enc, frac, off)
        check_status(st, msg, "bool_decode", wdec, errs)
    return st, msg


def bool_streams(rng, enc):
    enc_fn = X.bool_plain_encode if enc == X.PLAIN else X.bool_rle_encode
    streams = []
    for n in (1, 5, 31, 33, 1000, 1024, 5000, 20_000):
        streams.append((enc_fn(rng.random(n) < rng.random()), n))
    streams.append((enc_fn(np.ones(3000, bool)), 3000))
    streams.append((enc_fn(np.zeros(2000, bool)), 2000))
    streams.append((enc_fn(np.arange(1500) % 2 == 0), 1500))
    k = 200
    streams.append((enc_fn(np.repeat(rng.random(k) < 0.5, rng.integers(1, 40, k))[:3000]), 3000))
    streams.append((enc_fn([]), 0))
    if enc == X.RLE:
        # run forms a writer may not produce: a repeated byte of 2 (true), count-1 runs, a literal run after them
        s = R.repeated_run(2, 50, 1) + b"".join(R.repeated_run(int(v), 1, 1) for v in rng.integers(0, 2, 40)) + R.literal_run([1, 0, 0, 1] * 30, 1)
        streams.append((len(s).to_bytes(4, "little") + s, 210))
    return streams


@gpu
@FLAVOURS
@pytest.mark.parametrize("enc", [X.PLAIN, X.RLE], ids=["plain", "rle"])
def test_bool_pages_share_bytes_and_words(ag, enc, dev):
    rng = np.random.default_rng(80 + enc + dev)
    streams = bool_streams(rng, enc)
    for frac in (None, 0.3, 1.0):
        for gap in (True, False):
            st, msg = compare_bool(ag, enc, streams, rng, dev, frac, gap)
            assert st == N.AG_OK, msg


@gpu
@FLAVOURS
def test_bool_errors(ag, dev):
    rng = np.random.default_rng(90 + dev)
    good_p = (X.bool_plain_encode(rng.random(100) < 0.5), 100)
    good_r = (X.bool_rle_encode(rng.random(100) < 0.5), 100)
    for enc, good, bad in ((X.PLAIN, good_p, (b"\xff", 9)),
                           (X.RLE, good_r, (b"\x01\x00", 3)),
                           (X.RLE, good_r, (b"\x10\0\0\0\x01", 3)),
                           (X.RLE, good_r, (X.bool_rle_encode([1] * 20 + [0] * 5), 3000)),   # unexpected EOF after 25 values
                           (X.RLE, good_r, (b"\x01\0\0\0\x00", 5)),                          # zero run
                           (X.RLE, good_r, (b"\x02\0\0\0\x09\x01", 100))):                   # truncated literal
        for frac in (None, 0.4):
            st, msg = compare_bool(ag, enc, [good, bad, good, bad], rng, dev, frac)
            assert frac is not None or st == N.AG_ERR_INVALID, msg


# -------------------------------------------------------------------------------------------------- end to end ----
E2E = [(k, nf, v, c) for k in F.KINDS for nf in (None, 0.1, 1.0) for v in F.PAGE_VERSIONS for c in ("NONE", "SNAPPY", "ZSTD")
       if c == "NONE" or nf == 0.1]


@gpu
@pytest.mark.parametrize("case", E2E, ids=lambda c: F.case_id(c[:3]) + "-" + c[3])
def test_pyarrow_files_end_to_end(ag, case, tmp_path):
    kind, nf, ver, codec = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    path = str(tmp_path / "c.parquet")
    arr = F.make_array(rng, kind, 3000 if kind == "fsb1000" else 20_000, nf)
    tbl = F.write_column(path, arr, nullable=nf is not None, encoding=F.KINDS[kind], version=ver, compression=codec,
                         data_page_size=8192, dictionary_pagesize_limit=2048 if kind.endswith("_dict") else None)
    plan = P.chunk_plan(path)
    values, valid = read_chunk_dev(ag, plan)
    want, wvalid = F.expected(tbl, plan)
    assert np.array_equal(valid, wvalid)
    assert values == want


@gpu
@pytest.mark.parametrize("name,column", [("alltypes_plain.snappy.parquet", "bool_col"), ("alltypes_plain.snappy.parquet", "timestamp_col"),
                                         ("datapage_v2.snappy.parquet", "d"), ("byte_stream_split.zstd.parquet", "f32"),
                                         ("byte_stream_split.zstd.parquet", "f64")])
def test_golden_fixtures(ag, name, column):
    import pyarrow.parquet as pq
    path = os.path.join(GOLDEN, name)
    f = pq.ParquetFile(path)
    plan = P.chunk_plan(path, column=[f.schema.column(i).name for i in range(len(f.schema))].index(column))
    values, valid = read_chunk_dev(ag, plan)
    want, wvalid = F.expected(pq.read_table(path, columns=[column], coerce_int96_timestamp_unit="ns"), plan)
    assert np.array_equal(valid, wvalid)
    assert values == want


BIG = ["bss_double", "bss_double_spaced", "bss_flba16", "dict_flba16_spaced", "plain_int96_spaced", "plain_flba1000_spaced",
       "bool_plain", "bool_plain_spaced", "bool_rle", "bool_rle_spaced"]


@gpu
@pytest.mark.parametrize("kind", BIG)
def test_hundred_million_values(ag, kind):
    """~100M values per kind in 190 pages of 2^19 (FIXED_LEN_BYTE_ARRAY(1000): 400K values, 400 MB), spaced kinds with
    10 % nulls; four page bodies reused round-robin, every page writing its own slots; compared through a checksum"""
    rng = np.random.default_rng(zlib.crc32(kind.encode()))
    width = {"bss_double": 8, "bss_double_spaced": 8, "bss_flba16": 16, "dict_flba16_spaced": 16, "plain_int96_spaced": 12,
             "plain_flba1000_spaced": 1000}.get(kind, 0)
    per, n_pages = (1 << 12, 100) if width == 1000 else (1 << 19, 190)
    n = per * n_pages
    spaced = kind.endswith("_spaced")
    valid = rng.random(n) >= 0.1 if spaced else None
    counts = valid.reshape(n_pages, per).sum(axis=1) if spaced else np.full(n_pages, per)
    dictionary = None
    if kind.startswith("bool"):
        enc = X.PLAIN if "plain" in kind else X.RLE
        rows = [(rng.random(per) < 0.5).astype(np.uint8) for _ in range(4)]
        bodies = [X.bool_plain_encode(r) if enc == X.PLAIN else X.bool_rle_encode(r) for r in rows]
    else:
        ptype = {8: X.DOUBLE, 12: X.INT96}.get(width, X.FLBA)
        rows = [rng.integers(0, 256, (per, width), dtype=np.uint8) for _ in range(4)]
        if kind.startswith("bss"):
            enc, bodies = X.BYTE_STREAM_SPLIT, [X.bss_encode(r) for r in rows]
        elif kind.startswith("dict"):
            dictionary = rng.integers(0, 256, (1 << 16, width), dtype=np.uint8)
            idx = [rng.integers(0, 1 << 16, per) for _ in range(4)]
            enc, bodies, rows = X.RLE_DICTIONARY, [X.dict_encode(i, bw=16) for i in idx], [dictionary[i] for i in idx]
        else:
            enc, bodies = X.PLAIN, [r.tobytes() for r in rows]
    offs = np.cumsum([0] + [len(b) for b in bodies])
    blob = np.frombuffer(b"".join(bodies) + bytes(16), np.uint8).copy()
    pages = [(int(offs[k % 4]), len(bodies[k % 4]), per, k * per) for k in range(n_pages)]
    want = np.zeros((n, width) if width else n, np.uint8)
    for k in range(n_pages):
        seg = want[k * per:(k + 1) * per]
        if spaced:
            seg[valid[k * per:(k + 1) * per]] = rows[k % 4][:counts[k]]
        else:
            seg[:] = rows[k % 4]
    db = Dev(blob)
    dv = Dev(np.packbits(valid, bitorder="little")) if spaced else None
    vp = dv.ptr if dv else None
    if not width:
        do = Dev(np.zeros(n // 8 + 8, np.uint8))
        ag.call("ag_parquet_bool_decode_dev", enc, db.ptr, N.page_table(pages), n_pages, vp, do.ptr, None, None)
        ag.call("ag_stream_sync", None)
        got, want = do.get()[:n // 8], np.packbits(want, bitorder="little")
    else:
        do = Dev(nbytes=n * width)
        dd = Dev(dictionary) if dictionary is not None else None
        ag.call("ag_parquet_fixed_decode_dev", ptype, width if ptype == X.FLBA else 0, enc, db.ptr, N.page_table(pages), n_pages, vp,
                dd.ptr if dd else None, 0 if dictionary is None else len(dictionary), do.ptr, None, None, None)
        ag.call("ag_stream_sync", None)
        got = do.get(np.uint8, n * width)
    assert zlib.crc32(got.tobytes()) == zlib.crc32(want.tobytes()), kind
