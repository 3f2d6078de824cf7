"""Device DELTA_BINARY_PACKED page decode (INT32 / INT64) against the Python restatement in tests/pq_delta_ref.py, host and
_dev flavours, byte for byte; pyarrow-written files end to end against pq.read_table; 100M values through a checksum."""
import json
import os
import zlib

import numpy as np
import pytest

import pq_delta_ref as D
import pq_files as F
import pq_pages as P
from arrow_go_b200 import _native as N
from helpers import Dev, checksum64, ptr
from pq_chunk import read_chunk_dev
from pq_pages import batch

gpu = pytest.mark.gpu
SHAPES = ((128, 4), (256, 4), (128, 1), (1024, 8), (4096, 1))   # values per miniblock 32, 64, 128, 128, 4096
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "parquet_delta.json")))
# 300 tiles of 1024 slots, the last one partial: the one-block scans over a page's tiles take a full 256-tile step and
# a partial one
SEAM_SLOTS = 307_195


def run_delta(ag, width, blob, pages, n_out, vbits=None, dev=False):
    """-> (status, message, out, decoded); out starts as -7 everywhere"""
    dt = np.int32 if width == 4 else np.int64
    tbl = N.page_table(pages)
    out = np.full(n_out, -7, dt)
    dec = np.full(len(pages), -1, np.int64)
    if not dev:
        st, msg = ag.call_status("ag_parquet_delta_decode", width, ptr(blob), tbl, len(pages), ptr(vbits), ptr(out), ptr(dec))
        return st, msg, out, dec
    db, do, ddec = Dev(blob), Dev(out), Dev(dec)
    dv = Dev(vbits) if vbits is not None else None
    st, msg = ag.call_status("ag_parquet_delta_decode_dev", width, db.ptr, tbl, len(pages), dv.ptr if dv else None, do.ptr, ddec.ptr, None)
    ag.call("ag_stream_sync", None)
    return st, msg, do.get(), ddec.get()


def expect(width, blob, pages, n_out, valid=None):
    """oracle: (out, decoded, [(page index, message)] of failing pages)"""
    want = np.full(n_out, -7, np.int32 if width == 4 else np.int64)
    dec, errs = [], []
    for k, (b, ln, nv, o) in enumerate(pages):
        v = nv if valid is None else valid[o:o + nv].copy()
        vals, slots, e, msg = D.delta_decode(bytes(blob[b:b + ln]), width, v)
        want[o:o + slots] = vals
        dec.append(slots)
        if e:
            errs.append((k, msg))
    return want, np.array(dec), errs


def decode_and_compare(ag, width, streams, rng, dev, frac=None, gap=True):
    """decode `streams` [(bytes, num_values)] as one batch (dense, or spaced with a null fraction) and compare with
    the oracle; returns (status, message, oracle errors)"""
    blob, pages, n_out = batch(streams, rng, gap=gap)
    valid = vbits = None
    if frac is not None:
        valid = rng.random(n_out + 64) >= frac
        vbits = np.packbits(valid, bitorder="little")
    st, msg, out, dec = run_delta(ag, width, blob, pages, n_out, vbits, dev)
    want, wdec, errs = expect(width, blob, pages, n_out, valid)
    assert dec.tolist() == wdec.tolist(), (msg, errs)
    assert out.tobytes() == want.tobytes(), (msg, errs)
    return st, msg, errs


def values_with_delta_width(rng, width, bw, n):
    """n values whose consecutive deltas are uniform over bw bits (wrapping at the type width)"""
    ut = np.uint32 if width == 4 else np.uint64
    if bw == 0:
        d = np.zeros(n, ut)
    elif bw == 64:
        d = rng.integers(0, 1 << 63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
    else:
        d = rng.integers(0, 1 << bw, n, dtype=np.uint64).astype(ut)
    with np.errstate(over="ignore"):
        v = np.cumsum(d, dtype=ut) + ut(int(rng.integers(0, 1 << 62)) & ((1 << (8 * width)) - 1))
    return v.view(np.int32 if width == 4 else np.int64)


@gpu
@FLAVOURS
@pytest.mark.parametrize("width", [4, 8], ids=["int32", "int64"])
def test_random_streams_every_bit_width(ag, width, dev):
    rng = np.random.default_rng(31 + width)
    for bw in range(0, 8 * width + 1):
        streams = []
        for block, mini in SHAPES:
            n = int(rng.integers(1, 3000)) if block < 4096 else int(rng.integers(4000, 9000))
            streams.append((D.delta_encode(values_with_delta_width(rng, width, bw, n), width, block, mini), n))
        for frac in (None, 0.3):
            st, msg, errs = decode_and_compare(ag, width, streams, rng, dev, frac)
            assert st == N.AG_OK and not errs, (bw, frac, msg)
    seam = [(D.delta_encode(values_with_delta_width(rng, width, 8 * width - 3, SEAM_SLOTS), width), SEAM_SLOTS)]
    st, msg, errs = decode_and_compare(ag, width, seam, rng, dev, 0.1)
    assert st == N.AG_OK and not errs, msg


@gpu
@FLAVOURS
def test_wrapped_deltas(ag, dev):
    rng = np.random.default_rng(32)
    alt64 = np.where(np.arange(3000) % 2 == 0, np.iinfo(np.int64).min, np.iinfo(np.int64).max)
    alt32 = np.where(np.arange(3000) % 2 == 0, np.iinfo(np.int32).min, np.iinfo(np.int32).max).astype(np.int32)
    i32min, i32max = -2**31, 2**31 - 1
    boundary = [0, i32min, -1, i32max, -2, i32max - 1, i32max - 1, i32min + 1, 0, 1, i32min, i32max, i32min]
    for width, vals in ((8, alt64), (4, alt32), (4, np.array(boundary, np.int32))):
        streams = [(D.delta_encode(vals, width, b, m), vals.size) for b, m in SHAPES]
        for frac in (None, 0.5):
            st, msg, errs = decode_and_compare(ag, width, streams, rng, dev, frac)
            assert st == N.AG_OK and not errs, msg
        st, msg, out, dec = run_delta(ag, width, *batch(streams[:1], rng, gap=False), dev=dev)
        assert out[:vals.size].tolist() == vals.tolist()


@gpu
@FLAVOURS
def test_edge_cases(ag, dev):
    rng = np.random.default_rng(33)
    vals = (np.arange(10_000, dtype=np.int64) * 37) % 1001 - 500
    enc = D.delta_encode(vals[:300], 8)                                        # 128/4, 6-byte header
    b1 = len(D.delta_encode(vals[:129], 8))                                    # block 1 starts here
    enc140 = bytearray(D.delta_encode(vals[:140], 8))
    w0 = D._uvarint(enc140, b1)[1]                                             # block 1's width bytes
    enc140[w0 + 1:w0 + 4] = b"\xff\xff\xff"                                    # garbage widths of unused miniblocks
    enc4k = D.delta_encode(vals, 8, 4096, 1)
    cut4k = enc4k[:len(D.delta_encode(vals[:4097], 8, 4096, 1))]              # exactly one 4096-value block
    dense = [
        (D.delta_encode(vals[:100], 8), 150),       # total < num_values: a short count
        (D.delta_encode([], 8), 5),                 # total 0
        (D.delta_encode([], 8), 0),                 # num_values 0
        (D.delta_encode(vals[:1], 8), 1),           # header only
        (bytes(enc140), 140),
        (enc, 300),
    ]
    st, msg, errs = decode_and_compare(ag, 8, dense, rng, dev)
    assert st == N.AG_OK and not errs, msg
    # spaced: need < total, and streams that end right after the last needed miniblock / at a block boundary
    for stream, total, need in ((enc[:b1], 300, 129), (enc, 300, 200), (cut4k, 10_000, 4097), (enc4k, 10_000, 5000)):
        valid = np.zeros(total + 64, bool)
        valid[np.sort(rng.choice(total, need, replace=False))] = True
        blob, pages, n_out = batch([(stream, total)], rng, gap=False)
        st, msg, out, dec = run_delta(ag, 8, blob, pages, n_out, np.packbits(valid, bitorder="little"), dev)
        want, wdec, errs = expect(8, blob, pages, n_out, valid)
        assert st == N.AG_OK and not errs, msg
        assert dec.tolist() == wdec.tolist() == [total] and out.tobytes() == want.tobytes()


def error_cases():
    """(name, width, page bytes, num_values, null fraction or None)"""
    out = [(c["name"], c["width"], bytes(c["bytes"]), c["num_values"], None) for c in GOLD["decode"]]
    vals = np.arange(200, dtype=np.int64) ** 2
    wide = bytearray(D.delta_encode(vals, 8))
    wide[6 + 1 + 2] = 70                                                       # block 0, miniblock 2: width 70
    blk1 = bytearray(D.delta_encode(vals, 8))
    b1 = len(D.delta_encode(vals[:129], 8))
    out += [
        ("empty_page", 4, b"", 1, None),
        ("truncated_header_varint", 4, b"\x80", 1, None),
        ("header_varint_over_64_bits", 8, b"\x80" * 9 + b"\x02", 1, None),
        ("bad_header_with_no_values", 4, b"\x00", 0, None),
        ("min_delta_missing", 8, bytes([128, 1, 4, 2, 0]), 2, None),
        ("width_bytes_cut", 8, bytes([128, 1, 4, 2, 0, 0, 1]), 2, None),
        ("block_1_min_delta_cut", 8, bytes(blk1[:b1]), 200, None),
        ("width_70_dense", 8, bytes(wide), 200, None),
        ("width_70_spaced", 8, bytes(wide), 200, 0.2),
        ("truncated_miniblock_spaced", 8, bytes([128, 8, 1, 129, 8, 0, 0, 1, 0, 0, 0, 0]), 1025, 0.1),
        ("spaced_fewer_values_than_valid_slots", 4, D.delta_encode(np.arange(10), 4), 20, 0.0),
    ]
    return out


@gpu
@FLAVOURS
@pytest.mark.parametrize("case", error_cases(), ids=lambda c: c[0])
def test_error_cases(ag, case, dev):
    name, width, stream, nv, frac = case
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    good = D.delta_encode(np.arange(500) * 3 - 7, width)
    st, msg, errs = decode_and_compare(ag, width, [(good, 500), (stream, nv)], rng, dev, frac, gap=False)
    assert len(errs) == 1 and errs[0][0] == 1, errs
    assert st == N.AG_ERR_INVALID and f"delta_decode: page 1: {errs[0][1]} (" in msg, (msg, errs)


@gpu
def test_invalid_arguments(ag):
    blob = np.frombuffer(D.delta_encode([1, 2, 3], 4) + bytes(8), np.uint8).copy()
    out = np.zeros(8, np.int64)
    for w in (0, 2, 16):
        st, msg = ag.call_status("ag_parquet_delta_decode", w, ptr(blob), N.page_table([(0, 10, 3, 0)]), 1, None, ptr(out), None)
        assert st == N.AG_ERR_INVALID and "value_width" in msg
    dout = Dev(nbytes=64)
    st, msg = ag.call_status("ag_parquet_delta_decode_dev", 8, Dev(blob).ptr, N.page_table([(0, 10, 3, 0)]), 1, None, dout.ptr + 4, None, None)
    assert st == N.AG_ERR_INVALID and "aligned" in msg


@gpu
@pytest.mark.parametrize("case", F.delta_cases(), ids=F.case_id)
def test_pyarrow_delta_files_end_to_end(ag, case, tmp_path):
    rng = np.random.default_rng(zlib.crc32(F.case_id(case).encode()))
    path = str(tmp_path / "c.parquet")
    tbl = F.write_numeric_case(path, rng, ("delta",) + case + (None,))
    plan = P.chunk_plan(path)
    values, valid = read_chunk_dev(ag, plan)
    want, wvalid = F.expected(tbl, plan)
    assert P.encodings(plan) == {P.DELTA_BINARY_PACKED} and plan["dict"] is None
    assert np.array_equal(valid, wvalid)
    assert values == want


@gpu
def test_delta_decode_100m_values_device(ag):
    """100M int64 timestamps-like values in 2^19-value pages (256/4 blocks), 10 % nulls: two windows of pages against
    the oracle, the whole output through a checksum."""
    rng = np.random.default_rng(34)
    per_page, n_pages = 1 << 19, 100_000_000 // (1 << 19)
    n = per_page * n_pages
    valid = rng.random(n) >= 0.1
    vbits = np.packbits(valid, bitorder="little")
    bodies, encs = [], []
    for k in range(4):                                         # a few page bodies reused; each page has its own slots
        v = np.cumsum(rng.integers(0, 1000, per_page)) + (k << 40)
        v[rng.integers(0, per_page, 8)] = rng.integers(-(1 << 62), 1 << 62, 8)
        bodies.append(v)
        encs.append(D.delta_encode(v, 8, 256, 4))
    blob, offs = bytearray(), []
    for e in encs:
        offs.append(len(blob))
        blob += e
    blob += bytes(16)
    pages = [(offs[p % 4], len(encs[p % 4]), per_page, p * per_page) for p in range(n_pages)]
    db, dv = Dev(np.frombuffer(bytes(blob), np.uint8).copy()), Dev(vbits)
    dout, ddec = Dev(nbytes=8 * n), Dev(np.zeros(n_pages, np.int64))
    ag.call("ag_parquet_delta_decode_dev", 8, db.ptr, N.page_table(pages), n_pages, dv.ptr, dout.ptr, ddec.ptr, None)
    ag.call("ag_stream_sync", None)
    assert (ddec.get() == per_page).all()
    for k in range(4):                                         # the oracle's dense decode of every body
        vals, slots, e, _ = D.delta_decode(encs[k], 8, per_page)
        assert e == D.DERR_NONE and np.array_equal(vals, bodies[k])
    want_all = np.zeros(n, np.int64)
    for p in range(n_pages):                                   # spaced = the page's first `need` values at its valid slots
        o = p * per_page
        m = valid[o:o + per_page]
        want_all[o:o + per_page][m] = bodies[p % 4][:int(m.sum())]
    for p in (0, 1, n_pages - 1):
        o = p * per_page
        vals, slots, e, _ = D.delta_decode(encs[p % 4], 8, valid[o:o + per_page].copy())
        assert e == D.DERR_NONE and slots == per_page and np.array_equal(vals, want_all[o:o + per_page])
        got = dout.buf.to_numpy(np.int64, per_page, 8 * o)
        assert np.array_equal(got, want_all[o:o + per_page]), p
    res = Dev(np.zeros(1, np.uint64))
    ag.call("ag_checksum64_dev", dout.ptr, n, res.ptr, None)
    ag.call("ag_stream_sync", None)
    assert int(res.get()[0]) == checksum64(want_all.view(np.uint64))
