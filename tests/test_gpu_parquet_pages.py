"""Device Parquet page decode (levels, dictionary, PLAIN spaced) against the Python restatement in tests/pq_ref.py,
host and _dev flavours, and pyarrow-written files end to end against pq.read_table."""
import ctypes as C
import zlib

import numpy as np
import pytest

import pq_files as F
import pq_pages as P
import pq_ref as R
from arrow_go_b200 import _native as N
from helpers import Dev, checksum64, ptr
from pq_chunk import read_chunk_dev
from pq_pages import batch

gpu = pytest.mark.gpu
# 300 tiles of 1024 slots, the last one partial: the one-block scan of a page's tile valid counts takes a full
# 256-tile step and a partial one
SEAM_SLOTS = 307_195


def run_dict(ag, width, dictionary, blob, pages, n_out, valid=None, dev=False):
    """-> (status, message, out, decoded, bad_pos)"""
    dt = np.int32 if width == 4 else np.int64
    tbl = N.page_table(pages)
    out = np.full(n_out, -7, dt)
    dec = np.full(len(pages), -1, np.int64)
    if not dev:
        bad = C.c_int64(-1)
        st, msg = ag.call_status("ag_parquet_dict_decode", width, ptr(dictionary), dictionary.size, ptr(blob), tbl, len(pages),
                                 ptr(valid), ptr(out), ptr(dec), C.byref(bad))
        return st, msg, out, dec, bad.value
    dd, db, dv = Dev(dictionary), Dev(blob), Dev(valid) if valid is not None else None
    do, ddec, dbad = Dev(out), Dev(dec), Dev(np.array([-1], np.int64))
    st, msg = ag.call_status("ag_parquet_dict_decode_dev", width, dd.ptr, dictionary.size, db.ptr, tbl, len(pages),
                             dv.ptr if dv else None, do.ptr, ddec.ptr, dbad.ptr, None)
    ag.call("ag_stream_sync", None)
    return st, msg, do.get(), ddec.get(), int(dbad.get()[0])


def run_levels(ag, max_level, enc, blob, pages, n_out, dev=False):
    tbl = N.page_table(pages)
    out = np.full(n_out, -7, np.int16)
    dec = np.full(len(pages), -1, np.int64)
    if not dev:
        st, msg = ag.call_status("ag_parquet_levels_decode", max_level, enc, ptr(blob), tbl, len(pages), ptr(out), ptr(dec))
        return st, msg, out, dec
    db, do, ddec = Dev(blob), Dev(out), Dev(dec)
    st, msg = ag.call_status("ag_parquet_levels_decode_dev", max_level, enc, db.ptr, tbl, len(pages), do.ptr, ddec.ptr, None)
    ag.call("ag_stream_sync", None)
    return st, msg, do.get(), ddec.get()


def expect_dict(blob, pages, n_out, dictionary, valid=None):
    want = np.full(n_out, -7, dictionary.dtype)
    dec, err, bad = [], R.ERR_NONE, None
    for (b, ln, nv, o) in pages:
        v = nv if valid is None else valid[o:o + nv].copy()
        vals, slots, e, bd = R.dict_decode(bytes(blob[b:b + ln]), dictionary, v)
        want[o:o + slots] = vals
        dec.append(slots)
        err = err or e
        if bd is not None and (bad is None or o + bd < bad):
            bad = o + bd
    return want, np.array(dec), err, bad


def streams_for_width(rng, bw):
    hi = 1 << min(bw, 20)
    out = []
    n = int(rng.integers(1, 5000))
    v = rng.integers(0, hi, n) if bw else np.zeros(n, np.int64)
    out.append(v)                                                               # random: mostly literal
    out.append(np.full(int(rng.integers(1, 3000)), int(rng.integers(0, hi))))  # all repeated
    out.append(np.arange(int(rng.integers(1, 2000))) % 2 * (hi > 1))           # alternating: one long literal
    k = int(rng.integers(10, 200))
    out.append(np.repeat(rng.integers(0, hi, k), rng.integers(1, 30, k)))      # mixed runs
    return [(R.rle_encode(x.tolist(), bw), x.size) for x in out]


@gpu
@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_dict_random_streams_every_width(ag, dev):
    rng = np.random.default_rng(21)
    dictionary = rng.integers(-(1 << 62), 1 << 62, 1 << 20)
    for width in (4, 8):
        d = dictionary.astype(np.int32 if width == 4 else np.int64)
        for bw in range(0, 33):
            streams = [(bytes([bw]) + s, nv) for s, nv in streams_for_width(rng, bw)]
            blob, pages, n_out = batch(streams, rng)
            st, msg, out, dec, bad = run_dict(ag, width, d, blob, pages, n_out, dev=dev)
            want, wdec, err, wbad = expect_dict(blob, pages, n_out, d)
            assert st == N.AG_OK and err == R.ERR_NONE, (bw, msg)
            assert dec.tolist() == wdec.tolist() and bad == N.NO_ERROR_POS, bw
            assert out.tobytes() == want.tobytes(), (width, bw)


@gpu
@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_levels_streams_and_odd_shapes(ag, dev):
    rng = np.random.default_rng(22)
    for max_level in (0, 1, 3, 255, 40000):
        bw = max_level.bit_length()
        hi = max_level + 1
        raw = []
        raw.append((R.literal_run(rng.integers(0, hi, 1000).tolist(), bw), 1000))           # literal run > 504 values
        raw.append((b"".join(R.repeated_run(int(x), 1, bw) for x in rng.integers(0, hi, 300)), 300))  # runs of count 1
        raw.append((R.rle_encode(rng.integers(0, hi, 101).tolist(), bw), 101))               # padded last group
        raw.append((R.rle_encode(rng.integers(0, hi, 64).tolist(), bw), 50))                 # page asks for fewer
        raw.append((R.rle_encode([1 % hi] * 20, bw), 40))                                    # stream ends early
        raw.append((b"", 0))                                                                 # empty
        raw.append((R.rle_encode([0] * 8, bw), 0))                                           # num_values 0
        for v1 in (False, True):
            streams = [((len(s).to_bytes(4, "little") + s) if v1 else s, nv) for s, nv in raw]
            if v1:
                streams[5] = (b"\0\0\0\0", 0)
            blob, pages, n_out = batch(streams, rng)
            enc = N.PQ_LEVELS_V1_RLE if v1 else N.PQ_LEVELS_V2_RLE
            st, msg, out, dec = run_levels(ag, max_level, enc, blob, pages, n_out, dev=dev)
            assert st == N.AG_OK, msg
            want = np.full(n_out, -7, np.int16)
            for k, (b, ln, nv, o) in enumerate(pages):
                lv, e = R.levels_decode_page(bytes(blob[b:b + ln]), max_level, v1, nv)
                assert e == R.ERR_NONE
                want[o:o + lv.size] = lv
                assert dec[k] == lv.size, (max_level, v1, k)
            assert out.tobytes() == want.tobytes(), (max_level, v1)


@gpu
@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_spaced_dict_and_plain_odd_offsets(ag, dev):
    rng = np.random.default_rng(23)
    dictionary = rng.integers(-(1 << 40), 1 << 40, 5000).astype(np.int64)
    for frac in (0.0, 0.1, 0.5, 1.0):
        slots = [int(x) for x in rng.integers(0, 4000, 6)] + [0, 7]
        if frac == 0.1:
            slots.insert(0, SEAM_SLOTS)
        n_total = sum(slots) + 100
        valid = rng.random(n_total) >= frac
        streams, plain, o = [], [], 3
        # pages are laid out by batch() at consecutive slot ranges starting at 3 without gaps
        for nv in slots:
            k = int(valid[o:o + nv].sum())
            streams.append((bytes([13]) + R.rle_encode(rng.integers(0, 5000, k).tolist(), 13), nv))
            plain.append((rng.integers(-(1 << 40), 1 << 40, k).astype(np.int64).tobytes(), nv))
            o += nv
        blob, pages, n_out = batch(streams, rng, gap=False)
        pages = [(b, ln, nv, o + 3) for (b, ln, nv, o) in pages]
        vbits = np.packbits(np.concatenate([valid, np.zeros(64, bool)]), bitorder="little")
        st, msg, out, dec, bad = run_dict(ag, 8, dictionary, blob, pages, n_out + 3, valid=vbits, dev=dev)
        want, wdec, err, wbad = expect_dict(blob, pages, n_out + 3, dictionary, valid=np.concatenate([valid, np.zeros(64, bool)]))
        assert st == N.AG_OK, msg
        assert dec.tolist() == wdec.tolist() and out.tobytes() == want.tobytes(), frac
        # PLAIN spaced, same slots
        pblob, ppages, _ = batch(plain, rng, gap=False)
        ppages = [(b, ln, nv, o + 3) for (b, ln, nv, o) in ppages]
        pout = np.full(n_out + 3, -7, np.int64)
        tbl = N.page_table(ppages)
        if dev:
            db, dv, do = Dev(pblob), Dev(vbits), Dev(pout)
            ag.call("ag_parquet_plain_decode_spaced_dev", 8, db.ptr, tbl, len(ppages), dv.ptr, do.ptr, None)
            ag.call("ag_stream_sync", None)
            pout = do.get()
        else:
            ag.call("ag_parquet_plain_decode_spaced", 8, ptr(pblob), tbl, len(ppages), ptr(vbits), ptr(pout))
        pwant = np.full(n_out + 3, -7, np.int64)
        for (b, ln, nv, o) in ppages:
            vals, e = R.plain_decode_spaced(bytes(pblob[b:b + ln]), np.int64, valid[o:o + nv])
            pwant[o:o + nv] = vals
        assert pout.tobytes() == pwant.tobytes(), frac


@gpu
def test_error_cases(ag):
    rng = np.random.default_rng(24)
    d = np.arange(16, dtype=np.int64)
    good = bytes([4]) + R.rle_encode(rng.integers(0, 16, 100).tolist(), 4)

    def dict_err(stream, nv, dev=False):
        blob, pages, n_out = batch([(good, 100), (stream, nv)], rng, gap=False)
        return run_dict(ag, 8, d, blob, pages, n_out, dev=dev)

    for stream, nv, text in ((b"\x04\x00", 8, "count of 0"), (b"\x04\x80\x80", 8, "varint"),
                             (b"\x04\x81\x80\x80\x80\x80\x01", 8, "varint"), (b"\x21\x02\x00", 8, "bit width")):
        st, msg, out, dec, bad = dict_err(stream, nv)
        assert st == N.AG_ERR_INVALID and "page 1" in msg and text in msg, msg
    # truncated repeated value (16-bit index, one byte left)
    st, msg, *_ = dict_err(b"\x10\x08\x01", 8)
    assert st == N.AG_ERR_INVALID and "repeated run value truncated" in msg
    # truncated literal runs deliver their whole 32-value groups (bit_reader_test.go:513-566), host and device
    for payload in (7, 4):
        for dev in (False, True):
            st, msg, out, dec, bad = dict_err(bytes([1, 17]) + b"\xff" * payload, 64, dev=dev)
            assert st == N.AG_ERR_INVALID and "page 1" in msg and "truncated" in msg and dec[1] == 32
            assert (out[100:132] == 1).all() and (out[132:164] == -7).all()
    # index out of range: lowest offending output slot, dense and spaced
    bad_stream = bytes([5]) + R.literal_run([1, 2, 20, 3, 17, 0, 0, 0], 5)
    for dev in (False, True):
        st, msg, out, dec, bad = dict_err(bad_stream, 8, dev=dev)
        assert st == N.AG_ERR_INVALID and "invalid index values found for dictionary converter" in msg and bad == 102
        assert out[102] == 0 and out[101] == 2
    blob, pages, n_out = batch([(bad_stream, 12)], rng, gap=False)
    valid = np.array([0, 1, 1, 0, 1, 1, 1, 1, 1, 1, 0, 0] + [0] * 20, bool)
    st, msg, out, dec, bad = run_dict(ag, 8, d, blob, pages, n_out, valid=np.packbits(valid, bitorder="little"))
    assert st == N.AG_ERR_INVALID and bad == 4
    # levels: v1 framing, bit width, BIT_PACKED
    for page, text in ((b"\x01\x00", "invalid levels"), (b"\x09\x00\x00\x00\x02\x01", "invalid number of bytes")):
        blob = np.frombuffer(page + bytes(8), np.uint8).copy()
        st, msg, *_ = run_levels(ag, 1, N.PQ_LEVELS_V1_RLE, blob, [(0, len(page), 4, 0)], 8)
        assert st == N.AG_ERR_INVALID and text in msg, msg
    blob = np.zeros(16, np.uint8)
    st, _, *_ = run_levels(ag, 1, N.PQ_LEVELS_BIT_PACKED, blob, [(0, 4, 4, 0)], 8)
    assert st == N.AG_ERR_NOT_IMPLEMENTED
    st, _, *_ = run_levels(ag, 1 << 16, N.PQ_LEVELS_V2_RLE, blob, [(0, 4, 4, 0)], 8)
    assert st == N.AG_ERR_INVALID
    # PLAIN page shorter than its valid slots
    pblob = np.zeros(64, np.uint8)
    vbits = np.full(8, 0xFF, np.uint8)
    pout = np.zeros(16, np.int64)
    st, msg = ag.call_status("ag_parquet_plain_decode_spaced", 8, ptr(pblob), N.page_table([(0, 40, 6, 0)]), 1, ptr(vbits), ptr(pout))
    assert st == N.AG_ERR_INVALID and "eof exception decode plain" in msg


@gpu
@pytest.mark.parametrize("case", F.cases(), ids=F.case_id)
def test_pyarrow_files_end_to_end(ag, case, tmp_path):
    rng = np.random.default_rng(zlib.crc32(F.case_id(case).encode()))
    path = str(tmp_path / "c.parquet")
    tbl = F.write_numeric_case(path, rng, ("dict",) + case)
    plan = P.chunk_plan(path)
    values, valid = read_chunk_dev(ag, plan)
    want, wvalid = F.expected(tbl, plan)
    assert np.array_equal(valid, wvalid)
    assert values == want
    if case[4]:
        assert P.PLAIN in P.encodings(plan)


@gpu
def test_dict_decode_100m_values_device(ag):
    """100M int64 values over ~1 MB pages of 17-bit dictionary indices (literal runs with repeated runs between them),
    10 % nulls: checked against the oracle on two windows of pages, and on the whole output through a checksum."""
    rng = np.random.default_rng(25)
    dictionary = rng.integers(-(1 << 62), 1 << 62, 100_000)
    per_page, n_pages = 1 << 19, 100_000_000 // (1 << 19)
    n = per_page * n_pages
    valid = rng.random(n) >= 0.1
    vbits = np.packbits(valid, bitorder="little")
    # a few distinct page bodies reused (encoding 100M values in Python is slow); each page gets its own slot range
    bodies = []
    for k in range(4):
        idx = rng.integers(0, 100_000, per_page)
        idx[1000 * k:1000 * k + 5000] = 7
        bodies.append(idx)
    blob, pages, encs = bytearray(), [], []
    for k in range(4):
        encs.append(bytes([17]) + R.rle_encode(bodies[k].tolist(), 17))
    offs = []
    for k in range(4):
        offs.append(len(blob))
        blob += encs[k]
    blob += bytes(16)
    pages = [(offs[p % 4], len(encs[p % 4]), per_page, p * per_page) for p in range(n_pages)]
    dd, db, dv = Dev(dictionary), Dev(np.frombuffer(bytes(blob), np.uint8).copy()), Dev(vbits)
    dout, ddec, dbad = Dev(nbytes=8 * n), Dev(np.zeros(n_pages, np.int64)), Dev(np.zeros(1, np.int64))
    ag.call("ag_parquet_dict_decode_dev", 8, dd.ptr, dictionary.size, db.ptr, N.page_table(pages), n_pages, dv.ptr, dout.ptr,
            ddec.ptr, dbad.ptr, None)
    ag.call("ag_stream_sync", None)
    assert (ddec.get() == per_page).all() and dbad.get()[0] == N.NO_ERROR_POS
    want_all = np.empty(n, np.int64)
    for p in range(n_pages):
        o = p * per_page
        vals, slots, e, bad = R.dict_decode(encs[p % 4], dictionary, valid[o:o + per_page])
        assert slots == per_page and e == R.ERR_NONE
        want_all[o:o + per_page] = vals
    for p in (0, 1, n_pages - 1):
        got = dout.buf.to_numpy(np.int64, per_page, 8 * p * per_page)
        assert np.array_equal(got, want_all[p * per_page:(p + 1) * per_page]), p
    res = Dev(np.zeros(1, np.uint64))
    ag.call("ag_checksum64_dev", dout.ptr, n, res.ptr, None)
    ag.call("ag_stream_sync", None)
    assert int(res.get()[0]) == checksum64(want_all.view(np.uint64))
