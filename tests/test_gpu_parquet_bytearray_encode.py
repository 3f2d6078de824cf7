"""Device BYTE_ARRAY page encoders, host and _dev flavours, offset widths 4 and 8, byte for byte against the
restatements (pq_bytearray_ref.plain_encode / dlba_encode / dba_encode) with guard bytes around every page section:
page sizes around the tile edges, shuffled pages with gaps, shared slots, null slots with nonzero lengths, values past
64 KiB, empty and repeated values; pyarrow's own column buffers encoded into its files' value sections; round trips
through the device decoder; every error with nothing written; and one batch past 2^31 data and output bytes."""
import ctypes as C

import numpy as np
import pytest

import pq_bytearray_ref as B
import pq_files as F
import pq_pages as P
from arrow_go_b200 import _native as N
from helpers import Dev, ptr

pytestmark = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
WIDTHS = pytest.mark.parametrize("ow", [4, 8])
ENCS = pytest.mark.parametrize("enc", [B.PLAIN, B.DELTA_LENGTH_BYTE_ARRAY, B.DELTA_BYTE_ARRAY], ids=["plain", "dlba", "dba"])
EXPECT = {B.PLAIN: B.plain_encode, B.DELTA_LENGTH_BYTE_ARRAY: B.dlba_encode, B.DELTA_BYTE_ARRAY: B.dba_encode}
GUARD = 0xA5


def bound(ag, enc, n, span):
    s = C.c_int64()
    ag.call("ag_parquet_byte_array_max_size", enc, n, span, C.byref(s))
    return s.value


def arrow(vals, ow):
    """values -> (offsets, data) of an Arrow Binary (ow 4) or LargeBinary (ow 8) array"""
    lens = np.array([len(v) for v in vals], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32 if ow == 4 else np.int64)
    data = np.frombuffer(b"".join(vals) + b"\0", np.uint8).copy()
    return offsets, data


def layout(ag, enc, offsets, spans, rng, gap=True):
    """[(in, n)] -> pages [(in, n, out, capacity)] with outputs in shuffled order at odd offsets with gaps; bytes"""
    order = rng.permutation(len(spans)) if gap else np.arange(len(spans))
    outs, pos = {}, 0
    for k in order:
        pos += int(rng.integers(1, 19)) if gap else 0
        i0, n = spans[k]
        outs[k] = (pos, bound(ag, enc, n, int(offsets[i0 + n]) - int(offsets[i0])))
        pos += outs[k][1]
    return [(i0, n, *outs[k]) for k, (i0, n) in enumerate(spans)], pos + 8


def encode(ag, enc, ow, offsets, data, valid, pages, n_out, dev):
    """-> (status, message, out bytes, lengths, bad_pos)"""
    tbl = N.enc_page_table(pages)
    out = np.full(n_out + 64, GUARD, np.uint8)
    lens = np.full(len(pages), -1, np.int64)
    bp = np.full(1, -5, np.int64)
    vb = None if valid is None else np.packbits(valid, bitorder="little")
    if not dev:
        st, msg = ag.call_status("ag_parquet_byte_array_encode", enc, ow, ptr(offsets), ptr(data), ptr(vb), tbl, len(pages),
                                 ptr(out), ptr(lens), ptr(bp))
        return st, msg, out, lens, int(bp[0])
    do, dd, dv, dout, dl, db = Dev(offsets), Dev(data), None if vb is None else Dev(vb), Dev(out), Dev(lens), Dev(bp)
    st, msg = ag.call_status("ag_parquet_byte_array_encode_dev", enc, ow, do.ptr, dd.ptr, None if dv is None else dv.ptr, tbl,
                             len(pages), dout.ptr, dl.ptr, db.ptr, None)
    ag.call("ag_stream_sync", None)
    return st, msg, dout.get(), dl.get(), int(db.get()[0])


def expected(enc, vals, valid, i0, n):
    return EXPECT[enc]([vals[s] for s in range(i0, i0 + n) if valid is None or valid[s]])


def check(ag, enc, ow, vals, valid, spans, rng, dev, gap=True):
    offsets, data = arrow(vals, ow)
    pages, n_out = layout(ag, enc, offsets, spans, rng, gap)
    st, msg, out, lens, bad = encode(ag, enc, ow, offsets, data, valid, pages, n_out, dev)
    assert st == N.AG_OK, msg
    assert bad == N.NO_ERROR_POS
    written = np.zeros(out.size, bool)
    for k, (i0, n, o, cap) in enumerate(pages):
        want = expected(enc, vals, valid, i0, n)
        assert lens[k] == len(want), (k, i0, n)
        assert out[o:o + len(want)].tobytes() == want, (k, i0, n)
        written[o:o + len(want)] = True
    assert (out[~written] == GUARD).all()
    return pages, out, lens


def strings(rng, n, null_lengths=True):
    vals = F.random_strings(rng, n)
    valid = rng.random(n) >= 0.1
    if not null_lengths:
        vals = [v if ok else b"" for v, ok in zip(vals, valid)]
    return vals, valid


@ENCS
@WIDTHS
@FLAVOURS
def test_page_sizes_around_tile_edges(ag, enc, ow, dev):
    rng = np.random.default_rng(enc * 10 + ow + dev)
    sizes = [0, 1, 2, 3, 255, 256, 1023, 1024, 1025, 2047, 2048, 2049, 4097, 100_000]
    vals, valid = strings(rng, sum(sizes) + 8 * len(sizes) + 13)
    spans, i0 = [], 5                                   # first slots that are not multiples of 8, gaps between pages
    for n in sizes:
        spans.append((i0, n))
        i0 += n + int(rng.integers(0, 8))
    check(ag, enc, ow, vals, valid, spans, rng, dev)
    check(ag, enc, ow, vals, None, spans, rng, dev)


@ENCS
@WIDTHS
@FLAVOURS
def test_shared_slots_and_sorted_keys(ag, enc, ow, dev):
    rng = np.random.default_rng(7 + enc + ow)
    vals = F.random_strings(rng, 9000, sorted_keys=True)
    valid = rng.random(9000) >= 0.2
    valid[1030:3100] = False                            # whole null tiles: the previous value comes from two tiles back
    spans = [(0, 9000), (1000, 5000), (1000, 5000), (4093, 1), (8999, 1), (3, 2049)]
    check(ag, enc, ow, vals, valid, spans, rng, dev)


@ENCS
@FLAVOURS
def test_long_equal_and_empty_values(ag, enc, dev):
    rng = np.random.default_rng(3)
    big = bytes(rng.integers(0, 256, 200_000, dtype=np.uint8))
    vals = [b"", big, big, big[:70_000], big[:70_000] + b"x", b"", b"", big[5:], b"a" * 65_537, b"a" * 65_537, b"b"]
    vals = vals * 3 + [bytes(rng.integers(0, 256, int(m), dtype=np.uint8)) for m in rng.integers(0, 40, 3000)]
    valid = np.ones(len(vals), bool)
    valid[[2, 14, 20]] = False
    check(ag, enc, 8, vals, valid, [(0, len(vals)), (1, 10), (6, 30), (0, 1)], rng, dev)
    check(ag, enc, 4, vals, None, [(0, len(vals)), (2, 5)], rng, dev)


@pytest.mark.parametrize("encoding", ["PLAIN", "DELTA_LENGTH_BYTE_ARRAY", "DELTA_BYTE_ARRAY"])
@pytest.mark.parametrize("large", [False, True], ids=["binary", "large_binary"])
@FLAVOURS
def test_pyarrow_column_end_to_end(ag, tmp_path, encoding, large, dev):
    pa = pytest.importorskip("pyarrow")
    rng = np.random.default_rng(len(encoding) + large)
    n = 30_000
    vals = F.random_strings(rng, n, sorted_keys=encoding == "DELTA_BYTE_ARRAY")
    valid = rng.random(n) >= 0.1
    arr = pa.array(vals, type=pa.large_binary() if large else pa.binary(), mask=~valid)
    path = str(tmp_path / "s.parquet")
    F.write_column(path, arr, nullable=True, encoding=encoding, version="2.0", data_page_size=1 << 13)
    plan = P.chunk_plan(path)
    dst = P.host_decompress(plan)
    sections = P.value_sections(plan, dst)
    assert len(sections) > 3
    ow = 8 if large else 4
    vbuf, obuf, dbuf = arr.buffers()
    offsets = np.frombuffer(obuf, np.int32 if ow == 4 else np.int64)[:n + 1].copy()
    data = np.frombuffer(dbuf, np.uint8).copy()
    vbits = np.unpackbits(np.frombuffer(vbuf, np.uint8), bitorder="little")[:n].astype(bool)
    enc = {"PLAIN": B.PLAIN, "DELTA_LENGTH_BYTE_ARRAY": B.DELTA_LENGTH_BYTE_ARRAY, "DELTA_BYTE_ARRAY": B.DELTA_BYTE_ARRAY}[encoding]
    pages, n_out = layout(ag, enc, offsets, [(slot, nv) for _, (_, _, nv, slot) in sections], rng, gap=False)
    st, msg, out, lens, _ = encode(ag, enc, ow, offsets, data, vbits, pages, n_out, dev)
    assert st == N.AG_OK, msg
    for (_, (vd, vl, _, _)), (_, _, o, _), ln in zip(sections, pages, lens):
        assert ln == vl and out[o:o + ln].tobytes() == dst[vd:vd + vl]


def decode_dev(ag, enc, ow, dpages, out, pages, n_slots, dvalid, cap):
    """the encoded sections decoded on the device into (offsets, data) of n_slots slots, cap data bytes"""
    dsrc = out if isinstance(out, Dev) else Dev(out)
    doff = Dev(np.zeros(n_slots + 1, np.int32 if ow == 4 else np.int64))
    ddata = Dev(nbytes=cap)
    total = C.c_int64(-1)
    tbl = N.page_table([(o, ln, n, i0) for (i0, n, o, _), ln in zip(pages, dpages)])
    ag.call("ag_parquet_byte_array_decode_dev", enc, ow, dsrc.ptr, tbl, len(pages), n_slots,
            None if dvalid is None else dvalid.ptr, None, None, 0, 0, doff.ptr, ddata.ptr, cap, C.byref(total), None, None, None)
    ag.call("ag_stream_sync", None)
    return doff, ddata, total.value


@ENCS
@WIDTHS
def test_round_trip_through_the_decoder(ag, enc, ow):
    rng = np.random.default_rng(enc + ow)
    vals, valid = strings(rng, 50_001, null_lengths=False)
    offsets, data = arrow(vals, ow)
    spans = [(0, 20_000), (20_000, 17), (20_017, 29_984)]              # consecutive slots: decoded into one array
    pages, n_out = layout(ag, enc, offsets, spans, rng)
    st, msg, out, lens, _ = encode(ag, enc, ow, offsets, data, valid, pages, n_out, True)
    assert st == N.AG_OK, msg
    dvalid = Dev(np.packbits(valid, bitorder="little"))
    doff, ddata, total = decode_dev(ag, enc, ow, lens, out, pages, 50_001, dvalid, data.size)
    assert total == offsets[-1]
    assert (doff.get() == offsets).all()
    assert ddata.get(count=total).tobytes() == data[:total].tobytes()


def error_case(ag, enc, ow, offsets, data, valid, pages, dev):
    st, msg, out, lens, bad = encode(ag, enc, ow, offsets, data, valid, pages, max(o + c for _, _, o, c in pages), dev)
    assert st == N.AG_ERR_INVALID
    assert (out == GUARD).all() and (lens == -1).all()
    return msg, bad


@ENCS
@FLAVOURS
def test_errors_write_nothing(ag, enc, dev):
    rng = np.random.default_rng(1)
    vals, valid = strings(rng, 6000)
    for ow in (4, 8):
        offsets, data = arrow(vals, ow)
        pages, _ = layout(ag, enc, offsets, [(0, 1000), (1000, 2000), (3000, 3000)], rng, gap=False)
        short = [list(p) for p in pages]
        short[2][3] -= 1                                   # capacity one byte below the bound
        msg, bad = error_case(ag, enc, ow, offsets, data, valid, [tuple(p) for p in short], dev)
        assert "page 2: capacity" in msg and bad == N.NO_ERROR_POS
        dec = offsets.copy()
        dec[2500] = dec[2502] + 1                          # offsets decrease after slot 2500, inside page 1
        msg, bad = error_case(ag, enc, ow, dec, data, valid, [tuple(p) for p in short], dev)
        assert "page 1: offsets decrease" in msg and bad == 2500
        neg = offsets.copy()
        neg[:1001] -= int(neg[1000]) + 1                   # pages 0 and 1 start at negative offsets
        msg, bad = error_case(ag, enc, ow, neg, data, valid, pages, dev)
        assert "page 0: negative offset at slot 0" in msg and bad == 0
        msg, bad = error_case(ag, enc, ow, neg, data, valid, pages[1:], dev)
        assert "page 0: negative offset at slot 1000" in msg and bad == 1000
    # a valid value longer than 2^31-1 bytes: the checking pass reads no data, so a small buffer will do
    offsets = np.array([0, 5, 5 + (1 << 31), 6 + (1 << 31)], np.int64)
    data = np.zeros(16, np.uint8)
    pages = [(0, 1, 0, 256), (1, 2, 256, 64)]               # a slot error is reported before the page's capacity
    msg, bad = error_case(ag, enc, 8, offsets, data, None, pages, dev)
    assert "page 1: value at slot 1 longer than 2^31-1 bytes" in msg and bad == 1


@FLAVOURS
def test_host_refusals(ag, dev):
    offsets = np.arange(9, dtype=np.int32)
    data = np.zeros(16, np.uint8)
    tbl = N.enc_page_table([(0, 8, 0, 4096)])
    out = np.zeros(4096, np.uint8)
    fn = "ag_parquet_byte_array_encode" + ("_dev" if dev else "")
    tail = (None, None, None) if dev else (None, None)
    d = Dev(offsets) if dev else None
    o = d.ptr if dev else ptr(offsets)
    dd = Dev(data).ptr if dev else ptr(data)
    do = Dev(out).ptr if dev else ptr(out)
    for enc, ow, op, dp, outp, t in [(B.RLE_DICTIONARY, 4, o, dd, do, tbl), (B.PLAIN, 2, o, dd, do, tbl), (B.PLAIN, 4, None, dd, do, tbl),
                                     (B.PLAIN, 4, o, None, do, tbl), (B.PLAIN, 4, o, dd, None, tbl),
                                     (B.PLAIN, 4, o, dd, do, N.enc_page_table([(0, -1, 0, 4096)]))]:
        assert ag.call_status(fn, enc, ow, op, dp, None, t, 1, outp, *tail)[0] == N.AG_ERR_INVALID


@pytest.mark.parametrize("enc", [B.PLAIN, B.DELTA_BYTE_ARRAY], ids=["plain", "dba"])
def test_large_batch_past_2_31(ag, enc):
    """int64 offsets over 2.2 GB of data, the second page's section past 2^31 in the output"""
    rng = np.random.default_rng(enc)
    n = 2200
    lens = rng.integers(900_000, 1_100_000, n).astype(np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    total = int(offsets[-1])
    assert total > (1 << 31)
    base = np.frombuffer(rng.bytes(1 << 20), np.uint8)
    data = np.resize(base, total + 16)
    data[offsets[:-1]] = np.arange(n, dtype=np.uint8)                 # values differ from their first byte on
    spans = [(0, 1000), (1000, n - 1000)]
    caps = [bound(ag, enc, nv, int(offsets[i0 + nv] - offsets[i0])) for i0, nv in spans]
    pages = [(0, 1000, 0, caps[0]), (1000, n - 1000, (1 << 31) + 3, caps[1])]
    n_out = pages[1][2] + caps[1]
    assert n_out > (1 << 31)
    do, dd, dout = Dev(offsets), Dev(data), Dev(nbytes=n_out)
    dl = Dev(np.zeros(2, np.int64))
    ag.call("ag_parquet_byte_array_encode_dev", enc, 8, do.ptr, dd.ptr, None, N.enc_page_table(pages), 2, dout.ptr, dl.ptr, None, None)
    ag.call("ag_stream_sync", None)
    lens_w = dl.get()
    assert pages[1][2] + lens_w[1] > (1 << 31)
    doff, ddata, tot = decode_dev(ag, enc, 8, lens_w, dout, pages, n, None, total + 16)
    assert tot == total
    assert (doff.get() == offsets).all()
    assert np.array_equal(ddata.get(count=total), data[:total])


def test_dba_after_a_long_null_run_costs_what_dlba_does(ag):
    """A page of 32M leading nulls, then sorted keys.  Each tile finds the page's previous valid value in one load of
    a per-page max-scan of the tiles' last valid slots; a walk back over the 32768 null tiles from every tile would
    cost about 32768^2 / 2 dependent loads, far more than the DELTA_LENGTH_BYTE_ARRAY call on the same page."""
    import time
    rng = np.random.default_rng(11)
    n, tail = 32 << 20, 5000
    keys = F.random_strings(rng, tail, sorted_keys=True)
    lens = np.zeros(n, np.int64)
    lens[-tail:] = [len(k) for k in keys]
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    data = np.frombuffer(b"".join(keys) + b"\0", np.uint8).copy()
    valid = np.zeros(n, bool)
    valid[-tail:] = True
    do, dd, dv = Dev(offsets), Dev(data), Dev(np.packbits(valid, bitorder="little"))
    ms = {}
    for enc in (B.DELTA_LENGTH_BYTE_ARRAY, B.DELTA_BYTE_ARRAY):
        cap = bound(ag, enc, n, int(offsets[-1]))
        dout, dl = Dev(nbytes=cap), Dev(np.zeros(1, np.int64))
        tbl = N.enc_page_table([(0, n, 0, cap)])
        call = lambda: ag.call("ag_parquet_byte_array_encode_dev", enc, 4, do.ptr, dd.ptr, dv.ptr, tbl, 1, dout.ptr, dl.ptr,  # noqa: E731
                               None, None)
        call()
        ag.call("ag_stream_sync", None)
        t0 = time.perf_counter()
        for _ in range(3):
            call()
        ag.call("ag_stream_sync", None)
        ms[enc] = (time.perf_counter() - t0) * 1e3 / 3
        want = EXPECT[enc](keys)
        assert int(dl.get()[0]) == len(want)
        assert dout.get(count=len(want)).tobytes() == want
    assert ms[B.DELTA_BYTE_ARRAY] < 4 * ms[B.DELTA_LENGTH_BYTE_ARRAY] + 10, ms
