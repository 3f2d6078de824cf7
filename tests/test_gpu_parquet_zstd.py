"""Device ZSTD page decompression against the Python restatement in tests/zstd_ref.py (host and _dev flavours, byte for
byte), pyarrow-written ZSTD files end to end against pq.read_table, every page of the byte_stream_split.zstd fixture
against pyarrow's host decompression, and ~200 MB of output through a checksum."""
import os
import zlib

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import pq_files as F
import pq_pages as P
import zstd_ref as R
from arrow_go_b200 import _native as N
from helpers import Dev, checksum64, ptr
from pq_chunk import read_chunk_dev
from pq_pages import compressed_batch

gpu = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
CANARY = 0xA5
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def run_zstd(ag, src, pages, n_out, dev=False):
    """-> (status, message, out, written); out starts as the canary everywhere"""
    tbl = N.compressed_table(pages)
    out = np.full(n_out, CANARY, np.uint8)
    w = np.full(len(pages), -1, np.int64)
    if not dev:
        st, msg = ag.call_status("ag_parquet_zstd_decompress", ptr(src), tbl, len(pages), ptr(out), ptr(w))
        return st, msg, out, w
    ds, do, dw = Dev(src), Dev(out), Dev(w)
    st, msg = ag.call_status("ag_parquet_zstd_decompress_dev", ds.ptr, tbl, len(pages), do.ptr, dw.ptr, None)
    ag.call("ag_stream_sync", None)
    return st, msg, do.get(), dw.get()


def expect(src, pages, n_out):
    """restatement: (out, written, [(page index, message)] of failing pages)"""
    want = np.full(n_out, CANARY, np.uint8)
    w, errs = [], []
    for k, (s, sl, d, dl) in enumerate(pages):
        got, e, arg = R.decode(bytes(src[s:s + sl]), dl)
        want[d:d + len(got)] = np.frombuffer(got, np.uint8)
        w.append(len(got))
        if e:
            errs.append((k, R.message(e, arg, dl)))
    return want, w, errs


def decode_and_compare(ag, streams, rng, dev, gap=True):
    src, pages, n_out = compressed_batch(streams, rng, gap)
    st, msg, out, w = run_zstd(ag, src, pages, n_out, dev)
    want, ww, errs = expect(src, pages, n_out)
    assert w.tolist() == ww, (msg, errs)
    assert out.tobytes() == want.tobytes(), (msg, errs)          # the canary outside every written range survives
    return st, msg, errs, pages


@gpu
@FLAVOURS
def test_every_form(ag, dev):
    rng = np.random.default_rng(81)
    streams = [(s, len(x)) for _, s, x in R.forms()]
    for name in ("zstd_checksum.zst", "zstd_no_content_size.zst"):
        streams.append((open(os.path.join(GOLDEN, name), "rb").read(), len(R.golden_payload())))
    for gap in (True, False):
        st, msg, errs, _ = decode_and_compare(ag, streams, rng, dev, gap)
        assert st == N.AG_OK and not errs, msg


@gpu
@FLAVOURS
def test_page_sizes(ag, dev):
    rng = np.random.default_rng(82)
    streams = []
    for n in (0, 1, (1 << 17) - 1, 1 << 17, (1 << 17) + 1, 1 << 22):
        x = (np.cumsum(rng.integers(0, 1000, (n + 7) // 8)) + (1 << 40)).astype(np.int64).tobytes()[:n]
        streams.append((pa.compress(x, codec="zstd", asbytes=True), n))
        streams.append((R.reframe(pa.compress(x, codec="zstd", asbytes=True), fcs=False, checksum=True), n))
    streams.append((b"", 0))
    st, msg, errs, _ = decode_and_compare(ag, streams, rng, dev)
    assert st == N.AG_OK and not errs, msg


def error_rows():
    rows = [(name, s, n) for name, s, n, _ in R.corrupt_rows()]
    x = b"0123456789" * 100
    good = pa.compress(x, codec="zstd", asbytes=True)
    nofcs = R.reframe(good, fcs=False)
    rows += [("size_from_header_small", good, len(x) - 1), ("size_from_header_large", good, len(x) + 1),
             ("size_from_header_two_frames", good + good, len(x)), ("size_after_decoding_small", nofcs, len(x) - 1),
             ("size_after_decoding_large", nofcs, len(x) + 1), ("empty_page_with_output", b"", 3)]
    return rows


@gpu
@FLAVOURS
@pytest.mark.parametrize("row", error_rows(), ids=lambda r: r[0])
def test_error_rows(ag, row, dev):
    name, s, n = row
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = rng.integers(0, 3, 5000, dtype=np.uint8).tobytes()
    good = pa.compress(x, codec="zstd", asbytes=True)
    # the failing page twice (pages 1 and 3 in the caller's order): the message names page 1
    src, pages, n_out = compressed_batch([(good, len(x)), (s, n), (good, len(x)), (s, n)], rng, gap=False)
    st, msg, out, w = run_zstd(ag, src, pages, n_out, dev)
    want, ww, errs = expect(src, pages, n_out)
    assert [e[0] for e in errs] == [1, 3]
    assert w.tolist() == ww and out.tobytes() == want.tobytes(), (msg, errs)
    assert st == N.AG_ERR_INVALID and f"zstd_decompress: page 1: {errs[0][1]} ({ww[1]} bytes written)" in msg, (msg, errs)
    assert ww[0] == ww[2] == len(x)


@gpu
@FLAVOURS
def test_invalid_arguments(ag, dev):
    src = np.frombuffer(pa.compress(b"abcdabcdabcd", codec="zstd", asbytes=True), np.uint8).copy()
    n = len(src)
    bad = [
        ([(-1, n, 0, 12)], "page 0: negative field"),
        ([(0, n, 0, 12), (0, -1, 20, 12)], "page 1: negative field"),
        ([(0, n, 0, 12), (0, n, -4, 12)], "page 1: negative field"),
        ([(0, n, 0, -12)], "page 0: negative field"),
        ([(0, 1 << 32, 0, 12)], "more than 2^32-1 bytes"),
        ([(0, n, 0, 1 << 32)], "more than 2^32-1 bytes"),
        ([(0, n, 0, 12), (0, n, 30, 12), (0, n, 11, 12)], "pages 0 and 2: overlapping dst ranges"),
    ]
    out = Dev(nbytes=256)
    for pages, text in bad:
        if dev:
            st, msg = ag.call_status("ag_parquet_zstd_decompress_dev", Dev(src).ptr, N.compressed_table(pages), len(pages), out.ptr, None, None)
        else:
            h = np.zeros(256, np.uint8)
            st, msg = ag.call_status("ag_parquet_zstd_decompress", ptr(src), N.compressed_table(pages), len(pages), ptr(h), None)
        assert st == N.AG_ERR_INVALID and "zstd_decompress" in msg and text in msg, (pages, msg)
    pages = [(0, n, 0, 12), (0, 0, 5, 0), (0, n, 12, 12)]
    st, msg, o, w = run_zstd(ag, np.concatenate([src, np.zeros(8, np.uint8)]), pages, 32, dev)
    assert st == N.AG_OK and w.tolist() == [12, 0, 12] and o[:24].tobytes() == b"abcdabcdabcd" * 2, msg


@gpu
@pytest.mark.parametrize("case", F.compressed_cases(), ids=F.compressed_case_id)
def test_pyarrow_zstd_files_end_to_end(ag, case, tmp_path):
    rng = np.random.default_rng(zlib.crc32(F.compressed_case_id(case).encode()))
    path = str(tmp_path / "c.parquet")
    tbl = F.write_numeric_case(path, rng, case, compression="ZSTD")
    plan = P.chunk_plan(path)
    assert plan["codec"] == "ZSTD" and (P.DELTA_BINARY_PACKED in P.encodings(plan)) == (case[0] == "delta")
    values, valid = read_chunk_dev(ag, plan)
    want, wvalid = F.expected(tbl, plan)
    assert np.array_equal(valid, wvalid)
    assert values == want


@gpu
@FLAVOURS
def test_fixture_pages_against_host(ag, dev):
    """every page of every column of byte_stream_split.zstd.parquet, compared as decompressed bytes"""
    path = os.path.join(GOLDEN, "byte_stream_split.zstd.parquet")
    rng = np.random.default_rng(83)
    for c in range(pq.ParquetFile(path).metadata.num_columns):
        chunk, pages = P.column_chunk(path, column=c)
        regions, comp, n_dst = P.decompress_table(pages)
        streams = [(chunk[regions[k][0]:regions[k][0] + regions[k][1]], regions[k][3]) for k in comp]
        assert streams
        src, tbl, n_out = compressed_batch(streams, rng)
        st, msg, out, w = run_zstd(ag, src, tbl, n_out, dev)
        assert st == N.AG_OK, (c, msg)
        for (s, sl, d, dl), k in zip(tbl, w):
            want = pa.decompress(bytes(src[s:s + sl]), decompressed_size=dl, codec="zstd", asbytes=True) if dl else b""
            assert k == dl and out[d:d + dl].tobytes() == want, c


@gpu
def test_decompress_200mb_device(ag):
    """~200 MB of output over 2^19-value int64 timestamp pages and 17-bit index pages, one of each kind checksummed and
    without a content size: three pages against pyarrow, the whole output through a checksum against the host twin."""
    rng = np.random.default_rng(84)
    per_page = 1 << 19
    bodies = [(np.cumsum(rng.integers(0, 1000, per_page)) + (k << 40)).astype(np.int64).tobytes() for k in range(2)]
    bodies += [(rng.integers(0, 100_000, per_page) & 0x1FFFF).astype(np.uint32).tobytes() for _ in range(2)]
    encs = [pa.compress(b, codec="zstd", asbytes=True) for b in bodies]
    encs[1] = R.reframe(encs[1], fcs=False, checksum=True)
    offs, blob = [], bytearray()
    for e in encs:
        offs.append(len(blob))
        blob += e
    blob += bytes(16)
    pages, d, want = [], 0, []
    while d < 200_000_000:
        k = len(pages) % 4
        pages.append((offs[k], len(encs[k]), d, len(bodies[k])))
        want.append(bodies[k])
        d += len(bodies[k])
    ds, dout, dw = Dev(np.frombuffer(bytes(blob), np.uint8).copy()), Dev(nbytes=d), Dev(np.zeros(len(pages), np.int64))
    ag.call("ag_parquet_zstd_decompress_dev", ds.ptr, N.compressed_table(pages), len(pages), dout.ptr, dw.ptr, None)
    ag.call("ag_stream_sync", None)
    assert dw.get().tolist() == [p[3] for p in pages]
    for p in (0, 1, 3, len(pages) - 1):
        assert dout.buf.to_numpy(np.uint8, pages[p][3], pages[p][2]).tobytes() == want[p]
    allw = np.frombuffer(b"".join(want), np.uint64)
    res = Dev(np.zeros(1, np.uint64))
    ag.call("ag_checksum64_dev", dout.ptr, allw.size, res.ptr, None)
    ag.call("ag_stream_sync", None)
    assert int(res.get()[0]) == checksum64(allw)
