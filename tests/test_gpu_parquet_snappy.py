"""Device SNAPPY page decompression against the Python restatement in tests/snappy_ref.py (host and _dev flavours, byte
for byte), pyarrow-written SNAPPY files end to end against pq.read_table, every page of four parquet-testing fixtures
against pyarrow's host decompression, and ~200 MB of output through a checksum."""
import os
import zlib

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import pq_files as F
import pq_pages as P
import snappy_ref as S
from arrow_go_b200 import _native as N
from helpers import Dev, checksum64, ptr
from pq_chunk import read_chunk_dev
from pq_pages import compressed_batch

gpu = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
CANARY = 0xA5
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FIXTURES = ("alltypes_plain.snappy.parquet", "datapage_v2.snappy.parquet", "datapage_v2_empty_datapage.snappy.parquet",
            "datapage_v1-snappy-compressed-checksum.parquet")


def run_snappy(ag, src, pages, n_out, dev=False):
    """-> (status, message, out, written); out starts as the canary everywhere"""
    tbl = N.compressed_table(pages)
    out = np.full(n_out, CANARY, np.uint8)
    w = np.full(len(pages), -1, np.int64)
    if not dev:
        st, msg = ag.call_status("ag_parquet_snappy_decompress", ptr(src), tbl, len(pages), ptr(out), ptr(w))
        return st, msg, out, w
    ds, do, dw = Dev(src), Dev(out), Dev(w)
    st, msg = ag.call_status("ag_parquet_snappy_decompress_dev", ds.ptr, tbl, len(pages), do.ptr, dw.ptr, None)
    ag.call("ag_stream_sync", None)
    return st, msg, do.get(), dw.get()


def expect(src, pages, n_out):
    """restatement: (out, written, [(page index, message)] of failing pages)"""
    want = np.full(n_out, CANARY, np.uint8)
    w, errs = [], []
    for k, (s, sl, d, dl) in enumerate(pages):
        got, e, pre = S.decode(bytes(src[s:s + sl]), dl)
        want[d:d + len(got)] = np.frombuffer(got, np.uint8)
        w.append(len(got))
        if e:
            errs.append((k, S.MESSAGE[e].format(dl, pre)))
    return want, w, errs


def decode_and_compare(ag, streams, rng, dev, gap=True):
    src, pages, n_out = compressed_batch(streams, rng, gap)
    st, msg, out, w = run_snappy(ag, src, pages, n_out, dev)
    want, ww, errs = expect(src, pages, n_out)
    assert w.tolist() == ww, (msg, errs)
    assert out.tobytes() == want.tobytes(), (msg, errs)          # the canary outside every written range survives
    return st, msg, errs, pages


@gpu
@FLAVOURS
def test_every_element_form(ag, dev):
    rng = np.random.default_rng(61)
    streams = [(s, len(x)) for _, s, x in S.forms()]
    for name, x in (("random", rng.integers(0, 256, 50_000, dtype=np.uint8).tobytes()), ("zeros", bytes(70_000)),
                    ("timestamps", (np.cumsum(rng.integers(0, 1000, 9000)) + (1 << 40)).astype(np.int64).tobytes())):
        streams.append((pa.compress(x, codec="snappy", asbytes=True), len(x)))
        streams.append((S.encode(x, copy_form=4), len(x)))
    for gap in (True, False):
        st, msg, errs, _ = decode_and_compare(ag, streams, rng, dev, gap)
        assert st == N.AG_OK and not errs, msg


@gpu
@FLAVOURS
def test_page_sizes(ag, dev):
    rng = np.random.default_rng(62)
    streams = []
    for n in (0, 1, 65535, 65536, 65537):
        x = (rng.integers(0, 4, n, dtype=np.uint8) * 17).tobytes()
        streams.append((pa.compress(x, codec="snappy", asbytes=True), n))
    streams.append((b"", 0))                                      # an empty v2 value region
    st, msg, errs, _ = decode_and_compare(ag, streams, rng, dev)
    assert st == N.AG_OK and not errs, msg
    # 16 MB: longer than the parse window many times over; literal-heavy, copy-heavy and long-literal regions
    big = bytearray(rng.integers(0, 256, 1 << 24, dtype=np.uint8).tobytes())
    big[1 << 22:1 << 23] = bytes(1 << 22)
    big[1 << 23:(1 << 23) + (1 << 22)] = (np.cumsum(rng.integers(0, 1000, 1 << 19)) + (1 << 40)).astype(np.int64).tobytes()
    big = bytes(big)
    lit = S.stream(300_000, [S.literal(big[:300_000], 3)])       # one literal longer than the window
    src, pages, n_out = compressed_batch([(pa.compress(big, codec="snappy", asbytes=True), len(big)), (lit, 300_000)], rng)
    st, msg, out, w = run_snappy(ag, src, pages, n_out, dev)
    assert st == N.AG_OK, msg
    for (s, sl, d, dl), k in zip(pages, w):
        assert k == dl
        want = big if dl == len(big) else big[:300_000]
        assert out[d:d + dl].tobytes() == want
    assert (out[:min(p[2] for p in pages)] == CANARY).all()


def error_rows():
    rows = [(name, s, n) for name, s, n, _ in S.corrupt_rows() if n < 1 << 32]
    good = S.stream(20, [S.literal(b"0123456789"), S.copy(10, 10, 1)])
    rows += [("size_mismatch_small", good, 19), ("size_mismatch_large", good, 21),
             ("size_mismatch_corrupt_body", S.stream(20, [S.literal(b"0123456789"), b"\xf0"]), 25),
             ("empty_stream_with_output", b"", 3)]
    return rows


@gpu
@FLAVOURS
@pytest.mark.parametrize("row", error_rows(), ids=lambda r: r[0])
def test_error_rows(ag, row, dev):
    name, s, n = row
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = rng.integers(0, 3, 5000, dtype=np.uint8).tobytes()
    good = pa.compress(x, codec="snappy", asbytes=True)
    # the failing page twice (pages 1 and 3 in the caller's order): the message names page 1
    src, pages, n_out = compressed_batch([(good, len(x)), (s, n), (good, len(x)), (s, n)], rng, gap=False)
    st, msg, out, w = run_snappy(ag, src, pages, n_out, dev)
    want, ww, errs = expect(src, pages, n_out)
    assert [e[0] for e in errs] == [1, 3]
    assert w.tolist() == ww and out.tobytes() == want.tobytes(), msg
    assert st == N.AG_ERR_INVALID and f"snappy_decompress: page 1: {errs[0][1]} ({ww[1]} bytes written)" in msg, (msg, errs)
    assert ww[0] == ww[2] == len(x)


@gpu
@FLAVOURS
def test_invalid_arguments(ag, dev):
    src = np.frombuffer(S.encode(b"abcdabcdabcd"), np.uint8).copy()
    n = len(src)
    bad = [
        ([(-1, n, 0, 12)], "page 0: negative field"),
        ([(0, n, 0, 12), (0, -1, 20, 12)], "page 1: negative field"),
        ([(0, n, 0, 12), (0, n, -4, 12)], "page 1: negative field"),
        ([(0, n, 0, -12)], "page 0: negative field"),
        ([(0, 1 << 32, 0, 12)], "more than 2^32-1 bytes"),
        ([(0, n, 0, 1 << 32)], "more than 2^32-1 bytes"),
        ([(0, n, 0, 12), (0, n, 30, 12), (0, n, 11, 12)], "pages 0 and 2: overlapping dst ranges"),
        ([(0, n, 40, 12), (0, n, 0, 12), (0, n, 51, 12)], "pages 0 and 2: overlapping dst ranges"),
    ]
    out = Dev(nbytes=256)
    for pages, text in bad:
        if dev:
            st, msg = ag.call_status("ag_parquet_snappy_decompress_dev", Dev(src).ptr, N.compressed_table(pages), len(pages), out.ptr, None, None)
        else:
            h = np.zeros(256, np.uint8)
            st, msg = ag.call_status("ag_parquet_snappy_decompress", ptr(src), N.compressed_table(pages), len(pages), ptr(h), None)
        assert st == N.AG_ERR_INVALID and text in msg, (pages, msg)
    # empty ranges overlap nothing; adjacent ranges do not overlap
    pages = [(0, n, 0, 12), (0, 0, 5, 0), (0, n, 12, 12)]
    st, msg, o, w = run_snappy(ag, np.concatenate([src, np.zeros(8, np.uint8)]), pages, 32, dev)
    assert st == N.AG_OK and w.tolist() == [12, 0, 12] and o[:24].tobytes() == b"abcdabcdabcd" * 2, msg


@gpu
@pytest.mark.parametrize("case", F.compressed_cases(), ids=F.compressed_case_id)
def test_pyarrow_snappy_files_end_to_end(ag, case, tmp_path):
    rng = np.random.default_rng(zlib.crc32(F.compressed_case_id(case).encode()))
    path = str(tmp_path / "c.parquet")
    tbl = F.write_numeric_case(path, rng, case, compression="SNAPPY")
    plan = P.chunk_plan(path)
    assert plan["codec"] == "SNAPPY" and (P.DELTA_BINARY_PACKED in P.encodings(plan)) == (case[0] == "delta")
    values, valid = read_chunk_dev(ag, plan)
    want, wvalid = F.expected(tbl, plan)
    assert np.array_equal(valid, wvalid)
    assert values == want


@gpu
@FLAVOURS
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_pages_against_host(ag, name, dev):
    """every page of every column (BYTE_ARRAY, BOOLEAN and INT96 included: decompression is type-agnostic)"""
    path = os.path.join(GOLDEN, name)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    for c in range(pq.ParquetFile(path).metadata.num_columns):
        chunk, pages = P.column_chunk(path, column=c)
        regions, comp, n_dst = P.decompress_table(pages)
        streams = [(chunk[regions[k][0]:regions[k][0] + regions[k][1]], regions[k][3]) for k in comp]
        src, tbl, n_out = compressed_batch(streams, rng)
        st, msg, out, w = run_snappy(ag, src, tbl, n_out, dev)
        assert st == N.AG_OK, (c, msg)
        for (s, sl, d, dl), k in zip(tbl, w):
            want = pa.decompress(bytes(src[s:s + sl]), decompressed_size=dl, codec="snappy", asbytes=True) if dl else b""
            assert k == dl and out[d:d + dl].tobytes() == want, (name, c)


@gpu
def test_decompress_200mb_device(ag):
    """~200 MB of output over 2^19-value int64 pages (timestamps, copy-heavy) and 17-bit index pages (literal-heavy):
    two pages against pyarrow, the whole output through a checksum against the host twin."""
    rng = np.random.default_rng(63)
    per_page = 1 << 19
    bodies = [(np.cumsum(rng.integers(0, 1000, per_page)) + (k << 40)).astype(np.int64).tobytes() for k in range(2)]
    bodies += [(rng.integers(0, 100_000, per_page) & 0x1FFFF).astype(np.uint32).tobytes() for _ in range(2)]
    encs = [pa.compress(b, codec="snappy", asbytes=True) for b in bodies]
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
    ag.call("ag_parquet_snappy_decompress_dev", ds.ptr, N.compressed_table(pages), len(pages), dout.ptr, dw.ptr, None)
    ag.call("ag_stream_sync", None)
    assert dw.get().tolist() == [p[3] for p in pages]
    for p in (0, 3, len(pages) - 1):
        assert dout.buf.to_numpy(np.uint8, pages[p][3], pages[p][2]).tobytes() == want[p]
    allw = np.frombuffer(b"".join(want), np.uint64)
    res = Dev(np.zeros(1, np.uint64))
    ag.call("ag_checksum64_dev", dout.ptr, allw.size, res.ptr, None)
    ag.call("ag_stream_sync", None)
    assert int(res.get()[0]) == checksum64(allw)
