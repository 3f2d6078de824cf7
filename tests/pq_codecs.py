"""Test helper: the four Parquet page codecs the library decompresses (SNAPPY, ZSTD, GZIP, LZ4_RAW) in one table, one
way to run a batch of pages through either flavour of a codec and compare it byte for byte with the codec's Python
restatement, and the checks every codec's test file runs: argument checks, failing pages, the codec's parquet-testing
fixtures against pyarrow, pyarrow-written files end to end through read_chunk_dev, and ~200 MB of output through a
checksum.  Not product code."""
import os
import zlib
from typing import Callable, NamedTuple

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

import gzip_ref
import lz4_ref
import pq_files as F
import pq_pages as P
import snappy_ref
import zstd_ref
from arrow_go_b200 import _native as N
from helpers import Dev, checksum64, ptr
from pq_chunk import read_chunk_dev
from pq_pages import compressed_batch

CANARY = 0xA5
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


class Codec(NamedTuple):
    name: str              # pyarrow's codec name
    parquet: str           # the writer's `compression`, and the chunk's codec in a pq_pages plan
    prefix: str            # message prefix of the entry points
    entry: str             # host entry point; entry + "_dev" is the device flavour
    restate: Callable      # (bytes, dst_len) -> (output, message or None)
    sample: Callable       # () -> (stream, payload) of a short valid page
    error_rows: Callable   # () -> [(name, stream, dst_len)] of failing pages
    fixtures: tuple        # parquet-testing files under tests/golden
    big: Callable          # () -> (bodies, streams) of the four pages the 200 MB run repeats


def _snappy(buf, dl):
    got, e, pre = snappy_ref.decode(buf, dl)
    return got, snappy_ref.MESSAGE[e].format(dl, pre) if e else None


def _zstd(buf, dl):
    got, e, arg = zstd_ref.decode(buf, dl)
    return got, zstd_ref.message(e, arg, dl) if e else None


def _gzip(buf, dl):
    got, outcome, arg = gzip_ref.decode(buf, dl)
    return got, gzip_ref.message(outcome, arg, dl) if outcome != gzip_ref.OK else None


def _lz4(buf, dl):
    got, outcome, arg = lz4_ref.decode(buf, dl)
    return got, lz4_ref.message(outcome, arg, dl) if outcome != lz4_ref.OK else None


def _snappy_rows():
    S = snappy_ref
    rows = [(name, s, n) for name, s, n, _ in S.corrupt_rows() if n < 1 << 32]
    good = S.stream(20, [S.literal(b"0123456789"), S.copy(10, 10, 1)])
    rows += [("size_mismatch_small", good, 19), ("size_mismatch_large", good, 21),
             ("size_mismatch_corrupt_body", S.stream(20, [S.literal(b"0123456789"), b"\xf0"]), 25),
             ("empty_stream_with_output", b"", 3)]
    return rows


def _zstd_rows():
    R = zstd_ref
    rows = [(name, s, n) for name, s, n, _ in R.corrupt_rows()]
    x = b"0123456789" * 100
    good = pa.compress(x, codec="zstd", asbytes=True)
    nofcs = R.reframe(good, fcs=False)
    rows += [("size_from_header_small", good, len(x) - 1), ("size_from_header_large", good, len(x) + 1),
             ("size_from_header_two_frames", good + good, len(x)), ("size_after_decoding_small", nofcs, len(x) - 1),
             ("size_after_decoding_large", nofcs, len(x) + 1), ("empty_page_with_output", b"", 3)]
    return rows


def _gzip_rows():
    return [(name, s, n) for name, s, n, _ in gzip_ref.corrupt_rows()]


def _lz4_rows():
    R = lz4_ref
    return [r[:3] for r in R.corrupt_rows()] + [r[:3] for r in R.differences() if r[3][0] != R.OK]


def _bodies(seed):
    """2^19-value int64 timestamp pages (copy-heavy) and 17-bit index pages (literal-heavy)"""
    rng = np.random.default_rng(seed)
    per_page = 1 << 19
    bodies = [(np.cumsum(rng.integers(0, 1000, per_page)) + (k << 40)).astype(np.int64).tobytes() for k in range(2)]
    return bodies + [(rng.integers(0, 100_000, per_page) & 0x1FFFF).astype(np.uint32).tobytes() for _ in range(2)]


def _snappy_big():
    bodies = _bodies(63)
    return bodies, [pa.compress(b, codec="snappy", asbytes=True) for b in bodies]


def _zstd_big():
    """one timestamp page checksummed and without a content size"""
    bodies = _bodies(84)
    encs = [pa.compress(b, codec="zstd", asbytes=True) for b in bodies]
    encs[1] = zstd_ref.reframe(encs[1], fcs=False, checksum=True)
    return bodies, encs


def _gzip_big():
    """two pages of three members with FHCRC headers"""
    R = gzip_ref
    bodies = _bodies(94)
    encs = [pa.compress(b, codec="gzip", asbytes=True) for b in bodies]
    for k in (1, 2):
        b, third = bodies[k], len(bodies[k]) // 3
        parts = [b[:third], b[third:2 * third], b[2 * third:]]
        encs[k] = b"".join(R.member(R.gz(p)[10:-8], hcrc=True, name=b"part", payload=p) for p in parts)
    return bodies, encs


def _lz4_big():
    """timestamps, 17-bit indices and runs, every body a whole number of 8-byte words"""
    R = lz4_ref
    per_page = 1 << 19
    bodies = [R.timestamps(8 * per_page, k) for k in range(2)] + [R.dict_indices(17 * per_page // 8, 2), R.runs(4 * per_page, 3)]
    return bodies, [pa.compress(b, codec="lz4_raw", asbytes=True) for b in bodies]


SNAPPY = Codec("snappy", "SNAPPY", "snappy_decompress", "ag_parquet_snappy_decompress", _snappy,
               lambda: (snappy_ref.encode(b"abcdabcdabcd"), b"abcdabcdabcd"), _snappy_rows,
               ("alltypes_plain.snappy.parquet", "datapage_v2.snappy.parquet", "datapage_v2_empty_datapage.snappy.parquet",
                "datapage_v1-snappy-compressed-checksum.parquet"), _snappy_big)
ZSTD = Codec("zstd", "ZSTD", "zstd_decompress", "ag_parquet_zstd_decompress", _zstd,
             lambda: (pa.compress(b"abcdabcdabcd", codec="zstd", asbytes=True), b"abcdabcdabcd"), _zstd_rows,
             ("byte_stream_split.zstd.parquet",), _zstd_big)
GZIP = Codec("gzip", "GZIP", "gzip_decompress", "ag_parquet_gzip_decompress", _gzip,
             lambda: (pa.compress(b"abcdabcdabcd", codec="gzip", asbytes=True), b"abcdabcdabcd"), _gzip_rows,
             ("concatenated_gzip_members.parquet", "byte_stream_split_extended.gzip.parquet"), _gzip_big)
LZ4 = Codec("lz4_raw", "LZ4", "lz4_raw_decompress", "ag_parquet_lz4_raw_decompress", _lz4,
            lambda: (lz4_ref.block(lz4_ref.seq(b"abcd", 4, 8)), b"abcdabcdabcd" + lz4_ref.TAIL), _lz4_rows,
            ("lz4_raw_compressed.parquet", "lz4_raw_compressed_larger.parquet"), _lz4_big)


def run(ag, codec, src, pages, n_out, dev=False):
    """-> (status, message, out, written); out starts as the canary everywhere"""
    tbl = N.compressed_table(pages)
    out = np.full(n_out, CANARY, np.uint8)
    w = np.full(len(pages), -1, np.int64)
    if not dev:
        st, msg = ag.call_status(codec.entry, ptr(src), tbl, len(pages), ptr(out), ptr(w))
        return st, msg, out, w
    ds, do, dw = Dev(src), Dev(out), Dev(w)
    st, msg = ag.call_status(codec.entry + "_dev", ds.ptr, tbl, len(pages), do.ptr, dw.ptr, None)
    ag.call("ag_stream_sync", None)
    return st, msg, do.get(), dw.get()


def expect(codec, src, pages, n_out):
    """restatement: (out, written, [(page index, message)] of failing pages)"""
    want = np.full(n_out, CANARY, np.uint8)
    w, errs = [], []
    for k, (s, sl, d, dl) in enumerate(pages):
        got, msg = codec.restate(bytes(src[s:s + sl]), dl)
        want[d:d + len(got)] = np.frombuffer(got, np.uint8)
        w.append(len(got))
        if msg is not None:
            errs.append((k, msg))
    return want, w, errs


def decode_and_compare(ag, codec, streams, rng, dev, gap=True):
    """-> (status, message, [(page index, message)] the restatement gives)"""
    src, pages, n_out = compressed_batch(streams, rng, gap)
    st, msg, out, w = run(ag, codec, src, pages, n_out, dev)
    want, ww, errs = expect(codec, src, pages, n_out)
    assert w.tolist() == ww, (msg, errs)
    assert out.tobytes() == want.tobytes(), (msg, errs)          # the canary outside every written range survives
    return st, msg, errs


def invalid_arguments(ag, codec, dev):
    stream, payload = codec.sample()
    src = np.frombuffer(stream, np.uint8).copy()
    n, L = len(src), len(payload)
    bad = [
        ([(-1, n, 0, L)], "page 0: negative field"),
        ([(0, n, 0, L), (0, -1, 2 * L, L)], "page 1: negative field"),
        ([(0, n, 0, L), (0, n, -4, L)], "page 1: negative field"),
        ([(0, n, 0, -L)], "page 0: negative field"),
        ([(0, 1 << 32, 0, L)], "more than 2^32-1 bytes"),
        ([(0, n, 0, 1 << 32)], "more than 2^32-1 bytes"),
        ([(0, n, 0, L), (0, n, 2 * L + 4, L), (0, n, L - 1, L)], "pages 0 and 2: overlapping dst ranges"),
        ([(0, n, 3 * L + 4, L), (0, n, 0, L), (0, n, 4 * L + 3, L)], "pages 0 and 2: overlapping dst ranges"),
    ]
    out = Dev(nbytes=256)
    for pages, text in bad:
        if dev:
            st, msg = ag.call_status(codec.entry + "_dev", Dev(src).ptr, N.compressed_table(pages), len(pages), out.ptr, None, None)
        else:
            h = np.zeros(256, np.uint8)
            st, msg = ag.call_status(codec.entry, ptr(src), N.compressed_table(pages), len(pages), ptr(h), None)
        assert st == N.AG_ERR_INVALID and codec.prefix in msg and text in msg, (pages, msg)
    # empty ranges overlap nothing; adjacent ranges do not overlap
    pages = [(0, n, 0, L), (0, 0, 5, 0), (0, n, L, L)]
    st, msg, o, w = run(ag, codec, np.concatenate([src, np.zeros(8, np.uint8)]), pages, 2 * L + 8, dev)
    assert st == N.AG_OK and w.tolist() == [L, 0, L] and o[:2 * L].tobytes() == payload * 2, msg


def error_row(ag, codec, row, dev):
    """a failing page among good ones: the restatement's output, written counts and message"""
    name, s, n = row
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = rng.integers(0, 3, 5000, dtype=np.uint8).tobytes()
    good = pa.compress(x, codec=codec.name, asbytes=True)
    # the failing page twice (pages 1 and 3 in the caller's order): the message names page 1
    src, pages, n_out = compressed_batch([(good, len(x)), (s, n), (good, len(x)), (s, n)], rng, gap=False)
    st, msg, out, w = run(ag, codec, src, pages, n_out, dev)
    want, ww, errs = expect(codec, src, pages, n_out)
    assert [e[0] for e in errs] == [1, 3]
    assert w.tolist() == ww and out.tobytes() == want.tobytes(), (msg, errs)
    assert st == N.AG_ERR_INVALID and f"{codec.prefix}: page 1: {errs[0][1]} ({ww[1]} bytes written)" in msg, (msg, errs)
    assert ww[0] == ww[2] == len(x)


def fixture_pages(ag, codec, name, dev):
    """every page of every column (BYTE_ARRAY, BOOLEAN and INT96 included: decompression is type-agnostic) against
    pyarrow's host decompression, and every flat numeric column end to end against pq.read_table"""
    path = os.path.join(GOLDEN, name)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    tbl = pq.read_table(path)
    schema = pq.ParquetFile(path).schema
    for c in range(len(schema)):
        chunk, pages = P.column_chunk(path, column=c)
        regions, comp, _ = P.decompress_table(pages)
        streams = [(chunk[regions[k][0]:regions[k][0] + regions[k][1]], regions[k][3]) for k in comp]
        assert streams
        src, pt, n_out = compressed_batch(streams, rng)
        st, msg, out, w = run(ag, codec, src, pt, n_out, dev)
        assert st == N.AG_OK, (c, msg)
        for (s, sl, d, dl), k in zip(pt, w):
            want = pa.decompress(bytes(src[s:s + sl]), decompressed_size=dl, codec=codec.name, asbytes=True) if dl else b""
            assert k == dl and out[d:d + dl].tobytes() == want, c
        col = schema.column(c)
        if col.physical_type in ("INT32", "INT64", "FLOAT", "DOUBLE") and col.max_repetition_level == 0:
            plan = P.chunk_plan(path, c)
            values, valid = read_chunk_dev(ag, plan)
            want, wvalid = F.expected(tbl.select([c]), plan)
            assert np.array_equal(valid, wvalid) and values == want, c


def check_chunk(ag, codec, tbl, plan):
    """read_chunk_dev of a planned chunk against pq.read_table"""
    assert plan["codec"] == codec.parquet
    values, valid = read_chunk_dev(ag, plan)
    want, wvalid = F.expected(tbl, plan)
    assert np.array_equal(valid, wvalid)
    assert values == want


def pyarrow_file(ag, codec, case, tmp_path):
    """one compressed_cases() row written by pyarrow, end to end"""
    rng = np.random.default_rng(zlib.crc32(F.compressed_case_id(case).encode()))
    path = str(tmp_path / "c.parquet")
    tbl = F.write_numeric_case(path, rng, case, compression=codec.parquet)
    plan = P.chunk_plan(path)
    assert (P.DELTA_BINARY_PACKED in P.encodings(plan)) == (case[0] == "delta")
    check_chunk(ag, codec, tbl, plan)


def pyarrow_file_other_type(ag, codec, kind, tmp_path):
    """a BYTE_ARRAY, FIXED_LEN_BYTE_ARRAY or BOOLEAN column in v1 pages, end to end"""
    rng = np.random.default_rng(zlib.crc32(kind.encode()))
    path = str(tmp_path / "c.parquet")
    if kind == "byte_array":
        arr, enc = F.make_string_column(rng, "RLE_DICTIONARY", 8000, 0.1), "RLE_DICTIONARY"
    else:
        arr, enc = F.make_array(rng, kind, 20_000, 0.1), F.KINDS[kind]
    tbl = F.write_column(path, arr, nullable=True, encoding=enc, version="1.0", compression=codec.parquet, data_page_size=8192)
    plan = P.chunk_plan(path)
    # v1 pages: their bodies are always compressed, so every page of these columns goes through the codec
    assert len(plan["comp"]) == len(plan["pages"]) + (1 if plan["dict"] else 0)
    check_chunk(ag, codec, tbl, plan)


def decompress_200mb(ag, codec):
    """~200 MB of output over the codec's four page bodies, repeated: the first four pages and the last against the
    host bodies, the whole output through a checksum against the host twin."""
    bodies, encs = codec.big()
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
    ag.call(codec.entry + "_dev", ds.ptr, N.compressed_table(pages), len(pages), dout.ptr, dw.ptr, None)
    ag.call("ag_stream_sync", None)
    assert dw.get().tolist() == [p[3] for p in pages]
    for p in (0, 1, 2, 3, len(pages) - 1):
        assert dout.buf.to_numpy(np.uint8, pages[p][3], pages[p][2]).tobytes() == want[p]
    allw = np.frombuffer(b"".join(want), np.uint64)
    res = Dev(np.zeros(1, np.uint64))
    ag.call("ag_checksum64_dev", dout.ptr, allw.size, res.ptr, None)
    ag.call("ag_stream_sync", None)
    assert int(res.get()[0]) == checksum64(allw)
