"""Device GZIP page decompression against the Python restatement in tests/gzip_ref.py (host and _dev flavours, byte for
byte, the canary outside every written range), pyarrow-written GZIP files end to end (read_gzip_chunk_dev) against
pq.read_table, every page of the two parquet-testing GZIP fixtures against pyarrow's host decompression, ~200 MB of
output through a checksum, and the plain-C consumer."""
import os
import subprocess
import zlib

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import gzip_ref as R
import pq_files as F
import pq_pages as P
import test_c_programs
from arrow_go_b200 import _native as N
from helpers import Dev, checksum64, ptr
from pq_chunk import read_chunk_dev
from pq_pages import compressed_batch

gpu = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
CANARY = 0xA5
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FIXTURES = ("concatenated_gzip_members.parquet", "byte_stream_split_extended.gzip.parquet")


def run_gzip(ag, src, pages, n_out, dev=False):
    """-> (status, message, out, written); out starts as the canary everywhere"""
    tbl = N.compressed_table(pages)
    out = np.full(n_out, CANARY, np.uint8)
    w = np.full(len(pages), -1, np.int64)
    if not dev:
        st, msg = ag.call_status("ag_parquet_gzip_decompress", ptr(src), tbl, len(pages), ptr(out), ptr(w))
        return st, msg, out, w
    ds, do, dw = Dev(src), Dev(out), Dev(w)
    st, msg = ag.call_status("ag_parquet_gzip_decompress_dev", ds.ptr, tbl, len(pages), do.ptr, dw.ptr, None)
    ag.call("ag_stream_sync", None)
    return st, msg, do.get(), dw.get()


def expect(src, pages, n_out):
    """restatement: (out, written, [(page index, message)] of failing pages)"""
    want = np.full(n_out, CANARY, np.uint8)
    w, errs = [], []
    for k, (s, sl, d, dl) in enumerate(pages):
        got, outcome, arg = R.decode(bytes(src[s:s + sl]), dl)
        want[d:d + len(got)] = np.frombuffer(got, np.uint8)
        w.append(len(got))
        if outcome != R.OK:
            errs.append((k, R.message(outcome, arg, dl)))
    return want, w, errs


def decode_and_compare(ag, streams, rng, dev, gap=True):
    src, pages, n_out = compressed_batch(streams, rng, gap)
    st, msg, out, w = run_gzip(ag, src, pages, n_out, dev)
    want, ww, errs = expect(src, pages, n_out)
    assert w.tolist() == ww, (msg, errs)
    assert out.tobytes() == want.tobytes(), (msg, errs)          # the canary outside every written range survives
    return st, msg, errs


@gpu
@FLAVOURS
def test_every_form(ag, dev):
    rng = np.random.default_rng(91)
    streams = [(s, len(x)) for _, s, x in R.forms()]
    x = R.payload(40000, 9)
    streams += [(R.gz(x, lv, st), len(x)) for lv in (0, 1, 6, 9) for st in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED)]
    for gap in (True, False):
        st, msg, errs = decode_and_compare(ag, streams, rng, dev, gap)
        assert st == N.AG_OK and not errs, msg


@gpu
@FLAVOURS
def test_page_sizes(ag, dev):
    rng = np.random.default_rng(92)
    streams = []
    for n in (0, 1, 32767, 32768, 32769, 65535, 65536, 1 << 22):
        x = (np.cumsum(rng.integers(0, 1000, (n + 7) // 8)) + (1 << 40)).astype(np.int64).tobytes()[:n]
        streams.append((pa.compress(x, codec="gzip", asbytes=True), n))
        streams.append((R.gz(x, 0), n))                         # stored blocks
    streams.append((b"", 0))
    st, msg, errs = decode_and_compare(ag, streams, rng, dev)
    assert st == N.AG_OK and not errs, msg


@gpu
@FLAVOURS
@pytest.mark.parametrize("row", R.corrupt_rows(), ids=lambda r: r[0])
def test_error_rows(ag, row, dev):
    name, s, n, _ = row
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = rng.integers(0, 3, 5000, dtype=np.uint8).tobytes()
    good = pa.compress(x, codec="gzip", asbytes=True)
    # the failing page twice (pages 1 and 3 in the caller's order): the message names page 1
    src, pages, n_out = compressed_batch([(good, len(x)), (s, n), (good, len(x)), (s, n)], rng, gap=False)
    st, msg, out, w = run_gzip(ag, src, pages, n_out, dev)
    want, ww, errs = expect(src, pages, n_out)
    assert [e[0] for e in errs] == [1, 3]
    assert w.tolist() == ww and out.tobytes() == want.tobytes(), (msg, errs)
    assert st == N.AG_ERR_INVALID and f"gzip_decompress: page 1: {errs[0][1]} ({ww[1]} bytes written)" in msg, (msg, errs)
    assert ww[0] == ww[2] == len(x)


@gpu
@FLAVOURS
def test_invalid_arguments(ag, dev):
    src = np.frombuffer(pa.compress(b"abcdabcdabcd", codec="gzip", asbytes=True), np.uint8).copy()
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
            st, msg = ag.call_status("ag_parquet_gzip_decompress_dev", Dev(src).ptr, N.compressed_table(pages), len(pages), out.ptr, None, None)
        else:
            h = np.zeros(256, np.uint8)
            st, msg = ag.call_status("ag_parquet_gzip_decompress", ptr(src), N.compressed_table(pages), len(pages), ptr(h), None)
        assert st == N.AG_ERR_INVALID and "gzip_decompress" in msg and text in msg, (pages, msg)
    pages = [(0, n, 0, 12), (0, 0, 5, 0), (0, n, 12, 12)]
    st, msg, o, w = run_gzip(ag, np.concatenate([src, np.zeros(8, np.uint8)]), pages, 32, dev)
    assert st == N.AG_OK and w.tolist() == [12, 0, 12] and o[:24].tobytes() == b"abcdabcdabcd" * 2, msg


def read_gzip_chunk_dev(ag, plan):
    """INTEGRATION.md §6 for a GZIP chunk -> (values, validity): upload the chunk as it sits in the file, one
    ag_parquet_gzip_decompress_dev call (and device copies of the pages that are not compressed) into `dst`, checked
    byte for byte against pyarrow's host decompression.  read_chunk_dev then decodes the levels and values from exactly
    those bytes, handed to it as an uncompressed tail of the chunk: every page body is one device copy away from its
    offset in `dst`, and v2 levels keep their offsets in the chunk."""
    dchunk, ddst = Dev(P.as_array(plan["chunk"])), Dev(nbytes=plan["n_dst"])
    dw = Dev(np.full(len(plan["comp"]) + 1, -1, np.int64))
    ag.call("ag_parquet_gzip_decompress_dev", dchunk.ptr, N.compressed_table(plan["comp"]), len(plan["comp"]), ddst.ptr, dw.ptr, None)
    for s, d, k in plan["copies"]:
        ag.call("ag_copy_dev", ddst.ptr + d, dchunk.ptr + s, k, None)
    ag.call("ag_stream_sync", None)
    assert dw.get().tolist()[:len(plan["comp"])] == [c[3] for c in plan["comp"]]
    dst = ddst.get(np.uint8, plan["n_dst"]).tobytes()
    assert dst == P.host_decompress(plan)
    chunk = bytes(plan["chunk"])
    return read_chunk_dev(ag, dict(plan, chunk=chunk + dst, comp=[], copies=[(len(chunk), 0, plan["n_dst"])]))


def check_file(ag, tbl, path):
    """-> the number of GZIP page bodies in the chunk (a v2 page whose body GZIP would not shrink is stored as is)"""
    plan = P.chunk_plan(path)
    assert plan["codec"] == "GZIP"
    values, valid = read_gzip_chunk_dev(ag, plan)
    want, wvalid = F.expected(tbl, plan)
    assert np.array_equal(valid, wvalid)
    assert values == want
    return len(plan["comp"])


@gpu
@pytest.mark.parametrize("case", F.compressed_cases(), ids=F.compressed_case_id)
def test_pyarrow_gzip_files_end_to_end(ag, case, tmp_path):
    rng = np.random.default_rng(zlib.crc32(F.compressed_case_id(case).encode()))
    path = str(tmp_path / "c.parquet")
    check_file(ag, F.write_numeric_case(path, rng, case, compression="GZIP"), path)


@gpu
@pytest.mark.parametrize("kind", ["byte_array", "fsb12", "bool"])
def test_pyarrow_gzip_files_other_types(ag, kind, tmp_path):
    rng = np.random.default_rng(zlib.crc32(kind.encode()))
    path = str(tmp_path / "c.parquet")
    if kind == "byte_array":
        arr, enc = F.make_string_column(rng, "RLE_DICTIONARY", 8000, 0.1), "RLE_DICTIONARY"
    else:
        arr, enc = F.make_array(rng, kind, 20_000, 0.1), F.KINDS[kind]
    # v1 pages: their bodies are always GZIP, so every page of these columns goes through the codec
    tbl = F.write_column(path, arr, nullable=True, encoding=enc, version="1.0", compression="GZIP", data_page_size=8192)
    assert check_file(ag, tbl, path) == len(P.chunk_plan(path)["pages"]) + (1 if P.chunk_plan(path)["dict"] else 0)


@gpu
@FLAVOURS
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_pages_against_host(ag, name, dev):
    """every page of every column, compared as decompressed bytes with pyarrow's, and the whole file with pq.read_table"""
    path = os.path.join(GOLDEN, name)
    rng = np.random.default_rng(93)
    tbl = pq.read_table(path)
    for c in range(pq.ParquetFile(path).metadata.num_columns):
        chunk, pages = P.column_chunk(path, column=c)
        regions, comp, _ = P.decompress_table(pages)
        streams = [(chunk[regions[k][0]:regions[k][0] + regions[k][1]], regions[k][3]) for k in comp]
        assert streams
        src, pt, n_out = compressed_batch(streams, rng)
        st, msg, out, w = run_gzip(ag, src, pt, n_out, dev)
        assert st == N.AG_OK, (c, msg)
        for (s, sl, d, dl), k in zip(pt, w):
            want = pa.decompress(bytes(src[s:s + sl]), decompressed_size=dl, codec="gzip", asbytes=True) if dl else b""
            assert k == dl and out[d:d + dl].tobytes() == want, c
        plan = P.chunk_plan(path, c)
        if plan["ptype"] in (P.INT32, P.INT64, P.FLOAT, P.DOUBLE):
            values, valid = read_gzip_chunk_dev(ag, plan)
            want, wvalid = F.expected(tbl.select([c]), plan)
            assert np.array_equal(valid, wvalid) and values == want, c


@gpu
def test_decompress_200mb_device(ag):
    """~200 MB of output over 2^19-value int64 timestamp pages and 17-bit index pages, some of them three members with
    FHCRC headers: three pages against pyarrow, the whole output through a checksum against the host twin."""
    rng = np.random.default_rng(94)
    per_page = 1 << 19
    bodies = [(np.cumsum(rng.integers(0, 1000, per_page)) + (k << 40)).astype(np.int64).tobytes() for k in range(2)]
    bodies += [(rng.integers(0, 100_000, per_page) & 0x1FFFF).astype(np.uint32).tobytes() for _ in range(2)]
    encs = [pa.compress(b, codec="gzip", asbytes=True) for b in bodies]
    for k in (1, 2):
        b, third = bodies[k], len(bodies[k]) // 3
        parts = [b[:third], b[third:2 * third], b[2 * third:]]
        encs[k] = b"".join(R.member(R.gz(p)[10:-8], hcrc=True, name=b"part", payload=p) for p in parts)
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
    ag.call("ag_parquet_gzip_decompress_dev", ds.ptr, N.compressed_table(pages), len(pages), dout.ptr, dw.ptr, None)
    ag.call("ag_stream_sync", None)
    assert dw.get().tolist() == [p[3] for p in pages]
    for p in (0, 1, 2, len(pages) - 1):
        assert dout.buf.to_numpy(np.uint8, pages[p][3], pages[p][2]).tobytes() == want[p]
    allw = np.frombuffer(b"".join(want), np.uint64)
    res = Dev(np.zeros(1, np.uint64))
    ag.call("ag_checksum64_dev", dout.ptr, allw.size, res.ptr, None)
    ag.call("ag_stream_sync", None)
    assert int(res.get()[0]) == checksum64(allw)


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_c_smoke_is_refused_without_gpu(tmp_path):
    out = subprocess.run([test_c_programs.build("pq_gzip_smoke", str(tmp_path))], capture_output=True, text=True, timeout=120)
    assert out.returncode == 77, (out.returncode, out.stdout, out.stderr)


@gpu
def test_c_smoke_on_gpu(tmp_path):
    out = subprocess.run([test_c_programs.build("pq_gzip_smoke", str(tmp_path))], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
    assert "pq_gzip_smoke ok" in out.stdout
