"""Device LZ4_RAW page decompression against the Python restatement in tests/lz4_ref.py (host and _dev flavours, byte for
byte, the canary outside every written range), the seams of the shared-memory window and the span chain walk,
pyarrow-written LZ4 files end to end (read_lz4_chunk_dev) against pq.read_table, every page of the two parquet-testing
LZ4_RAW fixtures against liblz4, ~200 MB of output through a checksum, and the plain-C consumer."""
import os
import subprocess
import zlib

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import lz4_ref as R
import pq_files as F
import pq_pages as P
import test_c_programs
from arrow_go_b200 import _native as N
from helpers import Dev, checksum64, ptr
from pq_chunk import read_chunk_dev
from pq_pages import compressed_batch
from test_gpu_parquet_window import RESIDUES, SPAN, WIN, at_residues, upload

gpu = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
CANARY = 0xA5
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FIXTURES = ("lz4_raw_compressed.parquet", "lz4_raw_compressed_larger.parquet")
EXT = 16                 # extension bytes the parse reads from the window (kExt); a longer run leaves it
LOOK = 2 * EXT + 3       # bytes past a span a short sequence's header reaches (kLook)


def run_lz4(ag, src, pages, n_out, dev=False):
    """-> (status, message, out, written); out starts as the canary everywhere"""
    tbl = N.compressed_table(pages)
    out = np.full(n_out, CANARY, np.uint8)
    w = np.full(len(pages), -1, np.int64)
    if not dev:
        st, msg = ag.call_status("ag_parquet_lz4_raw_decompress", ptr(src), tbl, len(pages), ptr(out), ptr(w))
        return st, msg, out, w
    ds, do, dw = Dev(src), Dev(out), Dev(w)
    st, msg = ag.call_status("ag_parquet_lz4_raw_decompress_dev", ds.ptr, tbl, len(pages), do.ptr, dw.ptr, None)
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
    st, msg, out, w = run_lz4(ag, src, pages, n_out, dev)
    want, ww, errs = expect(src, pages, n_out)
    assert w.tolist() == ww, (msg, errs)
    assert out.tobytes() == want.tobytes(), (msg, errs)          # the canary outside every written range survives
    return st, msg, errs


@gpu
@FLAVOURS
def test_every_form(ag, dev):
    rng = np.random.default_rng(81)
    streams = [(s, len(x)) for _, s, x in R.forms()]
    streams += [(s, n) for _, s, n, (outcome, _), _ in R.differences() if outcome == R.OK]
    for gap in (True, False):
        st, msg, errs = decode_and_compare(ag, streams, rng, dev, gap)
        assert st == N.AG_OK and not errs, msg


@gpu
@FLAVOURS
def test_page_sizes(ag, dev):
    rng = np.random.default_rng(82)
    streams = []
    for n in (0, 1, 12, 13, 4095, 16384, 65535, 65536, 65537, 1 << 22):
        for make in (R.timestamps, R.dict_indices, R.runs, R.noise):
            x = make(n, n)
            streams.append((pa.compress(x, codec="lz4_raw", asbytes=True), n))
    streams.append((b"", 0))
    st, msg, errs = decode_and_compare(ag, streams, rng, dev)
    assert st == N.AG_OK and not errs, msg


@gpu
@FLAVOURS
@pytest.mark.parametrize("row", R.corrupt_rows() + [r[:4] + (None,) for r in R.differences() if r[3][0] != R.OK],
                         ids=lambda r: r[0])
def test_error_rows(ag, row, dev):
    name, s, n, _, _ = row
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = rng.integers(0, 3, 5000, dtype=np.uint8).tobytes()
    good = pa.compress(x, codec="lz4_raw", asbytes=True)
    # the failing page twice (pages 1 and 3 in the caller's order): the message names page 1
    src, pages, n_out = compressed_batch([(good, len(x)), (s, n), (good, len(x)), (s, n)], rng, gap=False)
    st, msg, out, w = run_lz4(ag, src, pages, n_out, dev)
    want, ww, errs = expect(src, pages, n_out)
    assert [e[0] for e in errs] == [1, 3]
    assert w.tolist() == ww and out.tobytes() == want.tobytes(), (msg, errs)
    assert st == N.AG_ERR_INVALID and f"lz4_raw_decompress: page 1: {errs[0][1]} ({ww[1]} bytes written)" in msg, (msg, errs)
    assert ww[0] == ww[2] == len(x)


@gpu
@FLAVOURS
def test_invalid_arguments(ag, dev):
    src = np.frombuffer(R.block(R.seq(b"abcd", 4, 8)), np.uint8).copy()
    n = len(src)
    bad = [
        ([(-1, n, 0, 28)], "page 0: negative field"),
        ([(0, n, 0, 28), (0, -1, 40, 28)], "page 1: negative field"),
        ([(0, n, 0, 28), (0, n, -4, 28)], "page 1: negative field"),
        ([(0, n, 0, -28)], "page 0: negative field"),
        ([(0, 1 << 32, 0, 28)], "more than 2^32-1 bytes"),
        ([(0, n, 0, 1 << 32)], "more than 2^32-1 bytes"),
        ([(0, n, 0, 28), (0, n, 60, 28), (0, n, 27, 28)], "pages 0 and 2: overlapping dst ranges"),
    ]
    out = Dev(nbytes=256)
    for pages, text in bad:
        if dev:
            st, msg = ag.call_status("ag_parquet_lz4_raw_decompress_dev", Dev(src).ptr, N.compressed_table(pages), len(pages), out.ptr, None, None)
        else:
            h = np.zeros(256, np.uint8)
            st, msg = ag.call_status("ag_parquet_lz4_raw_decompress", ptr(src), N.compressed_table(pages), len(pages), ptr(h), None)
        assert st == N.AG_ERR_INVALID and "lz4_raw_decompress" in msg and text in msg, (pages, msg)
    pages = [(0, n, 0, 28), (0, 0, 5, 0), (0, n, 28, 28)]
    st, msg, o, w = run_lz4(ag, np.concatenate([src, np.zeros(8, np.uint8)]), pages, 64, dev)
    want = b"abcdabcdabcd" + R.TAIL
    assert st == N.AG_OK and w.tolist() == [28, 0, 28] and o[:56].tobytes() == want * 2, msg


# ---------------------------------------------------------------- window and span seams ----
def seam_stream(rng, count):
    """[(sequence bytes, info)] of a valid stream built while replaying the parse for residue 0, so that sequences land
    on the seams: short sequences with extension runs of 1..5 bytes (across span ends), a probe in the last span of
    every window whose literals carry its offset and a 10-byte match extension run onto the window end, runs longer
    than EXT bytes, and one literal longer than the window.  info: start, end, last byte read, the literal
    extension, offset and match extension ranges, and whether a run is longer than EXT."""
    items, pos, out, cur, wend, cur0, probed, big = [], 0, 0, 0, WIN, 0, False, False

    def add(lit, off=None, ml=None):
        nonlocal pos, out, cur, wend, cur0, probed
        s = R.seq(lit, off, ml)
        ll = len(lit)
        kl = len(R.ext(ll - 15)) if ll >= 15 else 0
        po = pos + 1 + kl + ll if off is not None else None
        km = pos + len(s) - po - 2 if off is not None else 0
        inf = {"start": pos, "end": pos + len(s), "last": pos + len(s) - 1 if off is not None else pos + kl,
               "lx": (pos + 1, pos + 1 + kl), "off": (po, po + 2) if po is not None else None,
               "mx": (po + 2, po + 2 + km) if po is not None else None, "long": kl > EXT or km > EXT}
        items.append((s, inf))
        pos += len(s)
        out += ll + (ml or 0)
        if inf["long"] or inf["last"] >= wend or inf["end"] >= cur + SPAN:   # the span ends after this sequence
            cur = inf["end"]
            if cur + SPAN + LOOK > wend:
                cur0, probed = cur, False
                wend = cur - cur % 16 + WIN

    add(rng.integers(0, 256, 64, dtype=np.uint8).tobytes(), 64, 4)
    while len(items) < count:
        off = lambda ml_: int(rng.integers(1, min(out, 65535) + 1))
        if not probed and cur + SPAN - 120 <= pos < cur + SPAN and cur0 + WIN - 16 - pos < 4000:
            target = cur0 + WIN - 16 + 2                         # the offset's first byte, 3 below the highest window end
            for k in range(0, 20):
                ll = target - pos - 1 - k
                if ll >= 0 and (len(R.ext(ll - 15)) if ll >= 15 else 0) == k:
                    ml = 19 + 255 * 9 + 100                      # a 10-byte match extension run
                    add(rng.integers(0, 256, ll, dtype=np.uint8).tobytes(), off(ml), ml)
                    break
            probed = True
            continue
        u = rng.random()
        if u < 0.002 and not big:
            big = True
            add(rng.integers(0, 256, WIN + 700, dtype=np.uint8).tobytes(), 7, 30)    # literals longer than the window
            continue
        if u < 0.006:
            ml = 19 + 255 * int(rng.integers(EXT, EXT + 3)) + int(rng.integers(0, 255))   # a run longer than EXT bytes
            add(rng.integers(0, 256, int(rng.integers(0, 4)), dtype=np.uint8).tobytes(), off(ml), ml)
            continue
        if u < 0.008:
            ll = 15 + 255 * EXT + int(rng.integers(0, 255))
            add(rng.integers(0, 256, ll, dtype=np.uint8).tobytes(), 1, 4)
            continue
        ll = 15 + 255 * int(rng.integers(0, 5)) + int(rng.integers(0, 255)) if u < 0.03 else \
            int(rng.integers(15, 30)) if u < 0.12 else int(rng.integers(0, 13))
        ml = 19 + 255 * int(rng.integers(0, 5)) + int(rng.integers(0, 255)) if rng.random() < 0.15 else int(rng.integers(4, 19))
        add(rng.integers(0, 256, ll, dtype=np.uint8).tobytes(), off(ml), ml)
    add(R.TAIL)
    return items


def seam_spans(info, n, residue):
    """lz4_parse_kernel's spans over a valid stream: [(span start, first sequence, last sequence, window end, whether
    the last sequence left the window)]"""
    out, wlo, i = [], -(1 << 62), 0
    while i < len(info):
        cur = info[i]["start"]
        if min(cur + SPAN + LOOK, n) > wlo + WIN:
            wlo = cur - (residue + cur) % 16
        wend = wlo + WIN
        j = i
        while True:
            f = info[j]
            left = f["long"] or f["last"] >= wend
            if left or f["end"] >= cur + SPAN or f["end"] >= n:
                break
            j += 1
        out.append((cur, i, j, wend, left))
        i = j + 1
    return out


def seams(info, spans):
    """the seams the spans cross: (kind, boundary) for every field of a span's sequences that straddles the span end or
    the window end, the span positions of the spans' last tokens, and the kinds of sequences that left the window"""
    hit, last_q, left = set(), set(), set()
    for cur, i, j, wend, lft in spans:
        last_q.add(info[j]["start"] - cur)
        for k in range(i, j + 1):
            f = info[k]
            for field in ("lx", "off", "mx"):
                r = f[field]
                if r is None or r[1] <= r[0]:
                    continue
                for name, b in (("span", cur + SPAN), ("window", wend)):
                    if r[0] < b < r[1]:
                        hit.add((field, name))
        if lft:
            f = info[j]
            left.add("long_run" if f["long"] else "past_window")
            if f["off"] and f["off"][0] - f["start"] > WIN:
                left.add("literal_longer_than_window")
    return hit, last_q, left


@gpu
def test_lz4_sequences_at_span_and_window_edges(ag):
    rng = np.random.default_rng(820)
    items = seam_stream(rng, 40_000)
    good = b"".join(s for s, _ in items)
    info = [f for _, f in items]
    hit, last_q, left = set(), set(), set()
    for r in RESIDUES:
        h, q, lf = seams(info, seam_spans(info, len(good), r))
        hit |= h; last_q |= q; left |= lf
    assert {1020, 1021, 1022, 1023} <= last_q
    assert {("lx", "span"), ("off", "span"), ("mx", "span"), ("off", "window"), ("mx", "window")} <= hit, hit
    assert {"long_run", "past_window", "literal_longer_than_window"} <= left, left
    _, outcome, dlen = R.decode(good, 1 << 40)
    assert outcome == R.SIZE
    # offset 0 at the first sequence of a span and at the last (not one that leaves the window)
    sp = seam_spans(info, len(good), 0)
    first = next(i for cur, i, j, w, lft in sp[3:] if info[i]["off"])
    last = next(j for cur, i, j, w, lft in sp[3:] if info[j]["off"] and not lft and info[j]["start"] - cur >= 1000)
    streams = [good]
    for k in (first, last):
        b = bytearray(good)
        a = info[k]["off"][0]
        b[a:a + 2] = b"\0\0"
        streams.append(bytes(b))
    for s in streams:
        src, pages, n_out = at_residues(s, dlen)
        tbl = N.compressed_table([(o, ln, d, dl) for o, ln, dl, d in pages])
        ds, do, dw = upload(src), Dev(np.full(n_out, CANARY, np.uint8)), Dev(np.full(16, -1, np.int64))
        st, msg = ag.call_status("ag_parquet_lz4_raw_decompress_dev", ds.ptr, tbl, 16, do.ptr, dw.ptr, None)
        ag.call("ag_stream_sync", None)
        want, outcome, arg = R.decode(s, dlen)
        assert dw.get().tolist() == [len(want)] * 16, msg
        got = do.get().reshape(16, dlen)
        assert all(g[:len(want)].tobytes() == want and (g[len(want):] == CANARY).all() for g in got)
        if outcome != R.OK:
            assert st == N.AG_ERR_INVALID and f"page 0: {R.message(outcome, arg, dlen)} ({len(want)} bytes written)" in msg, msg
        else:
            assert st == N.AG_OK, msg


# ---------------------------------------------------------------- files ----
def read_lz4_chunk_dev(ag, plan):
    """INTEGRATION.md §6 for an LZ4_RAW chunk -> (values, validity): upload the chunk as it sits in the file, one
    ag_parquet_lz4_raw_decompress_dev call (and device copies of the pages that are not compressed) into `dst`, checked
    byte for byte against liblz4 (pyarrow's "lz4_raw" codec; "lz4" is the frame format).  read_chunk_dev then decodes
    the levels and values from exactly those bytes, handed to it as an uncompressed tail of the chunk."""
    dchunk, ddst = Dev(P.as_array(plan["chunk"])), Dev(nbytes=plan["n_dst"])
    dw = Dev(np.full(len(plan["comp"]) + 1, -1, np.int64))
    ag.call("ag_parquet_lz4_raw_decompress_dev", dchunk.ptr, N.compressed_table(plan["comp"]), len(plan["comp"]), ddst.ptr, dw.ptr, None)
    for s, d, k in plan["copies"]:
        ag.call("ag_copy_dev", ddst.ptr + d, dchunk.ptr + s, k, None)
    ag.call("ag_stream_sync", None)
    assert dw.get().tolist()[:len(plan["comp"])] == [c[3] for c in plan["comp"]]
    dst = ddst.get(np.uint8, plan["n_dst"]).tobytes()
    chunk = bytes(plan["chunk"])
    want = bytearray(plan["n_dst"])
    for s, sl, d, dl in plan["comp"]:
        if dl:
            want[d:d + dl] = pa.decompress(chunk[s:s + sl], decompressed_size=dl, codec="lz4_raw", asbytes=True)
    for s, d, k in plan["copies"]:
        want[d:d + k] = chunk[s:s + k]
    assert dst == bytes(want)
    return read_chunk_dev(ag, dict(plan, chunk=chunk + dst, comp=[], copies=[(len(chunk), 0, plan["n_dst"])]))


def check_file(ag, tbl, path):
    """-> the number of LZ4_RAW page bodies in the chunk (a v2 page whose body LZ4 would not shrink is stored as is)"""
    plan = P.chunk_plan(path)
    assert plan["codec"] == "LZ4"
    values, valid = read_lz4_chunk_dev(ag, plan)
    want, wvalid = F.expected(tbl, plan)
    assert np.array_equal(valid, wvalid)
    assert values == want
    return len(plan["comp"])


@gpu
@pytest.mark.parametrize("case", F.compressed_cases(), ids=F.compressed_case_id)
def test_pyarrow_lz4_files_end_to_end(ag, case, tmp_path):
    rng = np.random.default_rng(zlib.crc32(F.compressed_case_id(case).encode()))
    path = str(tmp_path / "c.parquet")
    check_file(ag, F.write_numeric_case(path, rng, case, compression="LZ4"), path)


@gpu
@pytest.mark.parametrize("kind", ["byte_array", "fsb12", "bool"])
def test_pyarrow_lz4_files_other_types(ag, kind, tmp_path):
    rng = np.random.default_rng(zlib.crc32(kind.encode()))
    path = str(tmp_path / "c.parquet")
    if kind == "byte_array":
        arr, enc = F.make_string_column(rng, "RLE_DICTIONARY", 8000, 0.1), "RLE_DICTIONARY"
    else:
        arr, enc = F.make_array(rng, kind, 20_000, 0.1), F.KINDS[kind]
    # v1 pages: their bodies are always compressed, so every page of these columns goes through the codec
    tbl = F.write_column(path, arr, nullable=True, encoding=enc, version="1.0", compression="LZ4", data_page_size=8192)
    assert check_file(ag, tbl, path) == len(P.chunk_plan(path)["pages"]) + (1 if P.chunk_plan(path)["dict"] else 0)


@gpu
@FLAVOURS
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_pages_against_host(ag, name, dev):
    """every page of every column, compared as decompressed bytes with liblz4's, and the numeric columns end to end"""
    path = os.path.join(GOLDEN, name)
    rng = np.random.default_rng(83)
    tbl = pq.read_table(path)
    for c in range(pq.ParquetFile(path).metadata.num_columns):
        chunk, pages = P.column_chunk(path, column=c)
        regions, comp, _ = P.decompress_table(pages)
        streams = [(chunk[regions[k][0]:regions[k][0] + regions[k][1]], regions[k][3]) for k in comp]
        assert streams
        src, pt, n_out = compressed_batch(streams, rng)
        st, msg, out, w = run_lz4(ag, src, pt, n_out, dev)
        assert st == N.AG_OK, (c, msg)
        for (s, sl, d, dl), k in zip(pt, w):
            want = pa.decompress(bytes(src[s:s + sl]), decompressed_size=dl, codec="lz4_raw", asbytes=True) if dl else b""
            assert k == dl and out[d:d + dl].tobytes() == want, c
        plan = P.chunk_plan(path, c)
        if plan["ptype"] in (P.INT32, P.INT64, P.FLOAT, P.DOUBLE):
            values, valid = read_lz4_chunk_dev(ag, plan)
            want, wvalid = F.expected(tbl.select([c]), plan)
            assert np.array_equal(valid, wvalid) and values == want, c


@gpu
def test_decompress_200mb_device(ag):
    """~200 MB of output over 2^19-value int64 timestamp pages, 17-bit index pages and runs: three pages against the
    host bodies, the whole output through a checksum against the host twin."""
    per_page = 1 << 19                                           # every body a whole number of 8-byte words
    bodies = [R.timestamps(8 * per_page, k) for k in range(2)] + [R.dict_indices(17 * per_page // 8, 2), R.runs(4 * per_page, 3)]
    encs = [pa.compress(b, codec="lz4_raw", asbytes=True) for b in bodies]
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
    ag.call("ag_parquet_lz4_raw_decompress_dev", ds.ptr, N.compressed_table(pages), len(pages), dout.ptr, dw.ptr, None)
    ag.call("ag_stream_sync", None)
    assert dw.get().tolist() == [p[3] for p in pages]
    for p in (0, 1, 2, 3, len(pages) - 1):
        assert dout.buf.to_numpy(np.uint8, pages[p][3], pages[p][2]).tobytes() == want[p]
    allw = np.frombuffer(b"".join(want), np.uint64)
    res = Dev(np.zeros(1, np.uint64))
    ag.call("ag_checksum64_dev", dout.ptr, allw.size, res.ptr, None)
    ag.call("ag_stream_sync", None)
    assert int(res.get()[0]) == checksum64(allw)


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_c_smoke_is_refused_without_gpu(tmp_path):
    out = subprocess.run([test_c_programs.build("pq_lz4_smoke", str(tmp_path))], capture_output=True, text=True, timeout=120)
    assert out.returncode == 77, (out.returncode, out.stdout, out.stderr)


@gpu
def test_c_smoke_on_gpu(tmp_path):
    out = subprocess.run([test_c_programs.build("pq_lz4_smoke", str(tmp_path))], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
    assert "pq_lz4_smoke ok" in out.stdout
