"""Device SNAPPY page compression (host and _dev flavours) against the parse of tests/snappy_encode_model.py, byte for
byte, with guard bytes around every page; argument errors before any launch; round trips through the device
decompressor and pyarrow, ~200 MB in one batch, output offsets past 2^31, and a pyarrow-written SNAPPY chunk
decompressed and recompressed on the device."""
import numpy as np
import pyarrow as pa
import pytest

import pq_codecs as H
import pq_files as F
import pq_pages as P
import snappy_encode_model as M
from arrow_go_b200 import _native as N
from helpers import Dev, checksum64, ptr

gpu = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
CANARY = 0xA5


def layout(bodies, rng, gap=True):
    """bodies at odd offsets of one input, each page's capacity (the bound plus some) with gaps between them, the page
    order shuffled.  -> (src, pages, n_out, bodies in page order)"""
    blob, pages, out = bytearray(), [], 3 if gap else 0
    for b in bodies:
        if gap:
            blob += bytes(int(rng.integers(0, 7)))
        cap = M.max_size(len(b)) + (int(rng.integers(0, 9)) if gap else 0)
        pages.append((len(blob), len(b), out, cap))
        blob += b
        out += cap + (int(rng.integers(1, 6)) if gap else 0)
    blob += bytes(8)
    order = rng.permutation(len(pages)) if gap else np.arange(len(pages))
    return P.as_array(blob), [pages[i] for i in order], out + 8, [bodies[i] for i in order]


def compress(ag, src, pages, n_out, dev):
    """-> (status, message, out, written); out starts as the canary everywhere"""
    tbl = N.compressed_table(pages)
    out = np.full(n_out, CANARY, np.uint8)
    w = np.full(len(pages), -1, np.int64)
    if not dev:
        st, msg = ag.call_status("ag_parquet_snappy_compress", ptr(src), tbl, len(pages), ptr(out), ptr(w))
        return st, msg, out, w
    ds, do, dw = Dev(src), Dev(out), Dev(w)
    st, msg = ag.call_status("ag_parquet_snappy_compress_dev", ds.ptr, tbl, len(pages), do.ptr, dw.ptr, None)
    ag.call("ag_stream_sync", None)
    return st, msg, do.get(), dw.get()


def device_round_trip(ag, out, pages, written, bodies):
    """every stream back through ag_parquet_snappy_decompress_dev"""
    back = [(d, int(k), 0, 0) for (_, _, d, _), k in zip(pages, written)]
    pos = 0
    for k, b in enumerate(bodies):
        back[k] = back[k][:2] + (pos, len(b))
        pos += len(b) + 1
    streams, res = Dev(out), Dev(nbytes=pos + 8)                 # held: a Dev frees its buffer when collected
    ag.call("ag_parquet_snappy_decompress_dev", streams.ptr, N.compressed_table(back), len(back), res.ptr, None, None)
    ag.call("ag_stream_sync", None)
    got = res.get(count=pos + 8)
    for (_, _, d, dl), b in zip(back, bodies):
        assert got[d:d + dl].tobytes() == b


def check_batch(ag, bodies, seed, gap=True):
    for dev in (False, True):
        rng = np.random.default_rng(seed)
        src, pages, n_out, order = layout(bodies, rng, gap)
        st, msg, out, w = compress(ag, src, pages, n_out, dev)
        assert st == N.AG_OK, msg
        want = np.full(n_out, CANARY, np.uint8)
        streams = [M.compress(b) for b in order]
        for (_, _, d, _), c in zip(pages, streams):
            want[d:d + len(c)] = np.frombuffer(c, np.uint8)
        assert w.tolist() == [len(c) for c in streams]
        assert out.tobytes() == want.tobytes()                   # guard bytes: nothing past written changes
        device_round_trip(ag, out, pages, w, order)


@gpu
def test_short_and_empty_pages(ag):
    rng = np.random.default_rng(1)
    bodies = [b"", b"a", b"ab", b"abc", b"", b"abcd", b"aaaaa", rng.integers(0, 256, 3, dtype=np.uint8).tobytes()]
    check_batch(ag, bodies, 1)
    check_batch(ag, bodies, 2, gap=False)


@gpu
def test_fragment_boundaries(ag):
    rng = np.random.default_rng(2)
    base = M.corpora(rng, 5 * 65536 + 100)
    bodies = []
    for n in (65535, 65536, 65537, 2 * 65536 - 1, 2 * 65536, 2 * 65536 + 3, 5 * 65536 + 77):
        bodies += [base["timestamps"][:n], base["emails"][:n]]
    bodies += [bytes(3 * 65536 + 5), rng.integers(0, 256, 2 * 65536 + 9, dtype=np.uint8).tobytes()]
    check_batch(ag, bodies, 3)


@gpu
def test_corpora(ag):
    rng = np.random.default_rng(4)
    bodies = list(M.corpora(rng, 300_000).values()) + [rng.integers(0, 256, 200_000, dtype=np.uint8).tobytes()]
    check_batch(ag, bodies, 4)


@gpu
def test_pyarrow_page_bodies(ag, tmp_path):
    rng = np.random.default_rng(5)
    n = 200_000
    path = str(tmp_path / "p.parquet")
    vals = pa.array(np.round(rng.lognormal(4, 1, n), 2), mask=rng.random(n) < 0.05)
    F.write_column(path, vals, nullable=True, encoding="PLAIN", version="1.0", compression="SNAPPY", data_page_size=1 << 17)
    plan = P.chunk_plan(path)
    dst = P.host_decompress(plan)
    check_batch(ag, [dst[d:d + dl] for _, _, d, dl in plan["comp"]], 5)


@gpu
@FLAVOURS
def test_invalid_arguments(ag, dev):
    src = np.frombuffer(b"abcdabcdabcdabcd", np.uint8).copy()
    cap = M.max_size(16)
    bad = [
        ([(-1, 16, 0, cap)], "page 0: negative field"),
        ([(0, 16, 0, cap), (0, -1, 200, cap)], "page 1: negative field"),
        ([(0, 16, 0, cap), (0, 16, -4, cap)], "page 1: negative field"),
        ([(0, 16, 0, -1)], "page 0: negative field"),
        ([(0, 16, 0, cap), (0, 1 << 32, 100, M.max_size(1 << 32))], "page 1: more than 2^32-1 bytes"),
        ([(0, 16, 0, cap), (0, 16, 100, cap - 1)], f"page 1: capacity {cap - 1} below the bound {cap}"),
        ([(0, 0, 0, 31)], "page 0: capacity 31 below the bound 32"),
        ([(0, 16, 0, cap), (0, 16, 2 * cap + 4, cap), (0, 16, cap - 1, cap)], "pages 0 and 2: overlapping dst ranges"),
    ]
    n_out = 4 * cap + 8
    for pages, text in bad:
        tbl = N.compressed_table(pages)
        if dev:
            ds, out = Dev(src), Dev(np.full(n_out, CANARY, np.uint8))
            st, msg = ag.call_status("ag_parquet_snappy_compress_dev", ds.ptr, tbl, len(pages), out.ptr, None, None)
            ag.call("ag_stream_sync", None)
            got = out.get()
        else:
            got = np.full(n_out, CANARY, np.uint8)
            st, msg = ag.call_status("ag_parquet_snappy_compress", ptr(src), tbl, len(pages), ptr(got), None)
        assert st == N.AG_ERR_INVALID and "snappy_compress" in msg and text in msg, (pages, msg)
        assert (got == CANARY).all()
    # adjacent capacities do not overlap; pages may share input
    st, msg, out, w = compress(ag, src, [(0, 16, 0, cap), (4, 12, cap, M.max_size(12))], n_out, dev)
    assert st == N.AG_OK and w.tolist() == [len(M.compress(src.tobytes())), len(M.compress(src[4:].tobytes()))], msg


@gpu
def test_200mb_round_trip(ag):
    """~200 MB of input in 4 MB pages, checked by round trip: pyarrow on a sample of pages, the device decompressor on
    all of them through a checksum"""
    bodies, _ = H.SNAPPY.big()
    offs, blob = [], bytearray()
    for b in bodies:
        offs.append(len(blob))
        blob += b
    pages, d = [], 0
    while sum(p[1] for p in pages) < 200_000_000:
        k = len(pages) % 4
        cap = M.max_size(len(bodies[k]))
        pages.append((offs[k], len(bodies[k]), d, cap))
        d += cap + 3
    ds, dout, dw = Dev(np.frombuffer(bytes(blob), np.uint8).copy()), Dev(nbytes=d), Dev(np.zeros(len(pages), np.int64))
    ag.call("ag_parquet_snappy_compress_dev", ds.ptr, N.compressed_table(pages), len(pages), dout.ptr, dw.ptr, None)
    ag.call("ag_stream_sync", None)
    w = dw.get()
    for i in (0, 1, 2, 3, len(pages) - 1):
        s = dout.buf.to_numpy(np.uint8, int(w[i]), pages[i][2]).tobytes()
        assert pa.decompress(s, decompressed_size=pages[i][1], codec="snappy", asbytes=True) == bodies[i % 4]
        assert len(s) <= 1.05 * len(pa.compress(bodies[i % 4], codec="snappy", asbytes=True))
    back, pos = [], 0
    for (_, sl, dd, _), k in zip(pages, w):
        back.append((dd, int(k), pos, sl))
        pos += sl
    res = Dev(nbytes=pos)
    ag.call("ag_parquet_snappy_decompress_dev", dout.ptr, N.compressed_table(back), len(back), res.ptr, None, None)
    ag.call("ag_stream_sync", None)
    want = np.frombuffer(b"".join(bodies[i % 4] for i in range(len(pages))), np.uint64)
    got = Dev(np.zeros(1, np.uint64))
    ag.call("ag_checksum64_dev", res.ptr, want.size, got.ptr, None)
    ag.call("ag_stream_sync", None)
    assert int(got.get()[0]) == checksum64(want)


@gpu
def test_output_offsets_past_2_31(ag):
    rng = np.random.default_rng(7)
    bodies = [M.corpora(rng, 150_000)["timestamps"], b"xyz", bytes(70_000)]
    src = P.as_array(b"".join(bodies) + bytes(8))
    base = (1 << 31) - 40
    pages, s, d = [], 0, base
    for b in bodies:
        pages.append((s, len(b), d, M.max_size(len(b))))
        s += len(b)
        d += M.max_size(len(b)) + 1
    ds, dout, dw = Dev(src), Dev(nbytes=d), Dev(np.zeros(len(pages), np.int64))
    ag.call("ag_parquet_snappy_compress_dev", ds.ptr, N.compressed_table(pages), len(pages), dout.ptr, dw.ptr, None)
    ag.call("ag_stream_sync", None)
    w = dw.get()
    for (_, _, dd, _), k, b in zip(pages, w, bodies):
        assert dout.buf.to_numpy(np.uint8, int(k), dd).tobytes() == M.compress(b)


@gpu
def test_pyarrow_chunk_recompressed_on_device(ag, tmp_path):
    """a pyarrow-written SNAPPY chunk decompressed on the device and compressed again there; pyarrow reads every page
    back to its original bytes"""
    rng = np.random.default_rng(8)
    n = 300_000
    path = str(tmp_path / "c.parquet")
    vals = pa.array(rng.integers(0, 3000, n).astype(np.int64), mask=rng.random(n) < 0.1)
    F.write_column(path, vals, nullable=True, encoding="RLE_DICTIONARY", version="1.0", compression="SNAPPY", data_page_size=1 << 16)
    plan = P.chunk_plan(path)
    assert len(plan["comp"]) > 2
    chunk, dec = Dev(P.as_array(plan["chunk"])), Dev(nbytes=plan["n_dst"])
    ag.call("ag_parquet_snappy_decompress_dev", chunk.ptr, N.compressed_table(plan["comp"]), len(plan["comp"]), dec.ptr, None, None)
    pages, d = [], 0
    for _, _, s, sl in plan["comp"]:
        pages.append((s, sl, d, M.max_size(sl)))
        d += M.max_size(sl)
    out, dw = Dev(nbytes=d), Dev(np.zeros(len(pages), np.int64))
    ag.call("ag_parquet_snappy_compress_dev", dec.ptr, N.compressed_table(pages), len(pages), out.ptr, dw.ptr, None)
    ag.call("ag_stream_sync", None)
    host = P.host_decompress(plan)
    for (s, sl, dd, _), k in zip(pages, dw.get()):
        stream = out.buf.to_numpy(np.uint8, int(k), dd).tobytes()
        assert stream == M.compress(host[s:s + sl])
        got = pa.decompress(stream, decompressed_size=sl, codec="snappy", asbytes=True) if sl else b""
        assert got == host[s:s + sl]
