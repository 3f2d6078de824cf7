"""The device SNAPPY compressor's parse (snappy_encode_model.py) on the CPU: its streams decode back to the input with
pyarrow's C++ Snappy and with snappy_ref.decode, and stay within 5 % of pyarrow's size, over the measured corpora, the
fragment edges, random bytes and page bodies of pyarrow-written files.  Also ag_parquet_snappy_max_size, and the
compress entry points failing with AG_ERR_CUDA when no GPU is usable."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

import pq_files as F
import pq_pages as P
import snappy_encode_model as M
import snappy_ref as S


def _round_trip(x, ratio=True):
    c = M.compress(x)
    assert len(c) <= M.max_size(len(x))
    got, err, pre = S.decode(c, len(x))
    assert err == S.OK and pre == len(x) and got == x
    if x:
        assert pa.decompress(c, decompressed_size=len(x), codec="snappy", asbytes=True) == x
    if ratio and len(x) >= 4096:
        assert len(c) <= 1.05 * len(pa.compress(x, codec="snappy", asbytes=True))
    return c


@pytest.mark.parametrize("name", list(M.corpora(np.random.default_rng(0), 64)))
def test_corpora(name):
    _round_trip(M.corpora(np.random.default_rng(20261018), 1 << 20)[name])


def test_short_pages():
    assert M.compress(b"") == b"\x00"
    for n in range(1, 4):
        assert M.compress(b"abc"[:n]) == S.put_uvarint(n) + S.literal(b"abc"[:n])
    for n in range(6):
        _round_trip(b"aaaaa"[:n])
        _round_trip(bytes(range(n)))


@pytest.mark.parametrize("n", [65535, 65536, 65537, 3 * 65536 + 5])
def test_fragment_edges(n):
    rng = np.random.default_rng(n)
    for x in M.corpora(rng, n).values():
        _round_trip(x[:n])
    _round_trip((rng.integers(0, 4, n, dtype=np.uint8) * 17).tobytes(), ratio=False)
    _round_trip(rng.integers(0, 256, n, dtype=np.uint8).tobytes())


def test_fragments_are_independent():
    """a repeat of the first fragment in the second is not a copy across the boundary"""
    rng = np.random.default_rng(3)
    a = rng.integers(0, 256, 1 << 16, dtype=np.uint8).tobytes()
    c = M.compress(a + a)
    assert len(c) > 2 << 16
    assert c == S.put_uvarint(2 << 16) + 2 * M.compress(a)[3:]


def test_element_forms():
    """a 1-byte-offset copy, a 2-byte-offset copy, and 64 + 60 + tail pieces of a long copy"""
    x = b"0123456789abcdef" + b"0123456789"
    assert M.compress(x) == S.put_uvarint(len(x)) + S.literal(x[:16]) + S.copy(16, 10, 1)
    c = M.compress(b"z" * 196)                                   # a copy of 195: 64, 64, then 67 = 60 + 7
    assert c == S.put_uvarint(196) + S.literal(b"z") + S.copy(1, 64, 2) + S.copy(1, 64, 2) + S.copy(1, 60, 2) + S.copy(1, 7, 1)
    rng = np.random.default_rng(5)
    far = rng.integers(0, 256, 3000, dtype=np.uint8).tobytes()
    c = M.compress(far + far[:8])                                # offset 3000 >= 2048: the 2-byte-offset form
    assert c[-3] & 3 == 2 and int.from_bytes(c[-2:], "little") == 3000


def test_incompressible():
    rng = np.random.default_rng(9)
    for n in (100, 5000, 300_000):
        x = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        c = _round_trip(x)
        frags = -(-n // M.FRAGMENT)
        assert len(c) <= len(S.put_uvarint(n)) + n + 3 * frags


@pytest.mark.parametrize("encoding", ["PLAIN", "RLE_DICTIONARY", "DELTA_BINARY_PACKED"])
def test_pyarrow_page_bodies(tmp_path, encoding):
    rng = np.random.default_rng(len(encoding))
    n = 300_000
    vals = (np.cumsum(rng.integers(0, 1000, n)) + (1 << 40)).astype(np.int64)
    if encoding == "RLE_DICTIONARY":
        vals = rng.integers(0, 3000, n).astype(np.int64)
    path = str(tmp_path / "p.parquet")
    F.write_column(path, pa.array(vals, mask=rng.random(n) < 0.05), nullable=True, encoding=encoding, version="1.0",
                   compression="SNAPPY", data_page_size=1 << 18)
    plan = P.chunk_plan(path)
    dst = P.host_decompress(plan)
    assert len(plan["comp"]) > 1
    for _, _, d, dl in plan["comp"]:
        _round_trip(dst[d:d + dl])


# ------------------------------------------------------------------------------------------- the entry points ----
def test_max_size():
    from arrow_go_b200 import _native as N
    size = C.c_int64()
    for n in (0, 1, 5, 6, 65536, 1 << 31, (1 << 32) - 1):
        N.call("ag_parquet_snappy_max_size", n, C.byref(size))
        assert size.value == 32 + n + n // 6 == M.max_size(n)
    for n in (-1, 1 << 32):
        st, msg = N.call_status("ag_parquet_snappy_max_size", n, C.byref(size))
        assert st == N.AG_ERR_INVALID and "snappy_max_size" in msg


def test_compress_needs_a_gpu():
    from arrow_go_b200 import _native as N
    if N.call_status("ag_init", 0)[0] == N.AG_OK:
        pytest.skip("a GPU is usable here")
    src = np.zeros(16, np.uint8)
    out = np.zeros(64, np.uint8)
    tbl = N.compressed_table([(0, 16, 0, 64)])
    for name, tail in (("ag_parquet_snappy_compress", ()), ("ag_parquet_snappy_compress_dev", (None,))):
        assert N.call_status(name, src.ctypes.data, tbl, 1, out.ctypes.data, None, *tail)[0] == N.AG_ERR_CUDA, name
