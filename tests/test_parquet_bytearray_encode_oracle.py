"""The BYTE_ARRAY page encoders' oracle: the restatements of PlainByteArrayEncoder, DeltaLengthByteArrayEncoder and
DeltaByteArrayEncoder (pq_bytearray_ref.plain_encode / dlba_encode / dba_encode) against the value sections of the
pages pyarrow writes, byte for byte, and ag_parquet_byte_array_max_size.  CPU only; the last test checks that the
encode entry points fail with AG_ERR_CUDA when no GPU is usable."""
import ctypes as C
import zlib

import numpy as np
import pytest

import pq_bytearray_ref as B
import pq_files as F
import pq_pages as P
from arrow_go_b200 import _native as N

ENCODERS = {"PLAIN": B.plain_encode, "DELTA_LENGTH_BYTE_ARRAY": B.dlba_encode, "DELTA_BYTE_ARRAY": B.dba_encode}
ENC_IDS = {"PLAIN": B.PLAIN, "DELTA_LENGTH_BYTE_ARRAY": B.DELTA_LENGTH_BYTE_ARRAY, "DELTA_BYTE_ARRAY": B.DELTA_BYTE_ARRAY}


def shared_prefix_keys(rng, n):
    """sorted keys behind a 300-byte common prefix, runs of equal keys, and empty values"""
    head = b"tenant/" + bytes(rng.integers(97, 123, 293, dtype=np.uint8))
    keys = [head + f"{k:08d}".encode() * int(rng.integers(1, 4)) for k in np.sort(rng.integers(0, 10 ** 6, n))]
    for i in rng.integers(0, n, n // 50):
        keys[i] = keys[i - 1] if i else b""
    keys[0] = b""
    return keys


def column(rng, corpus, n):
    if corpus == "short":
        return F.random_strings(rng, n)
    if corpus == "sorted":
        return F.random_strings(rng, n, sorted_keys=True)
    return shared_prefix_keys(rng, n)


def check_file(tmp_path, vals, valid, encoding, version, typ, page_size=1 << 12):
    pa = pytest.importorskip("pyarrow")
    arr = pa.array(vals, type=typ, mask=None if valid is None else ~valid)
    path = str(tmp_path / "s.parquet")
    F.write_column(path, arr, nullable=valid is not None, encoding=encoding, version=version, data_page_size=page_size)
    plan = P.chunk_plan(path)
    dst = P.host_decompress(plan)
    sections = P.value_sections(plan, dst)
    ok = np.ones(len(vals), bool) if valid is None else valid
    for enc, (vd, vl, nv, slot) in sections:
        assert enc == ENC_IDS[encoding]
        page = [bytes(v) if isinstance(v, bytes) else v.encode() for v, k in zip(vals[slot:slot + nv], ok[slot:slot + nv]) if k]
        assert dst[vd:vd + vl] == ENCODERS[encoding](page), (slot, nv)
    return len(sections)


@pytest.mark.parametrize("encoding", list(ENCODERS))
@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("null_frac", [None, 0.1])
@pytest.mark.parametrize("corpus", ["short", "sorted", "prefix"])
def test_pages_match_pyarrow(tmp_path, encoding, version, null_frac, corpus):
    pa = pytest.importorskip("pyarrow")
    rng = np.random.default_rng(zlib.crc32(f"{encoding}{version}{corpus}".encode()))
    n = 20_000
    vals = column(rng, corpus, n)
    valid = None if null_frac is None else rng.random(n) >= null_frac
    pages = check_file(tmp_path, vals, valid, encoding, version, pa.binary())
    assert pages >= 3


@pytest.mark.parametrize("encoding", list(ENCODERS))
def test_string_column_and_all_null_pages(tmp_path, encoding):
    pa = pytest.importorskip("pyarrow")
    rng = np.random.default_rng(5)
    vals = [v.decode() for v in F.random_strings(rng, 8000)]
    assert check_file(tmp_path, vals, rng.random(8000) >= 0.3, encoding, "2.0", pa.string()) >= 2
    check_file(tmp_path, vals, np.zeros(8000, bool), encoding, "1.0", pa.string())


def max_size(enc, n, span):
    s = C.c_int64()
    st, msg = N.call_status("ag_parquet_byte_array_max_size", enc, n, span, C.byref(s))
    return st, s.value


def delta_bound(n):
    return 40 + ((n - 2) // 128 + 1) * (10 + 4 + 128 * 4) if n > 1 else 40


@pytest.mark.parametrize("n", [0, 1, 2, 129, 130, 1 << 20, (1 << 31) - 1])
def test_max_size(n):
    for span in (0, 7, 1 << 40):
        assert max_size(B.PLAIN, n, span) == (N.AG_OK, 4 * n + span)
        assert max_size(B.DELTA_LENGTH_BYTE_ARRAY, n, span) == (N.AG_OK, delta_bound(n) + span)
        assert max_size(B.DELTA_BYTE_ARRAY, n, span) == (N.AG_OK, 2 * delta_bound(n) + span)


def test_max_size_refuses():
    assert max_size(B.PLAIN, -1, 0)[0] == N.AG_ERR_INVALID
    assert max_size(B.PLAIN, 1 << 31, 0)[0] == N.AG_ERR_INVALID
    assert max_size(B.PLAIN, 1, -1)[0] == N.AG_ERR_INVALID
    assert max_size(B.RLE_DICTIONARY, 1, 0)[0] == N.AG_ERR_INVALID
    assert N.call_status("ag_parquet_byte_array_max_size", B.PLAIN, 1, 0, None)[0] == N.AG_ERR_INVALID


def test_encoders_need_a_gpu():
    if N.call_status("ag_init", 0)[0] == N.AG_OK:
        pytest.skip("a GPU is usable here")
    offsets = np.arange(17, dtype=np.int32)
    data = np.zeros(16, np.uint8)
    out = np.zeros(4096, np.uint8)
    tbl = N.enc_page_table([(0, 16, 0, 4096)])
    for enc in (B.PLAIN, B.DELTA_LENGTH_BYTE_ARRAY, B.DELTA_BYTE_ARRAY):
        args = (enc, 4, offsets.ctypes.data, data.ctypes.data, None, tbl, 1, out.ctypes.data, None)
        assert N.call_status("ag_parquet_byte_array_encode", *args, None)[0] == N.AG_ERR_CUDA
        assert N.call_status("ag_parquet_byte_array_encode_dev", *args, None, None)[0] == N.AG_ERR_CUDA
