"""The BYTE_ARRAY dictionary encoder's oracle: the restatement of DictByteArrayEncoder and the writer's fallback rule
(pq_dict_ref) rebuilds pyarrow's dictionary-encoded string column chunks byte for byte: the dictionary page and every
RLE_DICTIONARY data page with its bit width, v1 and v2 pages, required and nullable columns, chunked columns, and
chunks written with a small dictionary page limit (the cut, the prefix dictionary page, the PLAIN pages after it).
CPU only; the last tests check that the host argument errors come back before the device is touched and that the
calls return AG_ERR_CUDA without a GPU."""
import zlib

import numpy as np
import pytest

import pq_bytearray_ref as B
import pq_dict_ref as D
import pq_files as F
import pq_pages as P
from arrow_go_b200 import _native as N


def write(tmp_path, chunks, valids, version, limit=None, page_size=4096):
    """chunks of binary values (valids: per chunk None or a bool mask) -> (plan, dst, values, validity, chunk lengths)"""
    pa = pytest.importorskip("pyarrow")
    arrs = [pa.array(c, type=pa.binary(), mask=None if v is None else ~v) for c, v in zip(chunks, valids)]
    col = pa.chunked_array(arrs, type=pa.binary())
    path = str(tmp_path / "d.parquet")
    F.write_column(path, col, nullable=any(v is not None for v in valids), encoding="RLE_DICTIONARY", version=version,
                   data_page_size=page_size, dictionary_pagesize_limit=limit)
    plan = P.chunk_plan(path)
    vals = [bytes(x) for c in chunks for x in c]
    valid = np.concatenate([np.ones(len(c), bool) if v is None else v for c, v in zip(chunks, valids)])
    return plan, P.host_decompress(plan), vals, valid, [len(c) for c in chunks]


def rebuild(plan, dst, vals, valid, lengths, limit=None):
    """checks every page of the chunk against the restatement; returns (the cut or None, dictionary pages)"""
    entries, indices, first = D.dictionary(vals, valid)
    cut = D.fallback_cut(vals, first, lengths, limit) if limit else None
    n_dict = len(entries) if cut is None else D.mark_counts(vals, first, [cut])[0][0]
    d, dl, nv = plan["dict"]
    assert nv == n_dict
    assert dst[d:d + dl] == D.dictionary_page(entries[:n_dict])
    dense = np.concatenate([[0], np.cumsum(valid)])
    dict_pages = 0
    for enc, (vd, vl, nv, slot) in P.value_sections(plan, dst):
        if enc == B.RLE_DICTIONARY:
            assert cut is None or slot + nv <= cut
            ents = D.mark_counts(vals, first, [slot + nv])[0][0]
            want = D.index_section(indices[dense[slot]:dense[slot + nv]], ents)
            dict_pages += 1
        else:
            assert enc == B.PLAIN and cut is not None and slot >= cut, (enc, slot, cut)
            want = B.plain_encode([vals[s] for s in range(slot, slot + nv) if valid[s]])
        assert dst[vd:vd + vl] == want, (enc, slot, nv)
    return cut, dict_pages


def strings(rng, n, distinct, null_frac):
    """n values drawn from `distinct` random short strings (the same pool for a given rng state and `distinct`)"""
    pool = F.random_strings(np.random.default_rng(distinct), distinct)
    vals = [pool[i] for i in rng.integers(0, distinct, n)]
    return vals, None if null_frac is None else rng.random(n) >= null_frac


@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("null_frac", [None, 0.1])
@pytest.mark.parametrize("distinct", [1, 300, 5000])
def test_chunk_matches_pyarrow(tmp_path, version, null_frac, distinct):
    rng = np.random.default_rng(zlib.crc32(f"{version}{null_frac}{distinct}".encode()))
    vals, valid = strings(rng, 30_000, distinct, null_frac)
    plan, dst, v, ok, lens = write(tmp_path, [vals], [valid], version)
    cut, pages = rebuild(plan, dst, v, ok, lens)
    assert cut is None and pages >= 2


@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("null_frac", [None, 0.1])
def test_chunked_column(tmp_path, version, null_frac):
    rng = np.random.default_rng(11 if null_frac is None else 12)
    sizes = [700, 0, 1500, 3, 5000, 1024]
    chunks, valids = zip(*[strings(rng, n, 400, null_frac) for n in sizes])
    plan, dst, v, ok, lens = write(tmp_path, chunks, valids, version)
    rebuild(plan, dst, v, ok, lens)


@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("limit", [1000, 4000, 20_000])
@pytest.mark.parametrize("chunked", [False, True])
def test_fallback_after_dictionary_limit(tmp_path, version, limit, chunked):
    rng = np.random.default_rng(limit + chunked)
    sizes = [700, 2100, 6000] if chunked else [8800]
    chunks, valids = zip(*[strings(rng, n, 3000, 0.1) for n in sizes])
    plan, dst, v, ok, lens = write(tmp_path, chunks, valids, version, limit=limit)
    cut, _ = rebuild(plan, dst, v, ok, lens, limit)
    assert cut is not None
    if chunked and limit == 1000:
        assert cut == 700               # the first chunk's only batch ends the check
    assert any(enc == B.PLAIN for enc, _ in P.value_sections(plan, dst))


def test_bit_width_follows_the_entries_not_the_page():
    """a page holding only index 0 after 1024 distinct values is written at bit width 10"""
    assert D.bit_width(0) == 0 and D.bit_width(1) == 1 and D.bit_width(2) == 1 and D.bit_width(1024) == 10
    assert D.index_section(np.zeros(5, np.uint32), 1024)[0] == 10


def test_pyarrow_bit_width_after_many_entries(tmp_path):
    vals = [f"v{i:05d}".encode() for i in range(1024)] + [b"v00000"] * 3000
    plan, dst, v, ok, lens = write(tmp_path, [vals], [None], "2.0", page_size=1024)
    rebuild(plan, dst, v, ok, lens)
    last = P.value_sections(plan, dst)[-1][1]
    assert dst[last[0]] == 10


# ---------------------------------------------------------------- the entry points without a device ----
def call(dev, ow, chunks, marks, indices=True, counts=True, mark_counts=True):
    tbl = N.ba_chunk_table(chunks)
    mk = np.array(marks, np.int64)
    idx = np.zeros(64, np.uint32)
    mc = np.zeros(2 * max(len(marks), 1), np.int64)
    cnt = np.zeros(3, np.int64)
    args = (ow, tbl, len(chunks), mk.ctypes.data if len(marks) else None, len(marks), idx.ctypes.data if indices else None,
            mc.ctypes.data if mark_counts else None, cnt.ctypes.data if counts else None, None)
    return N.call_status("ag_parquet_byte_array_dict_encode_dev" if dev else "ag_parquet_byte_array_dict_encode",
                         *args, *((None,) if dev else ()))


OFFS = np.arange(33, dtype=np.int32)
DATA = np.zeros(64, np.uint8)
FIRST = np.zeros(8, np.uint32)


def chunk(offset=0, length=32, offsets=OFFS, data=DATA, first=FIRST):
    return (offsets.ctypes.data if offsets is not None else None, data.ctypes.data if data is not None else None, None,
            offset, length, first if first is None or isinstance(first, int) else first.ctypes.data)


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_host_errors_before_the_device(dev):
    bad = [
        call(dev, 2, [chunk()], []),
        call(dev, 4, [chunk(offset=-1)], []),
        call(dev, 4, [chunk(length=-1)], []),
        call(dev, 4, [chunk(offsets=None)], []),
        call(dev, 4, [chunk(data=None)], []),
        call(dev, 4, [chunk(first=None)], []),
        call(dev, 4, [chunk(first=FIRST.ctypes.data + 2)], []),
        call(dev, 4, [chunk()], [33]),
        call(dev, 4, [chunk()], [-1]),
        call(dev, 4, [chunk()], [0], mark_counts=False),
        call(dev, 4, [chunk()], [], indices=False),
        call(dev, 4, [chunk()], [], counts=False),
    ]
    for k, (st, msg) in enumerate(bad):
        assert st == N.AG_ERR_INVALID, (k, st, msg)
    big = [chunk(length=(1 << 30))] * 2
    assert call(dev, 4, big, [])[0] == N.AG_ERR_NOT_IMPLEMENTED
    # empty chunks need no pointers
    st, _ = call(dev, 4, [chunk(length=0, offsets=None, data=None, first=None)], [0], indices=False)
    assert st in (N.AG_OK, N.AG_ERR_CUDA)


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_calls_need_a_gpu(dev):
    if N.call_status("ag_init", 0)[0] == N.AG_OK:
        pytest.skip("a GPU is usable here")
    assert call(dev, 4, [chunk(), chunk(offset=3, length=20)], [0, 5, 52])[0] == N.AG_ERR_CUDA
    assert call(dev, 8, [], [])[0] == N.AG_ERR_CUDA
