"""Device BYTE_ARRAY dictionaries (ag_parquet_byte_array_dict_encode[_dev]), both flavours and both offset widths,
against the restatement of DictByteArrayEncoder (pq_dict_ref): indices, every chunk's first-appearance bitmap, the
counts and the per-mark counts, with guard bytes around every output.  Cases: all-distinct, one value, all-null and
empty chunks, empty strings, values that differ only in their last byte around the 16-byte pieces and the warp
threshold, values past 64 KiB, chunk offsets off the 8- and 32-slot grid, the full-size table forced through
ag_unique_set_policy, and the prefix property.  End to end, pyarrow's dictionary page and index pages are rebuilt on
the device (dict encode, PLAIN with `first`, RLE with the bit width of each page's mark), with and without fallback.
Every device error leaves the outputs untouched; one LargeBinary batch passes 2^31 data bytes."""
import ctypes as C

import numpy as np
import pytest

import pq_bytearray_ref as B
import pq_dict_ref as D
import pq_files as F
import pq_pages as P
from arrow_go_b200 import _native as N
from helpers import Dev

pytestmark = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
WIDTHS = pytest.mark.parametrize("ow", [4, 8])
GUARD = 0xA5A5A5A5


def arrow(vals, ow):
    lens = np.array([len(v) for v in vals], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32 if ow == 4 else np.int64)
    data = np.frombuffer(b"".join(bytes(v) for v in vals) + b"\0", np.uint8).copy()
    return offsets, data


def encode(ag, ow, chunks, marks, dev):
    """chunks [(vals, valid or None, offset)] (the chunk's slots are vals[offset:]) -> (status, message, indices,
    [first words], counts, mark_counts, bad_pos, all guards intact, valid slots)"""
    arrays, tbl_rows, firsts = [], [], []
    n_valid = 0
    for vals, valid, off in chunks:
        offsets, data = arrow(vals, ow)
        vb = None if valid is None else np.packbits(valid, bitorder="little")
        nw = (len(vals) + 31) // 32
        first = np.full(nw + 2, GUARD, np.uint32)            # one guard word after the chunk's words
        firsts.append(first)
        n_valid += int(np.sum(valid[off:])) if valid is not None else len(vals) - off
        arrays.append((offsets, data, vb, first))
    n_slots = sum(len(v) - o for v, _, o in chunks)
    idx = np.full(n_valid + 8, GUARD, np.uint32)
    mc = np.full(2 * len(marks) + 2, -7, np.int64)
    cnt = np.full(4, -7, np.int64)
    bp = np.full(1, -5, np.int64)
    mk = np.array(marks, np.int64)
    if not dev:
        for (vals, _, off), (offsets, data, vb, first) in zip(chunks, arrays):
            tbl_rows.append((offsets.ctypes.data, data.ctypes.data, None if vb is None else vb.ctypes.data, off,
                             len(vals) - off, first.ctypes.data))
        st, msg = ag.call_status("ag_parquet_byte_array_dict_encode", ow, N.ba_chunk_table(tbl_rows), len(chunks),
                                 mk.ctypes.data if len(marks) else None, len(marks), idx.ctypes.data, mc.ctypes.data,
                                 cnt.ctypes.data, bp.ctypes.data)
        out_first = firsts
    else:
        keep = []
        for (vals, _, off), (offsets, data, vb, first) in zip(chunks, arrays):
            d = (Dev(offsets), Dev(data), None if vb is None else Dev(vb), Dev(first))
            keep.append(d)
            tbl_rows.append((d[0].ptr, d[1].ptr, None if d[2] is None else d[2].ptr, off, len(vals) - off, d[3].ptr))
        di, dm, dc, db = Dev(idx), Dev(mc), Dev(cnt), Dev(bp)
        st, msg = ag.call_status("ag_parquet_byte_array_dict_encode_dev", ow, N.ba_chunk_table(tbl_rows), len(chunks),
                                 mk.ctypes.data if len(marks) else None, len(marks), di.ptr, dm.ptr, dc.ptr, db.ptr, None)
        ag.call("ag_stream_sync", None)
        idx, mc, cnt, bp = di.get(), dm.get(), dc.get(), db.get()
        out_first = [d[3].get() for d in keep]
    return st, msg, idx, out_first, cnt, mc, int(bp[0]), n_valid, n_slots


def check(ag, ow, chunks, dev, marks=None):
    """the call against the restatement over the slots of all chunks; returns (entries, indices)"""
    vals = [bytes(v) for vs, _, o in chunks for v in vs[o:]]
    valid = np.concatenate([np.ones(len(vs) - o, bool) if ok is None else ok[o:] for vs, ok, o in chunks]) if chunks else np.zeros(0, bool)
    entries, indices, first = D.dictionary(vals, valid)
    n = len(vals)
    if marks is None:
        marks = sorted({m for m in (0, n, n // 3, n // 2 + 1, n - 1) if 0 <= m <= n})
    st, msg, idx, firsts, cnt, mc, bad, n_valid, n_slots = encode(ag, ow, chunks, marks, dev)
    assert st == N.AG_OK, msg
    assert bad == N.NO_ERROR_POS
    assert n_valid == len(indices) and n_slots == n
    assert np.array_equal(idx[:n_valid], indices)
    assert (idx[n_valid:] == GUARD).all()
    assert list(cnt[:3]) == [len(entries), sum(len(e) for e in entries), n_valid] and cnt[3] == -7
    assert [tuple(mc[2 * j:2 * j + 2]) for j in range(len(marks))] == D.mark_counts(vals, first, marks)
    assert (mc[2 * len(marks):] == -7).all()
    g = 0
    for (vs, _, off), words in zip(chunks, firsts):
        ln = len(vs) - off
        w0, w1 = off // 32, (off + ln + 31) // 32
        if ln == 0:
            w0 = w1
        assert (words[:w0] == GUARD).all() and (words[w1:] == GUARD).all()
        bits = np.unpackbits(words[w0:w1].view(np.uint8), bitorder="little")
        want = np.zeros(32 * (w1 - w0), np.uint8)
        want[off - 32 * w0:off - 32 * w0 + ln] = first[g:g + ln]
        assert np.array_equal(bits, want)
        g += ln
    return entries, indices


def near_equal(rng):
    """pairs of values that differ only in their last byte, around the 16-byte pieces and the warp threshold"""
    out = []
    for n in (1, 15, 16, 17, 31, 32, 33, 255, 256, 257, 511, 512, 513):
        base = bytes(rng.integers(97, 123, n, dtype=np.uint8))
        out += [base, base[:-1] + b"#", base, base[:-1] + b"#" * (n > 1) + b"!" * (n == 1)]
    return out


def case(name, rng):
    """-> chunks [(vals, valid, offset)]"""
    if name == "distinct":
        vals = [f"k{i:07d}".encode() for i in rng.permutation(20000)]
        return [(vals, None, 0)]
    if name == "one":
        return [([b"same value"] * 5000, rng.random(5000) > 0.3, 0)]
    if name == "all_null":
        vals = F.random_strings(rng, 3000)
        return [(vals, np.zeros(3000, bool), 0), (vals[:10], None, 3)]
    if name == "empty_strings":
        vals = [b"" if i % 3 else b"x" for i in range(4000)]
        return [(vals, rng.random(4000) > 0.1, 0)]
    if name == "near_equal":
        vals = near_equal(rng) * 40
        rng.shuffle(vals)
        return [(vals, None, 0), (vals[::-1], rng.random(len(vals)) > 0.2, 5)]
    if name == "long":
        pool = [bytes(rng.integers(0, 256, n, dtype=np.uint8)) for n in (70_000, 65_537, 300, 100_000)]
        pool.append(pool[0][:-1] + bytes([pool[0][-1] ^ 1]))
        vals = [pool[i] for i in rng.integers(0, len(pool), 300)]
        return [(vals, None, 0)]
    if name == "chunks":                                   # offsets off the 8- and 32-slot grid, empty chunks
        pool = F.random_strings(rng, 700)
        out = []
        for n, off in ((1000, 0), (0, 0), (2500, 5), (37, 33), (0, 13), (4100, 70), (1, 31)):
            vals = [pool[i] for i in rng.integers(0, len(pool), n + off)]
            out.append((vals, rng.random(n + off) > 0.15, off))
        return out
    raise ValueError(name)


CASES = ["distinct", "one", "all_null", "empty_strings", "near_equal", "long", "chunks"]


@pytest.mark.parametrize("name", CASES)
@WIDTHS
@FLAVOURS
def test_against_restatement(ag, name, ow, dev):
    rng = np.random.default_rng(CASES.index(name) * 4 + ow + dev)
    check(ag, ow, case(name, rng), dev)


@FLAVOURS
def test_empty_call(ag, dev):
    check(ag, 4, [], dev, marks=[0, 0])
    check(ag, 8, [([b"a"], None, 1)], dev, marks=[0])


@WIDTHS
@FLAVOURS
def test_full_size_table(ag, ow, dev):
    """the small table overflows (more than small_slots/2 distinct values) and the full-size table takes over"""
    rng = np.random.default_rng(3 + ow)
    ag.call("ag_unique_set_policy", 1024, 1024)
    try:
        pool = [f"value-{i}".encode() * int(rng.integers(1, 4)) for i in range(3000)]
        vals = [pool[i] for i in rng.integers(0, 3000, 20000)]
        check(ag, ow, [(vals[:7000], rng.random(7000) > 0.1, 0), (vals[7000:], None, 0)], dev)
        check(ag, ow, [(vals[:400] * 10, None, 0)], dev)       # above small_rows, below the cap: the small table holds
    finally:
        ag.call("ag_unique_set_policy", 0, 0)


@WIDTHS
def test_prefix_property(ag, ow):
    rng = np.random.default_rng(ow)
    vals = F.random_strings(rng, 9000, distinct=2000)
    valid = rng.random(9000) > 0.1
    ent_all, idx_all = check(ag, ow, [(vals, valid, 0)], True)
    for c in (0, 1, 1023, 1024, 5000):
        ent, idx = check(ag, ow, [(vals[:c], valid[:c], 0)], True)
        assert ent == ent_all[:len(ent)]
        assert np.array_equal(idx, idx_all[:len(idx)])


# ---------------------------------------------------------------- device errors ----
@WIDTHS
@FLAVOURS
def test_device_errors_write_nothing(ag, ow, dev):
    vals = [b"abc", b"de", b"", b"fgh"] * 50
    offsets, data = arrow(vals, ow)
    cases = []
    o = offsets.copy()
    o[0] = -1                                              # negative first offset of the second chunk (slot 0)
    cases.append((o, 0, "negative offset"))
    o = offsets.copy()
    o[77] = o[76] - 1                                      # offsets decrease after slot 76 of the chunk
    cases.append((o, 76, "decrease"))
    if ow == 8:
        o = offsets.copy()
        o[101:] += 1 << 31                                 # slot 100 longer than 2^31-1 bytes
        cases.append((o, 100, "longer"))
    good_o, good_d = arrow([b"x"] * 40, ow)
    for o, slot, what in cases:
        rows, keep = [], []
        first0, first1 = np.full(4, GUARD, np.uint32), np.full(10, GUARD, np.uint32)
        arrs = [(good_o, good_d, first0, 40), (o, data, first1, len(vals))]
        for a_o, a_d, fw, n in arrs:
            if dev:
                d = (Dev(a_o), Dev(a_d), Dev(fw))
                keep.append(d)
                rows.append((d[0].ptr, d[1].ptr, None, 0, n, d[2].ptr))
            else:
                rows.append((a_o.ctypes.data, a_d.ctypes.data, None, 0, n, fw.ctypes.data))
        idx = np.full(300, GUARD, np.uint32)
        mc = np.full(4, -7, np.int64)
        cnt = np.full(3, -7, np.int64)
        bp = np.full(1, -5, np.int64)
        mk = np.array([0, 10], np.int64)
        if dev:
            di, dm, dc, db = Dev(idx), Dev(mc), Dev(cnt), Dev(bp)
            st, msg = ag.call_status("ag_parquet_byte_array_dict_encode_dev", ow, N.ba_chunk_table(rows), 2, mk.ctypes.data, 2,
                                     di.ptr, dm.ptr, dc.ptr, db.ptr, None)
            ag.call("ag_stream_sync", None)
            idx, mc, cnt, bp = di.get(), dm.get(), dc.get(), db.get()
            firsts = [k[2].get() for k in keep]
        else:
            st, msg = ag.call_status("ag_parquet_byte_array_dict_encode", ow, N.ba_chunk_table(rows), 2, mk.ctypes.data, 2,
                                     idx.ctypes.data, mc.ctypes.data, cnt.ctypes.data, bp.ctypes.data)
            firsts = [first0, first1]
        assert st == N.AG_ERR_INVALID, (what, msg)
        assert "chunk 1" in msg, msg
        assert int(bp[0]) == 40 + slot, what                # the global slot
        assert (idx == GUARD).all() and (mc == -7).all() and (cnt == -7).all()
        assert all((f == GUARD).all() for f in firsts)


# ---------------------------------------------------------------- end to end with pyarrow ----
def device_chunk(path):
    """pyarrow's own column buffers (int32 offsets, with the arrays' slice offsets) -> dictionary call on the device"""
    import pyarrow.parquet as pq
    col = pq.read_table(path).column(0)
    rows, keep = [], []
    for a in col.chunks:
        vb, ob, db = a.buffers()
        off = np.frombuffer(ob, np.int32)
        d = (Dev(off), Dev(np.frombuffer(db, np.uint8) if db is not None and db.size else np.zeros(1, np.uint8)),
             None if vb is None else Dev(np.frombuffer(vb, np.uint8)), Dev(nbytes=((a.offset + len(a) + 31) // 32) * 4 + 4))
        keep.append((d, a.offset, len(a)))
        rows.append((d[0].ptr, d[1].ptr, None if d[2] is None else d[2].ptr, a.offset, len(a), d[3].ptr))
    return rows, keep


def rebuild_on_device(ag, tmp_path, chunks, version, limit):
    pa = pytest.importorskip("pyarrow")
    arrs = [pa.array(c, type=pa.binary(), mask=~v) for c, v in chunks]
    path = str(tmp_path / "e.parquet")
    F.write_column(path, pa.chunked_array(arrs, type=pa.binary()), nullable=True, encoding="RLE_DICTIONARY", version=version,
                   data_page_size=4096, dictionary_pagesize_limit=limit)
    plan = P.chunk_plan(path)
    dst = P.host_decompress(plan)
    sections = P.value_sections(plan, dst)
    rows, keep = device_chunk(path)
    page_ends = [slot + nv for enc, (_, _, nv, slot) in sections if enc == B.RLE_DICTIONARY]
    batch_ends = D.batch_ends([len(c) for c, _ in chunks])
    marks = np.array(page_ends + batch_ends, np.int64)
    valid = np.concatenate([v for _, v in chunks])
    nv_all = int(valid.sum())
    di, dm, dc = Dev(nbytes=4 * nv_all + 4), Dev(nbytes=16 * len(marks)), Dev(nbytes=24)
    ag.call("ag_parquet_byte_array_dict_encode_dev", 4, N.ba_chunk_table(rows), len(rows), marks.ctypes.data, len(marks),
            di.ptr, dm.ptr, dc.ptr, None, None)
    ag.call("ag_stream_sync", None)
    mc = dm.get(np.int64, 2 * len(marks)).reshape(-1, 2)
    # the cut: the first batch end whose dictionary size reaches the limit
    cut = next((int(e) for e, (_, size) in zip(batch_ends, mc[len(page_ends):]) if size >= limit), None)
    n_dict = int(dc.get(np.int64, 3)[0]) if cut is None else int(mc[len(page_ends) + batch_ends.index(cut)][0])
    # the dictionary page: PLAIN over each chunk's slots below the cut with `first` as validity
    d, dl, pnv = plan["dict"]
    assert pnv == n_dict
    page, g = b"", 0
    for (dv, a_off, ln), row in zip(keep, rows):
        take = ln if cut is None else max(0, min(ln, cut - g))
        g += ln
        if take == 0:
            continue
        cap = 4 * take + dv[1].count
        out, ln_out = Dev(nbytes=cap), Dev(nbytes=8)
        ag.call("ag_parquet_byte_array_encode_dev", N.PQ_ENC_PLAIN, 4, dv[0].ptr, dv[1].ptr, dv[3].ptr,
                N.enc_page_table([(a_off, take, 0, cap)]), 1, out.ptr, ln_out.ptr, None, None)
        ag.call("ag_stream_sync", None)
        page += out.get(np.uint8, int(ln_out.get(np.int64, 1)[0])).tobytes()
    assert page == dst[d:d + dl]
    # the index pages: one RLE call per distinct bit width, each page at the width of the entries at its end
    dense = np.concatenate([[0], np.cumsum(valid)])
    by_width = {}
    for k, (enc, (vd, vl, pnv, slot)) in enumerate([s for s in sections if s[0] == B.RLE_DICTIONARY]):
        bw = D.bit_width(int(mc[k][0]))
        by_width.setdefault(bw, []).append((int(dense[slot]), int(dense[slot + pnv] - dense[slot]), vd, vl))
    for bw, pages in by_width.items():
        caps = []
        for _, cnt_v, _, _ in pages:
            s = C.c_int64()
            ag.call("ag_parquet_rle_max_size", bw, N.PQ_RLE_WIDTH, cnt_v, C.byref(s))
            caps.append(s.value)
        outs = np.concatenate([[0], np.cumsum(caps)])
        tbl = N.enc_page_table([(i0, cnt_v, int(outs[k]), caps[k]) for k, (i0, cnt_v, _, _) in enumerate(pages)])
        out, lens = Dev(nbytes=int(outs[-1]) + 8), Dev(nbytes=8 * len(pages))
        ag.call("ag_parquet_rle_encode_dev", bw, N.PQ_RLE_WIDTH, N.PQ_RLE_IN_U32, di.ptr, tbl, len(pages), out.ptr, lens.ptr, None, None)
        ag.call("ag_stream_sync", None)
        o, ls = out.get(np.uint8, int(outs[-1])), lens.get(np.int64, len(pages))
        for k, (_, _, vd, vl) in enumerate(pages):
            assert o[outs[k]:outs[k] + ls[k]].tobytes() == dst[vd:vd + vl], (bw, k)
    return cut


@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("limit", [1 << 20, 3000])
@pytest.mark.parametrize("chunked", [False, True])
def test_pyarrow_chunk_rebuilt_on_device(ag, tmp_path, version, limit, chunked):
    rng = np.random.default_rng(limit + chunked)
    pool = F.random_strings(np.random.default_rng(9), 2500)
    sizes = [700, 3000, 9000] if chunked else [12000]
    chunks = [([pool[i] for i in rng.integers(0, len(pool), n)], rng.random(n) > 0.1) for n in sizes]
    cut = rebuild_on_device(ag, tmp_path, chunks, version, limit)
    assert (cut is None) == (limit == 1 << 20)


# ---------------------------------------------------------------- past 2^31 data bytes ----
def test_large_binary_past_2_31(ag):
    """2049 values of 2^20 + 1 bytes (int64 offsets, 2^31 + 2049 data bytes): value i holds bytes (i * L + k) % 251, so
    values i and j are equal iff i = j mod 251"""
    import torch
    L, n = (1 << 20) + 1, 2049
    total = L * n
    assert total > (1 << 31)
    data = (torch.arange(total + 16, dtype=torch.int64, device="cuda") % 251).to(torch.uint8)
    offsets = torch.arange(n + 1, dtype=torch.int64, device="cuda") * L
    first = torch.full(((n + 31) // 32 + 1,), -1, dtype=torch.int32, device="cuda")
    idx = torch.full((n + 1,), -1, dtype=torch.int32, device="cuda")
    mc = torch.zeros(4, dtype=torch.int64, device="cuda")
    cnt = torch.zeros(3, dtype=torch.int64, device="cuda")
    marks = np.array([251, n], np.int64)
    rows = [(offsets.data_ptr(), data.data_ptr(), None, 0, n, first.data_ptr())]
    ag.call("ag_parquet_byte_array_dict_encode_dev", 8, N.ba_chunk_table(rows), 1, marks.ctypes.data, 2, idx.data_ptr(),
            mc.data_ptr(), cnt.data_ptr(), None, None)
    ag.call("ag_stream_sync", None)
    want = np.arange(n) % 251
    assert np.array_equal(idx[:n].cpu().numpy(), want) and int(idx[n]) == -1
    assert cnt.cpu().tolist() == [251, 251 * L, n]
    assert mc.cpu().tolist() == [251, 251 * (L + 4), 251, 251 * (L + 4)]
    bits = np.unpackbits(first.cpu().numpy()[:(n + 31) // 32].view(np.uint8), bitorder="little")[:n]
    assert np.array_equal(bits, np.arange(n) < 251)
