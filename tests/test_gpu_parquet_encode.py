"""Device Parquet page encoders, host and _dev flavours, byte for byte: RLE/bit-packed streams against RleEncoder's
restatement (pq_ref.rle_encode) for every form, input kind and bit width; RLE booleans against bool_rle_encode;
DELTA_BINARY_PACKED against delta_encode; pages of pyarrow-written files rebuilt end to end on the device
(dictionary_encode, filter of the indices by validity, levels from the validity bitmap); round trips through the
device decoders; argument and value errors; offsets past 2^31."""
import ctypes as C

import numpy as np
import pytest

import pq_delta_ref as D
import pq_files as F
import pq_fixed_ref as FX
import pq_pages as P
import pq_ref as R
from arrow_go_b200 import _native as N
from helpers import Dev, ptr

pytestmark = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])


def rle_bound(ag, bw, form, n):
    s = C.c_int64()
    ag.call("ag_parquet_rle_max_size", bw, form, n, C.byref(s))
    return s.value


def delta_bound(ag, width, block, mini, n):
    s = C.c_int64()
    ag.call("ag_parquet_delta_max_size", width, block, mini, n, C.byref(s))
    return s.value


def layout(sizes, bound, rng, gap=True):
    """[(in, n, out, capacity)] of pages over consecutive input, outputs in shuffled order with gaps; total bytes"""
    order = rng.permutation(len(sizes)) if gap else np.arange(len(sizes))
    outs, pos = {}, 0
    for k in order:
        pos += int(rng.integers(0, 9)) if gap else 0
        outs[k] = pos
        pos += bound(sizes[k])
    pages, i0 = [], 0
    for k, n in enumerate(sizes):
        pages.append((i0, n, outs[k], bound(n)))
        i0 += n
    return pages, pos


def run(ag, fn, head, values, pages, n_out, dev, bad=True):
    """-> (status, message, out bytes, lengths, bad_pos or None)"""
    tbl = N.enc_page_table(pages)
    out = np.full(n_out + 64, 0xA5, np.uint8)
    lens = np.full(len(pages), -1, np.int64)
    bp = np.full(1, -5, np.int64)
    if not dev:
        tail = (ptr(lens), ptr(bp)) if bad else (ptr(lens),)
        st, msg = ag.call_status(fn, *head, ptr(values), tbl, len(pages), ptr(out), *tail)
        return st, msg, out, lens, (int(bp[0]) if bad else None)
    dv, do, dl, db = Dev(values), Dev(out), Dev(lens), Dev(bp)
    tail = (dl.ptr, db.ptr) if bad else (dl.ptr,)
    st, msg = ag.call_status(fn + "_dev", *head, dv.ptr, tbl, len(pages), do.ptr, *tail, None)
    ag.call("ag_stream_sync", None)
    return st, msg, do.get(), dl.get(), (int(db.get()[0]) if bad else None)


def rle_expect(vals, bw, form):
    s = R.rle_encode([int(x) for x in vals], bw)
    return {N.PQ_RLE_BARE: b"", N.PQ_RLE_LEN4: len(s).to_bytes(4, "little"), N.PQ_RLE_WIDTH: bytes([bw])}[form] + s


def check_rle(ag, bw, form, inp, values, pages, n_out, dev, logical):
    st, msg, out, lens, bad = run(ag, "ag_parquet_rle_encode", (bw, form, inp), values, pages, n_out, dev)
    assert st == N.AG_OK, msg
    assert bad == N.NO_ERROR_POS
    for k, (i0, n, o, cap) in enumerate(pages):
        want = rle_expect(logical[i0:i0 + n], bw, form)
        assert lens[k] == len(want), (k, n)
        assert out[o:o + lens[k]].tobytes() == want, (k, n, bw, form)


def sample(rng, kind, n, bw):
    top = (1 << bw) - 1
    if kind == "random":
        return rng.integers(0, top + 1, n, dtype=np.uint64)
    if kind == "clustered":
        lens = rng.integers(1, 65, n // 4 + 2)
        v = np.repeat(rng.integers(0, top + 1, lens.size, dtype=np.uint64), lens)
        return v[:n] if v.size >= n else np.concatenate([v, np.zeros(n - v.size, np.uint64)])
    # adversarial: runs of 7, 8 and 9 on every residue, literal stretches of 62..64 groups, short equal tails
    parts = []
    while sum(p.size for p in parts) < n:
        c = int(rng.integers(0, 6))
        if c < 3:
            parts.append(np.full(int(rng.choice([7, 8, 9, 15, 16, 17])), rng.integers(0, top + 1), np.uint64))
        elif c < 5:
            parts.append(rng.integers(0, top + 1, int(rng.integers(1, 8)), dtype=np.uint64))
        else:
            g = int(rng.choice([62, 63, 64, 126]))
            parts.append(((np.arange(8 * g) % 2) ^ (np.arange(8 * g) // 3 % 2)).astype(np.uint64) * np.uint64(top))
    return np.concatenate(parts)[:n]


SIZES = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 4095, 4096, 4097, 20_000, 0, 37, 511, 512, 513]


@FLAVOURS
@pytest.mark.parametrize("bw", range(33))
def test_rle_indices_every_width(ag, bw, dev):
    rng = np.random.default_rng(bw)
    for kind in ("random", "clustered", "adversarial"):
        logical = sample(rng, kind, sum(SIZES), bw)
        vals = logical.astype(np.uint32)
        for form in (N.PQ_RLE_BARE, N.PQ_RLE_LEN4, N.PQ_RLE_WIDTH):
            pages, n_out = layout(SIZES, lambda n: rle_bound(ag, bw, form, n), rng)
            check_rle(ag, bw, form, N.PQ_RLE_IN_U32, vals, pages, n_out, dev, logical)


@FLAVOURS
@pytest.mark.parametrize("bw", range(17))
def test_rle_levels(ag, bw, dev):
    rng = np.random.default_rng(100 + bw)
    for kind in ("random", "clustered", "adversarial"):
        logical = sample(rng, kind, sum(SIZES), min(bw, 15))       # levels are non-negative int16
        vals = logical.astype(np.int16)
        for form in (N.PQ_RLE_BARE, N.PQ_RLE_LEN4):
            pages, n_out = layout(SIZES, lambda n: rle_bound(ag, bw, form, n), rng)
            check_rle(ag, bw, form, N.PQ_RLE_IN_I16, vals, pages, n_out, dev, logical)


@FLAVOURS
def test_rle_bitmap_levels_and_booleans(ag, dev):
    rng = np.random.default_rng(3)
    for kind in ("random", "clustered", "adversarial"):
        bits = sample(rng, kind, sum(SIZES) + 5, 1)
        packed = np.packbits(bits.astype(np.uint8), bitorder="little")
        for form in (N.PQ_RLE_BARE, N.PQ_RLE_LEN4):
            pages, n_out = layout(SIZES, lambda n: rle_bound(ag, 1, form, n), rng)
            pages = [(i0 + 5, n, o, c) for i0, n, o, c in pages]          # bit offsets off the byte grid
            check_rle(ag, 1, form, N.PQ_RLE_IN_BITMAP, packed, pages, n_out, dev, bits)
            if form == N.PQ_RLE_LEN4:
                st, msg, out, lens, _ = run(ag, "ag_parquet_rle_encode", (1, form, N.PQ_RLE_IN_BITMAP), packed, pages, n_out, dev)
                for k, (i0, n, o, c) in enumerate(pages):
                    assert out[o:o + lens[k]].tobytes() == FX.bool_rle_encode(bits[i0:i0 + n])


@FLAVOURS
def test_rle_many_small_pages_and_long_page(ag, dev):
    rng = np.random.default_rng(9)
    sizes = [int(x) for x in rng.integers(0, 40, 3000)] + [1_000_003]
    logical = sample(rng, "clustered", sum(sizes), 17)
    pages, n_out = layout(sizes, lambda n: rle_bound(ag, 17, N.PQ_RLE_WIDTH, n), rng)
    check_rle(ag, 17, N.PQ_RLE_WIDTH, N.PQ_RLE_IN_U32, logical.astype(np.uint32), pages, n_out, dev, logical)


@FLAVOURS
@pytest.mark.parametrize("width,block,mini", [(4, 128, 4), (8, 128, 4), (8, 256, 4), (4, 128, 1), (8, 1024, 8), (4, 4096, 1)])
def test_delta_against_restatement(ag, width, block, mini, dev):
    rng = np.random.default_rng(block + width + mini)
    dt = np.int32 if width == 4 else np.int64
    info = np.iinfo(dt)
    sizes = SIZES + [block + 1, 2 * block, 2 * block + 1, 100_000]
    for kind in ("random", "timestamps", "extremes", "constant"):
        n = sum(sizes)
        if kind == "random":
            v = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
        elif kind == "timestamps":
            v = (np.cumsum(rng.integers(0, 1000, n)) + 1_700_000_000).astype(dt)
        elif kind == "extremes":
            v = rng.choice(np.array([info.min, info.max, 0, -1, 1], dt), n)
        else:
            v = np.full(n, 77, dt)
        pages, n_out = layout(sizes, lambda k: delta_bound(ag, width, block, mini, k), rng)
        st, msg, out, lens, _ = run(ag, "ag_parquet_delta_encode", (width, block, mini), v, pages, n_out, dev, bad=False)
        assert st == N.AG_OK, msg
        for k, (i0, cnt, o, cap) in enumerate(pages):
            want = D.delta_encode(v[i0:i0 + cnt], width, block, mini)
            assert lens[k] == len(want) and out[o:o + lens[k]].tobytes() == want, (kind, k, cnt)


# ------------------------------------------------------------------------------------ pyarrow, end to end ----
def _pages_of(path):
    plan = P.chunk_plan(path)
    return plan, P.host_decompress(plan)


def _dict_width(ndict):
    return 0 if ndict == 0 else max(1, (ndict - 1).bit_length())


@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("dtype", ["int64", "int32", "float64"])
def test_dictionary_pages_end_to_end(ag, tmp_path, version, dtype):
    pa = pytest.importorskip("pyarrow")
    rng = np.random.default_rng(21)
    n = 200_000
    vals = rng.integers(0, 3000, n).astype(dtype)
    if dtype == "float64":
        vals = vals * 0.25 - 100.0
    valid = rng.random(n) >= 0.1
    valid[50_000:60_000] = False
    path = str(tmp_path / "d.parquet")
    F.write_column(path, pa.array(vals, mask=~valid), nullable=True, encoding="RLE_DICTIONARY", version=version,
                   data_page_size=1 << 17)
    plan, dst = _pages_of(path)
    width = vals.dtype.itemsize
    vbits = np.packbits(valid, bitorder="little")
    dv, dvalid = Dev(vals), Dev(vbits)
    didx = Dev(nbytes=4 * n)
    didx_valid = Dev(nbytes=(n + 31) // 32 * 4)
    ddict = Dev(nbytes=width * n)
    counts = Dev(np.zeros(3, np.int64))
    chunks = N.dict_chunk_table([(dv.ptr, dvalid.ptr, 0, n, didx.ptr, didx_valid.ptr)])
    ag.call("ag_dictionary_encode_dev", 8 * width, chunks, 1, N.NULL_ENCODING_MASK, ddict.ptr, None, counts.ptr, None)
    ag.call("ag_stream_sync", None)
    ndict = int(counts.get()[0])
    d0, dl, _ = plan["dict"]
    assert ddict.get(np.uint8, ndict * width).tobytes() == dst[d0:d0 + dl]
    # the valid indices, dense
    dense = Dev(nbytes=4 * n)
    dlen = Dev(np.zeros(1, np.int64))
    ag.call("ag_filter_primitive_dev", 32, didx.ptr, None, 0, dvalid.ptr, None, 0, n, N.DROP_NULLS, dense.ptr, None, n, dlen.ptr, None)
    ag.call("ag_stream_sync", None)
    assert int(dlen.get()[0]) == int(valid.sum())
    bw = _dict_width(ndict)
    before = np.concatenate([[0], np.cumsum(valid)])
    secs = P.value_sections(plan, dst)
    ipages, lpages, o_i, o_l = [], [], 0, 0
    lform = N.PQ_RLE_LEN4 if version == "1.0" else N.PQ_RLE_BARE
    for _, (_, _, nv, slot) in secs:
        k = int(before[slot + nv] - before[slot])
        cap = rle_bound(ag, bw, N.PQ_RLE_WIDTH, k)
        ipages.append((int(before[slot]), k, o_i, cap))
        o_i += cap
        cap = rle_bound(ag, 1, lform, nv)
        lpages.append((slot, nv, o_l, cap))
        o_l += cap
    iout, lout = Dev(nbytes=o_i), Dev(nbytes=o_l)
    ilen, llen = Dev(np.zeros(len(secs), np.int64)), Dev(np.zeros(len(secs), np.int64))
    ag.call("ag_parquet_rle_encode_dev", bw, N.PQ_RLE_WIDTH, N.PQ_RLE_IN_U32, dense.ptr, N.enc_page_table(ipages), len(ipages),
            iout.ptr, ilen.ptr, None, None)
    ag.call("ag_parquet_rle_encode_dev", 1, lform, N.PQ_RLE_IN_BITMAP, dvalid.ptr, N.enc_page_table(lpages), len(lpages),
            lout.ptr, llen.ptr, None, None)
    ib, lb, il, ll = iout.get(), lout.get(), ilen.get(), llen.get()
    for k, ((_, (vd, vl, nv, slot)), (_, lv, _)) in enumerate(zip(secs, plan["pages"])):
        assert ib[ipages[k][2]:ipages[k][2] + il[k]].tobytes() == dst[vd:vd + vl], k
        d, dl2, _, _ = lv
        want = dst[d:d + 4 + int.from_bytes(dst[d:d + 4], "little")] if version == "1.0" else plan["chunk"][d:d + dl2]
        assert lb[lpages[k][2]:lpages[k][2] + ll[k]].tobytes() == want, k


@pytest.mark.parametrize("width,block", [(4, 128), (8, 256)])
def test_delta_pages_end_to_end(ag, tmp_path, width, block):
    pa = pytest.importorskip("pyarrow")
    rng = np.random.default_rng(width)
    n = 300_000
    if width == 8:
        vals = (1_700_000_000_000_000_000 + np.cumsum(rng.integers(0, 5_000_000, n))).astype(np.int64)
    else:
        vals = rng.integers(-(1 << 31), 1 << 31, n).astype(np.int32)
    path = str(tmp_path / "t.parquet")
    F.write_column(path, pa.array(vals), nullable=False, encoding="DELTA_BINARY_PACKED", version="2.0", data_page_size=1 << 18)
    plan, dst = _pages_of(path)
    secs = P.value_sections(plan, dst)
    pages, o = [], 0
    for _, (_, _, nv, slot) in secs:
        cap = delta_bound(ag, width, block, 4, nv)
        pages.append((slot, nv, o, cap))
        o += cap
    st, msg, out, lens, _ = run(ag, "ag_parquet_delta_encode", (width, block, 4), vals, pages, o, True, bad=False)
    assert st == N.AG_OK, msg
    for k, (_, (vd, vl, nv, slot)) in enumerate(secs):
        assert out[pages[k][2]:pages[k][2] + lens[k]].tobytes() == dst[vd:vd + vl], k


# --------------------------------------------------------------------------- round trips through the decoders ----
def test_round_trips_through_decoders(ag):
    rng = np.random.default_rng(31)
    sizes = [0, 1, 9, 4097, 70_000]
    # levels (max level 5 -> bit width 3), v1 form
    lv = sample(rng, "clustered", sum(sizes), 3).astype(np.int16) % 6
    pages, n_out = layout(sizes, lambda n: rle_bound(ag, 3, N.PQ_RLE_LEN4, n), rng, gap=False)
    st, msg, out, lens, _ = run(ag, "ag_parquet_rle_encode", (3, N.PQ_RLE_LEN4, N.PQ_RLE_IN_I16), lv, pages, n_out, True)
    assert st == N.AG_OK, msg
    dp = [(o, int(lens[k]), n, i0) for k, (i0, n, o, c) in enumerate(pages)]
    got = np.zeros(lv.size, np.int16)
    ag.call("ag_parquet_levels_decode", 5, N.PQ_LEVELS_V1_RLE, ptr(out), N.page_table(dp), len(dp), ptr(got), None)
    assert (got == lv).all()
    # dictionary indices, width form
    dic = np.arange(1000, dtype=np.int64) * 3
    idx = sample(rng, "adversarial", sum(sizes), 10).astype(np.uint32) % 1000
    pages, n_out = layout(sizes, lambda n: rle_bound(ag, 10, N.PQ_RLE_WIDTH, n), rng, gap=False)
    st, msg, out, lens, _ = run(ag, "ag_parquet_rle_encode", (10, N.PQ_RLE_WIDTH, N.PQ_RLE_IN_U32), idx, pages, n_out, True)
    assert st == N.AG_OK, msg
    dp = [(o, int(lens[k]), n, i0) for k, (i0, n, o, c) in enumerate(pages)]
    got = np.zeros(idx.size, np.int64)
    ag.call("ag_parquet_dict_decode", 8, ptr(dic), dic.size, ptr(out), N.page_table(dp), len(dp), None, ptr(got), None, None)
    assert (got == dic[idx]).all()
    # booleans
    bits = sample(rng, "random", sum(sizes), 1).astype(np.uint8)
    packed = np.packbits(bits, bitorder="little")
    pages, n_out = layout(sizes, lambda n: rle_bound(ag, 1, N.PQ_RLE_LEN4, n), rng, gap=False)
    st, msg, out, lens, _ = run(ag, "ag_parquet_rle_encode", (1, N.PQ_RLE_LEN4, N.PQ_RLE_IN_BITMAP), packed, pages, n_out, False)
    assert st == N.AG_OK, msg
    dp = [(o, int(lens[k]), n, i0) for k, (i0, n, o, c) in enumerate(pages)]
    gotb = np.zeros((bits.size + 7) // 8, np.uint8)
    ag.call("ag_parquet_bool_decode", N.PQ_ENC_RLE, ptr(out), N.page_table(dp), len(dp), None, ptr(gotb), None)
    assert (np.unpackbits(gotb, bitorder="little")[:bits.size] == bits).all()
    # DELTA INT64
    v = rng.integers(-(1 << 62), 1 << 62, sum(sizes))
    pages, n_out = layout(sizes, lambda n: delta_bound(ag, 8, 256, 4, n), rng, gap=False)
    st, msg, out, lens, _ = run(ag, "ag_parquet_delta_encode", (8, 256, 4), v, pages, n_out, True, bad=False)
    assert st == N.AG_OK, msg
    dp = [(o, int(lens[k]), n, i0) for k, (i0, n, o, c) in enumerate(pages)]
    gotv = np.zeros(v.size, np.int64)
    ag.call("ag_parquet_delta_decode", 8, ptr(out), N.page_table(dp), len(dp), None, ptr(gotv), None)
    assert (gotv == v).all()


# ---------------------------------------------------------------------------------------------------- errors ----
@FLAVOURS
def test_value_wider_than_bit_width(ag, dev):
    rng = np.random.default_rng(41)
    vals = rng.integers(0, 32, 30_000).astype(np.uint32)
    vals[[17_000, 25_000]] = 32
    sizes = [10_000, 10_000, 10_000]
    pages, n_out = layout(sizes, lambda n: rle_bound(ag, 5, N.PQ_RLE_BARE, n), rng)
    st, msg, _, _, bad = run(ag, "ag_parquet_rle_encode", (5, N.PQ_RLE_BARE, N.PQ_RLE_IN_U32), vals, pages, n_out, dev)
    assert st == N.AG_ERR_INVALID and bad == 17_000 and "page 1" in msg, msg
    lv = np.zeros(100, np.int16)
    lv[40] = -1
    pages = [(0, 100, 0, rle_bound(ag, 16, N.PQ_RLE_BARE, 100))]
    st, msg, _, _, bad = run(ag, "ag_parquet_rle_encode", (16, N.PQ_RLE_BARE, N.PQ_RLE_IN_I16), lv, pages, pages[0][3], dev)
    assert st == N.AG_ERR_INVALID and bad == 40, msg


@FLAVOURS
def test_refused_arguments(ag, dev):
    vals = np.zeros(64, np.uint32)
    ok = rle_bound(ag, 4, N.PQ_RLE_BARE, 64)
    cases = [((4, N.PQ_RLE_BARE, N.PQ_RLE_IN_U32), ok - 1),     # capacity below the bound
             ((33, N.PQ_RLE_BARE, N.PQ_RLE_IN_U32), 4096), ((-1, N.PQ_RLE_BARE, N.PQ_RLE_IN_U32), 4096),
             ((17, N.PQ_RLE_BARE, N.PQ_RLE_IN_I16), 4096), ((2, N.PQ_RLE_BARE, N.PQ_RLE_IN_BITMAP), 4096),
             ((4, 3, N.PQ_RLE_IN_U32), 4096), ((4, N.PQ_RLE_BARE, 3), 4096)]
    for head, cap in cases:
        st, msg, _, _, bad = run(ag, "ag_parquet_rle_encode", head, vals, [(0, 64, 0, cap)], cap, dev)
        assert st == N.AG_ERR_INVALID, (head, cap)
    okd = delta_bound(ag, 8, 128, 4, 64)
    dcases = [((8, 128, 4), okd - 1), ((2, 128, 4), 8192), ((8, 100, 4), 8192), ((8, 128, 3), 8192),
              ((8, 128, 8), 8192), ((8, 0, 4), 8192)]
    v64 = np.zeros(64, np.int64)
    for head, cap in dcases:
        st, msg, _, _, _ = run(ag, "ag_parquet_delta_encode", head, v64, [(0, 64, 0, cap)], cap, dev, bad=False)
        assert st == N.AG_ERR_INVALID, (head, cap)
    s = C.c_int64()
    assert ag.call_status("ag_parquet_rle_max_size", 33, 0, 10, C.byref(s))[0] == N.AG_ERR_INVALID
    assert ag.call_status("ag_parquet_delta_max_size", 8, 128, 3, 10, C.byref(s))[0] == N.AG_ERR_INVALID


def test_offsets_past_2_31(ag):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(51)
    vals = sample(rng, "clustered", 9000, 12).astype(np.uint32)
    i0 = (1 << 31) + 17
    big = torch.zeros(i0 + vals.size, dtype=torch.int32, device="cuda")
    big[i0:] = torch.from_numpy(vals.view(np.int32)).cuda()
    torch.cuda.synchronize()
    cap = rle_bound(ag, 12, N.PQ_RLE_WIDTH, 4000)
    o0 = (1 << 31) + 3
    outbuf = torch.zeros(o0 + 2 * cap + 64, dtype=torch.uint8, device="cuda")
    pages = [(i0, 4000, o0 + cap, cap), (i0 + 4000, 4000, o0, cap)]
    lens = Dev(np.zeros(2, np.int64))
    ag.call("ag_parquet_rle_encode_dev", 12, N.PQ_RLE_WIDTH, N.PQ_RLE_IN_U32, big.data_ptr(), N.enc_page_table(pages), 2,
            outbuf.data_ptr(), lens.ptr, None, None)
    ln = lens.get()
    for k, (a, n, o, c) in enumerate(pages):
        got = outbuf[o:o + int(ln[k])].cpu().numpy()
        assert got.tobytes() == rle_expect(vals[a - i0:a - i0 + n], 12, N.PQ_RLE_WIDTH), k
