"""The seams of the shared-memory page window and the span chain walk (csrc/pq_window.cuh), against the Python
restatements: RLE/bit-packed run headers (pq_runs_kernel), DELTA_BINARY_PACKED block headers (delta_walk_kernel), Snappy
elements (snappy_parse_kernel) and PLAIN BYTE_ARRAY length prefixes (ba_plain_parse_kernel).

The window is 16-byte aligned to the absolute address, so where its edges fall depends on where a page starts: every
stream runs as 16 pages, one at each page-start residue mod 16.  Each generator is checked by a replay of the kernel's
window and span positions, so that the seams it is meant to hit are asserted to occur."""
import ctypes as C

import numpy as np
import pytest

import pq_bytearray_ref as B
import pq_delta_ref as D
import pq_ref as R
import snappy_ref as S
from arrow_go_b200 import _native as N
from helpers import Dev
from pq_pages import as_array

pytestmark = pytest.mark.gpu

WIN = 16384        # bytes of the shared-memory window (kWinBytes)
SPAN = 1024        # candidate element starts per parse step (kSpan)
LOOK = 4           # bytes past its start that a Snappy element header or a BYTE_ARRAY length prefix reads
RESIDUES = range(16)


def layout(streams):
    """[(bytes, num_values or dst_len)] -> (blob, [(offset, len, n, first output)], n_out): stream k starts at an
    offset congruent to k mod 16, outputs back to back"""
    blob, pages, out = bytearray(), [], 0
    for k, (s, n) in enumerate(streams):
        blob += bytes((k - len(blob)) % 16)
        pages.append((len(blob), len(s), n, out))
        blob += s
        out += n
    return as_array(blob + bytes(16)), pages, out


def at_residues(stream, n):
    return layout([(stream, n)] * 16)


def upload(blob):
    d = Dev(blob)
    assert d.ptr % 16 == 0
    return d


# ---------------------------------------------------------------- RLE hybrid run headers ----
def rle_page(rng, bw):
    """repeated runs (1- or 2-byte header, (bw+7)/8-byte value) and literal runs of 1..40 payload bytes, so that run
    sizes vary from 2 to about 40 bytes, and one literal run whose payload spans more than a window"""
    runs, vals, hi = [], [], 2 if bw == 1 else 4096
    while sum(len(r) for r in runs) < 10 * WIN:
        if len(runs) == 40:
            x = rng.integers(0, hi, 8 * (2 * WIN // bw + 8))
        elif rng.random() < 0.5:
            c, v = int(rng.integers(1, 200)), int(rng.integers(0, hi))
            runs.append(R.repeated_run(v, c, bw)); vals.append(np.full(c, v))
            continue
        else:
            x = rng.integers(0, hi, 8 * int(rng.integers(1, max(2, 40 // bw + 1))))
        runs.append(R.literal_run(x, bw)); vals.append(x)
    return b"".join(runs), int(sum(v.size for v in vals)), hi


def rle_seams(stream, bw, residue):
    """pq_runs_kernel's windows: (offsets wend - pos of run headers 1..16 bytes before a window end, whether a literal
    payload skipped a whole window)"""
    nrep, seen, skipped = (bw + 7) // 8, set(), False
    pos, n = 0, len(stream)
    while pos < n:
        wend = WIN - (residue + pos) % 16 + pos                 # the window starts at the aligned start of pos
        while pos < n:
            if 1 <= wend - pos <= 16:
                seen.add(wend - pos)
            if pos + 16 > wend and wend < n:
                break
            ind, k = 0, 0
            while True:
                c = stream[pos + k]
                ind |= (c & 0x7F) << (7 * k)
                k += 1
                if not c & 0x80:
                    break
            body = pos + k
            pos = body + (ind >> 1) * bw if ind & 1 else body + nrep
            skipped |= bool(ind & 1) and body < wend and pos > wend + WIN
    return seen, skipped


@pytest.mark.parametrize("bw", [1, 17, 24, 32])
def test_rle_run_headers_at_window_ends(ag, bw):
    rng = np.random.default_rng(700 + bw)
    stream, nv, hi = rle_page(rng, bw)
    seen, skipped = set(), False
    for r in RESIDUES:
        s, k = rle_seams(stream, bw, r)
        seen |= s
        skipped |= k
    assert seen == set(range(1, 17)) and skipped
    page = bytes([bw]) + stream                                  # the page's bit-width byte, then the hybrid stream
    blob, pages, n_out = layout([(page, nv)] * 16)
    dictionary = np.random.default_rng(bw).integers(-(1 << 62), 1 << 62, hi)
    dd, db, do, ddec = Dev(dictionary), upload(blob), Dev(np.full(n_out, -7, np.int64)), Dev(np.full(16, -1, np.int64))
    dbad = Dev(np.array([-1], np.int64))
    st, msg = ag.call_status("ag_parquet_dict_decode_dev", 8, dd.ptr, dictionary.size, db.ptr, N.page_table(pages), 16, None,
                             do.ptr, ddec.ptr, dbad.ptr, None)
    ag.call("ag_stream_sync", None)
    want, slots, err, bad = R.dict_decode(page, dictionary, nv)
    assert st == N.AG_OK and err == R.ERR_NONE and bad is None and slots == nv, msg
    assert ddec.get().tolist() == [nv] * 16 and int(dbad.get()[0]) == N.NO_ERROR_POS
    assert np.array_equal(do.get(), np.tile(want, 16))


# ---------------------------------------------------------------- DELTA_BINARY_PACKED block headers ----
def delta_page(rng, width, block, minis, windows):
    """about `windows` windows of blocks: most of one constant delta (every miniblock 0 bits wide, so the block is its
    header), the rest of random widths; min deltas of every varint length"""
    vpm, lim = block // minis, 8 * width - 2
    deltas, size = [], 0
    while size < windows * WIN:
        base = int(rng.integers(-(1 << int(rng.integers(0, lim))), 1 << int(rng.integers(0, lim))))
        k = 0 if rng.random() < 0.95 else int(rng.integers(0, 9))
        for _ in range(minis):
            deltas.append(base + (rng.integers(0, 1 << k, vpm) if k else np.zeros(vpm, np.int64)))
        size += len(D.varint(D.zigzag(base))) + minis + block * k // 8
    d = np.concatenate(deltas)
    with np.errstate(over="ignore"):
        vals = np.concatenate([[int(rng.integers(-1000, 1000))], d]).cumsum(dtype=np.int64)
    vals = vals.astype(np.int32) if width == 4 else vals
    return D.delta_encode(vals, width, block, minis), vals.size


def delta_seams(page, residue):
    """delta_walk_kernel's windows: (wend - pos, varint length, header length) of every block header that crosses a
    window end"""
    pos, out = 0, []
    block, pos = D._uvarint(page, pos)
    minis, pos = D._uvarint(page, pos)
    total, pos = D._uvarint(page, pos)
    _, pos = D._uvarint(page, pos)
    vpm, want = block // minis, (total - 2) // (block // minis) + 1
    nmb, wend = 0, 0
    while nmb < want:
        if pos >= wend:
            wend = WIN - (residue + pos) % 16 + pos
        _, p2 = D._uvarint(page, pos)
        if pos < wend < p2 + minis:
            out.append((wend - pos, p2 - pos, p2 + minis - pos))
        pos = p2 + minis
        for bw in page[p2:p2 + minis]:
            if nmb == want:
                break
            nmb += 1
            pos += vpm * bw // 8
    return out


@pytest.mark.parametrize("width", [4, 8], ids=["int32", "int64"])
@pytest.mark.parametrize("shape", [(128, 4, 3), (512, 16, 2)], ids=["128x4", "512x16"])
def test_delta_block_headers_across_window_ends(ag, width, shape):
    rng = np.random.default_rng(710 + width + shape[1])
    page, nv = delta_page(rng, width, *shape)
    cross = [c for r in RESIDUES for c in delta_seams(page, r)]
    in_varint = {d for d, v, h in cross if d < v}
    in_widths = {d for d, v, h in cross if d >= v}
    assert len(in_varint) >= 2 and len(in_widths) >= 3, cross
    assert any(v > 1 and d < v for d, v, h in cross)             # a multi-byte min delta cut by the window end
    blob, pages, n_out = at_residues(page, nv)
    dt = np.int32 if width == 4 else np.int64
    db, do, ddec = upload(blob), Dev(np.full(n_out, -7, dt)), Dev(np.full(16, -1, np.int64))
    st, msg = ag.call_status("ag_parquet_delta_decode_dev", width, db.ptr, N.page_table(pages), 16, None, do.ptr, ddec.ptr, None)
    ag.call("ag_stream_sync", None)
    want, slots, err, _ = D.delta_decode(page, width, nv)
    assert st == N.AG_OK and err == D.DERR_NONE and slots == nv, msg
    assert ddec.get().tolist() == [nv] * 16 and np.array_equal(do.get(), np.tile(want, 16))


# ---------------------------------------------------------------- the span chain: Snappy and PLAIN BYTE_ARRAY ----
# The first element of each stream is FIRST bytes long, so that the second span's look-ahead ends FIRST + SPAN + LOOK
# bytes after the first span's start, between 8 bytes short of and 7 bytes past the end of the window loaded there.
FIRST = WIN - SPAN - LOOK - 7


def span_seams(starts, n, residue):
    """the parse kernels' spans over elements starting at `starts` (stream offsets, the first span at starts[0]):
    [(span start, index of its first element, index of its last element, window margin)], the margin being the bytes
    between the span's look-ahead end and the end of the window loaded before it (negative: the span loads a new one)"""
    out, wlo, i = [], -(1 << 62), 0
    while i < len(starts):
        cur = starts[i]
        hi = min(cur + SPAN + LOOK, n)
        margin = wlo + WIN - hi
        if margin < 0:
            wlo = cur - (residue + cur) % 16
        j = i
        while j + 1 < len(starts) and starts[j + 1] < cur + SPAN:
            j += 1
        out.append((cur, i, j, margin))
        i = j + 1
    return out


def snappy_elements(rng, count):
    """a FIRST-byte literal, then literals of 1..8 bytes and copies of every form with offsets no shorter than their
    length"""
    els, out = [S.literal(rng.integers(0, 256, FIRST - 3, dtype=np.uint8).tobytes(), 2)], FIRST - 3
    for _ in range(count):
        f = int(rng.integers(0, 4))
        if f == 0:
            x = rng.integers(0, 256, int(rng.integers(1, 9)), dtype=np.uint8).tobytes()
            els.append(S.literal(x)); out += len(x)
        else:
            ln = int(rng.integers(4, 12)) if f == 1 else int(rng.integers(1, 65))
            off = int(rng.integers(ln, min(out, 2047 if f == 1 else 65535) + 1))
            els.append(S.copy(off, ln, (1, 2, 4)[f - 1])); out += ln
    return els, out


def corrupt(el):
    """the same copy element with offset 0 (a copy-1 tag holds the offset's high bits)"""
    return bytes([el[0] & 0x1F if el[0] & 3 == 1 else el[0]]) + bytes(len(el) - 1)


def test_snappy_elements_at_span_and_window_edges(ag):
    rng = np.random.default_rng(720)
    els, dlen = snappy_elements(rng, 24_000)
    pre = S.put_uvarint(dlen)
    starts = list(len(pre) + np.concatenate([[0], np.cumsum([len(e) for e in els])[:-1]]))
    good = pre + b"".join(els)
    spans = [s for r in RESIDUES for s in span_seams(starts, len(good), r)]
    last_q = {starts[j] - cur for cur, i, j, m in spans}
    assert {1020, 1021, 1022, 1023} <= last_q
    assert {0, -1} <= {m for *_, m in spans}                      # a span that reads the window's last byte, or one past it
    # a copy with offset 0 at the first and at the last element of a span
    sp = span_seams(starts, len(good), 0)
    first = next(i for cur, i, j, m in sp[3:] if els[i][0] & 3)
    last = next(j for cur, i, j, m in sp[3:] if els[j][0] & 3 and starts[j] - cur >= 1020)
    streams = [(good, dlen)]
    for k in (first, last):
        streams.append((pre + b"".join(els[:k] + [corrupt(els[k])] + els[k + 1:]), dlen))
    for s, n in streams:
        src, pages, n_out = at_residues(s, n)
        tbl = N.compressed_table([(o, ln, d, dl) for o, ln, dl, d in pages])
        ds, do, dw = upload(src), Dev(np.full(n_out, 0xA5, np.uint8)), Dev(np.full(16, -1, np.int64))
        st, msg = ag.call_status("ag_parquet_snappy_decompress_dev", ds.ptr, tbl, 16, do.ptr, dw.ptr, None)
        ag.call("ag_stream_sync", None)
        want, err, _ = S.decode(s, n)
        assert dw.get().tolist() == [len(want)] * 16, msg
        got = do.get().reshape(16, n)
        assert all(g[:len(want)].tobytes() == want and (g[len(want):] == 0xA5).all() for g in got)
        if err:
            assert st == N.AG_ERR_INVALID and f"page 0: {S.MESSAGE[err]} ({len(want)} bytes written)" in msg, msg
        else:
            assert st == N.AG_OK, msg


def ba_values(rng, count):
    """a FIRST-byte element, then values of 0..6 bytes"""
    return [bytes(FIRST - 4)] + [rng.integers(97, 123, int(rng.integers(0, 7)), dtype=np.uint8).tobytes() for _ in range(count)]


def ba_starts(vals):
    return list(np.concatenate([[0], np.cumsum([4 + len(v) for v in vals])[:-1]]))


@pytest.mark.parametrize("spaced", [False, True], ids=["dense", "spaced"])
def test_plain_byte_array_prefixes_at_span_and_window_edges(ag, spaced):
    rng = np.random.default_rng(730 + spaced)
    vals = ba_values(rng, 30_000)
    good = B.plain_encode(vals)
    starts = ba_starts(vals)
    spans = [s for r in RESIDUES for s in span_seams(starts, len(good), r)]
    last_q = {starts[j] - cur for cur, i, j, m in spans}
    assert {1021, 1022, 1023} <= last_q                           # a length prefix across the span end
    assert any(starts[j] - cur + 4 + len(vals[j]) == SPAN for cur, i, j, m in spans)   # a value ends at the span end
    assert {0, -1} <= {m for *_, m in spans}
    sp = span_seams(starts, len(good), 0)
    first = sp[5][1]
    last = next(j for cur, i, j, m in sp[7:] if starts[j] - cur >= SPAN - 3)   # its length prefix crosses the span end
    cases = [(good, len(vals))]
    for k in (first, last):
        neg = bytearray(good)
        neg[starts[k]:starts[k] + 4] = (-3).to_bytes(4, "little", signed=True)
        cases.append((bytes(neg), len(vals)))
        cut = good[:starts[k] + 4 + len(vals[k]) - 1] if vals[k] else good[:starts[k] + 3]
        cases.append((cut, len(vals)))
    for page, nv in cases:
        streams, valid = [(page, nv)] * 16, None
        if spaced:                                               # the page's values at random slots among 25 % nulls
            slots = nv + nv // 3
            pv = np.zeros(slots, bool)
            pv[np.sort(rng.choice(slots, nv, replace=False))] = True
            streams, valid = [(page, slots)] * 16, np.tile(pv, 16)
        blob, pages, n_out = layout(streams)
        cap = 16 * len(page) + 64
        db, do, ddat = upload(blob), Dev(np.full(n_out + 1, -9, np.int64)), Dev(nbytes=cap)
        ddec, total = Dev(np.full(16, -1, np.int64)), C.c_int64(-1)
        dv = Dev(np.packbits(np.concatenate([valid, np.zeros(64, bool)]), bitorder="little")) if spaced else None
        st, msg = ag.call_status("ag_parquet_byte_array_decode_dev", B.PLAIN, 8, db.ptr, N.page_table(pages), 16, n_out,
                                 dv.ptr if dv else None, None, None, 0, 0, do.ptr, ddat.ptr, cap, C.byref(total),
                                 ddec.ptr, None, None)
        ag.call("ag_stream_sync", None)
        want, wslots, wmsg = B.plain_decode(page, pv if spaced else nv)
        assert ddec.get().tolist() == [wslots] * 16, (msg, wmsg)
        if wmsg:
            assert st == N.AG_ERR_INVALID and f"page 0: {wmsg} ({wslots} values decoded)" in msg, (msg, wmsg)
        else:
            assert st == N.AG_OK, msg
            data = b"".join(want) * 16
            assert do.get().tolist() == np.concatenate([[0], np.cumsum(np.tile([len(v) for v in want], 16))]).tolist()
            assert total.value == len(data) and ddat.get()[:len(data)].tobytes() == data
