"""Device LZ4_RAW page decompression against the Python restatement in tests/lz4_ref.py (host and _dev flavours, byte
for byte, the canary outside every written range): every form, page sizes, and the seams of the shared-memory window and
the span chain walk. Then what every codec does, through pq_codecs: argument checks, failing pages, the parquet-testing
fixtures against pyarrow, pyarrow-written files end to end, and ~200 MB of output through a checksum."""
import numpy as np
import pyarrow as pa
import pytest

import lz4_ref as R
import pq_codecs as H
import pq_files as F
from arrow_go_b200 import _native as N
from helpers import Dev
from test_gpu_parquet_window import RESIDUES, SPAN, WIN, at_residues, upload

gpu = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
EXT = 16                 # extension bytes the parse reads from the window (kExt); a longer run leaves it
LOOK = 2 * EXT + 3       # bytes past a span a short sequence's header reaches (kLook)


@gpu
@FLAVOURS
def test_every_form(ag, dev):
    rng = np.random.default_rng(81)
    streams = [(s, len(x)) for _, s, x in R.forms()]
    streams += [(s, n) for _, s, n, (outcome, _), _ in R.differences() if outcome == R.OK]
    for gap in (True, False):
        st, msg, errs = H.decode_and_compare(ag, H.LZ4, streams, rng, dev, gap)
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
    st, msg, errs = H.decode_and_compare(ag, H.LZ4, streams, rng, dev)
    assert st == N.AG_OK and not errs, msg


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
        ds, do, dw = upload(src), Dev(np.full(n_out, H.CANARY, np.uint8)), Dev(np.full(16, -1, np.int64))
        st, msg = ag.call_status("ag_parquet_lz4_raw_decompress_dev", ds.ptr, tbl, 16, do.ptr, dw.ptr, None)
        ag.call("ag_stream_sync", None)
        want, outcome, arg = R.decode(s, dlen)
        assert dw.get().tolist() == [len(want)] * 16, msg
        got = do.get().reshape(16, dlen)
        assert all(g[:len(want)].tobytes() == want and (g[len(want):] == H.CANARY).all() for g in got)
        if outcome != R.OK:
            assert st == N.AG_ERR_INVALID and f"page 0: {R.message(outcome, arg, dlen)} ({len(want)} bytes written)" in msg, msg
        else:
            assert st == N.AG_OK, msg


# ---------------------------------------------------------------- what every codec does (pq_codecs) ----
@gpu
@FLAVOURS
def test_invalid_arguments(ag, dev):
    H.invalid_arguments(ag, H.LZ4, dev)


@gpu
@FLAVOURS
@pytest.mark.parametrize("row", H.LZ4.error_rows(), ids=lambda r: r[0])
def test_error_rows(ag, row, dev):
    H.error_row(ag, H.LZ4, row, dev)


@gpu
@FLAVOURS
@pytest.mark.parametrize("name", H.LZ4.fixtures)
def test_fixture_pages_against_host(ag, name, dev):
    H.fixture_pages(ag, H.LZ4, name, dev)


@gpu
@pytest.mark.parametrize("case", F.compressed_cases(), ids=F.compressed_case_id)
def test_pyarrow_lz4_files_end_to_end(ag, case, tmp_path):
    H.pyarrow_file(ag, H.LZ4, case, tmp_path)


@gpu
@pytest.mark.parametrize("kind", ["byte_array", "fsb12", "bool"])
def test_pyarrow_lz4_files_other_types(ag, kind, tmp_path):
    H.pyarrow_file_other_type(ag, H.LZ4, kind, tmp_path)


@gpu
def test_decompress_200mb_device(ag):
    H.decompress_200mb(ag, H.LZ4)
