"""The device kernels past 2^31 rows, 2^32 bits and 2^32-row tables.

Every length, offset and index of the C ABI is 64-bit, but several kernels mix 32-bit and 64-bit arithmetic on
purpose (32-bit bitmap words, 32-bit per-row arithmetic in take's partition pass, 32-bit look-back payloads).  A row,
bit or output position narrowed to 32 bits only shows past 2^31 or 2^32, so each case here crosses that boundary.

All operands are carved from one device arena allocated once for the module, and every large input is produced on
the device by ag_generate_dev.  The generator is counter-based (value i = f(mix64(seed + i))), so its CPU twin
rebuilds any window [start, start + n) by seeding itself with seed + start; nothing multi-GB ever comes back to the
host.  Results are checked three ways: 1M-row windows around row 0, 2^31, 2^32 and the end against the oracle on the
regenerated window; device-side identities (popcounts, sums, ag_checksum64_dev); and whole-column totals that the
host computes by regenerating the column in chunks.  The CPU helpers that do this are pinned by the CPU tests at the
top of the file."""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from arrow_go_b200 import _native as N
from helpers import Dev
from oracle import oracle

MASK64 = (1 << 64) - 1
CHUNK = 1 << 24                     # rows per host chunk: 128 MB for the widest (8-byte) column
WORKERS = max(1, min(8, os.cpu_count() or 1))
W = 1 << 20                         # rows in a checked window
ARENA_BYTES = 17_500_000_000        # 2^31 + 2^16 + 3 int64 values (case 8, the largest) plus headroom
CANARY = 0xA5
SHIPPED_TAKE_POLICY = (0, 32 << 20, 160 << 20, 8 << 20)
_NP_KIND = {0: np.uint64, 1: np.int64, 2: np.int32, 3: np.float64}


# ---------------------------------------------------------------------------------------------------------------
# CPU twin of ag_generate_dev, and chunked host reductions over a regenerated column

def window(kind, seed, lo, hi, start, n):
    """Rows [start, start + n) of what ag_generate_dev(kind, seed, lo, hi) writes (kinds 0-4).  Kind 4 returns the
    packed LSB-first bitmap bytes of bits [start, start + n), with the bits past n clear; its start must be a
    multiple of 8, because the device writes whole bytes."""
    if kind == 4:
        assert start % 8 == 0, "kind 4 windows start on a byte"
        out = np.zeros((n + 7) // 8, dtype=np.uint8)
    else:
        out = np.empty(n, dtype=_NP_KIND[kind])
    if n:
        oracle.cpu().ref_generate(kind, (seed + start) & MASK64, lo, hi, out.ctypes.data, n)
    return out


def byte_column_window(seed, start, n):
    """Bytes [start, start + n) of a kind-0 column read as uint8: byte j is byte j & 7 of mix64(seed + (j >> 3))."""
    w0 = start >> 3
    words = window(0, seed, 0, 0, w0, ((start + n + 7) >> 3) - w0)
    return words.view(np.uint8)[start - 8 * w0:start - 8 * w0 + n]


def bits_window(seed, lo, hi, start, n):
    """Bits [start, start + n) of a kind-4 bitmap as bools, for any start."""
    s8 = start & ~7
    b = window(4, seed, lo, hi, s8, start - s8 + n)
    return np.unpackbits(b, bitorder="little")[start - s8:start - s8 + n].astype(bool)


def chunked(fn, n, chunk=CHUNK):
    """[fn(start, count) for each chunk of [0, n)], the chunks run on a thread pool (the twin releases the GIL)."""
    with ThreadPoolExecutor(WORKERS) as ex:
        return list(ex.map(lambda s: fn(s, min(chunk, n - s)), range(0, n, chunk)))


def bitmap_popcount(seed, lo, hi, off, nbits, chunk=CHUNK):
    """Set bits in [off, off + nbits) of a kind-4 bitmap."""
    def part(s, c):
        a = off + s
        s8 = a & ~7
        b = window(4, seed, lo, hi, s8, a - s8 + c)
        b[0] &= (0xFF << (a - s8)) & 0xFF
        return int(np.bitwise_count(b).sum(dtype=np.int64))
    return sum(chunked(part, nbits, chunk))


def int8_prefix(seed, n, rows, valid=None, chunk=CHUNK):
    """Wrapping int8 prefix sums (rows 0..r inclusive) of a kind-0 byte column read as int8, at each of `rows`, and
    the exact sum of the whole column.  valid = (seed, lo, hi, off): row i counts only when bit off + i of that
    kind-4 bitmap is set."""
    def vals(s, c):
        v = byte_column_window(seed, s, c).view(np.int8).astype(np.int64)
        if valid is not None:
            v *= bits_window(valid[0], valid[1], valid[2], valid[3] + s, c)
        return v
    sums = np.array(chunked(lambda s, c: int(vals(s, c).sum()), n, chunk), dtype=np.int64)
    before = np.concatenate(([0], np.cumsum(sums)))
    out = []
    for r in rows:
        c0 = (r // chunk) * chunk
        out.append(int(before[r // chunk]) + int(vals(c0, r - c0 + 1).sum()))
    return np.array(out, dtype=np.int64).astype(np.int8), int(before[-1])


def wrapping_sum(kind, seed, lo, hi, n, chunk=CHUNK):
    """Sum of a kind-1 (int64) or kind-3 (float64, integer-valued) column modulo 2^64, as an unsigned int."""
    def part(s, c):
        v = window(kind, seed, lo, hi, s, c)
        return int(v.astype(np.int64).view(np.uint64).sum(dtype=np.uint64))
    return sum(chunked(part, n, chunk)) & MASK64


def selection_counts(select, n, chunk=CHUNK):
    """Per-chunk counts of selected rows.  select(start, count) returns the packed LSB-first bitmap of rows
    [start, start + count), bits past count clear (start is a multiple of the chunk)."""
    return np.array(chunked(lambda s, c: int(np.bitwise_count(select(s, c)).sum(dtype=np.int64)), n, chunk), dtype=np.int64)


def kth_selected(select, n, counts, k, chunk=CHUNK):
    """Row of the k-th (0-based) selected row, given selection_counts(select, n, chunk)."""
    cum = np.cumsum(counts)
    c = int(np.searchsorted(cum, k, side="right"))
    s = c * chunk
    bits = np.unpackbits(select(s, min(chunk, n - s)), bitorder="little")
    return s + int(np.flatnonzero(bits)[k - int(cum[c] - counts[c])])


def mix64_np(z):
    with np.errstate(over="ignore"):    # modulo 2^64 by design
        z = np.asarray(z, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def checksum_part(words, w0):
    """ag_checksum64_dev's terms for `words` starting at word index w0, summed modulo 2^64."""
    return int((mix64_np(np.arange(w0, w0 + words.size, dtype=np.uint64)) * words.view(np.uint64)).sum(dtype=np.uint64))


def byte_words(b):
    """uint8 array -> little-endian uint64 words, zero-padded to whole words."""
    pad = np.zeros((b.size + 7) // 8 * 8, dtype=np.uint8)
    pad[:b.size] = b
    return pad.view(np.uint64)


# ---------------------------------------------------------------------------------------------------------------
# CPU tests pinning the helpers

@pytest.mark.parametrize("kind,lo,hi", [(0, 0, 0), (1, -5, 1 << 20), (1, 0, (1 << 32) - 1), (2, -(1 << 31), (1 << 31) - 1),
                                        (3, -(1 << 20), 1 << 20)])
def test_window_is_a_slice_of_one_generate_call(cpu, kind, lo, hi):
    n = 5000
    full = np.empty(n, dtype=_NP_KIND[kind])
    cpu.ref_generate(kind, 0xC0FFEE, lo, hi, full.ctypes.data, n)
    for start, cnt in ((0, n), (1, 100), (7, 9), (8, 1), (999, 4001), (n - 1, 1)):
        assert window(kind, 0xC0FFEE, lo, hi, start, cnt).tobytes() == full[start:start + cnt].tobytes(), (start, cnt)
    assert window(kind, 0xC0FFEE, lo, hi, 5, 10).tobytes() != full[4:14].tobytes()


def test_bitmap_window_at_byte_starts(cpu):
    n = 20_000
    full = np.zeros((n + 7) // 8, dtype=np.uint8)
    cpu.ref_generate(4, 0xBEEF, 3, 5, full.ctypes.data, n)
    bits = np.unpackbits(full, bitorder="little")[:n].astype(bool)
    assert 0.55 < bits.mean() < 0.65
    for start, cnt in ((0, n), (8, 13), (64, 8), (1000, 17_001), (n - 16, 16)):
        got = window(4, 0xBEEF, 3, 5, start, cnt)
        assert np.array_equal(np.unpackbits(got, bitorder="little")[:cnt].astype(bool), bits[start:start + cnt]), start
        assert not np.unpackbits(got, bitorder="little")[cnt:].any()
    for start, cnt in ((1, 100), (3, 7), (12_345, 999)):
        assert np.array_equal(bits_window(0xBEEF, 3, 5, start, cnt), bits[start:start + cnt]), start
    with pytest.raises(AssertionError):
        window(4, 0xBEEF, 3, 5, 4, 8)


def test_byte_column_window(cpu):
    words = np.empty(1000, dtype=np.uint64)
    cpu.ref_generate(0, 0xABC, 0, 0, words.ctypes.data, words.size)
    b = words.view(np.uint8)
    for start, cnt in ((0, 8000), (1, 1), (7, 2), (8, 9), (13, 6000), (7999, 1)):
        assert np.array_equal(byte_column_window(0xABC, start, cnt), b[start:start + cnt]), start
    assert not np.array_equal(byte_column_window(0xABC, 9, 100), b[8:108])


def test_chunked_reductions_match_numpy(cpu):
    n, chunk = 3_000_017, 1 << 16
    # byte popcount of a bitmap at an odd offset
    full = window(4, 0x51, 2, 7, 0, n + 11)
    bits = np.unpackbits(full, bitorder="little")[:n + 11].astype(bool)
    assert bitmap_popcount(0x51, 2, 7, 11, n, chunk) == int(bits[11:].sum())
    assert bitmap_popcount(0x51, 2, 7, 3, n - 5, chunk) == int(bits[3:n - 2].sum())
    # wrapping int8 prefix, without and with validity
    v = byte_column_window(0x52, 0, n).view(np.int8).astype(np.int64)
    vb = bits_window(0x53, 7, 8, 5, n)
    rows = [0, 1, chunk - 1, chunk, chunk + 1, 1_234_567, n - 1]
    for valid, x in ((None, v), ((0x53, 7, 8, 5), v * vb)):
        got, total = int8_prefix(0x52, n, rows, valid, chunk)
        c = np.cumsum(x)
        assert np.array_equal(got, c[rows].astype(np.int8)) and total == int(c[-1])
    # wrapping int64 sum (past 2^64) and exact float64 sum
    big = window(1, 0x54, 1 << 50, (1 << 50) + (1 << 32) - 1, 0, n)
    assert wrapping_sum(1, 0x54, 1 << 50, (1 << 50) + (1 << 32) - 1, n, chunk) == sum(int(x) for x in big) & MASK64
    f = window(3, 0x55, -(1 << 20), 1 << 20, 0, n)
    assert wrapping_sum(3, 0x55, -(1 << 20), 1 << 20, n, chunk) == int(f.sum()) & MASK64
    # the k-th selected row
    sel = lambda s, c: window(4, 0x56, 3, 5, s, c)
    counts = selection_counts(sel, n, chunk)
    where = np.flatnonzero(np.unpackbits(window(4, 0x56, 3, 5, 0, n), bitorder="little")[:n])
    assert counts.sum() == where.size
    for k in (0, 1, int(counts[0]) - 1, int(counts[0]), int(counts[:7].sum()) + 3, where.size - 1):
        assert kth_selected(sel, n, counts, k, chunk) == where[k], k


def test_checksum_part_matches_the_oracle(cpu):
    w = window(0, 0x57, 0, 0, 0, 1001)
    assert (checksum_part(w[:400], 0) + checksum_part(w[400:], 400)) & MASK64 == cpu.ref_checksum64(w.ctypes.data, w.size)
    b = w.view(np.uint8)[:8003]
    assert np.array_equal(byte_words(b)[:1000], w[:1000]) and byte_words(b)[1000] == int(w[1000]) & 0xFFFFFF


# ---------------------------------------------------------------------------------------------------------------
# device plumbing

@pytest.fixture(scope="module")
def arena(ag):
    """One device allocation that every case carves its operands from, so peak use is this plus the library's own
    scratch.  Skips the module when the device cannot hold it."""
    from arrow_go_b200.device import DeviceBuffer
    try:
        buf = DeviceBuffer(ARENA_BYTES)
    except N.NativeError as e:
        if e.status == N.AG_ERR_OOM:
            pytest.skip(f"a {ARENA_BYTES / 1e9:.1f} GB device arena does not fit: {e}")
        raise
    yield buf.ptr
    N.call("ag_stream_sync", None)
    buf.free()


def carve(base, *sizes):
    """Consecutive 256-byte aligned pointers for operands of the given byte sizes."""
    ptrs, off = [], 0
    for s in sizes:
        ptrs.append(base + off)
        off = (off + int(s) + 255) & ~255
    assert off <= ARENA_BYTES, off
    return ptrs


def gen(kind, seed, lo, hi, ptr, n):
    N.call("ag_generate_dev", kind, seed, lo, hi, ptr, n, None)


def dl(ptr, dtype, count):
    out = np.empty(count, dtype=dtype)
    N.call("ag_download", out.ctypes.data, ptr, out.nbytes, None)
    N.call("ag_stream_sync", None)
    return out


def ul(ptr, arr):
    arr = np.ascontiguousarray(arr)
    N.call("ag_upload", ptr, arr.ctypes.data, arr.nbytes, None)
    N.call("ag_stream_sync", None)


def memset(ptr, byte, nbytes):
    N.call("ag_dev_memset", ptr, byte, nbytes, None)


def word(init=0):
    return Dev(np.array([init], dtype=np.int64))


def read(w, dtype=np.int64):
    N.call("ag_stream_sync", None)
    return w.get(dtype)[0]


def dev_popcount(ptr, off, nbits):
    c = word()
    N.call("ag_bitmap_popcount_dev", ptr, off, nbits, c.ptr, None)
    return int(read(c))


def dev_checksum(ptr, n_words):
    c = word()
    N.call("ag_checksum64_dev", ptr, n_words, c.ptr, None)
    return int(read(c, np.uint64))


def assert_outside_bits_kept(ptr, off, n, canary=CANARY):
    """Bits [0, off) of the first byte and the bits past off + n up to the next 8 bytes still hold the canary."""
    head = dl(ptr, np.uint8, 1)[0]
    assert head & ((1 << off) - 1) == canary & ((1 << off) - 1)
    e = off + n
    tail = dl(ptr + e // 8, np.uint8, 8)
    keep = np.unpackbits(tail, bitorder="little")[e % 8:]
    assert np.array_equal(keep, np.unpackbits(np.full(8, canary, np.uint8), bitorder="little")[e % 8:])


def around(n):
    """Starts of the checked windows: row 0, around 2^31, around 2^32 (when n is past it) and the end."""
    starts = [0, (1 << 31) - W // 2]
    if n > (1 << 32) + W:
        starts.append((1 << 32) - W // 2)
    return starts + [n - W]


def words8(n):
    return (n + 7) // 8


GPU = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------
# 1. compare: uint8 GT / LE against a scalar, past 2^32 rows, output at bit offset 5

@GPU
@pytest.mark.timeout(600)
def test_compare_u8_past_2_32_rows(arena, cpu):
    n, off, seed = (1 << 32) + (1 << 20) + 37, 5, 0x1001
    s = np.array([100], dtype=np.uint8)
    nbm = (off + n + 7) // 8 + 8
    vals, gt, le = carve(arena, words8(n) * 8, nbm, nbm)
    gen(0, seed, 0, 0, vals, words8(n))
    for out, cmp in ((gt, N.CMP_GT), (le, N.CMP_LE)):
        memset(out, CANARY, nbm)
        N.call("ag_compare_dev", N.UINT8, cmp, N.SHAPE_AS, vals, s.ctypes.data, out, n, off, None)
    n_gt, n_le = dev_popcount(gt, off, n), dev_popcount(le, off, n)
    assert n_gt + n_le == n
    assert n_gt == sum(chunked(lambda a, c: int(np.count_nonzero(byte_column_window(seed, a, c) > s[0])), n))
    for out, cmp in ((gt, N.CMP_GT), (le, N.CMP_LE)):
        assert_outside_bits_kept(out, off, n)
        for r0 in around(n):
            a = off + r0
            got = dl(out + a // 8, np.uint8, (a % 8 + W + 7) // 8)
            want = got.copy()
            v = byte_column_window(seed, r0, W)
            assert cpu.ref_compare(N.UINT8, cmp, N.SHAPE_AS, v.ctypes.data, s.ctypes.data, want.ctypes.data, W, a % 8) == 0
            assert np.array_equal(got, want), (cmp, r0)


# ---------------------------------------------------------------------------------------------------------------
# 2. bitmap ops, copy, invert and popcount over 2^32 + 2^16 + 29 bits, an odd offset on every operand

@GPU
@pytest.mark.timeout(600)
def test_bitmap_ops_past_2_32_bits(arena, cpu):
    nbits, loff, roff, ooff = (1 << 32) + (1 << 16) + 29, 3, 5, 7
    L, R = (0x2001, 1, 2), (0x2002, 2, 3)            # (seed, lo, hi): P(bit) = 1/2 and 2/3
    nb = (nbits + 8 + 7) // 8 + 8
    lp, rp, op = carve(arena, nb, nb, nb)
    gen(4, *L, lp, loff + nbits)
    gen(4, *R, rp, roff + nbits)
    pl, pr = dev_popcount(lp, loff, nbits), dev_popcount(rp, roff, nbits)
    assert pl == bitmap_popcount(*L, loff, nbits)
    assert pr == bitmap_popcount(*R, roff, nbits)

    def src(spec, off, j0, w):
        a = off + j0
        return window(4, *spec, a & ~7, a % 8 + w), a % 8

    def check(name, ref_call):
        assert_outside_bits_kept(op, ooff, nbits)
        for j0, w in (((1 << 32) - 64, 128), ((1 << 32) - W // 2, nbits - ((1 << 32) - W // 2)), ((1 << 31) - W // 2, W), (nbits - W, W)):
            a = ooff + j0
            got = dl(op + a // 8, np.uint8, (a % 8 + w + 7) // 8)
            want = got.copy()
            ref_call(j0, w, want, a % 8)
            assert np.array_equal(got, want), (name, j0)

    pc = {}
    for bop in (N.BITOP_AND, N.BITOP_OR, N.BITOP_XOR, N.BITOP_ANDNOT, N.BITOP_XNOR):
        memset(op, CANARY, nb)
        N.call("ag_bitmap_op_dev", bop, lp, loff, rp, roff, op, ooff, nbits, None)
        pc[bop] = dev_popcount(op, ooff, nbits)

        def ref_op(j0, w, want, osub, bop=bop):
            (lb, ls), (rb, rs) = src(L, loff, j0, w), src(R, roff, j0, w)
            assert cpu.ref_bitmap_op(bop, lb.ctypes.data, ls, rb.ctypes.data, rs, want.ctypes.data, osub, w) == 0
        check(bop, ref_op)
    assert pc[N.BITOP_AND] + pc[N.BITOP_ANDNOT] == pl
    assert pc[N.BITOP_OR] + pc[N.BITOP_AND] == pl + pr
    assert pc[N.BITOP_XOR] == pc[N.BITOP_OR] - pc[N.BITOP_AND]
    assert pc[N.BITOP_XNOR] == nbits - pc[N.BITOP_XOR]

    for name, fn, ref_fn, want_pc in (("copy", "ag_bitmap_copy_dev", cpu.ref_bitmap_copy, pl),
                                      ("invert", "ag_bitmap_invert_dev", cpu.ref_bitmap_invert, nbits - pl)):
        memset(op, CANARY, nb)
        N.call(fn, lp, loff, nbits, op, ooff, None)
        assert dev_popcount(op, ooff, nbits) == want_pc, name

        def ref_one(j0, w, want, osub, ref_fn=ref_fn):
            lb, ls = src(L, loff, j0, w)
            ref_fn(lb.ctypes.data, ls, w, want.ctypes.data, osub)
        check(name, ref_one)


# ---------------------------------------------------------------------------------------------------------------
# 3. filter with EMIT_NULLS: more than 2^32 rows in, more than 2^32 rows out

@GPU
@pytest.mark.timeout(900)
def test_filter_u8_emit_nulls_past_2_32_output_rows(arena):
    n, vseed = (1 << 32) + (1 << 20) + 37, 0x3001
    M = (0x3002, (1 << 14) - 1, 1 << 14)               # mask: P(set) = 1 - 2^-14
    V = (0x3003, 15, 16)                                # mask validity: 1 in 16 slots null
    nbm = (n + 7) // 8 + 8
    vals, mask, mvalid, out, ovalid = carve(arena, words8(n) * 8, nbm, nbm, n + 64, (n + 31) // 32 * 4 + 64)
    gen(0, vseed, 0, 0, vals, words8(n))
    gen(4, *M, mask, n)
    gen(4, *V, mvalid, n)

    def emitted(s, c):   # a null mask slot is emitted (as a null row) as well as a set, valid one
        return window(4, *M, s, c) | ~window(4, *V, s, c) & np.packbits(np.ones(c, bool), bitorder="little")
    counts = selection_counts(emitted, n)
    total = int(counts.sum())
    assert total > (1 << 32)

    ln = word(-1)
    N.call("ag_filter_output_size_dev", mask, mvalid, 0, n, N.EMIT_NULLS, ln.ptr, None)
    assert read(ln) == total
    N.call("ag_filter_primitive_dev", 8, vals, None, 0, mask, mvalid, 0, n, N.EMIT_NULLS, out, ovalid, total, ln.ptr, None)
    assert read(ln) == total

    for p0 in (0, (1 << 31) - W // 2, (1 << 32) - W // 2, total - W):
        first = kth_selected(emitted, n, counts, p0)      # the row that lands at output position p0
        r0 = first & ~7
        span = min(2 * W, n - r0)
        rows = r0 + np.flatnonzero(np.unpackbits(emitted(r0, span), bitorder="little")[:span])
        rows = rows[rows >= first][:W]
        assert rows.size == W
        ok = bits_window(V[0], V[1], V[2], r0, span)[rows - r0]
        want = np.where(ok, byte_column_window(vseed, r0, span)[rows - r0], 0).astype(np.uint8)
        got = dl(out + p0, np.uint8, W)
        assert np.array_equal(got, want), p0
        gv = np.unpackbits(dl(ovalid + p0 // 8, np.uint8, W // 8 + 1), bitorder="little")[p0 % 8:p0 % 8 + W].astype(bool)
        assert np.array_equal(gv, ok), p0


# ---------------------------------------------------------------------------------------------------------------
# 4. fused compare + filter (int32, 2^31 + 2^20 + 37 rows) against compare then filter

@GPU
@pytest.mark.timeout(600)
def test_fused_compare_filter_i32_past_2_31_rows(arena):
    n, seed, lo, hi = (1 << 31) + (1 << 20) + 37, 0x4001, -(1 << 31), (1 << 31) - 1
    s = np.array([hi - 429_496_730], dtype=np.int32)  # about 10 % of the rows are greater
    sel = lambda a, c: np.packbits(window(2, seed, lo, hi, a, c) > s[0], bitorder="little")
    counts = selection_counts(sel, n)
    total = int(counts.sum())
    cap_bytes = (total * 4 + 7) // 8 * 8
    vals, mask, out1, out2 = carve(arena, n * 4, (n + 7) // 8 + 8, cap_bytes, cap_bytes)
    gen(2, seed, lo, hi, vals, n)
    memset(out1, 0, cap_bytes)
    memset(out2, 0, cap_bytes)
    N.call("ag_compare_dev", N.INT32, N.CMP_GT, N.SHAPE_AS, vals, s.ctypes.data, mask, n, 0, None)
    la, lb, lc = word(-1), word(-1), word(-1)
    N.call("ag_filter_output_size_dev", mask, None, 0, n, N.DROP_NULLS, la.ptr, None)
    N.call("ag_filter_primitive_dev", 32, vals, None, 0, mask, None, 0, n, N.DROP_NULLS, out2, None, total, lb.ptr, None)
    N.call("ag_filter_compare_scalar_dev", N.INT32, N.CMP_GT, vals, s.ctypes.data, n, out1, total, lc.ptr, None)
    assert read(la) == read(lb) == read(lc) == total
    assert dev_checksum(out1, cap_bytes // 8) == dev_checksum(out2, cap_bytes // 8)
    r = kth_selected(sel, n, counts, total - W)
    v = window(2, seed, lo, hi, r, n - r)
    assert np.array_equal(dl(out1 + 4 * (total - W), np.int32, W), v[v > s[0]])


# ---------------------------------------------------------------------------------------------------------------
# 5. take_indices: uint32 row positions up to 2^32 - 3, and the 2^32 - 1 row limit

@GPU
@pytest.mark.timeout(600)
def test_take_indices_u32_positions_past_2_31(arena):
    n, M = (1 << 32) - 2, (0x5001, 1, 1024)           # about 4M rows selected
    want = np.concatenate(chunked(lambda s, c: s + np.flatnonzero(np.unpackbits(window(4, *M, s, c), bitorder="little")[:c]), n))
    want = np.union1d(want, [n - 1]).astype(np.uint64)
    mask, out = carve(arena, (1 << 29) + 64, want.size * 4 + 64)
    gen(4, *M, mask, n)
    last = dl(mask + (n - 1) // 8, np.uint8, 1)
    last[0] |= 1 << ((n - 1) % 8)                      # the last row is selected too
    ul(mask + (n - 1) // 8, last)
    ln = word(-1)
    N.call("ag_take_indices_dev", 32, mask, None, 0, n, N.DROP_NULLS, out, None, want.size, ln.ptr, None)
    assert read(ln) == want.size
    got = dl(out, np.uint32, want.size).astype(np.uint64)
    assert np.count_nonzero(got > (1 << 31)) > want.size // 3
    assert got[-1] == n - 1
    assert np.array_equal(got, want)

    memset(out, CANARY, 64)
    ln = word(-7)
    st, msg = N.call_status("ag_take_indices_dev", 32, mask, None, 0, n + 1, N.DROP_NULLS, out, None, want.size, ln.ptr, None)
    assert st == N.AG_ERR_NOT_IMPLEMENTED, msg
    assert read(ln) == -7
    assert (dl(out, np.uint8, 64) == CANARY).all()


# ---------------------------------------------------------------------------------------------------------------
# 6. take from a uint8 table of 2^32 + 2^22 rows: direct, forced windowed and automatic routing

@pytest.fixture
def take_policy(ag):
    yield ag
    ag.call("ag_take_set_policy", *SHIPPED_TAKE_POLICY)


@GPU
@pytest.mark.timeout(900)
def test_take_into_table_past_2_32_rows(arena, take_policy):
    ag = take_policy
    vlen, tseed = (1 << 32) + (1 << 22), 0x6001
    n = (1 << 29) + (1 << 19) + 37                     # n * 8 >= vlen: the automatic policy routes to the windowed path
    h = n // 2
    I1 = (0x6002, 0, (1 << 32) - 1)                    # rows [0, h)
    I2 = (0x6003, 1 << 22, (1 << 32) + (1 << 22) - 1)  # rows [h, n)
    table, idx, out = carve(arena, words8(vlen) * 8, n * 8, n + 64)
    gen(0, tseed, 0, 0, table, words8(vlen))
    gen(1, *I1, idx, h)
    gen(1, *I2, idx + 8 * h, n - h)
    planted = {}

    def table_bytes(v):
        v = np.asarray(v, dtype=np.uint64)
        return ((mix64_np(np.uint64(tseed) + (v >> np.uint64(3))) >> ((v & np.uint64(7)) * np.uint64(8))) & np.uint64(0xFF)).astype(np.uint8)

    def idx_window(s, c):
        a = window(1, *I1, s, max(0, min(h, s + c) - s))
        b = window(1, *I2, max(s, h) - h, max(0, s + c - max(s, h)))
        v = np.concatenate((a, b))
        for r, x in planted.items():
            if s <= r < s + c:
                v[r - s] = x
        return v

    # in-range indices past 2^32 whose low 32 bits point at a row holding a different byte
    hi_idx = [v for v in range((1 << 32) + (1 << 21), (1 << 32) + (1 << 21) + 64)
              if table_bytes(v) != table_bytes(v & 0xFFFFFFFF)][:8]
    assert len(hi_idx) == 8
    for r, v in zip((5, (1 << 28) + 1, h + 12_345, n - 1), hi_idx):
        planted[r] = v
    # out of range, though their low 32 bits are in range; and one negative index
    bad_rows = {(1 << 27) + 11: -1, 3 * (1 << 26) + 7: vlen, (1 << 28) + 77: vlen + 5, 500_000_000: (1 << 32) + vlen}
    for r, v in list(planted.items()) + list(bad_rows.items()):
        ul(idx + 8 * r, np.array([v], dtype=np.int64))

    policies = {"direct": (1, 0, 0, 0), "windowed": (2, 0, 0, 8 << 20), "automatic": SHIPPED_TAKE_POLICY}
    bad = word()

    def run(policy, iptr, iw, signed, count):
        ag.call("ag_take_set_policy", *policies[policy])
        ag.call("ag_error_word_reset_dev", bad.ptr, None)
        memset(out, 0, count + 64)
        ag.call("ag_take_primitive_dev", 8, table, None, 0, vlen, iw, signed, iptr, None, 0, count, 1, out, None, bad.ptr, None)
        return int(read(bad))

    # the first offender is reported by every policy; then it is replaced by an in-range index past 2^32
    for r in sorted(bad_rows):
        for policy in policies:
            assert run(policy, idx, 64, 1, n) == r, (policy, r)
        planted[r] = hi_idx[len(planted)]
        ul(idx + 8 * r, np.array([planted[r]], dtype=np.int64))

    def host_checksum(s, c):   # chunks start on a multiple of 8 rows
        return checksum_part(byte_words(table_bytes(idx_window(s, c))), s // 8)
    want_sum = sum(chunked(host_checksum, n, CHUNK // 4)) & MASK64
    starts = [0, 1 << 28, n - W] + [max(0, r - 3) for r in planted]
    for policy in policies:
        assert run(policy, idx, 64, 1, n) == N.NO_ERROR_POS, policy
        assert dev_checksum(out, words8(n)) == want_sum, policy
        for r0 in starts:
            c = min(W, n - r0)
            assert np.array_equal(dl(out + r0, np.uint8, c), table_bytes(idx_window(r0, c))), (policy, r0)
        for r, v in planted.items():
            assert dl(out + r, np.uint8, 1)[0] == table_bytes(v) != table_bytes(v & 0xFFFFFFFF), (policy, r)

    # uint32 indices into the same table: every one is in range (the all_fit side of the partition pass)
    n32, I3 = (1 << 28) + 37, (0x6004, -(1 << 31), (1 << 31) - 1)
    gen(2, *I3, idx, n32)
    sums = []
    for policy in ("windowed", "direct"):
        assert run(policy, idx, 32, 0, n32) == N.NO_ERROR_POS, policy
        sums.append(dev_checksum(out, words8(n32)))
        for r0 in (0, 1 << 27, n32 - W):
            v = window(2, *I3, r0, W).view(np.uint32)
            assert np.array_equal(dl(out + r0, np.uint8, W), table_bytes(v)), (policy, r0)
    assert sums[0] == sums[1]


# ---------------------------------------------------------------------------------------------------------------
# 7. cumulative_sum over int8, past 2^32 rows, without and with validity (skip_nulls)

@GPU
@pytest.mark.timeout(900)
def test_cumsum_i8_past_2_32_rows(arena):
    n, seed, voff, ooff = (1 << 32) + (1 << 20) + 13, 0x7001, 3, 5
    V = (0x7002, 7, 8)                                 # 1 in 8 rows null
    nbm = (n + 8 + 7) // 8 + 8
    inp, out, valid, ovalid = carve(arena, words8(n) * 8, n + 64, nbm, nbm)
    gen(0, seed, 0, 0, inp, words8(n))
    gen(4, *V, valid, voff + n)
    state = Dev(np.zeros(4, dtype=np.int64))
    starts = around(n)

    for with_valid in (False, True):
        spec = (*V, voff) if with_valid else None
        pref, total = int8_prefix(seed, n, [r0 - 1 for r0 in starts if r0 > 0], spec)
        bases = dict(zip([r0 for r0 in starts if r0 > 0], pref.astype(np.int64)))
        memset(ovalid, CANARY, nbm)
        N.call("ag_cumulative_sum_state_init_dev", state.ptr, N.INT8, None, None)
        N.call("ag_cumulative_sum_dev", N.INT8, inp, valid if with_valid else None, voff if with_valid else 0, n, 1, 0, out,
               ovalid if with_valid else None, ooff, state.ptr, None, None)
        N.call("ag_stream_sync", None)
        st = state.get()
        nulls = n - bitmap_popcount(*V, voff, n) if with_valid else 0
        assert int(st[0]) == total and int(st[3]) == nulls, (with_valid, st)
        for r0 in starts:
            x = byte_column_window(seed, r0, W).view(np.int8).astype(np.int64)
            ok = bits_window(*V, voff + r0, W) if with_valid else np.ones(W, bool)
            want = np.where(ok, (bases.get(r0, 0) + np.cumsum(x * ok)).astype(np.int8), 0).astype(np.int8)
            assert np.array_equal(dl(out + r0, np.int8, W), want), (with_valid, r0)
            if with_valid:
                a = ooff + r0
                gv = np.unpackbits(dl(ovalid + a // 8, np.uint8, W // 8 + 1), bitorder="little")[a % 8:a % 8 + W].astype(bool)
                assert np.array_equal(gv, ok), r0
        if with_valid:
            assert_outside_bits_kept(ovalid, ooff, n)


# ---------------------------------------------------------------------------------------------------------------
# 8. Sum over 2^31 + 2^16 + 3 int64 / uint64 / float64 values

@GPU
@pytest.mark.timeout(900)
def test_sum_past_2_31_rows(arena):
    n, k = (1 << 31) + (1 << 16) + 3, (1 << 31) - 1
    buf = carve(arena, n * 8)[0]
    res = Dev(np.zeros(3, dtype=np.uint64))
    for fn, kind, spec, dt in (("ag_sum_i64_dev", 1, (0x8001, -(1 << 31), (1 << 31) - 1), np.int64),
                               ("ag_sum_u64_dev", 1, (0x8002, 1 << 40, (1 << 40) + (1 << 32) - 1), np.uint64),
                               ("ag_sum_f64_dev", 3, (0x8003, -(1 << 20), 1 << 20), np.float64)):
        gen(kind, *spec, buf, n)
        N.call(fn, buf, n, res.ptr, None)
        N.call(fn, buf, k, res.ptr + 8, None)
        N.call(fn, buf + 8 * k, n - k, res.ptr + 16, None)
        N.call("ag_stream_sync", None)
        whole, head, tail = res.get(dt)[:3]
        want = wrapping_sum(kind, *spec, n)
        if dt is np.float64:
            assert float(whole) == float(want - (1 << 64) if want >> 63 else want), fn    # every partial sum is an exact integer
            assert head + tail == whole, fn
        else:
            assert int(np.array(whole, dt).view(np.uint64)) == want, fn
            assert (int(np.array(head, dt).view(np.uint64)) + int(np.array(tail, dt).view(np.uint64))) & MASK64 == want, fn


# ---------------------------------------------------------------------------------------------------------------
# 9. min_max over int8 / uint8 past 2^32 rows, the extremes planted past 2^32

@GPU
@pytest.mark.timeout(600)
def test_min_max_8bit_past_2_32_rows(arena):
    n = (1 << 32) + (1 << 20) + 5
    vals = carve(arena, n + 64)[0]
    mm = Dev(np.zeros(8, dtype=np.uint8))
    for t, dt in ((N.INT8, np.int8), (N.UINT8, np.uint8)):
        # int32 values 0x30303030 .. 0x3030303F read as bytes: every byte in [0x30, 0x3F]
        gen(2, 0x9001, 0x30303030, 0x3030303F, vals, (n + 3) // 4)
        N.call("ag_min_max_dev", t, vals, n, mm.ptr, None)
        N.call("ag_stream_sync", None)
        assert list(mm.get(dt)[:2]) == [0x30, 0x3F], t
        info = np.iinfo(dt)
        ul(vals + (1 << 32) + 3, np.array([info.min], dtype=dt))
        ul(vals + n - 1, np.array([info.max], dtype=dt))
        N.call("ag_min_max_dev", t, vals, n, mm.ptr, None)
        N.call("ag_stream_sync", None)
        assert list(mm.get(dt)[:2]) == [info.min, info.max], t
        N.call("ag_min_max_dev", t, vals, n - 1, mm.ptr, None)          # without the last row: the maximum is gone
        N.call("ag_stream_sync", None)
        assert list(mm.get(dt)[:2]) == [info.min, 0x3F], t


# ---------------------------------------------------------------------------------------------------------------
# 10. arith (chunked spans), cast and is_in over one uint8 column of more than 2^32 rows

@GPU
@pytest.mark.timeout(900)
def test_arith_cast_is_in_u8_past_2_32_rows(arena, cpu):
    n, seed = (1 << 32) + (1 << 20) + 13, 0xA001
    col, out, bits = carve(arena, words8(n) * 8, words8(n) * 8, (n + 31) // 32 * 4 + 64)
    gen(0, seed, 0, 0, col, words8(n))
    full_words = n // 8
    col_sum = dev_checksum(col, full_words)

    # ADD with shape AS over three spans, one of them longer than 2^32 rows
    s = np.array([77], dtype=np.uint8)
    l1, l2 = (1 << 32) + (1 << 19) + 1, 1000
    cuts = [0, l1, l1 + l2, n]
    spans = N.span_table([(col + a, s.ctypes.data, out + a, b - a) for a, b in zip(cuts, cuts[1:])])
    N.call("ag_arith_binary_spans_dev", N.UINT8, N.OP_ADD, N.SHAPE_AS, spans, 3, None)
    for r0 in around(n) + [l1 - W // 2, l1 + l2 - W // 4]:          # the last two windows cross the span boundaries
        w = min(W, n - r0)
        v = byte_column_window(seed, r0, w)
        want = np.empty(w, dtype=np.uint8)
        assert cpu.ref_arith_binary(N.UINT8, N.OP_ADD, N.SHAPE_AS, v.ctypes.data, s.ctypes.data, want.ctypes.data, w) == 0
        assert np.array_equal(dl(out + r0, np.uint8, w), want), r0
    N.call("ag_arith_binary_dev", N.UINT8, N.OP_SUB, N.SHAPE_AS, out, s.ctypes.data, out, n, None)
    assert dev_checksum(out, full_words) == col_sum
    assert np.array_equal(dl(out + 8 * full_words, np.uint8, n % 8), byte_column_window(seed, 8 * full_words, n % 8))

    # cast uint8 -> int8
    memset(out, 0, words8(n) * 8)
    N.call("ag_cast_numeric_dev", N.UINT8, N.INT8, col, out, n, None)
    assert dev_checksum(out, full_words) == col_sum
    for r0 in around(n):
        v = byte_column_window(seed, r0, W)
        want, fb = np.empty(W, dtype=np.int8), C.c_int64()
        assert cpu.ref_cast_numeric(N.UINT8, N.INT8, v.ctypes.data, None, 0, want.ctypes.data, W, 1, 1, C.byref(fb)) == 0
        assert np.array_equal(dl(out + r0, np.int8, W), want), r0

    # is_in against a 40-value set: the 256-bit membership bitmap path
    vset = np.random.default_rng(0xA002).choice(256, 40, replace=False).astype(np.uint8)
    dset = Dev(vset)
    N.call("ag_is_in_dev", 8, col, None, 0, n, dset.ptr, None, 0, vset.size, 0, bits, None, None, None)
    lut = np.zeros(256, dtype=np.int64)
    lut[vset] = 1
    assert dev_popcount(bits, 0, n) == sum(chunked(lambda a, c: int(lut[byte_column_window(seed, a, c)].sum()), n))
    for r0 in [r & ~31 for r in around(n)]:
        w = min(W + 32, n - r0)
        v = byte_column_window(seed, r0, w)
        want, wv, nn = np.zeros(w // 8 + 1, np.uint8), np.zeros(w // 8 + 1, np.uint8), C.c_int64()
        assert cpu.ref_is_in(8, v.ctypes.data, None, 0, w, vset.ctypes.data, None, 0, vset.size, 0, want.ctypes.data, wv.ctypes.data,
                             C.byref(nn)) == 0
        got = np.unpackbits(dl(bits + r0 // 8, np.uint8, w // 8 + 1), bitorder="little")[:w]
        assert np.array_equal(got, np.unpackbits(want, bitorder="little")[:w]), r0


# ---------------------------------------------------------------------------------------------------------------
# 11. documented row limits: unique and dictionary_encode refuse 2^31 rows and write nothing

@GPU
@pytest.mark.timeout(300)
def test_unique_and_dictionary_encode_refuse_2_31_rows(arena):
    n = 1 << 31
    vals, outp = carve(arena, n, n)
    gen(0, 0xB001, 0, 0, vals, n // 8)
    ln = word(-7)
    st, msg = N.call_status("ag_unique_dev", 8, vals, None, 0, n, outp, None, n, ln.ptr, None)
    assert st == N.AG_ERR_NOT_IMPLEMENTED, msg
    assert read(ln) == -7

    half = n // 2                                      # two chunks over the same 1 GB of values
    vals, idx, dct = carve(arena, half, half * 4, n)
    counts = Dev(np.full(4, -7, dtype=np.int64))
    chunks = N.dict_chunk_table([(vals, None, 0, half, idx, None), (vals, None, 0, half, idx, None)])
    st, msg = N.call_status("ag_dictionary_encode_dev", 8, chunks, 2, N.NULL_ENCODING_MASK, dct, None, counts.ptr, None)
    assert st == N.AG_ERR_NOT_IMPLEMENTED, msg
    N.call("ag_stream_sync", None)
    assert (counts.get() == -7).all()
