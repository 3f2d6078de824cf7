"""float32 / float64 cumulative_sum on the device against the scan model (tests/cumsum_float_ref.py): the outputs and
the carried state (state.lo) bit for bit, except that a NaN equals any NaN (the device returns a canonical NaN);
validity and null counts against oracle/cpu_ref.c.  Sizes around the lane, warp segment, tile, group and super-group
edges; general, ill-conditioned, subnormal, overflowing, signed-zero and non-finite data; nulls, starts, both
flavours, element-aligned operands and chunked sequences."""
import ctypes as C

import numpy as np
import pytest

import cumsum_float_ref as M
from arrow_go_b200 import _native as N
from helpers import Dev, oracle_cumsum, pack_bits, ptr, unpack_bits
from sum_f64_ref import gensum

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float64]
DT_IDS = ["float32", "float64"]
TYPE_OF = {np.float32: N.FLOAT32, np.float64: N.FLOAT64}
STARTS = [None, 5.0, -0.0, np.inf]


def same(a, b):
    """Bit-exact, except that a NaN equals any NaN."""
    a, b = np.atleast_1d(np.asarray(a)), np.atleast_1d(np.asarray(b))
    na, nb = np.isnan(a), np.isnan(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


def first_diff(a, b):
    """(the first three rows that differ, with both values; how many differ)"""
    u = np.dtype(f"u{a.itemsize}")
    na, nb = np.isnan(a), np.isnan(b)
    bad = np.flatnonzero((na != nb) | (~na & ~nb & (a.view(u) != b.view(u))))
    return [(int(i), a[i], b[i]) for i in bad[:3]], bad.size


def run_dev(ag, chunks, valids, skip, start, in_off=0, out_off=0, voff=3):
    """ag_cumulative_sum_dev over the chunks of one sequence on one device state; the input of every chunk sits
    in_off elements and the output out_off elements past an aligned allocation.  (values, state value, output
    validity, null count)."""
    dt = chunks[0].dtype
    t, isz = TYPE_OF[dt.type], dt.itemsize
    total = sum(len(c) for c in chunks)
    valids = valids if valids is not None else [None] * len(chunks)
    state = Dev(np.zeros(4, dtype=np.int64))
    sv = np.array([start], dtype=dt) if start is not None else None
    ag.call("ag_cumulative_sum_state_init_dev", state.ptr, t, ptr(sv), None)
    dout = Dev(np.zeros(out_off + total + 8, dtype=dt))
    dov = Dev(np.zeros((total + 7) // 8 + 8, dtype=np.uint8)) if any(v is not None for v in valids) else None
    keep, pos = [], 0
    for x, v in zip(chunks, valids):
        dx = Dev(np.concatenate([np.zeros(in_off, dtype=dt), x]) if len(x) + in_off else np.zeros(1, dtype=dt))
        dv = Dev(pack_bits(v, offset=voff)) if v is not None else None
        keep += [dx, dv]
        ag.call("ag_cumulative_sum_dev", t, dx.ptr + in_off * isz, dv.ptr if dv else None, voff, len(x), int(skip), 0,
                dout.ptr + (out_off + pos) * isz, dov.ptr if dov else None, pos, state.ptr, None, None)
        pos += len(x)
    ag.call("ag_stream_sync", None)
    st = state.get()
    lo = np.array([st[0]], dtype=np.int64).view(np.uint64)
    value = lo.view(np.float64)[0] if dt == np.float64 else lo.astype(np.uint32).view(np.float32)[0]
    valid = unpack_bits(dov.get(), 0, total).astype(bool) if dov else np.ones(total, dtype=bool)
    return dout.get()[out_off:out_off + total], value, valid, int(st[3])


def run_host(ag, x, valid, skip, start, voff=5):
    """ag_cumulative_sum (host pointers, one call): (values, output validity, null count)."""
    dt = x.dtype
    n = len(x)
    out = np.zeros(n, dtype=dt)
    ov = np.zeros((n + 7) // 8 + 1, dtype=np.uint8)
    bm = pack_bits(valid, offset=voff) if valid is not None else None
    sv = np.array([start], dtype=dt) if start is not None else None
    nulls, bad = C.c_int64(-1), C.c_int64(-1)
    ag.call("ag_cumulative_sum", TYPE_OF[dt.type], ptr(x), ptr(bm), voff, n, ptr(sv), int(skip), 0, ptr(out), ptr(ov),
            C.byref(nulls), C.byref(bad))
    return out, unpack_bits(ov, 0, n).astype(bool), nulls.value


def check(ag, cpu, chunks, valids, skip, start, where, via="dev", **layout):
    """One call (or chunked sequence) against the model and the oracle; returns the device's values."""
    want, wstate = M.cumulative_sum(chunks, valids, skip, start)
    _, wv, wn, _ = oracle_cumsum(cpu, chunks, valids, skip, start)
    if via == "host":
        assert len(chunks) == 1
        out, v, nulls = run_host(ag, chunks[0], valids[0] if valids else None, skip, start)
    else:
        out, state, v, nulls = run_dev(ag, chunks, valids, skip, start, **layout)
        assert same(state, wstate), (where, "state", state, wstate)
    assert same(out, want), (where, first_diff(out, want))
    if valids is not None and any(x is not None for x in valids):
        assert np.array_equal(v, wv) and nulls == wn, (where, "validity")
    return out


# ---- data -------------------------------------------------------------------------------------------------------
def data(kind, dt, n, rng):
    dt = np.dtype(dt)
    fi = np.finfo(dt)
    if kind == "normal":
        return rng.standard_normal(n).astype(dt)
    if kind == "wide":      # exponents over most of the range, mixed signs
        emax = 100 if dt == np.float32 else 900
        return (rng.choice([-1.0, 1.0], n) * (1 + rng.random(n)) * 2.0 ** rng.integers(-emax, emax // 8, n)).astype(np.float64).astype(dt)
    if kind in ("gensum8", "gensum32"):
        return gensum(n, 1e8 if kind == "gensum8" else 1e32, 7).astype(dt)
    if kind == "subnormal":  # subnormals and the smallest normals: their sums cross the normal boundary
        k = rng.integers(-(1 << 20), 1 << 20, n).astype(np.float64)
        return (k * float(fi.smallest_subnormal)).astype(dt)
    if kind == "overflow":  # near the top of the range: partial sums overflow to +inf and -inf, and meet as NaN
        return (rng.choice([-1.0, 1.0, 1.0], n) * float(fi.max) * (0.25 + 0.5 * rng.random(n))).astype(dt)
    if kind == "negzero":
        return np.full(n, -0.0, dtype=dt)
    if kind == "mixedzero":
        return np.where(rng.random(n) < 0.7, -0.0, 0.0).astype(dt)
    if kind == "nonfinite":  # ±inf and NaN at tile edges and on both sides of the group boundaries
        tile, seg, e = M.geometry(dt)
        x = rng.standard_normal(n).astype(dt)
        spots = [e - 1, seg, tile - 1, tile, 3 * tile + 1, 128 * tile - 1, 128 * tile, 256 * tile + 2]
        vals = [np.inf, -np.inf, np.inf, np.nan, -np.inf, np.inf, -np.inf, np.nan]
        for p, v in zip(spots, vals):
            if p < n and (p > n // 2 or rng.random() < 0.5):
                x[p] = v
        return x
    raise ValueError(kind)


KINDS = ["normal", "wide", "gensum8", "gensum32", "subnormal", "overflow", "negzero", "mixedzero", "nonfinite"]


def sizes(dt):
    tile, seg, e = M.geometry(dt)
    other = M.geometry(np.float64 if dt == np.float32 else np.float32)[0]
    return [1, 2, e - 1, e + 1, seg - 1, seg + 1, tile - 1, tile, tile + 1, other - 1, other + 1,
            127 * tile + 301, 128 * tile + 5, (2 * 128 + 3) * tile]


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_cumulative_sum_sizes_data_starts(ag, cpu, dt, kind):
    rng = np.random.default_rng(100 * KINDS.index(kind) + np.dtype(dt).itemsize)
    for i, n in enumerate(sizes(dt)):
        x = data(kind, dt, n, rng)
        start = STARTS[i % len(STARTS)]
        if kind in ("negzero", "mixedzero"):
            start = [-0.0, None, 0.0, -0.0][i % 4]
        check(ag, cpu, [x], None, False, start, (kind, n, start))


# ---- validity ---------------------------------------------------------------------------------------------------
def validity(mode, dt, n, rng):
    tile, _, _ = M.geometry(dt)
    if mode in ("sparse_skip", "sparse"):
        return rng.random(n) > 0.02
    if mode == "early_null":  # no skip: the sequence dies inside the first tile
        v = np.ones(n, dtype=bool)
        v[min(n - 1, 1000)] = False
        return v
    if mode == "null_tiles":  # whole tiles null, and a tile that is null but for one row
        v = rng.random(n) > 0.001
        v[tile:2 * tile] = False
        v[3 * tile:4 * tile] = False
        v[3 * tile + 77:3 * tile + 78] = True
        return v
    raise ValueError(mode)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("mode", ["sparse_skip", "sparse", "early_null", "null_tiles"])
def test_gpu_cumulative_sum_validity(ag, cpu, dt, mode):
    rng = np.random.default_rng(300)
    tile, _, _ = M.geometry(dt)
    skip = mode in ("sparse_skip", "null_tiles")
    for n in (tile + 1, 4 * tile + 77, 129 * tile + 5):
        for kind, start in (("normal", 5.0), ("mixedzero", -0.0)):
            x = data(kind, dt, n, rng)
            v = validity(mode, dt, n, rng)
            for voff in (0, 5):   # bitmap offset
                check(ag, cpu, [x], [v], skip, start, (mode, n, kind, voff), voff=voff)
            check(ag, cpu, [x], [v], skip, start, (mode, n, kind, "host"), via="host")


# ---- layouts ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_gpu_cumulative_sum_element_aligned_operands_give_aligned_bits(ag, cpu, dt):
    """Inputs and outputs 1-3 elements past a 16-byte boundary (cp.async pieces, piece stores) and the host flavour
    give the aligned path's bits."""
    rng = np.random.default_rng(400)
    tile, _, _ = M.geometry(dt)
    for n in (tile - 1, 3 * tile + 77, 128 * tile + 5):
        x = data("normal", dt, n, rng)
        for valid, skip in ((None, False), (rng.random(n) > 0.01, True)):
            vs = [valid]
            aligned = check(ag, cpu, [x], vs, skip, 5.0, (n, "aligned"))
            for off in (1, 2, 3):
                got = check(ag, cpu, [x], vs, skip, 5.0, (n, "in", off), in_off=off)
                assert got.tobytes() == aligned.tobytes()
                got = check(ag, cpu, [x], vs, skip, 5.0, (n, "out", off), out_off=off)
                assert got.tobytes() == aligned.tobytes()
            got = check(ag, cpu, [x], vs, skip, 5.0, (n, "host"), via="host")
            assert got.tobytes() == aligned.tobytes()


# ---- chunked sequences ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_gpu_cumulative_sum_chunked_sequences(ag, cpu, dt):
    """Several calls on one state: cuts inside tiles and at tile and group edges; the state each call leaves
    (excl + tile_total of its last tile) is the next call's start."""
    rng = np.random.default_rng(500)
    tile, _, e = M.geometry(dt)
    n = (128 + 6) * tile + 33
    cuts = [0, 3, e + 3, tile, tile + 1, 2 * tile + 500, 128 * tile, 128 * tile + 1, n]
    for kind in ("normal", "gensum32", "mixedzero"):
        x = data(kind, dt, n, rng)
        chunks = [x[a:b] for a, b in zip(cuts, cuts[1:])]
        for start in (-0.0, 5.0):
            check(ag, cpu, chunks, None, False, start, (kind, start))
        for skip in (False, True):
            valid = rng.random(n) > 0.0003
            valid[:tile + 10] = True
            valids = [valid[a:b] for a, b in zip(cuts, cuts[1:])]
            valids[3] = None       # a chunk without a bitmap inside the sequence
            check(ag, cpu, chunks, valids, skip, -0.0, (kind, skip, "nulls"))


def test_gpu_cumulative_sum_compute_api_chunked_negative_zero_start():
    """compute.CumulativeSum over a chunked float64 column with Start = -0.0: the chunks are one sequence."""
    from arrow_go_b200 import compute as pc
    rng = np.random.default_rng(600)
    tile, _, _ = M.geometry(np.float64)
    n = 3 * tile + 700
    x = rng.standard_normal(n)
    x[:tile + 9] = -0.0
    cuts = [0, 5, tile + 1, 2 * tile, n]
    chunks = [x[a:b] for a, b in zip(cuts, cuts[1:])]
    col = pc.Chunked([pc.Array.from_numpy(c) for c in chunks], pc.FLOAT64)
    vals, valid, nulls = pc.CumulativeSum(col, start=pc.Scalar(-0.0, pc.FLOAT64)).to_numpy()
    want, _ = M.cumulative_sum(chunks, None, False, -0.0)
    assert valid.all() and nulls == 0
    assert same(vals, want), first_diff(vals, want)
    assert np.signbit(vals[:tile + 9]).all()


# ---- past the super-group -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_gpu_cumulative_sum_past_super_group(ag, cpu, dt):
    """4096 tiles + 77 rows: the inclusive prefix of the first super-group hands the sum to the last tile."""
    rng = np.random.default_rng(700)
    tile, _, _ = M.geometry(dt)
    x = data("normal", dt, M.SUPER * M.GROUP * tile + 77, rng)
    check(ag, cpu, [x], None, False, 0.3, "super")


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_gpu_cumulative_sum_deterministic(ag, dt):
    """Two runs of the same call are byte-identical (state included)."""
    rng = np.random.default_rng(800)
    x = rng.standard_normal(3_000_017).astype(dt)
    a = run_dev(ag, [x], None, False, None)
    b = run_dev(ag, [x], None, False, None)
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
