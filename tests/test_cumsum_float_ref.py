"""The float cumulative_sum model (tests/cumsum_float_ref.py) held to the kernel source and to the reference, no GPU:
  * a literal per-thread transcription of cumsum_stream_kernel gives the model's bits;
  * on data whose partial sums are all exact the model gives oracle/cpu_ref.c:ref_cumulative_sum's bits, signed
    zeros included;
  * on general data every output and the carried state lie within the summation bound of the exact prefix for the
    depth of the model's addition tree, and ±inf / NaN land in the reference's classes;
  * the model's constants are scan.cu's."""
import itertools
import os
import re

import numpy as np
import pytest

import cumsum_float_ref as M
from helpers import oracle_cumsum
from sum_f64_ref import gensum

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [np.float32, np.float64]
DT_IDS = ["float32", "float64"]


def same(a, b):
    """Bit-exact, except that a NaN equals any NaN."""
    a, b = np.atleast_1d(np.asarray(a)), np.atleast_1d(np.asarray(b))
    na, nb = np.isnan(a), np.isnan(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


def boundary_sizes(dt):
    tile, seg, e = M.geometry(dt)
    return [1, 2, e - 1, e, e + 1, seg - 1, seg, seg + 1, tile - 1, tile, tile + 1, 3 * tile + 77,
            127 * tile + 5, 128 * tile, 128 * tile + 1, (2 * 128 + 3) * tile]


# ---- the literal transcription --------------------------------------------------------------------------------------
def hs32(v):
    for d in (1, 2, 4, 8, 16):
        v = [v[l - d] + v[l] if l >= d else v[l] for l in range(32)]
    return v


def literal_lookback(agg, start):
    """cumsum_lookback, tile by tile: statuses are dictionaries written once, read when the loops reach them."""
    z = type(agg[0])(-0.0)
    gagg, sincl, excl = {}, {}, []
    for t, total in enumerate(agg):
        g, qpos = divmod(t, M.GROUP)
        sg, gq = divmod(g, M.SUPER)
        x = [hs32([agg[g * M.GROUP + r * 32 + l] if r * 32 + l < qpos else z for l in range(32)]) for r in range(4)]
        part = z
        for r in range(4):
            part = part + x[r][31]
        if qpos == M.GROUP - 1:
            gagg[g] = part + total
        gpart = hs32([gagg[sg * M.SUPER + l] if l < gq else z for l in range(32)])[31]
        base = sincl[sg - 1] if sg > 0 else start
        e = (base + gpart) + part
        if qpos == M.GROUP - 1 and gq == M.SUPER - 1:
            sincl[sg] = e + total
        excl.append(e)
    return excl


def literal_kernel(x, valid, skip, start):
    """cumsum_stream_kernel<T, *, false> written thread by thread: (out, state)."""
    dt = x.dtype
    f = dt.type
    z = f(-0.0)
    tile, seg, e_rows = M.geometry(dt)
    n = len(x)
    limit = n
    if valid is not None and not skip and not valid.all():
        limit = int(np.argmin(valid))
    xs = list(x)
    counts = [(valid is None or bool(valid[r])) and r < limit for r in range(n)]
    n_tiles = (n + tile - 1) // tile
    agg, lane_excl, warp_excl = [], {}, {}
    for t in range(n_tiles):
        s_warp = []
        for w in range(M.WARPS):
            tot = []
            for lane in range(32):
                acc = z
                for i in range(e_rows):
                    r = t * tile + w * seg + lane * e_rows + i
                    if r < n and counts[r]:
                        acc = acc + xs[r]
                tot.append(acc)
            incl = hs32(tot)
            for lane in range(32):
                lane_excl[t, w, lane] = incl[lane - 1] if lane > 0 else z
            s_warp.append(incl[31])
        total = z
        for w in range(M.WARPS):
            warp_excl[t, w] = total
            total = total + s_warp[w]
        agg.append(total)
    excl = literal_lookback(agg, f(start))
    out = np.zeros(n, dtype=dt)
    for t in range(n_tiles):
        for w in range(M.WARPS):
            for lane in range(32):
                run = warp_excl[t, w] + lane_excl[t, w, lane]
                for i in range(e_rows):
                    r = t * tile + w * seg + lane * e_rows + i
                    if r < n and counts[r]:
                        run = run + xs[r]
                        out[r] = excl[t] + run
    return out, excl[-1] + agg[-1]


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_literal_transcription_matches_model(dt):
    tile, seg, e = M.geometry(dt)
    rng = np.random.default_rng(11 + np.dtype(dt).itemsize)
    cases = [(n, None, False, 0.0) for n in (1, e - 1, e + 1, seg - 1, seg + 1, tile - 1, tile + 1, 2 * tile + 77)]
    cases += [(tile + 100, "sparse", True, 0.375), (tile + 100, "sparse", False, -0.0), (3 * seg + 5, None, False, -0.0)]
    cases += [(128 * tile + 5, None, False, 0.1)]           # the group boundary: tile 128 reads a group total
    with np.errstate(all="ignore"):
        for n, vmode, skip, start in cases:
            x = rng.standard_normal(n).astype(dt)
            valid = None
            if vmode == "sparse":
                valid = rng.random(n) > 0.05
                valid[:40] = True
            want_out, want_state = literal_kernel(x, valid, skip, start)
            out, state = M.scan_call(x, valid, skip, start)
            assert same(out, want_out) and same(state, want_state), (n, vmode, skip, start)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_literal_lookback_past_super_group(dt):
    """The third level: the inclusive prefix of a super-group (4096 tiles) hands the sum on to the next one."""
    rng = np.random.default_rng(12)
    n_tiles = 2 * M.SUPER * M.GROUP + 3 * M.GROUP + 17
    totals = (rng.standard_normal(n_tiles) * 64).astype(dt)
    start = dt(0.3)
    want = literal_lookback(list(totals), start)
    assert same(M.lookback(totals, start), np.array(want, dtype=dt))


# ---- exactly summable data: the reference's bits ----------------------------------------------------------------
def exact_data(rng, dt, n):
    """Multiples of 1/4 in [-3/4, 3/4] with signed zeros: every partial sum over any range is exact while
    |prefix| < 2^(p-3)."""
    k = rng.integers(-3, 4, n)
    x = (k * 0.25).astype(dt)
    x[(k == 0) & (rng.random(n) < 0.5)] = dt(-0.0)
    return x


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_exactly_summable_equals_oracle(cpu, dt):
    rng = np.random.default_rng(21)
    tile, _, _ = M.geometry(dt)
    for n in boundary_sizes(dt):
        x = exact_data(rng, dt, n)
        for vmode, skip, start in ((None, False, None), ("sparse", True, 5.0), ("sparse", False, -0.0), (None, False, 0.75)):
            valid = None if vmode is None else rng.random(n) > 0.01
            want, _, _, wstate = oracle_cumsum(cpu, [x], [valid], skip, start)
            got, state = M.cumulative_sum([x], [valid], skip, start)
            assert same(got, want) and same(state, wstate), (n, vmode, skip, start)
    # chunked: cut inside a tile, at a tile edge and at a group edge
    n = (128 + 9) * tile + 11
    x = exact_data(rng, dt, n)
    cuts = [0, 7, tile, tile + 300, 128 * tile, n]
    chunks = [x[a:b] for a, b in zip(cuts, cuts[1:])]
    for skip in (False, True):
        valid = rng.random(n) > 0.0005
        valid[:tile + 400] = True
        valids = [valid[a:b] for a, b in zip(cuts, cuts[1:])]
        want, _, _, wstate = oracle_cumsum(cpu, chunks, valids, skip, -0.0)
        got, state = M.cumulative_sum(chunks, valids, skip, -0.0)
        assert same(got, want) and same(state, wstate), skip


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_exactly_summable_past_super_group(cpu, dt):
    rng = np.random.default_rng(22)
    tile, _, _ = M.geometry(dt)
    n = M.SUPER * M.GROUP * tile + 77
    x = exact_data(rng, dt, n)
    for valid, start in ((None, 11.0), (rng.random(n) > 0.001, -0.0)):
        want, _, _, wstate = oracle_cumsum(cpu, [x], [valid], True, start)
        got, state = M.cumulative_sum([x], [valid], True, start)
        assert same(got, want) and same(state, wstate), start


# ---- signed zeros -----------------------------------------------------------------------------------------------
def signed_zero_cases(dt):
    """(chunks, valids, skip, start): every partial sum is exact, so the reference's zero signs are the answer."""
    tile, seg, e = M.geometry(dt)
    nz, pz = dt(-0.0), dt(0.0)
    rng = np.random.default_rng(31)
    cases = [([np.array([nz, nz, 1.0], dtype=dt)], None, False, -0.0),
             ([np.array([nz, nz, 1.0], dtype=dt)], None, False, 0.0)]
    for n in (1, e + 3, seg + 1, tile - 1, tile, tile + 5, 3 * tile + 77):
        for start in (-0.0, 0.0, None):
            cases.append(([np.full(n, nz, dtype=dt)], None, False, start))                # all -0.0, padding in the last tile
        mixed = np.where(rng.random(n) < 0.5, nz, pz).astype(dt)
        cases.append(([mixed], None, False, -0.0))
        v = np.ones(n, dtype=bool)
        v[n // 2] = False
        for skip in (False, True):
            cases.append(([np.full(n, nz, dtype=dt)], [v], skip, -0.0))                    # -0.0 before and after a null
    # chunked: 1 + -1 cancels to +0, which the -0.0 rows after it keep; and a -0.0 start carried through -0.0 chunks
    x =np.concatenate([np.array([1.0, -1.0], dtype=dt), np.full(tile + 3, nz, dtype=dt)])
    cases.append(([x[:1], x[1:5], x[5:]], None, False, -0.0))
    cases.append(([np.full(5, nz, dtype=dt), np.full(tile + 1, nz, dtype=dt)], None, False, -0.0))
    return cases


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_signed_zeros_equal_oracle(cpu, dt):
    for chunks, valids, skip, start in signed_zero_cases(dt):
        want, _, _, wstate = oracle_cumsum(cpu, chunks, valids, skip, start)
        got, state = M.cumulative_sum(chunks, valids, skip, start)
        where = ([len(c) for c in chunks], valids is not None, skip, start)
        assert same(got, want), (where, np.flatnonzero(np.signbit(got) != np.signbit(want))[:4])
        assert same(state, wstate), where


# ---- the error bound --------------------------------------------------------------------------------------------
def depth(dt, n):
    """Longest chain of roundings from one input to one output or the state in the model's tree."""
    tile, _, e = M.geometry(dt)
    n_super = -(-n // (tile * M.GROUP * M.SUPER))
    return 3 * e + 60 + 3 * n_super


def assert_within_bound(dt, x, counted, start, out, state):
    """|got - exact| <= gamma_D * (|start| + sum |x_j|), in exact integer arithmetic on a common binary scale."""
    p = np.finfo(dt).nmant + 1
    d = depth(dt, len(x))
    terms = np.concatenate([[start], np.where(counted, x, 0)]).astype(np.float64)
    got = np.concatenate([out[counted], [state]]).astype(np.float64)
    assert np.isfinite(terms).all() and np.isfinite(got).all()
    m_all, e_all = np.frexp(np.concatenate([terms, got]))
    nz = m_all != 0
    s = int((e_all[nz] - 53).min()) if nz.any() else 0

    def ints(v):
        m, e = np.frexp(v)
        mant = (m * 2.0 ** 53).astype(np.int64).tolist()
        sh = (e - 53 - s).tolist()
        return [a << b if a >= 0 else -((-a) << b) for a, b in zip(mant, sh)]

    t_int = ints(terms)
    exact = list(itertools.accumulate(t_int))
    scale = list(itertools.accumulate(abs(v) for v in t_int))
    rows = [0] + list(1 + np.flatnonzero(counted))              # prefix index of every output: start + x[:i+1]
    g_int = ints(got)
    for k, gi in enumerate(g_int):
        i = rows[k + 1] if k + 1 < len(rows) else len(t_int) - 1
        err = abs(gi - exact[i])
        assert err * ((1 << p) - d) <= d * scale[i], (k, i)


def general_data(kind, dt, n, rng):
    if kind == "normal":
        return rng.standard_normal(n).astype(dt)
    if kind == "wide":
        emax = 60 if dt == np.float32 else 300
        return (rng.choice([-1.0, 1.0], n) * (1 + rng.random(n)) * 2.0 ** rng.integers(-emax, emax // 2, n)).astype(dt)
    return gensum(n, 1e8 if kind == "gensum8" else 1e32, 41).astype(dt)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("kind", ["normal", "wide", "gensum8", "gensum32"])
def test_general_data_within_bound(dt, kind):
    rng = np.random.default_rng(51)
    tile, seg, e = M.geometry(dt)
    for n in (e + 1, seg + 3, tile + 1, 3 * tile + 77, 128 * tile + 77):
        x = general_data(kind, dt, n, rng)
        if not np.isfinite(x).all():
            continue
        for valid, skip, start in ((None, False, 0.0), (rng.random(n) > 0.01, True, 5.0)):
            out, state = M.cumulative_sum([x], [valid], skip, start)
            counted = M.counted_rows(n, valid, skip)
            assert_within_bound(dt, x, counted, dt(start), out, state)


# ---- non-finite values ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_nonfinite_classes_equal_oracle(cpu, dt):
    tile, _, _ = M.geometry(dt)
    group = M.GROUP * tile
    n = group + 3 * tile + 77
    rng = np.random.default_rng(61)
    base = rng.standard_normal(n).astype(dt)
    spots = [0, 100, tile - 1, tile, 5 * tile + 17, group - 1, group, group + tile + 3, n - 1]
    cases = [{p: v} for p in spots for v in (np.inf, -np.inf, np.nan)]
    cases += [{group - 1: np.inf, group: -np.inf}, {tile - 1: -np.inf, group + 5: np.inf}, {tile: np.nan, group + 1: np.inf}]
    for spot in cases:
        x = base.copy()
        for i, v in spot.items():
            x[i] = v
        want, _, _, wstate = oracle_cumsum(cpu, [x], None, False, None)
        got, state = M.cumulative_sum([x])
        for cls in (np.isnan, np.isposinf, np.isneginf, np.isfinite):
            assert np.array_equal(cls(got), cls(want)), (spot, cls.__name__)
            assert cls(state) == cls(wstate), (spot, cls.__name__)


# ---- constants --------------------------------------------------------------------------------------------------
def test_constants_match_scan_cu():
    src = open(os.path.join(ROOT, "arrow_go_b200", "csrc", "scan.cu")).read()

    def const(name):
        m = re.search(r"constexpr int %s = ([^;]+);" % name, src)
        assert m, name
        return m.group(1).split("//")[0].strip()

    threads = int(const("kScThreads"))
    warps = const("kScWarps")
    assert warps == "kScThreads / 32" and threads // 32 == M.WARPS
    assert int(const("kScRows")) == M.VEC_ROWS
    assert const("kScTileBytes") == "kScThreads * kScRows * 16" and threads * M.VEC_ROWS * 16 == M.TILE_BYTES
    assert int(const("kScGroup")) == M.GROUP
    assert int(const("kScSuper")) == M.SUPER
    # the accumulator identity is -0.0 in the float policy
    assert re.search(r"struct Pol<T, true>.*?zero\(\) \{ return T\(-0\.0\); \}", src, re.S)
