"""CPU: the model of the default float64 Sum (tests/sum_f64_ref.py) against math.fsum, against the Sum2 error bound,
against the class rules of IEEE addition on non-finite input, and against a literal per-thread transcription of
sum_kernel<double> at sizes small enough to loop over every thread."""
import math
from fractions import Fraction

import numpy as np
import pytest

import sum_f64_ref as M

CAP_N = 2 * M.TILE_PAIRS * M.MAX_BLOCKS          # the smallest even n that fills the one-wave grid
SEAM_SIZES = [1, 2, 3, 4095, 4096, 4097, 2 * M.TILE_PAIRS * 3 + 7, CAP_N - 1, CAP_N, CAP_N + 1,
              2 * M.TILE_PAIRS * (M.MAX_BLOCKS + 9) + 1001]


def _literal_sum(x):
    """sum_kernel<double> as written, one thread at a time, in Python floats (IEEE double, round to nearest)."""
    def add(p, v):
        s, c = p
        t = s + v
        z = t - s
        e = (s - (t - z)) + (v - z)
        return (t, c + e)

    def merge(p, o):
        s, c = add(p, o[0])
        return (s, c + o[1])

    def tree(v):                                    # block_tree_sum over 256 threads, thread 0's pair
        for m in (16, 8, 4, 2, 1):
            v = [merge(v[i], v[i ^ m]) for i in range(len(v))]
        r = [v[32 * w] for w in range(8)]
        for m in (4, 2, 1):
            r = [merge(r[i], r[i ^ m]) for i in range(8)]
        return r[0]

    x = [float(v) for v in x]
    n = len(x)
    n_pairs = n >> 1
    n_tiles = (n_pairs + M.TILE_PAIRS - 1) // M.TILE_PAIRS
    G = M.grid(n_pairs)
    partials = []
    for b in range(G):
        threads = []
        for t in range(M.THREADS):
            ax = [(0.0, 0.0)] * M.ACC
            ay = [(0.0, 0.0)] * M.ACC
            for tile in range(b, n_tiles, G):
                for k in range(M.LOADS):
                    jj = tile * M.TILE_PAIRS + t + k * M.THREADS
                    if jj < n_pairs:
                        ax[k % M.ACC] = add(ax[k % M.ACC], x[2 * jj])
                        ay[k % M.ACC] = add(ay[k % M.ACC], x[2 * jj + 1])
            for k in range(M.ACC):
                ax[k] = merge(ax[k], ay[k])
            ax[0] = merge(ax[0], ax[1])
            ax[2] = merge(ax[2], ax[3])
            threads.append(merge(ax[0], ax[2]))
        partials.append(tree(threads))
    if G == 1:
        acc = partials[0]
    else:
        folded = []
        for t in range(M.THREADS):
            a = (0.0, 0.0)
            for i in range(t, G, M.THREADS):
                a = merge(a, partials[i])
            folded.append(a)
        acc = tree(folded)
    if n & 1:
        acc = add(acc, x[n - 1])
    s, c = acc
    return s + c if math.isfinite(s) else s


def _wide_range(rng, n):
    """data whose every partial sum rounds: random signs, exponents over 2^-30 .. 2^30"""
    return rng.standard_normal(n) * 2.0 ** rng.integers(-30, 31, n)


@pytest.mark.parametrize("n", [1, 2, 3, 5, 4095, 4096, 4097, 2 * M.TILE_PAIRS * 2 + 2 * 700 + 1, 2 * M.TILE_PAIRS * 3 + 7])
def test_model_equals_literal_transcription(n):
    """Vectorised model == the kernel's loops written out thread by thread, bit for bit, on data where the order
    shows (every add rounds): one block, several blocks, a masked last tile and an odd tail."""
    rng = np.random.default_rng(0x5EED + n)
    x = _wide_range(rng, n)
    assert np.float64(_literal_sum(x)).tobytes() == M.sum_f64(x).tobytes()
    x[rng.integers(0, n)] = np.inf
    assert np.float64(_literal_sum(x)).tobytes() == M.sum_f64(x).tobytes()


@pytest.mark.parametrize("n", SEAM_SIZES)
def test_model_exact_on_integer_data(n):
    """Integer-valued data: every partial sum is exact, so every grid shape must return math.fsum."""
    x = np.random.default_rng(n).integers(-(1 << 20), (1 << 20) + 1, n).astype(np.float64)
    assert M.sum_f64(x) == math.fsum(x)
    assert M.global_sum_f64([x[: n // 3], x[n // 3:]]) == math.fsum(x)


def test_model_grid_rule():
    assert [M.grid(p) for p in (0, 1, 2048, 2049, 2048 * 528, 2048 * 528 + 1, 10 ** 9)] == [1, 1, 1, 2, 528, 528, 528]


@pytest.mark.parametrize("cond", [1e10, 1e18, 1e30, 1e48])
@pytest.mark.parametrize("n", [4097, 8192, 2 * M.TILE_PAIRS * 40 + 3, CAP_N + 1])
def test_model_within_sum2_bound(n, cond):
    """GenSum-style data: |model - fsum| <= 2 eps |fsum| + gamma_n^2 sum|x| at every condition number."""
    x = M.gensum(n, cond, seed=n ^ int(math.log10(cond)))
    exact = math.fsum(x)
    got = M.sum_f64(x)
    assert abs(Fraction(float(got)) - Fraction(exact)) <= M.sum2_error_bound(x, exact), (got, exact)
    assert M.expected_class(x) == "finite" and np.isfinite(got)


def test_model_one_ulp_when_well_conditioned():
    """N(0,1): gamma_n^2 sum|x| is far below eps |S|, so the result is within 1 ULP of fsum."""
    for n in (4097, 100_003, CAP_N + 1):
        x = np.random.default_rng(n).standard_normal(n)
        got, exact = M.sum_f64(x), math.fsum(x)
        assert abs(int(got.view(np.int64)) - int(np.float64(exact).view(np.int64))) <= 1


@pytest.mark.parametrize("n", [1, 2, 3, 4097, 2 * M.TILE_PAIRS * 5 + 1, CAP_N + 1])
def test_model_nonfinite_classes(n):
    """Planted ±inf / NaN give the class any IEEE summation gives; finite data that overflows with one sign gives the
    infinity of that sign (not NaN)."""
    rng = np.random.default_rng(n + 17)
    base = rng.standard_normal(n)
    spots = sorted({0, n - 1, n // 2, min(n - 1, 2 * M.TILE_PAIRS * 2 + 1)})
    for planted in ([np.inf], [-np.inf], [np.nan], [np.inf, -np.inf], [np.inf, np.nan], [np.inf, np.inf]):
        for first in spots:
            x = base.copy()
            for k, v in enumerate(planted):
                x[(first + k * (n // 2 + 1)) % n] = v
            want = M.expected_class(x)
            assert want is not None and M.float_class(M.sum_f64(x)) == want, (planted, first, want)
    big = rng.uniform(0.6, 1.0, n) * np.finfo(np.float64).max
    for sign in (1.0, -1.0):
        got = M.sum_f64(sign * big)
        assert (got == sign * np.inf) if n > 1 else np.isfinite(got)
    assert M.sum_f64(np.array([1.0, np.inf, 2.0])) == np.inf
    assert M.sum_f64(np.full(4, 1.7e308)) == np.inf
    assert M.sum_f64(np.full(5, -np.inf)) == -np.inf


def test_model_global_fold_nonfinite():
    """The cross-rank fold keeps the class: one rank's +inf gives +inf on every rank, +inf and -inf give NaN."""
    x = np.random.default_rng(3).standard_normal(30_001)
    a, b, c = x[:10_000].copy(), x[10_000:20_000].copy(), x[20_000:].copy()
    b[5] = np.inf
    assert M.global_sum_f64([a, b, c]) == np.inf
    c[7] = -np.inf
    assert np.isnan(M.global_sum_f64([a, b, c]))
    assert M.global_sum_f64([a[:0], b]) == np.inf
