"""float64 Sum on the GPU at the inputs where a compensated sum goes wrong: ±inf and NaN, overflow, subnormals, signed
zeros and ill-conditioned data, at the sizes where the kernel's grid and tiles change shape.

The default mode is compared bit for bit with its model (tests/sum_f64_ref.py) through the host flavour and the device
flavour at a 16-byte- and an 8-byte-aligned pointer; the class of every result is checked against the class rules of
IEEE addition, which do not depend on the order, and finite results against the Sum2 error bound.  The reference-order
mode is compared with the reference's own AVX2 loop on the same data, and the global Sum with the model's rank-order
fold."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest

import sum_f64_ref as M
from arrow_go_b200 import sharding
from helpers import Dev, ptr

pytestmark = pytest.mark.gpu

CAP_N = 2 * M.TILE_PAIRS * M.MAX_BLOCKS             # the smallest even n that fills the one-wave grid
SIZES = [1, 2, 3, 4095, 4096, 4097,                 # one block and its edge
         CAP_N - 1, CAP_N, CAP_N + 1,               # the grid cap
         3_000_001,                                 # two tiles for some blocks, a masked last tile, an odd tail
         10_000_000]
DBL_MAX = np.finfo(np.float64).max
FAMILIES = ["normal", "gensum_1e10", "gensum_1e18", "gensum_1e30", "gensum_1e48", "subnormal", "overflow_pos",
            "overflow_neg", "neg_zero", "mixed_zero"]


def make(family, n, seed):
    rng = np.random.default_rng(seed)
    if family == "normal":
        return rng.standard_normal(n)
    if family.startswith("gensum_"):
        return M.gensum(n, float(family[len("gensum_"):]), seed)
    if family == "subnormal":
        k = rng.integers(-(1 << 52) + 1, 1 << 52, n)
        k[k == 0] = 1
        return k.astype(np.float64) * 2.0 ** -1074
    if family in ("overflow_pos", "overflow_neg"):
        x = rng.uniform(0.6, 1.0, n) * DBL_MAX      # any two of them overflow
        return x if family == "overflow_pos" else -x
    if family == "neg_zero":
        return np.full(n, -0.0)
    if family == "mixed_zero":
        return np.where(rng.random(n) < 0.5, -0.0, 0.0)
    raise ValueError(family)


def bits(v):
    return np.float64(v).tobytes()


def ulp_dist(a, b):
    return abs(int(np.float64(a).view(np.int64)) - int(np.float64(b).view(np.int64)))


def sum_three_ways(ag, x):
    """(host flavour, device flavour at a 16-byte-aligned pointer, device flavour at an 8-byte-aligned one)"""
    r = C.c_double(123.0)
    ag.call("ag_sum_f64", ptr(x), x.size, C.byref(r))
    got = [np.float64(r.value)]
    out = Dev(np.zeros(2))
    devs = [Dev(x), Dev(x, byte_offset=8)]
    for k, d in enumerate(devs):
        assert d.ptr % 16 == 8 * k
        ag.call("ag_sum_f64_dev", d.ptr, x.size, out.ptr + 8 * k, None)
    ag.call("ag_stream_sync", None)
    got += [np.float64(v) for v in out.get()]
    return got


def check_against_model(ag, x, what):
    want = M.sum_f64(x)
    got = sum_three_ways(ag, x)
    for g, flavour in zip(got, ("host", "dev16", "dev8")):
        assert bits(g) == bits(want), (what, flavour, g, want)
    cls = M.expected_class(x)
    if cls is not None:
        assert M.float_class(want) == cls, (what, want, cls)
    return want


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("n", SIZES)
def test_sum_special_data_matches_model(ag, n, family):
    x = make(family, n, seed=n * 31 + FAMILIES.index(family))
    got = check_against_model(ag, x, (n, family))
    if family.startswith("overflow"):
        sign = 1.0 if family == "overflow_pos" else -1.0
        assert got == sign * np.inf if n > 1 else got == x[0]   # one sign overflows to that infinity, not NaN
        return
    assert np.isfinite(got)
    if family.endswith("zero"):
        assert bits(got) == bits(0.0)                           # zeros start from +0.0, as the reference's do
        return
    exact = math.fsum(x)
    assert abs(Fraction(float(got)) - Fraction(exact)) <= M.sum2_error_bound(x, exact), (got, exact)
    if family in ("normal", "subnormal"):
        assert ulp_dist(got, exact) <= 1, (got, exact)


def placements(n):
    """[(name, {index: value})] for the planted non-finite cases that exist at size n"""
    n_pairs = n >> 1
    G = M.grid(n_pairs)
    cases = []
    for v, vn in ((np.inf, "+inf"), (-np.inf, "-inf"), (np.nan, "nan")):
        cases.append((f"element0_{vn}", {0: v}))
        if n & 1 and n > 1:
            cases.append((f"odd_tail_{vn}", {n - 1: v}))
        if n_pairs % M.TILE_PAIRS:
            cases.append((f"masked_last_tile_{vn}", {2 * (n_pairs - 1): v}))
    if G > 1:
        last = 2 * ((G - 1) * M.TILE_PAIRS + 3)
        cases.append(("pinf_block0_ninf_last_block", {11: np.inf, last: -np.inf}))
        cases.append(("pinf_last_block_nan_block0", {last: np.inf, 11: np.nan}))
    if n_pairs:
        j = n_pairs // 2 + 5 if n_pairs > 10 else 0
        cases.append(("pinf_x_chain_ninf_y_chain", {2 * j: np.inf, 2 * j + 1: -np.inf}))
        cases.append(("pinf_x_chain_pinf_y_chain", {2 * j: np.inf, 2 * j + 1: np.inf}))
    return cases


PLANTED = [(n, name, spots) for n in SIZES for name, spots in placements(n)]


@pytest.mark.parametrize("n,name,spots", PLANTED, ids=[f"{n}-{name}" for n, name, _ in PLANTED])
def test_sum_planted_nonfinite(ag, n, name, spots):
    """±inf / NaN anywhere: any NaN or both infinities give NaN, infinities of one sign give that infinity."""
    x = np.random.default_rng(n).standard_normal(n)
    for i, v in spots.items():
        x[i] = v
    got = check_against_model(ag, x, (n, name))
    vals = list(spots.values())
    if any(np.isnan(v) for v in vals) or (np.inf in vals and -np.inf in vals):
        assert np.isnan(got)
    else:
        assert got == vals[0]


def test_sum_nonfinite_known_answers(ag):
    for x, want in (([1.0, np.inf, 2.0], np.inf), ([1.7e308] * 4, np.inf), ([-np.inf] * 5, -np.inf),
                    ([-1.7e308] * 4, -np.inf), ([np.inf, np.nan], np.nan)):
        for got in sum_three_ways(ag, np.array(x)):
            assert bits(got) == bits(want) if not np.isnan(want) else np.isnan(got), (x, got)
    x = np.random.default_rng(3).standard_normal(3_000_000)
    x[1_234_567] = np.inf
    assert all(g == np.inf for g in sum_three_ways(ag, x))


# ---- reference-order mode: the reference's AVX2 loop on the same data ------------------------------------------------
REF_SIZES = [1, 3, 31, 32, 33, 4097, 100_003]


def ref_cases(n):
    rng = np.random.default_rng(n + 5)
    cases = [make(f, n, seed=n) for f in ("gensum_1e30", "subnormal", "overflow_pos", "overflow_neg", "neg_zero",
                                          "mixed_zero")]
    for spots in ({0: np.inf}, {n - 1: -np.inf}, {n // 2: np.nan}, {0: np.inf, n - 1: -np.inf}):
        x = rng.standard_normal(n)
        for i, v in spots.items():
            x[i] = v
        cases.append(x)
    mixed = rng.uniform(0.6, 1.0, n) * DBL_MAX * np.where(rng.random(n) < 0.5, -1.0, 1.0)
    cases.append(mixed)                             # a sign-mixed overflow: the class follows the order
    return cases


@pytest.mark.parametrize("n", REF_SIZES)
def test_reference_order_mode_special_data(ag, ref, n):
    """ag_sum_f64_reforder reproduces the reference's AVX2 association: equal bits wherever the result is not NaN,
    NaN where it is NaN (x86 and CUDA give NaNs of different sign)."""
    for x in ref_cases(n):
        want = C.c_double()
        ref.sum_float64_avx2(ptr(x), n, C.addressof(want))
        r = C.c_double(123.0)
        ag.call("ag_sum_f64_reforder", ptr(x), n, C.byref(r))
        d, out = Dev(x), Dev(np.zeros(1))
        ag.call("ag_sum_f64_reforder_dev", d.ptr, n, out.ptr, None)
        ag.call("ag_stream_sync", None)
        for got in (r.value, out.get()[0]):
            if np.isnan(want.value):
                assert np.isnan(got), (n, got)
            else:
                assert bits(got) == bits(want.value), (n, got, want.value)


# ---- global Sum: ranks on one GPU fold their pairs in rank order ------------------------------------------------------
def global_sums(ag, shards):
    """`len(shards)` ranks on device 0 (ag_comm_create_local with the same device per rank), one stream each."""
    world = len(shards)
    comms = (C.c_void_p * world)()
    ag.call("ag_comm_create_local", comms, world, (C.c_int * world)(*([0] * world)))
    streams, bufs, outs = [], [], []
    for k in range(world):
        st = C.c_void_p()
        ag.call("ag_stream_create", C.byref(st))
        streams.append(st)
        bufs.append(Dev(shards[k]) if len(shards[k]) else Dev(np.zeros(1)))
        outs.append(Dev(np.full(1, 123.0)))
    for k in range(world):
        ag.call("ag_sum_f64_global_dev", C.c_void_p(comms[k]), bufs[k].ptr, len(shards[k]), outs[k].ptr, streams[k])
    for st in streams:
        ag.call("ag_stream_sync", st)
    res = [np.float64(o.get()[0]) for o in outs]
    for k in range(world):
        ag.call("ag_stream_destroy", streams[k])
        ag.call("ag_comm_destroy", C.c_void_p(comms[k]))
    return res


@pytest.mark.timeout(300)
@pytest.mark.parametrize("world", [2, 3])
def test_global_sum_nonfinite_ranks(ag, world):
    ag.call("ag_init_all", None)
    n = 3_000_011
    x = np.random.default_rng(world).standard_normal(n)
    cuts = [sharding.shard_range(n, r, world) for r in range(world)]
    base = [x[a:b].copy() for a, b in cuts]
    cases = []
    s = [v.copy() for v in base]; s[-1][17] = np.inf
    cases.append(("one rank +inf", s, np.inf))
    s = [v.copy() for v in base]; s[0][5] = np.inf; s[-1][len(s[-1]) - 1] = -np.inf
    cases.append(("+inf and -inf on two ranks", s, np.nan))
    s = [v.copy() for v in base]; s[0] = s[0][:0]; s[1][0] = -np.inf
    cases.append(("an empty rank, -inf on another", s, -np.inf))
    s = [v.copy() for v in base]; s[1] = s[1][:0]
    cases.append(("an empty rank", s, None))
    for what, shards, cls in cases:
        want = M.global_sum_f64(shards)
        got = global_sums(ag, shards)
        for r, g in enumerate(got):
            assert bits(g) == bits(want), (what, world, r, g, want)
        if cls is None:
            assert np.isfinite(want)
        elif np.isnan(cls):
            assert np.isnan(want)
        else:
            assert want == cls
