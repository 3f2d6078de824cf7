"""cumulative_sum / cumulative_sum_checked (arrow/compute/internal/kernels/vector_cumulative.go).

CPU part: the restatement (oracle/cpu_ref.c:ref_cumulative_sum) against the literal vectors of
arrow/compute/vector_cumulative_test.go (tests/golden/cumulative_sum.json) and against an
independent numpy model.  GPU part: the single-pass CUDA scan through the C ABI vs the oracle:
bit-exact for integers and for floats whose partial sums are exactly representable (signed zeros
included); for general floats the deviation from the reference's left-to-right loop is bounded and,
because the scan's association is fixed, identical from run to run.  Float outputs and the carried
state are bit-exact with tests/cumsum_float_ref.py on any input (tests/test_gpu_cumsum_float.py);
that state is the last tile's excl + tile_total and may differ from the last output by rounding,
unlike the reference's."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from arrow_go_b200 import _native as N
from helpers import ALL_TYPES, INT_TYPES, NP_OF, TYPE_NAME, Dev, pack_bits, ptr, random_values, unpack_bits

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = json.load(open(os.path.join(HERE, "golden", "cumulative_sum.json")))["cases"]
ID_OF = {v: k for k, v in TYPE_NAME.items()}
NO_POS = (1 << 63) - 1


class OracleState(C.Structure):
    _fields_ = [("cur", C.c_uint8 * 8), ("encountered_null", C.c_int64)]


def state_with(t, start):
    st = OracleState()
    raw = np.array([0 if start is None else start], dtype=NP_OF[t]).tobytes()
    for i, b in enumerate(raw):
        st.cur[i] = b
    return st


def oracle_chunks(cpu, t, chunks, valids, skip, checked, start=None):
    """chunks: list of numpy arrays; valids: list of bool arrays or None.  Returns (status, values, valid, nulls, bad)."""
    st = state_with(t, start)
    total = sum(len(c) for c in chunks)
    out = np.zeros(total, dtype=NP_OF[t])
    ovalid = np.full((total + 7) // 8 + 1, 0, dtype=np.uint8)
    pos, nulls_total, status, bad_row = 0, 0, 0, NO_POS
    for x, v in zip(chunks, valids):
        n = len(x)
        bm = pack_bits(v, offset=3) if v is not None else None
        nulls, bad = C.c_int64(0), C.c_int64(0)
        o = np.zeros(n, dtype=NP_OF[t])
        rc = cpu.ref_cumulative_sum(t, ptr(x), ptr(bm) if bm is not None else None, 3, n, int(skip), int(checked),
                                    ptr(o), ptr(ovalid), pos, C.byref(st), C.byref(nulls), C.byref(bad))
        out[pos:pos + n] = o
        nulls_total += nulls.value
        if rc != 0:
            status, bad_row = rc, pos + bad.value
            break
        pos += n
    return status, out, unpack_bits(ovalid, 0, total).astype(bool), nulls_total, bad_row


def case_chunks(case):
    t = ID_OF[case["type"]]
    chunks = [np.array([0 if v is None else v for v in c], dtype=NP_OF[t]) for c in case["chunks"]]
    valids = [np.array([v is not None for v in c], dtype=bool) for c in case["chunks"]]
    if all(v.all() for v in valids):
        valids = [None] * len(chunks)
    return t, chunks, valids


def check_case(case, run):
    t, chunks, valids = case_chunks(case)
    status, out, valid, nulls, bad = run(t, chunks, valids, bool(case.get("skip_nulls")), bool(case.get("checked")), case.get("start"))
    if case.get("fails"):
        assert status != 0, case
        return
    assert status == 0, case
    want = case["out"]
    assert len(out) == len(want)
    for i, w in enumerate(want):
        if w is None:
            assert not valid[i], (case, i)
        else:
            assert valid[i] and out[i] == np.array(w, dtype=NP_OF[t]), (case, i, out[i])
    assert nulls == sum(w is None for w in want)


def test_oracle_reference_vectors(cpu):
    for case in CASES:
        check_case(case, lambda *a: oracle_chunks(cpu, *a))


def model(t, x, valid, skip, start=0):
    """numpy model: wrapping cumsum of the valid values; dead after the first null unless skip."""
    dt = np.dtype(NP_OF[t])
    v = np.ones(len(x), dtype=bool) if valid is None else valid.copy()
    if not skip and not v.all():
        v[int(np.argmin(v)):] = False
    contrib = np.where(v, x, 0).astype(dt)
    with np.errstate(over="ignore"):
        run = (np.cumsum(contrib.astype(np.uint64 if dt.kind != "f" else dt), dtype=np.uint64 if dt.kind != "f" else dt)
               + np.array(start, dtype=dt).astype(np.uint64 if dt.kind != "f" else dt))
    out = run.astype(dt) if dt.kind == "f" else run.astype(np.uint64).view(np.uint64).astype(dt)
    return np.where(v, out, 0).astype(dt), v


@pytest.mark.parametrize("t", INT_TYPES, ids=lambda t: TYPE_NAME[t])
def test_oracle_matches_numpy_model_integers(cpu, t):
    rng = np.random.default_rng(t)
    for n in (0, 1, 7, 100, 4099):
        for skip in (False, True):
            for with_nulls in (False, True):
                x = random_values(rng, t, n)
                valid = (rng.random(n) > 0.01) if with_nulls else None
                st, out, v, nulls, _ = oracle_chunks(cpu, t, [x], [valid], skip, False, start=3)
                want, wv = model(t, x, valid, skip, start=3)
                assert st == 0 and np.array_equal(v, wv) and np.array_equal(out, want), (TYPE_NAME[t], n, skip, with_nulls)
                assert nulls == int((~wv).sum())


# ------------------------------------------------------------------ GPU -----------------
gpu = pytest.mark.gpu


def gpu_chunks(ag, t, chunks, valids, skip, checked, start=None, via="dev", in_off=0, out_off=0):
    """in_off / out_off (dev only): the input and output pointers are that many elements past an aligned allocation."""
    total = sum(len(c) for c in chunks)
    isz = np.dtype(NP_OF[t]).itemsize
    if via == "host":
        assert len(chunks) == 1
        x, v = chunks[0], valids[0]
        out = np.zeros(total, dtype=NP_OF[t])
        ov = np.full((total + 7) // 8 + 1, 0xA5, dtype=np.uint8)
        bm = pack_bits(v, offset=5) if v is not None else None
        nulls, bad = C.c_int64(-1), C.c_int64(-1)
        sv = np.array([start], dtype=NP_OF[t]) if start is not None else None
        st, _ = ag.call_status("ag_cumulative_sum", t, ptr(x), ptr(bm) if bm is not None else None, 5, total, ptr(sv) if sv is not None else None,
                               int(skip), int(checked), ptr(out), ptr(ov), C.byref(nulls), C.byref(bad))
        if total % 8:
            assert ov[total // 8] >> (total % 8) == 0xA5 >> (total % 8)  # bits past n untouched
        return st, out, unpack_bits(ov, 0, total).astype(bool), nulls.value, bad.value
    state = Dev(np.zeros(4, dtype=np.int64))
    sv = np.array([start], dtype=NP_OF[t]) if start is not None else None
    ag.call("ag_cumulative_sum_state_init_dev", state.ptr, t, ptr(sv) if sv is not None else None, None)
    bad = Dev(np.zeros(1, dtype=np.int64))
    ag.call("ag_error_word_reset_dev", bad.ptr, None)
    dout = Dev(np.zeros(out_off + total + 8, dtype=NP_OF[t]))
    any_nulls = any(v is not None for v in valids)
    dov = Dev(np.zeros((total + 7) // 8 + 8, dtype=np.uint8)) if any_nulls else None
    keep, pos = [], 0
    for x, v in zip(chunks, valids):
        n = len(x)
        dx = Dev(np.concatenate([np.zeros(in_off, dtype=NP_OF[t]), x]) if n + in_off else np.zeros(1, dtype=NP_OF[t]))
        dv = Dev(pack_bits(v, offset=3)) if v is not None else None
        keep += [dx, dv]
        ag.call("ag_cumulative_sum_dev", t, dx.ptr + in_off * isz, dv.ptr if dv else None, 3, n, int(skip), int(checked),
                dout.ptr + (out_off + pos) * isz, dov.ptr if dov else None, pos, state.ptr, bad.ptr, None)
        pos += n
    ag.call("ag_stream_sync", None)
    b = int(bad.get()[0])
    stt = state.get()
    out = dout.get()[out_off:out_off + total]
    valid = unpack_bits(dov.get(), 0, total).astype(bool) if dov else np.ones(total, dtype=bool)
    return (N.AG_ERR_INVALID if (checked and b != NO_POS) else 0), out, valid, int(stt[3]), b


@gpu
@pytest.mark.parametrize("via", ["dev", "host"])
def test_gpu_reference_vectors(ag, via):
    for case in CASES:
        if via == "host" and len(case["chunks"]) != 1:
            continue
        check_case(case, lambda *a: gpu_chunks(ag, *a, via=via))


@gpu
@pytest.mark.parametrize("t", ALL_TYPES, ids=lambda t: TYPE_NAME[t])
def test_gpu_matches_oracle(ag, cpu, t):
    rng = np.random.default_rng(500 + t)
    isf = t in (N.FLOAT32, N.FLOAT64)
    for n in (1, 31, 1000, 4096, 4097, 70_001, (1 << 20) + 13):
        for skip in (False, True):
            for null_mode in ("none", "sparse", "late"):
                if isf:  # exactly summable floats: every partial sum is an integer below 2^24
                    x = rng.integers(-3, 4, n).astype(NP_OF[t])
                else:
                    x = random_values(rng, t, n)
                valid = None
                if null_mode == "sparse":
                    valid = rng.random(n) > 0.02
                elif null_mode == "late":
                    valid = np.ones(n, dtype=bool)
                    valid[int(n * 0.9):] = rng.random(n - int(n * 0.9)) > 0.5
                start = None if n % 2 else 5
                wst, wout, wv, wn, _ = oracle_chunks(cpu, t, [x], [valid], skip, False, start)
                for via in ("dev", "host"):
                    st, out, v, nulls, _ = gpu_chunks(ag, t, [x], [valid], skip, False, start, via=via)
                    assert st == 0 and np.array_equal(v, wv), (TYPE_NAME[t], n, skip, null_mode, via)
                    assert out.tobytes() == wout.tobytes(), (TYPE_NAME[t], n, skip, null_mode, via)
                    assert nulls == wn


@gpu
@pytest.mark.parametrize("t", INT_TYPES, ids=lambda t: TYPE_NAME[t])
def test_gpu_checked_overflow_row(ag, cpu, t):
    """Planted overflow: status and first failing row equal the sequential loop's."""
    rng = np.random.default_rng(900 + t)
    info = np.iinfo(NP_OF[t])
    for n in (2, 1000, 300_007):
        small = rng.integers(0, 2, n).astype(NP_OF[t])            # running sum stays tiny
        wst, wout, _, _, _ = oracle_chunks(cpu, t, [small], [None], False, True)
        st, out, _, _, bad = gpu_chunks(ag, t, [small], [None], False, True)
        if wst == 0:
            assert st == 0 and np.array_equal(out, wout)
        x = small.copy()
        pos = int(rng.integers(1, n))
        x[pos] = info.max                                          # pushes the sum over the top (or exactly to max)
        x[0] = 1
        wst, wout, _, _, wbad = oracle_chunks(cpu, t, [x], [None], False, True)
        st, out, _, _, bad = gpu_chunks(ag, t, [x], [None], False, True)
        assert (st != 0) == (wst != 0) and (wst == 0 or bad == wbad), (TYPE_NAME[t], n, pos, bad, wbad)
        # the same from a slice (input 1 element past a 16-byte boundary) into an output 3 elements past one
        st, out, _, _, bad = gpu_chunks(ag, t, [x], [None], False, True, in_off=1, out_off=3)
        assert (st != 0) == (wst != 0) and (wst == 0 or bad == wbad), (TYPE_NAME[t], n, pos, bad, wbad, "sliced")
        # a null in front of the offender (no skip) hides it: the sequence is dead before the overflow
        valid = np.ones(n, dtype=bool)
        valid[0] = False
        wst, wout, wv, _, _ = oracle_chunks(cpu, t, [x], [valid], False, True)
        st, out, v, _, _ = gpu_chunks(ag, t, [x], [valid], False, True)
        assert st == wst == 0 and np.array_equal(v, wv) and np.array_equal(out, wout)


@gpu
@pytest.mark.parametrize("t", [N.INT64, N.FLOAT64, N.INT32], ids=lambda t: TYPE_NAME[t])
def test_gpu_large_crosses_super_group(ag, cpu, t):
    """> 4096 tiles (128 MB of input): the third look-back level (inclusive prefix per super-group); checked int64 runs
    it with three-word status entries."""
    rng = np.random.default_rng(4242)
    n = 4100 * (32768 // np.dtype(NP_OF[t]).itemsize) + 77
    x = rng.integers(-3, 4, n).astype(NP_OF[t])
    for valid in (None, rng.random(n) > 0.001):
        for checked in ((False, True) if t == N.INT64 else (False,)):
            wst, wout, wv, wn, _ = oracle_chunks(cpu, t, [x], [valid], True, checked, 11)
            st, out, v, nulls, _ = gpu_chunks(ag, t, [x], [valid], True, checked, 11)
            assert st == wst == 0 and np.array_equal(v, wv) and out.tobytes() == wout.tobytes() and nulls == wn, checked


@gpu
def test_gpu_chunked_state_carry(ag, cpu):
    rng = np.random.default_rng(77)
    for t in (N.INT64, N.INT32, N.FLOAT64):
        cuts = [0, 5, 5, 4101, 70_000, 200_003]
        n = cuts[-1]
        x = rng.integers(-1000, 1000, n).astype(NP_OF[t])
        for skip in (False, True):
            valid = rng.random(n) > 0.0005
            valid[:4200] = True
            chunks = [x[a:b] for a, b in zip(cuts, cuts[1:])]
            valids = [valid[a:b] for a, b in zip(cuts, cuts[1:])]
            wst, wout, wv, wn, _ = oracle_chunks(cpu, t, chunks, valids, skip, False, 7)
            st, out, v, nulls, _ = gpu_chunks(ag, t, chunks, valids, skip, False, 7)
            assert st == 0 and np.array_equal(v, wv) and out.tobytes() == wout.tobytes() and nulls == wn, (TYPE_NAME[t], skip)


@gpu
def test_gpu_general_floats_bounded_and_deterministic(ag, cpu):
    """General data: not bit-identical to a left-to-right loop (no parallel scan can be), but
    (a) within the standard summation bound of the exact prefix sums, no worse than the reference's
    own error, and (b) identical from run to run (fixed association)."""
    rng = np.random.default_rng(1)
    n = 3_000_017
    x = rng.standard_normal(n)
    _, ref_out, _, _, _ = oracle_chunks(cpu, N.FLOAT64, [x], [None], False, False)
    _, a, _, _, _ = gpu_chunks(ag, N.FLOAT64, [x], [None], False, False)
    _, b, _, _, _ = gpu_chunks(ag, N.FLOAT64, [x], [None], False, False)
    assert a.tobytes() == b.tobytes()
    exact = np.cumsum(x.astype(np.longdouble))
    scale = np.cumsum(np.abs(x))
    eps = np.finfo(np.float64).eps
    gpu_err = np.abs(a.astype(np.longdouble) - exact)
    ref_err = np.abs(ref_out.astype(np.longdouble) - exact)
    assert (gpu_err <= 64 * eps * scale).all()          # log-depth tree: far inside the n*eps bound
    assert gpu_err.max() <= max(ref_err.max(), eps) * 4  # and no worse than the sequential loop in practice


@gpu
@pytest.mark.parametrize("t", [N.FLOAT64, N.FLOAT32], ids=lambda t: TYPE_NAME[t])
def test_gpu_nonfinite_prefix_classes(ag, cpu, t):
    """±inf and NaN planted inside a tile, at tile edges and on both sides of a look-back group boundary (kScGroup =
    128 tiles of 32 KB): every prefix has the sequential loop's class (finite, +inf, -inf or NaN) — NaN and infinity
    bit patterns pass through the look-back's status words — and the finite prefixes before the first planted value
    keep the bound of test_gpu_general_floats_bounded_and_deterministic.  N(0,1) data: no finite prefix overflows."""
    dt = NP_OF[t]
    tile = 32768 // np.dtype(dt).itemsize
    group = 128 * tile                              # first group boundary: row 524,288 (float64), 1,048,576 (float32)
    n = group + 3 * tile + 77
    rng = np.random.default_rng(600 + t)
    base = rng.standard_normal(n).astype(dt)
    eps = np.finfo(dt).eps
    spots = [100, tile - 1, tile, 5 * tile + 17, group - 1, group, group + tile + 3]
    cases = [{p: v} for p in spots for v in (np.inf, -np.inf, np.nan)]
    cases += [{group - 1: np.inf, group: -np.inf}, {tile - 1: -np.inf, group + 5: np.inf}, {tile: np.nan, group + 1: np.inf},
              {100: np.inf, tile: np.inf, group: np.inf}]
    for spot in cases:
        x = base.copy()
        for i, v in spot.items():
            x[i] = v
        _, want, _, _, _ = oracle_chunks(cpu, t, [x], [None], False, False)
        st, got, _, _, _ = gpu_chunks(ag, t, [x], [None], False, False)
        assert st == 0
        for cls in (np.isnan, np.isposinf, np.isneginf, np.isfinite):
            bad = np.flatnonzero(cls(got) != cls(want))
            assert bad.size == 0, (TYPE_NAME[t], spot, cls.__name__, bad[:5])
        first = min(spot)
        exact = np.cumsum(x[:first].astype(np.longdouble))
        scale = np.cumsum(np.abs(x[:first]).astype(np.longdouble))
        assert (np.abs(got[:first].astype(np.longdouble) - exact) <= 64 * eps * scale).all(), (TYPE_NAME[t], spot)


@gpu
def test_gpu_chunks_with_and_without_bitmap_share_one_sequence(ag, cpu):
    """Chunks without a bitmap and chunks with one alternate inside one sequence; once a null was met (no skip) a
    later bitmap-free chunk is all null and leaves the carried value alone."""
    rng = np.random.default_rng(78)
    for t in (N.INT64, N.INT16, N.FLOAT64, N.FLOAT32):
        cuts = [0, 4096 * 16, 4096 * 16 + 48_000, 300_000 + 16, 300_000 + 16 + 70_000 + 32, 500_000]
        n = cuts[-1]
        x = rng.integers(-3, 4, n).astype(NP_OF[t])
        for skip in (False, True):
            valids = [None, None, rng.random(cuts[3] - cuts[2]) > 0.001, None, None]
            valids[2][:100] = True
            chunks = [x[a:b] for a, b in zip(cuts, cuts[1:])]
            wst, wout, wv, wn, _ = oracle_chunks(cpu, t, chunks, valids, skip, False, 3)
            st, out, v, nulls, _ = gpu_chunks(ag, t, chunks, valids, skip, False, 3)
            assert st == 0 and np.array_equal(v, wv) and out.tobytes() == wout.tobytes() and nulls == wn, (TYPE_NAME[t], skip)


@gpu
def test_gpu_element_aligned_input_streams(ag, cpu):
    """An Arrow slice: the values pointer is only element-aligned (1, 2 or 3 elements past a 16-byte boundary).  4- and
    8-byte types are fetched in 4- / 8-byte cp.async pieces, 1- / 2-byte types below 4-byte alignment by plain loads
    (the others in 4-byte pieces).  Each input runs three ways: into an aligned output, into an output just as far past
    a 16-byte boundary (stored in pieces), and checked (status, first failing row and values equal the oracle's); with
    and without a validity bitmap, lengths around the 32 KB tile edges."""
    rng = np.random.default_rng(79)
    for t in (N.INT64, N.FLOAT64, N.INT32, N.FLOAT32, N.UINT32, N.INT16, N.UINT8):
        dt = NP_OF[t]; isz = np.dtype(dt).itemsize
        for off_elems in (1, 2, 3):
            for n in (1, 4095, 4096, 4097, 8193, 70_001, 300_017):
                base = rng.integers(-3, 4, n + off_elems + 16).astype(dt) if np.dtype(dt).kind != "u" else rng.integers(0, 4, n + off_elems + 16).astype(dt)
                x = base[off_elems:off_elems + n]
                for p_null, skip in ((0.0, False), (0.05, True), (0.05, False)):
                    valid = rng.random(n) >= p_null if p_null else None
                    for out_off, checked in ((0, False), (off_elems, False), (0, True)):
                        wst, wout, wv, wn, wbad = oracle_chunks(cpu, t, [x], [valid], skip, checked, 2)
                        # device call on a pointer off_elems elements past an aligned allocation
                        dbase = Dev(base)
                        state = Dev(np.zeros(4, dtype=np.int64)); sv = np.array([2], dtype=dt)
                        ag.call("ag_cumulative_sum_state_init_dev", state.ptr, t, ptr(sv), None)
                        bad = Dev(np.zeros(1, dtype=np.int64)); ag.call("ag_error_word_reset_dev", bad.ptr, None)
                        dout = Dev(np.zeros(out_off + n + 8, dtype=dt))
                        dv = Dev(pack_bits(valid, offset=3)) if valid is not None else None
                        dov = Dev(np.zeros((n + 7) // 8 + 8, dtype=np.uint8)) if valid is not None else None
                        ag.call("ag_cumulative_sum_dev", t, dbase.ptr + off_elems * isz, dv.ptr if dv else None, 3, n, int(skip),
                                int(checked), dout.ptr + out_off * isz, dov.ptr if dov else None, 0, state.ptr, bad.ptr, None)
                        ag.call("ag_stream_sync", None)
                        where = (TYPE_NAME[t], off_elems, n, p_null, skip, out_off, checked)
                        got_bad = int(bad.get()[0])
                        if wst != 0:  # a checked narrow type whose running sum leaves its range
                            assert got_bad == wbad, where
                            continue
                        assert got_bad == NO_POS, where
                        out = dout.get()[out_off:out_off + n]
                        assert out.tobytes() == wout.tobytes(), where
                        if valid is not None:
                            assert np.array_equal(unpack_bits(dov.get(), 0, n).astype(bool), wv) and int(state.get()[3]) == wn, where
