"""The logical-column model of tests/exec_model.py pinned against pyarrow.compute (Arrow C++), for the functions where
Arrow C++ and arrow-go agree, and the layout generator checked to flatten back to its logical column.  No GPU and no
call into the library: these define what tests/test_gpu_exec_differential.py holds the device to."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pac
import pytest

import exec_model as M
from arrow_go_b200 import compute as pc

PA_TYPE = {pc.BOOL: pa.bool_(), pc.UINT8: pa.uint8(), pc.INT8: pa.int8(), pc.UINT16: pa.uint16(), pc.INT16: pa.int16(),
           pc.UINT32: pa.uint32(), pc.INT32: pa.int32(), pc.UINT64: pa.uint64(), pc.INT64: pa.int64(),
           pc.FLOAT32: pa.float32(), pc.FLOAT64: pa.float64()}
TYPE_OF_PA = {v: k for k, v in PA_TYPE.items()}


def to_pa(a):
    if isinstance(a, M.Sca):
        return pa.scalar(a.value, type=PA_TYPE[a.type])
    return pa.array(a.values, type=PA_TYPE[a.type], mask=None if a.valid is None else ~a.valid)


def col(rng, t, n, p_null=0.2, lo=None, hi=None):
    if t == pc.BOOL:
        v = rng.random(n) < 0.5
    elif t in M.FLOATS:
        v = rng.integers(-50, 51, n).astype(pc.NP_OF[t]) * (rng.random(n) + 0.5).astype(pc.NP_OF[t])
    else:
        info = np.iinfo(pc.NP_OF[t])
        lo = info.min if lo is None else max(lo, info.min)
        hi = info.max if hi is None else min(hi, info.max)
        v = rng.integers(lo, hi, n, endpoint=True, dtype=pc.NP_OF[t])
    return M.Col(t, v, rng.random(n) >= p_null if p_null else None)


def assert_same(out, want, what):
    """`out` (model Out / Fail) equals the pyarrow result `want` (an Array, or an exception)."""
    if isinstance(want, Exception):
        assert isinstance(out, M.Fail), (what, out, want)
        return
    assert not isinstance(out, M.Fail), (what, out)
    assert PA_TYPE[out.type] == want.type, (what, out.type, want.type)
    assert len(out) == len(want), what
    wv = ~np.asarray(want.is_null().to_numpy(zero_copy_only=False), dtype=bool)
    assert np.array_equal(out.valid, wv), what
    got = np.asarray(out.values)[wv]
    exp = want.filter(pa.array(wv)).to_numpy(zero_copy_only=False)
    if got.dtype.kind == "f":
        assert np.array_equal(np.isnan(got), np.isnan(exp)) and got[~np.isnan(got)].tobytes() == exp[~np.isnan(exp)].astype(got.dtype).tobytes(), what
    else:
        assert np.array_equal(got, exp.astype(got.dtype)), what


def pa_call(fn, *a, **kw):
    try:
        r = fn(*a, **kw)
        return r if isinstance(r, pa.Array) else r.combine_chunks() if isinstance(r, pa.ChunkedArray) else r
    except (pa.ArrowInvalid, pa.ArrowNotImplementedError, IndexError) as e:
        return e


PA_ARITH = {"add": "add_checked", "add_unchecked": "add", "subtract": "subtract_checked", "subtract_unchecked": "subtract",
            "multiply": "multiply_checked", "multiply_unchecked": "multiply"}


@pytest.mark.parametrize("name", list(PA_ARITH))
def test_model_arithmetic_matches_pyarrow(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    for t in M.NUMERIC:
        for case in range(12):
            n = int(rng.integers(0, 300))
            narrow = case % 3 == 0                      # small values: few overflows, so the values get compared
            l = col(rng, t, n, lo=-20 if narrow else None, hi=20 if narrow else None)
            r = col(rng, t, n, lo=-20 if narrow else None, hi=20 if narrow else None)
            if name == "multiply" and t in M.INTS and l.valid is not None:
                # arrow-go's MultiplyChecked runs under ScalarBinary, so it checks null slots too
                # (arrow/compute/internal/kernels/base_arithmetic.go:279-286); Arrow C++ skips them.  No overflow under nulls.
                l.values[~l.validity()] = 0
            if name in ("add", "subtract") and t in M.SIGNED and not narrow:
                # arrow-go's checked add / sub use the unsigned carry test on signed values (base_arithmetic.go:249-277):
                # add catches only overflow past the maximum, sub only past the minimum.  Arrow C++ catches both, so
                # the operands keep to the side both see: add of non-negatives, sub of a non-positive minus a non-negative.
                mx = np.iinfo(pc.NP_OF[t]).max
                l.values &= mx
                r.values &= mx
                if name == "subtract":
                    l.values[:] = -l.values
            shapes = [(l, r), (l, M.Sca(t, r.values[0].item() if n else 1)), (M.Sca(t, l.values[0].item() if n else 1), r),
                      (l, M.Sca(t, None))]
            for a, b in shapes:
                out = M.model(name, [a, b])
                want = pa_call(getattr(pac, PA_ARITH[name]), to_pa(a), to_pa(b))
                if isinstance(want, pa.Scalar):
                    continue
                assert_same(out, want, (name, M.NAME[t], n, type(a).__name__, type(b).__name__))


def test_model_promotion_matches_pyarrow():
    rng = np.random.default_rng(7)
    for lt in M.NUMERIC:
        for rt in M.NUMERIC:
            if lt == rt:
                continue
            # values that fit every numeric type, then a planted one that the promoted type may not hold
            l, r = col(rng, lt, 50, lo=0, hi=100), col(rng, rt, 50, lo=0, hi=100)
            to = M.common_numeric(lt, rt)
            for name in ("add_unchecked", "greater_equal"):
                want = pa_call(getattr(pac, {"add_unchecked": "add"}.get(name, name)), to_pa(l), to_pa(r))
                out = M.model(name, [l, r])
                assert_same(out, want, (name, lt, rt))
                assert out.type == (to if name == "add_unchecked" else pc.BOOL)
            if lt == pc.UINT64 and rt in M.SIGNED:
                l.values[7] = np.uint64(1 << 63)
                l.valid = np.ones(50, dtype=bool)
                out = M.model("add", [l, r])
                assert isinstance(out, M.Fail) and out.msg == f"integer value {1 << 63} not in range: 0 to {(1 << 63) - 1}"
                assert isinstance(pa_call(pac.add_checked, to_pa(l), to_pa(r)), Exception)


@pytest.mark.parametrize("name", list(M.CMP))
def test_model_compare_matches_pyarrow(name):
    rng = np.random.default_rng(3 + len(name))
    for t in M.NUMERIC:
        for n in (0, 1, 9, 200):
            l, r = col(rng, t, n, lo=-3, hi=3), col(rng, t, n, lo=-3, hi=3)
            if t in M.FLOATS and n > 4:
                l.values[:3] = [np.nan, -0.0, 0.0]
                r.values[:3] = [np.nan, 0.0, np.nan]
            for a, b in ((l, r), (l, M.Sca(t, 1)), (M.Sca(t, 1), r), (M.Sca(t, None), r)):
                assert_same(M.model(name, [a, b]), pa_call(getattr(pac, name), to_pa(a), to_pa(b)), (name, M.NAME[t], n))


@pytest.mark.parametrize("name", ["and", "or", "and_kleene", "or_kleene"])
def test_model_boolean_matches_pyarrow(name):
    rng = np.random.default_rng(11)
    for n in (0, 1, 8, 9, 300):
        l, r = col(rng, pc.BOOL, n, 0.3), col(rng, pc.BOOL, n, 0.3)
        for a, b in ((l, r), (l, M.Sca(pc.BOOL, True)), (M.Sca(pc.BOOL, False), r), (l, M.Sca(pc.BOOL, None)), (M.Sca(pc.BOOL, None), r)):
            want = pa_call(getattr(pac, name), to_pa(a), to_pa(b))
            assert_same(M.model(name, [a, b]), want, (name, n))


def test_model_safe_cast_matches_pyarrow():
    rng = np.random.default_rng(5)
    for src in M.NUMERIC:
        for dst in M.NUMERIC:
            for case in range(6):
                c = col(rng, src, 64, lo=-300 if case < 3 else None, hi=300 if case < 3 else None)
                if src in M.FLOATS:
                    if case >= 3 and dst in M.INTS:
                        # float -> int: Arrow C++ also refuses out-of-range values with its own check; arrow-go only
                        # checks truncation, and its conversion of an out-of-range float is the loop's (undefined in C)
                        # value: compare on whole numbers inside the target range
                        c.values[:] = np.clip(np.trunc(c.values.astype(np.float64) / 2), *M._int_range(dst)).astype(c.values.dtype)
                    if dst in M.INTS and case == 1:
                        c.values[5] = 2.5                # truncated
                if src in M.INTS and dst in M.FLOATS and case == 4:
                    c.values[:] = 0
                    if M.width(src) >= (32 if dst == pc.FLOAT32 else 64):
                        c.values[9] = c.values.dtype.type(np.iinfo(c.values.dtype).max)   # beyond the mantissa
                want = pa_call(pac.cast, to_pa(c), PA_TYPE[dst], safe=True)
                out = M.model("cast", [c], {"to": dst})
                assert_same(out, want, ("cast", M.NAME[src], M.NAME[dst], case))


def test_model_filter_take_match_pyarrow():
    rng = np.random.default_rng(9)
    for t in M.NUMERIC + [pc.BOOL]:
        for n in (0, 1, 7, 64, 65, 500):
            v, m = col(rng, t, n, 0.2), col(rng, pc.BOOL, n, 0.2)
            for sel, pa_sel in ((pc.DROP_NULLS, "drop"), (pc.EMIT_NULLS, "emit_null")):
                want = pa_call(pac.filter, to_pa(v), to_pa(m), null_selection_behavior=pa_sel)
                assert_same(M.model("filter", [v, m], {"null_selection": sel}), want, ("filter", M.NAME[t], n, sel))
            for it in (pc.INT8, pc.UINT16, pc.INT32, pc.INT64, pc.UINT64):
                idx = col(rng, it, int(rng.integers(0, 80)), 0.2, lo=0, hi=max(n - 1, 0))
                if n == 0:
                    idx = M.Col(it, np.zeros(0, pc.NP_OF[it]))
                want = pa_call(pac.take, to_pa(v), to_pa(idx), boundscheck=True)
                assert_same(M.model("take", [v, idx]), want, ("take", M.NAME[t], M.NAME[it], n))
                if len(idx) and idx.validity()[0] and n + 3 <= np.iinfo(pc.NP_OF[it]).max:
                    idx.values[0] = n + 3
                    assert_same(M.model("take", [v, idx]), pa_call(pac.take, to_pa(v), to_pa(idx)), ("take oob", n))
                    assert M.model("take", [v, idx]).msg == f"{n + 3} out of bounds"


@pytest.mark.parametrize("checked", [False, True])
def test_model_cumulative_sum_matches_pyarrow(checked):
    rng = np.random.default_rng(13 + checked)
    for t in M.NUMERIC:
        for n in (0, 1, 17, 400):
            for skip in (False, True):
                for p_null in (0.0, 0.01):
                    c = col(rng, t, n, p_null, lo=-3 if t in M.SIGNED else 0, hi=3)
                    if t in M.INTS and n > 5 and rng.random() < 0.5:
                        c.values[4] = np.iinfo(c.values.dtype).max                   # an overflow
                    start = M.Sca(t, 2) if rng.random() < 0.5 else None
                    fn = pac.cumulative_sum_checked if checked else pac.cumulative_sum
                    want = pa_call(fn, to_pa(c), start=None if start is None else to_pa(start), skip_nulls=skip)
                    out = M.model("cumulative_sum_checked" if checked else "cumulative_sum", [c], {"skip_nulls": skip, "start": start})
                    assert_same(out, want, (checked, M.NAME[t], n, skip, p_null))


def test_model_is_in_unique_sort_indices_match_pyarrow():
    rng = np.random.default_rng(17)
    for t in M.NUMERIC:
        for n in (0, 1, 30, 700):
            c = col(rng, t, n, 0.2, lo=0, hi=20)
            if t in M.FLOATS and n > 8:
                c.values[:4] = [np.nan, -0.0, 0.0, np.nan]
            s = col(rng, t, 9, 0.2, lo=0, hi=20)
            # MATCH and SKIP are Arrow C++'s skip_nulls=False / True; arrow-go's EMIT_NULL and INCONCLUSIVE have no
            # Arrow C++ counterpart to pin them against (the GPU file checks them against the oracle's ref_is_in)
            for beh, skip in ((pc.NULL_MATCH, False), (pc.NULL_SKIP, True)):
                want = pa_call(pac.is_in, to_pa(c), value_set=to_pa(s), skip_nulls=skip)
                assert_same(M.model("is_in", [c], {"value_set": s, "null_behavior": beh}), want, ("is_in", M.NAME[t], n, beh))
            assert_same(M.model("unique", [c]), pa_call(pac.unique, to_pa(c)), ("unique", M.NAME[t], n))
            for order, pa_order in ((pc.ASCENDING, "ascending"), (pc.DESCENDING, "descending")):
                for placement, pa_place in ((pc.NULLS_AT_END, "at_end"), (pc.NULLS_AT_START, "at_start")):
                    want = pa_call(pac.array_sort_indices, to_pa(c), order=pa_order, null_placement=pa_place)
                    out = M.model("sort_indices", [c], {"order": order, "placement": placement})
                    assert_same(out, want, ("sort_indices", M.NAME[t], n, order, placement))


# ------------------------------------------------------------------------------------------ layouts
@pytest.mark.parametrize("t", [pc.BOOL, pc.UINT8, pc.INT16, pc.FLOAT32, pc.INT64])
def test_layouts_flatten_to_their_column(t):
    rng = np.random.default_rng(23 + t)
    seen = set()
    for case in range(200):
        n = int(rng.choice([0, 1, 7, 8, 9, 63, 64, 65, 1000]))
        lay = M.random_layout(rng, n, max_chunks=int(rng.choice([3, 8, 120])))
        pattern = M.VALIDITY[case % len(M.VALIDITY)]
        valid, bitmap = M.random_validity(rng, n, pattern, lay)
        c = col(rng, t, n, 0)
        c.valid = valid
        pieces = lay.pieces(c, bitmap)
        vals, v = M.flatten(pieces, t)
        assert np.array_equal(vals.view(np.uint8), c.values.view(np.uint8)) and np.array_equal(v, c.validity()), (lay, pattern)
        assert all((p.valid is None) == (not bitmap) for p in pieces)
        # through pyarrow: the same buffers as Arrow arrays with offsets flatten to the same column
        arrs = [pa.Array.from_buffers(PA_TYPE[t], p.length, [None if p.valid is None else pa.py_buffer(np.packbits(p.valid, bitorder="little")),
                                                             pa.py_buffer(np.packbits(p.values, bitorder="little") if t == pc.BOOL else p.values)],
                                      offset=p.offset) for p in pieces]
        flat = pa.chunked_array(arrs, type=PA_TYPE[t]).combine_chunks() if arrs else pa.array([], PA_TYPE[t])
        assert flat.to_pylist() == to_pa(c).to_pylist(), (lay, pattern)
        if lay.chunked:
            lens = [b - a for a, b, _ in lay.ranges(n)]
            seen.update({"empty" for x in lens if x == 0} | {"one" for x in lens if x == 1})
            seen.update({"sliced" for _, _, o in lay.ranges(n) if o})
            seen.update({"in_byte" for a in lay.cuts if a % 8})
        elif lay.form == "slice":
            assert 1 <= lay.offsets[0] <= 17
            seen.add("slice")
        if pattern == "null_chunk" and lay.chunked and n:
            nonempty = [(a, b) for a, b, _ in lay.ranges(n) if b > a]
            assert any(not c.validity()[a:b].any() for a, b in nonempty)
    assert seen >= {"empty", "one", "sliced", "in_byte", "slice"}, seen


def test_independent_cuts_give_hundreds_of_spans():
    """Two operands cut independently into ~120 chunks each give 100-300 aligned spans."""
    rng = np.random.default_rng(29)
    for n in (4097, 8193):
        a, b = M.random_cuts(rng, n, 120), M.random_cuts(rng, n, 120)
        spans = len(set(a) | set(b)) - 1
        assert 100 <= spans <= 300, spans
