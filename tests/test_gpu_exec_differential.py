"""Every registered compute function against the logical-column model of tests/exec_model.py, in the argument shapes
the executor produces: plain arrays, slices at offsets 1-17, chunked arrays with random cuts (empty and one-row
chunks, chunks that are slices, binary operands cut independently into 100-300 spans), valid and null scalars on
either side, five validity patterns, mixed types that promote, and planted failures for the checked functions (in
rows valid on both sides, in rows null in the other operand, and next to span cuts).

Each call is checked for output type and kind, length, null count, every validity bit, the values at valid rows
(floats by bit pattern; NaN equals NaN), the error sentinel and message, and that no input changed."""
import zlib

import numpy as np
import pytest

import exec_model as M
from arrow_go_b200 import compute as pc

gpu = pytest.mark.gpu
TILE_EDGES = {w: [32768 // w - 1, 32768 // w, 32768 // w + 1] for w in (1, 2, 4, 8)}   # a 32 KB tile of each width
SHORT = [0, 1, 7, 8, 9, 63, 64, 65]
EDGES = [4095, 4096, 4097, 8191, 8192, 8193]
WAVES = [1_000_003, 3_000_001]


@pytest.fixture(autouse=True)
def _init(request):
    if request.node.get_closest_marker("gpu"):   # the registry check runs without a device
        request.getfixturevalue("ag")


def rng_for(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


def lengths(rng, t, k=5):
    """k lengths: short ones, 4K/8K edges and the type's tile edges."""
    w = max(M.width(t) // 8, 1)
    pool = SHORT + EDGES + TILE_EDGES[w]
    return [int(x) for x in rng.choice(pool, size=k, replace=False)]


# ------------------------------------------------------------------------------------------ building datums
class Arg:
    """A logical argument and its physical form on the device."""

    def __init__(self, col, layout=None, bitmap=True):
        self.col, self.layout = col, layout
        self.parents = []
        if isinstance(col, M.Sca):
            self.datum = pc.Scalar(col.value, col.type)
            return
        arrs = []
        for p in layout.pieces(col, bitmap):
            full = pc.Array.from_numpy(p.values, p.valid, col.type)
            self.parents.append((full, p))
            arrs.append(full if (p.offset == 0 and p.values.size == p.length) else full.slice(p.offset, p.length))
        self.datum = pc.Chunked(arrs, col.type) if layout.chunked else arrs[0]

    def describe(self):
        if isinstance(self.col, M.Sca):
            return f"scalar {M.NAME[self.col.type]} {self.col.value!r}"
        nulls = "no bitmap" if not self.parents or self.parents[0][1].valid is None else f"{int((~self.col.validity()).sum())} nulls"
        return f"{M.NAME[self.col.type]}[{len(self.col)}] {self.layout!r} {nulls}"

    def check_unchanged(self, what):
        for full, p in self.parents:
            vals, valid, _ = full.to_numpy()
            same = np.array_equal(vals, p.values) if p.values.dtype == np.bool_ else vals.tobytes() == p.values.tobytes()
            assert same, f"{what}: the call changed an input's values ({self.describe()})"
            want_valid = np.ones(p.values.size, dtype=bool) if p.valid is None else p.valid
            assert np.array_equal(valid, want_valid), f"{what}: the call changed an input's validity ({self.describe()})"


def first_diffs(a, b, k=3):
    rows = np.flatnonzero(a != b)[:k]
    return [(int(i), a[i].item(), b[i].item()) for i in rows]


def float_bits_equal(got, want):
    gn, wn = np.isnan(got), np.isnan(want)
    return (gn == wn) & ((got.view(f"u{got.itemsize}") == want.view(f"u{want.itemsize}")) | gn)


def check(name, args, want, call, opts=None):
    """Run `call()` and hold the result to the model's answer `want`."""
    what = f"{name}({', '.join(a.describe() for a in args)}" + (f", {opts}" if opts else "") + ")"
    try:
        got = call()
    except pc.ArrowError as e:
        assert isinstance(want, M.Fail), f"{what}: failed with {e.sentinel}: {e.msg}, the model says it succeeds"
        assert e.sentinel == want.sentinel, f"{what}: {e.sentinel}: {e.msg}, want {want}"
        if want.sentinel != "ErrNotImplemented":
            assert e.msg == want.msg, f"{what}: message {e.msg!r}, want {want.msg!r}"
        got = None
    if got is not None:
        assert not isinstance(want, M.Fail), f"{what}: succeeded, the model says {want}"
        compare(got, want, what)
    for a in args:
        a.check_unchanged(what)


def compare(got, want, what):
    assert got.type == want.type, f"{what}: type {got.type}, want {want.type}"
    assert got.kind == want.kind, f"{what}: kind {got.kind}, want {want.kind}"
    assert len(got) == len(want), f"{what}: length {len(got)}, want {len(want)}"
    if want.type == pc.DICTIONARY:
        idx, valid, nulls = got.indices().to_numpy()
        dvals, dvalid, _ = got.dictionary().to_numpy()
        wd, wdv = want.extra["dictionary"], want.extra["dictionary_valid"]
        assert got.value_type == want.extra["value_type"]
        assert dvals.tobytes() == np.ascontiguousarray(wd).tobytes(), f"{what}: dictionary differs"
        assert np.array_equal(dvalid, np.ones(len(wd), bool) if wdv is None else wdv), f"{what}: dictionary validity differs"
        vals = idx
    else:
        vals, valid, nulls = got.to_numpy()
    assert np.array_equal(valid, want.valid), f"{what}: validity differs at rows (row, got, want) {first_diffs(valid, want.valid)}"
    assert nulls == want.null_count, f"{what}: null count {nulls}, want {want.null_count}"
    care = want.valid
    g, w = np.ascontiguousarray(vals[care]), np.ascontiguousarray(np.asarray(want.values)[care])
    ok = float_bits_equal(g, w) if g.dtype.kind == "f" else (g == w)
    if not ok.all():
        rows = np.flatnonzero(care)[np.flatnonzero(~ok)[:3]]
        diffs = [(int(r), vals[r].item(), np.asarray(want.values)[r].item()) for r in rows]
        raise AssertionError(f"{what}: values differ at rows (row, got, want) {diffs}")


# ------------------------------------------------------------------------------------------ value generators
def values(rng, t, n, kind="full"):
    """'full': the whole range; 'small': a few values around zero (floats: whole numbers, so any sum order is exact);
    'bool': booleans."""
    if t == pc.BOOL:
        return rng.random(n) < 0.5
    dt = np.dtype(pc.NP_OF[t])
    if dt.kind == "f":
        if kind == "small":
            return rng.integers(-8, 9, n).astype(dt)
        v = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)).astype(dt)
        if n > 8:
            v[rng.integers(0, n, 4)] = [np.nan, -0.0, np.inf, 0.0]
        return v
    info = np.iinfo(dt)
    if kind == "small":
        return rng.integers(max(info.min, -8), min(info.max, 8), n, endpoint=True).astype(dt)
    return rng.integers(info.min, info.max, n, endpoint=True, dtype=dt)


def column(rng, t, n, kind="full", layout=None, pattern=None):
    pattern = pattern or M.VALIDITY[int(rng.integers(0, len(M.VALIDITY)))]
    valid, bitmap = M.random_validity(rng, n, pattern, layout)
    return M.Col(t, values(rng, t, n, kind), valid), bitmap


def layout(rng, n, many=False):
    return M.random_layout(rng, n, max_chunks=120 if many else 8)


def cut_rows(layouts, n):
    """Rows on both sides of every cut of the chunked layouts."""
    rows = set()
    for lay in layouts:
        if lay is not None and lay.chunked:
            for c in lay.cuts[1:-1]:
                rows.update(r for r in (c - 1, c) if 0 <= r < n)
    return sorted(rows)


def plant(rng, n, layouts, k=4):
    """Rows for planted failures: random rows and rows next to span cuts."""
    cuts = cut_rows(layouts, n)
    rows = list(rng.integers(0, n, k)) if n else []
    if cuts:
        rows += list(rng.choice(cuts, size=min(k, len(cuts)), replace=False))
    return sorted(set(int(r) for r in rows))


def set_valid(col, rows, flag):
    if not rows:
        return
    if col.valid is None:
        col.valid = np.ones(len(col), dtype=bool)
    col.valid[rows] = flag


# ------------------------------------------------------------------------------------------ binary scalar functions
def failing_pair(name, t):
    """(left, right) values that make the checked kernel of `name` fail on type t, or None."""
    info = np.iinfo(pc.NP_OF[t]) if t in M.INTS else None
    if name in ("add", "sub", "subtract", "multiply") and info is not None:
        return {"add": (info.max, info.max), "multiply": (info.max, info.max)}.get(name, (info.min, info.max))
    if name.startswith("divide"):
        return (7, 0) if (info is not None or name == "divide") else None
    if name.startswith("shift"):
        return (1, M.width(t))
    return None


PROMOTE_PAIRS = [(pc.INT8, pc.UINT8), (pc.UINT16, pc.INT32), (pc.INT32, pc.INT64), (pc.UINT64, pc.INT8), (pc.UINT32, pc.FLOAT32),
                 (pc.INT64, pc.FLOAT64), (pc.FLOAT32, pc.INT16), (pc.UINT8, pc.UINT32)]


def out_of_range(lt, rt):
    """A value of type lt that the promotion of (lt, rt) cannot hold, or None."""
    to = M.common_numeric(lt, rt)
    if lt == pc.UINT64 and to == pc.INT64:
        return np.uint64(1 << 63)
    if lt in (pc.INT64, pc.UINT32, pc.INT32) and to in M.FLOATS:
        return pc.NP_OF[lt]((1 << (24 if to == pc.FLOAT32 else 53)) + 3)
    return None


def binary_cases(name, types, kind="full"):
    """(left, right, opts) cases for a binary scalar function over `types` and promoting pairs."""
    rng = rng_for(name)
    pairs = [(t, t) for t in types]
    if name in M.PROMOTING:
        int_only = name in M.INT_ONLY
        pairs += [p for p in PROMOTE_PAIRS if not (int_only and any(x in M.FLOATS for x in p))]
    for lt, rt in pairs:
        ns = lengths(rng, lt, 3)
        if lt == rt and lt in (pc.INT32, pc.FLOAT64, pc.BOOL):
            ns.append(int(rng.choice(WAVES)))
        for n in ns:
            for shape in ("aa", "aa_many", "as", "sa", "null_l", "null_r"):
                if n > 100_000 and shape not in ("aa", "as"):
                    continue
                many = shape == "aa_many"
                la, lb = layout(rng, n, many), layout(rng, n, many)
                vk = "bool" if lt == pc.BOOL else ("small" if name in ("multiply", "multiply_unchecked") or name.startswith("shift") else kind)
                l, lbm = column(rng, lt, n, vk, la)
                r, rbm = column(rng, rt, n, vk, lb)
                if name.startswith("shift") and rt in M.INTS:
                    r.values[:] = np.abs(r.values.astype(np.int64) % max(M.width(rt) - 1, 1)).astype(r.values.dtype)
                if name.startswith("divide") and rt in M.INTS:
                    r.values[r.values == 0] = 1
                fp = failing_pair(name, lt) if lt == rt else None
                if fp is not None and n:
                    rows = plant(rng, n, [la, lb])
                    for row in rows:
                        l.values[row], r.values[row] = fp
                    # most planted rows are hidden by a null in the other operand; one in three cases keeps one valid
                    hide_right = rng.random() < 0.5
                    set_valid(r if hide_right else l, rows, False)
                    set_valid(l if hide_right else r, rows, True)
                    if rng.random() < 0.33:
                        set_valid(r if hide_right else l, rows[:1], True)
                    lbm = rbm = True
                oor = out_of_range(lt, rt) if lt != rt else None
                if oor is not None and n and rng.random() < 0.5:
                    row = int(rng.integers(0, n))
                    l.values[row] = oor
                    if rng.random() < 0.5:
                        set_valid(l, [row], False)
                        lbm = True
                left, right = Arg(l, la, lbm), Arg(r, lb, rbm)
                if shape in ("as", "null_r") and n:
                    right = Arg(M.Sca(rt, None if shape == "null_r" else r.values[int(rng.integers(0, n))].item()))
                if shape in ("sa", "null_l") and n:
                    left = Arg(M.Sca(lt, None if shape == "null_l" else l.values[int(rng.integers(0, n))].item()))
                yield left, right


def run_binary(name, left, right, opts=None):
    args = [left, right]
    chunked = [i for i, a in enumerate(args) if a.layout is not None and a.layout.chunked]
    want = M.model(name, [left.col, right.col], chunked=chunked)
    check(name, args, want, lambda: pc.CallFunction(name, [left.datum, right.datum], opts))


ARITH_TYPES = {n: (M.INTS if n in M.INT_ONLY else M.NUMERIC) for n in list(M.ARITH) + list(M.NOT_NULL_ARITH)}


@gpu
@pytest.mark.parametrize("name", sorted(ARITH_TYPES))
def test_binary_arithmetic(name):
    for left, right in binary_cases(name, ARITH_TYPES[name]):
        run_binary(name, left, right)


@gpu
@pytest.mark.parametrize("name", sorted(M.CMP))
def test_compare(name):
    for left, right in binary_cases(name, M.NUMERIC, "small"):
        run_binary(name, left, right)


@gpu
@pytest.mark.parametrize("name", sorted(M.BITOP) + sorted(M.KLEENE))
def test_boolean_binary(name):
    rng = rng_for(name, "scalars")
    for left, right in binary_cases(name, [pc.BOOL], "bool"):
        run_binary(name, left, right)
        # both truth values of a valid scalar on either side
        if isinstance(right.col, M.Sca) and right.col.valid:
            run_binary(name, left, Arg(M.Sca(pc.BOOL, not right.col.value)))
        if isinstance(left.col, M.Sca) and left.col.valid:
            run_binary(name, Arg(M.Sca(pc.BOOL, bool(rng.random() < 0.5))), right)


# ------------------------------------------------------------------------------------------ unary scalar functions
UNARY_TYPES = {"abs": M.NUMERIC, "abs_unchecked": M.NUMERIC, "negate": M.SIGNED + M.FLOATS, "negate_unchecked": M.NUMERIC,
               "sign": M.NUMERIC, "bit_wise_not": M.INTS, "not": [pc.BOOL], "is_null": M.NUMERIC + [pc.BOOL],
               "is_not_null": M.NUMERIC + [pc.BOOL], "is_nan": M.NUMERIC}


@gpu
@pytest.mark.parametrize("name", sorted(UNARY_TYPES))
def test_unary(name):
    rng = rng_for(name)
    for t in UNARY_TYPES[name]:
        for n in lengths(rng, t, 4) + ([int(rng.choice(WAVES))] if t in (pc.INT64, pc.FLOAT32, pc.BOOL) else []):
            lay = layout(rng, n, many=rng.random() < 0.3)
            c, bm = column(rng, t, n, "full", lay)
            if name in ("abs", "negate") and t in M.SIGNED and n and rng.random() < 0.5:
                rows = plant(rng, n, [lay], 2)
                c.values[rows] = np.iinfo(pc.NP_OF[t]).min       # fails in a null row too: every slot is checked
            a = Arg(c, lay, bm)
            want = M.model(name, [c], chunked=[0] if lay.chunked else [])
            check(name, [a], want, lambda: pc.CallFunction(name, [a.datum]))


# ------------------------------------------------------------------------------------------ cast
@gpu
@pytest.mark.parametrize("src", M.NUMERIC, ids=lambda t: M.NAME[t])
def test_cast(src):
    rng = rng_for("cast", src)
    for dst in M.NUMERIC:
        for n in lengths(rng, src, 3):
            lay = layout(rng, n, many=rng.random() < 0.3)
            c, bm = column(rng, src, n, "small", lay)
            if src in M.FLOATS and dst in M.INTS:
                c.values[:] = np.trunc(c.values)
            elif src in M.INTS:
                c.values[:] = values(rng, src, n, "full")
                if dst in M.INTS:     # mostly in range, a few rows that are not
                    lo, hi = M.safe_bounds(src, dst)
                    c.values[:] = np.clip(c.values.astype(object), lo, hi).astype(c.values.dtype) if n else c.values
            if n and rng.random() < 0.7:
                rows = plant(rng, n, [lay], 2)
                bad = 2.5 if src in M.FLOATS else (np.iinfo(pc.NP_OF[src]).max if src in M.INTS else None)
                if bad is not None and not (src in M.FLOATS and dst in M.FLOATS):
                    c.values[rows] = bad
                    set_valid(c, rows[1:], False)            # one failing row is valid, the others hidden by a null
                    set_valid(c, rows[:1], rng.random() < 0.7)
                    bm = True
            a = Arg(c, lay, bm)
            opts = {"to": dst}
            if src in M.INTS and dst in M.INTS and rng.random() < 0.2:
                opts["allow_int_overflow"] = True
            want = M.model("cast", [c], opts, chunked=[0] if lay.chunked else [])
            check("cast", [a], want, lambda: pc.Cast(a.datum, dst, allow_int_overflow=opts.get("allow_int_overflow", False)), opts)


@gpu
@pytest.mark.parametrize("t", M.NUMERIC, ids=lambda t: M.NAME[t])
def test_cast_function_without_options_is_invalid(t):
    """cast_<type> called by name with no CastOptions is refused (arrow-go: "function '%s' cannot be called without
    options") rather than dereferencing the missing options, and with options of another kind likewise."""
    fname = {pc.FLOAT32: "cast_float", pc.FLOAT64: "cast_double"}.get(t, "cast_" + M.NAME[t])
    a = pc.Array.from_numpy(np.arange(3, dtype=np.int16))
    with pytest.raises(pc.ArrowError) as e:
        pc.CallFunction(fname, [a])
    assert e.value.sentinel == "ErrInvalid" and e.value.msg == f"function '{fname}' cannot be called without options"
    with pytest.raises(pc.ArrowError) as e:
        pc.CallFunction(fname, [a], ("filter", pc.DROP_NULLS))
    assert e.value.sentinel == "ErrInvalid" and e.value.msg == f"{fname}: expected CastOptions, got FilterOptions"


# ------------------------------------------------------------------------------------------ filter / take
@gpu
@pytest.mark.parametrize("name", ["filter", "array_filter"])
def test_filter(name):
    rng = rng_for(name)
    for t in M.NUMERIC + [pc.BOOL]:
        for n in lengths(rng, t, 3) + ([int(rng.choice(WAVES))] if t in (pc.INT64, pc.BOOL) else []):
            for sel in (pc.DROP_NULLS, pc.EMIT_NULLS):
                many = n < 100_000 and rng.random() < 0.4
                lv, lm = layout(rng, n, many), layout(rng, n, many)
                v, vbm = column(rng, t, n, "full", lv)
                m, mbm = column(rng, pc.BOOL, n, "bool", lm)
                a, b = Arg(v, lv, vbm), Arg(m, lm, mbm)
                chunked = [i for i, x in enumerate((a, b)) if x.layout.chunked]
                want = M.model(name, [v, m], {"null_selection": sel}, chunked=chunked)
                check(name, [a, b], want, lambda: pc.CallFunction(name, [a.datum, b.datum], ("filter", sel)), {"null_selection": sel})


@gpu
@pytest.mark.parametrize("name", ["take", "array_take"])
def test_take(name):
    rng = rng_for(name)
    for t in M.NUMERIC + [pc.BOOL]:
        for it in (pc.INT8, pc.UINT16, pc.INT32, pc.UINT32, pc.INT64, pc.UINT64):
            for n in lengths(rng, t, 2):
                nv = int(rng.choice([1, 5, 127, 4097, 70_000])) if n else int(rng.choice([0, 3]))
                nv = min(nv, int(np.iinfo(pc.NP_OF[it]).max) - 3)
                # values: chunked (through the concatenation of its chunks) except booleans and array_take
                lv = layout(rng, nv, many=rng.random() < 0.3) if (t != pc.BOOL and name == "take") else M.random_layout(rng, nv, form=str(rng.choice(["array", "slice"])))
                li = layout(rng, n) if name == "take" else M.random_layout(rng, n, form=str(rng.choice(["array", "slice"])))
                v, vbm = column(rng, t, nv, "full", lv)
                idx, ibm = column(rng, it, n, "full", li)
                idx.values[:] = rng.integers(0, max(nv, 1), n) if nv else 0
                if n and rng.random() < 0.3:
                    rows = plant(rng, n, [li], 2)
                    idx.values[rows] = nv + int(rng.integers(0, 3))
                    set_valid(idx, rows[1:], False)
                    set_valid(idx, rows[:1], rng.random() < 0.6)
                    ibm = True
                if nv == 0 and n:
                    idx.valid = np.zeros(n, dtype=bool)
                    ibm = True
                a, b = Arg(v, lv, vbm), Arg(idx, li, ibm)
                want = M.model(name, [v, idx], chunked=[i for i, x in enumerate((a, b)) if x.layout.chunked])
                check(name, [a, b], want, lambda: pc.CallFunction(name, [a.datum, b.datum]))


# ------------------------------------------------------------------------------------------ cumulative_sum
@gpu
@pytest.mark.parametrize("name", ["cumulative_sum", "cumulative_sum_checked"])
def test_cumulative_sum(name):
    rng = rng_for(name)
    checked = name.endswith("_checked")
    for t in M.NUMERIC:
        for n in lengths(rng, t, 3) + ([int(rng.choice(WAVES))] if t in (pc.INT64, pc.FLOAT64) else []):
            for skip in (False, True):
                lay = layout(rng, n, many=n < 100_000 and rng.random() < 0.3)
                pattern = str(rng.choice(["none", "zero_nulls", "nulls_10", "null_chunk"])) if rng.random() < 0.5 else "none"
                c, bm = column(rng, t, n, "small", lay, pattern)
                if t in M.INTS and c.values.dtype.kind == "u":
                    c.values[:] = np.abs(c.values.astype(np.int64)).astype(c.values.dtype)
                if t in M.INTS and n and rng.random() < 0.4:
                    c.values[plant(rng, n, [lay], 1)] = np.iinfo(pc.NP_OF[t]).max
                # no start, a start of another type (safe-cast to t, 300 fails for 8-bit t), a null start
                start = [None, None, M.Sca(pc.INT8, 3), M.Sca(pc.INT64, 300), M.Sca(pc.FLOAT64, 2.0), M.Sca(t, 1),
                         M.Sca(pc.INT64, None)][int(rng.integers(0, 7))]
                a = Arg(c, lay, bm)
                opts = {"skip_nulls": skip, "start": start}
                want = M.model(name, [c], opts, chunked=[0] if lay.chunked else [])
                sd = None if start is None else pc.Scalar(start.value, start.type)
                check(name, [a], want, lambda: pc.CumulativeSum(a.datum, start=sd, skip_nulls=skip, checked=checked),
                      {"skip_nulls": skip, "start": None if start is None else (M.NAME[start.type], start.value)})


@gpu
@pytest.mark.parametrize("checked", [False, True])
def test_cumulative_sum_empty_input_checks_start(checked):
    """The start value is checked when the kernel state is set up, which happens for every call: an empty input with a
    null start, or a start the safe cast refuses, fails like a non-empty one."""
    for empty in (pc.Array.from_numpy(np.zeros(0, np.uint64)), pc.Array.from_numpy(np.arange(4, dtype=np.int8)).slice(4, 0),
                  pc.Chunked([pc.Array.from_numpy(np.zeros(0, np.int32))], pc.INT32)):
        with pytest.raises(pc.ArrowError) as e:
            pc.CumulativeSum(empty, start=pc.Scalar(None, pc.INT64), checked=checked)
        assert e.value.sentinel == "ErrInvalid" and e.value.msg == "cumulative sum start value must be valid"
    with pytest.raises(pc.ArrowError) as e:
        pc.CumulativeSum(pc.Array.from_numpy(np.zeros(0, np.int8)), start=pc.Scalar(300, pc.INT64), checked=checked)
    assert e.value.msg == "cannot cast cumulative sum start value to int8: integer value 300 not in range: -128 to 127"
    out = pc.CumulativeSum(pc.Array.from_numpy(np.zeros(0, np.int8)), start=pc.Scalar(3, pc.INT64), checked=checked)
    assert out.type == pc.INT8 and len(out) == 0


# ------------------------------------------------------------------------------------------ sort_indices / unique / is_in
def one_array_layout(rng, n):
    form = str(rng.choice(["array", "slice", "one_chunk"]))
    if form != "one_chunk":
        return M.random_layout(rng, n, form=form)
    return M.Layout("chunked", cuts=[0, n], offsets=[int(rng.integers(0, 18))], pad=3, seed=int(rng.integers(0, 1 << 31)))


@gpu
@pytest.mark.parametrize("name", ["sort_indices", "unique", "is_in"])
def test_one_array_functions(name):
    rng = rng_for(name)
    for t in M.NUMERIC:
        for n in lengths(rng, t, 3) + ([int(rng.choice(WAVES))] if t in (pc.INT32, pc.FLOAT64) else []):
            lay = one_array_layout(rng, n)
            c, bm = column(rng, t, n, "small" if rng.random() < 0.6 else "full", lay)
            a = Arg(c, lay, bm)
            chunked = [0] if lay.chunked else []
            if name == "sort_indices":
                order, place = int(rng.integers(0, 2)), int(rng.integers(0, 2))
                want = M.model(name, [c], {"order": order, "placement": place}, chunked=chunked)
                check(name, [a], want, lambda: pc.SortIndices(a.datum, order, place), {"order": order, "placement": place})
            elif name == "unique":
                # compare() reads values at valid rows only, which skips the unspecified value under unique's null slot
                check(name, [a], M.model(name, [c], chunked=chunked), lambda: pc.Unique(a.datum))
            else:
                s, _ = column(rng, t, int(rng.integers(0, 40)), "small")
                sd = pc.Array.from_numpy(s.values, s.valid, t)
                for beh in range(4):
                    want = M.model(name, [c], {"value_set": s, "null_behavior": beh}, chunked=chunked)
                    check(name, [a], want, lambda: pc.IsIn(a.datum, sd, beh), {"null_behavior": beh})
        # a column of several chunks is refused
        c = M.Col(t, values(rng, t, 10))
        lay = M.Layout("chunked", cuts=[0, 4, 10], offsets=[0, 1], seed=1)
        a = Arg(c, lay)
        call = {"sort_indices": lambda: pc.SortIndices(a.datum), "unique": lambda: pc.Unique(a.datum),
                "is_in": lambda: pc.IsIn(a.datum, pc.Array.from_numpy(c.values[:2]))}[name]
        check(name, [a], M.model(name, [c], {"chunks": 2, "value_set": M.Col(t, c.values[:2])}, chunked=[0]), call)


# ------------------------------------------------------------------------------------------ dictionary_encode / run ends
@gpu
def test_dictionary_encode():
    rng = rng_for("dictionary_encode")
    for t in M.NUMERIC:
        for n in lengths(rng, t, 3):
            for enc in (pc.NULL_ENCODING_MASK, pc.NULL_ENCODING_ENCODE):
                lay = layout(rng, n, many=rng.random() < 0.3)
                c, bm = column(rng, t, n, "small", lay)
                a = Arg(c, lay, bm)
                want = M.model("dictionary_encode", [c], {"null_encoding": enc}, chunked=[0] if lay.chunked else [])
                check("dictionary_encode", [a], want, lambda: pc.DictionaryEncode(a.datum, enc), {"null_encoding": enc})


def runs_column(rng, t, n, lay):
    """A column of runs: few distinct values repeated, nulls in runs too."""
    c, bm = column(rng, t, n, "bool" if t == pc.BOOL else "small", lay)
    if n:
        reps = rng.integers(1, 40, n)
        src = np.repeat(np.arange(n), reps)[:n]
        c.values[:] = c.values[src]
        if c.valid is not None:
            c.valid[:] = c.valid[src]
    return c, bm


@gpu
def test_run_end_encode_and_decode():
    rng = rng_for("run_end")
    for t in M.NUMERIC + [pc.BOOL]:
        for n in lengths(rng, t, 3):
            rt = [pc.INT16, pc.INT32, pc.INT64][int(rng.integers(0, 3))]
            if rt == pc.INT16 and n > 32767:
                rt = pc.INT32
            lay = layout(rng, n, many=rng.random() < 0.3)
            c, bm = runs_column(rng, t, n, lay)
            a = Arg(c, lay, bm)
            what = f"run_end_encode({a.describe()}, {M.NAME[rt]})"
            out = pc.RunEndEncode(a.datum, rt)
            a.check_unchanged(what)
            assert out.type == pc.RUN_END_ENCODED and out.run_end_type == rt and out.value_type == t, what
            assert out.kind == (pc.KIND_CHUNKED if lay.chunked else pc.KIND_ARRAY) and len(out) == n, what
            # chunk by chunk: runs never cross a chunk boundary, and an empty chunk is dropped
            spans = [(s, e) for s, e, _ in lay.ranges(n) if e > s] if lay.chunked else [(0, n)]
            if lay.chunked and not spans:
                spans = [(0, 0)]
            chunks = out.chunks() if lay.chunked else [out]
            assert len(chunks) == len(spans), (what, len(chunks), len(spans))
            for (s, e), ch in zip(spans, chunks):
                ends, vals, rvalid = M.run_end_encode(c.values[s:e], None if c.valid is None else c.valid[s:e], rt)
                gends = ch.run_ends().to_numpy()[0]
                gvals, gvalid, _ = ch.values().to_numpy()
                assert np.array_equal(gends.astype(np.int64), ends), (what, s, e, first_diffs(gends.astype(np.int64), ends) if gends.size == ends.size else (gends.size, ends.size))
                wv = np.ones(len(vals), bool) if rvalid is None else rvalid
                assert np.array_equal(gvalid, wv), (what, s, e)
                assert gvals[wv].tobytes() == np.asarray(vals)[wv].tobytes(), (what, s, e)
            # run_end_decode gives the logical column back, whole and from a slice of each encoded array
            dec = pc.RunEndDecode(out)
            compare(dec, M.Out(t, c.values, c.valid, out.kind), f"run_end_decode({what})")
            if n >= 3 and not lay.chunked:
                o, k = int(rng.integers(1, n // 2 + 1)), int(rng.integers(0, n // 2))
                dec = pc.RunEndDecode(out.slice(o, k))
                compare(dec, M.Out(t, c.values[o:o + k], None if c.valid is None else c.valid[o:o + k], pc.KIND_ARRAY),
                        f"run_end_decode(slice({o}, {k}) of {what})")


# ------------------------------------------------------------------------------------------ registry coverage
COVERED = (set(ARITH_TYPES) | set(M.CMP) | set(M.BITOP) | set(M.KLEENE) | set(UNARY_TYPES)
           | {"cast", "filter", "array_filter", "take", "array_take", "cumulative_sum", "cumulative_sum_checked",
              "sort_indices", "unique", "is_in", "dictionary_encode", "run_end_encode", "run_end_decode"})
# cast_<type> are the kernels behind "cast"; test_cast runs every one of them through it, and
# test_cast_function_without_options_is_invalid calls each by name
EXCLUDED = {f"cast_{x}": "runs under 'cast' in test_cast (it needs CastOptions, which CallFunction by name cannot pass)"
            for x in ("int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float", "double")}


def test_registry_is_covered():
    """Every registered function is either exercised here or excluded with a reason."""
    names = set(pc.function_names())
    missing = names - COVERED - set(EXCLUDED)
    assert not missing, f"registered functions that tests/test_gpu_exec_differential.py neither covers nor excludes: {sorted(missing)}"
    stale = (COVERED | set(EXCLUDED)) - names
    assert not stale, f"covered or excluded names that are not registered: {sorted(stale)}"
