"""ExecuteScalarExpression: expression trees over record batches and tables, evaluated as one fused device program.

The contract is the tree evaluated node by node with CallFunction (post-order, arguments left to right): the same
type, validity and values at valid rows, and on failure the same error sentinel and message.  Every tree is checked
against two oracles: (a) the tree walked in Python through pc.CallFunction / pc.Cast, and (b) a fold of
exec_model.model over the tree, which computes every slot with the C restatements of the kernels and never runs the
library.  test_fused_coverage checks that the trees really run as one expr_eval_kernel launch.
"""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

from arrow_go_b200 import _native as N
from arrow_go_b200 import compute as pc

import exec_model as M

SHORT = [0, 1, 7, 8, 9, 63, 64, 65]
EDGES = [1023, 1024, 1025, 4095, 4096, 4097]
BIG = [1_000_003, 3_000_017]

gpu = pytest.mark.gpu


def _rng(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


# ---------------------------------------------------------------- trees -----------------------------------------
# ("field", i) | ("lit", value, type) | ("call", name, [args], options) | ("cast", arg, type, allow_int, allow_float)
def build(t):
    if t[0] == "field":
        return pc.Field(t[1])
    if t[0] == "lit":
        return pc.Literal(t[1], t[2])
    if t[0] == "cast":
        return pc.CastExpr(build(t[1]), t[2], t[3], t[4])
    return pc.Call(t[1], [build(a) for a in t[2]], t[3])


def node_by_node(t, cols):
    if t[0] == "field":
        return cols[t[1]]
    if t[0] == "lit":
        return pc.Scalar(t[1], t[2])
    if t[0] == "cast":
        return pc.Cast(node_by_node(t[1], cols), t[2], t[3], t[4])
    return pc.CallFunction(t[1], [node_by_node(a, cols) for a in t[2]], t[3])


def cast_model(a, to, allow_int, allow_float):
    if a.type == to:
        return a
    if a.type == pc.BOOL or to == pc.BOOL:
        return M.Fail("ErrNotImplemented", None)
    if isinstance(a, M.Sca):
        if a.value is None:
            return M.Sca(to, None)
        c, f = M.cast_col(M.Col(a.type, a.raw()), to, allow_int, allow_float)
        return f or M.Sca(to, c.values[0].item())
    c, f = M.cast_col(a, to, allow_int, allow_float)
    return f or c


def fold(t, mcols):
    """Oracle (b): exec_model.model folded over the tree; an M.Col / M.Sca, or an M.Fail (message None where the model
    does not word it: a call that does not dispatch, an all-literal call)."""
    if t[0] == "field":
        return mcols[t[1]]
    if t[0] == "lit":
        return M.Sca(t[2], t[1])
    if t[0] == "cast":
        a = fold(t[1], mcols)
        return a if isinstance(a, M.Fail) else cast_model(a, t[2], t[3], t[4])
    args = []
    for a in t[2]:
        r = fold(a, mcols)
        if isinstance(r, M.Fail):
            return r
        args.append(r)
    arity = ARITY.get(t[1], 1 if t[1].startswith("cast_") else None)
    if arity is None or arity != len(args):   # no function registered / the wrong number of arguments
        return M.Fail("ErrInvalid", None)
    if all(isinstance(a, M.Sca) for a in args):
        return M.Fail("ErrNotImplemented", None)
    try:
        pc.dispatch_best(t[1], [a.type for a in args])
    except pc.ArrowError as e:
        return M.Fail(e.sentinel, None)
    if t[1].startswith("cast_"):   # cast_<type> by name: its CastOptions are the call's
        if t[3] is None:
            return M.Fail("ErrInvalid", None)
        return cast_model(args[0], *t[3][1])
    r = M.model(t[1], args)
    return r if isinstance(r, M.Fail) else M.Col(r.type, r.values, r.valid)


def model_columns(cols):
    out = []
    for c in cols:
        v, m, _ = c.to_numpy()
        out.append(M.Col(c.type, v, m))
    return out


def same_as_model(got, want):
    assert got.type == want.type
    if isinstance(want, M.Sca):
        assert repr(pc.scalar_value(got)) == repr(want.value)
        return
    gv, gm, _ = got.to_numpy()
    wm = want.validity()
    assert np.array_equal(gm, wm), "validity (model)"
    wv = want.values
    if want.type in (pc.FLOAT32, pc.FLOAT64):
        gn, wn = np.isnan(gv[wm]), np.isnan(wv[wm])
        assert np.array_equal(gn, wn)
        assert np.array_equal(gv[wm][~gn].view(np.uint8), wv[wm][~wn].view(np.uint8))
    else:
        assert np.array_equal(gv[wm], wv[wm].astype(gv.dtype))


def outcome(fn):
    try:
        return "ok", fn()
    except pc.ArrowError as e:
        return "err", (e.sentinel, e.msg)


def snapshot(cols):
    return [c.to_numpy()[:2] if c.type == pc.BOOL or c.type in pc.NP_OF else (np.zeros(0), np.zeros(0)) for c in cols]


def same_logical(got, want):
    assert got.type == want.type
    assert got.kind == want.kind
    if want.kind == pc.KIND_SCALAR:
        assert repr(pc.scalar_value(got)) == repr(pc.scalar_value(want))
        return
    assert len(got) == len(want)
    gv, gm, _ = got.to_numpy()
    wv, wm, _ = want.to_numpy()
    assert np.array_equal(gm, wm), "validity"
    if want.type in (pc.FLOAT32, pc.FLOAT64):
        gn, wn = np.isnan(gv[wm]), np.isnan(wv[wm])
        assert np.array_equal(gn, wn)
        assert np.array_equal(gv[wm][~gn].view(np.uint8), wv[wm][~wn].view(np.uint8))
    else:
        assert np.array_equal(gv[wm], wv[wm])


def check(tree, cols, table):
    """The fused result against the node-by-node oracle, and the inputs unchanged."""
    before = snapshot(cols)
    data = pc.Table(cols) if table else pc.RecordBatch(cols)
    got = outcome(lambda: pc.ExecuteScalarExpression(build(tree), data))
    want = outcome(lambda: node_by_node(tree, cols))
    assert got[0] == want[0], (got, want, tree)
    if got[0] == "err":
        assert got[1] == want[1], tree
    else:
        same_logical(got[1], want[1])
    if all(c.type == pc.BOOL or c.type in pc.NP_OF for c in cols):
        m = fold(tree, model_columns(cols))
        if got[0] == "err":
            assert isinstance(m, M.Fail) and m.sentinel == got[1][0], (m, got, tree)
            assert m.msg is None or m.msg == got[1][1], (m, got, tree)
        else:
            assert not isinstance(m, M.Fail), (m, tree)
            same_as_model(got[1], m)
    after = snapshot(cols)
    for (bv, bm), (av, am) in zip(before, after):
        assert np.array_equal(bm, am) and bv.tobytes() == av.tobytes()
    return got


# ---------------------------------------------------------------- inputs ----------------------------------------
def values(rng, t, n):
    if t == pc.BOOL:
        return rng.random(n) < 0.5
    dt = np.dtype(M.np_of(t))
    if t in M.FLOATS:
        v = rng.standard_normal(n) * 100
        v[rng.random(n) < 0.02] = np.nan
        return v.astype(dt)
    info = np.iinfo(dt)
    small = rng.integers(max(info.min, -100), min(info.max, 100), n, endpoint=True)
    big = rng.integers(info.min, info.max, n, endpoint=True, dtype=dt)
    return np.where(rng.random(n) < 0.1, big, small.astype(dt)).astype(dt)


def column(rng, t, n, table, nulls=None):
    v = values(rng, t, n)
    pattern = nulls if nulls is not None else rng.choice(["none", "zero_nulls", "nulls_10", "nulls_90"])
    valid = {"none": None, "zero_nulls": np.ones(n, bool), "nulls_10": rng.random(n) >= 0.1, "nulls_90": rng.random(n) >= 0.9}[pattern]
    off = int(rng.integers(0, 13))   # a slice at an odd element offset and a bitmap offset that is not a multiple of 8
    pad_v = np.concatenate([values(rng, t, off), v]) if off else v
    pad_m = None if valid is None else np.concatenate([rng.random(off) < 0.5, valid])
    arr = pc.Array.from_numpy(pad_v, valid=pad_m, type_id=t).slice(off, n) if off else pc.Array.from_numpy(v, valid=valid, type_id=t)
    if not table:
        return arr
    k = int(rng.choice([1, 2, 16])) if n else int(rng.choice([0, 1]))
    cuts = sorted(rng.integers(0, n + 1, max(k - 1, 0)).tolist()) if n else []
    bounds = [0] + cuts + [n]
    return pc.Chunked([arr.slice(a, b - a) for a, b in zip(bounds[:-1], bounds[1:])] if k else [], t)


# ---------------------------------------------------------------- random trees ----------------------------------
BINARY = list(M.ARITH) + list(M.NOT_NULL_ARITH) + list(M.CMP)
BOOLEAN = list(M.BITOP) + list(M.KLEENE)
UNARY_NUM = list(M.UNARY)
ARITY = {**{n: 2 for n in BINARY + BOOLEAN}, **{n: 1 for n in UNARY_NUM + ["not", "is_null", "is_not_null", "is_nan"]}}


def random_tree(rng, types, depth, vals=values):
    """A tree whose leaves are the columns `types` (indices) and literals (drawn by `vals`); mixed types so promotion
    (and its failures) happen."""
    r = rng.random()
    if depth <= 0 or r < 0.15:
        if rng.random() < 0.8:
            return ("field", int(rng.integers(0, len(types))))
        t = int(rng.choice(M.NUMERIC))
        return ("lit", None if rng.random() < 0.15 else vals(rng, t, 1)[0].item(), t)
    kind = rng.random()
    if kind < 0.45:
        name = str(rng.choice(BINARY))
        return ("call", name, [random_tree(rng, types, depth - 1, vals), random_tree(rng, types, depth - 1, vals)], None)
    if kind < 0.6:
        name = str(rng.choice(BOOLEAN))
        args = [("call", str(rng.choice(list(M.CMP))), [random_tree(rng, types, depth - 2, vals), random_tree(rng, types, depth - 2, vals)], None)
                if rng.random() < 0.7 else ("call", str(rng.choice(["is_null", "is_not_null", "is_nan"])), [random_tree(rng, types, depth - 2, vals)], None)
                for _ in range(2)]
        return ("call", name, args, None)
    if kind < 0.65:
        return ("call", "not", [("call", str(rng.choice(list(M.CMP))), [random_tree(rng, types, depth - 1, vals), random_tree(rng, types, depth - 1, vals)], None)], None)
    if kind < 0.85:
        return ("call", str(rng.choice(UNARY_NUM)), [random_tree(rng, types, depth - 1, vals)], None)
    return ("cast", random_tree(rng, types, depth - 1, vals), int(rng.choice(M.NUMERIC)), bool(rng.random() < 0.5), bool(rng.random() < 0.5))


CASES = [(n, table, seed) for n in SHORT + EDGES for table in (False, True) for seed in range(3)]


@gpu
@pytest.mark.parametrize("n,table,seed", CASES)
def test_random_trees(n, table, seed):
    rng = _rng("expr", n, table, seed)
    types = [int(rng.choice(M.NUMERIC)) for _ in range(int(rng.integers(2, 5)))]
    cols = [column(rng, t, n, table) for t in types]
    for _ in range(6):
        check(random_tree(rng, types, int(rng.integers(1, 6))), cols, table)


@gpu
@pytest.mark.parametrize("n", BIG)
@pytest.mark.parametrize("table", [False, True])
def test_random_trees_large(n, table):
    rng = _rng("expr-large", n, table)
    types = [pc.INT32, pc.FLOAT64, pc.INT64, pc.UINT8]
    cols = [column(rng, t, n, table, nulls="nulls_10") for t in types]
    for _ in range(3):
        check(random_tree(rng, types, 4), cols, table)


def small_values(rng, t, n):
    """Values in [1, 5]: no checked op, shift, division or cast fails on them, so a tree fails only where it does not
    dispatch."""
    if t == pc.BOOL:
        return rng.random(n) < 0.5
    return rng.integers(1, 6, n).astype(M.np_of(t))


FUSED_NAMES = set(BINARY) | set(BOOLEAN) | set(UNARY_NUM) | {"not", "is_null", "is_not_null", "is_nan", "cast"}


def call_names(t):
    if t[0] == "cast":
        return {"cast"} | call_names(t[1])
    if t[0] == "call":
        return {t[1]}.union(*[call_names(a) for a in t[2]])
    return set()


@gpu
@pytest.mark.parametrize("table", [False, True])
def test_fused_coverage(table):
    """Every random tree that succeeds and is rooted at a call runs as exactly one expr_eval_kernel launch, and every
    fused function occurs in such a tree: the differential above does not pass on the node-by-node route alone."""
    pytest.importorskip("torch")
    rng = _rng("coverage", table)
    n = 3000
    types = [pc.INT32, pc.INT64, pc.FLOAT64, pc.UINT16, pc.INT8, pc.FLOAT32]
    cols = []
    for t in types:
        arr = pc.Array.from_numpy(small_values(rng, t, n), valid=rng.random(n) >= 0.1, type_id=t)
        cols.append(pc.Chunked([arr.slice(0, 1000), arr.slice(1000, 2000)], t) if table else arr)
    data = pc.Table(cols) if table else pc.RecordBatch(cols)
    # one tree per fused function, then random ones
    f0, f1, f2 = ("field", 0), ("field", 1), ("field", 2)
    trees = [("call", b, [f0, f1], None) for b in BINARY] + [("call", u, [f0], None) for u in UNARY_NUM]
    trees += [("call", b, [("call", "greater", [f0, f1], None), ("call", "less", [f2, f0], None)], None) for b in BOOLEAN]
    trees += [("call", "not", [("call", "equal", [f0, f2], None)], None), ("cast", f0, pc.FLOAT32, False, False)]
    trees += [("call", u, [f2], None) for u in ("is_null", "is_not_null", "is_nan")]
    trees += [random_tree(rng, types, int(rng.integers(1, 4)), vals=small_values) for _ in range(100)]
    seen, fused, unfused = set(), 0, []
    for tree in trees:
        if tree[0] not in ("call", "cast"):
            continue
        if tree[0] == "cast" and tree[1][0] == "field" and types[tree[1][1]] == tree[2]:
            continue   # a cast to the column's own type is the column: nothing to run
        res = {}
        names = _kernel_names(lambda: res.update(r=outcome(lambda: pc.ExecuteScalarExpression(build(tree), data))))
        if res["r"][0] != "ok" or res["r"][1].kind == pc.KIND_SCALAR:
            continue
        if sum("expr_eval_kernel" in k for k in names) == 1:
            fused += 1
            seen |= call_names(tree)
        else:
            unfused.append(tree)
        check(tree, cols, table)
    assert not unfused, unfused[:3]
    assert fused >= 40, fused
    assert FUSED_NAMES <= seen, sorted(FUSED_NAMES - seen)


@gpu
@pytest.mark.parametrize("table", [False, True])
def test_is_in_in_an_expression(table):
    a = i64([1, 2, 3, 4, 5, 2], [True, True, False, True, True, True])
    vs = i64([2, 4, 9])
    col = pc.Chunked([a], pc.INT64) if table else a   # is_in takes one array (a chunk)
    data = pc.Table([col]) if table else pc.RecordBatch([col])
    e = pc.Call("and_kleene", [pc.IsInExpr(pc.Field(0), vs), pc.Call("greater", [pc.Field(0), pc.Literal(3, pc.INT64)])])
    got = pc.ExecuteScalarExpression(e, data)
    want = pc.CallFunction("and_kleene", [pc.IsIn(col, vs), pc.CallFunction("greater", [col, pc.Scalar(3, pc.INT64)])])
    same_logical(got, want)
    assert got.to_pylist() == [False, False, False, True, False, False]   # is_in of a null row is false (NullMatchingMatch)
    names = _kernel_names(lambda: pc.ExecuteScalarExpression(e, data))
    assert sum("expr_eval_kernel" in k for k in names) == 1, names


@gpu
def test_cast_functions_by_name():
    f = pc.Array.from_numpy(np.array([1.0, 2.5, 300.0, -4.0]), valid=np.array([True, True, True, False]), type_id=pc.FLOAT64)
    cases = [
        (("call", "cast_int32", [("field", 0)], ("cast", (pc.INT32, False, True))), "ok"),
        (("call", "cast_int32", [("field", 0)], ("cast", (pc.INT32, False, False))), "err"),   # 2.5 is truncated
        (("call", "cast_int8", [("call", "abs", [("field", 0)], None)], ("cast", (pc.INT8, False, False))), "err"),   # 2.5
        (("call", "cast_int8", [("call", "abs", [("field", 0)], None)], ("cast", (pc.INT8, False, True))), "ok"),   # 300 wraps
        (("call", "cast_int8", [("field", 0)], ("cast", (pc.INT8, True, True))), "ok"),
        (("call", "cast_uint16", [("field", 0)], None), "err"),   # called without options
        (("call", "add", [("call", "cast_double", [("field", 0)], ("cast", (pc.FLOAT64, False, False))),
                          ("cast", ("lit", 7, pc.INT32), pc.FLOAT64, False, False)], None), "ok"),   # a cast literal folds
    ]
    for tree, want in cases:
        assert check(tree, [f], False)[0] == want, tree
        assert check(tree, [pc.Chunked([f.slice(0, 1), f.slice(1, 3)], pc.FLOAT64)], True)[0] == want, tree


# ---------------------------------------------------------------- values under nulls ----------------------------
def i64(vals, valid=None):
    return pc.Array.from_numpy(np.array(vals, dtype=np.int64), valid=None if valid is None else np.array(valid), type_id=pc.INT64)


@gpu
def test_payload_under_null_decides():
    big = 1 << 40
    a = i64([1, big, 3], [True, False, True])
    b = i64([1, big, 3])
    # add_unchecked computes every slot (big + big under the null); the checked multiply fails there
    t = ("call", "multiply", [("call", "add_unchecked", [("field", 0), ("field", 1)], None), ("lit", 1 << 30, pc.INT64)], None)
    assert check(t, [a, b], False)[0] == "err"
    # the checked add writes 0 under a null, so the same multiply passes
    t = ("call", "multiply", [("call", "add", [("field", 0), ("field", 1)], None), ("lit", 1 << 30, pc.INT64)], None)
    assert check(t, [a, b], False)[0] == "ok"
    # a checked add over a null slot whose payload would overflow does not fail
    m = i64([1, (1 << 63) - 1, 2], [True, False, True])
    assert check(("call", "add", [("field", 0), ("lit", 5, pc.INT64)], None), [m], False)[0] == "ok"
    # a null literal on a checked op: nothing is computed, the other side still runs
    assert check(("call", "multiply", [("field", 0), ("lit", None, pc.INT64)], None), [a], False)[0] == "ok"
    assert check(("call", "multiply", [("call", "negate", [("lit", None, pc.INT64)], None), ("field", 0)], None), [a], False)[0] == "err"


@gpu
def test_divide_shift_and_casts():
    a = i64([4, 5, 6])
    z = i64([2, 0, 3], [True, True, True])
    zn = i64([2, 0, 3], [True, False, True])
    assert check(("call", "divide", [("field", 0), ("field", 1)], None), [a, z], False)[0] == "err"
    assert check(("call", "divide", [("field", 0), ("field", 1)], None), [a, zn], False)[0] == "ok"
    assert check(("call", "shift_left", [("field", 0), ("lit", 70, pc.INT64)], None), [a], False)[0] == "err"
    assert check(("call", "shift_left_unchecked", [("field", 0), ("lit", 70, pc.INT64)], None), [a], False)[0] == "ok"
    # uint64 beyond INT64_MAX meeting int8: the implicit safe cast to int64 fails
    u = pc.Array.from_numpy(np.array([1, 1 << 63], dtype=np.uint64), type_id=pc.UINT64)
    s = pc.Array.from_numpy(np.array([1, 2], dtype=np.int8), type_id=pc.INT8)
    assert check(("call", "add", [("field", 0), ("field", 1)], None), [u, s], False)[0] == "err"
    # an explicit cast fails, and passes with its allow flags
    f = pc.Array.from_numpy(np.array([1.5, 300.0]), type_id=pc.FLOAT64)
    assert check(("cast", ("field", 0), pc.INT8, False, False), [f], False)[0] == "err"
    assert check(("cast", ("field", 0), pc.INT8, True, True), [f], False)[0] == "ok"
    assert check(("cast", ("call", "abs", [("field", 0)], None), pc.INT32, False, True), [pc.Chunked([f], pc.FLOAT64)], True)[0] == "ok"


# ---------------------------------------------------------------- refusals --------------------------------------
@gpu
def test_refusals():
    a = i64([1, 2, 3])
    d = pc.DictionaryEncode(a)
    r = pc.RunEndEncode(a, pc.INT32)
    # no CallFunction equivalent: a field index out of range, and vector or meta functions (exec.go:625-627)
    for e in (pc.Call("add", [pc.Field(5), pc.Field(0)]), pc.Call("cumulative_sum", [pc.Field(0)]), pc.Call("unique", [pc.Field(0)]),
              pc.Call("sort_indices", [pc.Field(0)])):
        with pytest.raises(pc.ArrowError) as err:
            pc.ExecuteScalarExpression(e, pc.RecordBatch([a]))
        assert err.value.sentinel == "ErrInvalid"
    # the same status and message as CallFunction node by node
    cases = [
        (("call", "add", [("lit", 1, pc.INT64), ("lit", 2, pc.INT64)], None), [a], "ErrNotImplemented"),
        (("call", "no_such_function", [("field", 0)], None), [a], "ErrInvalid"),
        (("call", "add", [("field", 0)], None), [a], "ErrInvalid"),
        (("call", "add", [("field", 0), ("field", 0)], None), [d], "ErrNotImplemented"),
        (("call", "add", [("field", 0), ("field", 0)], None), [r], "ErrNotImplemented"),
    ]
    for tree, cols, sentinel in cases:
        got = check(tree, cols, False)
        assert got[0] == "err" and got[1][0] == sentinel, (tree, got)


# ---------------------------------------------------------------- capacity --------------------------------------
@gpu
@pytest.mark.parametrize("table", [False, True])
def test_deeper_and_wider_than_one_program(table):
    rng = _rng("capacity", table)
    n = 5000
    cols = [column(rng, pc.FLOAT64 if j % 2 else pc.INT32, n, table) for j in range(20)]

    def balanced(lo, hi):
        if hi - lo == 1:
            return ("field", lo)
        mid = (lo + hi) // 2
        return ("call", "add_unchecked", [balanced(lo, mid), balanced(mid, hi)], None)

    # 20 distinct columns (> AG_EXPR_MAX_COLS) and a full binary tree of depth 9 (> AG_EXPR_MAX_REGS registers)
    check(balanced(0, 20), cols, table)

    def full(d, k):
        if d == 0:
            return ("field", k % 20)
        return ("call", "add_unchecked" if d % 2 else "multiply_unchecked", [full(d - 1, 2 * k), full(d - 1, 2 * k + 1)], None)

    check(full(9, 0), cols, table)


# ---------------------------------------------------------------- layouts ---------------------------------------
@gpu
@pytest.mark.parametrize("nchunks", [1, 16, 1000])
def test_table_layouts(nchunks):
    rng = _rng("layouts", nchunks)
    n = 20000
    cols = []
    for j, t in enumerate([pc.INT32, pc.FLOAT64, pc.BOOL]):
        arr = pc.Array.from_numpy(values(rng, t, n), valid=rng.random(n) >= 0.1, type_id=t)
        cuts = sorted(rng.integers(0, n + 1, nchunks - 1).tolist())
        bounds = [0] + cuts + [n]
        cols.append(pc.Chunked([arr.slice(a, b - a) for a, b in zip(bounds[:-1], bounds[1:])], t))
    t = ("call", "or_kleene", [("call", "greater", [("call", "multiply", [("field", 0), ("lit", 3, pc.INT32)], None), ("field", 1)], None),
                              ("field", 2)], None)
    check(t, cols, True)


@gpu
def test_empty_inputs():
    empty = pc.Chunked([], pc.INT32)
    e0 = pc.Chunked([pc.Array.from_numpy(np.zeros(0, np.int32), type_id=pc.INT32)], pc.INT32)
    t = ("call", "add", [("field", 0), ("field", 1)], None)
    check(t, [empty, e0], True)
    check(t, [pc.Array.from_numpy(np.zeros(0, np.int32), type_id=pc.INT32)] * 2, False)


# ---------------------------------------------------------------- one launch ------------------------------------
def _kernel_names(fn):
    torch = pytest.importorskip("torch")
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
            and "memset" not in e.name.lower()]


@gpu
def test_one_launch():
    rng = _rng("one-launch")
    n = 100_000
    e = pc.Call("and_kleene", [pc.Call("greater", [pc.Call("add", [pc.Call("multiply", [pc.Field(0), pc.Field(1)]), pc.Field(2)]), pc.Field(3)]),
                               pc.Call("is_not_null", [pc.Field(0)])])
    arrays = [pc.Array.from_numpy(values(rng, pc.FLOAT64, n), valid=rng.random(n) >= 0.1, type_id=pc.FLOAT64) for _ in range(4)]
    batch = pc.RecordBatch(arrays)
    pc.ExecuteScalarExpression(e, batch)   # warm
    names = _kernel_names(lambda: pc.ExecuteScalarExpression(e, batch))
    assert sum("expr_eval_kernel" in k for k in names) == 1, names
    assert all("expr_eval_kernel" in k or "reset_error_word" in k for k in names), names
    chunked = []
    for a in arrays:
        cuts = sorted(rng.integers(0, n + 1, 999).tolist())
        bounds = [0] + cuts + [n]
        chunked.append(pc.Chunked([a.slice(x, y - x) for x, y in zip(bounds[:-1], bounds[1:])], pc.FLOAT64))
    table = pc.Table(chunked)
    pc.ExecuteScalarExpression(e, table)
    names = _kernel_names(lambda: pc.ExecuteScalarExpression(e, table))
    assert sum("expr_eval_kernel" in k for k in names) == 1, names
    assert all("expr_eval_kernel" in k or "reset_error_word" in k for k in names), names


# ---------------------------------------------------------------- past 2^31 rows --------------------------------
@gpu
def test_past_2_31_rows():
    n = (1 << 31) + 100
    x = np.zeros(n, dtype=np.int8)
    x[-200:] = np.arange(200, dtype=np.int64).astype(np.int8)
    x[:64] = 5
    y = np.ones(n, dtype=np.int8)
    b = np.zeros(n, dtype=bool)
    b[-50:] = True
    cols = [pc.Array.from_numpy(x, type_id=pc.INT8), pc.Array.from_numpy(y, type_id=pc.INT8), pc.Array.from_numpy(b, type_id=pc.BOOL)]
    e = pc.Call("or", [pc.Call("greater", [pc.Field(0), pc.Field(1)]), pc.Field(2)])
    got = pc.ExecuteScalarExpression(e, pc.RecordBatch(cols))
    del cols
    vals, valid, _ = got.to_numpy()
    want = (x > y) | b
    assert valid.all()
    assert np.array_equal(vals[:1000], want[:1000]) and np.array_equal(vals[-1000:], want[-1000:])
    assert int(vals.sum()) == int(want.sum())
    assert zlib.crc32(np.packbits(vals, bitorder="little").tobytes()) == zlib.crc32(np.packbits(want, bitorder="little").tobytes())


# ---------------------------------------------------------------- the C ABI -------------------------------------
class Instr(C.Structure):
    _fields_ = [("op", C.c_int32), ("type", C.c_int32), ("out_type", C.c_int32), ("dst", C.c_int32), ("a", C.c_int32),
                ("b", C.c_int32), ("flags", C.c_int32), ("bits", C.c_uint64)]


class Program(C.Structure):
    _fields_ = [("n_instr", C.c_int32), ("instr", C.POINTER(Instr)), ("n_cols", C.c_int32), ("col_types", C.POINTER(C.c_int32)),
                ("out_reg", C.c_int32)]


class Chunk(C.Structure):   # ag_sort_chunk
    _fields_ = [("vals", C.c_void_p), ("valid", C.c_void_p), ("offset", C.c_int64), ("length", C.c_int64)]


LOAD, CONST, ADD, MUL_CHECKED, GT, CAST = 0, 1, 3, 8, 27, 42


def program(instrs, col_types, out_reg):
    arr = (Instr * len(instrs))(*[Instr(*i) for i in instrs])
    ct = (C.c_int32 * max(len(col_types), 1))(*col_types)
    p = Program(len(instrs), arr, len(col_types), ct, out_reg)
    p._keep = (arr, ct)
    return p


def host_eval(p, cols, n):
    spans = (Chunk * len(cols))(*[Chunk(c.ctypes.data, None, 0, n) for c in cols])
    out = np.zeros(max(n, 1) * 8, dtype=np.uint8)
    valid = np.zeros((n + 7) // 8 + 8, dtype=np.uint8)
    bad = C.c_int64()
    st, msg = N.call_status("ag_eval_program", C.byref(p), 1, spans, out.ctypes.data, valid.ctypes.data, C.byref(bad))
    return st, msg, out, valid, bad.value


@gpu
def test_c_abi_programs():
    n = 1000
    a = np.arange(n, dtype=np.int64)
    b = np.full(n, 7, dtype=np.int64)
    p = program([(LOAD, pc.INT64, pc.INT64, 0, 0, 0, 0, 0), (LOAD, pc.INT64, pc.INT64, 1, 1, 0, 0, 0),
                 (ADD, pc.INT64, pc.INT64, 0, 0, 1, 0, 0), (CONST, pc.INT64, pc.INT64, 1, 0, 0, 1, 500),
                 (GT, pc.INT64, pc.BOOL, 0, 0, 1, 0, 0)], [pc.INT64, pc.INT64], 0)
    st, msg, out, valid, _ = host_eval(p, [a, b], n)
    assert st == 0, msg
    assert np.array_equal(np.unpackbits(out, bitorder="little")[:n].astype(bool), a + 7 > 500)
    assert np.unpackbits(valid, bitorder="little")[:n].all()
    # a failing program: checked multiply overflows at row 3
    big = np.zeros(n, dtype=np.int64)
    big[3] = 1 << 62
    p = program([(LOAD, pc.INT64, pc.INT64, 0, 0, 0, 0, 0), (CONST, pc.INT64, pc.INT64, 1, 0, 0, 1, 4),
                 (MUL_CHECKED, pc.INT64, pc.INT64, 0, 0, 1, 0, 0)], [pc.INT64], 0)
    st, msg, _, _, bad = host_eval(p, [big], n)
    assert st == N.AG_ERR_INVALID and bad == 3, msg
    # the device flavour over device buffers
    torch = pytest.importorskip("torch")
    da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    dout = torch.zeros(n, dtype=torch.int64, device="cuda")
    word = torch.full((1,), (1 << 63) - 1, dtype=torch.int64, device="cuda")
    p = program([(LOAD, pc.INT64, pc.INT64, 0, 0, 0, 0, 0), (LOAD, pc.INT64, pc.INT64, 1, 1, 0, 0, 0),
                 (ADD, pc.INT64, pc.INT64, 0, 0, 1, 0, 0)], [pc.INT64, pc.INT64], 0)
    spans = (Chunk * 2)(Chunk(da.data_ptr(), None, 0, n), Chunk(db.data_ptr(), None, 0, n))
    N.call("ag_eval_program_dev", C.byref(p), 1, spans, dout.data_ptr(), None, word.data_ptr(), None)
    torch.cuda.synchronize()
    assert torch.equal(dout.cpu(), torch.from_numpy(a + b)) and int(word.item()) == (1 << 63) - 1


MALFORMED = [
    ("unknown op", [(99, pc.INT64, pc.INT64, 0, 0, 0, 0, 0)], [pc.INT64], 0),
    ("register out of range", [(LOAD, pc.INT64, pc.INT64, 8, 0, 0, 0, 0)], [pc.INT64], 8),
    ("column out of range", [(LOAD, pc.INT64, pc.INT64, 0, 1, 0, 0, 0)], [pc.INT64], 0),
    ("column type mismatch", [(LOAD, pc.INT32, pc.INT32, 0, 0, 0, 0, 0)], [pc.INT64], 0),
    ("operand types", [(LOAD, pc.INT64, pc.INT64, 0, 0, 0, 0, 0), (CONST, pc.INT32, pc.INT32, 1, 0, 0, 1, 1),
                       (ADD, pc.INT64, pc.INT64, 0, 0, 1, 0, 0)], [pc.INT64], 0),
    ("undefined operand", [(LOAD, pc.INT64, pc.INT64, 0, 0, 0, 0, 0), (ADD, pc.INT64, pc.INT64, 0, 0, 3, 0, 0)], [pc.INT64], 0),
    ("float checked op", [(LOAD, pc.FLOAT64, pc.FLOAT64, 0, 0, 0, 0, 0), (MUL_CHECKED, pc.FLOAT64, pc.FLOAT64, 0, 0, 0, 0, 0)], [pc.FLOAT64], 0),
    ("bad result type", [(LOAD, pc.INT64, pc.INT64, 0, 0, 0, 0, 0), (GT, pc.INT64, pc.INT64, 0, 0, 0, 0, 0)], [pc.INT64], 0),
    ("output register empty", [(LOAD, pc.INT64, pc.INT64, 0, 0, 0, 0, 0)], [pc.INT64], 3),
]


@gpu
@pytest.mark.parametrize("what,instrs,col_types,out_reg", MALFORMED, ids=[m[0] for m in MALFORMED])
def test_malformed_programs(what, instrs, col_types, out_reg):
    n = 64
    a = np.arange(n, dtype=np.int64)
    p = program(instrs, col_types, out_reg)
    before = N.raw().ag_kernel_launch_count()
    st, msg, _, _, _ = host_eval(p, [a] * len(col_types), n)
    assert st == N.AG_ERR_INVALID, (what, msg)
    assert N.raw().ag_kernel_launch_count() == before
    spans = (Chunk * len(col_types))(*[Chunk(a.ctypes.data, None, 0, n) for _ in col_types])
    st, _ = N.call_status("ag_eval_program_dev", C.byref(p), 1, spans, None, None, None, None)
    assert st == N.AG_ERR_INVALID
    assert N.raw().ag_kernel_launch_count() == before


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_no_cpu_fallback_without_gpu():
    """Without a device ag_eval_program fails with AG_ERR_CUDA and computes nothing."""
    a = np.arange(16, dtype=np.int64)
    p = program([(LOAD, pc.INT64, pc.INT64, 0, 0, 0, 0, 0)], [pc.INT64], 0)
    st, _, out, _, _ = host_eval(p, [a], 16)
    assert st == N.AG_ERR_CUDA and not out.any()
