"""A model of what a compute call must return, and a generator of the physical forms one logical column can take.

The model works from the flattened logical inputs only: every argument is a logical column (`Col`), a valid scalar
or a null scalar (`Sca`), and each function is the oracle's per-element loop (oracle/cpu_ref.c) applied to the whole
column in one call, or tests/dictionary_encode_ref.py / tests/run_end_ref.py.  Nothing here knows how the library
cuts its arguments into spans.  It answers with an `Out` (type, kind, values, validity) or a `Fail` (sentinel,
message).

The layout generator presents a logical column as a plain array, a slice of a larger array, or a chunked array
(random cuts, empty and one-row chunks, chunks that are slices).  `Layout.pieces` gives the physical buffers as
numpy arrays; tests/test_gpu_exec_differential.py uploads them.  Bytes outside a piece's logical rows are random,
so a kernel that reads past its offset picks up garbage rather than a lucky zero.
"""
import ctypes as C

import numpy as np

import dictionary_encode_ref
import run_end_ref
from arrow_go_b200 import compute as pc   # type ids and option values only
from helpers import pack_bits, ptr, unpack_bits

NUMERIC = [pc.UINT8, pc.INT8, pc.UINT16, pc.INT16, pc.UINT32, pc.INT32, pc.UINT64, pc.INT64, pc.FLOAT32, pc.FLOAT64]
INTS = NUMERIC[:8]
SIGNED = [pc.INT8, pc.INT16, pc.INT32, pc.INT64]
FLOATS = [pc.FLOAT32, pc.FLOAT64]
NAME = {pc.BOOL: "bool", pc.UINT8: "uint8", pc.INT8: "int8", pc.UINT16: "uint16", pc.INT16: "int16", pc.UINT32: "uint32",
        pc.INT32: "int32", pc.UINT64: "uint64", pc.INT64: "int64", pc.FLOAT32: "float32", pc.FLOAT64: "float64"}
NO_ERROR_POS = (1 << 63) - 1

# oracle op / comparison / shape codes (include/arrowgpu.h)
OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_ABS, OP_NEG, OP_SIGN = 0, 1, 2, 3, 4, 5, 20
OP_ADD_C, OP_SUB_C, OP_MUL_C, OP_DIV_C, OP_ABS_C, OP_NEG_C = 21, 22, 23, 24, 25, 26
OP_BIT_AND, OP_BIT_OR, OP_BIT_XOR, OP_BIT_NOT, OP_SHL, OP_SHR, OP_SHL_C, OP_SHR_C = 64, 65, 66, 67, 68, 69, 70, 71
SH_AA, SH_AS, SH_SA = 0, 1, 2
BITOP = {"and": 0, "or": 1, "xor": 2, "and_not": 3}
KLEENE = {"and_kleene": 0, "or_kleene": 1, "and_not_kleene": 2}
CMP = {"equal": 0, "not_equal": 1, "greater": 2, "greater_equal": 3, "less": 4, "less_equal": 5}

OVERFLOW, DIV_ZERO = "overflow", "divide by zero"
SHIFT_MSG = "shift amount must be >= 0 and less than precision of type"
# name -> (op, checked-integer kernel?, failure message); the checked integer kernels run ScalarBinaryNotNull
# (ref_arith_checked), everything else every slot (ref_arith_binary)
ARITH = {
    "add": (OP_ADD_C, True, OVERFLOW), "add_unchecked": (OP_ADD, False, None),
    "sub": (OP_SUB_C, True, OVERFLOW), "sub_unchecked": (OP_SUB, False, None),
    "subtract": (OP_SUB_C, True, OVERFLOW), "subtract_unchecked": (OP_SUB, False, None),
    "multiply": (OP_MUL_C, True, OVERFLOW), "multiply_unchecked": (OP_MUL, False, None),
    "bit_wise_and": (OP_BIT_AND, False, None), "bit_wise_or": (OP_BIT_OR, False, None), "bit_wise_xor": (OP_BIT_XOR, False, None),
}
# every type through ref_arith_checked (ScalarBinaryNotNull)
NOT_NULL_ARITH = {
    "divide": (OP_DIV_C, DIV_ZERO), "divide_unchecked": (OP_DIV, DIV_ZERO),
    "shift_left": (OP_SHL_C, SHIFT_MSG), "shift_left_unchecked": (OP_SHL, SHIFT_MSG),
    "shift_right": (OP_SHR_C, SHIFT_MSG), "shift_right_unchecked": (OP_SHR, SHIFT_MSG),
}
UNARY = {"abs": OP_ABS_C, "abs_unchecked": OP_ABS, "negate": OP_NEG_C, "negate_unchecked": OP_NEG, "sign": OP_SIGN,
         "bit_wise_not": OP_BIT_NOT}
INT_ONLY = {"bit_wise_and", "bit_wise_or", "bit_wise_xor", "bit_wise_not", "shift_left", "shift_left_unchecked",
            "shift_right", "shift_right_unchecked"}
PROMOTING = set(ARITH) | set(NOT_NULL_ARITH) | set(CMP)


def np_of(t):
    return np.bool_ if t == pc.BOOL else pc.NP_OF[t]


def width(t):
    return 1 if t == pc.BOOL else np.dtype(pc.NP_OF[t]).itemsize * 8


class Col:
    """A logical column: `values` (every row, null rows included), `valid` (bool per row, or None: no nulls)."""

    def __init__(self, t, values, valid=None):
        self.type = t
        self.values = np.ascontiguousarray(values, dtype=np_of(t))
        self.valid = None if valid is None else np.ascontiguousarray(valid, dtype=bool)

    def __len__(self):
        return self.values.size

    def validity(self):
        return np.ones(len(self), dtype=bool) if self.valid is None else self.valid


class Sca:
    """A scalar: `value` None is a null scalar."""

    def __init__(self, t, value):
        self.type, self.value = t, value

    @property
    def valid(self):
        return self.value is not None

    def raw(self):
        return np.array([0 if self.value is None else self.value], dtype=np_of(self.type))


class Out:
    """What a call must return.  `kind` is pc.KIND_ARRAY or pc.KIND_CHUNKED; `values` are specified at valid rows
    only (a null row's value, e.g. under unique's null slot, is not)."""

    def __init__(self, t, values, valid, kind, **extra):
        self.type, self.kind = t, kind
        self.values = np.asarray(values)
        self.valid = np.ones(self.values.size, dtype=bool) if valid is None else np.asarray(valid, dtype=bool)
        self.extra = extra

    def __len__(self):
        return self.values.size

    @property
    def null_count(self):
        return int((~self.valid).sum())


class Fail:
    def __init__(self, sentinel, msg):
        self.sentinel, self.msg = sentinel, msg

    def __repr__(self):
        return f"Fail({self.sentinel}: {self.msg})"


_cpu = None


def cpu():
    global _cpu
    if _cpu is None:
        from oracle import oracle
        _cpu = oracle.cpu()
    return _cpu


def bits(b):
    """A bool array as an LSB-first bitmap at bit 0 (pack_bits with zero padding)."""
    return pack_bits(np.asarray(b, dtype=bool), 0, fill=0)


# ------------------------------------------------------------------------------------------ promotion and casts
def common_numeric(a, b):
    """The promoted type of a binary call (commonNumeric, pinned by test_host_cpu.py::test_common_numeric_table):
    floats win; otherwise the narrowest integer type holding both ranges, saturating at int64."""
    if pc.FLOAT64 in (a, b):
        return pc.FLOAT64
    if pc.FLOAT32 in (a, b):
        return pc.FLOAT32
    (wa, sa), (wb, sb) = (width(a), a in SIGNED), (width(b), b in SIGNED)
    if sa == sb:
        w, s = max(wa, wb), sa
    else:
        ws, wu = (wa, wb) if sa else (wb, wa)
        w, s = min(64, ws if ws > wu else 2 * wu), True
    return {(8, False): pc.UINT8, (16, False): pc.UINT16, (32, False): pc.UINT32, (64, False): pc.UINT64,
            (8, True): pc.INT8, (16, True): pc.INT16, (32, True): pc.INT32, (64, True): pc.INT64}[(w, s)]


def _int_range(t):
    info = np.iinfo(pc.NP_OF[t])
    return int(info.min), int(info.max)


def safe_bounds(src, dst):
    """The range a safe cast names in its message (getSafeMinMax / checkIntToFloatTrunc)."""
    if dst in FLOATS:
        hi = 1 << (24 if dst == pc.FLOAT32 else 53)
        return (-hi if src in SIGNED else 0), hi
    (a, b), (c, d) = _int_range(src), _int_range(dst)
    return max(a, c), min(b, d)


def cast_col(col, to, allow_int_overflow=False, allow_float_truncate=False):
    """(Col, None) or (None, Fail): the numeric cast of every row; valid rows are checked, the first failing row
    names the error."""
    if col.type == to:
        return col, None
    out = np.zeros(len(col), dtype=pc.NP_OF[to])
    bad = C.c_int64(NO_ERROR_POS)
    vb = None if col.valid is None else bits(col.valid)
    cpu().ref_cast_numeric(col.type, to, ptr(col.values), ptr(vb), 0, ptr(out), len(col), int(allow_int_overflow),
                           int(allow_float_truncate), C.byref(bad))
    if bad.value != NO_ERROR_POS:
        v = col.values[bad.value]
        if col.type in FLOATS:
            return None, Fail("ErrInvalid", "float value %f was truncated converting to %s" % (float(v), NAME[to]))
        lo, hi = safe_bounds(col.type, to)
        return None, Fail("ErrInvalid", f"integer value {int(v)} not in range: {lo} to {hi}")
    return Col(to, out, col.valid), None


def cast_arg(a, to):
    if isinstance(a, Col):
        return cast_col(a, to)
    if a.value is None or a.type == to:
        return Sca(to, a.value), None
    c, f = cast_col(Col(a.type, a.raw()), to)
    return (None, f) if f else (Sca(to, c.values[0].item()), None)


# ------------------------------------------------------------------------------------------ the model
def _kind(args):
    return pc.KIND_CHUNKED if any(getattr(a, "chunked", False) for a in args) else pc.KIND_ARRAY


def _length(args):
    return next(len(a) for a in args if isinstance(a, Col))


def _intersection(args, n):
    v = np.ones(n, dtype=bool)
    for a in args:
        if isinstance(a, Sca):
            if not a.valid:
                v[:] = False
        elif a.valid is not None:
            v &= a.valid
    return v


def _shape_ptrs(l, r):
    shape = SH_AA if isinstance(l, Col) and isinstance(r, Col) else (SH_AS if isinstance(l, Col) else SH_SA)
    lv = l.values if isinstance(l, Col) else l.raw()
    rv = r.values if isinstance(r, Col) else r.raw()
    return shape, lv, rv


def _broadcast_bool(a, n):
    """(values, valid) of a boolean argument as full columns."""
    if isinstance(a, Col):
        return a.values, a.validity()
    return np.full(n, bool(a.value)), np.full(n, a.valid)


def model(name, args, opts=None, chunked=()):
    """What CallFunction(name, args) must give.  `args` are Col / Sca; `chunked` holds the indices of the
    arguments presented as chunked arrays (a chunked input gives a chunked output)."""
    opts = opts or {}
    for i, a in enumerate(args):
        a.chunked = i in chunked
    kind = _kind(args)
    if name in PROMOTING and len({a.type for a in args}) > 1:
        to = common_numeric(args[0].type, args[1].type)
        cast = []
        for a in args:
            c, f = cast_arg(a, to)
            if f:
                return f
            c.chunked = a.chunked
            cast.append(c)
        args = cast
    t = args[0].type
    if name in ARITH or name in NOT_NULL_ARITH:
        return _binary_arith(name, args, kind)
    if name in CMP:
        n = _length(args)
        shape, lv, rv = _shape_ptrs(*args)
        ob = np.zeros(n // 8 + 8, dtype=np.uint8)
        cpu().ref_compare(t, CMP[name], shape, ptr(lv), ptr(rv), ptr(ob), n, 0)
        return Out(pc.BOOL, unpack_bits(ob, 0, n), _intersection(args, n), kind)
    if name in BITOP or name in KLEENE:
        n = _length(args)
        (ld, lv), (rd, rv) = _broadcast_bool(args[0], n), _broadcast_bool(args[1], n)
        od, ov = np.zeros(n // 8 + 8, dtype=np.uint8), np.zeros(n // 8 + 8, dtype=np.uint8)
        lvb, ldb, rvb, rdb = bits(lv), bits(ld), bits(rv), bits(rd)   # kept alive across the calls
        if name in BITOP:
            cpu().ref_bitmap_op(BITOP[name], ptr(ldb), 0, ptr(rdb), 0, ptr(od), 0, n)
            return Out(pc.BOOL, unpack_bits(od, 0, n), _intersection(args, n), kind)
        cpu().ref_kleene(KLEENE[name], ptr(lvb), ptr(ldb), 0, ptr(rvb), ptr(rdb), 0, ptr(ov), ptr(od), 0, n)
        return Out(pc.BOOL, unpack_bits(od, 0, n), unpack_bits(ov, 0, n), kind)
    a = args[0]
    n = len(a)
    if name in UNARY:
        op = UNARY[name]
        out = np.zeros(n, dtype=pc.NP_OF[t])
        if op in (OP_ABS_C, OP_NEG_C) and t in SIGNED:   # AbsoluteValueChecked / NegateChecked: every slot
            bad = C.c_int64(NO_ERROR_POS)
            cpu().ref_arith_unary_checked(t, op, ptr(a.values), ptr(out), n, C.byref(bad))
            if bad.value != NO_ERROR_POS:
                return Fail("ErrInvalid", OVERFLOW)
        else:
            cpu().ref_arith_unary_same(t, op, ptr(a.values), ptr(out), n)
        return Out(t, out, a.valid, kind)
    if name == "not":
        return Out(pc.BOOL, ~a.values, a.valid, kind)
    if name == "is_null":
        return Out(pc.BOOL, ~a.validity(), None, kind)
    if name == "is_not_null":
        return Out(pc.BOOL, a.validity(), None, kind)
    if name == "is_nan":
        return Out(pc.BOOL, np.isnan(a.values) if t in FLOATS else np.zeros(n, dtype=bool), None, kind)
    if name == "cast":
        c, f = cast_col(a, opts["to"], opts.get("allow_int_overflow", False), opts.get("allow_float_truncate", False))
        return f or Out(c.type, c.values, c.valid, kind)
    if name in ("filter", "array_filter"):
        return _filter(a, args[1], opts.get("null_selection", pc.DROP_NULLS), kind)
    if name in ("take", "array_take"):
        return _take(a, args[1], opts.get("bounds_check", True), pc.KIND_CHUNKED if a.chunked or args[1].chunked else pc.KIND_ARRAY)
    if name in ("cumulative_sum", "cumulative_sum_checked"):
        return _cumulative_sum(a, name.endswith("_checked"), opts.get("skip_nulls", False), opts.get("start"), kind)
    if name in ("sort_indices", "unique", "is_in"):
        if a.chunked and opts.get("chunks", 1) != 1:
            return Fail("ErrNotImplemented", f"{name}: the GPU kernel takes one array")
        return _one_array(name, a, opts)
    if name == "dictionary_encode":
        enc = opts.get("null_encoding", pc.NULL_ENCODING_MASK)
        (chunk,), dictionary, dict_valid = dictionary_encode_ref.dictionary_encode_ref([(a.values, a.valid)], enc)
        idx, ivalid, _ = chunk
        return Out(pc.DICTIONARY, idx, ivalid, kind, dictionary=dictionary, dictionary_valid=dict_valid, value_type=t)
    raise KeyError(name)


def _binary_arith(name, args, kind):
    l, r = args
    t = l.type
    n = _length(args)
    valid = _intersection(args, n)
    out = np.zeros(n, dtype=pc.NP_OF[t])
    if name in NOT_NULL_ARITH or (ARITH[name][1] and t not in FLOATS):
        op, msg = NOT_NULL_ARITH[name] if name in NOT_NULL_ARITH else (ARITH[name][0], ARITH[name][2])
        if not all(a.valid for a in args if isinstance(a, Sca)):
            return Out(t, out, valid, kind)      # one side entirely null: nothing is computed, nothing fails
        shape, lv, rv = _shape_ptrs(l, r)
        lb = bits(l.valid) if isinstance(l, Col) and l.valid is not None else None
        rb = bits(r.valid) if isinstance(r, Col) and r.valid is not None else None
        bad = C.c_int64(NO_ERROR_POS)
        cpu().ref_arith_checked(t, op, shape, ptr(lv), ptr(lb), 0, ptr(rv), ptr(rb), 0, ptr(out), n, C.byref(bad))
        if bad.value != NO_ERROR_POS:
            return Fail("ErrInvalid", msg)
        return Out(t, out, valid, kind)
    shape, lv, rv = _shape_ptrs(l, r)
    cpu().ref_arith_binary(t, ARITH[name][0], shape, ptr(lv), ptr(rv), ptr(out), n)
    return Out(t, out, valid, kind)


def _filter(values, mask, sel, kind):
    n = len(values)
    if len(mask) != n:
        return Fail("ErrInvalid", "vector kernel arguments must all be the same length")
    bw = width(values.type)
    vals = bits(values.values) if values.type == pc.BOOL else values.values
    out = np.zeros(n // 8 + 8, dtype=np.uint8) if values.type == pc.BOOL else np.zeros(max(n, 1), dtype=values.values.dtype)
    ov = np.zeros(n // 8 + 8, dtype=np.uint8)
    ln, nn = C.c_int64(), C.c_int64()
    vb = None if values.valid is None else bits(values.valid)
    mb = None if mask.valid is None else bits(mask.valid)
    md = bits(mask.values)
    cpu().ref_filter_primitive(bw, ptr(vals), ptr(vb), 0, ptr(md), ptr(mb), 0, n, sel, ptr(out), ptr(ov),
                               C.byref(ln), C.byref(nn))
    k = ln.value
    res = unpack_bits(out, 0, k) if values.type == pc.BOOL else out[:k]
    return Out(values.type, res, unpack_bits(ov, 0, k) if (vb is not None or mb is not None) else None, kind)


def _take(values, indices, bounds_check, kind):
    n = len(indices)
    bw, iw = width(values.type), width(indices.type)
    vals = bits(values.values) if values.type == pc.BOOL else values.values
    out = np.zeros(n // 8 + 8, dtype=np.uint8) if values.type == pc.BOOL else np.zeros(max(n, 1), dtype=values.values.dtype)
    ov = np.zeros(n // 8 + 8, dtype=np.uint8)
    nn, pos, bad = C.c_int64(), C.c_int64(NO_ERROR_POS), C.c_int64()
    vb = None if values.valid is None else bits(values.valid)
    ib = None if indices.valid is None else bits(indices.valid)
    cpu().ref_take_primitive(bw, ptr(vals), ptr(vb), 0, len(values), iw, int(indices.type in SIGNED), ptr(indices.values), ptr(ib),
                             0, n, int(bounds_check), ptr(out), ptr(ov), C.byref(nn), C.byref(pos), C.byref(bad))
    if bounds_check and pos.value != NO_ERROR_POS:
        return Fail("ErrIndex", f"{int(indices.values[pos.value])} out of bounds")
    res = unpack_bits(out, 0, n) if values.type == pc.BOOL else out[:n]
    return Out(values.type, res, unpack_bits(ov, 0, n) if (vb is not None or ib is not None) else None, kind)


class _CumsumState(C.Structure):
    _fields_ = [("cur", C.c_uint8 * 8), ("encountered_null", C.c_int64)]


def _cumulative_sum(a, checked, skip, start, kind):
    t = a.type
    if t not in NUMERIC:
        return Fail("ErrType", f"cumulative sum input type must be numeric, got {NAME[t]}")
    st = _CumsumState()
    if start is not None:
        if not start.valid:
            return Fail("ErrInvalid", "cumulative sum start value must be valid")
        s, f = cast_arg(start, t)
        if f:
            return Fail("ErrInvalid", f"cannot cast cumulative sum start value to {NAME[t]}: {f.msg}")
        for i, b in enumerate(s.raw().tobytes()):
            st.cur[i] = b
    n = len(a)
    out = np.zeros(max(n, 1), dtype=pc.NP_OF[t])
    ov = np.zeros(n // 8 + 8, dtype=np.uint8)
    nn, bad = C.c_int64(), C.c_int64(NO_ERROR_POS)
    vb = bits(a.validity())
    cpu().ref_cumulative_sum(t, ptr(a.values), ptr(vb), 0, n, int(skip), int(checked), ptr(out), ptr(ov), 0,
                             C.byref(st), C.byref(nn), C.byref(bad))
    if checked and bad.value != NO_ERROR_POS:
        return Fail("ErrInvalid", OVERFLOW)
    return Out(t, out[:n], unpack_bits(ov, 0, n), kind)


def _one_array(name, a, opts):
    n, t = len(a), a.type
    vb = None if a.valid is None else bits(a.valid)
    if name == "sort_indices":
        out = np.zeros(max(n, 1), dtype=np.uint64)
        nn, nan = C.c_int64(), C.c_int64()
        cpu().ref_sort_indices(t, ptr(a.values), ptr(vb), 0, n, opts.get("order", pc.ASCENDING), opts.get("placement", pc.NULLS_AT_END),
                               ptr(out), C.byref(nn), C.byref(nan))
        return Out(pc.UINT64, out[:n], None, pc.KIND_ARRAY)
    bw = width(t)
    if name == "unique":
        out = np.zeros(max(n, 1), dtype=pc.NP_OF[t])
        ov = np.zeros(n // 8 + 8, dtype=np.uint8)
        ln, nn = C.c_int64(), C.c_int64()
        cpu().ref_unique(bw, ptr(a.values), ptr(vb), 0, n, ptr(out), ptr(ov), C.byref(ln), C.byref(nn))
        k = ln.value
        return Out(t, out[:k], unpack_bits(ov, 0, k) if vb is not None else None, pc.KIND_ARRAY)
    s = opts["value_set"]
    sb = None if s.valid is None else bits(s.valid)
    od, ov = np.zeros(n // 8 + 8, dtype=np.uint8), np.zeros(n // 8 + 8, dtype=np.uint8)
    nn = C.c_int64()
    cpu().ref_is_in(bw, ptr(a.values), ptr(vb), 0, n, ptr(s.values), ptr(sb), 0, len(s), opts.get("null_behavior", pc.NULL_MATCH),
                    ptr(od), ptr(ov), C.byref(nn))
    return Out(pc.BOOL, unpack_bits(od, 0, n), unpack_bits(ov, 0, n), pc.KIND_ARRAY)


def run_end_encode(values, valid, run_end_type):
    """(run_ends, run_values, run_valid or None) of one chunk, the run ends counted from the chunk's first row."""
    rt = {pc.INT16: "int16", pc.INT32: "int32", pc.INT64: "int64"}[run_end_type]
    ends, vals, rvalid, _ = run_end_ref.encode(values, valid, rt)
    return ends, vals, rvalid


# ------------------------------------------------------------------------------------------ layouts
class Piece:
    """One physical array: `values` / `valid` (None: no bitmap) are the whole buffers, rows [offset, offset+length)
    are the logical ones."""

    def __init__(self, values, valid, offset, length):
        self.values, self.valid, self.offset, self.length = values, valid, offset, length


class Layout:
    """One physical form of a logical column: 'array', 'slice' or 'chunked'.  `pieces(col)` builds the buffers."""

    def __init__(self, form, cuts=None, offsets=None, pad=0, seed=0):
        self.form, self.cuts, self.offsets, self.pad, self.seed = form, cuts, offsets, pad, seed

    def __repr__(self):
        if self.form == "chunked":
            return f"chunked(cuts={self.cuts}, chunk_offsets={self.offsets})" if len(self.cuts) <= 40 else \
                f"chunked({len(self.cuts) - 1} chunks, cuts[:40]={self.cuts[:40]}..., chunk_offsets[:40]={self.offsets[:40]}...)"
        return "array" if self.form == "array" else f"slice(offset={self.offsets[0]})"

    @property
    def chunked(self):
        return self.form == "chunked"

    def ranges(self, n):
        """[(start, stop, element offset inside its buffer)] of every piece."""
        if self.form == "chunked":
            return [(a, b, o) for a, b, o in zip(self.cuts, self.cuts[1:], self.offsets)]
        return [(0, n, self.offsets[0] if self.form == "slice" else 0)]

    def pieces(self, col, bitmap=True):
        """The physical buffers.  `bitmap` False drops the validity bitmap (the column must have no nulls); a
        column with valid None and bitmap True gets a bitmap with zero nulls."""
        rng = np.random.default_rng(self.seed)
        dt = np_of(col.type)
        out = []
        for a, b, off in self.ranges(len(col)):
            pad = self.pad if off else 0
            m = off + (b - a) + pad
            if col.type == pc.BOOL:
                buf = rng.random(m) < 0.5
            elif dt in (np.float32, np.float64):
                buf = rng.standard_normal(m).astype(dt)
            else:
                buf = rng.integers(0, 256, m * np.dtype(dt).itemsize, dtype=np.uint8).view(dt)
            buf[off:off + b - a] = col.values[a:b]
            valid = None
            if bitmap:
                valid = rng.random(m) < 0.5
                valid[off:off + b - a] = col.validity()[a:b]
            out.append(Piece(buf, valid, off, b - a))
        return out


def flatten(pieces, t):
    """The logical column a list of pieces holds (numpy only)."""
    dt = np_of(t)
    vals = [p.values[p.offset:p.offset + p.length] for p in pieces]
    valid = [np.ones(p.length, dtype=bool) if p.valid is None else p.valid[p.offset:p.offset + p.length] for p in pieces]
    return (np.concatenate(vals) if vals else np.zeros(0, dtype=dt)), (np.concatenate(valid) if valid else np.zeros(0, dtype=bool))


def random_cuts(rng, n, chunks):
    """Cut points over [0, n] with zero-length and one-row chunks and cuts inside a byte."""
    inner = rng.integers(0, n + 1, max(chunks - 1, 0)) if n else np.zeros(max(chunks - 1, 0), dtype=np.int64)
    cuts = sorted([0, n] + inner.tolist())
    # a zero-length and a one-row chunk wherever there is room
    if n >= 2 and chunks >= 3:
        k = int(rng.integers(1, len(cuts) - 1))
        cuts.insert(k, cuts[k])
        p = int(rng.integers(0, n - 1))
        cuts += [p, p + 1]
        cuts.sort()
    return cuts


def random_layout(rng, n, form=None, max_chunks=8):
    form = form or ["array", "slice", "chunked"][int(rng.integers(0, 3))]
    seed = int(rng.integers(0, 1 << 31))
    if form == "array":
        return Layout("array", seed=seed)
    if form == "slice":
        return Layout("slice", offsets=[int(rng.integers(1, 18))], pad=int(rng.integers(0, 9)), seed=seed)
    cuts = random_cuts(rng, n, int(rng.integers(1, max_chunks + 1)))
    offs = [int(rng.integers(1, 18)) if rng.random() < 0.5 else 0 for _ in cuts[1:]]
    return Layout("chunked", cuts=cuts, offsets=offs, pad=int(rng.integers(0, 9)), seed=seed)


VALIDITY = ("none", "zero_nulls", "nulls_10", "nulls_90", "null_chunk")


def random_validity(rng, n, pattern, layout=None):
    """(valid or None, bitmap?) of a validity pattern: 'none' has no bitmap at all, 'zero_nulls' a bitmap without
    nulls, 'nulls_10' / 'nulls_90' about that share of nulls, 'null_chunk' one all-null chunk among valid ones."""
    if pattern == "none":
        return None, False
    if pattern == "zero_nulls":
        return None, True
    if pattern in ("nulls_10", "nulls_90"):
        return rng.random(n) >= (0.1 if pattern == "nulls_10" else 0.9), True
    v = np.ones(n, dtype=bool)
    if layout is not None and layout.chunked:
        spans = [(a, b) for a, b, _ in layout.ranges(n) if b > a]
        a, b = spans[int(rng.integers(0, len(spans)))] if spans else (0, 0)
    else:
        a = int(rng.integers(0, n + 1))
        b = int(rng.integers(a, n + 1))
    v[a:b] = False
    return v, True
