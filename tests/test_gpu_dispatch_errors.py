"""Every stream-ordered entry point that picks a kernel instantiation from an argument (a type id, a bit width,
an index width, an op, an operand shape or a comparison operator) refuses a value it has no kernel for with a
fixed status and message, and reports the first bad argument when several are bad."""
import numpy as np
import pytest

from arrow_go_b200 import _native as N
from helpers import Dev, dev_scalar_i64

pytestmark = pytest.mark.gpu

BAD = 99   # no type id, bit width or index width is 99
BAD_SHAPE = 7
BAD_CMP = 9
NBYTES = 256
n = 4


class Bufs:
    def __init__(self):
        self.a, self.b, self.o = Dev(nbytes=NBYTES), Dev(nbytes=NBYTES), Dev(nbytes=NBYTES)
        self.mask, self.valid = Dev(nbytes=NBYTES), Dev(nbytes=NBYTES)
        self.word = dev_scalar_i64(N.NO_ERROR_POS)
        self.state = Dev(nbytes=NBYTES)
        self.host_scalar = np.zeros(1, dtype=np.int64)
        self.spans = N.span_table([(self.a.ptr, self.b.ptr, self.o.ptr, n)])


def binary(t, op, shape):
    return lambda d: ("ag_arith_binary_dev", t, op, shape, d.a.ptr, d.b.ptr, d.o.ptr, n, None)


def spans(t, op, shape):
    return lambda d: ("ag_arith_binary_spans_dev", t, op, shape, d.spans, 1, None)


def unary_same(t, op):
    return lambda d: ("ag_arith_unary_same_dev", t, op, d.a.ptr, d.o.ptr, n, None)


def unary_diff(it, ot, op):
    return lambda d: ("ag_arith_unary_diff_dev", it, ot, op, d.a.ptr, d.o.ptr, n, None)


def checked(t, op, shape):
    return lambda d: ("ag_arith_checked_dev", t, op, shape, d.a.ptr, None, 0, d.b.ptr, None, 0, d.o.ptr, n, d.word.ptr, None)


def unary_checked(t, op):
    return lambda d: ("ag_arith_unary_checked_dev", t, op, d.a.ptr, d.o.ptr, n, d.word.ptr, None)


def compare(t, cmp, shape):
    return lambda d: ("ag_compare_dev", t, cmp, shape, d.a.ptr, d.b.ptr, d.o.ptr, n, 0, None)


def cast(it, ot):
    return lambda d: ("ag_cast_numeric_dev", it, ot, d.a.ptr, d.o.ptr, n, None)


def cumsum(t):
    return lambda d: ("ag_cumulative_sum_dev", t, d.a.ptr, None, 0, n, 0, 0, d.o.ptr, None, 0, d.state.ptr, None, None)


def cumsum_init(t):
    return lambda d: ("ag_cumulative_sum_state_init_dev", d.state.ptr, t, d.host_scalar.ctypes.data, None)


def sort(t):
    return lambda d: ("ag_sort_indices_dev", t, d.a.ptr, None, 0, n, 0, 0, d.o.ptr, None, None, None)


def min_max(t):
    return lambda d: ("ag_min_max_dev", t, d.a.ptr, n, d.o.ptr, None)


def filt(bw):
    return lambda d: ("ag_filter_primitive_dev", bw, d.a.ptr, None, 0, d.mask.ptr, None, 0, n, N.DROP_NULLS, d.o.ptr, None, n,
                      d.word.ptr, None)


def filter_compare(t, cmp):
    return lambda d: ("ag_filter_compare_scalar_dev", t, cmp, d.a.ptr, d.host_scalar.ctypes.data, n, d.o.ptr, n, d.word.ptr, None)


def take_indices(iw):
    return lambda d: ("ag_take_indices_dev", iw, d.mask.ptr, None, 0, n, N.DROP_NULLS, d.o.ptr, None, n, d.word.ptr, None)


def take(bw, iw):
    return lambda d: ("ag_take_primitive_dev", bw, d.a.ptr, None, 0, n, iw, 1, d.b.ptr, None, 0, n, 0, d.o.ptr, None, None, None)


def is_in(bw):
    return lambda d: ("ag_is_in_dev", bw, d.a.ptr, None, 0, n, d.b.ptr, None, 0, n, 0, d.o.ptr, d.valid.ptr, None, None)


def unique(bw):
    return lambda d: ("ag_unique_dev", bw, d.a.ptr, None, 0, n, d.o.ptr, None, n, d.word.ptr, None)


INV, IDX, NI, TY = N.AG_ERR_INVALID, N.AG_ERR_INDEX, N.AG_ERR_NOT_IMPLEMENTED, N.AG_ERR_TYPE
NO_SIGN = "arith: sign with differing types needs an integer input"
NO_MINMAX = "min_max: type id {} is not an integer type (internal/utils/min_max.go covers the 8 integer types)"

CASES = {
    "binary-type": (binary(BAD, N.OP_ADD, N.SHAPE_AA), TY, "arith: unsupported type id 99"),
    "binary-op": (binary(N.INT32, N.OP_DIV, N.SHAPE_AA), NI, "arith: binary op 3 has no native kernel (the reference has none either)"),
    "binary-bitwise-float": (binary(N.FLOAT64, N.OP_BIT_AND, N.SHAPE_AA), TY, "arith: bitwise ops take integer types"),
    "binary-shape": (binary(N.INT32, N.OP_ADD, BAD_SHAPE), INV, "arith: bad operand shape 7"),
    "binary-bitwise-float-before-shape": (binary(N.FLOAT32, N.OP_BIT_XOR, BAD_SHAPE), TY, "arith: bitwise ops take integer types"),
    "binary-op-before-shape": (binary(N.UINT8, N.OP_DIV, BAD_SHAPE), NI, "arith: binary op 3 has no native kernel (the reference has none either)"),
    "spans-type": (spans(BAD, N.OP_ADD, N.SHAPE_AA), TY, "arith: unsupported type id 99"),
    "spans-op": (spans(N.INT64, N.OP_DIV, N.SHAPE_AA), NI, "arith: binary op 3 has no native kernel"),
    "spans-bitwise-float": (spans(N.FLOAT32, N.OP_BIT_OR, N.SHAPE_AA), TY, "arith: bitwise ops take integer types"),
    "spans-shape": (spans(N.INT16, N.OP_MUL, BAD_SHAPE), INV, "arith: bad operand shape 7"),
    "unary-same-type": (unary_same(BAD, N.OP_ABS), TY, "arith: unsupported type id 99"),
    "unary-same-op": (unary_same(N.INT32, N.OP_ADD), NI, "arith: unary op 0 has no native kernel"),
    "unary-same-bitnot-float": (unary_same(N.FLOAT64, N.OP_BIT_NOT), TY, "arith: bit_wise_not takes integer types"),
    "unary-diff-op": (unary_diff(N.INT32, N.INT8, N.OP_ABS), NI, "arith: unary_diff_type only implements SIGN (base_arithmetic.cc:427-438)"),
    "unary-diff-float-input": (unary_diff(N.FLOAT64, N.INT8, N.OP_SIGN), NI, NO_SIGN),
    "unary-diff-itype": (unary_diff(BAD, N.INT8, N.OP_SIGN), NI, NO_SIGN),
    "unary-diff-otype": (unary_diff(N.INT32, BAD, N.OP_SIGN), TY, "arith: unsupported output type id 99"),
    "unary-diff-itype-before-otype": (unary_diff(N.FLOAT32, BAD, N.OP_SIGN), NI, NO_SIGN),
    "checked-type": (checked(BAD, N.OP_ADD_CHECKED, N.SHAPE_AA), TY, "arith_checked: type id 99 is not a numeric type"),
    "checked-abs-checked": (checked(N.INT32, N.OP_ABS_CHECKED, N.SHAPE_AA), NI, "arith_checked: op 25 is not a checked integer op"),
    "checked-float-op": (checked(N.FLOAT64, N.OP_ADD_CHECKED, N.SHAPE_AA), NI,
                         "arith_checked: op 21 on a floating point type (only DIV / DIV_CHECKED have NotNull float kernels)"),
    "checked-shape": (checked(N.INT32, N.OP_ADD_CHECKED, BAD_SHAPE), INV, "arith_checked: bad operand shape 7"),
    "checked-float-shape": (checked(N.FLOAT32, N.OP_DIV, BAD_SHAPE), INV, "arith_checked: bad operand shape 7"),
    "checked-op-before-shape": (checked(N.UINT16, N.OP_BIT_AND, BAD_SHAPE), NI, "arith_checked: op 64 is not a checked integer op"),
    "unary-checked-op": (unary_checked(N.INT32, N.OP_ADD), NI, "arith_unary_checked: op 0"),
    "unary-checked-type": (unary_checked(BAD, N.OP_ABS_CHECKED), TY, "arith: unsupported type id 99"),
    "compare-type": (compare(BAD, N.CMP_EQ, N.SHAPE_AA), TY, "compare: unsupported type id 99"),
    "compare-cmp": (compare(N.INT32, BAD_CMP, N.SHAPE_AA), INV, "compare: bad operator 9"),
    "compare-eq-shape": (compare(N.INT32, N.CMP_EQ, BAD_SHAPE), INV, "compare: bad operand shape 7"),
    "compare-gt-shape": (compare(N.INT32, N.CMP_GT, BAD_SHAPE), INV, "compare: bad operand shape 7"),
    "compare-type-before-cmp": (compare(BAD, BAD_CMP, BAD_SHAPE), TY, "compare: unsupported type id 99"),
    "compare-cmp-before-shape": (compare(N.INT8, BAD_CMP, BAD_SHAPE), INV, "compare: bad operator 9"),
    "cast-itype": (cast(BAD, N.INT32), TY, "cast: unsupported input type id 99"),
    "cast-otype": (cast(N.INT32, BAD), TY, "cast: unsupported output type id 99"),
    "cast-itype-before-otype": (cast(N.FLOAT16, BAD), TY, "cast: unsupported input type id 10"),
    "cumsum-type": (cumsum(BAD), TY, "cumulative_sum: input type must be numeric, got type id 99"),
    "cumsum-init-type": (cumsum_init(BAD), TY, "cumulative_sum: input type must be numeric, got type id 99"),
    "sort-type": (sort(BAD), NI, "sort_indices: unsupported type id 99 (fixed-width numeric columns only)"),
    "min-max-float": (min_max(N.FLOAT64), TY, NO_MINMAX.format(N.FLOAT64)),
    "min-max-type": (min_max(BAD), TY, NO_MINMAX.format(BAD)),
    "filter-width": (filt(24), TY, "filter: invalid values bit width 24"),
    "filter-compare-narrow-type": (filter_compare(N.INT16, N.CMP_GT), NI,
                                   "filter_compare: fused path covers 32/64-bit types; use compare + filter for type id 5"),
    "filter-compare-type": (filter_compare(BAD, N.CMP_GT), NI,
                            "filter_compare: fused path covers 32/64-bit types; use compare + filter for type id 99"),
    "filter-compare-cmp": (filter_compare(N.INT64, BAD_CMP), INV, "filter_compare: bad operator 9"),
    "filter-compare-type-before-cmp": (filter_compare(N.UINT8, BAD_CMP), NI,
                                       "filter_compare: fused path covers 32/64-bit types; use compare + filter for type id 2"),
    "take-indices-width": (take_indices(8), TY, "take_indices: index width must be 16 or 32"),
    "take-value-width": (take(24, 32), INV, "take: invalid values byte width for take"),
    "take-index-width": (take(64, 24), IDX, "take: invalid indices byte width"),
    "take-bool-index-width": (take(1, 24), IDX, "take: invalid indices byte width"),
    "take-value-before-index-width": (take(24, 24), INV, "take: invalid values byte width for take"),
    "is-in-width": (is_in(24), NI, "is_in: fixed-width values of 1/2/4/8 bytes only (got 24 bits)"),
    "unique-width": (unique(24), NI, "unique: fixed-width values of 1/2/4/8 bytes only (got 24 bits)"),
}


@pytest.fixture(scope="module")
def bufs(ag):
    return Bufs()


@pytest.mark.parametrize("case", list(CASES))
def test_dispatch_rejects(ag, bufs, case):
    make, status, message = CASES[case]
    name, *args = make(bufs)
    st, msg = ag.call_status(name, *args)
    assert (st, msg) == (status, message)
    ag.call("ag_stream_sync", None)   # a refused call leaves the stream usable
