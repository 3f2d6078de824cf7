"""ag_arith_binary_spans[_dev] with more spans than one launch of the span kernel takes (256 non-empty spans per launch):
the call runs as several launches of the same kernel, each with its own slice of the span table.  Checked span by span
against the oracle's restatement of the reference's SIMD loop (the one test_gpu_arith.py checks against the reference
itself), through test_gpu_arith._spans_case."""
import numpy as np
import pytest

from arrow_go_b200 import _native as N
from helpers import NP_OF, TYPE_NAME
from test_gpu_arith import _spans_case

pytestmark = pytest.mark.gpu

CAP = 256   # non-empty spans per launch (kSpanTable in csrc/elementwise.cu)
TYPES = [N.FLOAT64, N.INT32, N.UINT16, N.UINT8]
SHAPES = [N.SHAPE_AA, N.SHAPE_AS, N.SHAPE_SA]


class _Restatement:
    """The `ref` interface of _spans_case (arithmetic_{binary,arr_scalar,scalar_arr}_<isa>) over oracle/cpu_ref.c."""

    def __init__(self, cpu):
        self.cpu = cpu

    def __getattr__(self, name):
        shape = {"arithmetic_binary_": N.SHAPE_AA, "arithmetic_arr_scalar_": N.SHAPE_AS, "arithmetic_scalar_arr_": N.SHAPE_SA}[name[:name.rindex("_") + 1]]

        def fn(type_id, op, l, r, out, n):
            assert self.cpu.ref_arith_binary(type_id, op, shape, l, r, out, n) == 0
        return fn


def _lens(rng, count, tile, empties_at=()):
    """`count` non-empty spans, mostly a few hundred rows, every 16th longer than a tile; empty spans inserted before
    the non-empty spans whose index is in `empties_at`."""
    out = []
    for k in range(count):
        if k in empties_at:
            out += [0, 0]
        out.append(tile + int(rng.integers(1, 50)) if k % 16 == 5 else int(rng.integers(1, 400)))
    return out


def _cases(rng, tile):
    """Span lengths crossing the per-launch cap: one below, exactly at it, one above, thousands; and empty
    spans at the cap boundary both when the non-empty spans fit one launch and when they do not."""
    return [_lens(rng, CAP - 1, tile), _lens(rng, CAP, tile), _lens(rng, CAP + 1, tile), _lens(rng, 2000, tile),
            _lens(rng, CAP, tile, empties_at=(CAP - 1,)) + [0, 0], _lens(rng, CAP + 1, tile, empties_at=(CAP - 1, CAP))]


def _offsets(rng, lens, nvec, phase):
    if phase == "aligned":
        return [(0, 0, 0)] * len(lens)
    if phase == "shared":      # one misalignment per span on every operand (what executeSpans produces)
        return [(k % nvec,) * 3 for k in range(len(lens))]
    # independent phases per operand (the shift path) in every launch after the first; the first launch stays aligned,
    # so one call mixes launches with and without the shift path
    out, seen = [], 0
    for ln in lens:
        out.append((0, 0, 0) if seen < CAP else tuple(int(x) for x in rng.integers(0, 2 * nvec, 3)))
        seen += ln > 0
    return out


@pytest.mark.parametrize("type_id", TYPES, ids=lambda t: TYPE_NAME[t])
@pytest.mark.parametrize("shape", SHAPES, ids=["aa", "as", "sa"])
@pytest.mark.parametrize("phase", ["aligned", "shared", "independent"])
def test_spans_past_one_launch(ag, cpu, isa, type_id, shape, phase):
    rng = np.random.default_rng(0x5BA3 + type_id * 13 + shape * 7 + len(phase))
    isz = np.dtype(NP_OF[type_id]).itemsize
    nvec, tile = 16 // isz, 16384 // isz   # rows per tile of the span kernel (kBinaryTileBytes)
    ref = _Restatement(cpu)
    for lens in _cases(rng, tile):
        _spans_case(ag, ref, isa, type_id, N.OP_ADD, shape, lens, _offsets(rng, lens, nvec, phase), rng)
    lens = _lens(rng, 600, tile)
    _spans_case(ag, ref, isa, type_id, N.OP_SUB_CHECKED, shape, lens, _offsets(rng, lens, nvec, phase), rng)


def test_host_spans_past_one_launch(ag, cpu, isa):
    rng = np.random.default_rng(0x5BA4)
    lens = _lens(rng, 2 * CAP + 3, 2048, empties_at=(CAP,))
    offs = [tuple(int(x) for x in rng.integers(0, 4, 3)) for _ in lens]
    _spans_case(ag, _Restatement(cpu), isa, N.FLOAT64, N.OP_ADD, N.SHAPE_AA, lens, offs, rng, host=True)
