"""CPU checks of tests/sort_keys_ref.py: the restatement of kernels.SortIndices reproduces the reference's literal
vectors, agrees with the model of the device order outside the NaN quirk, the model agrees with pyarrow, and the
quirk itself (DESIGN §2) is pinned."""
import json
import os

import numpy as np
import pytest

from sort_keys_ref import (ASC, AT_END, AT_START, DESC, golden_columns, quirk_possible, random_column,
                           reference_sort_indices, sort_keys_model)

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "sort_indices_keys.json")))
TYPES = ["bool", "uint8", "int8", "uint16", "int16", "uint32", "int32", "uint64", "int64", "float32", "float64"]


@pytest.mark.parametrize("case", GOLDEN["cases"], ids=[c["name"] for c in GOLDEN["cases"]])
def test_golden_restatement_and_model(case):
    cols = golden_columns(case)
    keys = [tuple(k) for k in case["keys"]]
    assert reference_sort_indices(cols, keys).tolist() == case["want"]
    assert sort_keys_model(cols, keys).tolist() == case["want"]


def test_golden_lists_left_out_cases():
    assert "TestVectorSortIndicesCppRecordBatchParity/MoreTypes" in GOLDEN["left_out"]
    assert len(GOLDEN["cases"]) >= 15


def _random_case(rng, n, nkeys, layout):
    ncols = max(1, nkeys - int(rng.integers(0, 2)))     # sometimes one column serves two keys
    types = [TYPES[int(rng.integers(0, len(TYPES)))] for _ in range(ncols)]
    if layout == "aligned":
        cuts = sorted(rng.integers(0, n + 1, int(rng.integers(0, 4))).tolist())
        lens = np.diff([0] + cuts + [n]).tolist()
    cols = []
    for ty in types:
        if layout == "misaligned":
            cuts = sorted(rng.integers(0, n + 1, int(rng.integers(0, 4))).tolist())
            lens = np.diff([0] + cuts + [n]).tolist()
        elif layout == "one":
            lens = [n]
        cols.append(random_column(rng, ty, lens, null_p=float(rng.choice([0, 0.1, 0.3])), nan_p=0.15,
                                  small=bool(rng.integers(0, 2))))
    keys = [(int(rng.integers(0, ncols)), int(rng.integers(0, 2)), int(rng.integers(0, 2))) for _ in range(nkeys)]
    return cols, keys


@pytest.mark.parametrize("seed", range(40))
def test_restatement_matches_model_outside_quirk(seed):
    rng = np.random.default_rng(seed)
    nkeys = [1, 2, 3, 5, 8, 9, 12][seed % 7]
    layout = ["one", "aligned", "misaligned"][seed % 3]
    cols, keys = _random_case(rng, int(rng.integers(0, 200)), nkeys, layout)
    if quirk_possible(cols, keys):   # keep NaN where order and placement agree: (asc, at end) or (desc, at start)
        keys = [(c, o, (o if np.asarray(cols[c][0][0]).dtype.kind == "f" else p) if cols[c] else p) for c, o, p in keys]
    assert reference_sort_indices(cols, keys).tolist() == sort_keys_model(cols, keys).tolist()


@pytest.mark.parametrize("seed", range(12))
def test_model_matches_pyarrow(seed):
    pa = pytest.importorskip("pyarrow")
    pc = pytest.importorskip("pyarrow.compute")
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.integers(0, 3000))
    cols, keys = _random_case(rng, n, 1 + seed % 5, ["aligned", "misaligned"][seed % 2])
    placement = seed % 2
    keys = [(c, o, placement) for c, o, _ in keys]   # pyarrow's null placement is one for all keys
    arrays = []
    for col in cols:
        arrays.append(pa.chunked_array([pa.array(v, mask=None if ok is None else ~ok) for v, ok in col],
                                       type=pa.from_numpy_dtype(np.asarray(col[0][0]).dtype) if col else pa.int32()))
    table = pa.table({f"c{i}": a for i, a in enumerate(arrays)})
    got = pc.sort_indices(table, sort_keys=[(f"c{c}", "descending" if o else "ascending") for c, o, _ in keys],
                          null_placement="at_start" if placement else "at_end").to_numpy()
    assert got.tolist() == sort_keys_model(cols, keys).tolist()


def test_quirk_chunked_nan_ascending_nulls_at_start():
    """One chunked float key, (Ascending, NullsAtStart): the reference's chunk merge puts NaN after the finite values
    (by order); the device keeps [null | NaN | finite] (by placement)."""
    f = np.float64
    cols = [[(np.array([np.nan, 2.0], f), None), (np.array([1.0, 0.0], f), np.array([True, False]))]]
    keys = [(0, ASC, AT_START)]
    assert sort_keys_model(cols, keys).tolist() == [3, 0, 2, 1]
    assert reference_sort_indices(cols, keys).tolist() != [3, 0, 2, 1]
    # one chunk: the partition rule on both sides
    one = [[(np.array([np.nan, 2.0, 1.0, 0.0], f), np.array([True, True, True, False]))]]
    assert reference_sort_indices(one, keys).tolist() == sort_keys_model(one, keys).tolist() == [3, 0, 2, 1]


def test_quirk_nan_in_later_key_with_nine_keys():
    """Nine keys: the tail comparator orders key 1 by order, so NaN goes after 1.0 under (Ascending, NullsAtStart); the
    device (and the reference with 8 keys) put it first."""
    a = [(np.zeros(3, np.int32), None)]
    b = [(np.array([1.0, np.nan, 0.5]), None)]
    cols = [a, b]
    nine = [(0, ASC, AT_END), (1, ASC, AT_START)] + [(0, ASC, AT_END)] * 7
    eight = nine[:8]
    assert sort_keys_model(cols, nine).tolist() == [1, 2, 0]
    assert reference_sort_indices(cols, eight).tolist() == [1, 2, 0]
    assert reference_sort_indices(cols, nine).tolist() == [2, 0, 1]
