"""The run_end_encode / run_end_decode restatement (tests/run_end_ref.py) against the reference's literal cases and
against pyarrow.  CPU only."""
import json
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import run_end_ref as ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "run_end_encode.json")
NP = {"bool": np.bool_, "uint8": np.uint8, "int8": np.int8, "uint16": np.uint16, "int16": np.int16, "uint32": np.uint32,
      "int32": np.int32, "uint64": np.uint64, "int64": np.int64, "float": np.float32, "double": np.float64,
      "float32": np.float32, "float64": np.float64}
TYPES = ["bool", "uint8", "int8", "uint16", "int16", "uint32", "int32", "uint64", "int64", "float32", "float64"]
RUN_END_TYPES = ["int16", "int32", "int64"]


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def _column(chunk, ty):
    """Literal chunk -> (values with null payload 0, valid or None)."""
    valid = np.array([v is not None for v in chunk], dtype=bool)
    vals = np.array([0 if v is None else v for v in chunk], dtype=NP[ty])
    return vals, (valid if not valid.all() else None)


@pytest.mark.parametrize("case", _golden(), ids=lambda c: f"{c['name']}-{c['run_end_type']}")
def test_oracle_matches_reference_literals(case):
    for chunk, ends, values in zip(case["chunks"], case["run_ends"], case["values"]):
        vals, valid = _column(chunk, case["type"])
        got_ends, got_vals, got_valid, _ = ref.encode(vals, valid, case["run_end_type"])
        assert got_ends.tolist() == ends
        got = [(v.item() if (got_valid is None or ok) else None) for v, ok in
               zip(got_vals, got_valid if got_valid is not None else [True] * len(got_vals))]
        assert got == values
        # and back
        dv, dvalid = ref.decode(got_ends, got_vals, got_valid, 0, len(chunk))
        assert dv.tolist() == vals.tolist()
        assert (dvalid is None and valid is None) or dvalid.tolist() == valid.tolist()


def _seeded(ty, n, run_len, null_rate, rng):
    runs = max(1, n // run_len)
    lens = rng.integers(1, 2 * run_len, runs)
    if ty == "bool":
        base = rng.integers(0, 2, runs).astype(bool)
    elif ty.startswith("float"):
        base = rng.integers(-3, 4, runs).astype(NP[ty])   # no NaN, no -0.0
        base[base == 0] = 1
    else:
        base = rng.integers(0, 4, runs).astype(NP[ty])
    vals = np.repeat(base, lens)[:n]
    valid = rng.random(len(vals)) >= null_rate if null_rate else None
    if valid is not None:
        vals = vals.copy()
        vals[~valid] = 0   # pyarrow writes 0 under a null
    return vals, valid


def _pa_array(vals, valid, ty, offset):
    """pyarrow array of (vals, valid) sliced at `offset` (pad rows in front)."""
    pad_v = np.zeros(offset, dtype=vals.dtype)
    arr = pa.array(np.concatenate([pad_v, vals]), mask=None if valid is None else ~np.concatenate([np.ones(offset, bool), valid]),
                   type=pa.bool_() if ty == "bool" else pa.from_numpy_dtype(NP[ty]))
    return arr.slice(offset)


@pytest.mark.parametrize("ty", TYPES)
@pytest.mark.parametrize("rt", RUN_END_TYPES)
def test_oracle_matches_pyarrow(ty, rt):
    rng = np.random.default_rng(hash((ty, rt)) & 0xFFFF)
    for run_len, null_rate, offset, chunks in [(1, 0.0, 0, 1), (3, 0.0, 5, 1), (4, 0.2, 3, 2), (16, 0.1, 0, 3), (40, 0.5, 7, 2)]:
        vals, valid = _seeded(ty, 500, run_len, null_rate, rng)
        cuts = sorted(rng.integers(0, len(vals), chunks - 1).tolist()) if chunks > 1 else []
        bounds = [0] + cuts + [len(vals)]
        for a, b in zip(bounds[:-1], bounds[1:]):   # chunkwise: every chunk on its own
            v, m = vals[a:b], None if valid is None else valid[a:b]
            want = pc.run_end_encode(_pa_array(v, m, ty, offset), run_end_type=getattr(pa, rt)())
            ends, rvals, rvalid, nulls = ref.encode(v, m, rt)
            assert ends.tolist() == want.run_ends.to_pylist()
            exp_vals = want.values.to_pylist()
            got_vals = [(x.item() if (rvalid is None or ok) else None) for x, ok in
                        zip(rvals, rvalid if rvalid is not None else [True] * len(rvals))]
            assert got_vals == exp_vals
            assert nulls == want.values.null_count
            # decode of a slice that cuts runs at both ends, against pyarrow's decode of the same slice
            if b - a > 4:
                off, ln = 1, b - a - 3
                dv, dm = ref.decode(ends, rvals, rvalid, off, ln)
                exp = pc.run_end_decode(want.slice(off, ln)).to_pylist()
                got = [(x.item() if (dm is None or ok) else None) for x, ok in zip(dv, dm if dm is not None else [True] * len(dv))]
                assert got == exp


def test_float_difference_from_pyarrow():
    """IEEE ==: NaN rows never merge and +0.0 / -0.0 share a run.  pyarrow compares raw bytes: equal NaN payloads merge
    and ±0 split.  The restatement follows the reference; this pins where the two differ."""
    for dt in (np.float32, np.float64):
        x = np.array([np.nan, np.nan, 0.0, -0.0, -0.0, 1.0], dtype=dt)
        ends, vals, _, _ = ref.encode(x, None, "int32")
        assert ends.tolist() == [1, 2, 5, 6]                 # NaN | NaN | 0.0 -0.0 -0.0 | 1.0
        assert np.signbit(vals[2]) == False                  # the run keeps the bits of its first row (+0.0)
        want = pc.run_end_encode(pa.array(x), run_end_type=pa.int32())
        assert want.run_ends.to_pylist() == [2, 3, 5, 6]     # pyarrow: NaN NaN | 0.0 | -0.0 -0.0 | 1.0


@pytest.mark.parametrize("rt,mx", [("int16", 32767), ("int32", 2 ** 31 - 1)])
def test_run_end_type_limits(rt, mx):
    ref.check_length(mx, rt)
    with pytest.raises(ref.RunEndLengthError, match=f"can hold: {mx}"):
        ref.check_length(mx + 1, rt)
    assert ref.encode(np.zeros(0, np.int8), None, "int16")[0].tolist() == []   # n == 0: no error even for int16


def test_malformed_run_ends():
    vals = np.arange(4)
    with pytest.raises(ref.MalformedRunEnds):
        ref.decode([2, 2, 5, 6], vals, None, 0, 6)      # a repeated run end
    with pytest.raises(ref.MalformedRunEnds):
        ref.decode([2, 4, 3, 6], vals, None, 0, 6)      # a decrease
    with pytest.raises(ref.MalformedRunEnds):
        ref.decode([2, 4, 5, 6], vals, None, 3, 4)      # the last run end is short of offset+length
    assert ref.decode([2, 4, 5, 6], vals, None, 1, 4)[0].tolist() == [0, 1, 1, 2]   # a slice that cuts runs at both ends
