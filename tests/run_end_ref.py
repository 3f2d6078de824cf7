"""NumPy restatement of run_end_encode / run_end_decode for BOOL and the numeric types (the oracle).

Semantics of arrow-go's kernels/vector_run_end_encode.go for fixed-width values:
- rows i-1 and i share a run iff their validity bits are equal AND their values compare equal with the physical
  type's == (:96-105), the payload under a null included: float NaN rows each start a run, +0.0 and -0.0 share one
  (the run keeps the bits of its first row);
- run r: run_ends[r] = the first row of run r+1 (n for the last run), values[r] = the value of its first row,
  values validity bit r = that row's validity;
- the values child has a validity bitmap iff the input has one;
- n greater than the run-end type's maximum is ErrInvalid (validateRunEndType :437-444);
- decode: row j of the slice [offset, offset+length) takes the run p with run_ends[p-1] <= offset+j < run_ends[p],
  the last run clipped at offset+length.
"""
import numpy as np

RUN_END_MAX = {"int16": (1 << 15) - 1, "int32": (1 << 31) - 1, "int64": (1 << 63) - 1}


class RunEndLengthError(ValueError):
    pass


def check_length(n, run_end_type):
    mx = RUN_END_MAX[run_end_type]
    if n > mx:
        raise RunEndLengthError(f"cannot run-end encode arrays with more elements than the run end type can hold: {mx}")


def boundaries(values, valid=None):
    """Bool array: row i starts a run.  `values` is a numpy array (bool for BOOL), `valid` a bool array or None."""
    values = np.asarray(values)
    n = len(values)
    b = np.zeros(n, dtype=bool)
    if n == 0:
        return b
    b[0] = True
    with np.errstate(invalid="ignore"):
        b[1:] = ~(values[1:] == values[:-1])   # IEEE == for floats, bit equality for integers and booleans
    if valid is not None:
        valid = np.asarray(valid, dtype=bool)
        b[1:] |= valid[1:] != valid[:-1]
    return b


def encode(values, valid=None, run_end_type="int32"):
    """(run_ends int64, run_values, run_valid or None, null_runs)."""
    values = np.asarray(values)
    n = len(values)
    check_length(n, run_end_type)
    b = boundaries(values, valid)
    starts = np.flatnonzero(b)
    ends = np.append(starts[1:], n).astype(np.int64) if n else np.zeros(0, np.int64)
    run_values = values[starts]
    if valid is None:
        return ends, run_values, None, 0
    run_valid = np.asarray(valid, dtype=bool)[starts]
    return ends, run_values, run_valid, int((~run_valid).sum())


def count(values, valid=None):
    """(runs, null runs) of CountNumberOfRuns."""
    b = boundaries(values, valid)
    runs = int(b.sum())
    if valid is None:
        return runs, 0
    return runs, int((b & ~np.asarray(valid, dtype=bool)).sum())


class MalformedRunEnds(ValueError):
    pass


def covering_runs(run_ends, offset, length):
    """(first, last): the runs that cover rows offset and offset+length-1; MalformedRunEnds when the run ends over
    [first, last] do not increase strictly or stop before offset+length."""
    run_ends = np.asarray(run_ends, dtype=np.int64)
    if length == 0:
        return 0, -1
    first = int(np.searchsorted(run_ends, offset, side="right"))
    last = int(np.searchsorted(run_ends, offset + length - 1, side="right"))
    if first >= len(run_ends) or last >= len(run_ends):
        raise MalformedRunEnds("the run ends stop before offset+length")
    seg = run_ends[max(first - 1, 0): last + 1]
    if np.any(np.diff(seg) <= 0) or last < first:
        raise MalformedRunEnds("the run ends do not increase strictly")
    return first, last


def decode(run_ends, run_values, run_valid=None, offset=0, length=None):
    """(values, valid or None) of the slice [offset, offset+length)."""
    run_ends = np.asarray(run_ends, dtype=np.int64)
    if length is None:
        length = int(run_ends[-1]) - offset if len(run_ends) else 0
    covering_runs(run_ends, offset, length)
    rows = np.arange(offset, offset + length, dtype=np.int64)
    p = np.searchsorted(run_ends, rows, side="right")
    vals = np.asarray(run_values)[p]
    if run_valid is None:
        return vals, None
    return vals, np.asarray(run_valid, dtype=bool)[p]
