"""A NumPy model of take on record batches and tables, FilterRecordBatch and FilterTable, output chunk lengths included.

It restates the reference's four selections (arrow/compute/selection.go):
  takeRecordImpl  (:160-204)  chunked indices are concatenated; every column becomes one array of len(indices) rows.
  takeTableImpl   (:117-158)  -> takeChunkedImpl (:246-300) -> ChunkedPrimitiveTake (kernels/vector_selection.go:1194-1228):
                              every column gets one chunk per index chunk (empty index chunks give empty chunks), an
                              array index gives one chunk.  A table without columns has no rows (array.NewTable(.., -1)).
  FilterRecordBatch (:679-722) the mask becomes indices (GetTakeIndices) and every column is taken without a bounds check.
  FilterTable     (:724-800)  columns and mask are cut at every chunk boundary of any of them
                              (exec.RechunkArraysConsistently); a span that selects no row gives no chunk; a table
                              without rows comes back as it is.
Per element these are PrimitiveTake: out = column[idx], valid = idx valid and column[idx] valid, value 0 where the
output is null.  Only valid index slots are bounds-checked (negative, or >= rows once read as unsigned), and the error
names the index of the first offending row: ErrIndex "<value> out of bounds".

A column is a list of (values, valid) chunks of logical rows (valid None: no nulls); indices and masks are a list of
(values, valid) chunks plus a flag saying whether they are chunked.
"""
import numpy as np

from exec_model import Fail

DROP_NULLS, EMIT_NULLS = 0, 1


def _flat(chunks, dtype=None):
    if not chunks:
        return np.zeros(0, dtype=dtype or np.int64), np.zeros(0, dtype=bool)
    vals = np.concatenate([np.asarray(v) for v, _ in chunks])
    valid = np.concatenate([np.ones(len(v), dtype=bool) if ok is None else np.asarray(ok, dtype=bool) for v, ok in chunks])
    return vals, valid


def _bad(idx, ivalid, nrows):
    """Row of the first valid out-of-bounds index, or None."""
    signed = np.issubdtype(idx.dtype, np.signedinteger)
    neg = (idx < 0) if signed else np.zeros(idx.size, dtype=bool)
    big = idx.astype(np.uint64) >= np.uint64(nrows) if idx.size else np.zeros(0, dtype=bool)
    oob = ivalid & (neg | big)
    return int(np.argmax(oob)) if oob.any() else None


def nullable(chunks):
    """Whether a column or index vector can hold nulls: some chunk has a validity bitmap with a null in it.  The output
    of a take has a validity bitmap exactly when its column or its indices can hold nulls."""
    return any(ok is not None and not np.all(ok) for _, ok in chunks)


def gather(col, idx, ivalid, bitmap=True):
    """PrimitiveTake of one flattened column: (values, valid).  An out-of-range valid index (no bounds check) gives value
    0, and a null only when the output has a validity bitmap (`bitmap`)."""
    vals, valid = col
    ok = ivalid.copy()
    n = vals.size
    safe = np.zeros(idx.size, dtype=np.int64)
    inb = ok & (idx.astype(np.int64) >= 0) & (idx.astype(np.uint64) < np.uint64(n)) if idx.size else ok
    safe[inb] = idx[inb].astype(np.int64)
    ok = inb & (valid[safe] if n else np.zeros(idx.size, dtype=bool))
    out = np.where(ok, vals[safe] if n else np.zeros(idx.size, dtype=vals.dtype), np.zeros(1, dtype=vals.dtype))
    return out.astype(vals.dtype), ok if bitmap else np.ones(idx.size, dtype=bool)


def take_record(cols, nrows, indices, bounds_check=True):
    """takeRecordImpl: [(values, valid)] per column and the row count, or a Fail."""
    idx, ivalid = _flat(indices[0])
    if cols and bounds_check:
        b = _bad(idx, ivalid, nrows)
        if b is not None:
            return Fail("ErrIndex", f"{idx[b]} out of bounds")
    inull = nullable(indices[0])
    return [gather(_flat(c), idx, ivalid, inull or nullable(c)) for c in cols], idx.size


def take_table(cols, nrows, indices, bounds_check=True):
    """takeTableImpl: [[(values, valid) per output chunk]] per column and the row count, or a Fail."""
    ichunks, _chunked = indices
    if cols and bounds_check:
        for v, ok in ichunks:   # checkIndexBoundsChunked: the first chunk in order that holds an offender
            v = np.asarray(v)
            b = _bad(v, np.ones(v.size, dtype=bool) if ok is None else np.asarray(ok), nrows)
            if b is not None:
                return Fail("ErrIndex", f"{v[b]} out of bounds")
    out = []
    inull = nullable(ichunks)
    for c in cols:
        flat = _flat(c)
        out.append([gather(flat, np.asarray(v), np.ones(len(v), dtype=bool) if ok is None else np.asarray(ok), inull or nullable(c))
                    for v, ok in ichunks])
    rows = sum(len(v) for v, _ in ichunks) if cols else 0
    return out, rows


def take_indices(mask, mvalid, sel):
    """GetTakeIndices: (row indices, index validity) of a mask span."""
    mvalid = np.ones(mask.size, dtype=bool) if mvalid is None else mvalid
    if sel == DROP_NULLS:
        rows = np.nonzero(mask & mvalid)[0]
        return rows, np.ones(rows.size, dtype=bool)
    rows = np.nonzero(mask | ~mvalid)[0]
    return rows, mvalid[rows]


def filter_record_batch(cols, nrows, mask, sel):
    m, mv = _flat(mask[0])
    if m.size != nrows:
        return Fail("ErrInvalid", "filter inputs must all be the same length")
    idx, ivalid = take_indices(m.astype(bool), mv, sel)
    return [gather(_flat(c), idx, ivalid) for c in cols], idx.size


def spans(lens):
    """RechunkArraysConsistently: [(start, length)] cut at every boundary of every argument, empty chunks skipped."""
    total = sum(lens[0]) if lens else 0
    cuts = {0, total}
    for ls in lens:
        cuts.update(np.cumsum([0] + list(ls)).tolist())
    cuts = sorted(cuts)
    return [(a, b - a) for a, b in zip(cuts, cuts[1:]) if b > a]


def filter_table(cols, nrows, mask, sel):
    """FilterTable: [[(values, valid) per output chunk]] per column and the row count, or a Fail; None when the table
    comes back unchanged (no rows)."""
    m, mv = _flat(mask[0])
    if m.size != nrows:
        return Fail("ErrInvalid", "filter inputs must all be the same length")
    if nrows == 0:
        return None
    flat = [_flat(c) for c in cols]
    lens = [[len(v) for v, _ in c] for c in cols] + [[len(v) for v, _ in mask[0]]]
    out = [[] for _ in cols]
    rows = 0
    for a, ln in spans(lens):
        idx, ivalid = take_indices(m[a:a + ln].astype(bool), mv[a:a + ln], sel)
        if idx.size == 0:
            continue
        rows += idx.size
        for c, (vals, valid) in enumerate(flat):
            out[c].append(gather((vals[a:a + ln], valid[a:a + ln]), idx, ivalid))
    return out, rows
