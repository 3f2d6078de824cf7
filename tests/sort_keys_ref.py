"""sort_indices over several keys and chunked columns: a restatement of the reference and a model of the device order.

A column is a list of chunks, each chunk a pair (values, valid): a NumPy array (bool for BOOL columns) and a bool array
of the same length, or None when the chunk has no nulls.  A key is (column, order, null_placement) with order
0 ascending / 1 descending and null_placement 0 at end / 1 at start; `columns[column]` is the key's column.

reference_sort_indices restates kernels.SortIndices (arrow/compute/internal/kernels/vector_sort.go:390-481) with its
four paths, comparisons included; it is written for clarity, not speed (a few thousand rows).

sort_keys_model is the order the device produces: for every key, first to last,
    NullsAtEnd   : [finite values in key order | NaN | null]
    NullsAtStart : [null | NaN | finite values in key order]
with ties (NaN and null rows included) ordered by the next key and ties on every key kept in row order.  It is one
stable np.lexsort over per-key (class, value rank) pairs.  It agrees with the reference except where the reference
places NaN by order (chunk merges and the tail comparator above 8 keys, vector_sort_support.go:120-137) - DESIGN §2.
"""
import functools

import numpy as np

ASC, DESC = 0, 1
AT_END, AT_START = 0, 1
MAX_RADIX_SORT_KEYS = 8   # vector_sort.go:84


def _flat(col):
    """(values, valid) of a whole column."""
    if not col:
        return np.zeros(0), np.zeros(0, dtype=bool)
    vals = np.concatenate([np.asarray(v) for v, _ in col])
    valid = np.concatenate([np.ones(len(v), dtype=bool) if ok is None else np.asarray(ok, dtype=bool) for v, ok in col])
    return vals, valid


# ---------------------------------------------------------------------------------------------------------------- model
def _key_ranks(col, order, placement):
    vals, valid = _flat(col)
    n = len(vals)
    is_float = vals.dtype.kind == "f"
    nan = valid & np.isnan(vals) if is_float else np.zeros(n, dtype=bool)
    fin = valid & ~nan
    cls = np.where(fin, 0, np.where(nan, 1, 2))
    code = cls if placement == AT_END else 2 - cls
    rank = np.zeros(n, dtype=np.int64)
    if fin.any():
        v = vals[fin]
        if is_float:
            v = np.where(v == 0, 0.0, v).astype(np.float64)   # -0.0 == +0.0
        elif v.dtype == np.bool_:
            v = v.astype(np.uint8)
        uniq, inv = np.unique(v, return_inverse=True)
        rank[fin] = (len(uniq) - 1 - inv) if order == DESC else inv
    return code, rank


def sort_keys_model(columns, keys):
    """uint64 permutation in the device's order (see the module docstring)."""
    arrays = []
    for c, order, placement in reversed(keys):   # np.lexsort: the last array is the primary key
        code, rank = _key_ranks(columns[c], order, placement)
        arrays += [rank, code]
    if not keys or len(arrays[0]) == 0:
        return np.zeros(0, dtype=np.uint64)
    return np.lexsort(arrays).astype(np.uint64)


# -------------------------------------------------------------------------------------------------------- restatement
class _Comparator:
    """physicalSort<T>Column (vector_sort_physical.go): row compare and the null / null-like tests."""

    def __init__(self, col):
        self.vals, self.valid = _flat(col)
        self.is_float = self.vals.dtype.kind == "f"
        self.validity_nulls = bool((~self.valid).any())          # columnHasValidityNulls (chunksHaveNulls)
        self.vals_py = self.vals.tolist()

    def is_null(self, i):
        return not self.valid[i]

    def has_null_like(self):                                  # hasNullLikeValues: true for float columns
        return self.is_float

    def is_null_like(self, i):                                # isNullLikeAt: NaN and not null
        return self.is_float and bool(self.valid[i]) and self.vals_py[i] != self.vals_py[i]

    def compare(self, i, j, key):                             # compareRowsForKey, vector_sort_physical.go:514-531
        _, order, placement = key
        if self.validity_nulls:                               # compareKeyedNulls, vector_sort_support.go:152-169
            ni, nj = not self.valid[i], not self.valid[j]
            if ni and nj:
                return 0
            if ni:
                return -1 if placement == AT_START else 1
            if nj:
                return 1 if placement == AT_START else -1
        vi, vj = self.vals_py[i], self.vals_py[j]
        if self.is_float:                                     # compareFloatNaNs, vector_sort_support.go:120-137
            ai, aj = vi != vi, vj != vj
            if ai and aj:
                return 0
            if ai:
                return 1 if order == ASC else -1
            if aj:
                return -1 if order == ASC else 1
        c = (vi > vj) - (vi < vj)                             # compareOrdered (-0.0 == +0.0)
        return -c if order == DESC else c


def _stable_sort(indices, lo, hi, cmp):
    indices[lo:hi] = sorted(indices[lo:hi], key=functools.cmp_to_key(cmp))


def _no_validity_nulls(lo, hi, placement):                   # nullPartitionNoValidityNulls, vector_sort_internal.go:142-148
    # (non_nulls_lo, non_nulls_hi, nulls_lo, nulls_hi)
    return (lo, hi, lo, lo) if placement == AT_START else (lo, hi, hi, hi)


def _partition(indices, lo, hi, placement, pred):
    """Stable partition of indices[lo:hi] by pred, the pred rows on the placement side (partitionNullsOnly /
    partitionNullLikes, vector_sort_internal.go:36-140)."""
    seg = indices[lo:hi]
    yes = [i for i in seg if pred(i)]
    no = [i for i in seg if not pred(i)]
    if not yes:
        return _no_validity_nulls(lo, hi, placement)
    if placement == AT_START:
        indices[lo:hi] = yes + no
        return (lo + len(yes), hi, lo, lo + len(yes))
    indices[lo:hi] = no + yes
    return (lo, lo + len(no), lo + len(no), hi)


def _partition_key(indices, comp, key, lo, hi):
    placement = key[2]
    if comp.validity_nulls:
        p = _partition(indices, lo, hi, placement, comp.is_null) if lo < hi else (lo, lo, lo, lo)
    else:
        p = _no_validity_nulls(lo, hi, placement)
    if comp.has_null_like() and p[0] < p[1]:
        q = _partition(indices, p[0], p[1], placement, comp.is_null_like)
    else:
        q = _no_validity_nulls(p[0], p[1], placement)
    return p, q


def _radix_range(indices, comps, keys, k, lo, hi):
    """radixRecordBatchSortRange, vector_sort_internal.go:170-204."""
    if hi - lo <= 1 or k >= len(keys):
        return
    key, comp = keys[k], comps[k]
    p, q = _partition_key(indices, comp, key, lo, hi)
    fin_lo, fin_hi, nan_lo, nan_hi = q
    null_lo, null_hi = p[2], p[3]
    _stable_sort(indices, fin_lo, fin_hi, lambda a, b: comp.compare(a, b, key))
    if k == len(keys) - 1:
        return
    _radix_range(indices, comps, keys, k + 1, nan_lo, nan_hi)
    _radix_range(indices, comps, keys, k + 1, null_lo, null_hi)
    rs = fin_lo                                               # visitConstantRanges, :153-167
    for t in range(fin_lo + 1, fin_hi + 1):
        if t < fin_hi and comp.compare(indices[t - 1], indices[t], key) == 0:
            continue
        _radix_range(indices, comps, keys, k + 1, rs, t)
        rs = t


def _tail(comps, keys, start):                                # makeTailComparator, :239-248
    def cmp(a, b):
        for i in range(start, len(keys)):
            v = comps[i].compare(a, b, keys[i])
            if v:
                return v
        return 0
    return cmp


def _multi_key_range(indices, comps, keys, lo, hi):
    """multipleKeyRecordBatchSortRange, vector_sort_internal.go:208-235 (more than 8 keys)."""
    if hi - lo <= 1:
        return
    key, comp = keys[0], comps[0]
    p, q = _partition_key(indices, comp, key, lo, hi)
    tail = _tail(comps, keys, 1)
    _stable_sort(indices, q[0], q[1], lambda a, b: comp.compare(a, b, key) or tail(a, b))
    _stable_sort(indices, q[2], q[3], tail)
    _stable_sort(indices, p[2], p[3], tail)


def _array_sort_range(indices, comp, key, lo, hi):
    """arraySortOneColumnRange, vector_sort_internal.go:252-273."""
    if hi - lo <= 1:
        return
    if not comp.validity_nulls and not comp.has_null_like():
        _stable_sort(indices, lo, hi, lambda a, b: comp.compare(a, b, key))
        return
    _, q = _partition_key(indices, comp, key, lo, hi)
    _stable_sort(indices, q[0], q[1], lambda a, b: comp.compare(a, b, key))


def _merge_spans(indices, spans, less):
    """pairwiseMergeSortedSpans + mergeAdjacentStable (vector_sort.go:254-304)."""
    cur = list(spans)
    while len(cur) > 1:
        nxt = []
        for i in range(0, len(cur), 2):
            if i + 1 < len(cur):
                (a0, a1), (b0, b1) = cur[i], cur[i + 1]
                a, b = indices[a0:a1], indices[b0:b1]
                out, x, y = [], 0, 0
                while x < len(a) and y < len(b):
                    if not less(b[y], a[x]):
                        out.append(a[x]); x += 1
                    else:
                        out.append(b[y]); y += 1
                indices[a0:b1] = out + a[x:] + b[y:]
                nxt.append((a0, b1))
            else:
                nxt.append(cur[i])
        cur = nxt


def _aligned_boundaries(columns):                            # alignedChunkBoundaries, vector_sort.go:308-332
    ch0 = columns[0]
    if not ch0:
        return None
    offs = [0]
    for i, (v, _) in enumerate(ch0):
        for col in columns[1:]:
            if len(col) != len(ch0) or len(col[i][0]) != len(v):
                return None
        offs.append(offs[-1] + len(v))
    return offs


def reference_sort_indices(columns, keys):
    """kernels.SortIndices (vector_sort.go:390-481) with sortColumns[i] = columns[keys[i][0]]."""
    if not keys:
        raise ValueError("must provide at least one sort key")
    cols = [columns[c] for c, _, _ in keys]
    n = len(_flat(cols[0])[0])
    comps = [_Comparator(c) for c in cols]
    indices = list(range(n))
    if len(keys) == 1:
        chunks, comp, key = cols[0], comps[0], keys[0]
        if len(chunks) > 1:                                   # sortIndicesSingleColumnChunked, :336-359
            lo, spans = 0, []
            for v, _ in chunks:
                _array_sort_range(indices, comp, key, lo, lo + len(v))
                spans.append((lo, lo + len(v)))
                lo += len(v)
            _merge_spans(indices, spans, lambda a, b: comp.compare(a, b, key) < 0)
        elif not comp.validity_nulls and not comp.has_null_like():
            _stable_sort(indices, 0, n, lambda a, b: comp.compare(a, b, key))
        else:
            _array_sort_range(indices, comp, key, 0, n)
    else:
        offs = _aligned_boundaries(cols)
        radix = len(keys) <= MAX_RADIX_SORT_KEYS
        if offs is not None and len(offs) - 1 > 1:            # sortIndicesMultiColumnAlignedChunks, :363-383
            for c in range(len(offs) - 1):
                if radix:
                    _radix_range(indices, comps, keys, 0, offs[c], offs[c + 1])
                else:
                    _multi_key_range(indices, comps, keys, offs[c], offs[c + 1])
            full = _tail(comps, keys, 0)
            _merge_spans(indices, [(offs[c], offs[c + 1]) for c in range(len(offs) - 1)], lambda a, b: full(a, b) < 0)
        elif radix:
            _radix_range(indices, comps, keys, 0, 0, n)
        else:
            _multi_key_range(indices, comps, keys, 0, n)
    return np.array(indices, dtype=np.uint64)


def quirk_possible(columns, keys):
    """True when the reference's result may place NaN by order rather than by placement: a single chunked key, aligned
    multi-chunk key columns, or more than 8 keys."""
    cols = [columns[c] for c, _, _ in keys]
    if len(keys) == 1:
        return len(cols[0]) > 1
    offs = _aligned_boundaries(cols)
    return (offs is not None and len(offs) > 2) or len(keys) > MAX_RADIX_SORT_KEYS


# ------------------------------------------------------------------------------------------------ shared test inputs
NP_OF_NAME = {"bool": np.bool_, "uint8": np.uint8, "int8": np.int8, "uint16": np.uint16, "int16": np.int16,
              "uint32": np.uint32, "int32": np.int32, "uint64": np.uint64, "int64": np.int64,
              "float32": np.float32, "float64": np.float64}


def golden_columns(case):
    """Columns of a case of tests/golden/sort_indices_keys.json in the form above."""
    cols = []
    for ty, chunks in zip(case["types"], case["columns"]):
        col = []
        for ch in chunks:
            valid = np.array([v is not None for v in ch], dtype=bool)
            vals = np.array([(0 if v is None else (float("nan") if v == "NaN" else v)) for v in ch]).astype(NP_OF_NAME[ty])
            col.append((vals, None if valid.all() else valid))
        cols.append(col)
    return cols


def random_column(rng, ty, chunk_lens, null_p=0.1, nan_p=0.1, small=False):
    """A column of chunk lengths `chunk_lens`: nulls, NaN, +-0.0, and small or full-range values."""
    dt = np.dtype(NP_OF_NAME[ty])
    col = []
    for ln in chunk_lens:
        if dt == np.bool_:
            v = rng.integers(0, 2, ln).astype(bool)
        elif dt.kind == "f":
            v = (rng.integers(-4, 5, ln) if small else rng.standard_normal(ln) * 1e3).astype(dt)
            v[rng.random(ln) < nan_p] = np.nan
            v[rng.random(ln) < 0.05] = -0.0
        else:
            info = np.iinfo(dt)
            lo, hi = (max(info.min, -5), min(info.max, 5)) if small else (info.min, info.max)
            v = rng.integers(lo, hi, ln, dtype=dt, endpoint=True)
        valid = rng.random(ln) >= null_p if null_p else None
        col.append((v, valid))
    return col
