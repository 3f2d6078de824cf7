"""NumPy restatement of dictionary_encode (arrow/compute/internal/kernels/vector_hash.go:144-241) for fixed-width
values: keys compare by raw bytes, the dictionary is the distinct keys in order of first appearance over the whole
column, and a null is either masked (index 0, null slot) or encoded as one more entry where it first appears."""
import numpy as np

MASK, ENCODE = 0, 1


def dictionary_encode_ref(chunks, null_encoding=MASK):
    """chunks: [(values ndarray, valid bool ndarray or None), ...].
    Returns ([(indices int32, valid bool ndarray or None, null_count), ...], dictionary ndarray, dictionary valid or None)."""
    dtype = chunks[0][0].dtype if chunks else np.dtype(np.int64)
    lens = [len(v) for v, _ in chunks]
    vals = np.concatenate([np.ascontiguousarray(v) for v, _ in chunks]) if chunks else np.zeros(0, dtype)
    valid = np.concatenate([np.ones(len(v), bool) if m is None else np.asarray(m, bool) for v, m in chunks]) if chunks else np.zeros(0, bool)
    bits = vals.view(np.dtype(f"u{dtype.itemsize}"))
    rows = np.flatnonzero(valid)
    keys, first, inverse = np.unique(bits[rows], return_index=True, return_inverse=True)
    first_rows = rows[first]
    null_rows = np.flatnonzero(~valid)
    encode_null = null_encoding == ENCODE and len(null_rows) > 0
    all_first = np.concatenate([first_rows, null_rows[:1]]) if encode_null else first_rows
    order = np.argsort(all_first, kind="stable")
    rank = np.empty(len(all_first), np.int64)
    rank[order] = np.arange(len(all_first))
    idx = np.zeros(len(vals), np.int32)
    idx[rows] = rank[:len(keys)][inverse.reshape(-1)]
    dict_bits = np.zeros(len(all_first), bits.dtype)
    dict_bits[rank[:len(keys)]] = keys
    dict_valid = None
    if encode_null:
        idx[null_rows] = rank[-1]
        dict_valid = np.ones(len(all_first), bool)
        dict_valid[rank[-1]] = False
    out, pos = [], 0
    for n, (_, m) in zip(lens, chunks):
        ci, cv = idx[pos:pos + n], valid[pos:pos + n]
        if null_encoding == MASK and m is not None and not cv.all():
            out.append((ci, cv, int((~cv).sum())))
        else:
            out.append((ci, None, 0))
        pos += n
    return out, dict_bits.view(dtype), dict_valid
