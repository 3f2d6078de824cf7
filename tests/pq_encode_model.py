"""The parallel formulation of RleEncoder (parquet/internal/utils/rle.go:314-445) that csrc/pq_encode.cu implements:
the specification of the device RLE/bit-packed encoder, pinned to pq_ref.rle_encode in test_parquet_encode_oracle.py.

The sequential encoder buffers values in groups of 8 from an origin (the page start, or the end of the last repeated
run) and resets its repeat count at every literal group it flushes.  So:
  - a repeated run is emitted exactly at the first group, on the origin's 8-alignment, whose 8 values are all equal;
    it covers that group up to the end of its equal-value run, and that end is the next origin;
  - only equal runs [a, b) of 8 or more values can be caught: with the incoming alignment residue r, the run is caught
    iff c = a + ((r - a) mod 8) satisfies c + 8 <= b, and then the residue becomes b mod 8, else it stays r.  Each
    long run is a map Z8 -> Z8 and the chain of residues is an associative scan of those maps;
  - the groups between an origin and the next caught group (or the page end) form literal runs, cut every 63 groups
    (a 1-byte header (g << 1) | 1, then g * bit_width bytes);
  - the tail after the last full group of the last stretch: with no literal pending (0 mod 63 groups in the stretch)
    and all its (< 8) values equal it is a repeated run of its length; otherwise it is padded with zeros to one last
    literal group.
"""
import numpy as np

from pq_ref import pack_group, varint

IDENTITY = tuple(range(8))


def run_map(a, b):
    """the Z8 -> Z8 map of the equal run [a, b): caught -> b mod 8, else unchanged"""
    return tuple(b % 8 if a + ((r - a) % 8) + 8 <= b else r for r in range(8))


def compose(f, g):
    """f then g"""
    return tuple(g[f[r]] for r in range(8))


def equal_runs(values):
    """(starts, ends) of the maximal runs of equal values"""
    v = np.asarray(values)
    n = v.size
    if n == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    heads = np.flatnonzero(np.concatenate([[True], v[1:] != v[:-1]]))
    return heads.astype(np.int64), np.append(heads[1:], n).astype(np.int64)


def caught_runs(values):
    """[(c, b)]: the repeated runs the encoder emits before the tail, as [first caught position, run end).  The residue
    entering every long run is an exclusive scan of the long runs' maps, applied to residue 0."""
    a, b = equal_runs(values)
    long_ = (b - a) >= 8
    la, lb = a[long_], b[long_]
    maps = [run_map(int(x), int(y)) for x, y in zip(la, lb)]
    prefix, acc = [], IDENTITY                                    # exclusive scan (any associative bracketing works)
    for m in maps:
        prefix.append(acc)
        acc = compose(acc, m)
    out = []
    for x, y, p in zip(la, lb, prefix):
        r = p[0]
        c = int(x) + ((r - int(x)) % 8)
        if c + 8 <= int(y):
            out.append((c, int(y)))
    return out


def literal_stretch(values, origin, groups, bw):
    """groups [origin, origin + 8 * groups) as literal runs of at most 63 groups"""
    out = bytearray()
    for g0 in range(0, groups, 63):
        g = min(63, groups - g0)
        out.append((g << 1) | 1)
        for k in range(g0, g0 + g):
            out += pack_group(values[origin + 8 * k: origin + 8 * k + 8], bw)
    return out


def rle_encode(values, bw):
    """the hybrid stream of `values` at bit width bw, built from the caught runs"""
    v = [int(x) for x in values]
    n = len(v)
    out = bytearray()
    origin = 0
    for c, b in caught_runs(v):
        out += literal_stretch(v, origin, (c - origin) // 8, bw)
        out += varint((b - c) << 1) + v[c].to_bytes((bw + 7) // 8, "little")
        origin = b
    full = (n - origin) // 8
    tail = v[origin + 8 * full:]
    if tail and full % 63 == 0 and len(set(tail)) == 1:
        out += literal_stretch(v, origin, full, bw)
        out += varint(len(tail) << 1) + tail[0].to_bytes((bw + 7) // 8, "little")
    else:
        padded = v[:origin + 8 * full] + tail + [0] * (-len(tail) % 8)
        out += literal_stretch(padded, origin, full + (1 if tail else 0), bw)
    return bytes(out)
