"""Test helper: a pure-Python restatement of LZ4_RAW page decompression as include/arrowgpu.h documents it (an LZ4
block as pierrec/lz4 v4's block decoder accepts it, plus the page outcomes), builders for every sequence form, including
ones liblz4's encoder never emits, and the corrupt rows.  Not product code.  decode() mirrors the device parse: a
sequence's literal run and its match are separate elements, and a corrupt stream delivers the bytes of the elements
before the failing one."""
import collections

import numpy as np

OK, CORRUPT, SIZE = "ok", "corrupt", "size"
PREFIX = "parquet: could not decompress page: "


def message(outcome, arg, dst_len):
    if outcome == SIZE:
        return f"parquet: metadata said {dst_len} bytes uncompressed data page, got {arg} bytes"
    return PREFIX + "lz4: invalid source or destination buffer too short"


def _length(buf, s, n, seen, kind):
    """a length field whose nibble is n: (length, next offset, complete); extension bytes are added up to the first
    byte that is not 255"""
    if n != 15:
        return n, s, True
    k = 0
    while True:
        if s >= len(buf):
            return n, s, False
        b = buf[s]
        s += 1
        k += 1
        n += b
        if b != 255:
            break
    if seen is not None:
        seen[f"{kind}_extension"] += 1
        if k >= 3:
            seen[f"{kind}_multi_255"] += 1
    return n, s, True


def decode(buf, dst_len, seen=None):
    """-> (output, outcome, arg): OK; CORRUPT with the bytes of the elements before the failing one; SIZE (a clean
    stream of arg bytes, arg != dst_len) with no output.  seen (a Counter) counts the forms met."""
    buf = bytes(buf)
    if not buf:
        return (b"", OK, None) if dst_len == 0 else (b"", CORRUPT, None)
    if seen is not None and buf == b"\x00":
        seen["lone_zero_token"] += 1
    out, s, n = bytearray(), 0, len(buf)
    while True:
        tok = buf[s]
        s += 1
        ll, s, ok = _length(buf, s, tok >> 4, seen, "literal")
        if not ok or ll > n - s or ll > dst_len - len(out):
            return bytes(out), CORRUPT, None
        if seen is not None:
            seen[f"literal_{ll}"] += 1
        out += buf[s:s + ll]
        s += ll
        if s == n:
            if tok & 15:
                return bytes(out), CORRUPT, None
            if seen is not None:
                seen["ends_in_literals"] += 1
            break
        if n - s < 2:
            return bytes(out), CORRUPT, None
        off = buf[s] | buf[s + 1] << 8
        s += 2
        ml, s, ok = _length(buf, s, tok & 15, seen, "match")
        ml += 4
        if not ok or off == 0 or off > len(out) or ml > dst_len - len(out):
            return bytes(out), CORRUPT, None
        if seen is not None:
            seen[f"nibble_{tok & 15}"] += 1
            seen[f"offset_{off}"] += 1
            if off < ml:
                seen["overlap"] += 1
        if off >= ml:
            out += out[len(out) - off:len(out) - off + ml]
        else:
            out += (bytes(out[-off:]) * (ml // off + 1))[:ml]
        if s == n:
            if seen is not None:
                seen["ends_in_match"] += 1
            break
    if len(out) != dst_len:
        return b"", SIZE, len(out)
    return bytes(out), OK, None


# ---- builders ----
def ext(n):
    """the extension bytes of a length field whose nibble is 15, for n = length - 15 (or match length - 19)"""
    return b"\xff" * (n // 255) + bytes([n % 255])


def seq(lit=b"", off=None, ml=None, nibble=0):
    """one sequence: the literals, then a match of ml bytes at offset off; off None: a literal-only sequence with the
    given match nibble (0 for a clean end)"""
    ln = len(lit)
    head = ext(ln - 15) if ln >= 15 else b""
    if off is None:
        return bytes([min(ln, 15) << 4 | nibble]) + head + bytes(lit)
    m = ml - 4
    tail = off.to_bytes(2, "little") + (ext(m - 15) if m >= 15 else b"")
    return bytes([min(ln, 15) << 4 | min(m, 15)]) + head + bytes(lit) + tail


TAIL = bytes(range(100, 116))          # a final literal run of 16 bytes: liblz4's end-of-block rules hold after it


def block(*seqs, tail=True):
    return b"".join(seqs) + (seq(TAIL) if tail else b"")


def noise(n, seed=1):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def forms():
    """[(name, stream, payload)] of every form; each ends in a 16-byte literal run, so liblz4 accepts it too"""
    r = noise(70_000, 61)
    rows = [(f"literal_{n}", block(seq(r[:n], 1, 4))) for n in (1, 14, 15, 15 + 254, 15 + 255, 15 + 255 * 3 + 7)]
    rows.append(("literal_0", block(seq(r[:10], 10, 4), seq(b"", 4, 9), seq(b"", 14, 20))))
    rows.append(("match_nibbles", block(seq(r[:40], 40, 4), *[seq(r[k:k + 1], 7, k + 4) for k in range(16)])))
    rows.append(("match_extensions", block(seq(r[:30], 30, 19 + 254), seq(r[:2], 30, 19 + 255), seq(b"", 9, 19 + 255 * 4 + 3))))
    rows += [(f"offset_{o}", block(seq(r[:o], o, 37))) for o in (1, 2, 7, 8)]
    rows.append(("offset_65535", block(seq(r[:65535], 65535, 100), seq(r[:3], 65535, 4))))
    rows.append(("overlap", block(seq(b"abc", 3, 50), seq(b"xy", 5, 19))))
    rows.append(("lone_zero_token", b"\x00"))
    return [(name, s, _payload(s)) for name, s in rows]


def _payload(s):
    out, outcome, arg = decode(s, 1 << 30)
    assert outcome == SIZE, outcome                              # clean: the restatement's length is the payload's
    return decode(s, arg)[0]


def differences():
    """[(name, stream, dst_len, (outcome, arg) here, liblz4 accepts)]: where this library (as pierrec) and liblz4 part"""
    r = noise(64, 62)
    return [
        ("ends_in_match", block(seq(r[:8], 8, 20), tail=False), 28, (OK, None), False),
        ("match_in_last_12_bytes", block(seq(r[:20], 20, 4), seq(r[:6]), tail=False), 30, (OK, None), False),
        ("final_literals_with_match_nibble", block(seq(r[:20], 20, 4), seq(r[:16], nibble=7), tail=False), 40, (CORRUPT, None), True),
        ("offset_0", block(seq(r[:20], 20, 4), seq(r[:3], 0, 4)), 47, (CORRUPT, None), True),
        ("empty_block", b"", 0, (OK, None), False),
    ]


def corrupt_rows():
    """[(name, stream, dst_len, (outcome, arg), bytes written)]: one row per rule"""
    ok = seq(b"0123456789", 10, 4)                               # 14 bytes out
    r = noise(40, 63)
    rows = [
        ("empty_source", b"", 5, 0),
        ("literal_extension_cut", ok + b"\xf0\xff\xff", 40, 14),
        ("literal_extension_missing", ok + b"\xf0", 40, 14),
        ("literals_cut", ok + b"\x50abc", 40, 14),
        ("offset_cut", ok + b"\x14x\x01", 40, 15),
        ("offset_missing_with_nibble", ok + b"\x13x", 40, 15),
        ("match_extension_cut", ok + b"\x1fx\x01\x00\xff", 40, 15),
        ("match_extension_missing", ok + b"\x1fx\x01\x00", 40, 15),
        ("offset_0", ok + seq(b"x", 0, 4) + seq(TAIL), 40, 15),
        ("offset_beyond_output", ok + seq(b"x", 16, 4) + seq(TAIL), 40, 15),
        ("offset_beyond_output_first", seq(b"", 1, 4) + seq(TAIL), 20, 0),
        ("literal_past_dst", ok + seq(r[:10]), 20, 14),
        ("match_past_dst", ok + seq(b"ab", 4, 10) + seq(TAIL), 20, 16),
        ("final_nonzero_nibble", ok + seq(r[:16], nibble=7), 30, 30),
        ("trailing_byte", block(ok) + b"\x00", 31, 30),
    ]
    out = [(name, s, n, (CORRUPT, None), w) for name, s, n, w in rows]
    good = block(ok)
    out += [("size_short", good, 31, (SIZE, 30), 0), ("size_lone_token", b"\x00", 3, (SIZE, 0), 0)]
    return out


def timestamps(n, seed=0):
    """n bytes of PLAIN int64 timestamps (increments in [0, 1000))"""
    rng = np.random.default_rng(seed)
    return (np.cumsum(rng.integers(0, 1000, (n + 7) // 8)) + (1 << 40)).astype(np.int64).tobytes()[:n]


def dict_indices(n, seed=0):
    """n bytes of 17-bit dictionary indices, bit-packed as an RLE/bit-packed literal run would hold them"""
    rng = np.random.default_rng(seed)
    bits = (rng.integers(0, 100_000, (8 * n + 16) // 17 + 1)[:, None] >> np.arange(17)) & 1
    return np.packbits(bits.astype(np.uint8).ravel(), bitorder="little").tobytes()[:n]


def runs(n, seed=0):
    """n bytes of runs of 1 to 5000 equal bytes"""
    rng = np.random.default_rng(seed)
    out = bytearray()
    while len(out) < n:
        out += bytes([int(rng.integers(0, 256))]) * int(rng.integers(1, 5000))
    return bytes(out[:n])


def count_forms(streams):
    seen = collections.Counter()
    for s, n in streams:
        decode(s, n, seen)
    return seen
