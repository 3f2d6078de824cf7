"""Python restatement of raw Snappy decoding as the device decompressor (csrc/snappy.cu) does it: golang/snappy's decode
checks, plus the page outcomes of include/arrowgpu.h.  And an encoder that can emit every element form: inline and
1-4-byte literal lengths, copy-1/2/4, overlapping copies; the streams of every form and the corrupt rows the tests
share.  Not product code."""
import numpy as np

OK, CORRUPT, SIZE = 0, 1, 2
MESSAGE = {CORRUPT: "parquet: could not decompress page: snappy: corrupt input",
           SIZE: "parquet: metadata said {} bytes uncompressed data page, got {} bytes"}


def uvarint(buf):
    """binary.Uvarint: (value, n); n == 0 buffer too short, n < 0 overflow"""
    x = 0
    for i, b in enumerate(buf[:10]):
        if b < 0x80:
            if i == 9 and b > 1:
                return 0, -(i + 1)
            return x | b << (7 * i), i + 1
        x |= (b & 0x7F) << (7 * i)
    return (0, -11) if len(buf) >= 10 else (0, 0)


def put_uvarint(v):
    out = bytearray()
    while v >= 0x80:
        out.append(v & 0x7F | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def decode(buf, dst_len=None):
    """-> (output, err, preamble).  CORRUPT: output holds the bytes of the elements before the failing one.  With
    dst_len: an empty stream and dst_len 0 is OK, and a preamble != dst_len is SIZE with no output."""
    buf = bytes(buf)
    if dst_len == 0 and not buf:
        return b"", OK, 0
    v, n = uvarint(buf)
    if n <= 0 or v > 0xFFFFFFFF:
        return b"", CORRUPT, 0
    if dst_len is not None and v != dst_len:
        return b"", SIZE, v
    out, s = bytearray(), n
    while s < len(buf):
        tag = buf[s]
        if tag & 3 == 0:
            x = tag >> 2
            if x < 60:
                s += 1
            else:
                nb = x - 59
                s += 1 + nb
                if s > len(buf):
                    return bytes(out), CORRUPT, v
                x = int.from_bytes(buf[s - nb:s], "little")
            length = x + 1
            if length > v - len(out) or length > len(buf) - s:
                return bytes(out), CORRUPT, v
            out += buf[s:s + length]
            s += length
            continue
        hdr = (0, 2, 3, 5)[tag & 3]
        s += hdr
        if s > len(buf):
            return bytes(out), CORRUPT, v
        if tag & 3 == 1:
            length, off = 4 + ((tag >> 2) & 7), (tag >> 5) << 8 | buf[s - 1]
        else:
            length, off = 1 + (tag >> 2), int.from_bytes(buf[s - hdr + 1:s], "little")
        if off <= 0 or len(out) < off or length > v - len(out):
            return bytes(out), CORRUPT, v
        if off >= length:
            out += out[len(out) - off:len(out) - off + length]
        else:
            for _ in range(length):
                out.append(out[-off])
    if len(out) != v:
        return bytes(out), CORRUPT, v
    return bytes(out), OK, v


# ---- encoder: elements ----
def literal(data, nbytes=None):
    """one literal element; nbytes = 0 for the inline length (<= 60 bytes), 1..4 for that many length bytes"""
    n = len(data) - 1
    if nbytes is None:
        nbytes = 0 if n < 60 else (n.bit_length() + 7) // 8
    if nbytes == 0:
        assert 0 <= n < 60
        return bytes([n << 2]) + bytes(data)
    assert n < 1 << (8 * nbytes)
    return bytes([(59 + nbytes) << 2]) + n.to_bytes(nbytes, "little") + bytes(data)


def copy(off, length, form=None):
    """one copy element; form 1 (length 4..11, offset < 2048), 2 (length 1..64, offset < 65536) or 4"""
    if form is None:
        form = 1 if 4 <= length <= 11 and off < 2048 else 2 if off < 65536 else 4
    if form == 1:
        assert 4 <= length <= 11 and off < 2048
        return bytes([(off >> 8) << 5 | (length - 4) << 2 | 1, off & 0xFF])
    assert 1 <= length <= 64
    if form == 2:
        return bytes([(length - 1) << 2 | 2]) + off.to_bytes(2, "little")
    return bytes([(length - 1) << 2 | 3]) + off.to_bytes(4, "little")


def stream(n, elements):
    return put_uvarint(n) + b"".join(elements)


def encode(data, copy_form=None, lit_bytes=None, max_copy=64):
    """greedy 4-byte-hash encoder; copy_form / lit_bytes force one form where it fits (copy-1 falls back to copy-2)"""
    data = bytes(data)
    els, last, i, lit0 = [], {}, 0, 0

    def flush(end):
        k = lit0
        while k < end:
            chunk = data[k:min(end, k + 65536)]
            fits = lit_bytes is not None and (len(chunk) <= 60 if lit_bytes == 0 else len(chunk) - 1 < 1 << (8 * lit_bytes))
            els.append(literal(chunk, lit_bytes if fits else None))
            k += len(chunk)

    while i + 4 <= len(data):
        key = data[i:i + 4]
        c = last.get(key)
        last[key] = i
        if c is None or i - c > 0xFFFFFFFF:
            i += 1
            continue
        m = 4
        while i + m < len(data) and data[c + m] == data[i + m]:
            m += 1
        flush(i)
        off = i - c
        while m > 0:
            ln = min(m, max_copy)
            if m - ln in (1, 2, 3) and ln > 4:                 # keep every copy at least 4 long
                ln -= 4
            f = copy_form
            if f == 1 and not (4 <= ln <= 11 and off < 2048):
                f = None
            if f == 2 and off >= 65536:
                f = 4
            els.append(copy(off, ln, f))
            i += ln
            m -= ln
        lit0 = i
    flush(len(data))
    return stream(len(data), els)


def forms():
    """(name, stream, expected output) covering every element form"""
    rng = np.random.default_rng(52)
    big = rng.integers(0, 256, 70_000, dtype=np.uint8).tobytes()
    far = big + big[:100]                                       # a copy 70 000 bytes back: copy-4
    out = [
        ("inline_literals", encode(b"abcdefgh" * 3 + bytes(range(40)), lit_bytes=0)),
        ("literal_1_byte_length", stream(200, [literal(big[:200], 1)])),
        ("literal_2_byte_length", stream(300, [literal(big[:300], 2)])),
        ("literal_3_byte_length", stream(70_000, [literal(big, 3)])),
        ("literal_4_byte_length", stream(61, [literal(big[:61], 4)])),
        ("literal_1_byte_length_short", stream(5, [literal(big[:5], 1)])),
        ("copy_1", stream(20, [literal(b"0123456789"), copy(10, 10, 1)])),
        ("copy_2", stream(74, [literal(b"0123456789"), copy(10, 64, 2)])),
        ("copy_4", stream(74, [literal(b"0123456789"), copy(10, 64, 4)])),
        ("offset_1_run", stream(1 + 64 * 3, [literal(b"z"), copy(1, 64, 2), copy(1, 64, 4), copy(64, 64, 2)])),
        ("overlap_offset_3", stream(3 + 11, [literal(b"abc"), copy(3, 11, 1)])),
        ("copy_of_length_1", stream(2, [literal(b"q"), copy(1, 1, 2)])),
        ("offset_beyond_64k", encode(far)),
        ("greedy_copy_2_only", encode(b"hello hello hello world " * 40, copy_form=2)),
        ("greedy_copy_4_only", encode(b"hello hello hello world " * 40, copy_form=4)),
        ("greedy_literal_4_bytes", encode(big[:5000] + big[:5000], lit_bytes=4)),
        ("empty_stream", stream(0, [])),
    ]
    return [(n, s, decode(s)[0]) for n, s in out]


def corrupt_rows():
    """(name, stream, dst_len, bytes the restatement delivers)"""
    ok = literal(b"0123456789")
    return [
        ("no_preamble", b"", 5, 0),
        ("preamble_cut", b"\x80", 5, 0),
        ("preamble_over_10_bytes", b"\xff" * 10 + b"\x01", 5, 0),
        ("preamble_over_32_bits", put_uvarint(1 << 32), 1 << 32, 0),
        ("literal_length_cut", stream(20, [ok, b"\xf0"]), 20, 10),
        ("literal_4_length_cut", stream(20, [ok, b"\xfc\x01\x00"]), 20, 10),
        ("literal_bytes_cut", stream(20, [ok, literal(b"abcdefghij")[:-1]]), 20, 10),
        ("literal_past_output", stream(15, [ok, literal(b"abcdefghij")]), 15, 10),
        ("copy_1_offset_cut", stream(20, [ok, copy(10, 10, 1)[:1]]), 20, 10),
        ("copy_2_offset_cut", stream(20, [ok, copy(10, 10, 2)[:2]]), 20, 10),
        ("copy_4_offset_cut", stream(20, [ok, copy(10, 10, 4)[:4]]), 20, 10),
        ("copy_offset_0", stream(20, [ok, copy(0, 10, 2)]), 20, 10),
        ("copy_offset_past_output", stream(30, [ok, copy(11, 10, 2)]), 30, 10),
        ("copy_past_output", stream(15, [ok, copy(10, 10, 2)]), 15, 10),
        ("stream_ends_early", stream(30, [ok, copy(10, 10, 1)]), 30, 20),
        ("trailing_element", stream(20, [ok, copy(10, 10, 1), literal(b"x")]), 20, 20),
        ("preamble_only", stream(7, []), 7, 0),
    ]
