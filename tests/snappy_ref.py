"""Python restatement of raw Snappy decoding as the device decompressor (csrc/snappy.cu) does it: golang/snappy's decode
checks, plus the page outcomes of include/arrowgpu.h.  And an encoder that can emit every element form: inline and
1-4-byte literal lengths, copy-1/2/4, overlapping copies.  Not product code."""
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
