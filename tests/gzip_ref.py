"""Test helper: a pure-Python restatement of GZIP page decompression as include/arrowgpu.h documents it (RFC 1952
members, RFC 1951 DEFLATE, the page outcomes as events in stream order), builders for the forms zlib does not emit, and
the corrupt rows.  Not product code.  decode() mirrors the device walk: it reports the first event in stream order
and the bytes written before the first decode event."""
import collections
import struct
import zlib

OK, EOF, SHORT, EXCEED, HEADER, CHECKSUM, CORRUPT = "ok", "unexpected EOF", "short", "exceeds", "header", "checksum", "corrupt"

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_BITS = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_BITS = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CLEN_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32
NAME_MAX = 512                      # FNAME / FCOMMENT: at most NAME_MAX - 1 bytes before the NUL


def _crc_table():
    t = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ 0xEDB88320 if c & 1 else c >> 1
        t.append(c)
    return t


_CRC = _crc_table()


def crc32(data, crc=0):
    """CRC-32 (IEEE, reflected), the gzip trailer's"""
    c = crc ^ 0xFFFFFFFF
    for b in data:
        c = _CRC[(c ^ b) & 255] ^ (c >> 8)
    return c ^ 0xFFFFFFFF


def message(outcome, arg, dst_len):
    pre = "parquet: could not decompress page: "
    if outcome == SHORT:
        return pre + ("EOF" if arg == 0 else "unexpected EOF")
    return pre + {EOF: "unexpected EOF", EXCEED: f"codec: gzip: decoded data exceeds destination size {dst_len}",
                  HEADER: "gzip: invalid header", CHECKSUM: "gzip: invalid checksum"}.get(outcome, f"gzip: {arg}")


class _Event(Exception):
    def __init__(self, kind, arg=None):
        super().__init__(kind, arg)
        self.kind, self.arg = kind, arg


class _Bits:
    """LSB-first bits of buf; bits past the end read as zeros (pos > 8 * len is a truncation)"""

    def __init__(self, buf, pos):
        self.buf, self.pos, self.end = buf, pos, 8 * len(buf)

    def peek(self, n):
        i = self.pos >> 3
        return (int.from_bytes(self.buf[i:i + 4], "little") >> (self.pos & 7)) & ((1 << n) - 1)

    def take(self, n):
        v = self.peek(n)
        self.pos += n
        return v

    def check(self):
        if self.pos > self.end:
            raise _Event(EOF)


def _rev(code, n):
    return int(f"{code:0{n}b}"[::-1], 2) if n else 0


def _build(lens, may_be_empty=False):
    """a complete code (or one symbol of length 1, or none when may_be_empty) -> (table, max length); table[peek] =
    (symbol, length) or None"""
    cnt = [0] * 16
    for n in lens:
        cnt[n] += 1
    cnt[0] = 0
    left = 1
    for n in range(1, 16):
        left = 2 * left - cnt[n]
        if left < 0:
            raise _Event(CORRUPT, "huffman")
    total = sum(cnt)
    if left > 0 and not ((total == 1 and cnt[1] == 1) or (total == 0 and may_be_empty)):
        raise _Event(CORRUPT, "huffman")
    mx = max([n for n in lens if n], default=1)
    code, nxt = 0, [0] * 16
    for n in range(1, 16):
        code = (code + cnt[n - 1]) << 1
        nxt[n] = code
    table = [None] * (1 << mx)
    for s, n in enumerate(lens):
        if n:
            r = _rev(nxt[n], n)
            nxt[n] += 1
            for k in range(r, 1 << mx, 1 << n):
                table[k] = (s, n)
    return table, mx


def _sym(br, code):
    e = code[0][br.peek(code[1])]
    if e is None:
        return -1
    br.pos += e[1]
    return e[0]


_FIXED = None


def _inflate(br, out, m0, dst_len, seen):
    global _FIXED
    while True:
        hdr = br.take(3)
        br.check()
        final, btype = hdr & 1, hdr >> 1
        if btype == 0:
            br.pos = (br.pos + 7) & ~7
            n, nn = br.take(16), br.take(16)
            br.check()
            if n != (~nn & 0xFFFF):
                raise _Event(CORRUPT, "stored length")
            if br.pos + 8 * n > br.end:
                raise _Event(EOF)
            seen["stored"] += 1
            seen["stored_len_0" if n == 0 else "stored_len_65535" if n == 65535 else "stored_len"] += 1
            i = br.pos >> 3
            out += br.buf[i:i + n]
            br.pos += 8 * n
            if len(out) > dst_len:
                raise _Event(EXCEED)
        elif btype == 3:
            raise _Event(CORRUPT, "block type")
        else:
            if btype == 1:
                seen["fixed"] += 1
                if _FIXED is None:
                    _FIXED = (_build(FIXED_LIT), _build(FIXED_DIST))
                lit, dist = _FIXED
            else:
                seen["dynamic"] += 1
                lit, dist = _dynamic_header(br, seen)
            _block(br, out, m0, dst_len, lit, dist, seen)
        if final:
            return


def _dynamic_header(br, seen):
    h = br.take(14)
    br.check()
    nlit, ndist, nclen = 257 + (h & 31), 1 + ((h >> 5) & 31), 4 + (h >> 10)
    if nlit > 286 or ndist > 30:
        raise _Event(CORRUPT, "code lengths")
    cl = [0] * 19
    for i in range(19):
        cl[CLEN_ORDER[i]] = br.take(3) if i < nclen else 0
    br.check()
    clen = _build(cl)
    lens, n = [], nlit + ndist
    while len(lens) < n:
        s = _sym(br, clen)
        br.check()
        if s < 0:
            raise _Event(CORRUPT, "code lengths")
        if s < 16:
            lens.append(s)
            continue
        if s == 16:
            if not lens:
                raise _Event(CORRUPT, "code lengths")
            v, rep = lens[-1], 3 + br.take(2)
            lim = (3, 6)
        elif s == 17:
            v, rep, lim = 0, 3 + br.take(3), (3, 10)
        else:
            v, rep, lim = 0, 11 + br.take(7), (11, 138)
        br.check()
        if len(lens) + rep > n:
            raise _Event(CORRUPT, "code lengths")
        seen[f"repeat_{s}"] += 1
        if rep in lim:
            seen[f"repeat_{s}_{rep}"] += 1
        lens += [v] * rep
    if lens[256] == 0:
        raise _Event(CORRUPT, "huffman")
    litc, distc = _build(lens[:nlit]), _build(lens[nlit:], may_be_empty=True)
    used = [x for x in lens[nlit:] if x]
    seen["no_distance_codes" if not used else "single_distance_code" if len(used) == 1 else "distance_codes"] += 1
    if max(lens[:nlit]) > 10:
        seen["code_longer_than_10_bits"] += 1
    if max(lens) == 15:
        seen["code_length_15"] += 1
    return litc, distc


def _block(br, out, m0, dst_len, lit, dist, seen):
    while True:
        s = _sym(br, lit)
        br.check()
        if s < 0:
            raise _Event(CORRUPT, "symbol")
        if s < 256:
            if len(out) >= dst_len:
                raise _Event(EXCEED)
            out.append(s)
            continue
        if s == 256:
            return
        if s >= 286:
            raise _Event(CORRUPT, "symbol")
        length = LEN_BASE[s - 257] + br.take(LEN_BITS[s - 257])
        br.check()
        d = _sym(br, dist)
        br.check()
        if d < 0 or d >= 30:
            raise _Event(CORRUPT, "symbol")
        dist_v = DIST_BASE[d] + br.take(DIST_BITS[d])
        br.check()
        if dist_v > len(out) - m0:
            raise _Event(CORRUPT, "distance")
        for k in ("len_3", "len_258", "dist_1", "dist_32768"):
            if (k[:3] == "len" and length == int(k[4:])) or (k[:4] == "dist" and dist_v == int(k[5:])):
                seen[k] += 1
        if dist_v >= length:
            out += out[len(out) - dist_v:len(out) - dist_v + length]
        else:
            for _ in range(length):
                out.append(out[-dist_v])
        if len(out) > dst_len:
            raise _Event(EXCEED)


def decode(buf, dst_len, forms=None):
    """-> (output written, outcome, arg).  arg: the check name of CORRUPT, the total of SHORT."""
    seen = forms if forms is not None else collections.Counter()
    buf = bytes(buf)
    n = len(buf)
    out = bytearray()
    ck_bad, ev, arg = False, None, None
    try:
        q = nmem = 0
        while q != n:
            if n - q < 10:
                raise _Event(EOF)
            if buf[q] != 0x1F or buf[q + 1] != 0x8B or buf[q + 2] != 8:
                raise _Event(HEADER)
            flg, h0 = buf[q + 3], q
            q += 10
            if flg & 0xE0:
                seen["reserved_flags"] += 1
            if flg & 4:
                if n - q < 2:
                    raise _Event(EOF)
                xlen = buf[q] | buf[q + 1] << 8
                q += 2
                if n - q < xlen:
                    raise _Event(EOF)
                q += xlen
                seen["fextra"] += 1
            for f, name in ((8, "fname"), (16, "fcomment")):
                if flg & f:
                    i = 0
                    while True:
                        if i >= NAME_MAX:
                            raise _Event(HEADER)
                        if q >= n:
                            raise _Event(EOF)
                        q += 1
                        if buf[q - 1] == 0:
                            break
                        i += 1
                    seen[name] += 1
                    if i == NAME_MAX - 1:
                        seen[name + "_511"] += 1
            if flg & 2:
                if n - q < 2:
                    raise _Event(EOF)
                if crc32(buf[h0:q]) & 0xFFFF != buf[q] | buf[q + 1] << 8:
                    raise _Event(HEADER)
                q += 2
                seen["fhcrc"] += 1
            m0 = len(out)
            br = _Bits(buf, 8 * q)
            _inflate(br, out, m0, dst_len, seen)
            q = (br.pos + 7) >> 3
            if n - q < 8:
                raise _Event(EOF)
            crc, isize = struct.unpack_from("<II", buf, q)
            if crc32(out[m0:]) != crc or isize != (len(out) - m0) & 0xFFFFFFFF:
                ck_bad = True
            q += 8
            nmem += 1
            seen["member"] += 1
            if nmem > 1:
                seen["multi_member"] += 1
            if len(out) == m0:
                seen["empty_member"] += 1
    except _Event as e:
        ev, arg = e.kind, e.arg
    written = bytes(out[:dst_len])
    if ck_bad:
        return written, CHECKSUM, None
    if ev:
        return written, ev, arg
    if len(out) < dst_len:
        return written, SHORT, len(out)
    return written, OK, None


# ------------------------------------------------------------------------------------------------------------ builders
class BitWriter:
    def __init__(self):
        self.acc, self.n = 0, 0

    def bits(self, v, n):
        self.acc |= (v & ((1 << n) - 1)) << self.n
        self.n += n
        return self

    def code(self, c, n):                  # Huffman codes go most significant bit first
        return self.bits(_rev(c, n), n)

    def align(self):
        self.n = (self.n + 7) & ~7
        return self

    def bytes(self):
        return self.acc.to_bytes((self.n + 7) // 8, "little")


def canonical(lens):
    """{symbol: code} of a code given by its lengths"""
    cnt = collections.Counter(n for n in lens if n)
    code, nxt = 0, {}
    for n in range(1, 16):
        code = (code + cnt.get(n - 1, 0)) << 1
        nxt[n] = code
    out = {}
    for s, n in enumerate(lens):
        if n:
            out[s] = (nxt[n], n)
            nxt[n] += 1
    return out


def complete_lengths(symbols, n):
    """lengths over n symbols giving `symbols` (sorted) a complete code: 2^b - k of length b - 1, the rest b"""
    k = len(symbols)
    lens = [0] * n
    if k == 1:
        lens[symbols[0]] = 1
        return lens
    b = (k - 1).bit_length()
    for i, s in enumerate(sorted(symbols)):
        lens[s] = b - 1 if i < (1 << b) - k else b
    return lens


def _len_sym(length):
    for i in range(28, -1, -1):
        if length >= LEN_BASE[i] and (i != 27 or length < 258):
            return 257 + i, length - LEN_BASE[i]


def _dist_sym(d):
    for i in range(29, -1, -1):
        if d >= DIST_BASE[i]:
            return i, d - DIST_BASE[i]


def expand(tokens, history=b""):
    """tokens (a literal byte, or (length, distance)) -> the bytes they produce after `history`"""
    out = bytearray(history)
    for t in tokens:
        if isinstance(t, int):
            out.append(t)
        else:
            for _ in range(t[0]):
                out.append(out[-t[1]])
    return bytes(out[len(history):])


def _huff_body(w, tokens, lit, dist):
    for t in tokens:
        if isinstance(t, int):
            w.code(*lit[t])
        else:
            s, e = _len_sym(t[0])
            w.code(*lit[s]).bits(e, LEN_BITS[s - 257])
            d, de = _dist_sym(t[1])
            w.code(*dist[d]).bits(de, DIST_BITS[d])
    w.code(*lit[256])


def stored_block(w, data, final=True):
    w.bits(final, 1).bits(0, 2).align().bits(len(data), 16).bits(~len(data) & 0xFFFF, 16)
    for b in data:
        w.bits(b, 8)
    return w


def fixed_block(w, tokens, final=True):
    w.bits(final, 1).bits(1, 2)
    _huff_body(w, tokens, canonical(FIXED_LIT), canonical(FIXED_DIST))
    return w


def rle_code_lengths(lens):
    """[(symbol, extra)] of the code-length alphabet for lens, greedy"""
    out, i = [], 0
    while i < len(lens):
        v, run = lens[i], 1
        while i + run < len(lens) and lens[i + run] == v:
            run += 1
        i += run
        if v == 0:
            while run >= 11:
                r = min(run, 138)
                out.append((18, r - 11))
                run -= r
            if run >= 3:
                out.append((17, run - 3))
                run = 0
            out += [(0, 0)] * run
        else:
            out.append((v, 0))
            run -= 1
            while run >= 3:
                r = min(run, 6)
                out.append((16, r - 3))
                run -= r
            out += [(v, 0)] * run
    return out


# a complete code-length code over all 19 symbols: 13 of length 4, 6 of length 5
CLEN_LENS = [4] * 13 + [5] * 6


def dynamic_block(w, tokens, lit_lens, dist_lens, final=True, clen_seq=None, clen_lens=CLEN_LENS, hlit=None, hdist=None):
    """a dynamic block with the given code lengths (len(lit_lens) = HLIT + 257, len(dist_lens) = HDIST + 1)"""
    nlit, ndist = len(lit_lens), len(dist_lens)
    w.bits(final, 1).bits(2, 2)
    w.bits((nlit - 257) if hlit is None else hlit, 5).bits((ndist - 1) if hdist is None else hdist, 5).bits(15, 4)
    for i in range(19):
        w.bits(clen_lens[CLEN_ORDER[i]], 3)
    cc = canonical(clen_lens)
    for s, e in (clen_seq if clen_seq is not None else rle_code_lengths(list(lit_lens) + list(dist_lens))):
        w.code(*cc[s])
        if s >= 16:
            w.bits(e, {16: 2, 17: 3, 18: 7}[s])
    if tokens is not None:
        _huff_body(w, tokens, canonical(lit_lens), canonical(dist_lens))
    return w


def member(body, flags=0, extra=None, name=None, comment=None, hcrc=False, payload=b"", crc=None, isize=None):
    """a gzip member around DEFLATE bytes `body` producing `payload`"""
    flg = flags | (4 if extra is not None else 0) | (8 if name is not None else 0) | (16 if comment is not None else 0) | (2 if hcrc else 0)
    h = bytearray(b"\x1f\x8b\x08" + bytes([flg]) + b"\x00\x00\x00\x00\x00\xff")
    if extra is not None:
        h += struct.pack("<H", len(extra)) + extra
    if name is not None:
        h += name + b"\x00"
    if comment is not None:
        h += comment + b"\x00"
    if hcrc:
        h += struct.pack("<H", crc32(h) & 0xFFFF)
    return bytes(h) + body + struct.pack("<II", crc32(payload) if crc is None else crc,
                                         len(payload) & 0xFFFFFFFF if isize is None else isize)


def gz(payload, level=6, strategy=zlib.Z_DEFAULT_STRATEGY):
    c = zlib.compressobj(level, zlib.DEFLATED, 31, 9, strategy)
    return c.compress(payload) + c.flush()


def payload(n, seed=1):
    """text-like bytes with repeats near and far, a long run and a stretch of noise"""
    import random
    r = random.Random(seed)
    words = [bytes(r.choice(b"abcdefghijklmnopqrstuvwxyz") for _ in range(r.randint(2, 9))) for _ in range(300)]
    out = bytearray()
    while len(out) < n:
        k = r.random()
        if k < 0.7:
            out += r.choice(words) + b" "
        elif k < 0.75:
            out += bytes([r.randrange(256)]) * r.randint(1, 400)
        elif k < 0.85:
            out += bytes(r.randrange(256) for _ in range(r.randint(1, 64)))
        elif len(out) > 300:
            a = r.randrange(len(out) - 258)
            out += out[a:a + r.randint(3, 258)]
    return bytes(out[:n])


def _lens_tokens():
    """the dynamic block whose code lengths hit every repeat-code limit: (lit_lens, dist_lens, tokens)"""
    used = [0, 139, 151, 155] + list(range(166, 174)) + [256, 257, 284, 285]
    lit = complete_lengths(used, 286)
    dist = [2, 2, 2, 2]
    toks = [0, 139, 151, 155] + list(range(166, 174)) + [(3, 1), (258, 2), (227, 4), (3, 3), 0]
    return lit, dist, toks


def forms():
    """[(name, stream, payload)] of hand-built forms zlib does not emit"""
    rows = []
    x = payload(3000, 7)
    raw = (lambda c: c.compress(x) + c.flush())(zlib.compressobj(6, zlib.DEFLATED, -15))
    rows.append(("header_fields", member(raw, extra=b"\x01\x02ab", name=b"page.bin", comment=b"a comment", hcrc=True, payload=x), x))
    rows.append(("name_511", member(raw, name=b"n" * 511, comment=b"c" * 511, payload=x), x))
    rows.append(("empty_extra", member(raw, extra=b"", payload=x), x))
    rows.append(("reserved_flags", member(raw, flags=0xE0, payload=x), x))
    empty = member(stored_block(BitWriter(), b"").bytes())
    rows.append(("empty_member", empty, b""))
    rows.append(("concatenated", gz(x[:1000]) + empty + gz(x[1000:], 9) + gz(b""), x))
    # stored blocks of LEN 0 and 65535, then a fixed block reaching back 32768 bytes with a length of 258
    big = payload(65535, 8)
    w = stored_block(BitWriter(), b"", final=False)
    stored_block(w, big, final=False)
    toks = [(258, 32768), (3, 1), 65, (258, 1)]
    fixed_block(w, toks)
    y = big + expand(toks, big)
    rows.append(("stored_and_far_copy", member(w.bytes(), payload=y), y))
    # fixed block with literal/length symbols 280..287 region (7-bit and 8-bit codes) and a short distance
    toks = [72, 105, (3, 2), 255, (10, 1), (257, 5)]
    y = expand(toks)
    rows.append(("fixed_block", member(fixed_block(BitWriter(), toks).bytes(), payload=y), y))
    # dynamic block: every repeat code at its limits
    lit, dist, toks = _lens_tokens()
    y = expand(toks)
    rows.append(("repeat_limits", member(dynamic_block(BitWriter(), toks, lit, dist).bytes(), payload=y), y))
    # dynamic block: literal/length code lengths 1..15 (codes longer than the device's primary table)
    used = [97 + i for i in range(15)] + [256]
    lit = [0] * 257
    for i, s in enumerate(used[:15]):
        lit[s] = i + 1
    lit[256] = 15
    toks = [97 + (i * 7) % 15 for i in range(200)] + [111, 110, 109]
    y = expand(toks)
    rows.append(("long_codes", member(dynamic_block(BitWriter(), toks, lit, [0]).bytes(), payload=y), y))
    # dynamic block: one distance code of length 1; and no distance code at all
    lit = complete_lengths([65, 66, 256, 257, 258], 259)
    toks = [65, 66, (3, 1), (4, 1), 66]
    y = expand(toks)
    rows.append(("single_distance_code", member(dynamic_block(BitWriter(), toks, lit, [1]).bytes(), payload=y), y))
    lit = complete_lengths([65, 66, 67, 256], 257)
    toks = [65, 66, 67, 67, 66]
    y = expand(toks)
    rows.append(("no_distance_codes", member(dynamic_block(BitWriter(), toks, lit, [0, 0]).bytes(), payload=y), y))
    return rows


def corrupt_rows():
    """[(name, stream, dst_len, (outcome, arg))]: one row per check, a truncation inside each part of a member"""
    x = payload(5000, 9)
    good = gz(x)
    raw = good[10:-8]
    hdr = member(raw, extra=b"xy", name=b"nm", comment=b"cm", hcrc=True, payload=x)
    n = len(x)
    # hdr: 10 fixed bytes, FEXTRA [10, 14), FNAME [14, 17), FCOMMENT [17, 20), FHCRC [20, 22)
    rows = [
        ("truncated_fixed_header", good[:6], n, (EOF, None)),
        ("truncated_fextra", hdr[:13], n, (EOF, None)),
        ("truncated_fname", hdr[:15], n, (EOF, None)),
        ("truncated_fcomment", hdr[:18], n, (EOF, None)),
        ("truncated_fhcrc", hdr[:21], n, (EOF, None)),
        ("truncated_deflate", good[:len(good) // 2], n, (EOF, None)),
        ("truncated_trailer", good[:-3], n, (EOF, None)),
        ("trailing_5_bytes", good + b"\x1f\x8b\x08\x00\x00", n, (EOF, None)),
        ("bad_magic", b"\x1f\x8c" + good[2:], n, (HEADER, None)),
        ("bad_cm", good[:2] + b"\x07" + good[3:], n, (HEADER, None)),
        ("fhcrc_mismatch", hdr[:20] + bytes([hdr[20] ^ 1]) + hdr[21:], n, (HEADER, None)),
        ("name_512", member(raw, name=b"n" * 512, payload=x), n, (HEADER, None)),
        ("zero_padding", good + bytes(16), n, (HEADER, None)),
        ("zlib_wrapper", zlib.compress(x), n, (HEADER, None)),
        ("raw_deflate", raw + bytes(10), n, (HEADER, None)),
        ("bad_crc", good[:-8] + struct.pack("<I", zlib.crc32(x) ^ 1) + good[-4:], n, (CHECKSUM, None)),
        ("bad_isize", good[:-4] + struct.pack("<I", n + 1), n, (CHECKSUM, None)),
        ("bad_crc_then_corrupt", gz(x[:100])[:-8] + b"\0\0\0\0" + gz(x[:100])[-4:] + b"\x1f\x8b\x08\x00" + bytes(8),
         n, (CHECKSUM, None)),
        ("block_type_3", member(BitWriter().bits(1, 1).bits(3, 2).bytes() + bytes(4)), 1, (CORRUPT, "block type")),
        ("stored_nlen", member(BitWriter().bits(1, 1).bits(0, 2).align().bits(3, 16).bits(3, 16).bytes() + b"abc"), 3,
         (CORRUPT, "stored length")),
        ("hlit_over", member(dynamic_block(BitWriter(), None, [1] * 257, [1], hlit=30).bytes() + bytes(40)), 1,
         (CORRUPT, "code lengths")),
        ("hdist_over", member(dynamic_block(BitWriter(), None, [1] * 257, [1], hdist=30).bytes() + bytes(40)), 1,
         (CORRUPT, "code lengths")),
        ("repeat_16_first", member(dynamic_block(BitWriter(), None, [0] * 257, [0], clen_seq=[(16, 0)]).bytes() + bytes(40)),
         1, (CORRUPT, "code lengths")),
        ("repeat_past_end", member(dynamic_block(BitWriter(), None, [0] * 257, [0], clen_seq=[(18, 127), (18, 127), (18, 127)]).bytes()
                                   + bytes(40)), 1, (CORRUPT, "code lengths")),
        ("oversubscribed", member(dynamic_block(BitWriter(), None, [1] * 3 + [0] * 253 + [1], [1]).bytes() + bytes(8)), 1,
         (CORRUPT, "huffman")),
        ("incomplete", member(dynamic_block(BitWriter(), None, [2] * 2 + [0] * 254 + [2], [1]).bytes() + bytes(8)), 1,
         (CORRUPT, "huffman")),
        ("no_end_of_block", member(dynamic_block(BitWriter(), None, [1, 1] + [0] * 255, [1]).bytes() + bytes(8)), 1,
         (CORRUPT, "huffman")),
        ("code_length_code_incomplete", member(dynamic_block(BitWriter(), None, [1] * 257, [1], clen_lens=[2] * 3 + [0] * 16,
                                                             clen_seq=[]).bytes() + bytes(8)), 1, (CORRUPT, "huffman")),
        ("fixed_symbol_286", member(BitWriter().bits(1, 1).bits(1, 2).code(0b11000110, 8).bytes() + bytes(4)), 1,
         (CORRUPT, "symbol")),
        ("fixed_distance_30", member(BitWriter().bits(1, 1).bits(1, 2).code(0b00110000, 8).code(0b0000001, 7)
                                     .code(30, 5).bytes() + bytes(4)), 5, (CORRUPT, "symbol")),
        ("empty_distance_code_used", member(dynamic_block(BitWriter(), None, complete_lengths([65, 256, 257], 258), [0])
                                            .code(0, 1).code(3, 2).bytes() + bytes(8)), 5, (CORRUPT, "symbol")),
        ("distance_too_far", member(fixed_block(BitWriter(), [65, 66, (3, 3)]).bytes(), payload=b"AB"), 5,
         (CORRUPT, "distance")),
        ("distance_across_members", gz(b"abcdef") + member(fixed_block(BitWriter(), [65, (3, 2)]).bytes(), payload=b"A"), 10,
         (CORRUPT, "distance")),
        ("exceeds", good, n - 1, (EXCEED, None)),
        ("exceeds_by_stored", gz(x, 0), n - 7, (EXCEED, None)),
        ("short", good, n + 1, (SHORT, n)),
        ("short_empty_member", gz(b""), 4, (SHORT, 0)),
        ("empty_page_with_output", b"", 3, (SHORT, 0)),
    ]
    return rows
