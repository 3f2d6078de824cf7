"""Python restatement of ZSTD page decompression (RFC 8878) as the device decompressor (csrc/zstd.cu) does it: the checks
and page outcomes of include/arrowgpu.h, XXH64, a counter of the format forms each decode meets, and stream-surgery
helpers that build the forms libzstd does not emit.  Not product code.

A page is checked in the order the device does it, so that both name the same check:
  1. the walk of frame and zstd-block headers (a failure here fails the block the walk stopped at);
  2. per zstd block: literals and sequences section headers, then the Huffman literals, then the sequences bitstream,
     then the execution checks (literal overrun, offsets, block output, content size), in sequence order.
"""
import collections

import numpy as np

OK, CORRUPT, SIZE, CHECKSUM = 0, 1, 2, 3
CHECKS = ("truncated", "bad magic", "frame header", "dictionary", "block type", "block size", "literals", "huffman",
          "fse", "sequences", "offset", "content size", "page size")
MESSAGE = {CORRUPT: "parquet: could not decompress page: zstd: {}",
           SIZE: "parquet: metadata said {} bytes uncompressed data page, got {} bytes",
           CHECKSUM: "parquet: could not decompress page: zstd: checksum mismatch"}

MAGIC = 0xFD2FB528
BLOCK_MAX = 1 << 17

LL_BASE = list(range(16)) + [16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536]
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BASE = [c + 3 for c in range(32)] + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195,
                                       16387, 32771, 65539]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
LL_DEFAULT = [4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1]
ML_DEFAULT = [1, 4, 3, 2, 2, 2, 2, 2, 2] + [1] * 37 + [-1] * 7
OF_DEFAULT = [1, 1, 1, 1, 1, 1, 2, 2, 2] + [1] * 15 + [-1] * 5
# per symbol type LL, OF, ML: (max accuracy log, max symbol, predefined distribution, predefined accuracy log)
SEQ_KIND = ((9, 35, LL_DEFAULT, 6), (8, 31, OF_DEFAULT, 5), (9, 52, ML_DEFAULT, 6))
SEQ_NAME = ("ll", "of", "ml")

M64 = (1 << 64) - 1
P1, P2, P3, P4, P5 = 11400714785074694791, 14029467366897019727, 1609587929392839161, 9650029242287828579, 2870177450012600261


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & M64


def _round(acc, v):
    return (_rotl((acc + v * P2) & M64, 31) * P1) & M64


def xxh64(data, seed=0):
    data = bytes(data)
    n, i = len(data), 0
    if n >= 32:
        v = [(seed + P1 + P2) & M64, (seed + P2) & M64, seed & M64, (seed - P1) & M64]
        while i + 32 <= n:
            for k in range(4):
                v[k] = _round(v[k], int.from_bytes(data[i + 8 * k:i + 8 * k + 8], "little"))
            i += 32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & M64
        for k in range(4):
            h = ((h ^ _round(0, v[k])) * P1 + P4) & M64
    else:
        h = (seed + P5) & M64
    h = (h + n) & M64
    while i + 8 <= n:
        h = (_rotl(h ^ _round(0, int.from_bytes(data[i:i + 8], "little")), 27) * P1 + P4) & M64
        i += 8
    if i + 4 <= n:
        h = (_rotl(h ^ (int.from_bytes(data[i:i + 4], "little") * P1) & M64, 23) * P2 + P3) & M64
        i += 4
    while i < n:
        h = (_rotl(h ^ (data[i] * P5) & M64, 11) * P1) & M64
        i += 1
    h ^= h >> 33
    h = (h * P2) & M64
    h ^= h >> 29
    h = (h * P3) & M64
    return h ^ (h >> 32)


class Corrupt(Exception):
    def __init__(self, check):
        assert check in CHECKS, check
        super().__init__(check)
        self.check = check


def le(b, off, n):
    return int.from_bytes(bytes(b[off:off + n]), "little")


# ---------------------------------------------------------------------------------------------------------------- bits
class Backward:
    """RFC 8878 backward bitstream: the highest set bit of the last byte is the padding marker"""

    def __init__(self, buf, check):
        buf = bytes(buf)
        if not buf or buf[-1] == 0:
            raise Corrupt(check)
        self.val = int.from_bytes(buf, "little")
        self.total = 8 * (len(buf) - 1) + buf[-1].bit_length() - 1
        self.pos = self.total
        self.check = check

    def peek(self, n):
        p = self.pos - n
        return ((self.val >> p) if p >= 0 else (self.val << -p)) & ((1 << n) - 1)

    def read(self, n):
        v = self.peek(n)
        self.pos -= n
        return v

    def overflowed(self):
        return self.pos < 0

    def finish(self):
        if self.pos != 0:
            raise Corrupt(self.check)


def read_ncount(buf, max_log, max_sym, check="fse"):
    """FSE table description (RFC 8878 4.1.1) -> (normalized counts, accuracy log, bytes used)"""
    buf = bytes(buf)
    val = int.from_bytes(buf, "little")
    pos = 0

    def peek(n):
        return (val >> pos) & ((1 << n) - 1)

    if not buf:
        raise Corrupt(check)
    al = peek(4) + 5
    pos = 4
    if al > max_log:
        raise Corrupt(check)
    remaining = (1 << al) + 1
    threshold = 1 << al
    nbits = al + 1
    norm, sym, prev0 = [], 0, False
    while remaining > 1:
        if sym > max_sym:
            raise Corrupt(check)
        if prev0:
            n0 = sym
            while peek(2) == 3:
                n0 += 3
                pos += 2
            n0 += peek(2)
            pos += 2
            if n0 > max_sym:
                raise Corrupt(check)
            while sym < n0:
                norm.append(0)
                sym += 1
            if pos > 8 * len(buf):
                raise Corrupt(check)
        mx = 2 * threshold - 1 - remaining
        low = peek(nbits - 1)
        if low < mx:
            count = low
            pos += nbits - 1
        else:
            count = peek(nbits)
            if count >= threshold:
                count -= mx
            pos += nbits
        count -= 1
        remaining -= -count if count < 0 else count
        norm.append(count)
        sym += 1
        prev0 = count == 0
        if remaining < threshold:
            if remaining <= 1:
                break
            nbits = remaining.bit_length()
            threshold = 1 << (nbits - 1)
        if pos > 8 * len(buf):
            raise Corrupt(check)
    if remaining != 1 or pos > 8 * len(buf):
        raise Corrupt(check)
    return norm, al, (pos + 7) // 8


def fse_table(norm, al):
    """decode table [(symbol, nbits, base)] of a normalized distribution"""
    size = 1 << al
    sym = [0] * size
    high = size - 1
    nxt = {}
    for s, c in enumerate(norm):
        if c == -1:
            sym[high] = s
            high -= 1
            nxt[s] = 1
        else:
            nxt[s] = c
    step = (size >> 1) + (size >> 3) + 3
    pos = 0
    for s, c in enumerate(norm):
        for _ in range(max(c, 0)):
            sym[pos] = s
            pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    if pos != 0:
        raise Corrupt("fse")
    out = []
    for u in range(size):
        s = sym[u]
        x = nxt[s]
        nxt[s] += 1
        nb = al - (x.bit_length() - 1)
        out.append((s, nb, (x << nb) - size))
    return out


# ------------------------------------------------------------------------------------------------------------- huffman
def huffman_weights(buf, forms):
    """Huffman tree description -> (weights of every symbol, bytes used)"""
    if not buf:
        raise Corrupt("huffman")
    hb = buf[0]
    if hb < 128:
        forms["huf_fse_weights"] += 1
        if 1 + hb > len(buf):
            raise Corrupt("huffman")
        norm, al, used = read_ncount(buf[1:1 + hb], 6, 255, "huffman")
        tbl = fse_table(norm, al)
        bits = Backward(buf[1 + used:1 + hb], "huffman")
        s1, s2 = bits.read(al), bits.read(al)
        w = []
        while True:
            if len(w) > 253:
                raise Corrupt("huffman")
            w.append(tbl[s1][0])
            s1 = tbl[s1][2] + bits.read(tbl[s1][1])
            if bits.overflowed():
                w.append(tbl[s2][0])
                break
            if len(w) > 253:
                raise Corrupt("huffman")
            w.append(tbl[s2][0])
            s2 = tbl[s2][2] + bits.read(tbl[s2][1])
            if bits.overflowed():
                w.append(tbl[s1][0])
                break
        used = 1 + hb
    else:
        forms["huf_direct_weights"] += 1
        n = hb - 127
        used = 1 + (n + 1) // 2
        if used > len(buf):
            raise Corrupt("huffman")
        w = []
        for i in range(n):
            b = buf[1 + i // 2]
            w.append(b >> 4 if i % 2 == 0 else b & 15)
    if any(x > 11 for x in w):
        raise Corrupt("huffman")
    total = sum(1 << (x - 1) for x in w if x)
    if total == 0:
        raise Corrupt("huffman")
    max_bits = total.bit_length()
    rest = (1 << max_bits) - total
    if max_bits > 11 or rest & (rest - 1):
        raise Corrupt("huffman")
    w.append(rest.bit_length())
    if sum(1 for x in w if x == 1) < 2 or sum(1 for x in w if x == 1) % 2:
        raise Corrupt("huffman")
    if max_bits == 11:
        forms["huf_max_bits_11"] += 1
    return w, max_bits, used


def huffman_table(w, max_bits):
    tbl = [None] * (1 << max_bits)
    i = 0
    for wt in range(1, max_bits + 1):
        for s, x in enumerate(w):
            if x == wt:
                for _ in range(1 << (wt - 1)):
                    tbl[i] = (s, max_bits + 1 - wt)
                    i += 1
    assert i == len(tbl)
    return tbl, max_bits


def huffman_stream(buf, n, table):
    tbl, max_bits = table
    bits = Backward(buf, "huffman")
    out = bytearray()
    for _ in range(n):
        s, nb = tbl[bits.peek(max_bits)]
        out.append(s)
        bits.read(nb)
        if bits.overflowed():
            raise Corrupt("huffman")
    bits.finish()
    return out


# -------------------------------------------------------------------------------------------------------------- frames
def walk(buf, forms):
    """frame and zstd-block headers -> (frames, fail); a frame is {fcs, window, checksum, blocks: [(type, start, size)],
    ck}; fail is (index of the block the walk stopped at, check) or None"""
    buf = bytes(buf)
    frames, pos, nblk = [], 0, 0
    while pos < len(buf):
        if len(buf) - pos < 4:
            return frames, (nblk, "truncated")
        magic = le(buf, pos, 4)
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            if len(buf) - pos < 8 or len(buf) - pos - 8 < le(buf, pos + 4, 4):
                return frames, (nblk, "truncated")
            forms["skippable_frame"] += 1
            pos += 8 + le(buf, pos + 4, 4)
            continue
        if magic != MAGIC:
            return frames, (nblk, "bad magic")
        pos += 4
        if pos >= len(buf):
            return frames, (nblk, "truncated")
        fhd = buf[pos]
        fcs_flag, single, reserved, ck, did_flag = fhd >> 6, fhd >> 5 & 1, fhd >> 3 & 1, fhd >> 2 & 1, fhd & 3
        if reserved:
            return frames, (nblk, "frame header")
        dsz = (0, 1, 2, 4)[did_flag]
        fsz = (single, 2, 4, 8)[fcs_flag]
        if pos + 1 + (1 - single) + dsz + fsz > len(buf):
            return frames, (nblk, "truncated")
        p = pos + 1
        window = None
        if not single:
            wd = buf[p]
            wlog = 10 + (wd >> 3)
            window = (1 << wlog) + ((1 << wlog) >> 3) * (wd & 7)
            p += 1
            forms["window_descriptor"] += 1
        else:
            forms["single_segment"] += 1
        did = le(buf, p, dsz)
        p += dsz
        if did_flag:
            forms["dictionary_id_field"] += 1
        if did:
            return frames, (nblk, "dictionary")
        fcs = None
        if fsz:
            fcs = le(buf, p, fsz) + (256 if fsz == 2 else 0)
            forms[f"content_size_{fsz}_bytes"] += 1
        else:
            forms["no_content_size"] += 1
        p += fsz
        if single:
            window = fcs
        pos = p
        bmax = min(window, BLOCK_MAX)
        fr = {"fcs": fcs, "window": window, "checksum": ck, "blocks": [], "ck": None, "complete": False}
        while True:
            if pos + 3 > len(buf):
                return frames + [fr] if fr["blocks"] else frames, (nblk, "truncated")
            bh = le(buf, pos, 3)
            last, btype, bsize = bh & 1, bh >> 1 & 3, bh >> 3
            if btype == 3:
                return frames + [fr] if fr["blocks"] else frames, (nblk, "block type")
            if bsize > bmax:
                return frames + [fr] if fr["blocks"] else frames, (nblk, "block size")
            stored = 1 if btype == 1 else bsize
            if pos + 3 + stored > len(buf):
                return frames + [fr] if fr["blocks"] else frames, (nblk, "truncated")
            fr["blocks"].append((btype, pos + 3, bsize))
            nblk += 1
            pos += 3 + stored
            if last:
                fr["complete"] = True
                break
        if ck:
            if pos + 4 > len(buf):
                return frames + [fr], (nblk, "truncated")
            fr["ck"] = le(buf, pos, 4)
            pos += 4
        frames.append(fr)
    return frames, None


class FrameState:
    def __init__(self):
        self.rep = [1, 4, 8]
        self.huf = None
        self.seq = [None, None, None]


def literals_header(d):
    """-> (type, size format, regenerated, compressed, header bytes, streams)"""
    if not d:
        raise Corrupt("literals")
    lt, sf = d[0] & 3, d[0] >> 2 & 3
    if lt < 2:
        if sf in (0, 2):
            return lt, sf, d[0] >> 3, 0, 1, 0
        if sf == 1:
            if len(d) < 2:
                raise Corrupt("literals")
            return lt, sf, (d[0] >> 4) + (d[1] << 4), 0, 2, 0
        if len(d) < 3:
            raise Corrupt("literals")
        return lt, sf, (d[0] >> 4) + (d[1] << 4) + (d[2] << 12), 0, 3, 0
    hl = (3, 3, 4, 5)[sf]
    if len(d) < hl:
        raise Corrupt("literals")
    v = le(d, 0, hl)
    bits = (10, 10, 14, 18)[sf]
    regen = (v >> 4) & ((1 << bits) - 1)
    comp = v >> (4 + bits)
    return lt, sf, regen, comp, hl, 1 if sf == 0 else 4


def block_headers(d, fs, seq_room, forms):
    """phase 1 of a compressed block: literals and sequences section headers.  -> dict"""
    lt, sf, regen, comp, hl, ns = literals_header(d)
    if regen > BLOCK_MAX:
        raise Corrupt("literals")
    if lt == 0:
        lend = hl + regen
    elif lt == 1:
        lend = hl + 1
    else:
        lend = hl + comp
        if ns == 4 and regen < 6:
            raise Corrupt("literals")
    if lend > len(d):
        raise Corrupt("literals")
    forms[("lit_raw", "lit_rle", "lit_huffman", "lit_treeless")[lt] + (f"_{ns}_streams" if lt >= 2 else "") + f"_sf{sf}"] += 1
    s = lend
    if s >= len(d):
        raise Corrupt("sequences")
    b0 = d[s]
    if b0 < 128:
        nseq, s = b0, s + 1
        forms["nseq_1_byte" if nseq else "nseq_0"] += 1
    elif b0 < 255:
        if s + 2 > len(d):
            raise Corrupt("sequences")
        nseq, s = ((b0 - 128) << 8) + d[s + 1], s + 2
        forms["nseq_2_bytes"] += 1
    else:
        if s + 3 > len(d):
            raise Corrupt("sequences")
        nseq, s = d[s + 1] + (d[s + 2] << 8) + 0x7F00, s + 3
        forms["nseq_3_bytes"] += 1
    modes = None
    if nseq == 0:
        if s != len(d):
            raise Corrupt("sequences")
    else:
        if s >= len(d):
            raise Corrupt("sequences")
        modes = d[s]
        if modes & 3:
            raise Corrupt("sequences")
        s += 1
        if nseq > seq_room:
            raise Corrupt("sequences")
    return {"lt": lt, "regen": regen, "comp": comp, "hl": hl, "ns": ns, "lend": lend, "nseq": nseq, "modes": modes, "s": s}


def literals(d, h, fs, forms):
    """phase 2: the block's literals"""
    lt, regen, hl = h["lt"], h["regen"], h["hl"]
    if lt == 0:
        return bytes(d[hl:hl + regen])
    if lt == 1:
        return bytes([d[hl]]) * regen
    body = d[hl:h["lend"]]
    if lt == 2:
        w, mb, used = huffman_weights(body, forms)
        fs.huf = huffman_table(w, mb)
        body = body[used:]
    elif fs.huf is None:
        raise Corrupt("huffman")
    if h["ns"] == 1:
        return bytes(huffman_stream(body, regen, fs.huf))
    if len(body) < 6:
        raise Corrupt("huffman")
    sz = [le(body, 0, 2), le(body, 2, 2), le(body, 4, 2)]
    sz.append(len(body) - 6 - sum(sz))
    if sz[3] < 0:
        raise Corrupt("huffman")
    seg = (regen + 3) // 4
    counts = [seg, seg, seg, regen - 3 * seg]
    out, p = bytearray(), 6
    for k in range(4):
        out += huffman_stream(body[p:p + sz[k]], counts[k], fs.huf)
        p += sz[k]
    return bytes(out)


def sequences(d, h, fs, forms):
    """phase 3: [(literal length, match length, offset value)]"""
    nseq = h["nseq"]
    if nseq == 0:
        return []
    s = h["s"]
    tables = []
    for k, sh in enumerate((6, 4, 2)):
        mode = h["modes"] >> sh & 3
        max_log, max_sym, default, dlog = SEQ_KIND[k]
        forms[f"{SEQ_NAME[k]}_" + ("predefined", "rle", "fse", "repeat")[mode]] += 1
        if mode == 0:
            t = fse_table(default, dlog)
        elif mode == 1:
            if s >= len(d):
                raise Corrupt("sequences")
            if d[s] > max_sym:
                raise Corrupt("sequences")
            t = [(d[s], 0, 0)]
            s += 1
        elif mode == 2:
            norm, al, used = read_ncount(d[s:], max_log, max_sym)
            if s + used > len(d):
                raise Corrupt("fse")
            t = fse_table(norm, al)
            s += used
            if al == max_log:
                forms[f"{SEQ_NAME[k]}_accuracy_log_{al}"] += 1
        else:
            if fs.seq[k] is None:
                raise Corrupt("sequences")
            t = fs.seq[k]
        tables.append(t)
    fs.seq = list(tables)
    bits = Backward(d[s:], "sequences")
    logs = [(len(t) - 1).bit_length() for t in tables]
    st = [bits.read(logs[0]), bits.read(logs[1]), bits.read(logs[2])]
    out = []
    for i in range(nseq):
        llc, ofc, mlc = tables[0][st[0]][0], tables[1][st[1]][0], tables[2][st[2]][0]
        ofv = (1 << ofc) + bits.read(ofc)
        ml = ML_BASE[mlc] + bits.read(ML_BITS[mlc])
        ll = LL_BASE[llc] + bits.read(LL_BITS[llc])
        out.append((ll, ml, ofv))
        if i + 1 < nseq:
            for k in (0, 2, 1):
                e = tables[k][st[k]]
                st[k] = e[2] + bits.read(e[1])
        if bits.overflowed():
            raise Corrupt("sequences")
    bits.finish()
    return out


def resolve(ofv, ll, rep, forms):
    """RFC 8878 3.1.2.5: the offset of one sequence, updating the repeat-offset history in place"""
    if ofv > 3:
        off = ofv - 3
        rep[:] = [off, rep[0], rep[1]]
        return off
    idx = ofv - 1 + (ll == 0)
    if ll == 0:
        forms["repeat_offset_ll0_shift"] += 1
    forms[f"repeat_offset_{idx}"] += 1
    if idx == 0:
        return rep[0]
    if idx == 1:
        off = rep[1]
        rep[:] = [rep[1], rep[0], rep[2]]
        return off
    if idx == 2:
        off = rep[2]
        rep[:] = [rep[2], rep[0], rep[1]]
        return off
    off = rep[0] - 1
    rep[:] = [off, rep[0], rep[1]]
    return off


def decode(buf, dst_len=None, forms=None):
    """-> (output, err, arg).  err OK; SIZE (arg = the size the frames give; no output); CORRUPT (arg = check; output =
    the bytes of the zstd blocks before the failing one); CHECKSUM (arg = None; output = every byte decoded)."""
    buf = bytes(buf)
    forms = forms if forms is not None else collections.Counter()
    sized = dst_len is not None                                         # None: decode without a page size
    if not sized:
        dst_len = 1 << 62
    if not buf and dst_len == 0:
        return b"", OK, None
    frames, fail = walk(buf, forms)
    if sized and fail is None and all(f["fcs"] is not None for f in frames):
        total = sum(f["fcs"] for f in frames)
        if total != dst_len:
            return b"", SIZE, total
    out = bytearray()
    nblk, fail_at, check, over, starts, ck_bad = 0, None, None, None, [], []
    seq_room = dst_len // 3
    for fi, fr in enumerate(frames):
        forms["frame"] += 1
        if fr["checksum"]:
            forms["checksum"] += 1
        if fr["fcs"] == 0:
            forms["empty_frame"] += 1
        fs = FrameState()
        f0 = len(out)
        bmax = min(fr["window"], BLOCK_MAX)
        for bi, (btype, start, bsize) in enumerate(fr["blocks"]):
            starts.append(len(out))
            k = nblk
            nblk += 1
            try:
                if btype == 0:
                    forms["block_raw"] += 1
                    out += buf[start:start + bsize]
                elif btype == 1:
                    forms["block_rle"] += 1
                    out += bytes([buf[start]]) * bsize
                else:
                    forms["block_compressed"] += 1
                    d = buf[start:start + bsize]
                    h = block_headers(d, fs, seq_room, forms)
                    seq_room -= h["nseq"]
                    lits = literals(d, h, fs, forms)
                    seqs = sequences(d, h, fs, forms)
                    b0, lp = len(out), 0
                    for ll, ml, ofv in seqs:
                        if lp + ll > len(lits):
                            raise Corrupt("sequences")
                        out += lits[lp:lp + ll]
                        lp += ll
                        off = resolve(ofv, ll, fs.rep, forms)
                        if off == 0 or off > len(out) - f0 or off > fr["window"]:
                            raise Corrupt("offset")
                        if off >= ml:
                            out += out[len(out) - off:len(out) - off + ml]
                        else:
                            out += (out[len(out) - off:] * (ml // off + 1))[:ml]
                    out += lits[lp:]
                    if len(out) - b0 > bmax:
                        raise Corrupt("block size")
                if fr["fcs"] is not None and (len(out) - f0 > fr["fcs"] or
                                              (fr["complete"] and bi + 1 == len(fr["blocks"]) and len(out) - f0 != fr["fcs"])):
                    raise Corrupt("content size")
            except Corrupt as e:
                fail_at, check = k, e.check
                del out[starts[k]:]
                break
            if over is None and len(out) > dst_len:
                over = k
        if fail_at is not None:
            break
        if len(frames[1:]) and fi == 0:
            forms["multi_frame"] += 1
        if fr["checksum"] and fr["ck"] is not None:
            if xxh64(out[f0:]) & 0xFFFFFFFF != fr["ck"]:
                ck_bad.append(len(out))                                  # where the frame's output ends
    if fail_at is None and fail is not None:
        fail_at, check = fail
        starts.append(len(out))
    if fail_at is None:
        if sized and len(out) != dst_len:
            return b"", SIZE, len(out)
        return bytes(out), (CHECKSUM if ck_bad else OK), None
    if over is not None and over < fail_at:
        fail_at, check = over, "page size"
        del out[starts[over]:]
    if any(e <= len(out) for e in ck_bad):                           # a frame whose output is out
        return bytes(out), CHECKSUM, None
    return bytes(out), CORRUPT, check


def message(err, arg, dst_len):
    if err == SIZE:
        return MESSAGE[SIZE].format(dst_len, arg)
    if err == CORRUPT:
        return MESSAGE[CORRUPT].format(arg)
    return MESSAGE[err]


# ------------------------------------------------------------------------------------------------------------- surgery
def frames_of(buf):
    """[(start, end)] of every frame (skippable frames included) of a valid page"""
    out, pos, buf = [], 0, bytes(buf)
    while pos < len(buf):
        frames, fail = walk(buf[pos:], collections.Counter())
        assert frames, fail
        one, _ = walk(buf[pos:], collections.Counter())
        fr = one[0]
        btype, start, bsize = fr["blocks"][-1]
        end = pos + start + (1 if btype == 1 else bsize) + (4 if fr["checksum"] else 0)
        out.append((pos, end))
        pos = end
    return out


def skippable(payload, nibble=0):
    return (0x184D2A50 | nibble).to_bytes(4, "little") + len(payload).to_bytes(4, "little") + bytes(payload)


def frame_header(fcs=None, window_log=None, checksum=False, single=None, dict_id=None, fcs_bytes=None):
    """a frame header.  single defaults to True when fcs is given and window_log is not"""
    if single is None:
        single = fcs is not None and window_log is None
    if fcs_bytes is None:
        fcs_bytes = 0 if fcs is None else (1 if single and fcs < 256 else 2 if 256 <= fcs < 65792 else 4 if fcs < 1 << 32 else 8)
    flag = {0: 0, 1: 0, 2: 1, 4: 2, 8: 3}[fcs_bytes]
    assert fcs_bytes != 1 or single
    dflag = {None: 0, 1: 1, 2: 2, 4: 3}[None if dict_id is None else dict_id[1]]
    fhd = flag << 6 | (1 if single else 0) << 5 | (4 if checksum else 0) | dflag
    out = MAGIC.to_bytes(4, "little") + bytes([fhd])
    if not single:
        out += bytes([(window_log - 10) << 3])
    if dict_id is not None:
        out += dict_id[0].to_bytes(dict_id[1], "little")
    if fcs_bytes:
        out += (fcs - (256 if fcs_bytes == 2 else 0)).to_bytes(fcs_bytes, "little")
    return out


def block(kind, body, last, size=None):
    """zstd block: kind 'raw' (body = bytes), 'rle' (body = one byte, size = count) or 'compressed'"""
    t = {"raw": 0, "rle": 1, "compressed": 2, "reserved": 3}[kind]
    n = len(body) if size is None else size
    return (last | t << 1 | n << 3).to_bytes(3, "little") + bytes(body)


def frame(blocks, fcs=None, checksum_of=None, **kw):
    """a frame from encoded zstd blocks; checksum_of = the frame's output (appends its XXH64)"""
    out = frame_header(fcs=fcs, checksum=checksum_of is not None, **kw) + b"".join(blocks)
    if checksum_of is not None:
        out += (xxh64(checksum_of) & 0xFFFFFFFF).to_bytes(4, "little")
    return out


def reframe(buf, fcs="keep", checksum="keep", window_log=None, fcs_bytes=None):
    """re-emit every zstd frame of a valid page with its content size present / absent and its checksum set / cleared"""
    buf = bytes(buf)
    out = bytearray()
    for s, e in frames_of(buf):
        if le(buf, s, 4) != MAGIC:
            out += buf[s:e]
            continue
        frames, _ = walk(buf[s:e], collections.Counter())
        fr = frames[0]
        body_start = fr["blocks"][0][1] - 3
        body_end = e - s - (4 if fr["checksum"] else 0)
        body = buf[s + body_start:s + body_end]
        data, err, _ = decode(buf[s:e])
        assert err == OK
        size = len(data) if fcs == "keep" and fr["fcs"] is not None or fcs is True else None
        ck = fr["checksum"] if checksum == "keep" else checksum
        wl = window_log
        if wl is None:
            w = fr["window"] or 1
            wl = max(10, (w - 1).bit_length())
        hdr = frame_header(fcs=size, window_log=wl, checksum=bool(ck), single=False, fcs_bytes=fcs_bytes if size is not None else None)
        out += hdr + body
        if ck:
            out += (xxh64(data) & 0xFFFFFFFF).to_bytes(4, "little")
    return bytes(out)


def direct_weights(buf):
    """re-emit the Huffman description of every compressed-literals zstd block that uses FSE-compressed weights (and
    has at most 128 of them) with direct 4-bit weights, fixing up the literal and block headers"""
    buf = bytes(buf)
    out = bytearray()
    changed = 0
    for s, e in frames_of(buf):
        if le(buf, s, 4) != MAGIC:
            out += buf[s:e]
            continue
        frames, _ = walk(buf[s:e], collections.Counter())
        fr = frames[0]
        out += buf[s:s + fr["blocks"][0][1] - 3]
        for k, (bt, start, bsize) in enumerate(fr["blocks"]):
            last = 1 if k + 1 == len(fr["blocks"]) else 0
            raw = buf[s + start - 3:s + start + (1 if bt == 1 else bsize)]
            d = raw[3:]
            if bt == 2:
                lt, sf, regen, comp, hl, ns = literals_header(d)
                if lt == 2 and d[hl] < 128:
                    w, mb, used = huffman_weights(d[hl:], collections.Counter())
                    w = w[:-1]
                    if len(w) <= 128:
                        desc = bytes([127 + len(w)]) + bytes((w[i] << 4) | (w[i + 1] if i + 1 < len(w) else 0)
                                                           for i in range(0, len(w), 2))
                        ncomp = comp - used + len(desc)
                        bits = (10, 10, 14, 18)[sf]
                        if ncomp < 1 << bits:
                            hdr = (lt | sf << 2 | regen << 4 | ncomp << (4 + bits)).to_bytes(hl, "little")
                            d = hdr + desc + d[hl + used:]
                            raw = block("compressed", d, last)
                            changed += 1
            out += raw
        out += buf[s + e - s - (4 if fr["checksum"] else 0):e] if fr["checksum"] else b""
    return bytes(out), changed


def rle_seq_block(lits, nseq, ll_code, of_code, ml_code, of_bits, last, repeat=False):
    """a compressed zstd block with raw literals and RLE modes for all three symbol types (repeat: Repeat modes, the
    previous zstd block's RLE codes): every sequence has the same codes; of_bits(i) gives sequence i's extra offset
    bits (of_code of them).  LL / ML codes must have no extra bits."""
    assert LL_BITS[ll_code] == 0 and ML_BITS[ml_code] == 0
    n = len(lits)
    lh = bytes([n << 3]) if n < 32 else (0 | 1 << 2 | (n & 15) << 4).to_bytes(1, "little") + bytes([n >> 4])
    if nseq < 128:
        sh = bytes([nseq])
    elif nseq < 0x7F00:
        sh = bytes([(nseq >> 8) + 128, nseq & 255])
    else:
        sh = bytes([255]) + (nseq - 0x7F00).to_bytes(2, "little")
    sh += bytes([0xFC]) if repeat else bytes([1 << 6 | 1 << 4 | 1 << 2, ll_code, of_code, ml_code])
    # the bitstream is read backward from its end: sequence 0's offset bits come first; write them first (MSB side)
    acc, nb = 1, 0                                                   # the padding marker
    for i in range(nseq):
        acc = acc << of_code | of_bits(i)
        nb += of_code
    stream = acc.to_bytes((nb + 8) // 8, "little")
    return block("compressed", lh + bytes(lits) + sh + stream, last)


# ---------------------------------------------------------------------------------------------------- test streams
LEVELS = (-5, 1, 3, 9, 19, 22)


def datasets(rng):
    return {
        "timestamps": (np.cumsum(rng.integers(0, 1000, 40_000)) + (1 << 40)).astype(np.int64).tobytes(),
        "dict_indices": (rng.integers(0, 100_000, 60_000) & 0x1FFFF).astype(np.uint32).tobytes(),
        "zeros": bytes(300_000),
        "random": rng.integers(0, 256, 150_000, dtype=np.uint8).tobytes(),
        "text": b" ".join(rng.choice([b"alpha", b"beta", b"gamma", b"delta", b"parquet", b"zstd"], 40_000)),
        "skewed": np.minimum(rng.geometric(0.03, 200_000), 255).astype(np.uint8).tobytes(),
        "one": b"x",
        "empty": b"",
    }


def corpus():
    """[(name, compressed, raw)] written by pyarrow"""
    rng = np.random.default_rng(71)
    import pyarrow as pa
    out = []
    for name, x in datasets(rng).items():
        for lvl in LEVELS:
            out.append((f"{name}-{lvl}", pa.Codec("zstd", compression_level=lvl).compress(x, asbytes=True), x))
    big = (np.cumsum(rng.integers(0, 1000, 1 << 19)) + (1 << 40)).astype(np.int64).tobytes()
    out.append(("timestamps-4MB-3", pa.compress(big, codec="zstd", asbytes=True), big))
    return out


def comp(x, level=3):
    import pyarrow as pa
    return pa.Codec("zstd", compression_level=level).compress(x, asbytes=True)


def surgery():
    """[(name, stream, raw)]: the forms libzstd does not emit"""
    import pyarrow as pa
    rng = np.random.default_rng(72)
    text = b" ".join(rng.choice([b"alpha", b"beta", b"gamma", b"delta"], 3000))
    ts = (np.cumsum(rng.integers(0, 1000, 5000)) + (1 << 40)).astype(np.int64).tobytes()
    letters = rng.integers(97, 123, 20_000, dtype=np.uint8).tobytes()
    assert direct_weights(comp(letters))[1] > 0
    a, b = comp(text), comp(ts, 19)
    rows = [
        ("concatenated", a + b, text + ts),
        ("skippable_frames", skippable(b"meta") + a + skippable(b"", 15) + b + skippable(bytes(100), 7), text + ts),
        ("checksum", reframe(a, checksum=True), text),
        ("no_content_size", reframe(b, fcs=False), ts),
        ("checksum_no_content_size", reframe(a + b, fcs=False, checksum=True), text + ts),
        ("content_size_2_bytes", reframe(comp(text[:5000]), fcs_bytes=2), text[:5000]),
        ("content_size_8_bytes", reframe(a, fcs_bytes=8), text),
        ("dictionary_id_zero", frame([block("raw", b"hello", 1)], fcs=5, dict_id=(0, 2)), b"hello"),
        ("raw_and_rle_blocks", frame([block("raw", b"hello", 0), block("rle", b"x", 1, size=1000)], fcs=1005),
         b"hello" + b"x" * 1000),
        ("empty_raw_block_frames", frame([block("raw", b"", 1)], fcs=0) * 3, b""),
        ("direct_weights", direct_weights(comp(letters))[0], letters),
        ("rle_literals", frame([block("compressed", bytes([20 << 3 | 1, ord("k"), 0]), 1)], fcs=20), b"k" * 20),
        ("repeat_modes", frame([block("raw", b"abcdefgh", 0), rle_seq_block(b"xyz", 3, 1, 0, 2, lambda i: 0, 0),
                                  rle_seq_block(b"uv", 2, 1, 0, 2, lambda i: 0, 1, repeat=True)], fcs=8 + 3 * 6 + 2 * 6),
         None),
        ("rle_modes_3_byte_count", frame([block("raw", b"abcdefgh", 0),
                                            rle_seq_block(b"", 33_000, 0, 0, 0, lambda i: 0, 1)], fcs=8 + 99_000), None),
        ("rep0_minus_1", frame([block("raw", bytes(range(64)), 0), rle_seq_block(b"", 4, 0, 5, 0, lambda i: 3, 0),
                                  rle_seq_block(b"zz", 5, 0, 1, 0, lambda i: 1, 1)], fcs=64 + 12 + 15 + 2), None),
        ("window_descriptor_1KB", frame([block("raw", b"q" * 1024, 0), block("rle", b"r", 1, size=1024)],
                                          window_log=10), b"q" * 1024 + b"r" * 1024),
    ]
    out = []
    for name, s, x in rows:
        if x is None:                                             # hand-built: libzstd decodes it the same way
            x, err, _ = decode(s)
            assert err == OK and pa.decompress(s, decompressed_size=len(x), codec="zstd", asbytes=True) == x, name
        out.append((name, s, x))
    return out


def forms():
    """every stream of the corpus and the surgery rows, for the device tests: [(name, stream, raw)]"""
    return [r for r in corpus() if len(r[2]) < 1 << 20] + surgery()


def corrupt_rows():
    """[(name, stream, dst_len, expected check or CHECKSUM)]: every row but the two
    window rows (test_zstd_oracle.WINDOW_ROWS) pa.decompress rejects too"""
    rng = np.random.default_rng(73)
    text = b" ".join(rng.choice([b"alpha", b"beta", b"gamma", b"delta"], 3000))
    good = comp(text)
    n = len(text)
    ck = reframe(good, checksum=True)
    hdr = frame_header(fcs=None, window_log=17, single=False)
    bad_ck = ck[:-1] + bytes([ck[-1] ^ 1])
    rows = [
        ("truncated_block", good[:-3], n, "truncated"),
        ("truncated_checksum", ck[:-2], n, "truncated"),
        ("truncated_skippable", skippable(b"abcdef")[:-2], n, "truncated"),
        ("bad_magic", b"\x28\xb5\x2f\xfe" + good[4:], n, "bad magic"),
        ("reserved_bit", good[:4] + bytes([good[4] | 8]) + good[5:], n, "frame header"),
        ("dictionary", frame([block("raw", b"hello", 1)], fcs=5, dict_id=(7, 1)), 5, "dictionary"),
        ("reserved_block_type", hdr + block("reserved", b"abc", 1), 3, "block type"),
        ("block_over_window", frame_header(window_log=10, single=False) + block("raw", bytes(2000), 1), 2000, "block size"),
        ("literals_past_block", hdr + block("compressed", bytes([31 << 3]) + b"ab", 1), 31, "literals"),
        ("treeless_without_table", hdr + block("compressed", bytes([3, 0, 0, 0]), 1), 0, "huffman"),
        ("fse_accuracy_too_high", hdr + block("raw", b"abcdefgh", 0) +
         block("compressed", bytes([0, 1, 2 << 6, 0x0F, 0, 0]), 1), 11, "fse"),
        ("repeat_without_table", hdr + block("raw", b"abcdefgh", 0) + block("compressed", bytes([0, 1, 0xFC, 1]), 1), 11,
         "sequences"),
        ("zero_sequences_trailing_bytes", hdr + block("compressed", bytes([0, 0, 7]), 1), 0, "sequences"),
        ("no_padding_marker", hdr + block("raw", b"abcdefgh", 0) + rle_seq_block(b"", 2, 0, 0, 0, lambda i: 0, 1)[:-1] +
         b"\x00", 14, "sequences"),
        ("literal_overrun", hdr + block("raw", b"abcdefgh", 0) + rle_seq_block(b"ab", 1, 5, 0, 0, lambda i: 0, 1), 16,
         "sequences"),
        ("offset_before_output", hdr + rle_seq_block(b"", 1, 0, 0, 0, lambda i: 0, 1), 3, "offset"),
        ("offset_zero", hdr + block("raw", b"abcdefgh", 0) + rle_seq_block(b"", 1, 0, 1, 0, lambda i: 1, 1), 11, "offset"),
        ("offset_beyond_window", frame_header(window_log=10, single=False) + block("raw", bytes(1024), 0) +
         block("raw", bytes(1024), 0) + rle_seq_block(b"", 1, 0, 10, 0, lambda i: 1503 - 1024, 1), 2051, "offset"),
        ("content_size_short", frame([block("raw", b"hello", 1)], fcs=10), 10, "content size"),
        ("content_size_long", frame([block("raw", b"hello", 0), block("raw", b"world", 1)], fcs=7), 7, "content size"),
        ("second_frame_corrupt", good + good[:-3], 2 * n, "truncated"),
        ("checksum_mismatch", bad_ck, n, CHECKSUM),
        ("checksum_mismatch_then_corrupt", bad_ck + good[:-3], 2 * n, CHECKSUM),
        ("page_size_then_corrupt", reframe(good, fcs=False) + good[:-3], n - 10, "page size"),
    ]
    return rows


def golden_payload():
    """the bytes the golden frames hold (tests/golden/gen_zstd_golden.py writes them)"""
    rng = np.random.default_rng(2024)
    ts = (np.cumsum(rng.integers(0, 1000, 40_000)) + (1 << 40)).astype(np.int64).tobytes()
    return ts + b" ".join(rng.choice([b"alpha", b"beta", b"gamma"], 20_000))
