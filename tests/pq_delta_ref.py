"""Python restatement of the Parquet DELTA_BINARY_PACKED encoder and decoder the device entry points implement (test
oracle only).

  deltaBitPackEncoder   parquet/internal/encoding/delta_bit_packing.go:362-494 (block shape configurable)
  deltaBitPackDecoder   delta_bit_packing.go:72-316 (SetData, initBlock, unpackNextMini, Decode, DecodeSpaced)

It follows the decisions include/arrowgpu.h documents where they differ from the reference (blocks read lazily; an
error in the block chain keeps the miniblocks before it).
"""
import numpy as np

from pq_ref import unpack, varint

# deltaBitPackEncoder / deltaBitPackDecoder, parquet/internal/encoding/delta_bit_packing.go.  Error codes match the
# device decoder's; DELTA_MESSAGES holds the reference's text for each.
(DERR_NONE, DERR_EOF, DERR_ZERO_BLOCK, DERR_BLOCK_SIZE, DERR_ZERO_MINI, DERR_TOO_MANY_MINI, DERR_MINI_DIVIDE, DERR_VPM,
 DERR_COUNT, DERR_FIRST32, DERR_MIN_DELTA32, DERR_WIDTH_BYTES, DERR_WIDTH, DERR_PAYLOAD, DERR_SHORT) = range(15)
DELTA_MESSAGES = {
    DERR_EOF: "parquet: eof exception",
    DERR_ZERO_BLOCK: "parquet: cannot have zero values per block",
    DERR_BLOCK_SIZE: "parquet: values per block must be a multiple of 128, got {0}",
    DERR_ZERO_MINI: "parquet: cannot have zero miniblock per block",
    DERR_TOO_MANY_MINI: "parquet: too many miniblocks per block: {0}",
    DERR_MINI_DIVIDE: "parquet: miniblocks per block must divide the block size, got {0} miniblocks for {1} values",
    DERR_VPM: "parquet: values per miniblock must be a nonzero multiple of 32, got {0}",
    DERR_COUNT: "parquet: invalid delta value count {0} for {1} buffered values",
    DERR_FIRST32: "parquet: initial delta value {0} exceeds INT32 range",
    DERR_MIN_DELTA32: "parquet: minimum delta {0} exceeds INT32 range",
    DERR_WIDTH_BYTES: "failed to read byte",
    DERR_WIDTH: "parquet: delta bit width {0} exceeds decoder width {1}",
    DERR_PAYLOAD: "unexpected EOF",
    DERR_SHORT: "parquet: number of values / definition levels read did not match",
}
_M64 = (1 << 64) - 1


def zigzag(v):
    return ((v << 1) ^ (v >> 63)) & _M64


def _wrap(v, width):
    """two's-complement value of v at 8*width bits"""
    bits = 8 * width
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def _pack_bits(vals, bw):
    """uint64 values of bw bits, LSB-first, as little-endian bytes (len(vals) * bw a multiple of 8)"""
    if bw == 0 or len(vals) == 0:
        return b""
    bits = ((vals[:, None] >> np.arange(bw, dtype=np.uint64)) & np.uint64(1)).astype(np.uint8).ravel()
    return np.packbits(bits, bitorder="little").tobytes()


def delta_encode(values, width, block=128, miniblocks=4):
    """deltaBitPackEncoder.Put + FlushValues (delta_bit_packing.go:362-494), byte for byte, with a configurable block
    shape (the reference fixes 128/4): deltas wrap at the type width, the width bytes of absent miniblocks of the last
    block stay 0, and the last miniblock is padded with zeros.  Vectorised per block."""
    dt = np.int32 if width == 4 else np.int64
    v = np.asarray(values).astype(dt)
    vpm = block // miniblocks
    out = bytearray()
    if v.size:
        d = (v[1:] - v[:-1]).astype(np.int64) if width == 8 else (v[1:].astype(np.int32) - v[:-1]).astype(np.int32).astype(np.int64)
        with np.errstate(over="ignore"):
            for b0 in range(0, d.size, block):
                blk = d[b0:b0 + block]
                mn = int(blk.min())
                out += varint(zigzag(mn))
                wpos = len(out)
                out += bytes(miniblocks)
                u = blk.view(np.uint64) - np.uint64(mn & _M64)         # wraps like uint64(val - minDelta)
                for i in range(miniblocks):
                    m = u[i * vpm:(i + 1) * vpm]
                    if m.size == 0:
                        break
                    bw = int(m.max()).bit_length()
                    out[wpos + i] = bw
                    out += _pack_bits(np.concatenate([m, np.zeros(vpm - m.size, np.uint64)]), bw)
    first = int(v[0]) if v.size else 0
    return varint(block) + varint(miniblocks) + varint(int(v.size)) + varint(zigzag(first)) + bytes(out)


def _uvarint(buf, pos):
    """binary.ReadUvarint: (value, new pos) or (None, pos)"""
    x = 0
    for i in range(10):
        if pos >= len(buf):
            return None, pos
        c = buf[pos]
        pos += 1
        if c < 0x80:
            if i == 9 and c > 1:
                return None, pos
            return x | c << (7 * i), pos
        x |= (c & 0x7F) << (7 * i)
    return None, pos


def _unzigzag(u):
    return (u >> 1) ^ -(u & 1)


def delta_decode(page, width, valid_or_n):
    """SetData(num_values) + Decode / DecodeSpaced of one page, with the decisions include/arrowgpu.h documents (lazy
    blocks; an error in the block chain keeps the miniblocks before it).  valid_or_n: number of slots (dense) or a bool
    array of the page's slots (spaced).  Returns (values of the slots written, slots written, error code, message)."""
    page = bytes(page)
    dense = not isinstance(valid_or_n, np.ndarray)
    nslots = valid_or_n if dense else valid_or_n.size
    need = nslots if dense else int(valid_or_n.sum())
    dt = np.int32 if width == 4 else np.int64
    err, args, pos = DERR_NONE, (), 0
    block, pos = _uvarint(page, pos)
    nmini = vpm = total = first = 0
    if block is None:
        err = DERR_EOF
    elif block == 0:
        err = DERR_ZERO_BLOCK
    elif block > 0xFFFFFFFF or block % 128:
        err, args = DERR_BLOCK_SIZE, (block,)
    else:
        nmini, pos = _uvarint(page, pos)
        if nmini is None:
            err = DERR_EOF
        elif nmini == 0:
            err = DERR_ZERO_MINI
        elif nmini > 0xFFFFFFFF:
            err, args = DERR_TOO_MANY_MINI, (nmini,)
        elif block % nmini:
            err, args = DERR_MINI_DIVIDE, (nmini, block)
        elif (block // nmini) % 32:
            err, args = DERR_VPM, (block // nmini,)
        else:
            vpm = block // nmini
            total, pos = _uvarint(page, pos)
            if total is None:
                err = DERR_EOF
            elif total > 0xFFFFFFFF or total > nslots:
                err, args = DERR_COUNT, (total, nslots)
            else:
                fz, pos = _uvarint(page, pos)
                if fz is None:
                    err = DERR_EOF
                else:
                    first = _unzigzag(fz)
                    if width == 4 and not -(1 << 31) <= first < (1 << 31):
                        err, args = DERR_FIRST32, (first,)
    if err:
        total = 0
    cap = min(need, total)
    want = (cap - 2) // vpm + 1 if cap > 1 else 0                  # miniblocks holding deltas 1..cap-1
    minis = []                                                    # (payload offset, width, min delta) of touched miniblocks
    while not err and len(minis) < want:
        mz, pos = _uvarint(page, pos)
        if mz is None:
            err = DERR_EOF
            break
        md = _unzigzag(mz)
        if width == 4 and not -(1 << 31) <= md < (1 << 31):
            err, args = DERR_MIN_DELTA32, (md,)
            break
        if len(page) - pos < nmini:
            err = DERR_WIDTH_BYTES
            break
        widths, pos = page[pos:pos + nmini], pos + nmini
        for bw in widths:
            if len(minis) == want:
                break
            if bw > 8 * width:
                err, args = DERR_WIDTH, (bw, 8 * width)
                break
            nb = vpm * bw // 8
            if nb > len(page) - pos:
                err = DERR_PAYLOAD
                break
            minis.append((pos, bw, md))
            pos += nb
    produced = cap if not err else (1 + len(minis) * vpm if cap > 0 else 0)
    if not err and not dense and total < need:
        err, produced = DERR_SHORT, 0
    msg = DELTA_MESSAGES[err].format(*args) if err else None
    # values: first, then the running sum of (unpacked + min delta), wrapping at 64 bits (and 32 for INT32)
    parts = [unpack(page[o:o + vpm * bw // 8], vpm, bw) + np.uint64(md & _M64) for o, bw, md in minis]
    deltas = np.concatenate(parts)[:max(produced - 1, 0)] if parts else np.zeros(0, np.uint64)
    with np.errstate(over="ignore"):
        vals = np.concatenate([np.array([first & _M64], np.uint64), deltas]).cumsum(dtype=np.uint64)[:produced]
    vals = (vals & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.int32) if width == 4 else vals.view(np.int64)
    if dense:
        return vals.astype(dt), produced, err, msg
    if err == DERR_SHORT:
        return np.zeros(0, dt), 0, err, msg
    pos_valid = np.flatnonzero(valid_or_n)
    slots = nslots if produced == need else int(pos_valid[produced])
    out = np.zeros(slots, dt)
    out[pos_valid[:produced]] = vals
    return out, slots, err, msg
