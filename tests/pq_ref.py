"""Python restatement of the Parquet hybrid-stream decoders the device entry points implement (test oracle only).

  RleEncoder      parquet/internal/utils/rle.go:314-445 (canonical streams: repeated runs of >= 8, literal runs of at
                  most 63 groups, a padded last group)
  RleDecoder      rle.go:123-239 (Next / GetBatch)
  LevelDecoder    parquet/internal/encoding/levels.go:188-297
  dictionary      decoder.go:125-160 over typed_rle_dict.go:143-236, dense and spaced
  PLAIN spaced    plain_encoding_types.go:98 -> spacedExpand (decoder.go:209)

It follows the decisions include/arrowgpu.h documents where they differ from the reference (errors on zero-count runs,
varint overruns, truncated repeated values, bit widths over 32 / 16, dictionary indices out of range in both paths).
"""
import numpy as np

OK, INVALID, NOT_IMPLEMENTED = 0, 1, 3
ERR_NONE, ERR_TRUNC_LITERAL, ERR_ZERO_RUN, ERR_VARINT, ERR_TRUNC_REPEATED, ERR_BIT_WIDTH, ERR_LEVELS_SHORT, ERR_LEVELS_LENGTH, ERR_PLAIN_SHORT = range(9)
NO_ERROR_POS = (1 << 63) - 1


def varint(v):
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def pack_group(vals, bw):
    """8 values of bw bits, LSB-first -> bw bytes"""
    acc = 0
    for i, v in enumerate(vals):
        acc |= int(v) << (i * bw)
    return acc.to_bytes(bw, "little") if bw else b""


def literal_run(vals, bw):
    """one literal run holding `vals` (padded with zeros to whole groups)"""
    vals = list(vals) + [0] * (-len(vals) % 8)
    groups = len(vals) // 8
    return varint(groups << 1 | 1) + b"".join(pack_group(vals[i:i + 8], bw) for i in range(0, len(vals), 8))


def repeated_run(value, count, bw):
    return varint(count << 1) + int(value).to_bytes((bw + 7) // 8, "little")


class RleEncoder:
    """RleEncoder.Put / Flush, byte for byte."""

    def __init__(self, bw):
        self.bw = bw
        self.out = bytearray()
        self.buffer = []
        self.cur = 0
        self.rep = 0
        self.lit = 0
        self.ind = -1

    def _flush_literal(self, update):
        if self.ind == -1:
            self.ind = len(self.out)
            self.out.append(0)
        if self.buffer:
            self.out += pack_group(self.buffer, self.bw)
        self.buffer = []
        if update:
            self.out[self.ind] = ((self.lit // 8) << 1 | 1) & 0xFF
            self.ind = -1
            self.lit = 0

    def _flush_repeated(self):
        self.out += varint(self.rep << 1) + int(self.cur).to_bytes((self.bw + 7) // 8, "little")
        self.rep = 0
        self.buffer = []

    def _flush_buffered(self, done):
        if self.rep >= 8:
            self.buffer = []
            if self.lit:
                self._flush_literal(True)
            return
        self.lit += len(self.buffer)
        self._flush_literal(True if self.lit // 8 + 1 >= 64 else done)
        self.rep = 0

    def put(self, v):
        if self.cur == v:
            self.rep += 1
            if self.rep > 8:
                return
        else:
            if self.rep >= 8:
                self._flush_repeated()
            self.rep = 1
            self.cur = v
        self.buffer.append(v)
        if len(self.buffer) == 8:
            self._flush_buffered(False)

    def flush(self):
        if self.lit > 0 or self.rep > 0 or self.buffer:
            all_rep = self.lit == 0 and (self.rep == len(self.buffer) or not self.buffer)
            if self.rep > 0 and all_rep:
                self._flush_repeated()
            else:
                self.buffer += [0] * ((8 - len(self.buffer)) % 8 if self.buffer else 0)
                self.lit += len(self.buffer)
                self._flush_literal(True)
                self.rep = 0
        return bytes(self.out)


def rle_encode(values, bw):
    e = RleEncoder(bw)
    for v in values:
        e.put(int(v))
    return e.flush()


def unpack(payload, count, bw):
    if bw == 0 or count == 0:
        return np.zeros(count, dtype=np.uint64)
    bits = np.unpackbits(np.frombuffer(payload, dtype=np.uint8), bitorder="little")[:count * bw].reshape(count, bw).astype(np.uint64)
    return (bits << np.arange(bw, dtype=np.uint64)).sum(axis=1, dtype=np.uint64)


def rle_decode(stream, bw, need):
    """Decode up to `need` values.  Returns (uint64 values, error code)."""
    out, produced, pos, n = [], 0, 0, len(stream)
    nrep = (bw + 7) // 8
    while produced < need and pos < n:
        ind, k = 0, 0
        while True:
            if pos + k >= n or k == 5:
                return _cat(out), ERR_VARINT
            c = stream[pos + k]
            ind |= (c & 0x7F) << (7 * k)
            k += 1
            if not c & 0x80:
                break
        body, count = pos + k, ind >> 1
        if count == 0:
            return _cat(out), ERR_ZERO_RUN
        if ind & 1:
            if count > 0x7FFFFFFF // 8:
                return _cat(out), ERR_VARINT
            take = min(count * 8, need - produced)
            avail = (n - body) * 8
            if take * bw > avail:
                got = min(take, avail // (32 * bw) * 32)
                out.append(unpack(stream[body:], got, bw))
                return _cat(out), ERR_TRUNC_LITERAL
            out.append(unpack(stream[body:body + count * bw], take, bw))
            produced += take
            pos = body + count * bw
        else:
            if count > 0x7FFFFFFF:
                return _cat(out), ERR_VARINT
            if body + nrep > n:
                return _cat(out), ERR_TRUNC_REPEATED
            v = int.from_bytes(stream[body:body + nrep], "little")
            take = min(count, need - produced)
            out.append(np.full(take, v, dtype=np.uint64))
            produced += take
            pos = body + nrep
    return _cat(out), ERR_NONE


def _cat(parts):
    return np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint64)


def levels_decode_page(page, max_level, v1, num_values):
    """LevelDecoder.SetData(RLE)/SetDataV2 + Decode: (int16 levels, error code)"""
    bw = int(max_level).bit_length()
    page = bytes(page)
    if v1:
        if len(page) < 4:
            return np.zeros(0, np.int16), ERR_LEVELS_SHORT
        nb = int.from_bytes(page[:4], "little", signed=True)
        if nb < 0 or nb > len(page) - 4:
            return np.zeros(0, np.int16), ERR_LEVELS_LENGTH
        page = page[4:4 + nb]
    vals, err = rle_decode(page, bw, num_values)
    return vals.astype(np.uint16).view(np.int16), err


def dict_decode(page, dictionary, valid_or_n):
    """dictDecoder.SetData + decode / decodeSpaced.  valid_or_n: number of slots (dense) or a bool array of the
    page's slots (spaced).  Returns (values, slots written, error code, lowest bad slot within the page or None)."""
    page = bytes(page)
    dense = not isinstance(valid_or_n, np.ndarray)
    nslots = valid_or_n if dense else valid_or_n.size
    need = nslots if dense else int(valid_or_n.sum())
    if len(page) == 0:
        bw, stream = 0, b""
    else:
        bw, stream = page[0], page[1:]
        if bw > 32:
            return np.zeros(0, dictionary.dtype), 0, ERR_BIT_WIDTH, None
    idx, err = rle_decode(stream, bw, need)
    produced = idx.size
    if dense:
        slots, valid = produced, None
        rank = np.arange(slots)
        vmask = np.ones(slots, bool)
    else:
        valid = valid_or_n
        pos = np.flatnonzero(valid)
        slots = nslots if produced == need else int(pos[produced])
        vmask = valid[:slots]
        rank = np.cumsum(vmask) - 1
    out = np.zeros(slots, dtype=dictionary.dtype)
    bad = None
    sel = np.flatnonzero(vmask)
    iv = idx[rank[sel]] if sel.size else np.zeros(0, np.uint64)
    okm = iv < dictionary.size
    out[sel[okm]] = dictionary[iv[okm].astype(np.int64)]
    if (~okm).any():
        bad = int(sel[~okm][0])
    return out, slots, err, bad


def plain_decode_spaced(page, dtype, valid):
    """PlainDecoder.DecodeSpaced: (values with 0 in null slots, error code)"""
    dtype = np.dtype(dtype)
    need = int(valid.sum())
    if need * dtype.itemsize > len(page):
        return np.zeros(0, dtype), ERR_PLAIN_SHORT
    vals = np.frombuffer(bytes(page[:need * dtype.itemsize]), dtype=dtype)
    out = np.zeros(valid.size, dtype=dtype)
    out[valid] = vals
    return out, ERR_NONE
