"""Python restatement of the Parquet BYTE_ARRAY encoders and decoders the device entry points implement (test oracle
only).

  PlainByteArrayDecoder         parquet/internal/encoding/byte_array_decoder.go:144-189
  DeltaLengthByteArrayDecoder   delta_length_byte_array.go:113-188
  DeltaByteArrayDecoder         delta_byte_array.go:166-303
  dictionary indices            pq_ref.dict_decode

It follows the decisions include/arrowgpu.h documents where they differ from the reference (a failing PLAIN value or
DELTA_BYTE_ARRAY prefix keeps the values before it).
"""
import numpy as np

import pq_delta_ref as D
import pq_ref as R

PLAIN, PLAIN_DICTIONARY, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY, RLE_DICTIONARY = 0, 2, 6, 7, 8
MSG_EOF = "parquet: eof reading bytearray"
MSG_NEG_PLAIN = "parquet: invalid BYTE_ARRAY value"
MSG_NEG_LEN = "parquet: negative delta byte array length {0}"
MSG_EXCEED = "parquet: delta byte array lengths exceed payload size"
MSG_COUNT = "parquet: delta prefix and suffix length counts do not match"
MSG_FIRST = "parquet: first delta byte array prefix length must be zero"
MSG_PREFIX = "parquet: invalid delta byte array prefix length {0}"
MSG_SHORT = "parquet: number of values / definition levels read did not match"


# ---------------------------------------------------------------- encoders ----
def plain_encode(values):
    return b"".join(len(v).to_bytes(4, "little") + bytes(v) for v in values)


def dlba_encode(values, block=128, miniblocks=4):
    """DeltaLengthByteArrayEncoder: the lengths as DELTA_BINARY_PACKED INT32, then the bytes"""
    return D.delta_encode(np.array([len(v) for v in values], np.int64), 4, block, miniblocks) + b"".join(bytes(v) for v in values)


def dba_encode(values, block=128, miniblocks=4):
    """DeltaByteArrayEncoder: prefix lengths shared with the previous value, then the suffixes as DELTA_LENGTH"""
    prefixes, suffixes, last = [], [], b""
    for v in values:
        v = bytes(v)
        n = 0
        while n < min(len(v), len(last)) and v[n] == last[n]:
            n += 1
        prefixes.append(n)
        suffixes.append(v[n:])
        last = v
    return D.delta_encode(np.array(prefixes, np.int64), 4, block, miniblocks) + dlba_encode(suffixes, block, miniblocks)


# ---------------------------------------------------------------- decoders ----
def _shape(valid_or_n):
    dense = not isinstance(valid_or_n, np.ndarray)
    nslots = valid_or_n if dense else valid_or_n.size
    need = nslots if dense else int(valid_or_n.sum())
    return dense, nslots, need


def _spread(vals, valid_or_n, produced, short=False):
    """dense values -> (slot values with b"" for nulls, slots written), as the device counts slots"""
    dense, nslots, need = _shape(valid_or_n)
    if short:
        return [], 0
    if dense:
        return list(vals[:produced]), produced
    pos = np.flatnonzero(valid_or_n)
    slots = nslots if produced >= need else int(pos[produced])
    out = [b""] * slots
    for r, s in enumerate(pos[:produced]):
        out[s] = vals[r]
    return out, slots


def plain_decode(page, valid_or_n):
    """-> (slot values, slots written, message or None)"""
    page = bytes(page)
    _, _, need = _shape(valid_or_n)
    vals, pos, msg = [], 0, None
    while len(vals) < need:
        if len(page) - pos < 4:
            msg = MSG_EOF
            break
        n = int.from_bytes(page[pos:pos + 4], "little", signed=True)
        if n < 0:
            msg = MSG_NEG_PLAIN
            break
        if len(page) - pos - 4 < n:
            msg = MSG_EOF
            break
        vals.append(page[pos + 4:pos + 4 + n])
        pos += 4 + n
    out, slots = _spread(vals, valid_or_n, len(vals))
    return out, slots, msg


def delta_end(page):
    """bytesRead() of a sound DELTA_BINARY_PACKED stream once every value is decoded: the end of the miniblock holding
    the last delta (or of the header)"""
    pos = 0
    block, pos = D._uvarint(page, pos)
    nmini, pos = D._uvarint(page, pos)
    total, pos = D._uvarint(page, pos)
    _, pos = D._uvarint(page, pos)
    vpm = block // nmini
    want = (total - 2) // vpm + 1 if total > 1 else 0
    got = 0
    while got < want:
        _, pos = D._uvarint(page, pos)
        widths, pos = page[pos:pos + nmini], pos + nmini
        for bw in widths:
            if got == want:
                break
            pos += vpm * bw // 8
            got += 1
    return pos


def _lengths(page, nslots):
    """a DELTA_BINARY_PACKED INT32 stream decoded in full: (lengths, bytes read, message or None)"""
    vals, produced, err, msg = D.delta_decode(page, 4, nslots)
    if err:
        return None, 0, msg
    return [int(x) for x in vals], delta_end(page), None


def _dlba_set_data(page, nslots):
    """SetData: (lengths, payload, message or None)"""
    lens, end, msg = _lengths(page, nslots)
    if msg:
        return None, None, msg
    payload = page[end:]
    run = 0
    for n in lens:
        if n < 0:
            return None, None, MSG_NEG_LEN.format(n)
        if n > len(payload) - run:
            return None, None, MSG_EXCEED
        run += n
    return lens, payload, None


def dlba_decode(page, valid_or_n):
    page = bytes(page)
    dense, nslots, need = _shape(valid_or_n)
    lens, payload, msg = _dlba_set_data(page, nslots)
    if msg:
        return (*_spread([], valid_or_n, 0), msg)
    if not dense and len(lens) < need:
        return [], 0, MSG_SHORT
    vals, pos = [], 0
    for n in lens[:need]:
        vals.append(payload[pos:pos + n])
        pos += n
    return (*_spread(vals, valid_or_n, len(vals)), None)


def dba_decode(page, valid_or_n):
    page = bytes(page)
    dense, nslots, need = _shape(valid_or_n)
    pre, end, msg = _lengths(page, nslots)
    if not msg:
        suf_lens, payload, msg = _dlba_set_data(page[end:], nslots)
        if not msg and len(pre) != len(suf_lens):
            msg = MSG_COUNT
    if msg:
        return (*_spread([], valid_or_n, 0), msg)
    n = min(need, len(suf_lens))
    vals, last, pos = [], b"", 0
    for k in range(n):
        p = pre[k]
        if k == 0 and p != 0:
            msg = MSG_FIRST
            break
        if p < 0 or p > len(last):
            msg = MSG_PREFIX.format(p)
            break
        last = last[:p] + payload[pos:pos + suf_lens[k]]
        pos += suf_lens[k]
        vals.append(last)
    if not msg and not dense and len(suf_lens) < need:
        return [], 0, MSG_SHORT
    return (*_spread(vals, valid_or_n, len(vals)), msg)


def dict_decode(page, dictionary, valid_or_n):
    """-> (slot values, slots written, error code, lowest bad slot or None); a slot with an out-of-range index is b\"\""""
    codes = np.arange(1, len(dictionary) + 1, dtype=np.int64)            # 0 = null or out of range
    out, slots, err, bad = R.dict_decode(page, codes, valid_or_n)
    return [dictionary[c - 1] if c else b"" for c in out.tolist()], slots, err, bad


def decode(encoding, page, valid_or_n, dictionary=None):
    """one page -> (slot values, slots written, message or error code or None, bad slot or None)"""
    if encoding == PLAIN:
        return (*plain_decode(page, valid_or_n), None)
    if encoding == DELTA_LENGTH_BYTE_ARRAY:
        return (*dlba_decode(page, valid_or_n), None)
    if encoding == DELTA_BYTE_ARRAY:
        return (*dba_decode(page, valid_or_n), None)
    vals, slots, err, bad = dict_decode(page, dictionary, valid_or_n)
    return vals, slots, (err or None), bad


def arrow_buffers(n_slots, placed, offset_base=0):
    """placed: [(first slot, [values])] -> (offsets int64 [n_slots + 1], data bytes) of the Arrow array the device writes"""
    lens = np.zeros(n_slots, np.int64)
    chunks = {}
    for o, vals in placed:
        for k, v in enumerate(vals):
            lens[o + k] = len(v)
            chunks[o + k] = v
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64) + offset_base
    data = b"".join(chunks[i] for i in sorted(chunks))
    return offsets, data
