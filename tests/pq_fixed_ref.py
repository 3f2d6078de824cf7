"""Python restatement of the BOOLEAN and fixed-width page decoders the device entry points implement (test oracle only).

  PlainBooleanDecoder / RleBooleanDecoder .DecodeToBitmap, decodeSpacedToBitmap   boolean_decoder.go:264-417
  PlainDecoder[T] (INT96 too)                                                   plain_encoding_types.go:61-110
  PlainFixedLenByteArrayDecoder, ByteStreamSplit*Decoder                       fixed_len_byte_array_decoder.go,
                                                                                byte_stream_split.go:98-250
  dictionary pages                                                              decoder.go:125-160 (as pq_ref.dict_decode)

It follows the decisions include/arrowgpu.h documents where they differ from the reference: a boolean null slot is 0,
an RLE boolean repeated byte is true when non-zero, a BYTE_STREAM_SPLIT page's value count is its stride.  Values are
rows of `width` bytes (uint8 arrays of shape (slots, width)); booleans are uint8 0/1 per slot.
"""
import numpy as np

import pq_ref as R

PLAIN, PLAIN_DICTIONARY, RLE, RLE_DICTIONARY, BYTE_STREAM_SPLIT = 0, 2, 3, 8, 9
INT32, INT64, INT96, FLOAT, DOUBLE, FLBA = 1, 2, 3, 4, 5, 7
WIDTH = {INT32: 4, FLOAT: 4, INT64: 8, DOUBLE: 8, INT96: 12}

RUN_MSG = {
    R.ERR_TRUNC_LITERAL: "literal run truncated (unexpected EOF in a bit-packed run)",
    R.ERR_ZERO_RUN: "run header with a count of 0",
    R.ERR_VARINT: "run header varint overruns the stream or the 32-bit run count",
    R.ERR_TRUNC_REPEATED: "repeated run value truncated",
    R.ERR_BIT_WIDTH: "invalid or corrupted bit width (dictionary indices take 0..32 bits)",
}
MSG_PLAIN_SHORT = "parquet: eof exception decode plain (fewer values than valid slots)"
MSG_EOF = "parquet: eof exception"
MSG_BSS_SIZE = "data size ({}) is too small for the number of values in in BYTE_STREAM_SPLIT ({})"
MSG_BSS_ALIGN = "ByteStreamSplit data size {} not aligned with byte_width: {}"
MSG_BSS_ALIGN_FLBA = "ByteStreamSplit data size {} not aligned with type FIXED_LEN_BYTE_ARRAY and byte_width: {}"
MSG_BSS_SHORT = "parquet: number of values / definitions levels read did not match"
MSG_BOOL_SHORT = "parquet: boolean data has {} bits available, need {}: unexpected EOF"
MSG_BOOL_LENGTH = "invalid length - {} (corrupt data page?)"
MSG_BOOL_BYTES = "received invalid number of bytes - {} (corrupt data page?)"
MSG_UNEXPECTED_EOF = "unexpected EOF"


def width_of(ptype, type_length=0):
    return type_length if ptype == FLBA else WIDTH[ptype]


def _need(valid_or_n):
    return valid_or_n if not isinstance(valid_or_n, np.ndarray) else int(valid_or_n.sum())


def spread(vals, valid_or_n, need):
    """dense values (rows) -> (slot rows with zeros in null slots, slots written); a short stream stops at the first
    valid slot whose value is missing"""
    vals = np.asarray(vals)
    if not isinstance(valid_or_n, np.ndarray):
        return vals, len(vals)
    valid = valid_or_n
    pos = np.flatnonzero(valid)
    slots = valid.size if len(vals) >= need else int(pos[len(vals)])
    out = np.zeros((slots,) + vals.shape[1:], vals.dtype)
    out[valid[:slots]] = vals[:int(valid[:slots].sum())]
    return out, slots


def _nothing(width):
    return np.zeros((0, width) if width else 0, np.uint8), 0


# ---------------------------------------------------------------------------------------------------- BOOLEAN ----
def bool_decode(enc, page, valid_or_n):
    """-> (uint8 0/1 per slot written, slots, message or None)"""
    page = bytes(page)
    need = _need(valid_or_n)
    msg = None
    if enc == PLAIN:
        if need > len(page) * 8:
            return (*_nothing(0), MSG_BOOL_SHORT.format(len(page) * 8, need))
        vals = np.unpackbits(np.frombuffer(page, np.uint8), bitorder="little")[:need]
    else:
        if len(page) < 4:
            return (*_nothing(0), MSG_BOOL_LENGTH.format(len(page)))
        nb = int.from_bytes(page[:4], "little")
        if nb > len(page) - 4:
            return (*_nothing(0), MSG_BOOL_BYTES.format(nb))
        raw, err = R.rle_decode(page[4:4 + nb], 1, need)
        vals = (raw != 0).astype(np.uint8)
        if err:
            msg = RUN_MSG[err]
        elif vals.size < need:
            msg = MSG_UNEXPECTED_EOF
    out, slots = spread(vals.astype(np.uint8), valid_or_n, need)
    return out, slots, msg


def bool_plain_encode(bits):
    return np.packbits(np.asarray(bits, np.uint8), bitorder="little").tobytes()


def bool_rle_encode(bits):
    s = R.rle_encode(np.asarray(bits, np.uint8).tolist(), 1)
    return len(s).to_bytes(4, "little") + s


# ------------------------------------------------------------------------------------------------ fixed width ----
def fixed_decode(ptype, width, enc, page, valid_or_n, dictionary=None):
    """-> (uint8 rows (slots, width), slots, message or None, lowest bad slot within the page or None)"""
    page = bytes(page)
    need = _need(valid_or_n)
    nslots = valid_or_n if not isinstance(valid_or_n, np.ndarray) else valid_or_n.size
    if enc == PLAIN:
        if need * width > len(page):
            if ptype == INT96:
                msg = f"parquet: eof exception decode plain INT96, nvals: {need}, nbytes: {need * 12}, datalen: {len(page)}"
            elif ptype == FLBA:
                msg = MSG_EOF
            else:
                msg = MSG_PLAIN_SHORT
            return (*_nothing(width), msg, None)
        vals = np.frombuffer(page[:need * width], np.uint8).reshape(need, width)
        out, slots = spread(vals, valid_or_n, need)
        return out, slots, None, None
    if enc == BYTE_STREAM_SPLIT:
        if nslots * width < len(page):
            return (*_nothing(width), MSG_BSS_SIZE.format(len(page), nslots), None)
        if len(page) % width:
            fmt = MSG_BSS_ALIGN_FLBA if ptype == FLBA else MSG_BSS_ALIGN
            return (*_nothing(width), fmt.format(len(page), width), None)
        stride = len(page) // width
        to_read = min(need, stride)
        if to_read * width > 0x7FFFFFFF:
            return (*_nothing(width), MSG_EOF, None)
        if isinstance(valid_or_n, np.ndarray) and to_read < need:
            return (*_nothing(width), MSG_BSS_SHORT, None)
        vals = np.frombuffer(page, np.uint8).reshape(width, stride).T[:to_read]
        out, slots = spread(np.ascontiguousarray(vals), valid_or_n, need)
        return out, slots, None, None
    # dictionary
    if len(page) == 0:
        bw, stream = 0, b""
    else:
        bw, stream = page[0], page[1:]
        if bw > 32:
            return (*_nothing(width), RUN_MSG[R.ERR_BIT_WIDTH], None)
    idx, err = R.rle_decode(stream, bw, need)
    dictionary = np.zeros((0, width), np.uint8) if dictionary is None else dictionary
    ok = idx < len(dictionary)
    rows = np.zeros((idx.size, width), np.uint8)
    rows[ok] = dictionary[idx[ok].astype(np.int64)]
    out, slots = spread(rows, valid_or_n, need)
    bad = None
    if (~ok).any():
        first = int(np.flatnonzero(~ok)[0])
        bad = first if not isinstance(valid_or_n, np.ndarray) else int(np.flatnonzero(valid_or_n)[first])
    return out, slots, RUN_MSG.get(err), bad


def bss_encode(rows):
    """rows (n, width) uint8 -> BYTE_STREAM_SPLIT page bytes"""
    return np.ascontiguousarray(np.asarray(rows, np.uint8).T).tobytes()


def dict_encode(indices, bw=None):
    """dictionary data page: bit width byte, then the RLE / bit-packed indices"""
    indices = np.asarray(indices)
    bw = max(int(indices.max(initial=0)).bit_length(), 1) if bw is None else bw
    return bytes([bw]) + R.rle_encode(indices.tolist(), bw)
