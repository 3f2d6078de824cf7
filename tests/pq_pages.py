"""Test helper: walk an uncompressed Parquet column chunk (as pyarrow writes it) and return its pages.

Only what the tests need: a Thrift compact-protocol reader for PageHeader, and the chunk's byte range from pyarrow's
column-chunk metadata (dictionary_page_offset, data_page_offset, total_compressed_size).  Not product code."""
import numpy as np

DATA_PAGE, DICTIONARY_PAGE, DATA_PAGE_V2 = 0, 2, 3
PLAIN, PLAIN_DICTIONARY, RLE_DICTIONARY = 0, 2, 8


class _Reader:
    def __init__(self, buf, pos):
        self.buf, self.pos = buf, pos

    def byte(self):
        b = self.buf[self.pos]
        self.pos += 1
        return b

    def uvarint(self):
        v, sh = 0, 0
        while True:
            b = self.byte()
            v |= (b & 0x7F) << sh
            sh += 7
            if not b & 0x80:
                return v

    def zigzag(self):
        v = self.uvarint()
        return (v >> 1) ^ -(v & 1)

    def value(self, t):
        if t in (1, 2):          # BOOLEAN_TRUE / BOOLEAN_FALSE inside a struct
            return t == 1
        if t == 3:
            return self.byte()
        if t in (4, 5, 6):
            return self.zigzag()
        if t == 7:
            self.pos += 8
            return None
        if t == 8:
            n = self.uvarint()
            self.pos += n
            return bytes(self.buf[self.pos - n:self.pos])
        if t in (9, 10):
            h = self.byte()
            n, et = h >> 4, h & 0x0F
            if n == 15:
                n = self.uvarint()
            return [self.byte() == 1 if et in (1, 2) else self.value(et) for _ in range(n)]
        if t == 11:
            n = self.uvarint()
            if n:
                kv = self.byte()
                return [(self.value(kv >> 4), self.value(kv & 0x0F)) for _ in range(n)]
            return []
        if t == 12:
            return self.struct()
        raise ValueError(f"thrift compact type {t}")

    def struct(self):
        out, fid = {}, 0
        while True:
            h = self.byte()
            if h == 0:
                return out
            delta, t = h >> 4, h & 0x0F
            fid = fid + delta if delta else self.zigzag()
            out[fid] = self.value(t)


def column_chunk_pages(path, row_group=0, column=0):
    """[{type, num_values, encoding, payload (bytes), def_len (v2), num_nulls (v2)}, ...] of one column chunk"""
    import pyarrow.parquet as pq
    meta = pq.ParquetFile(path).metadata.row_group(row_group).column(column)
    assert meta.compression == "UNCOMPRESSED", meta.compression
    start = meta.dictionary_page_offset if meta.has_dictionary_page else meta.data_page_offset
    with open(path, "rb") as f:
        f.seek(start)
        buf = f.read(meta.total_compressed_size)
    pages, pos = [], 0
    while pos < len(buf):
        r = _Reader(buf, pos)
        h = r.struct()
        size = h[3]
        payload = buf[r.pos:r.pos + size]
        pos = r.pos + size
        t = h[1]
        if t == DICTIONARY_PAGE:
            pages.append({"type": t, "num_values": h[7][1], "encoding": h[7][2], "payload": payload})
        elif t == DATA_PAGE:
            pages.append({"type": t, "num_values": h[5][1], "encoding": h[5][2], "payload": payload})
        elif t == DATA_PAGE_V2:
            d = h[8]
            pages.append({"type": t, "num_values": d[1], "num_nulls": d[2], "encoding": d[4], "def_len": d[5],
                          "rep_len": d[6], "payload": payload})
    return pages


def split_data_page(page, max_def):
    """(levels section offset, levels section length, values offset) of a flat column's data page: v1 pages carry
    `4-byte length + RLE levels` when the column is optional; v2 pages carry def_len bytes of levels."""
    p = page["payload"]
    if page["type"] == DATA_PAGE_V2:
        lo = page.get("rep_len", 0)
        return lo, page["def_len"], lo + page["def_len"]
    if max_def == 0:
        return 0, 0, 0
    nb = int.from_bytes(p[:4], "little")
    return 0, len(p), 4 + nb


def np_of(arrow_type):
    import pyarrow as pa
    return {pa.int32(): np.int32, pa.int64(): np.int64, pa.float32(): np.float32, pa.float64(): np.float64}[arrow_type]
