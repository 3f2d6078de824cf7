"""Test helper: walk a Parquet column chunk (as pyarrow writes it, or a parquet-testing fixture, any codec) and plan its
read: one upload of the chunk as it sits in the file, the batched decompression into one buffer, and the level /
dictionary / value page descriptors over it.  Also lays out synthetic page streams for the unit tests.  Not product
code."""
import numpy as np

DATA_PAGE, DICTIONARY_PAGE, DATA_PAGE_V2 = 0, 2, 3
PLAIN, PLAIN_DICTIONARY, RLE, DELTA_BINARY_PACKED, RLE_DICTIONARY, BYTE_STREAM_SPLIT = 0, 2, 3, 5, 8, 9
DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY = 6, 7
BOOLEAN, INT32, INT64, INT96, FLOAT, DOUBLE, BYTE_ARRAY, FIXED_LEN_BYTE_ARRAY = range(8)
PTYPES = {"BOOLEAN": BOOLEAN, "INT32": INT32, "INT64": INT64, "INT96": INT96, "FLOAT": FLOAT, "DOUBLE": DOUBLE,
          "BYTE_ARRAY": BYTE_ARRAY, "FIXED_LEN_BYTE_ARRAY": FIXED_LEN_BYTE_ARRAY}


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


def column_chunk(path, row_group=0, column=0):
    """(chunk bytes, [{type, num_values, encoding, payload_off, compressed_size, uncompressed_size, def_len, rep_len,
    is_compressed}]) of one column chunk; payload_off is the page body's offset in the chunk.  No page of an
    UNCOMPRESSED chunk is compressed."""
    import pyarrow.parquet as pq
    meta = pq.ParquetFile(path).metadata.row_group(row_group).column(column)
    start = meta.dictionary_page_offset if meta.has_dictionary_page else meta.data_page_offset
    with open(path, "rb") as f:
        f.seek(start)
        buf = f.read(meta.total_compressed_size)
    codec = meta.compression != "UNCOMPRESSED"
    pages, pos = [], 0
    while pos < len(buf):
        r = _Reader(buf, pos)
        h = r.struct()
        pg = {"type": h[1], "uncompressed_size": h[2], "compressed_size": h[3], "payload_off": r.pos,
              "def_len": 0, "rep_len": 0, "is_compressed": codec}
        if h[1] == DICTIONARY_PAGE:
            pg.update(num_values=h[7][1], encoding=h[7][2])
        elif h[1] == DATA_PAGE:
            pg.update(num_values=h[5][1], encoding=h[5][2])
        elif h[1] == DATA_PAGE_V2:
            d = h[8]
            pg.update(num_values=d[1], encoding=d[4], def_len=d[5], rep_len=d[6], is_compressed=codec and d.get(7, True))
        pos = r.pos + h[3]
        pages.append(pg)
    return buf, pages


def decompress_table(pages):
    """(region of every page in the decompressed buffer [(src, src_len, dst, dst_len)], indices of the compressed
    regions, buffer size).  A v2 page's levels are never compressed and stay out; a page that is not compressed is a
    plain copy.  Every page's output starts 8-byte aligned."""
    regions, comp, dst = [], [], 0
    for k, pg in enumerate(pages):
        lv = pg["rep_len"] + pg["def_len"]
        regions.append((pg["payload_off"] + lv, pg["compressed_size"] - lv, dst, pg["uncompressed_size"] - lv))
        if pg["is_compressed"]:
            comp.append(k)
        dst += pg["uncompressed_size"] - lv
        dst += -dst % 8
    return regions, comp, dst + 8


def chunk_plan(path, column=0):
    """Everything a reader needs for column `column` of row group 0, any physical type and codec:
       chunk, codec            the column chunk's bytes as they sit in the file, and its codec
       comp, n_dst             [(src, src_len, dst, dst_len)] of the decompression into one buffer `dst` of n_dst bytes
       copies                  [(src, dst, len)] of the page bodies that are not compressed (chunk -> dst)
       ptype, type_length, max_def
       v1                      the levels encoding, the same on every data page: v1 levels (4-byte length + RLE) sit at
                               the start of their page in `dst`, v2 levels (RLE) straight in `chunk`
       dict                    (dst offset, len, num_values) of the dictionary page or None
       pages                   [(encoding, levels (data, len, num_values, out) or None, values (data, len, num_values,
                               out))] of the data pages; value_sections() finds the values of v1 pages with levels
       n_slots"""
    import pyarrow.parquet as pq
    f = pq.ParquetFile(path)
    col = f.schema.column(column)
    chunk, pages = column_chunk(path, column=column)
    regions, comp, n_dst = decompress_table(pages)
    plan = {"chunk": chunk, "codec": f.metadata.row_group(0).column(column).compression, "n_dst": n_dst,
            "comp": [regions[k] for k in comp], "copies": [(r[0], r[2], r[3]) for k, r in enumerate(regions) if k not in comp],
            "ptype": PTYPES[col.physical_type], "type_length": col.length or 0, "max_def": col.max_definition_level,
            "v1": None, "dict": None, "pages": []}
    slot = 0
    for pg, (s, sl, d, dl) in zip(pages, regions):
        nv = pg["num_values"]
        if pg["type"] == DICTIONARY_PAGE:
            plan["dict"] = (d, dl, nv)
            continue
        v1 = pg["type"] == DATA_PAGE
        assert plan["v1"] in (None, v1), "v1 and v2 data pages in one chunk"
        plan["v1"] = v1
        levels = None
        if plan["max_def"]:
            levels = (d, dl, nv, slot) if v1 else (pg["payload_off"] + pg["rep_len"], pg["def_len"], nv, slot)
        plan["pages"].append((pg["encoding"], levels, (d, dl, nv, slot)))
        slot += nv
    plan["n_slots"] = slot
    return plan


def host_decompress(plan):
    """the decompressed buffer `dst` built on the host with pyarrow (a Parquet "LZ4" chunk is LZ4_RAW, pyarrow's
    "lz4_raw"; its "lz4" is the frame format)"""
    import pyarrow as pa
    codec = {"LZ4": "lz4_raw"}.get(plan["codec"], plan["codec"].lower())
    out = bytearray(plan["n_dst"])
    for s, sl, d, dl in plan["comp"]:
        if dl:
            out[d:d + dl] = pa.decompress(plan["chunk"][s:s + sl], decompressed_size=dl, codec=codec, asbytes=True)
    for s, d, n in plan["copies"]:
        out[d:d + n] = plan["chunk"][s:s + n]
    return bytes(out)


def value_sections(plan, dst):
    """[(encoding, (data, len, num_values, out))] of the data pages' values in `dst`: a v1 page of an optional column
    holds a 4-byte level length and the levels first, so its values start after them"""
    out = []
    for enc, _, (d, dl, nv, slot) in plan["pages"]:
        if plan["v1"] and plan["max_def"]:
            nb = int.from_bytes(bytes(dst[d:d + 4]), "little")
            d, dl = d + 4 + nb, dl - 4 - nb
        out.append((enc, (d, dl, nv, slot)))
    return out


def encodings(plan):
    return {e for e, _, _ in plan["pages"]}


def as_array(buf):
    return np.frombuffer(bytes(buf), np.uint8).copy()


def batch(streams, rng, gap=True):
    """Lay `streams` [(bytes, num_values)] out in one buffer at odd byte offsets, give each page an output range
    (with gaps, at odd element offsets), and shuffle the page order.  Returns (blob, pages, n_out)."""
    blob, pages, slot = bytearray(), [], 3 if gap else 0
    for s, nv in streams:
        if gap:
            blob += bytes(int(rng.integers(0, 7)))
        pages.append((len(blob), len(s), nv, slot))
        blob += s
        slot += nv + (int(rng.integers(0, 5)) if gap else 0)
    blob += bytes(8)
    order = rng.permutation(len(pages)) if gap else np.arange(len(pages))
    return as_array(blob), [pages[i] for i in order], slot + 8


def compressed_batch(streams, rng, gap=True):
    """batch() for ag_pq_compressed tables: `streams` [(bytes, dst_len)] at odd byte offsets, each page's output range
    at odd byte offsets with gaps between them, the page order shuffled.  Returns (src, pages, n_out)."""
    blob, pages, out = bytearray(), [], 3 if gap else 0
    for s, n in streams:
        if gap:
            blob += bytes(int(rng.integers(0, 7)))
        pages.append((len(blob), len(s), out, n))
        blob += s
        out += n + (int(rng.integers(1, 6)) if gap else 0)
    blob += bytes(8)
    order = rng.permutation(len(pages)) if gap else np.arange(len(pages))
    return as_array(blob), [pages[i] for i in order], out + 8
