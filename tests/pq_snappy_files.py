"""Test helper: walk a SNAPPY Parquet column chunk (as pyarrow writes it, or a parquet-testing fixture) and plan its
device decode: one upload of the chunk as it sits in the file, the batched decompression into one buffer, and the
level / dictionary / PLAIN / DELTA_BINARY_PACKED page descriptors that chunk_plan (pq_files.py) builds, over the
decompressed buffer.  Not product code."""
import numpy as np

import pq_pages as P

DELTA_BINARY_PACKED = 5


def column_chunk(path, row_group=0, column=0):
    """(chunk bytes, [{type, num_values, encoding, payload_off, compressed_size, uncompressed_size, def_len, rep_len,
    is_compressed}]) of one column chunk; payload_off is the page body's offset in the chunk"""
    import pyarrow.parquet as pq
    meta = pq.ParquetFile(path).metadata.row_group(row_group).column(column)
    start = meta.dictionary_page_offset if meta.has_dictionary_page else meta.data_page_offset
    with open(path, "rb") as f:
        f.seek(start)
        buf = f.read(meta.total_compressed_size)
    pages, pos = [], 0
    while pos < len(buf):
        r = P._Reader(buf, pos)
        h = r.struct()
        pg = {"type": h[1], "uncompressed_size": h[2], "compressed_size": h[3], "payload_off": r.pos,
              "def_len": 0, "rep_len": 0, "is_compressed": True}
        if h[1] == P.DICTIONARY_PAGE:
            pg.update(num_values=h[7][1], encoding=h[7][2])
        elif h[1] == P.DATA_PAGE:
            pg.update(num_values=h[5][1], encoding=h[5][2])
        elif h[1] == P.DATA_PAGE_V2:
            d = h[8]
            pg.update(num_values=d[1], encoding=d[4], def_len=d[5], rep_len=d[6], is_compressed=d.get(7, True))
        pos = r.pos + h[3]
        pages.append(pg)
    return buf, pages


def decompress_table(pages):
    """(region of every page in the decompressed buffer [(src, src_len, dst, dst_len)], indices of the compressed
    regions, buffer size).  A v2 page's levels are never compressed and stay out; a v2 page with is_compressed false
    is a plain copy.  Every page's output starts 8-byte aligned."""
    regions, comp, dst = [], [], 0
    for k, pg in enumerate(pages):
        lv = pg["rep_len"] + pg["def_len"]
        regions.append((pg["payload_off"] + lv, pg["compressed_size"] - lv, dst, pg["uncompressed_size"] - lv))
        if pg["is_compressed"]:
            comp.append(k)
        dst += pg["uncompressed_size"] - lv
        dst += -dst % 8
    return regions, comp, dst + 8


def snappy_chunk_plan(path):
    """Everything the device calls need for column 0 of row group 0:
       chunk     the column chunk's bytes as they sit in the file
       comp      [(src, src_len, dst, dst_len)] of the decompression, n_dst the decompressed buffer's size
       copies    [(src, dst, len)] of uncompressed v2 page bodies (chunk -> dst)
       levels    [(data, len, num_values, out)]; offsets into `dst` (v1) or into `chunk` (v2, levels_in == "chunk")
       dict      (dst offset, num_values) of the dictionary page or None
       dpages / ppages / delta   value page descriptors over `dst`; other: encodings of any other data pages
       n_slots, max_def, v1"""
    import pyarrow.parquet as pq
    max_def = pq.ParquetFile(path).schema.column(0).max_definition_level
    chunk, pages = column_chunk(path)
    regions, comp, n_dst = decompress_table(pages)
    plan = {"chunk": chunk, "comp": [regions[k] for k in comp], "n_dst": n_dst,
            "copies": [(r[0], r[2], r[3]) for k, r in enumerate(regions) if k not in comp], "dict": None, "levels": [], "dpages": [], "ppages": [],
            "delta": [], "other": [], "max_def": max_def, "v1": None, "levels_in": "dst"}
    slot = 0
    for pg, (s, sl, d, dl) in zip(pages, regions):
        if pg["type"] == P.DICTIONARY_PAGE:
            plan["dict"] = (d, pg["num_values"])
            continue
        nv = pg["num_values"]
        plan["v1"] = pg["type"] == P.DATA_PAGE
        if plan["v1"]:
            if max_def:
                plan["levels"].append((d, dl, nv, slot))    # 4-byte length + levels; value_sections finds the values
        else:
            plan["levels_in"] = "chunk"
            if max_def:
                plan["levels"].append((pg["payload_off"] + pg["rep_len"], pg["def_len"], nv, slot))
        desc = (d, dl, nv, slot)
        if pg["encoding"] in (P.PLAIN_DICTIONARY, P.RLE_DICTIONARY):
            plan["dpages"].append(desc)
        elif pg["encoding"] == P.PLAIN:
            plan["ppages"].append(desc)
        elif pg["encoding"] == DELTA_BINARY_PACKED:
            plan["delta"].append(desc)
        else:
            plan["other"].append(pg["encoding"])
        slot += nv
    plan["n_slots"] = slot
    return plan


def host_decompressed(plan):
    """the decompressed buffer built on the host with pyarrow (for comparisons)"""
    import pyarrow as pa
    out = bytearray(plan["n_dst"])
    for s, sl, d, dl in plan["comp"]:
        if dl:
            out[d:d + dl] = pa.decompress(plan["chunk"][s:s + sl], decompressed_size=dl, codec="snappy", asbytes=True)
    for s, d, n in plan["copies"]:
        out[d:d + n] = plan["chunk"][s:s + n]
    return bytes(out)


def value_sections(plan, dst):
    """v1 pages of an optional column: the value section starts after the levels and their 4-byte length, which is
    known once the page is decompressed (pq_pages.split_data_page)"""
    if not plan["v1"] or not plan["max_def"]:
        return plan
    for key in ("dpages", "ppages", "delta"):
        out = []
        for (d, dl, nv, slot) in plan[key]:
            nb = int.from_bytes(bytes(dst[d:d + 4]), "little")
            out.append((d + 4 + nb, dl - 4 - nb, nv, slot))
        plan[key] = out
    return plan


def write_snappy_file(path, tbl, version, use_dictionary=True, column_encoding=None, data_page_size=None):
    import pyarrow.parquet as pq
    kw = {"data_page_size": data_page_size} if data_page_size else {}
    if column_encoding:
        kw["column_encoding"] = column_encoding
    pq.write_table(tbl, path, compression="SNAPPY", use_dictionary=use_dictionary, data_page_version=version, **kw)


def as_array(buf):
    return np.frombuffer(bytes(buf), np.uint8).copy()
