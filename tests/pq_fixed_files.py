"""Test helper: pyarrow-written Parquet files with BOOLEAN, FIXED_LEN_BYTE_ARRAY, INT96 and BYTE_STREAM_SPLIT columns,
the plan that turns one column chunk (uncompressed, SNAPPY or ZSTD) into batched page descriptors over its decompressed
pages, and the physical values pq.read_table's result stands for.  Not product code."""
import decimal

import numpy as np

import pq_fixed_ref as X
import pq_pages as P
import pq_snappy_files as Z

NULL_FRACS = (None, 0.0, 0.1, 1.0)
PTYPES = {"BOOLEAN": 0, "INT32": X.INT32, "INT64": X.INT64, "INT96": X.INT96, "FLOAT": X.FLOAT, "DOUBLE": X.DOUBLE,
          "FIXED_LEN_BYTE_ARRAY": X.FLBA}
# (kind, arrow type maker, encoding): every flat kind this change decodes
KINDS = {
    "bool": "PLAIN", "fsb1": "PLAIN", "fsb3": "PLAIN", "fsb12": "PLAIN", "fsb16": "PLAIN", "fsb1000": "PLAIN",
    "decimal": "PLAIN", "float16": "PLAIN", "int96": "PLAIN", "fsb16_dict": "RLE_DICTIONARY", "int96_dict": "RLE_DICTIONARY",
    "bss_float": "BYTE_STREAM_SPLIT", "bss_double": "BYTE_STREAM_SPLIT", "bss_int32": "BYTE_STREAM_SPLIT",
    "bss_int64": "BYTE_STREAM_SPLIT", "bss_fsb5": "BYTE_STREAM_SPLIT",
}


def make_array(rng, kind, n, null_frac):
    import pyarrow as pa
    mask = None if null_frac is None else rng.random(n) < null_frac
    if kind == "bool":
        return pa.array(rng.random(n) < 0.4, pa.bool_(), mask=mask)
    if kind.startswith("fsb") or kind == "bss_fsb5":
        w = 5 if kind == "bss_fsb5" else int(kind[3:].split("_")[0])
        pool = [bytes(rng.integers(0, 256, w, dtype=np.uint8)) for _ in range(200 if "dict" in kind else n)]
        vals = pool if "dict" not in kind else [pool[i] for i in rng.integers(0, len(pool), n)]
        return pa.array(vals, pa.binary(w), mask=mask)
    if kind == "decimal":
        vals = [decimal.Decimal(int(v)).scaleb(-3) for v in rng.integers(-(10 ** 17), 10 ** 17, n)]
        return pa.array(vals, pa.decimal128(20, 3), mask=mask)
    if kind == "float16":
        return pa.array(rng.standard_normal(n).astype(np.float16), pa.float16(), mask=mask)
    if kind.startswith("int96"):
        base = rng.integers(-(10 ** 18), 10 ** 18, 150 if "dict" in kind else n)
        ns = base if "dict" not in kind else base[rng.integers(0, base.size, n)]
        return pa.array(ns, pa.timestamp("ns"), mask=mask)
    t = {"bss_float": np.float32, "bss_double": np.float64, "bss_int32": np.int32, "bss_int64": np.int64}[kind]
    v = rng.standard_normal(n).astype(t) if t in (np.float32, np.float64) else rng.integers(-(1 << 30), 1 << 30, n).astype(t)
    return pa.array(v, mask=mask)


def write_file(path, rng, kind, null_frac, version, n=6000, data_page_size=None, compression="NONE", dictionary_pagesize_limit=None):
    import pyarrow as pa
    import pyarrow.parquet as pq
    arr = make_array(rng, kind, n, null_frac)
    tbl = pa.Table.from_arrays([arr], schema=pa.schema([pa.field("c", arr.type, nullable=null_frac is not None)]))
    enc = KINDS[kind]
    kw = {"data_page_size": data_page_size} if data_page_size else {}
    if dictionary_pagesize_limit:
        kw["dictionary_pagesize_limit"] = dictionary_pagesize_limit
    if kind.startswith("int96"):
        kw["use_deprecated_int96_timestamps"] = True
    if enc == "RLE_DICTIONARY":
        pq.write_table(tbl, path, compression=compression, use_dictionary=True, data_page_version=version, **kw)
    elif kind == "bool":
        pq.write_table(tbl, path, compression=compression, use_dictionary=False, data_page_version=version, **kw)
    else:
        pq.write_table(tbl, path, compression=compression, use_dictionary=False, column_encoding={"c": enc},
                       data_page_version=version, **kw)
    return tbl


def host_decompress(plan, codec):
    import pyarrow as pa
    out = bytearray(plan["n_dst"])
    for s, sl, d, dl in plan["comp"]:
        if dl:
            src = plan["chunk"][s:s + sl]
            out[d:d + dl] = src if codec == "UNCOMPRESSED" else pa.decompress(src, decompressed_size=dl, codec=codec.lower(), asbytes=True)
    for s, d, n in plan["copies"]:
        out[d:d + n] = plan["chunk"][s:s + n]
    return bytes(out)


def chunk_plan(path, column=0):
    """column `column` of row group 0:
       chunk, comp, copies, n_dst   as pq_snappy_files.snappy_chunk_plan (the decompression of every page)
       codec, ptype, type_length
       dict      (dst offset, len, num_values) of the dictionary page or None
       pages     [(encoding, (dst offset, len, num_values, out))] of the data pages' value sections; v1 pages of an
                 optional column hold levels first, so value_sections() finds those once the pages are decompressed
       n_slots, max_def, v1"""
    import pyarrow.parquet as pq
    f = pq.ParquetFile(path)
    col = f.schema.column(column)
    meta = f.metadata.row_group(0).column(column)
    chunk, pages = Z.column_chunk(path, column=column)
    regions, comp, n_dst = Z.decompress_table(pages)
    plan = {"chunk": chunk, "comp": [regions[k] for k in comp], "n_dst": n_dst,
            "copies": [(r[0], r[2], r[3]) for k, r in enumerate(regions) if k not in comp], "dict": None, "pages": [],
            "codec": meta.compression, "ptype": PTYPES[col.physical_type], "type_length": col.length or 0,
            "max_def": col.max_definition_level, "v1": None}
    slot = 0
    for pg, (s, sl, d, dl) in zip(pages, regions):
        if pg["type"] == P.DICTIONARY_PAGE:
            plan["dict"] = (d, dl, pg["num_values"])
            continue
        plan["v1"] = pg["type"] == P.DATA_PAGE
        plan["pages"].append((pg["encoding"], (d, dl, pg["num_values"], slot)))
        slot += pg["num_values"]
    plan["n_slots"] = slot
    return plan


def value_sections(plan, dst):
    """v1 pages of an optional column: the values start after the 4-byte level length and the levels"""
    if not plan["v1"] or not plan["max_def"]:
        return plan
    out = []
    for enc, (d, dl, nv, slot) in plan["pages"]:
        nb = int.from_bytes(bytes(dst[d:d + 4]), "little")
        out.append((enc, (d + 4 + nb, dl - 4 - nb, nv, slot)))
    plan["pages"] = out
    return plan


def int96_of_ns(ns):
    """INT96 physical bytes (nanoseconds of the day, then the Julian day, little-endian) of timestamps in ns"""
    ns = np.asarray(ns, np.int64)
    day, nod = np.divmod(ns, 86_400_000_000_000)
    out = np.zeros((ns.size, 12), np.uint8)
    out[:, :8] = nod.astype("<i8").view(np.uint8).reshape(-1, 8)
    out[:, 8:] = (day + 2440588).astype("<u4").view(np.uint8).reshape(-1, 4)
    return out


def expected(tbl, ptype, width):
    """(physical values as uint8 rows (n, width) with zeros in null slots; booleans: uint8 0/1, validity)"""
    import pyarrow as pa
    col = tbl.column(0).combine_chunks()
    valid = np.asarray(col.is_valid())
    n = len(col)
    if ptype == 0:
        return np.asarray(col.fill_null(False)).astype(np.uint8), valid
    t = col.type
    if pa.types.is_timestamp(t):
        ns = np.asarray(col.cast(pa.int64()).fill_null(0))
        rows = int96_of_ns(ns)
    elif pa.types.is_decimal(t):
        rows = np.zeros((n, width), np.uint8)
        for i, v in enumerate(col.to_pylist()):
            if v is not None:
                unscaled = int(v.scaleb(t.scale))
                rows[i] = np.frombuffer(unscaled.to_bytes(width, "big", signed=True), np.uint8)
    elif pa.types.is_fixed_size_binary(t):
        rows = np.zeros((n, width), np.uint8)
        for i, v in enumerate(col.to_pylist()):
            if v is not None:
                rows[i] = np.frombuffer(v, np.uint8)
    elif pa.types.is_float16(t):
        rows = np.asarray(col.fill_null(0)).astype(np.float16).view(np.uint8).reshape(n, 2).copy()
    else:
        rows = np.asarray(col.fill_null(0)).view(np.uint8).reshape(n, width).copy()
    rows[~valid] = 0
    return rows, valid
