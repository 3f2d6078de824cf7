"""Test helper: pyarrow-written Parquet files with one string column `c` in each BYTE_ARRAY encoding, and the plan that
turns its column chunk into batched page descriptors.  Not product code."""
import itertools

import numpy as np

import pq_pages as P
from pq_files import PAGE_VERSIONS

ENCODINGS = ("PLAIN", "RLE_DICTIONARY", "DELTA_LENGTH_BYTE_ARRAY", "DELTA_BYTE_ARRAY")
NULL_FRACS = (None, 0.1, 1.0)


def random_strings(rng, n, sorted_keys=False, distinct=None):
    """short and empty strings, a few long ones; sorted keys share prefixes"""
    if sorted_keys:
        return [f"key_{k:09d}".encode() for k in np.sort(rng.integers(0, 10 ** 9, n))]
    lens = rng.choice([0, 1, 3, 8, 20, 70], n, p=[0.05, 0.1, 0.25, 0.3, 0.2, 0.1])
    pool = [bytes(rng.integers(97, 123, int(m), dtype=np.uint8)) for m in lens]
    if distinct:
        pool = [pool[i] for i in rng.integers(0, distinct, n)]
    return pool


def write_file(path, rng, encoding, null_frac, version, n=20_000, data_page_size=None, compression="NONE", dictionary_pagesize_limit=None):
    import pyarrow as pa
    import pyarrow.parquet as pq
    vals = random_strings(rng, n, sorted_keys=encoding == "DELTA_BYTE_ARRAY", distinct=300 if encoding == "RLE_DICTIONARY" else None)
    mask = None if null_frac is None else rng.random(n) < null_frac
    field = pa.field("c", pa.binary(), nullable=null_frac is not None)
    tbl = pa.Table.from_arrays([pa.array(vals, type=pa.binary(), mask=mask)], schema=pa.schema([field]))
    kw = {"data_page_size": data_page_size} if data_page_size else {}
    if dictionary_pagesize_limit:
        kw["dictionary_pagesize_limit"] = dictionary_pagesize_limit
    if encoding == "RLE_DICTIONARY":
        pq.write_table(tbl, path, compression=compression, use_dictionary=True, data_page_version=version, **kw)
    else:
        pq.write_table(tbl, path, compression=compression, use_dictionary=False, column_encoding={"c": encoding},
                       data_page_version=version, **kw)
    return tbl


def chunk_plan(path):
    """column 0 of row group 0 (uncompressed):
       data      every page payload back to back
       dict      (data, len, num_values) of the dictionary page or None
       pages     [(encoding, (data, len, num_values, out))] of the data pages' value sections
       n_slots"""
    import pyarrow.parquet as pq
    max_def = pq.ParquetFile(path).schema.column(0).max_definition_level
    pages = P.column_chunk_pages(path)
    blob, base = bytearray(), []
    for pg in pages:
        base.append(len(blob))
        blob += pg["payload"]
        blob += b"\0" * (-len(blob) % 8)
    plan = {"dict": None, "pages": []}
    slot = 0
    for pg, b in zip(pages, base):
        if pg["type"] == P.DICTIONARY_PAGE:
            plan["dict"] = (b, len(pg["payload"]), pg["num_values"])
            continue
        _, _, vo = P.split_data_page(pg, max_def)
        nv = pg["num_values"]
        plan["pages"].append((pg["encoding"], (b + vo, len(pg["payload"]) - vo, nv, slot)))
        slot += nv
    plan["data"] = bytes(blob) + bytes(16)
    plan["n_slots"] = slot
    return plan


def expected(tbl):
    """(values with b"" for nulls, validity) of column 0"""
    col = tbl.column(0).combine_chunks()
    vals = [b"" if v is None else v for v in col.to_pylist()]
    return vals, np.asarray(col.is_valid())


def cases():
    """(encoding, null_frac, version, data_page_size)"""
    return list(itertools.product(ENCODINGS, NULL_FRACS, PAGE_VERSIONS, (None, 4096)))


def case_id(c):
    e, nf, v, ps = c
    return f"{e}-{'req' if nf is None else f'null{int(nf * 100)}'}-v{v[0]}" + (f"-page{ps}" if ps else "")
