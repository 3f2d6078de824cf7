"""Test helper: pyarrow-written Parquet files with DELTA_BINARY_PACKED INT32 / INT64 columns, and the plan that turns one
column chunk into batched page descriptors (levels / delta values).  Not product code."""
import itertools

import numpy as np

import pq_pages as P
from pq_files import PAGE_VERSIONS

DELTA_BINARY_PACKED = 5


def delta_chunk_plan(path):
    """Everything the device calls need for column 0 of row group 0:
       data      one bytes object holding every page payload back to back
       levels    [(data, len, num_values, out)] for the levels decode (optional columns)
       delta     [(data, len, num_values, out)] of DELTA_BINARY_PACKED data pages (value sections)
       other     encodings of any other data pages (none in a delta-only chunk)
       n_slots   total slots;  max_def;  v1"""
    import pyarrow.parquet as pq
    max_def = pq.ParquetFile(path).schema.column(0).max_definition_level
    pages = P.column_chunk_pages(path)
    blob, base = bytearray(), []
    for pg in pages:
        base.append(len(blob))
        blob += pg["payload"]
        blob += b"\0" * (-len(blob) % 8)
    plan = {"levels": [], "delta": [], "other": [], "max_def": max_def, "v1": None}
    slot = 0
    for pg, b in zip(pages, base):
        if pg["type"] == P.DICTIONARY_PAGE:
            plan["other"].append(pg["encoding"])
            continue
        lo, ll, vo = P.split_data_page(pg, max_def)
        nv = pg["num_values"]
        plan["v1"] = pg["type"] == P.DATA_PAGE
        if max_def:
            plan["levels"].append((b + lo, ll, nv, slot))
        if pg["encoding"] == DELTA_BINARY_PACKED:
            plan["delta"].append((b + vo, len(pg["payload"]) - vo, nv, slot))
        else:
            plan["other"].append(pg["encoding"])
        slot += nv
    plan["data"] = bytes(blob)
    plan["n_slots"] = slot
    return plan


# columns: INT32 / INT64, required / 10 % / 100 % nulls, both page versions, default and small pages
DELTA_TYPES = ("int32", "int64")
DELTA_NULL_FRACS = (None, 0.1, 1.0)


def write_delta_file(path, rng, type_name, null_frac, version, n=20_000, data_page_size=None):
    """sorted timestamps-like runs with some random jumps (both wide and narrow miniblocks) in one column `c`"""
    import pyarrow as pa
    import pyarrow.parquet as pq
    at = {"int32": pa.int32(), "int64": pa.int64()}[type_name]
    hi = (1 << 31) - 1 if type_name == "int32" else (1 << 62)
    vals = np.cumsum(rng.integers(0, 1000, n)) - (1 << 20)
    jumps = rng.integers(0, n, 20)
    vals[jumps] = rng.integers(-hi, hi, jumps.size)
    arr = vals.astype(P.np_of(at))
    mask = None if null_frac is None else rng.random(n) < null_frac
    field = pa.field("c", at, nullable=null_frac is not None)
    tbl = pa.Table.from_arrays([pa.array(arr, type=at, mask=mask)], schema=pa.schema([field]))
    kw = {"data_page_size": data_page_size} if data_page_size else {}
    pq.write_table(tbl, path, compression="NONE", use_dictionary=False, column_encoding={"c": "DELTA_BINARY_PACKED"},
                   data_page_version=version, **kw)
    return tbl


def delta_cases():
    """(type, null_frac, version, data_page_size)"""
    return [(t, nf, v, ps) for t, nf, v, ps in itertools.product(DELTA_TYPES, DELTA_NULL_FRACS, PAGE_VERSIONS, (None, 2048))]


def delta_case_id(c):
    t, nf, v, ps = c
    return f"{t}-{'req' if nf is None else f'null{int(nf * 100)}'}-v{v[0]}" + (f"-page{ps}" if ps else "")
