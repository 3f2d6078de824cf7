"""Test helper: pyarrow-written Parquet files covering the page shapes the device decoders take, and the plan that
turns one column chunk into batched page descriptors (levels / dictionary / PLAIN).  Not product code."""
import itertools

import numpy as np

import pq_pages as P

TYPES = ("int32", "int64", "float", "double")
NULL_FRACS = (None, 0.0, 0.1, 1.0)     # None = required column
PAGE_VERSIONS = ("1.0", "2.0")


def make_column(rng, type_name, n, null_frac, distinct):
    import pyarrow as pa
    at = {"int32": pa.int32(), "int64": pa.int64(), "float": pa.float32(), "double": pa.float64()}[type_name]
    pool = rng.integers(-(1 << 30), 1 << 30, distinct)
    vals = pool[rng.integers(0, distinct, n)]
    # some long repeats so that both run kinds occur
    for s in rng.integers(0, n, 8):
        vals[s:s + 300] = vals[s]
    arr = np.asarray(vals).astype(P.np_of(at))
    mask = None if null_frac is None else rng.random(n) < null_frac
    return pa.array(arr, type=at, mask=mask), at


def write_file(path, rng, type_name, null_frac, version, n=20_000, distinct=300, data_page_size=None, dict_limit=None):
    import pyarrow as pa
    import pyarrow.parquet as pq
    col, at = make_column(rng, type_name, n, null_frac, distinct)
    field = pa.field("c", at, nullable=null_frac is not None)
    tbl = pa.Table.from_arrays([col], schema=pa.schema([field]))
    kw = {}
    if data_page_size:
        kw["data_page_size"] = data_page_size
    if dict_limit:
        kw["dictionary_pagesize_limit"] = dict_limit
    pq.write_table(tbl, path, compression="NONE", use_dictionary=True, data_page_version=version, **kw)
    return tbl


def cases():
    """(type, null_frac, version, data_page_size, dict_limit): every type x nullability x page version at the
    default page size, plus many small pages and a dictionary limit small enough to force PLAIN fallback pages"""
    out = [(t, nf, v, None, None) for t, nf, v in itertools.product(TYPES, NULL_FRACS, PAGE_VERSIONS)]
    out += [(t, nf, v, 2048, None) for t, nf, v in itertools.product(("int64", "float"), (None, 0.1), PAGE_VERSIONS)]
    out += [(t, nf, v, 4096, 512) for t, nf, v in itertools.product(TYPES, (None, 0.1), PAGE_VERSIONS)]
    return out


def case_id(c):
    t, nf, v, ps, dl = c
    return f"{t}-{'req' if nf is None else f'null{int(nf * 100)}'}-v{v[0]}" + (f"-page{ps}" if ps else "") + (f"-dict{dl}" if dl else "")


def chunk_plan(path):
    """Everything the device calls need for column 0 of row group 0:
       data      one bytes object holding every page payload back to back
       dict      (payload offset, num_values) of the dictionary page or None
       levels    [(data, len, num_values, out)] for the levels decode (optional columns)
       dpages    [(data, len, num_values, out)] of dictionary-encoded data pages (value streams)
       ppages    [(data, len, num_values, out)] of PLAIN data pages
       n_slots   total slots;  max_def;  v1"""
    import pyarrow.parquet as pq
    pf = pq.ParquetFile(path)
    max_def = pf.schema.column(0).max_definition_level
    pages = P.column_chunk_pages(path)
    blob, base = bytearray(), []
    for pg in pages:
        base.append(len(blob))
        blob += pg["payload"]
        blob += b"\0" * (-len(blob) % 8)
    plan = {"dict": None, "levels": [], "dpages": [], "ppages": [], "max_def": max_def, "v1": None}
    slot = 0
    for pg, b in zip(pages, base):
        if pg["type"] == P.DICTIONARY_PAGE:
            plan["dict"] = (b, pg["num_values"])
            continue
        lo, ll, vo = P.split_data_page(pg, max_def)
        nv = pg["num_values"]
        plan["v1"] = pg["type"] == P.DATA_PAGE
        if max_def:
            plan["levels"].append((b + lo, ll, nv, slot))
        desc = (b + vo, len(pg["payload"]) - vo, nv, slot)
        if pg["encoding"] in (P.PLAIN_DICTIONARY, P.RLE_DICTIONARY):
            plan["dpages"].append(desc)
        else:
            assert pg["encoding"] == P.PLAIN, pg["encoding"]
            plan["ppages"].append(desc)
        slot += nv
    plan["data"] = bytes(blob)
    plan["n_slots"] = slot
    return plan


def expected(tbl):
    """(values with 0 in null slots, validity) of column 0 as pq.read_table gives it"""
    col = tbl.column(0).combine_chunks()
    valid = np.ones(len(col), bool) if col.null_count == 0 else col.is_valid().to_numpy(zero_copy_only=False)
    dt = col.type.to_pandas_dtype()
    vals = col.fill_null(0).to_numpy(zero_copy_only=False).astype(dt) if len(col) else np.zeros(0, dt)
    vals = np.where(valid, vals, np.zeros(1, dt)).astype(dt)
    return vals, valid
