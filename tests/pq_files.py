"""Test helper: pyarrow-written Parquet files covering the page shapes the device decoders take (the column makers of
each family, one writer, the case lists and their ids), and what pq.read_table's result stands for in a column
reader's output form.  Not product code."""
import decimal
import itertools

import numpy as np

import pq_fixed_ref as X
import pq_pages as P

PAGE_VERSIONS = ("1.0", "2.0")


def write_column(path, arr, *, nullable, encoding, version, compression="NONE", data_page_size=None,
                 dictionary_pagesize_limit=None):
    """`arr` as column `c` of a one-column file -> the table written.  encoding "RLE_DICTIONARY" writes a dictionary
    (and PLAIN pages once it is full), None the writer's own choice without one, anything else that encoding.  A
    timestamp column is written as INT96."""
    import pyarrow as pa
    import pyarrow.parquet as pq
    tbl = pa.Table.from_arrays([arr], schema=pa.schema([pa.field("c", arr.type, nullable=nullable)]))
    kw = {"use_dictionary": encoding == "RLE_DICTIONARY"}
    if encoding not in (None, "RLE_DICTIONARY"):
        kw["column_encoding"] = {"c": encoding}
    if data_page_size:
        kw["data_page_size"] = data_page_size
    if dictionary_pagesize_limit:
        kw["dictionary_pagesize_limit"] = dictionary_pagesize_limit
    if pa.types.is_timestamp(arr.type):
        kw["use_deprecated_int96_timestamps"] = True
    pq.write_table(tbl, path, compression=compression, data_page_version=version, **kw)
    return tbl


def case_id(c):
    """`name-req|nullNN-vN`, then `-pageN` and `-dictN` when the case sets a page size and a dictionary limit"""
    name, nf, version, *rest = c
    out = f"{name}-{'req' if nf is None else f'null{int(nf * 100)}'}-v{version[0]}"
    for tag, x in zip(("-page", "-dict"), rest):
        out += f"{tag}{x}" if x else ""
    return out


def int96_of_ns(ns):
    """INT96 physical bytes (nanoseconds of the day, then the Julian day, little-endian) of timestamps in ns"""
    ns = np.asarray(ns, np.int64)
    day, nod = np.divmod(ns, 86_400_000_000_000)
    out = np.zeros((ns.size, 12), np.uint8)
    out[:, :8] = nod.astype("<i8").view(np.uint8).reshape(-1, 8)
    out[:, 8:] = (day + 2440588).astype("<u4").view(np.uint8).reshape(-1, 4)
    return out


def expected(tbl, plan):
    """(values, validity) of column 0 in the column reader's output form: b"" per null slot and the bytes of every
    other slot for BYTE_ARRAY; otherwise the physical bytes of every slot, zero bytes for a null one (BOOLEAN: one
    0 / 1 byte per slot)"""
    import pyarrow as pa
    col = tbl.column(0).combine_chunks()
    valid = np.asarray(col.is_valid())
    n = len(col)
    if plan["ptype"] == P.BYTE_ARRAY:
        return [b"" if v is None else v for v in col.to_pylist()], valid
    if plan["ptype"] == P.BOOLEAN:
        return np.asarray(col.fill_null(False)).astype(np.uint8).tobytes(), valid
    width = X.width_of(plan["ptype"], plan["type_length"])
    t = col.type
    if pa.types.is_timestamp(t):
        rows = int96_of_ns(np.asarray(col.cast(pa.int64()).fill_null(0)))
    elif pa.types.is_decimal(t):
        rows = np.zeros((n, width), np.uint8)
        for i, v in enumerate(col.to_pylist()):
            if v is not None:
                rows[i] = np.frombuffer(int(v.scaleb(t.scale)).to_bytes(width, "big", signed=True), np.uint8)
    elif pa.types.is_fixed_size_binary(t):
        rows = np.zeros((n, width), np.uint8)
        for i, v in enumerate(col.to_pylist()):
            if v is not None:
                rows[i] = np.frombuffer(v, np.uint8)
    else:
        rows = np.asarray(col.fill_null(0)).view(np.uint8).reshape(n, width).copy()
    rows[~valid] = 0
    return rows.tobytes(), valid


# ----------------------------------------------------------------- INT32 / INT64 / FLOAT / DOUBLE, dictionary + PLAIN
TYPES = ("int32", "int64", "float", "double")
NULL_FRACS = (None, 0.0, 0.1, 1.0)     # None = required column
NP_OF = {"int32": np.int32, "int64": np.int64, "float": np.float32, "double": np.float64}


def make_column(rng, type_name, n, null_frac, distinct):
    import pyarrow as pa
    at = {"int32": pa.int32(), "int64": pa.int64(), "float": pa.float32(), "double": pa.float64()}[type_name]
    pool = rng.integers(-(1 << 30), 1 << 30, distinct)
    vals = pool[rng.integers(0, distinct, n)]
    # some long repeats so that both run kinds occur
    for s in rng.integers(0, n, 8):
        vals[s:s + 300] = vals[s]
    arr = np.asarray(vals).astype(NP_OF[type_name])
    mask = None if null_frac is None else rng.random(n) < null_frac
    return pa.array(arr, type=at, mask=mask), at


def cases():
    """(type, null_frac, version, data_page_size, dict_limit): every type x nullability x page version at the
    default page size, plus many small pages and a dictionary limit small enough to force PLAIN fallback pages"""
    out = [(t, nf, v, None, None) for t, nf, v in itertools.product(TYPES, NULL_FRACS, PAGE_VERSIONS)]
    out += [(t, nf, v, 2048, None) for t, nf, v in itertools.product(("int64", "float"), (None, 0.1), PAGE_VERSIONS)]
    out += [(t, nf, v, 4096, 512) for t, nf, v in itertools.product(TYPES, (None, 0.1), PAGE_VERSIONS)]
    return out


# ------------------------------------------------------------------------------- DELTA_BINARY_PACKED INT32 / INT64
# columns: INT32 / INT64, required / 10 % / 100 % nulls, both page versions, default and small pages
DELTA_TYPES = ("int32", "int64")
DELTA_NULL_FRACS = (None, 0.1, 1.0)


def make_delta_column(rng, type_name, n, null_frac):
    """sorted timestamps-like runs with some random jumps (both wide and narrow miniblocks)"""
    import pyarrow as pa
    hi = (1 << 31) - 1 if type_name == "int32" else (1 << 62)
    vals = np.cumsum(rng.integers(0, 1000, n)) - (1 << 20)
    jumps = rng.integers(0, n, 20)
    vals[jumps] = rng.integers(-hi, hi, jumps.size)
    mask = None if null_frac is None else rng.random(n) < null_frac
    return pa.array(vals.astype(NP_OF[type_name]), mask=mask)


def delta_cases():
    """(type, null_frac, version, data_page_size)"""
    return [(t, nf, v, ps) for t, nf, v, ps in itertools.product(DELTA_TYPES, DELTA_NULL_FRACS, PAGE_VERSIONS, (None, 2048))]


def compressed_cases():
    """cases() shapes (dictionary / PLAIN fallback) plus DELTA_BINARY_PACKED files, v1 and v2, for every codec"""
    return [("dict",) + c for c in cases()] + [("delta",) + c + (None,) for c in delta_cases()]


def compressed_case_id(c):
    return c[0] + "-" + case_id(c[1:])


def write_numeric_case(path, rng, case, compression="NONE"):
    """the file of one compressed_cases() row -> the table written"""
    kind, t, nf, v, ps, dl = case
    if kind == "dict":
        arr, enc = make_column(rng, t, 20_000, nf, 300)[0], "RLE_DICTIONARY"
    else:
        arr, enc = make_delta_column(rng, t, 20_000, nf), "DELTA_BINARY_PACKED"
    return write_column(path, arr, nullable=nf is not None, encoding=enc, version=v, compression=compression,
                        data_page_size=ps, dictionary_pagesize_limit=dl)


# ------------------------------------------------------------------------------------------------------ BYTE_ARRAY
BA_ENCODINGS = ("PLAIN", "RLE_DICTIONARY", "DELTA_LENGTH_BYTE_ARRAY", "DELTA_BYTE_ARRAY")
BA_NULL_FRACS = (None, 0.1, 1.0)


def random_strings(rng, n, sorted_keys=False, distinct=None):
    """short and empty strings, a few long ones; sorted keys share prefixes"""
    if sorted_keys:
        return [f"key_{k:09d}".encode() for k in np.sort(rng.integers(0, 10 ** 9, n))]
    lens = rng.choice([0, 1, 3, 8, 20, 70], n, p=[0.05, 0.1, 0.25, 0.3, 0.2, 0.1])
    pool = [bytes(rng.integers(97, 123, int(m), dtype=np.uint8)) for m in lens]
    if distinct:
        pool = [pool[i] for i in rng.integers(0, distinct, n)]
    return pool


def make_string_column(rng, encoding, n, null_frac):
    """binary values suited to `encoding`: sorted keys for DELTA_BYTE_ARRAY, 300 distinct ones for a dictionary"""
    import pyarrow as pa
    vals = random_strings(rng, n, sorted_keys=encoding == "DELTA_BYTE_ARRAY", distinct=300 if encoding == "RLE_DICTIONARY" else None)
    mask = None if null_frac is None else rng.random(n) < null_frac
    return pa.array(vals, type=pa.binary(), mask=mask)


def ba_cases():
    """(encoding, null_frac, version, data_page_size)"""
    return list(itertools.product(BA_ENCODINGS, BA_NULL_FRACS, PAGE_VERSIONS, (None, 4096)))


# ------------------------------------------------------------- BOOLEAN, FIXED_LEN_BYTE_ARRAY, INT96, BYTE_STREAM_SPLIT
FIXED_NULL_FRACS = (None, 0.0, 0.1, 1.0)
# kind -> encoding (None: the writer's own, PLAIN in v1 pages and RLE in v2 pages): every flat kind the fixed decoders take
KINDS = {
    "bool": None, "fsb1": "PLAIN", "fsb3": "PLAIN", "fsb12": "PLAIN", "fsb16": "PLAIN", "fsb1000": "PLAIN",
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
