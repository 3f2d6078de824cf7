"""The Python restatement of the BOOLEAN / fixed-width decoders (tests/pq_fixed_ref.py) pinned against pq.read_table on
pyarrow-written files, against its own encoders and error cases; and the new header constants against parquet.thrift."""
import itertools
import re
import zlib

import numpy as np
import pytest

import pq_files as F
import pq_fixed_ref as X
import pq_pages as P
import pq_ref as R
from pq_chunk import read_chunk_oracle
from arrow_go_b200 import _native as N


def write_and_read(path, rng, kind, nf, version, n, **kw):
    """write one fixed-width case, read it back through the oracle -> (plan, values, validity, table)"""
    tbl = F.write_column(path, F.make_array(rng, kind, n, nf), nullable=nf is not None, encoding=F.KINDS[kind], version=version, **kw)
    plan = P.chunk_plan(path)
    return (plan, *read_chunk_oracle(plan, P.host_decompress(plan)), tbl)


CASES = [(k, nf, v) for k, nf, v in itertools.product(F.KINDS, F.FIXED_NULL_FRACS, F.PAGE_VERSIONS)]


@pytest.mark.parametrize("case", CASES, ids=F.case_id)
def test_oracle_matches_pyarrow(case, tmp_path):
    kind, nf, ver = case
    rng = np.random.default_rng(zlib.crc32(F.case_id(case).encode()))
    plan, values, valid, tbl = write_and_read(str(tmp_path / "c.parquet"), rng, kind, nf, ver, 600 if kind == "fsb1000" else 3000,
                                              data_page_size=512)
    encs = P.encodings(plan)
    if kind == "bool":
        assert encs == ({X.PLAIN} if ver == "1.0" else {X.RLE})
    elif F.KINDS[kind] == "BYTE_STREAM_SPLIT":
        assert encs == {X.BYTE_STREAM_SPLIT}
    want, wvalid = F.expected(tbl, plan)
    assert np.array_equal(valid, wvalid)
    assert values == want


@pytest.mark.parametrize("kind", ["fsb16_dict", "int96_dict"])
def test_oracle_dictionary_fallback_chunk(kind, tmp_path):
    rng = np.random.default_rng(7)
    plan, values, valid, tbl = write_and_read(str(tmp_path / "c.parquet"), rng, kind, 0.1, "1.0", 20_000, data_page_size=4096,
                                              dictionary_pagesize_limit=1024)
    encs = P.encodings(plan)
    assert plan["dict"] and X.PLAIN in encs and (X.RLE_DICTIONARY in encs or X.PLAIN_DICTIONARY in encs)
    want, wvalid = F.expected(tbl, plan)
    assert np.array_equal(valid, wvalid)
    assert values == want


def test_round_trips_and_run_forms():
    rng = np.random.default_rng(3)
    bits = rng.random(5000) < 0.3
    for enc, page in ((X.PLAIN, X.bool_plain_encode(bits)), (X.RLE, X.bool_rle_encode(bits))):
        out, slots, msg = X.bool_decode(enc, page, bits.size)
        assert msg is None and slots == bits.size and out.tolist() == bits.astype(np.uint8).tolist()
    # every run form: repeated runs of 0, 1 and a non-0/1 byte (true), a literal run, a padded last group
    s = R.repeated_run(0, 9, 1) + R.repeated_run(1, 3, 1) + R.repeated_run(2, 4, 1) + R.literal_run([1, 0, 1], 1)
    out, slots, msg = X.bool_decode(X.RLE, len(s).to_bytes(4, "little") + s, 19)
    assert msg is None and out.tolist() == [0] * 9 + [1] * 7 + [1, 0, 1]
    rows = rng.integers(0, 256, (777, 13), dtype=np.uint8)
    out, slots, msg, _ = X.fixed_decode(X.FLBA, 13, X.BYTE_STREAM_SPLIT, X.bss_encode(rows), 777)
    assert msg is None and out.tobytes() == rows.tobytes()
    valid = np.zeros(1000, bool)
    valid[np.sort(rng.choice(1000, 777, replace=False))] = True
    out, slots, msg, _ = X.fixed_decode(X.FLBA, 13, X.BYTE_STREAM_SPLIT, X.bss_encode(rows), valid)
    assert msg is None and slots == 1000 and out[valid].tobytes() == rows.tobytes() and not out[~valid].any()


def test_error_messages():
    assert X.bool_decode(X.PLAIN, b"\xff", 9)[2] == X.MSG_BOOL_SHORT.format(8, 9)
    assert X.bool_decode(X.RLE, b"\x01\x00", 3)[2] == X.MSG_BOOL_LENGTH.format(2)
    assert X.bool_decode(X.RLE, b"\x10\0\0\0\x01", 3)[2] == X.MSG_BOOL_BYTES.format(16)
    out, slots, msg = X.bool_decode(X.RLE, X.bool_rle_encode([1] * 20), 30)
    assert (slots, msg) == (20, X.MSG_UNEXPECTED_EOF)
    assert X.fixed_decode(X.INT32, 4, X.BYTE_STREAM_SPLIT, bytes(16), 1)[2] == X.MSG_BSS_SIZE.format(16, 1)
    assert X.fixed_decode(X.INT32, 4, X.BYTE_STREAM_SPLIT, bytes(6), 2)[2] == X.MSG_BSS_ALIGN.format(6, 4)
    assert X.fixed_decode(X.FLBA, 4, X.BYTE_STREAM_SPLIT, bytes(6), 2)[2] == X.MSG_BSS_ALIGN_FLBA.format(6, 4)
    assert X.fixed_decode(X.DOUBLE, 8, X.BYTE_STREAM_SPLIT, bytes(16), np.ones(3, bool))[2] == X.MSG_BSS_SHORT
    assert X.fixed_decode(X.INT96, 12, X.PLAIN, bytes(20), 2)[2] == \
        "parquet: eof exception decode plain INT96, nvals: 2, nbytes: 24, datalen: 20"
    assert X.fixed_decode(X.FLBA, 3, X.PLAIN, bytes(5), 2)[2] == X.MSG_EOF
    assert X.fixed_decode(X.INT64, 8, X.PLAIN, bytes(5), 1)[2] == X.MSG_PLAIN_SHORT


def test_enums_match_parquet_thrift():
    # parquet/internal/gen-go/parquet/parquet.go:37-46 (Type) and :445-457 (Encoding), generated from parquet.thrift
    assert (N.PQ_TYPE_INT32, N.PQ_TYPE_INT64, N.PQ_TYPE_INT96, N.PQ_TYPE_FLOAT, N.PQ_TYPE_DOUBLE, N.PQ_TYPE_FIXED_LEN_BYTE_ARRAY) == (1, 2, 3, 4, 5, 7)
    assert (N.PQ_ENC_PLAIN, N.PQ_ENC_PLAIN_DICTIONARY, N.PQ_ENC_RLE, N.PQ_ENC_RLE_DICTIONARY, N.PQ_ENC_BYTE_STREAM_SPLIT) == (0, 2, 3, 8, 9)
    assert (X.INT32, X.INT64, X.INT96, X.FLOAT, X.DOUBLE, X.FLBA) == (1, 2, 3, 4, 5, 7)
    text = open(N.HEADER_PATH).read()
    for name, val in (("AG_PQ_ENC_RLE", 3), ("AG_PQ_ENC_BYTE_STREAM_SPLIT", 9), ("AG_PQ_TYPE_INT32", 1), ("AG_PQ_TYPE_INT64", 2),
                      ("AG_PQ_TYPE_INT96", 3), ("AG_PQ_TYPE_FLOAT", 4), ("AG_PQ_TYPE_DOUBLE", 5), ("AG_PQ_TYPE_FIXED_LEN_BYTE_ARRAY", 7)):
        assert re.search(rf"#define {name}\s+{val}\b", text), name
