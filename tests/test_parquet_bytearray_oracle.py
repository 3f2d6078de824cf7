"""The Python restatement of the BYTE_ARRAY decoders (tests/pq_bytearray_ref.py) pinned against pq.read_table on
pyarrow-written files, and against its own encoders and error cases."""
import json
import os
import zlib

import numpy as np
import pytest

import pq_bytearray_ref as B
import pq_files as F
import pq_pages as P
from pq_chunk import read_chunk_oracle


def write_and_read(path, rng, enc, nf, version, n, **kw):
    """write one string case, read it back through the oracle -> (plan, values, validity, table)"""
    tbl = F.write_column(path, F.make_string_column(rng, enc, n, nf), nullable=nf is not None, encoding=enc, version=version, **kw)
    plan = P.chunk_plan(path)
    return (plan, *read_chunk_oracle(plan, P.host_decompress(plan)), tbl)


@pytest.mark.parametrize("case", F.ba_cases(), ids=F.case_id)
def test_oracle_matches_pyarrow(case, tmp_path):
    enc, nf, ver, ps = case
    rng = np.random.default_rng(zlib.crc32(F.case_id(case).encode()))
    plan, values, valid, tbl = write_and_read(str(tmp_path / "c.parquet"), rng, enc, nf, ver, 5000, data_page_size=ps)
    assert P.encodings(plan) <= {B.PLAIN, B.PLAIN_DICTIONARY, B.RLE_DICTIONARY, B.DELTA_LENGTH_BYTE_ARRAY, B.DELTA_BYTE_ARRAY}
    want, wvalid = F.expected(tbl, plan)
    assert np.array_equal(valid, wvalid)
    assert values == want


def test_oracle_dictionary_fallback_chunk(tmp_path):
    rng = np.random.default_rng(5)
    plan, values, valid, tbl = write_and_read(str(tmp_path / "c.parquet"), rng, "RLE_DICTIONARY", 0.1, "1.0", 30_000,
                                              dictionary_pagesize_limit=2048)
    encs = P.encodings(plan)
    assert plan["dict"] and B.PLAIN in encs and (B.RLE_DICTIONARY in encs or B.PLAIN_DICTIONARY in encs)
    want, wvalid = F.expected(tbl, plan)
    assert np.array_equal(valid, wvalid)
    assert values == want


@pytest.mark.parametrize("enc", [B.PLAIN, B.DELTA_LENGTH_BYTE_ARRAY, B.DELTA_BYTE_ARRAY])
def test_round_trip(enc):
    rng = np.random.default_rng(enc)
    vals = F.random_strings(rng, 3000) + [b"", b"x" * 20_000] + F.random_strings(rng, 500, sorted_keys=True)
    page = {B.PLAIN: B.plain_encode, B.DELTA_LENGTH_BYTE_ARRAY: B.dlba_encode, B.DELTA_BYTE_ARRAY: B.dba_encode}[enc](vals)
    out, slots, msg, _ = B.decode(enc, page, len(vals))
    assert msg is None and slots == len(vals) and out == vals
    valid = np.zeros(len(vals) + 50, bool)
    valid[np.sort(rng.choice(valid.size, len(vals), replace=False))] = True
    got, slots, msg, _ = B.decode(enc, page, valid)
    assert msg is None and slots == valid.size and [got[i] for i in np.flatnonzero(valid)] == vals


def test_error_messages():
    assert B.plain_decode(b"\x05\0\0\0ab", 1)[2] == B.MSG_EOF
    assert B.plain_decode(b"\xff\xff\xff\xff", 1)[2] == B.MSG_NEG_PLAIN
    out, slots, msg = B.plain_decode(B.plain_encode([b"a", b"bc"]) + b"\x01", 3)
    assert (out, slots, msg) == ([b"a", b"bc"], 2, B.MSG_EOF)
    assert B.plain_decode(B.plain_encode([b"a"]) + b"junk", 1)[2] is None
    import pq_delta_ref as D
    assert B.dlba_decode(D.delta_encode([1, -2], 4) + b"x", 2)[2] == B.MSG_NEG_LEN.format(-2)
    assert B.dlba_decode(D.delta_encode([1, 2], 4) + b"xy", 2)[2] == B.MSG_EXCEED
    assert B.dba_decode(D.delta_encode([1, 0], 4) + B.dlba_encode([b"a", b"b"]), 2)[2] == B.MSG_FIRST
    out, slots, msg = B.dba_decode(D.delta_encode([0, 1, 3], 4) + B.dlba_encode([b"ab", b"c", b"d"]), 3)
    assert (out, slots, msg) == ([b"ab", b"ac"], 2, B.MSG_PREFIX.format(3))
    assert B.dba_decode(D.delta_encode([0], 4) + B.dlba_encode([b"a", b"b"]), 2)[2] == B.MSG_COUNT


GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "parquet_bytearray.json")))


@pytest.mark.parametrize("case", GOLD["cases"], ids=lambda c: c["name"])
def test_reference_vectors(case):
    import pq_delta_ref as D
    page = bytes(case["bytes"])
    if "prefixes" in case:                                       # the page is what the reference's encoders produce
        assert page == D.delta_encode(case["prefixes"], 4) + B.dlba_encode([s.encode() for s in case["suffixes"]])
    vals, slots, msg, _ = B.decode(case["encoding"], page, case["num_values"])
    assert msg == case["error"]
    assert vals == [v.encode() for v in case["values"]] and slots == len(case["values"])
