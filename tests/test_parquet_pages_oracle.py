"""The Python restatement of the Parquet page decoders (tests/pq_ref.py) against the reference's literal test vectors
(tests/golden/parquet_rle.json) and against pq.read_table on pyarrow-written files, page by page.  CPU only: this pins
the oracle the device tests compare with."""
import json
import os
import zlib

import numpy as np
import pytest

import pq_files as F
import pq_pages as P
import pq_ref as R
from pq_chunk import read_chunk_oracle

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "parquet_rle.json")))


@pytest.mark.parametrize("case", GOLD["rle_encode"], ids=lambda c: c["name"])
def test_encoder_matches_reference_vectors(case):
    for w in case["widths"]:
        enc = R.rle_encode(case["values"], w)
        if "bytes" in case:
            assert list(enc) == case["bytes"], w
        elif case["length"] == "2*(1+ceil(w/8))":
            assert len(enc) == 2 * (1 + (w + 7) // 8), w
        else:
            assert len(enc) == 1 + (w * 104 + 7) // 8, w
        vals, err = R.rle_decode(enc, w, len(case["values"]))
        assert err == R.ERR_NONE and vals.tolist() == case["values"], w


@pytest.mark.parametrize("case", GOLD["rle_decode"], ids=lambda c: c["name"])
def test_decoder_matches_reference_vectors(case):
    vals, err = R.rle_decode(bytes(case["bytes"]), case["width"], case["num_values"])
    assert vals.size == case["decoded"] and (vals == case["value"]).all()
    assert (err != R.ERR_NONE) == case["error"]


@pytest.mark.parametrize("case", GOLD["levels"], ids=lambda c: c["name"])
def test_levels_match_reference_vectors(case):
    if "bytes" in case:
        lv, err = R.levels_decode_page(bytes(case["bytes"]), case["max_level"], case["v1"], case["num_values"])
        assert lv.size == case["decoded"] and (lv == case["value"]).all() and (err != R.ERR_NONE) == case["error"]
        return
    levels = case["levels"]
    bw = case["max_level"].bit_length()
    enc = R.rle_encode(levels, bw)
    page = len(enc).to_bytes(4, "little") + enc
    lv, err = R.levels_decode_page(page, case["max_level"], True, len(levels))
    assert err == R.ERR_NONE and lv.tolist() == levels
    lv, err = R.levels_decode_page(enc, case["max_level"], False, len(levels))
    assert err == R.ERR_NONE and lv.tolist() == levels


def test_encoder_round_trip_random():
    rng = np.random.default_rng(11)
    for bw in range(0, 33):
        for shape in ("random", "runs", "alternating"):
            n = int(rng.integers(1, 3000))
            hi = 1 << bw
            if shape == "random":
                v = rng.integers(0, hi, n, dtype=np.uint64) if bw else np.zeros(n, np.uint64)
            elif shape == "runs":
                v = np.repeat(rng.integers(0, hi, n // 20 + 1, dtype=np.uint64), rng.integers(1, 40, n // 20 + 1))[:n]
            else:
                v = (np.arange(n) % 2).astype(np.uint64) & np.uint64(hi - 1)
            enc = R.rle_encode(v.tolist(), bw)
            got, err = R.rle_decode(enc, bw, v.size)
            assert err == R.ERR_NONE and np.array_equal(got, v), (bw, shape)


def test_error_cases():
    assert R.rle_decode(b"\x00", 8, 4)[1] == R.ERR_ZERO_RUN
    assert R.rle_decode(b"\x01", 8, 4)[1] == R.ERR_ZERO_RUN
    assert R.rle_decode(b"\x80\x80", 8, 4)[1] == R.ERR_VARINT
    assert R.rle_decode(b"\x81\x80\x80\x80\x80\x01", 8, 4)[1] == R.ERR_VARINT
    assert R.rle_decode(b"\x08\x01", 16, 4)[1] == R.ERR_TRUNC_REPEATED
    assert R.levels_decode_page(b"\x01\x00", 1, True, 4)[1] == R.ERR_LEVELS_SHORT
    assert R.levels_decode_page(b"\x09\x00\x00\x00\x02\x01", 1, True, 4)[1] == R.ERR_LEVELS_LENGTH
    d = np.arange(4, dtype=np.int64)
    assert R.dict_decode(b"\x21\x02\x00", d, 1)[2] == R.ERR_BIT_WIDTH
    out, slots, err, bad = R.dict_decode(b"\x03" + R.literal_run([1, 0, 2, 0, 6, 0, 0, 0], 3), d, 8)
    assert err == R.ERR_NONE and bad == 4 and out[4] == 0 and slots == 8


@pytest.mark.parametrize("case", F.cases(), ids=F.case_id)
def test_oracle_decodes_pyarrow_files(case, tmp_path):
    rng = np.random.default_rng(zlib.crc32(F.case_id(case).encode()))
    path = str(tmp_path / "c.parquet")
    tbl = F.write_numeric_case(path, rng, ("dict",) + case)
    plan = P.chunk_plan(path)
    values, valid = read_chunk_oracle(plan, P.host_decompress(plan))
    want, wvalid = F.expected(tbl, plan)
    assert np.array_equal(valid, wvalid)
    assert values == want
    if case[3]:
        assert len(plan["pages"]) > 3
    if case[4]:
        assert P.PLAIN in P.encodings(plan), "no PLAIN fallback page was written"
