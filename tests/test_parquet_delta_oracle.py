"""The Python restatement of the DELTA_BINARY_PACKED encoder and decoder (tests/pq_delta_ref.py) against the reference's
literal test vectors (tests/golden/parquet_delta.json) and against pq.read_table on pyarrow-written files, page by page.
CPU only: this pins the oracle the device tests compare with."""
import json
import os
import zlib

import numpy as np
import pytest

import pq_delta_ref as D
import pq_files as F
import pq_pages as P
from pq_chunk import read_chunk_oracle

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "parquet_delta.json")))


def miniblock_widths(page):
    """every width byte of the miniblocks that hold values (checkDeltaBitPackedWidths, encoding_test.go:708-745)"""
    block, pos = D._uvarint(page, 0)
    nmini, pos = D._uvarint(page, pos)
    total, pos = D._uvarint(page, pos)
    _, pos = D._uvarint(page, pos)
    vpm, remaining, widths = block // nmini, total - 1, []
    while remaining > 0:
        _, pos = D._uvarint(page, pos)
        ws, pos = page[pos:pos + nmini], pos + nmini
        for w in ws:
            if remaining <= 0:
                break
            widths.append(w)
            pos += vpm * w // 8
            remaining -= min(vpm, remaining)
    assert pos == len(page)
    return widths


@pytest.mark.parametrize("case", GOLD["decode"], ids=lambda c: c["name"])
def test_decoder_rejects_reference_vectors(case):
    err = getattr(D, "DERR_" + case["error"])
    out, slots, e, msg = D.delta_decode(bytes(case["bytes"]), case["width"], case["num_values"])
    assert e == err and msg == D.DELTA_MESSAGES[err].format(*case["args"]), msg
    # a header error delivers nothing; a chain error keeps the first value (all of these fail in the first miniblock)
    assert slots == (1 if err in (D.DERR_MIN_DELTA32, D.DERR_WIDTH, D.DERR_PAYLOAD) else 0)


@pytest.mark.parametrize("case", GOLD["encode"], ids=lambda c: c["name"])
def test_encoder_matches_reference_bytes(case):
    enc = D.delta_encode(case["values"], case["width"])
    assert list(enc) == case["bytes"]
    out, slots, err, _ = D.delta_decode(enc, case["width"], len(case["values"]))
    assert err == D.DERR_NONE and out.tolist() == case["values"]


@pytest.mark.parametrize("case", GOLD["overflow"], ids=lambda c: c["name"])
def test_wrapped_deltas_round_trip(case):
    vals = case.get("values") or [case["alternate"][i % 2] for i in range(case["n"])]
    enc = D.delta_encode(vals, case["width"])
    widths = miniblock_widths(enc)
    assert widths and max(widths) <= case["max_bit_width"]
    out, slots, err, _ = D.delta_decode(enc, case["width"], len(vals))
    assert err == D.DERR_NONE and slots == len(vals) and out.tolist() == vals


def test_encoder_layout():
    # width bytes of absent miniblocks stay 0, the last miniblock is padded to vpm values
    enc = D.delta_encode(np.arange(40) * 5, 8, 256, 4)              # header, min delta 5, four zero widths, no payload
    assert list(enc) == [128, 2, 4, 40, 0, 10, 0, 0, 0, 0]
    enc = D.delta_encode([0, 3, 1, 7], 4)
    md, pos = D._uvarint(enc, 5)
    assert D._unzigzag(md) == -2 and list(enc[pos:pos + 4]) == [4, 0, 0, 0] and len(enc) == pos + 4 + 16   # deltas - min: 5, 0, 8


def test_lazy_blocks_and_short_pages():
    vals = np.arange(300, dtype=np.int64) * 7
    enc = D.delta_encode(vals, 8)                                  # 128/4: blocks of 128 deltas, 6-byte header
    b1 = len(D.delta_encode(vals[:129], 8))                        # where block 1 starts
    # 129 valid slots need block 0 only: the stream may end right after it
    valid = np.zeros(300, bool)
    valid[:129] = True
    out, slots, err, _ = D.delta_decode(enc[:b1], 8, valid)
    assert err == D.DERR_NONE and slots == 300 and out[:129].tolist() == vals[:129].tolist() and not out[129:].any()
    # the width bytes of unused trailing miniblocks are not looked at
    enc140 = bytearray(D.delta_encode(vals[:140], 8))
    w0 = D._uvarint(enc140, b1)[1]                                 # block 1's width bytes, after its min delta
    enc140[w0 + 1:w0 + 4] = b"\xff\xff\xff"
    out, slots, err, _ = D.delta_decode(bytes(enc140), 8, 140)
    assert err == D.DERR_NONE and out.tolist() == vals[:140].tolist()
    # dense, total < num_values: a short count, not an error; spaced: an error and nothing written
    out, slots, err, _ = D.delta_decode(enc, 8, 400)
    assert err == D.DERR_NONE and slots == 300 and out.tolist() == vals.tolist()
    out, slots, err, msg = D.delta_decode(enc, 8, np.ones(400, bool))
    assert err == D.DERR_SHORT and slots == 0 and "did not match" in msg
    # total 0 and num_values 0
    assert D.delta_decode(D.delta_encode([], 4), 4, 5)[1:3] == (0, D.DERR_NONE)
    assert D.delta_decode(D.delta_encode([], 4), 4, 0)[1:3] == (0, D.DERR_NONE)
    assert D.delta_decode(b"\x00", 4, 0)[2] == D.DERR_ZERO_BLOCK        # the header is parsed even when nothing is needed


def test_chain_error_keeps_earlier_miniblocks():
    vals = np.arange(200, dtype=np.int64) ** 2
    enc = bytearray(D.delta_encode(vals, 8))
    enc[6 + 1 + 2] = 70                                            # 6-byte header, min delta: block 0, miniblock 2 gets width 70
    out, slots, err, msg = D.delta_decode(bytes(enc), 8, 200)
    assert err == D.DERR_WIDTH and msg.endswith("delta bit width 70 exceeds decoder width 64")
    assert slots == 1 + 2 * 32 and out.tolist() == vals[:65].tolist()
    valid = np.zeros(400, bool)
    valid[1::2] = True
    out, slots, err, _ = D.delta_decode(bytes(enc), 8, valid)
    assert err == D.DERR_WIDTH and slots == 2 * 65 + 1 and out[1::2].tolist() == vals[:65].tolist() and not out[0::2].any()


@pytest.mark.parametrize("case", F.delta_cases(), ids=F.case_id)
def test_oracle_decodes_pyarrow_delta_files(case, tmp_path):
    t, nf, v, ps = case
    rng = np.random.default_rng(zlib.crc32(F.case_id(case).encode()))
    path = str(tmp_path / "c.parquet")
    tbl = F.write_numeric_case(path, rng, ("delta",) + case + (None,))
    plan = P.chunk_plan(path)
    dst = P.host_decompress(plan)
    values, valid = read_chunk_oracle(plan, dst)
    want, wvalid = F.expected(tbl, plan)
    assert P.encodings(plan) == {P.DELTA_BINARY_PACKED} and plan["dict"] is None
    assert np.array_equal(valid, wvalid)
    assert values == want
    if ps and nf != 1.0:
        assert len(plan["pages"]) > 3
    # pyarrow's block shape: 128/4 for INT32, 256/4 for INT64
    _, (b, ln, nv, o) = P.value_sections(plan, dst)[0]
    block, pos = D._uvarint(dst, b)
    assert (block, dst[pos]) == ((128 if t == "int32" else 256), 4)
