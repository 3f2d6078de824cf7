"""Pins the Snappy restatement in tests/snappy_ref.py against pyarrow's C++ Snappy in both directions: the restatement
decodes pyarrow's encodings, pyarrow decodes every form the restatement's encoder emits, and every corrupt row of the
restatement is also rejected by pyarrow.  CPU only."""
import numpy as np
import pyarrow as pa
import pytest

import snappy_ref as S


def pa_decompress(buf, n):
    return pa.decompress(buf, decompressed_size=n, codec="snappy", asbytes=True)


def samples():
    rng = np.random.default_rng(51)
    ts = (np.cumsum(rng.integers(0, 1000, 4000)) + (1 << 40)).astype(np.int64).tobytes()
    return {
        "empty": b"",
        "one": b"\x07",
        "random": rng.integers(0, 256, 70_000, dtype=np.uint8).tobytes(),
        "zeros": bytes(100_000),
        "repetitive": (b"parquet-snappy " * 5000)[:70_001],
        "timestamps": ts,
        "dict_indices": (rng.integers(0, 100_000, 8000) & 0x1FFFF).astype(np.uint32).tobytes(),
    }


@pytest.mark.parametrize("name", list(samples()))
def test_restatement_decodes_pyarrow(name):
    x = samples()[name]
    out, err, pre = S.decode(pa.compress(x, codec="snappy", asbytes=True), len(x))
    assert err == S.OK and pre == len(x) and out == x


def forms():
    """(name, stream, expected output) covering every element form"""
    rng = np.random.default_rng(52)
    big = rng.integers(0, 256, 70_000, dtype=np.uint8).tobytes()
    far = big + big[:100]                                       # a copy 70 000 bytes back: copy-4
    out = [
        ("inline_literals", S.encode(b"abcdefgh" * 3 + bytes(range(40)), lit_bytes=0)),
        ("literal_1_byte_length", S.stream(200, [S.literal(big[:200], 1)])),
        ("literal_2_byte_length", S.stream(300, [S.literal(big[:300], 2)])),
        ("literal_3_byte_length", S.stream(70_000, [S.literal(big, 3)])),
        ("literal_4_byte_length", S.stream(61, [S.literal(big[:61], 4)])),
        ("literal_1_byte_length_short", S.stream(5, [S.literal(big[:5], 1)])),
        ("copy_1", S.stream(20, [S.literal(b"0123456789"), S.copy(10, 10, 1)])),
        ("copy_2", S.stream(74, [S.literal(b"0123456789"), S.copy(10, 64, 2)])),
        ("copy_4", S.stream(74, [S.literal(b"0123456789"), S.copy(10, 64, 4)])),
        ("offset_1_run", S.stream(1 + 64 * 3, [S.literal(b"z"), S.copy(1, 64, 2), S.copy(1, 64, 4), S.copy(64, 64, 2)])),
        ("overlap_offset_3", S.stream(3 + 11, [S.literal(b"abc"), S.copy(3, 11, 1)])),
        ("copy_of_length_1", S.stream(2, [S.literal(b"q"), S.copy(1, 1, 2)])),
        ("offset_beyond_64k", S.encode(far)),
        ("greedy_copy_2_only", S.encode(b"hello hello hello world " * 40, copy_form=2)),
        ("greedy_copy_4_only", S.encode(b"hello hello hello world " * 40, copy_form=4)),
        ("greedy_literal_4_bytes", S.encode(big[:5000] + big[:5000], lit_bytes=4)),
        ("empty_stream", S.stream(0, [])),
    ]
    return [(n, s, S.decode(s)[0]) for n, s in out]


@pytest.mark.parametrize("case", forms(), ids=lambda c: c[0])
def test_pyarrow_decodes_every_form(case):
    name, s, x = case
    out, err, pre = S.decode(s, len(x))
    assert err == S.OK and out == x
    assert pa_decompress(s, len(x)) == x
    if name == "offset_beyond_64k":
        assert any(b & 3 == 3 for b in _tags(s)), "no copy-4 element"


def _tags(s):
    """the tag bytes of a valid stream"""
    _, s_ = S.uvarint(s)
    out = []
    while s_ < len(s):
        t = s[s_]
        out.append(t)
        if t & 3 == 0:
            x = t >> 2
            nb = 0 if x < 60 else x - 59
            n = (x if x < 60 else int.from_bytes(s[s_ + 1:s_ + 1 + nb], "little")) + 1
            s_ += 1 + nb + n
        else:
            s_ += (0, 2, 3, 5)[t & 3]
    return out


def corrupt_rows():
    """(name, stream, dst_len, bytes the restatement delivers)"""
    ok = S.literal(b"0123456789")
    return [
        ("no_preamble", b"", 5, 0),
        ("preamble_cut", b"\x80", 5, 0),
        ("preamble_over_10_bytes", b"\xff" * 10 + b"\x01", 5, 0),
        ("preamble_over_32_bits", S.put_uvarint(1 << 32), 1 << 32, 0),
        ("literal_length_cut", S.stream(20, [ok, b"\xf0"]), 20, 10),
        ("literal_4_length_cut", S.stream(20, [ok, b"\xfc\x01\x00"]), 20, 10),
        ("literal_bytes_cut", S.stream(20, [ok, S.literal(b"abcdefghij")[:-1]]), 20, 10),
        ("literal_past_output", S.stream(15, [ok, S.literal(b"abcdefghij")]), 15, 10),
        ("copy_1_offset_cut", S.stream(20, [ok, S.copy(10, 10, 1)[:1]]), 20, 10),
        ("copy_2_offset_cut", S.stream(20, [ok, S.copy(10, 10, 2)[:2]]), 20, 10),
        ("copy_4_offset_cut", S.stream(20, [ok, S.copy(10, 10, 4)[:4]]), 20, 10),
        ("copy_offset_0", S.stream(20, [ok, S.copy(0, 10, 2)]), 20, 10),
        ("copy_offset_past_output", S.stream(30, [ok, S.copy(11, 10, 2)]), 30, 10),
        ("copy_past_output", S.stream(15, [ok, S.copy(10, 10, 2)]), 15, 10),
        ("stream_ends_early", S.stream(30, [ok, S.copy(10, 10, 1)]), 30, 20),
        ("trailing_element", S.stream(20, [ok, S.copy(10, 10, 1), S.literal(b"x")]), 20, 20),
        ("preamble_only", S.stream(7, []), 7, 0),
    ]


@pytest.mark.parametrize("row", corrupt_rows(), ids=lambda r: r[0])
def test_corrupt_rows_rejected_by_both(row):
    name, s, n, delivered = row
    out, err, _ = S.decode(s, n)
    assert err == S.CORRUPT and len(out) == delivered
    if n < 1 << 32:
        with pytest.raises(OSError, match="Corrupt snappy compressed data"):
            pa_decompress(s, n)


def test_size_mismatch_is_checked_before_the_body():
    s = S.stream(20, [S.literal(b"0123456789"), b"\xf0"])    # corrupt body, preamble 20
    assert S.decode(s, 21) == (b"", S.SIZE, 20)
    assert S.decode(b"", 0) == (b"", S.OK, 0)
    assert S.decode(b"", 1)[1] == S.CORRUPT
