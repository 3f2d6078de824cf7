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


@pytest.mark.parametrize("case", S.forms(), ids=lambda c: c[0])
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


@pytest.mark.parametrize("row", S.corrupt_rows(), ids=lambda r: r[0])
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
