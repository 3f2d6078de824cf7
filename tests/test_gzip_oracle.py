"""The GZIP restatement (tests/gzip_ref.py) against zlib and pyarrow: byte for byte on zlib's output at every level and
strategy, on pyarrow's GZIP output and on gzip.compress; every form in REQUIRED met; every corrupt row rejected by zlib
too (or by pyarrow, for trailing bytes); CRC32 pinned; every page of the two parquet-testing GZIP fixtures."""
import collections
import gzip
import os
import zlib

import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import gzip_ref as R
import pq_pages as P

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FIXTURES = ("concatenated_gzip_members.parquet", "byte_stream_split_extended.gzip.parquet")
STRATEGIES = {"default": zlib.Z_DEFAULT_STRATEGY, "filtered": zlib.Z_FILTERED, "huffman_only": zlib.Z_HUFFMAN_ONLY,
              "rle": zlib.Z_RLE, "fixed": zlib.Z_FIXED}

REQUIRED = [
    "member", "multi_member", "empty_member", "fextra", "fname", "fcomment", "fhcrc", "fname_511", "fcomment_511",
    "reserved_flags", "stored", "stored_len_0", "stored_len_65535", "fixed", "dynamic", "len_3", "len_258", "dist_1",
    "dist_32768", "repeat_16_3", "repeat_16_6", "repeat_17_3", "repeat_17_10", "repeat_18_11", "repeat_18_138",
    "single_distance_code", "no_distance_codes", "code_longer_than_10_bits", "code_length_15",
]


def zlib_decode(s):
    """every member through zlib.decompressobj(31); raises on anything zlib refuses, including a truncated member"""
    out = b""
    while True:
        d = zlib.decompressobj(31)
        out += d.decompress(s)
        if not d.eof:
            raise zlib.error("truncated")
        s = d.unused_data
        if not s:
            return out


@pytest.mark.parametrize("strategy", list(STRATEGIES))
@pytest.mark.parametrize("level", range(10))
def test_restatement_matches_zlib(level, strategy):
    x = R.payload(40000 if (level, strategy) == (9, "default") else 12000, level)
    s = R.gz(x, level, STRATEGIES[strategy])
    got, outcome, arg = R.decode(s, len(x))
    assert outcome == R.OK and got == x, (outcome, arg)


def test_restatement_matches_pyarrow_and_gzip_module():
    x = R.payload(30000, 3)
    for s in (pa.compress(x, codec="gzip", asbytes=True), gzip.compress(x), gzip.compress(x, mtime=0, compresslevel=1)):
        got, outcome, arg = R.decode(s, len(x))
        assert outcome == R.OK and got == x, (outcome, arg)


def test_every_form_is_covered():
    seen = collections.Counter()
    x = R.payload(40000, 9)
    R.decode(R.gz(x, 9), len(x), seen)
    for name, s, y in R.forms():
        got, outcome, arg = R.decode(s, len(y), seen)
        assert outcome == R.OK and got == y, (name, outcome, arg)
        if name != "reserved_flags":                             # zlib refuses reserved FLG bits
            assert zlib_decode(s) == y, name
    missing = [f for f in REQUIRED if not seen[f]]
    assert not missing, missing


# Where the restatement follows Go's reader and not zlib: reserved FLG bits are ignored (a form above), a name of 512
# bytes or more is a bad header.  Trailing bytes after a member are refused by pyarrow, not by zlib's one-member
# decompressobj or Python's gzip module (which skips zero padding).
ZLIB_ACCEPTS = ("name_512",)
TRAILING = ("trailing_5_bytes", "zero_padding")


@pytest.mark.parametrize("row", R.corrupt_rows(), ids=lambda r: r[0])
def test_corrupt_rows(row):
    name, s, n, want = row
    got, outcome, arg = R.decode(s, n)
    assert (outcome, arg) == want
    assert len(got) <= n
    if outcome in (R.EXCEED, R.SHORT):
        return
    if name in TRAILING:
        with pytest.raises(Exception):
            pa.decompress(s, decompressed_size=n, codec="gzip", asbytes=True)
    elif name in ZLIB_ACCEPTS:
        zlib_decode(s)
    else:
        with pytest.raises(zlib.error):
            zlib_decode(s)


def test_messages():
    assert R.message(R.SHORT, 0, 5).endswith(": EOF")
    assert R.message(R.SHORT, 3, 5).endswith(": unexpected EOF")
    assert R.message(R.EXCEED, None, 7) == "parquet: could not decompress page: codec: gzip: decoded data exceeds destination size 7"
    assert R.message(R.CORRUPT, "distance", 7) == "parquet: could not decompress page: gzip: distance"
    assert R.decode(b"", 0) == (b"", R.OK, None)


def test_crc32_against_zlib():
    for data in (b"", b"a", bytes(range(256)) * 3, R.payload(10000, 4)):
        assert R.crc32(data) == zlib.crc32(data)
    assert R.crc32(b"123456789") == 0xCBF43926


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_pages_against_pyarrow(name):
    path = os.path.join(GOLDEN, name)
    seen = collections.Counter()
    for c in range(pq.ParquetFile(path).metadata.num_columns):
        chunk, pages = P.column_chunk(path, column=c)
        regions, comp, _ = P.decompress_table(pages)
        assert comp
        for k in comp:
            s, sl, _, dl = regions[k][:4]
            body = bytes(chunk[s:s + sl])
            got, outcome, arg = R.decode(body, dl, seen)
            want = pa.decompress(body, decompressed_size=dl, codec="gzip", asbytes=True) if dl else b""
            assert outcome == R.OK and got == want, (c, k, outcome, arg)
    assert seen["member"]
