"""The LZ4_RAW restatement (tests/lz4_ref.py) against liblz4 through pyarrow's "lz4_raw" codec: byte for byte on
pyarrow-compressed bodies of every kind and size, on every builder form and on every page of the two parquet-testing
LZ4_RAW fixtures; every form in REQUIRED met; every corrupt row refused by liblz4 too, except where the two decoders are
documented to part (DESIGN §2).  pa.decompress does not check the length it produces, so the size outcomes are pinned
against the restatement alone."""
import collections
import os

import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import lz4_ref as R
import pq_pages as P

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FIXTURES = ("lz4_raw_compressed.parquet", "lz4_raw_compressed_larger.parquet")

REQUIRED = ["literal_0", "literal_14", "literal_15", "literal_269", "literal_270", "literal_multi_255", "literal_extension",
            "match_extension", "match_multi_255", "offset_1", "offset_2", "offset_7", "offset_8", "offset_65535", "overlap",
            "lone_zero_token", "ends_in_literals"] + [f"nibble_{k}" for k in range(16)]


def liblz4(s, n):
    return pa.decompress(s, decompressed_size=n, codec="lz4_raw", asbytes=True)


def bodies():
    """(name, body) of pyarrow-compressible kinds at sizes from 0 to several MB"""
    out = []
    for n in (0, 1, 5, 12, 13, 64, 4095, 65536, 65537, 1 << 20, 5 << 20):
        out.append((f"noise_{n}", R.noise(n, n)))
        out.append((f"runs_{n}", R.runs(n, n)))
    for n in (100, 65536, 1 << 21):
        out.append((f"timestamps_{n}", R.timestamps(n, n)))
        out.append((f"dict_indices_{n}", R.dict_indices(n, n)))
    return out


@pytest.mark.parametrize("name,x", bodies(), ids=[b[0] for b in bodies()])
def test_restatement_matches_liblz4(name, x):
    s = pa.compress(x, codec="lz4_raw", asbytes=True)
    got, outcome, arg = R.decode(s, len(x))
    assert outcome == R.OK and got == x, (outcome, arg)
    assert liblz4(s, len(x)) == x


def test_every_form_is_covered():
    seen = collections.Counter()
    for name, s, y in R.forms():
        got, outcome, arg = R.decode(s, len(y), seen)
        assert outcome == R.OK and got == y, (name, outcome, arg)
        assert liblz4(s, len(y)) == y, name
    missing = [f for f in REQUIRED if not seen[f]]
    assert not missing, missing


@pytest.mark.parametrize("row", R.differences(), ids=lambda r: r[0])
def test_documented_differences_from_liblz4(row):
    """a stream ending in a match or with a match in its last 12 bytes and an empty block decode here and not in
    liblz4; a final literal-only sequence with a match nibble and offset 0 are corrupt here and pass liblz4"""
    name, s, n, want, lib_accepts = row
    got, outcome, arg = R.decode(s, n)
    assert (outcome, arg) == want
    if outcome == R.OK:
        assert len(got) == n
    if lib_accepts:
        liblz4(s, n)
    else:
        with pytest.raises(Exception):
            liblz4(s, n)


LIBLZ4_ACCEPTS = ("offset_0", "final_nonzero_nibble")


@pytest.mark.parametrize("row", R.corrupt_rows(), ids=lambda r: r[0])
def test_corrupt_rows(row):
    name, s, n, want, written = row
    got, outcome, arg = R.decode(s, n)
    assert (outcome, arg) == want
    assert len(got) == written
    if outcome == R.SIZE:
        return
    if name in LIBLZ4_ACCEPTS:
        liblz4(s, n)
    else:
        with pytest.raises(Exception):
            liblz4(s, n)


def test_messages():
    assert R.message(R.CORRUPT, None, 7) == "parquet: could not decompress page: lz4: invalid source or destination buffer too short"
    assert R.message(R.SIZE, 5, 8) == "parquet: metadata said 8 bytes uncompressed data page, got 5 bytes"
    assert R.decode(b"", 0) == (b"", R.OK, None)
    assert R.decode(b"\x00", 0) == (b"", R.OK, None)


def test_builder_lengths():
    """the extension bytes of every length form: 15 is one 0 byte, 15 + 255 is 255 then 0"""
    assert R.seq(bytes(14))[:1] == b"\xe0" and len(R.seq(bytes(14))) == 15
    assert R.seq(bytes(15))[:2] == b"\xf0\x00"
    assert R.seq(bytes(15 + 254))[:2] == b"\xf0\xfe"
    assert R.seq(bytes(15 + 255))[:3] == b"\xf0\xff\x00"
    assert R.seq(b"", 1, 19)[:4] == b"\x0f\x01\x00\x00"
    assert R.seq(b"", 1, 19 + 510)[:5] == b"\x0f\x01\x00\xff\xff" and R.seq(b"", 1, 19 + 510)[5] == 0


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_pages_against_liblz4(name):
    path = os.path.join(GOLDEN, name)
    for c in range(pq.ParquetFile(path).metadata.num_columns):
        chunk, pages = P.column_chunk(path, column=c)
        regions, comp, _ = P.decompress_table(pages)
        assert comp
        for k in comp:
            s, sl, _, dl = regions[k][:4]
            body = bytes(chunk[s:s + sl])
            got, outcome, arg = R.decode(body, dl)
            want = liblz4(body, dl) if dl else b""
            assert outcome == R.OK and got == want, (c, k, outcome, arg)
