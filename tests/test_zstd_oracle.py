"""The ZSTD restatement (tests/zstd_ref.py) against pyarrow's libzstd: byte for byte on pyarrow's output at levels from
negative to 22, every form of the format coverage met (forms libzstd does not emit come from stream surgery), every
corrupt row rejected by pa.decompress too, XXH64 pinned, and the libzstd-written golden frames."""
import collections
import os

import pyarrow as pa
import pytest

import zstd_ref as Z

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


REQUIRED = [
    "frame", "skippable_frame", "multi_frame", "empty_frame", "single_segment", "window_descriptor", "dictionary_id_field",
    "content_size_1_bytes", "content_size_2_bytes", "content_size_4_bytes", "content_size_8_bytes", "no_content_size",
    "checksum", "block_raw", "block_rle", "block_compressed", "huf_fse_weights", "huf_direct_weights", "huf_max_bits_11",
    "nseq_0", "nseq_1_byte", "nseq_2_bytes", "nseq_3_bytes", "ll_accuracy_log_9", "of_accuracy_log_8",
    "ml_accuracy_log_9", "repeat_offset_0", "repeat_offset_1", "repeat_offset_2", "repeat_offset_3",
    "repeat_offset_ll0_shift",
] + [f"{k}_{m}" for k in ("ll", "of", "ml") for m in ("predefined", "rle", "fse", "repeat")]
REQUIRED_PREFIX = ["lit_raw", "lit_rle", "lit_huffman_1_streams", "lit_huffman_4_streams", "lit_treeless"]


def test_restatement_decodes_pyarrow_output_and_covers_every_form():
    seen = collections.Counter()
    for name, s, x in Z.corpus() + Z.surgery():
        got, err, arg = Z.decode(s, len(x), seen)
        assert err == Z.OK and got == x, (name, err, arg)
    missing = [f for f in REQUIRED if not seen[f]] + [p for p in REQUIRED_PREFIX if not any(k.startswith(p) for k in seen)]
    assert not missing, missing


def test_xxh64_known_answers():
    assert Z.xxh64(b"") == 0xEF46DB3751D8E999
    for name in ("checksum", "checksum_no_content_size"):
        s, x = next((r[1], r[2]) for r in Z.surgery() if r[0] == name)
        assert pa.decompress(s, decompressed_size=len(x), codec="zstd", asbytes=True) == x   # libzstd verifies it


# libzstd's one-shot decompression (pa.decompress) keeps the whole output as history and accepts these; RFC 8878 bounds
# zstd blocks and offsets by the window, and so does the decoder the reference uses.
WINDOW_ROWS = ("block_over_window", "offset_beyond_window")


@pytest.mark.parametrize("row", Z.corrupt_rows(), ids=lambda r: r[0])
def test_corrupt_rows(row):
    name, s, n, want = row
    got, err, arg = Z.decode(s, n)
    if want == Z.CHECKSUM:
        assert err == Z.CHECKSUM, (err, arg)
    else:
        assert err == Z.CORRUPT and arg == want, (err, arg)
    if name in WINDOW_ROWS:
        return
    with pytest.raises(Exception):
        pa.decompress(s, decompressed_size=max(n, 1), codec="zstd", asbytes=True)


def test_size_outcomes():
    x = b"0123456789" * 100
    good = Z.comp(x)
    assert Z.decode(good, len(x) + 1)[1:] == (Z.SIZE, len(x))
    assert Z.decode(good + good, len(x))[1:] == (Z.SIZE, 2 * len(x))
    nofcs = Z.reframe(good, fcs=False)
    assert Z.decode(nofcs, len(x) - 1)[1:] == (Z.SIZE, len(x))
    assert Z.decode(nofcs, len(x) + 1)[1:] == (Z.SIZE, len(x))
    assert Z.decode(b"", 0) == (b"", Z.OK, None)
    assert Z.decode(b"", 5)[1:] == (Z.SIZE, 0)


def test_golden_libzstd_frames():
    """frames written by libzstd with the checksum flag set and the content-size flag cleared (gen_zstd_golden.py)"""
    x = Z.golden_payload()
    for name in ("zstd_checksum.zst", "zstd_no_content_size.zst"):
        s = open(os.path.join(GOLDEN, name), "rb").read()
        seen = collections.Counter()
        got, err, _ = Z.decode(s, len(x), seen)
        assert err == Z.OK and got == x, name
        assert seen["checksum" if "checksum" in name else "no_content_size"], name
