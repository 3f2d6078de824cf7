"""The ZSTD restatement (tests/zstd_ref.py) against pyarrow's libzstd: byte for byte on pyarrow's output at levels from
negative to 22, every form of the format coverage met (forms libzstd does not emit come from stream surgery), every
corrupt row rejected by pa.decompress too, XXH64 pinned, and the libzstd-written golden frames."""
import collections
import os

import numpy as np
import pyarrow as pa
import pytest

import zstd_ref as Z

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
LEVELS = (-5, 1, 3, 9, 19, 22)


def datasets(rng):
    return {
        "timestamps": (np.cumsum(rng.integers(0, 1000, 40_000)) + (1 << 40)).astype(np.int64).tobytes(),
        "dict_indices": (rng.integers(0, 100_000, 60_000) & 0x1FFFF).astype(np.uint32).tobytes(),
        "zeros": bytes(300_000),
        "random": rng.integers(0, 256, 150_000, dtype=np.uint8).tobytes(),
        "text": b" ".join(rng.choice([b"alpha", b"beta", b"gamma", b"delta", b"parquet", b"zstd"], 40_000)),
        "skewed": np.minimum(rng.geometric(0.03, 200_000), 255).astype(np.uint8).tobytes(),
        "one": b"x",
        "empty": b"",
    }


def corpus():
    """[(name, compressed, raw)] written by pyarrow"""
    rng = np.random.default_rng(71)
    out = []
    for name, x in datasets(rng).items():
        for lvl in LEVELS:
            out.append((f"{name}-{lvl}", pa.Codec("zstd", compression_level=lvl).compress(x, asbytes=True), x))
    big = (np.cumsum(rng.integers(0, 1000, 1 << 19)) + (1 << 40)).astype(np.int64).tobytes()
    out.append(("timestamps-4MB-3", pa.compress(big, codec="zstd", asbytes=True), big))
    return out


def comp(x, level=3):
    return pa.Codec("zstd", compression_level=level).compress(x, asbytes=True)


def surgery():
    """[(name, stream, raw)]: the forms libzstd does not emit"""
    rng = np.random.default_rng(72)
    text = b" ".join(rng.choice([b"alpha", b"beta", b"gamma", b"delta"], 3000))
    ts = (np.cumsum(rng.integers(0, 1000, 5000)) + (1 << 40)).astype(np.int64).tobytes()
    letters = rng.integers(97, 123, 20_000, dtype=np.uint8).tobytes()
    assert Z.direct_weights(comp(letters))[1] > 0
    a, b = comp(text), comp(ts, 19)
    rows = [
        ("concatenated", a + b, text + ts),
        ("skippable_frames", Z.skippable(b"meta") + a + Z.skippable(b"", 15) + b + Z.skippable(bytes(100), 7), text + ts),
        ("checksum", Z.reframe(a, checksum=True), text),
        ("no_content_size", Z.reframe(b, fcs=False), ts),
        ("checksum_no_content_size", Z.reframe(a + b, fcs=False, checksum=True), text + ts),
        ("content_size_2_bytes", Z.reframe(comp(text[:5000]), fcs_bytes=2), text[:5000]),
        ("content_size_8_bytes", Z.reframe(a, fcs_bytes=8), text),
        ("dictionary_id_zero", Z.frame([Z.block("raw", b"hello", 1)], fcs=5, dict_id=(0, 2)), b"hello"),
        ("raw_and_rle_blocks", Z.frame([Z.block("raw", b"hello", 0), Z.block("rle", b"x", 1, size=1000)], fcs=1005),
         b"hello" + b"x" * 1000),
        ("empty_raw_block_frames", Z.frame([Z.block("raw", b"", 1)], fcs=0) * 3, b""),
        ("direct_weights", Z.direct_weights(comp(letters))[0], letters),
        ("rle_literals", Z.frame([Z.block("compressed", bytes([20 << 3 | 1, ord("k"), 0]), 1)], fcs=20), b"k" * 20),
        ("repeat_modes", Z.frame([Z.block("raw", b"abcdefgh", 0), Z.rle_seq_block(b"xyz", 3, 1, 0, 2, lambda i: 0, 0),
                                  Z.rle_seq_block(b"uv", 2, 1, 0, 2, lambda i: 0, 1, repeat=True)], fcs=8 + 3 * 6 + 2 * 6),
         None),
        ("rle_modes_3_byte_count", Z.frame([Z.block("raw", b"abcdefgh", 0),
                                            Z.rle_seq_block(b"", 33_000, 0, 0, 0, lambda i: 0, 1)], fcs=8 + 99_000), None),
        ("rep0_minus_1", Z.frame([Z.block("raw", bytes(range(64)), 0), Z.rle_seq_block(b"", 4, 0, 5, 0, lambda i: 3, 0),
                                  Z.rle_seq_block(b"zz", 5, 0, 1, 0, lambda i: 1, 1)], fcs=64 + 12 + 15 + 2), None),
        ("window_descriptor_1KB", Z.frame([Z.block("raw", b"q" * 1024, 0), Z.block("rle", b"r", 1, size=1024)],
                                          window_log=10), b"q" * 1024 + b"r" * 1024),
    ]
    out = []
    for name, s, x in rows:
        if x is None:                                             # hand-built: libzstd decodes it the same way
            x, err, _ = Z.decode(s)
            assert err == Z.OK and pa.decompress(s, decompressed_size=len(x), codec="zstd", asbytes=True) == x, name
        out.append((name, s, x))
    return out


def forms():
    """every stream of the corpus and the surgery rows, for the device tests: [(name, stream, raw)]"""
    return [r for r in corpus() if len(r[2]) < 1 << 20] + surgery()


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
    for name, s, x in corpus() + surgery():
        got, err, arg = Z.decode(s, len(x), seen)
        assert err == Z.OK and got == x, (name, err, arg)
    missing = [f for f in REQUIRED if not seen[f]] + [p for p in REQUIRED_PREFIX if not any(k.startswith(p) for k in seen)]
    assert not missing, missing


def test_xxh64_known_answers():
    assert Z.xxh64(b"") == 0xEF46DB3751D8E999
    for name in ("checksum", "checksum_no_content_size"):
        s, x = next((r[1], r[2]) for r in surgery() if r[0] == name)
        assert pa.decompress(s, decompressed_size=len(x), codec="zstd", asbytes=True) == x   # libzstd verifies it


def corrupt_rows():
    """[(name, stream, dst_len, expected check or Z.CHECKSUM)]: every row but WINDOW_ROWS pa.decompress rejects too"""
    rng = np.random.default_rng(73)
    text = b" ".join(rng.choice([b"alpha", b"beta", b"gamma", b"delta"], 3000))
    good = comp(text)
    n = len(text)
    ck = Z.reframe(good, checksum=True)
    hdr = Z.frame_header(fcs=None, window_log=17, single=False)
    bad_ck = ck[:-1] + bytes([ck[-1] ^ 1])
    rows = [
        ("truncated_block", good[:-3], n, "truncated"),
        ("truncated_checksum", ck[:-2], n, "truncated"),
        ("truncated_skippable", Z.skippable(b"abcdef")[:-2], n, "truncated"),
        ("bad_magic", b"\x28\xb5\x2f\xfe" + good[4:], n, "bad magic"),
        ("reserved_bit", good[:4] + bytes([good[4] | 8]) + good[5:], n, "frame header"),
        ("dictionary", Z.frame([Z.block("raw", b"hello", 1)], fcs=5, dict_id=(7, 1)), 5, "dictionary"),
        ("reserved_block_type", hdr + Z.block("reserved", b"abc", 1), 3, "block type"),
        ("block_over_window", Z.frame_header(window_log=10, single=False) + Z.block("raw", bytes(2000), 1), 2000, "block size"),
        ("literals_past_block", hdr + Z.block("compressed", bytes([31 << 3]) + b"ab", 1), 31, "literals"),
        ("treeless_without_table", hdr + Z.block("compressed", bytes([3, 0, 0, 0]), 1), 0, "huffman"),
        ("fse_accuracy_too_high", hdr + Z.block("raw", b"abcdefgh", 0) +
         Z.block("compressed", bytes([0, 1, 2 << 6, 0x0F, 0, 0]), 1), 11, "fse"),
        ("repeat_without_table", hdr + Z.block("raw", b"abcdefgh", 0) + Z.block("compressed", bytes([0, 1, 0xFC, 1]), 1), 11,
         "sequences"),
        ("zero_sequences_trailing_bytes", hdr + Z.block("compressed", bytes([0, 0, 7]), 1), 0, "sequences"),
        ("no_padding_marker", hdr + Z.block("raw", b"abcdefgh", 0) + Z.rle_seq_block(b"", 2, 0, 0, 0, lambda i: 0, 1)[:-1] +
         b"\x00", 14, "sequences"),
        ("literal_overrun", hdr + Z.block("raw", b"abcdefgh", 0) + Z.rle_seq_block(b"ab", 1, 5, 0, 0, lambda i: 0, 1), 16,
         "sequences"),
        ("offset_before_output", hdr + Z.rle_seq_block(b"", 1, 0, 0, 0, lambda i: 0, 1), 3, "offset"),
        ("offset_zero", hdr + Z.block("raw", b"abcdefgh", 0) + Z.rle_seq_block(b"", 1, 0, 1, 0, lambda i: 1, 1), 11, "offset"),
        ("offset_beyond_window", Z.frame_header(window_log=10, single=False) + Z.block("raw", bytes(1024), 0) +
         Z.block("raw", bytes(1024), 0) + Z.rle_seq_block(b"", 1, 0, 10, 0, lambda i: 1503 - 1024, 1), 2051, "offset"),
        ("content_size_short", Z.frame([Z.block("raw", b"hello", 1)], fcs=10), 10, "content size"),
        ("content_size_long", Z.frame([Z.block("raw", b"hello", 0), Z.block("raw", b"world", 1)], fcs=7), 7, "content size"),
        ("second_frame_corrupt", good + good[:-3], 2 * n, "truncated"),
        ("checksum_mismatch", bad_ck, n, Z.CHECKSUM),
        ("checksum_mismatch_then_corrupt", bad_ck + good[:-3], 2 * n, Z.CHECKSUM),
        ("page_size_then_corrupt", Z.reframe(good, fcs=False) + good[:-3], n - 10, "page size"),
    ]
    return rows


# libzstd's one-shot decompression (pa.decompress) keeps the whole output as history and accepts these; RFC 8878 bounds
# zstd blocks and offsets by the window, and so does the decoder the reference uses.
WINDOW_ROWS = ("block_over_window", "offset_beyond_window")


@pytest.mark.parametrize("row", corrupt_rows(), ids=lambda r: r[0])
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
    good = comp(x)
    assert Z.decode(good, len(x) + 1)[1:] == (Z.SIZE, len(x))
    assert Z.decode(good + good, len(x))[1:] == (Z.SIZE, 2 * len(x))
    nofcs = Z.reframe(good, fcs=False)
    assert Z.decode(nofcs, len(x) - 1)[1:] == (Z.SIZE, len(x))
    assert Z.decode(nofcs, len(x) + 1)[1:] == (Z.SIZE, len(x))
    assert Z.decode(b"", 0) == (b"", Z.OK, None)
    assert Z.decode(b"", 5)[1:] == (Z.SIZE, 0)


def test_golden_libzstd_frames():
    """frames written by libzstd with the checksum flag set and the content-size flag cleared (gen_zstd_golden.py)"""
    x = golden_payload()
    for name in ("zstd_checksum.zst", "zstd_no_content_size.zst"):
        s = open(os.path.join(GOLDEN, name), "rb").read()
        seen = collections.Counter()
        got, err, _ = Z.decode(s, len(x), seen)
        assert err == Z.OK and got == x, name
        assert seen["checksum" if "checksum" in name else "no_content_size"], name


def golden_payload():
    """the bytes the golden frames hold (tests/golden/gen_zstd_golden.py writes them)"""
    rng = np.random.default_rng(2024)
    ts = (np.cumsum(rng.integers(0, 1000, 40_000)) + (1 << 40)).astype(np.int64).tobytes()
    return ts + b" ".join(rng.choice([b"alpha", b"beta", b"gamma"], 20_000))
