"""Device SNAPPY page decompression against the Python restatement in tests/snappy_ref.py (host and _dev flavours, byte
for byte): every element form, and page sizes up to 16 MB. Then what every codec does, through pq_codecs: argument
checks, failing pages, the parquet-testing fixtures against pyarrow, pyarrow-written files end to end, and ~200 MB of
output through a checksum."""
import numpy as np
import pyarrow as pa
import pytest

import pq_codecs as H
import pq_files as F
import snappy_ref as S
from arrow_go_b200 import _native as N
from pq_pages import compressed_batch

gpu = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])


@gpu
@FLAVOURS
def test_every_element_form(ag, dev):
    rng = np.random.default_rng(61)
    streams = [(s, len(x)) for _, s, x in S.forms()]
    for name, x in (("random", rng.integers(0, 256, 50_000, dtype=np.uint8).tobytes()), ("zeros", bytes(70_000)),
                    ("timestamps", (np.cumsum(rng.integers(0, 1000, 9000)) + (1 << 40)).astype(np.int64).tobytes())):
        streams.append((pa.compress(x, codec="snappy", asbytes=True), len(x)))
        streams.append((S.encode(x, copy_form=4), len(x)))
    for gap in (True, False):
        st, msg, errs = H.decode_and_compare(ag, H.SNAPPY, streams, rng, dev, gap)
        assert st == N.AG_OK and not errs, msg


@gpu
@FLAVOURS
def test_page_sizes(ag, dev):
    rng = np.random.default_rng(62)
    streams = []
    for n in (0, 1, 65535, 65536, 65537):
        x = (rng.integers(0, 4, n, dtype=np.uint8) * 17).tobytes()
        streams.append((pa.compress(x, codec="snappy", asbytes=True), n))
    streams.append((b"", 0))                                      # an empty v2 value region
    st, msg, errs = H.decode_and_compare(ag, H.SNAPPY, streams, rng, dev)
    assert st == N.AG_OK and not errs, msg
    # 16 MB: longer than the parse window many times over; literal-heavy, copy-heavy and long-literal regions
    big = bytearray(rng.integers(0, 256, 1 << 24, dtype=np.uint8).tobytes())
    big[1 << 22:1 << 23] = bytes(1 << 22)
    big[1 << 23:(1 << 23) + (1 << 22)] = (np.cumsum(rng.integers(0, 1000, 1 << 19)) + (1 << 40)).astype(np.int64).tobytes()
    big = bytes(big)
    lit = S.stream(300_000, [S.literal(big[:300_000], 3)])       # one literal longer than the window
    src, pages, n_out = compressed_batch([(pa.compress(big, codec="snappy", asbytes=True), len(big)), (lit, 300_000)], rng)
    st, msg, out, w = H.run(ag, H.SNAPPY, src, pages, n_out, dev)
    assert st == N.AG_OK, msg
    for (s, sl, d, dl), k in zip(pages, w):
        assert k == dl
        want = big if dl == len(big) else big[:300_000]
        assert out[d:d + dl].tobytes() == want
    assert (out[:min(p[2] for p in pages)] == H.CANARY).all()


# ---------------------------------------------------------------- what every codec does (pq_codecs) ----
@gpu
@FLAVOURS
def test_invalid_arguments(ag, dev):
    H.invalid_arguments(ag, H.SNAPPY, dev)


@gpu
@FLAVOURS
@pytest.mark.parametrize("row", H.SNAPPY.error_rows(), ids=lambda r: r[0])
def test_error_rows(ag, row, dev):
    H.error_row(ag, H.SNAPPY, row, dev)


@gpu
@FLAVOURS
@pytest.mark.parametrize("name", H.SNAPPY.fixtures)
def test_fixture_pages_against_host(ag, name, dev):
    H.fixture_pages(ag, H.SNAPPY, name, dev)


@gpu
@pytest.mark.parametrize("case", F.compressed_cases(), ids=F.compressed_case_id)
def test_pyarrow_snappy_files_end_to_end(ag, case, tmp_path):
    H.pyarrow_file(ag, H.SNAPPY, case, tmp_path)


@gpu
@pytest.mark.parametrize("kind", ["byte_array", "fsb12", "bool"])
def test_pyarrow_snappy_files_other_types(ag, kind, tmp_path):
    H.pyarrow_file_other_type(ag, H.SNAPPY, kind, tmp_path)


@gpu
def test_decompress_200mb_device(ag):
    H.decompress_200mb(ag, H.SNAPPY)
