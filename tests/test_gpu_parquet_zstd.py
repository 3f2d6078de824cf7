"""Device ZSTD page decompression against the Python restatement in tests/zstd_ref.py (host and _dev flavours, byte for
byte): every form, the golden frames, and page sizes around the 128 KiB block. Then what every codec does, through
pq_codecs: argument checks, failing pages, the parquet-testing fixtures against pyarrow, pyarrow-written files end to
end, and ~200 MB of output through a checksum."""
import os

import numpy as np
import pyarrow as pa
import pytest

import pq_codecs as H
import pq_files as F
import zstd_ref as R
from arrow_go_b200 import _native as N

gpu = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])


@gpu
@FLAVOURS
def test_every_form(ag, dev):
    rng = np.random.default_rng(81)
    streams = [(s, len(x)) for _, s, x in R.forms()]
    for name in ("zstd_checksum.zst", "zstd_no_content_size.zst"):
        streams.append((open(os.path.join(H.GOLDEN, name), "rb").read(), len(R.golden_payload())))
    for gap in (True, False):
        st, msg, errs = H.decode_and_compare(ag, H.ZSTD, streams, rng, dev, gap)
        assert st == N.AG_OK and not errs, msg


@gpu
@FLAVOURS
def test_page_sizes(ag, dev):
    rng = np.random.default_rng(82)
    streams = []
    for n in (0, 1, (1 << 17) - 1, 1 << 17, (1 << 17) + 1, 1 << 22):
        x = (np.cumsum(rng.integers(0, 1000, (n + 7) // 8)) + (1 << 40)).astype(np.int64).tobytes()[:n]
        streams.append((pa.compress(x, codec="zstd", asbytes=True), n))
        streams.append((R.reframe(pa.compress(x, codec="zstd", asbytes=True), fcs=False, checksum=True), n))
    streams.append((b"", 0))
    st, msg, errs = H.decode_and_compare(ag, H.ZSTD, streams, rng, dev)
    assert st == N.AG_OK and not errs, msg


# ---------------------------------------------------------------- what every codec does (pq_codecs) ----
@gpu
@FLAVOURS
def test_invalid_arguments(ag, dev):
    H.invalid_arguments(ag, H.ZSTD, dev)


@gpu
@FLAVOURS
@pytest.mark.parametrize("row", H.ZSTD.error_rows(), ids=lambda r: r[0])
def test_error_rows(ag, row, dev):
    H.error_row(ag, H.ZSTD, row, dev)


@gpu
@FLAVOURS
def test_fixture_pages_against_host(ag, dev):
    H.fixture_pages(ag, H.ZSTD, H.ZSTD.fixtures[0], dev)


@gpu
@pytest.mark.parametrize("case", F.compressed_cases(), ids=F.compressed_case_id)
def test_pyarrow_zstd_files_end_to_end(ag, case, tmp_path):
    H.pyarrow_file(ag, H.ZSTD, case, tmp_path)


@gpu
@pytest.mark.parametrize("kind", ["byte_array", "fsb12", "bool"])
def test_pyarrow_zstd_files_other_types(ag, kind, tmp_path):
    H.pyarrow_file_other_type(ag, H.ZSTD, kind, tmp_path)


@gpu
def test_decompress_200mb_device(ag):
    H.decompress_200mb(ag, H.ZSTD)
