"""Device GZIP page decompression against the Python restatement in tests/gzip_ref.py (host and _dev flavours, byte for
byte, the canary outside every written range): every form, zlib's levels and strategies, and page sizes around the 32
KiB window, stored blocks included. Then what every codec does, through pq_codecs: argument checks, failing pages, the
parquet-testing fixtures against pyarrow, pyarrow-written files end to end, and ~200 MB of output through a checksum."""
import zlib

import numpy as np
import pyarrow as pa
import pytest

import gzip_ref as R
import pq_codecs as H
import pq_files as F
from arrow_go_b200 import _native as N

gpu = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])


@gpu
@FLAVOURS
def test_every_form(ag, dev):
    rng = np.random.default_rng(91)
    streams = [(s, len(x)) for _, s, x in R.forms()]
    x = R.payload(40000, 9)
    streams += [(R.gz(x, lv, st), len(x)) for lv in (0, 1, 6, 9) for st in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED)]
    for gap in (True, False):
        st, msg, errs = H.decode_and_compare(ag, H.GZIP, streams, rng, dev, gap)
        assert st == N.AG_OK and not errs, msg


@gpu
@FLAVOURS
def test_page_sizes(ag, dev):
    rng = np.random.default_rng(92)
    streams = []
    for n in (0, 1, 32767, 32768, 32769, 65535, 65536, 1 << 22):
        x = (np.cumsum(rng.integers(0, 1000, (n + 7) // 8)) + (1 << 40)).astype(np.int64).tobytes()[:n]
        streams.append((pa.compress(x, codec="gzip", asbytes=True), n))
        streams.append((R.gz(x, 0), n))                         # stored blocks
    streams.append((b"", 0))
    st, msg, errs = H.decode_and_compare(ag, H.GZIP, streams, rng, dev)
    assert st == N.AG_OK and not errs, msg


# ---------------------------------------------------------------- what every codec does (pq_codecs) ----
@gpu
@FLAVOURS
def test_invalid_arguments(ag, dev):
    H.invalid_arguments(ag, H.GZIP, dev)


@gpu
@FLAVOURS
@pytest.mark.parametrize("row", H.GZIP.error_rows(), ids=lambda r: r[0])
def test_error_rows(ag, row, dev):
    H.error_row(ag, H.GZIP, row, dev)


@gpu
@FLAVOURS
@pytest.mark.parametrize("name", H.GZIP.fixtures)
def test_fixture_pages_against_host(ag, name, dev):
    H.fixture_pages(ag, H.GZIP, name, dev)


@gpu
@pytest.mark.parametrize("case", F.compressed_cases(), ids=F.compressed_case_id)
def test_pyarrow_gzip_files_end_to_end(ag, case, tmp_path):
    H.pyarrow_file(ag, H.GZIP, case, tmp_path)


@gpu
@pytest.mark.parametrize("kind", ["byte_array", "fsb12", "bool"])
def test_pyarrow_gzip_files_other_types(ag, kind, tmp_path):
    H.pyarrow_file_other_type(ag, H.GZIP, kind, tmp_path)


@gpu
def test_decompress_200mb_device(ag):
    H.decompress_200mb(ag, H.GZIP)
