"""include/arrowgpu.h's ZSTD block cites the reference path it replaces and lists every check the device names."""
from arrow_go_b200 import _native as N

import zstd_ref as Z


def test_zstd_header_cites_reference_and_lists_checks():
    text = open(N.HEADER_PATH).read()
    block = text[text.index("ZSTD page decompression"):text.index("ag_parquet_zstd_decompress_dev")]
    for needle in ("parquet/file/page_reader.go:597-621", "parquet/compress/zstd.go:115-118", "getdecoder (:100-105)",
                   "zstd.NewReader(nil)"):
        assert needle in block, needle
    for check in Z.CHECKS:
        assert f"*         {check} " in block, check
