"""Writes zstd_checksum.zst (content checksum on) and zstd_no_content_size.zst (content-size flag off): frames only
libzstd's advanced parameters can produce (pyarrow cannot set them).  Calls the system libzstd.so.1 through ctypes.

  python tests/golden/gen_zstd_golden.py
"""
import ctypes as C
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from zstd_ref import golden_payload  # noqa: E402

ZSTD_c_compressionLevel, ZSTD_c_contentSizeFlag, ZSTD_c_checksumFlag = 100, 200, 201


def compress(lib, data, level, checksum, content_size):
    cctx = lib.ZSTD_createCCtx()
    for p, v in ((ZSTD_c_compressionLevel, level), (ZSTD_c_checksumFlag, checksum), (ZSTD_c_contentSizeFlag, content_size)):
        assert not lib.ZSTD_isError(lib.ZSTD_CCtx_setParameter(cctx, p, v))
    cap = lib.ZSTD_compressBound(len(data))
    out = C.create_string_buffer(cap)
    n = lib.ZSTD_compress2(cctx, out, cap, data, len(data))
    assert not lib.ZSTD_isError(n)
    lib.ZSTD_freeCCtx(cctx)
    return out.raw[:n]


def main():
    lib = C.CDLL("libzstd.so.1")
    lib.ZSTD_createCCtx.restype = C.c_void_p
    lib.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.ZSTD_CCtx_setParameter.restype = C.c_size_t
    lib.ZSTD_compressBound.argtypes = [C.c_size_t]
    lib.ZSTD_compressBound.restype = C.c_size_t
    lib.ZSTD_compress2.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
    lib.ZSTD_compress2.restype = C.c_size_t
    lib.ZSTD_isError.argtypes = [C.c_size_t]
    lib.ZSTD_freeCCtx.argtypes = [C.c_void_p]
    x = golden_payload()
    for name, ck, cs in (("zstd_checksum.zst", 1, 1), ("zstd_no_content_size.zst", 0, 0)):
        with open(os.path.join(HERE, name), "wb") as f:
            f.write(compress(lib, x, 3, ck, cs))


if __name__ == "__main__":
    main()
