"""Parquet decode primitives (SURVEY §8f rank 4) against the reference's own SIMD loops assembled into oracle/_ref
(unpack32_avx2, bytes_to_bools_avx2, levels_to_bitmap_bmi2 / extract_bits_bmi2) and its literal test vectors
(parquet/file/level_conversion_test.go:42-140)."""
import ctypes as C

import numpy as np
import pytest

from arrow_go_b200 import _native as N
from helpers import Dev, ptr, unpack_bits

gpu = pytest.mark.gpu


def model_unpack(packed_words, n, bits):
    """bit-level model: value i = bits [i*b, (i+1)*b) of the little-endian stream"""
    stream = np.unpackbits(packed_words.view(np.uint8), bitorder="little")
    out = np.zeros(n, dtype=np.uint64)
    for j in range(bits):
        out |= stream[np.arange(n) * bits + j].astype(np.uint64) << np.uint64(j)
    return out.astype(np.uint32)


def def_levels_model(levels, def_level, ancestor, offset, valid_bits):
    """python restatement of defLevelsBatchToBitmap (level_conversion.go:134-176)"""
    levels = np.asarray(levels, dtype=np.int16)
    defined = levels > def_level - 1
    if ancestor >= 0:
        present = levels > ancestor - 1
        bits = defined[present]
    else:
        bits = defined
    out = np.unpackbits(valid_bits, bitorder="little").astype(bool)
    out[offset:offset + bits.size] = bits
    return np.packbits(out, bitorder="little"), int(bits.size), int(bits.sum())


def test_reference_asm_agrees_with_the_bit_model(ref):
    """Pin the model (and so the GPU test below) on the reference's instruction stream."""
    if not hasattr(ref, "unpack32_avx2"):
        pytest.skip("oracle/_ref built without the parquet objects")
    ref.unpack32_avx2.restype = C.c_int
    ref.unpack32_avx2.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    rng = np.random.default_rng(1)
    for bits in range(0, 33):
        n = 32 * 7
        words = rng.integers(0, 1 << 32, max(1, n * bits // 32) + 4, dtype=np.uint64).astype(np.uint32)
        out = np.full(n + 40, 0xEEEEEEEE, dtype=np.uint32)
        assert ref.unpack32_avx2(words.ctypes.data, out.ctypes.data, n + 5, bits) == n     # whole groups only
        assert np.array_equal(out[:n], model_unpack(words, n, bits)), bits
    ref.levels_to_bitmap_bmi2.restype = C.c_uint64
    ref.levels_to_bitmap_bmi2.argtypes = [C.c_void_p, C.c_int, C.c_int16]
    lv = np.tile(np.arange(8, dtype=np.int16), 8)
    for num, rhs, want in ((0, 0, 0), (64, 8, 0), (64, -1, 0xFFFFFFFFFFFFFFFF), (47, -1, 0x7FFFFFFFFFFF), (64, 6, 0x8080808080808080)):
        assert ref.levels_to_bitmap_bmi2(lv.ctypes.data, num, rhs) == want    # level_conversion_test.go:88-117


@gpu
def test_unpack32_all_widths(ag, ref):
    rng = np.random.default_rng(2)
    have_ref = hasattr(ref, "unpack32_avx2")
    if have_ref:
        ref.unpack32_avx2.restype = C.c_int
        ref.unpack32_avx2.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    for bits in range(0, 33):
        for n_req in (0, 31, 32, 1000, 32 * 4099 + 17):
            n = n_req // 32 * 32
            words = rng.integers(0, 1 << 32, max(1, n * bits // 32) + 4, dtype=np.uint64).astype(np.uint32)
            want = np.zeros(n, dtype=np.uint32)
            if n and have_ref:
                assert ref.unpack32_avx2(words.ctypes.data, want.ctypes.data, n_req, bits) == n
            elif n:
                want = model_unpack(words, n, bits)
            got = np.full(n + 8, 0xEEEEEEEE, dtype=np.uint32)
            cnt = C.c_int64()
            ag.call("ag_parquet_unpack32", ptr(words), ptr(got), n_req, bits, C.byref(cnt))
            assert cnt.value == n and np.array_equal(got[:n], want), (bits, n_req)
            assert np.all(got[n:] == 0xEEEEEEEE)
    st, _ = ag.call_status("ag_parquet_unpack32", ptr(words), ptr(got), 64, 33, C.byref(cnt))
    assert st == N.AG_ERR_INVALID


@gpu
def test_bytes_to_bools(ag, ref):
    rng = np.random.default_rng(3)
    for length, outlen in ((1, 8), (1, 3), (100, 800), (100, 795), (4099, 4099 * 8), (5, 100)):
        b = rng.integers(0, 256, length, dtype=np.uint8)
        want = np.full(outlen + 8, 0xEE, dtype=np.uint8)
        if hasattr(ref, "bytes_to_bools_avx2"):
            ref.bytes_to_bools_avx2.restype = None
            ref.bytes_to_bools_avx2.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
            ref.bytes_to_bools_avx2(b.ctypes.data, length, want.ctypes.data, outlen)
        else:
            k = min(outlen, length * 8)
            want[:k] = np.unpackbits(b, bitorder="little")[:k]
        got = np.full(outlen + 8, 0xEE, dtype=np.uint8)
        ag.call("ag_parquet_bytes_to_bools", ptr(b), length, ptr(got), outlen)
        assert np.array_equal(got, want), (length, outlen)


@gpu
def test_def_levels_reference_literals(ag):
    # TestDefLevelsToBitmap (level_conversion_test.go:42-67): RepLevel 1 with ancestor level 0 = every slot present
    vb = np.array([2, 0], dtype=np.uint8)
    lv = np.array([3, 3, 3, 2, 3, 3, 3, 3, 3], dtype=np.int16)
    rd, nc = C.c_int64(-1), C.c_int64(0)
    ag.call("ag_parquet_def_levels_to_bitmap", ptr(lv), 9, 3, 0, ptr(vb), 0, 9, C.byref(rd), C.byref(nc))
    assert rd.value == 9 and nc.value == 1
    cur = int(vb[1]); nc.value = 0
    ag.call("ag_parquet_def_levels_to_bitmap", ptr(lv), 0, 3, 0, ptr(vb), 0, 9, C.byref(rd), C.byref(nc))
    assert rd.value == 0 and nc.value == 0 and int(vb[1]) == cur
    # TestDefLevelsToBitmapPowerOf2 (:69-87)
    vb = np.array([1, 0], dtype=np.uint8)
    lv = np.array([3, 3, 3, 2, 3, 3, 3, 3], dtype=np.int16)
    nc.value = 0
    ag.call("ag_parquet_def_levels_to_bitmap", ptr(lv[4:]), 4, 3, 0, ptr(vb), 0, 8, C.byref(rd), C.byref(nc))
    assert rd.value == 4 and nc.value == 0
    # TestWithRepetitionlevelFiltersOutEmptyListValues (:119-143)
    vb = np.zeros(8, dtype=np.uint8)
    lv = np.array([0, 0, 0, 2, 2, 1, 0, 2], dtype=np.int16)
    nc.value = 5
    ag.call("ag_parquet_def_levels_to_bitmap", ptr(lv), 8, 2, 1, ptr(vb), 1, 64, C.byref(rd), C.byref(nc))
    assert "".join("1" if b else "0" for b in unpack_bits(vb, 0, 8)) == "01101000" and not vb[1:].any()
    assert nc.value == 6 and rd.value == 4
    # upper bound (level_conversion.go:138-140)
    st, msg = ag.call_status("ag_parquet_def_levels_to_bitmap", ptr(lv), 8, 2, -1, ptr(vb), 0, 4, C.byref(rd), C.byref(nc))
    assert st == N.AG_ERR_INVALID and "upper bound" in msg


@gpu
def test_def_levels_random_vs_model(ag):
    rng = np.random.default_rng(4)
    for n in (1, 63, 64, 65, 1000, 200_003):
        for ancestor in (-1, 0, 1, 2):
            for off in (0, 3, 13):
                lv = rng.integers(0, 4, n).astype(np.int16)
                vb = rng.integers(0, 256, (n + off) // 8 + 9, dtype=np.uint8)
                want, read, setc = def_levels_model(lv, 3, ancestor, off, vb.copy())
                got = vb.copy()
                rd, nc = C.c_int64(), C.c_int64(7)
                ag.call("ag_parquet_def_levels_to_bitmap", ptr(lv), n, 3, ancestor, ptr(got), off, n, C.byref(rd), C.byref(nc))
                assert rd.value == read and nc.value == 7 + read - setc, (n, ancestor, off)
                assert np.array_equal(unpack_bits(got, 0, off + read), unpack_bits(want, 0, off + read)), (n, ancestor, off)
                # bytes past the one holding the last bit read keep the caller's values
                assert np.array_equal(got[(off + read + 7) >> 3:], vb[(off + read + 7) >> 3:]), (n, ancestor, off)
                # device flavour
                dl, dv, dc = Dev(lv), Dev(vb.copy()), Dev(np.zeros(2, dtype=np.int64))
                ag.call("ag_parquet_def_levels_to_bitmap_dev", dl.ptr, n, 3, ancestor, dv.ptr, off, n, dc.ptr, None)
                ag.call("ag_stream_sync", None)
                assert dc.get().tolist() == [read, setc]
                assert np.array_equal(unpack_bits(dv.get(), 0, off + read), unpack_bits(want, 0, off + read))


@gpu
def test_unpack32_100m_values_device(ag):
    """100M 13-bit values (dictionary indices of a large page run): device flavour, checked against the bit model on
    two windows and through sum(values) == sum over the model of the whole stream computed in chunks."""
    n, bits = 100_000_000 // 32 * 32, 13
    words = np.random.default_rng(5).integers(0, 1 << 32, n * bits // 32 + 4, dtype=np.uint64).astype(np.uint32)
    din, dout = Dev(words), Dev(nbytes=n * 4)
    cnt = C.c_int64()
    ag.call("ag_parquet_unpack32_dev", din.ptr, dout.ptr, n, bits, C.byref(cnt), None)
    ag.call("ag_stream_sync", None)
    assert cnt.value == n
    for start in (0, n - 32 * 40_000):
        m = 32 * 40_000
        w0 = start * bits // 32
        want = model_unpack(words[w0:w0 + m * bits // 32 + 2], m, bits)
        assert np.array_equal(dout.buf.to_numpy(np.uint32, m, start * 4), want)
