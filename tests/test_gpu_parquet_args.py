"""Argument checks of every batch-of-pages Parquet decode entry point (levels, dict, plain-spaced, delta, bool, fixed,
byte_array), host and _dev flavours: the status, the `<fn>: ` prefix and the words of each message, and what a call
with no pages writes."""
import ctypes as C

import numpy as np
import pytest

from arrow_go_b200 import _native as N
from helpers import Dev, ptr

gpu = pytest.mark.gpu
FLAVOURS = pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
NO_ERROR_POS = (1 << 63) - 1
CANARY = 0xA7
SLOTS = 64                      # output slots of every call; every page below ends before it
ENTRIES = ["levels", "dict", "plain", "delta", "bool", "fixed", "byte_array"]
FN = {"levels": "levels_decode", "dict": "dict_decode", "plain": "plain_decode_spaced", "delta": "delta_decode",
      "bool": "bool_decode", "fixed": "fixed_decode", "byte_array": "byte_array_decode"}
SYMBOL = {"levels": "ag_parquet_levels_decode", "dict": "ag_parquet_dict_decode", "plain": "ag_parquet_plain_decode_spaced",
          "delta": "ag_parquet_delta_decode", "bool": "ag_parquet_bool_decode", "fixed": "ag_parquet_fixed_decode",
          "byte_array": "ag_parquet_byte_array_decode"}
HAS_BAD_POS = ("dict", "fixed", "byte_array")
OK_PAGE = (0, 2, 8, 0)


def run(ag, entry, dev, pages, n=None, *, width=4, dict_enc=False, null=(), out_off=0, dict_off=0,
        level_enc=N.PQ_LEVELS_V2_RLE, max_level=1, dict_len=4, data=None):
    """One call of `entry`.  `null` names the operands passed as NULL ("table", "data", "out", "dict"); out_off /
    dict_off move the _dev flavour's output / dictionary that many bytes past an aligned address.
    -> (status, message, bad position or None, output bytes after the call)."""
    n = len(pages) if n is None else n
    tbl = None if "table" in null else N.page_table(pages)
    dict_enc = dict_enc or entry == "dict"
    nout = {"levels": SLOTS * 2, "bool": SLOTS // 8, "byte_array": (SLOTS + 1) * width}.get(entry, SLOTS * width)
    data = np.zeros(64, np.uint8) if data is None else np.frombuffer(bytes(data), np.uint8).copy()
    valid = np.full(SLOTS // 8, 0xFF, np.uint8) if entry == "plain" else None
    out = np.full(nout, CANARY, np.uint8)
    dec = np.full(max(n, 1), -1, np.int64)
    if entry == "byte_array":
        dictionary = (np.arange(max(dict_len, 0) + 1) * 2).astype(np.int32 if width == 4 else np.int64).view(np.uint8)
        dict_data = np.zeros(2 * max(dict_len, 0) + 1, np.uint8)
    else:
        dictionary = np.zeros(max(dict_len, 0) * width + 1, np.uint8)
        dict_data = None
    if not dict_enc:
        dictionary = dict_data = None
    if "dict" in null:
        dictionary = None
    if dev:
        dd, dout, ddec = Dev(data), Dev(out, byte_offset=out_off), Dev(dec)
        dbad = Dev(np.array([-1], np.int64))
        dv = Dev(valid) if valid is not None else None
        ddict = Dev(dictionary, byte_offset=dict_off) if dictionary is not None else None
        ddata = Dev(dict_data) if dict_data is not None else None
        p_data, p_out, p_dec, p_bad = dd.ptr, dout.ptr, ddec.ptr, dbad.ptr
        p_valid, p_dict, p_dict_data = dv.ptr if dv else None, ddict.ptr if ddict else None, ddata.ptr if ddata else None
    else:
        bad = C.c_int64(-1)
        p_data, p_out, p_dec, p_bad = ptr(data), ptr(out), ptr(dec), C.byref(bad)
        p_valid, p_dict, p_dict_data = ptr(valid), ptr(dictionary), ptr(dict_data)
    if "data" in null:
        p_data = None
    if "out" in null:
        p_out = None
    dl = dict_len if dict_enc else 0
    enc = N.PQ_ENC_RLE_DICTIONARY if dict_enc else N.PQ_ENC_PLAIN
    if entry == "levels":
        args = [max_level, level_enc, p_data, tbl, n, p_out, p_dec]
    elif entry == "dict":
        args = [width, p_dict, dl, p_data, tbl, n, p_valid, p_out, p_dec, p_bad]
    elif entry == "plain":
        args = [width, p_data, tbl, n, p_valid, p_out]
    elif entry == "delta":
        args = [width, p_data, tbl, n, p_valid, p_out, p_dec]
    elif entry == "bool":
        args = [N.PQ_ENC_PLAIN, p_data, tbl, n, p_valid, p_out, p_dec]
    elif entry == "fixed":
        ptype = N.PQ_TYPE_INT32 if width == 4 else N.PQ_TYPE_INT64
        args = [ptype, 0, enc, p_data, tbl, n, p_valid, p_dict, dl, p_out, p_dec, p_bad]
    else:
        total = C.c_int64(-1)
        args = [enc, width, p_data, tbl, n, SLOTS if pages else 0, p_valid, p_dict, p_dict_data, dl, 0, p_out, None, 0, C.byref(total), p_dec, p_bad]
    st, msg = ag.call_status(SYMBOL[entry] + ("_dev" if dev else ""), *(args + [None] if dev else args))
    if dev:
        ag.call("ag_stream_sync", None)
        bad_value, got = int(dbad.get()[0]), dout.get()
    else:
        bad_value, got = bad.value, out
    return st, msg, (bad_value if entry in HAS_BAD_POS else None), got


def expect(st, msg, fn, *words, status=N.AG_ERR_INVALID):
    assert st == status, (fn, words, msg)
    assert msg.startswith(f"{fn}: "), (fn, msg)
    for w in words:
        assert w in msg, (fn, w, msg)


@gpu
@FLAVOURS
@pytest.mark.parametrize("entry", ENTRIES)
def test_negative_page_count(ag, entry, dev):
    st, msg, _, got = run(ag, entry, dev, [OK_PAGE], n=-1)
    expect(st, msg, FN[entry], "negative page")
    assert (got == CANARY).all()


@gpu
@FLAVOURS
@pytest.mark.parametrize("entry", ENTRIES)
def test_no_pages(ag, entry, dev):
    """n_pages == 0 succeeds, writes no output slot and still resets the bad position"""
    for null in ((), ("table",)):
        st, msg, bad, got = run(ag, entry, dev, [], null=null)
        assert st == N.AG_OK, (entry, msg)
        if entry == "byte_array":
            assert (got[4:] == CANARY).all()                                # offsets[0] = offset_base, nothing else
        else:
            assert (got == CANARY).all(), entry
        if entry in HAS_BAD_POS:
            assert bad == NO_ERROR_POS, (entry, bad)


@gpu
@FLAVOURS
@pytest.mark.parametrize("entry", ENTRIES)
def test_null_page_table(ag, entry, dev):
    st, msg, _, got = run(ag, entry, dev, [OK_PAGE], null=("table",))
    expect(st, msg, FN[entry], "NULL page table")
    assert (got == CANARY).all()


BAD_FIELDS = [(-1, 2, 8, 8), (0, -1, 8, 8), (0, 2, -8, 8), (0, 2, 8, -8)]
HUGE_FIELDS = [(0, 2, 1 << 31, 8), (0, 1 << 32, 8, 8)]


@gpu
@FLAVOURS
@pytest.mark.parametrize("entry", ENTRIES)
def test_bad_page_fields(ag, entry, dev):
    """the lowest bad page is named; the _dev flavour alone is given fields too large to stage"""
    for page in BAD_FIELDS + (HUGE_FIELDS if dev else []):
        st, msg, _, got = run(ag, entry, dev, [OK_PAGE, page])
        words = ["page 1: negative field"]
        if dev:
            words.append("page 1: negative field, more than 2^31-1 values or more than 2^32-1 bytes")
        expect(st, msg, FN[entry], *words)
        assert (got == CANARY).all()


@gpu
@FLAVOURS
@pytest.mark.parametrize("entry", ENTRIES)
def test_null_operands(ag, entry, dev):
    st, msg, _, got = run(ag, entry, dev, [OK_PAGE, (2, 3, 8, 8)], null=("data",))
    expect(st, msg, FN[entry], "NULL page data")
    st, msg, _, _ = run(ag, entry, dev, [OK_PAGE, (2, 3, 8, 8)], null=("out",))
    expect(st, msg, FN[entry], "NULL offsets" if entry == "byte_array" else "NULL output")
    if entry in HAS_BAD_POS:
        st, msg, _, got = run(ag, entry, dev, [OK_PAGE], dict_enc=True, null=("dict",))
        expect(st, msg, FN[entry], "NULL dictionary offsets" if entry == "byte_array" else "NULL dictionary")
        assert (got == CANARY).all()


@gpu
@pytest.mark.parametrize("entry", ["levels", "dict", "plain", "delta", "fixed", "byte_array"])
@pytest.mark.parametrize("width", [4, 8])
def test_misaligned_device_operands(ag, entry, width):
    """device outputs and dictionaries of 4- and 8-byte values must be aligned to their width (levels: int16)"""
    st, msg, _, got = run(ag, entry, True, [OK_PAGE], width=width, out_off=1 if entry == "levels" else width // 2)
    expect(st, msg, FN[entry], "offsets not aligned to offset_width" if entry == "byte_array" else "output not aligned to its")
    assert (got == CANARY).all()
    if entry in HAS_BAD_POS:
        st, msg, _, got = run(ag, entry, True, [OK_PAGE], width=width, dict_enc=True, dict_off=width // 2)
        expect(st, msg, FN[entry], "dictionary offsets not aligned" if entry == "byte_array" else "dictionary not aligned to its value width")
    if entry == "fixed":
        st, msg, _, _ = run(ag, entry, True, [OK_PAGE], width=width, dict_enc=True, out_off=width // 2)
        expect(st, msg, FN[entry], "output not aligned to its")


@gpu
@FLAVOURS
@pytest.mark.parametrize("entry", ["dict", "plain", "delta"])
def test_value_width(ag, entry, dev):
    for w in (0, 2, 12):
        st, msg, _, got = run(ag, entry, dev, [OK_PAGE], width=w)
        expect(st, msg, FN[entry], "value_width must be 4")
        assert (got == CANARY).all()
    if entry == "dict":
        st, msg, _, _ = run(ag, entry, dev, [OK_PAGE], dict_len=-1)
        expect(st, msg, FN[entry], "negative dictionary length")


@gpu
@FLAVOURS
def test_levels_encodings(ag, dev):
    run_ = 8 << 1                                                    # a repeated run of 8 levels
    for enc, data in ((N.PQ_LEVELS_V2_RLE, [run_, 1]), (N.PQ_LEVELS_V1_RLE, [2, 0, 0, 0, run_, 1])):
        st, msg, _, got = run(ag, "levels", dev, [(0, len(data), 8, 4)], level_enc=enc, data=data)
        assert st == N.AG_OK, msg
        lv = got.view(np.int16)
        assert lv[4:12].tolist() == [1] * 8 and (got[:8] == CANARY).all() and (got[24:] == CANARY).all()
    st, msg, _, _ = run(ag, "levels", dev, [(0, 3, 8, 0)], level_enc=N.PQ_LEVELS_V1_RLE)
    expect(st, msg, "levels_decode", "page 0: parquet: received invalid levels (corrupt data page?) (0 values decoded)")
    st, msg, _, _ = run(ag, "levels", dev, [OK_PAGE], level_enc=N.PQ_LEVELS_BIT_PACKED)
    expect(st, msg, "levels_decode", "deprecated BIT_PACKED", status=N.AG_ERR_NOT_IMPLEMENTED)
    st, msg, _, _ = run(ag, "levels", dev, [OK_PAGE], level_enc=5)
    expect(st, msg, "levels_decode", "unknown level encoding 5")
    for ml in (-1, 1 << 16):
        st, msg, _, _ = run(ag, "levels", dev, [OK_PAGE], max_level=ml)
        expect(st, msg, "levels_decode", "max_level must be 0..65535")
