"""The page encoders' oracles: the restatements of RleEncoder (pq_ref.rle_encode), RleBooleanEncoder
(pq_fixed_ref.bool_rle_encode) and deltaBitPackEncoder (pq_delta_ref.delta_encode) against the pages pyarrow writes,
byte for byte, and the parallel formulation of the RLE encoder the device kernel implements (pq_encode_model.py)
against the sequential restatement on adversarial inputs.  CPU only; the last test checks that the encode entry points
fail with AG_ERR_CUDA when no GPU is usable."""
import ctypes as C
import itertools

import numpy as np
import pytest

import pq_delta_ref as D
import pq_encode_model as M
import pq_files as F
import pq_fixed_ref as FX
import pq_pages as P
import pq_ref as R


# ------------------------------------------------------------------------------------------ the parallel model ----
def _check(values, bw):
    v = [int(x) for x in values]
    assert M.rle_encode(v, bw) == R.rle_encode(v, bw), (bw, v[:64], len(v))


@pytest.mark.parametrize("bw", [0, 1, 8, 17, 32])
def test_model_short_inputs(bw):
    hi = 1 if bw == 0 else 3
    for n in range(10):
        for v in itertools.product(range(hi), repeat=min(n, 5)):
            _check(list(v) + [0] * (n - len(v)), bw)


@pytest.mark.parametrize("bw", [0, 1, 8, 17, 32])
def test_model_runs_at_every_residue(bw):
    top = (1 << bw) - 1 if bw else 0
    for lead in range(17):                               # every residue, before and after a caught run
        for run in (7, 8, 9, 15, 16, 17):
            for tail in range(0, 12):
                lit = [(k * 5 + 1) & top for k in range(lead)]
                _check(lit + [top] * run + [(k * 3) & top for k in range(tail)], bw)


@pytest.mark.parametrize("bw", [1, 8, 17, 32])
def test_model_back_to_back_runs(bw):
    rng = np.random.default_rng(bw)
    top = (1 << bw) - 1
    for _ in range(300):
        parts = []
        for _ in range(rng.integers(1, 12)):
            ln = int(rng.choice([1, 2, 7, 8, 9, 10, 14, 15, 16, 23]))
            parts += [int(rng.integers(0, min(top, 3) + 1))] * ln
        _check(parts, bw)


@pytest.mark.parametrize("bw", [1, 8, 17, 32])
@pytest.mark.parametrize("groups", [62, 63, 64, 126, 127])
def test_model_literal_stretches_and_tails(bw, groups):
    top = (1 << bw) - 1
    lit = [(k % 2) ^ (k // 3 % 2) for k in range(8 * groups)]         # no 8 equal values in a row on any alignment
    lit = [x * top if x else 0 for x in lit]
    for tail in range(0, 8):
        _check(lit + [top // 2 + 1] * tail, bw)                       # equal tail
        _check(lit + [k & 1 for k in range(tail)], bw)                # mixed tail
        _check(lit + [5 & top] * (8 + tail) + lit[:8 * tail + 3], bw)  # caught run after the stretch


@pytest.mark.parametrize("groups", [0, 63, 126])
def test_model_equal_tails_after_literals(groups):
    lit = [(k % 2) ^ (k // 3 % 2) for k in range(8 * groups)]
    for tail in range(1, 8):
        for bw in (1, 8, 17, 32):
            _check(lit + [1] * tail, bw)


def test_model_random():
    rng = np.random.default_rng(20261018)
    for _ in range(1500):
        bw = int(rng.choice([0, 1, 2, 5, 8, 13, 17, 32]))
        n = int(rng.integers(0, 1300))
        vals, hi = [], (1 if bw == 0 else min(1 << bw, 5))
        while len(vals) < n:
            vals += [int(rng.integers(0, hi))] * int(rng.choice([1, 7, 8, 9, 16, 600]))
        _check(vals[:n], bw)


# ---------------------------------------------------------------------------------- pyarrow's pages, byte for byte ----
def _plan(path):
    plan = P.chunk_plan(path)
    return plan, P.host_decompress(plan)


def _level_sections(plan, dst):
    """the definition-level section of every data page (v1: 4-byte length + stream; v2: the stream)"""
    out = []
    for _, lv, _ in plan["pages"]:
        d, dl, nv, slot = lv
        if plan["v1"]:
            nb = int.from_bytes(dst[d:d + 4], "little")
            out.append((dst[d:d + 4 + nb], nv, slot))
        else:
            out.append((plan["chunk"][d:d + dl], nv, slot))
    return out


def _dict_width(ndict):
    return 0 if ndict == 0 else max(1, (ndict - 1).bit_length())


@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("shape", ["nulls", "all_null", "one_entry"])
def test_dictionary_pages_match_pyarrow(tmp_path, version, shape):
    pa = pytest.importorskip("pyarrow")
    rng = np.random.default_rng(7)
    n = 200_000
    vals = rng.integers(0, 3000, n).astype(np.int64)
    valid = rng.random(n) >= 0.1
    valid[50_000:60_000] = False
    if shape == "all_null":
        valid[:] = False
    if shape == "one_entry":
        vals[:] = 42
    arr = pa.array(vals, mask=~valid)
    path = str(tmp_path / "d.parquet")
    F.write_column(path, arr, nullable=True, encoding="RLE_DICTIONARY", version=version, data_page_size=1 << 17)
    plan, dst = _plan(path)
    assert len(plan["pages"]) >= (1 if shape == "all_null" else 5)
    # dictionary: first-occurrence order of the valid values, PLAIN
    _, first = np.unique(vals[valid], return_index=True)
    order = vals[valid][np.sort(first)]
    rank = {int(x): k for k, x in enumerate(order)}
    d, dl, nd = plan["dict"]
    assert dst[d:d + dl] == order.tobytes() and nd == order.size
    bw = _dict_width(order.size)
    for (enc, (vd, vl, nv, slot)), (lv, _, _) in zip(P.value_sections(plan, dst), _level_sections(plan, dst)):
        ok = valid[slot:slot + nv]
        idx = [rank[int(x)] for x in vals[slot:slot + nv][ok]]
        assert dst[vd:vd + vl] == bytes([bw]) + R.rle_encode(idx, bw)
        lev = R.rle_encode(ok.astype(np.uint8).tolist(), 1)
        assert lv == (len(lev).to_bytes(4, "little") + lev if version == "1.0" else lev)
    if shape == "all_null":
        assert all(dst[vd:vd + vl] == b"\x00" for _, (vd, vl, _, _) in P.value_sections(plan, dst))


@pytest.mark.parametrize("version", ["1.0", "2.0"])
def test_boolean_rle_pages_match_pyarrow(tmp_path, version):
    pa = pytest.importorskip("pyarrow")
    rng = np.random.default_rng(11)
    n = 100_000
    bits = rng.random(n) < 0.3
    bits[20_000:30_000] = True
    path = str(tmp_path / "b.parquet")
    F.write_column(path, pa.array(bits), nullable=False, encoding="RLE", version=version, data_page_size=1 << 12)
    plan, dst = _plan(path)
    assert len(plan["pages"]) > 1
    for enc, (vd, vl, nv, slot) in P.value_sections(plan, dst):
        assert enc == P.RLE
        assert dst[vd:vd + vl] == FX.bool_rle_encode(bits[slot:slot + nv])


@pytest.mark.parametrize("width,block", [(4, 128), (8, 256)])
def test_delta_pages_match_pyarrow(tmp_path, width, block):
    pa = pytest.importorskip("pyarrow")
    rng = np.random.default_rng(width)
    n = 300_000
    if width == 8:
        vals = (1_700_000_000_000_000_000 + np.cumsum(rng.integers(0, 5_000_000, n))).astype(np.int64)
    else:
        vals = rng.integers(-(1 << 31), 1 << 31, n).astype(np.int32)
    path = str(tmp_path / "t.parquet")
    F.write_column(path, pa.array(vals), nullable=False, encoding="DELTA_BINARY_PACKED", version="2.0", data_page_size=1 << 18)
    plan, dst = _plan(path)
    assert len(plan["pages"]) > 1
    for enc, (vd, vl, nv, slot) in P.value_sections(plan, dst):
        assert enc == P.DELTA_BINARY_PACKED
        assert dst[vd:vd + vl] == D.delta_encode(vals[slot:slot + nv], width, block, 4)


# ---------------------------------------------------------------------------------------------- without a GPU ----
def test_encoders_need_a_gpu():
    from arrow_go_b200 import _native as N
    ag = N
    if ag.call_status("ag_init", 0)[0] == N.AG_OK:
        pytest.skip("a GPU is usable here")
    size = C.c_int64()
    vals = np.zeros(16, np.uint32)
    out = np.zeros(64, np.uint8)
    tbl = N.enc_page_table([(0, 16, 0, 64)])
    calls = [("ag_parquet_rle_max_size", 1, N.PQ_RLE_BARE, 16, C.byref(size)),
             ("ag_parquet_rle_encode", 1, N.PQ_RLE_BARE, N.PQ_RLE_IN_U32, vals.ctypes.data, tbl, 1, out.ctypes.data, None, None),
             ("ag_parquet_rle_encode_dev", 1, N.PQ_RLE_BARE, N.PQ_RLE_IN_U32, vals.ctypes.data, tbl, 1, out.ctypes.data, None, None, None),
             ("ag_parquet_delta_max_size", 4, 128, 4, 16, C.byref(size)),
             ("ag_parquet_delta_encode", 4, 128, 4, vals.ctypes.data, tbl, 1, out.ctypes.data, None),
             ("ag_parquet_delta_encode_dev", 4, 128, 4, vals.ctypes.data, tbl, 1, out.ctypes.data, None, None)]
    for name, *args in calls:
        assert ag.call_status(name, *args)[0] == N.AG_ERR_CUDA, name
