"""arrow/math Sum on the GPU vs the oracle (reference asm order + restatement).

Mirrors arrow/math/float64_test.go:30-48 (sum 0..9999 == 49995000, empty == 0) and the
benchmark sizes of :60-86; parity rules are SURVEY.md §8d."""
import ctypes as C
import math

import numpy as np
import pytest

from helpers import Dev, misaligned, ptr

pytestmark = pytest.mark.gpu


def ulp_dist(a, b):
    ia = np.array([a], dtype=np.float64).view(np.int64)[0]
    ib = np.array([b], dtype=np.float64).view(np.int64)[0]
    return abs(int(ia) - int(ib))


def gpu_sum_f64(ag, x, fn="ag_sum_f64"):
    r = C.c_double(123.0)
    ag.call(fn, ptr(x), x.size, C.byref(r))
    return r.value


def gpu_sum_f64_dev(ag, x, fn="ag_sum_f64_dev", off_elems=0):
    d = Dev(x, byte_offset=off_elems * 8)
    out = Dev(np.zeros(1))
    ag.call(fn, d.ptr, x.size, out.ptr, None)
    ag.call("ag_stream_sync", None)
    return out.get()[0]


def test_reference_known_answers(ag):
    # arrow/math/float64_test.go:33-36, int64_test.go, uint64_test.go
    x = np.arange(10000, dtype=np.float64)
    assert gpu_sum_f64(ag, x) == 49995000.0
    assert gpu_sum_f64_dev(ag, x) == 49995000.0
    assert gpu_sum_f64(ag, x, "ag_sum_f64_reforder") == 49995000.0
    xi = np.arange(10000, dtype=np.int64)
    r = C.c_int64()
    ag.call("ag_sum_i64", ptr(xi), xi.size, C.byref(r))
    assert r.value == 49995000
    ru = C.c_uint64()
    xu = xi.astype(np.uint64)  # keep the buffer alive across the call
    ag.call("ag_sum_u64", ptr(xu), xu.size, C.byref(ru))
    assert ru.value == 49995000
    # empty (float64_test.go:43-48)
    e = np.zeros(0)
    assert gpu_sum_f64(ag, e) == 0.0
    assert gpu_sum_f64(ag, e, "ag_sum_f64_reforder") == 0.0
    ag.call("ag_sum_i64", None, 0, C.byref(r))
    assert r.value == 0
    # a NULL buffer with rows is an error and leaves the result untouched
    rf = C.c_double(123.0)
    st, _ = ag.call_status("ag_sum_f64", None, 4, C.byref(rf))
    assert st == ag.AG_ERR_INVALID and rf.value == 123.0


@pytest.mark.parametrize("n", [1, 2, 3, 31, 32, 33, 63, 64, 255, 256, 257, 1000, 2047, 2048, 8192, 100003, 1 << 20, (1 << 22) + 5])
def test_f64_exact_data_bit_exact_with_reference(ag, cpu, ref, isa, n):
    """Dataset E (integer-valued doubles): every association order gives the same bits, so the
    GPU tree must equal the reference's AVX2 result exactly."""
    rng = np.random.default_rng(0x94378165 + n)
    x = rng.integers(-(1 << 20), (1 << 20) + 1, n).astype(np.float64)
    want = C.c_double()
    getattr(ref, f"sum_float64_{isa}")(ptr(x), n, C.addressof(want))
    assert cpu.ref_sum_f64_avx2_order(ptr(x), n) == want.value or isa != "avx2"
    assert gpu_sum_f64(ag, x) == want.value
    assert gpu_sum_f64_dev(ag, x) == want.value
    assert gpu_sum_f64_dev(ag, x, off_elems=1) == want.value  # 8-byte (not 16-byte) aligned slice


@pytest.mark.parametrize("n", [1, 31, 32, 33, 100, 8192, 100003, 1 << 20])
def test_f64_reference_order_mode_bit_exact_on_general_data(ag, cpu, ref, n):
    rng = np.random.default_rng(0x0FF1CE + n)
    x = rng.standard_normal(n)
    want = C.c_double()
    ref.sum_float64_avx2(ptr(x), n, C.addressof(want))
    assert cpu.ref_sum_f64_avx2_order(ptr(x), n) == want.value
    assert gpu_sum_f64(ag, x, "ag_sum_f64_reforder") == want.value
    assert gpu_sum_f64_dev(ag, x, "ag_sum_f64_reforder_dev") == want.value


@pytest.mark.parametrize("n", [8192, 100003, 1 << 20, 10_000_000])
@pytest.mark.parametrize("dist", ["normal", "uniform", "cancelling"])
def test_f64_general_data_accuracy(ag, cpu, n, dist):
    """Dataset G, SURVEY §8d acceptance: the GPU sum is within 1 ULP of the exactly rounded sum (math.fsum) and no
    farther from the reference-order result than the reference is from exact (+1 ULP).  The kernel carries the
    rounding error of every addition (TwoSum, summed in floating point: Sum2), so |res - S| <= 2 eps |S| +
    gamma_n^2 sum|x|; 1 ULP holds while gamma_n^2 sum|x| is small against eps |S|, which covers these families —
    "cancelling" is N(0,1) data followed by its own negation plus a small tail (sum|x| / |sum x| ~ 1e9).  Worse
    conditioned data, where only the bound holds, and non-finite inputs are in test_gpu_sum_special.py."""
    rng = np.random.default_rng(0x94378165)
    if dist == "normal":
        x = rng.standard_normal(n)
    elif dist == "uniform":
        x = rng.random(n)
    else:
        h = rng.standard_normal(n // 2)
        x = np.concatenate([h, -h[::-1], rng.standard_normal(n - 2 * (n // 2) + 0) * 1e-3])[:n]
        x[-1] = 1e-3
    exact = math.fsum(x)
    refv = cpu.ref_sum_f64_avx2_order(ptr(x), n)
    got = gpu_sum_f64_dev(ag, x)
    assert got == gpu_sum_f64(ag, x), "host and device flavours must agree bit for bit"
    assert got == gpu_sum_f64_dev(ag, x, off_elems=1), "alignment must not change the result"
    assert ulp_dist(got, exact) <= 1, (got, exact, ulp_dist(got, exact))
    assert ulp_dist(got, refv) <= ulp_dist(refv, exact) + 1


def test_f64_dataset_g_100m_rows_reports_ulp(ag, cpu, record_property):
    """BASELINE config size, dataset G (N(0,1), seed 0x94378165): report the ULP distance of the GPU sum to the exactly
    rounded sum and to the reference-order (AVX2) result, and of the reference to exact (SURVEY §8d asks for the
    numbers); accept on <= 1 ULP from exact, which the Sum2 bound (2 eps |S| + gamma_n^2 sum|x|) gives for N(0,1) data
    even at 100M rows.  The reference-order mode must reproduce the AVX2 bits at this size too."""
    n = 100_000_000
    x = np.random.default_rng(0x94378165).standard_normal(n)
    exact = math.fsum(x)
    refv = cpu.ref_sum_f64_avx2_order(ptr(x), n)
    d = Dev(x)
    out = Dev(np.zeros(2))
    ag.call("ag_sum_f64_dev", d.ptr, n, out.ptr, None)
    ag.call("ag_sum_f64_reforder_dev", d.ptr, n, out.ptr + 8, None)
    ag.call("ag_stream_sync", None)
    got, got_ref_order = (float(v) for v in out.get())
    report = {"rows": n, "gpu_vs_exact_ulp": ulp_dist(got, exact), "gpu_vs_reference_order_ulp": ulp_dist(got, refv),
              "reference_order_vs_exact_ulp": ulp_dist(refv, exact), "reforder_mode_bit_exact": got_ref_order == refv,
              "exact": exact, "gpu": got, "reference_order": refv}
    for k, v in report.items():
        record_property(k, v)
    print("\nsum f64 dataset G 100M:", report)
    try:
        import json, os
        os.makedirs("gpurun_out", exist_ok=True)
        json.dump(report, open("gpurun_out/sum_f64_ulp_100m.json", "w"), indent=1)
    except OSError:
        pass
    assert got_ref_order == refv
    assert ulp_dist(got, exact) <= 1
    assert ulp_dist(got, refv) <= ulp_dist(refv, exact) + 1


def test_f64_deterministic(ag):
    x = np.random.default_rng(7).standard_normal(3_000_001)
    d = Dev(x)
    out = Dev(np.zeros(1))
    vals = set()
    for _ in range(5):
        ag.call("ag_sum_f64_dev", d.ptr, x.size, out.ptr, None)
        ag.call("ag_stream_sync", None)
        vals.add(out.get()[0].tobytes())
    assert len(vals) == 1


@pytest.mark.parametrize("n", [1, 2, 3, 255, 256, 257, 8192, 100003, (1 << 22) + 3])
def test_int_sums_wrap_bit_exact(ag, cpu, ref, isa, n):
    rng = np.random.default_rng(0x94378165 + n)
    x = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, dtype=np.int64, endpoint=True)
    want = C.c_int64()
    getattr(ref, f"sum_int64_{isa}")(ptr(x), n, C.addressof(want))
    assert cpu.ref_sum_i64(ptr(x), n) == want.value
    r = C.c_int64()
    ag.call("ag_sum_i64", ptr(x), n, C.byref(r))
    assert r.value == want.value
    xm = misaligned(x, 1)
    d = Dev(xm, byte_offset=8)
    out = Dev(np.zeros(1, dtype=np.int64))
    ag.call("ag_sum_i64_dev", d.ptr, n, out.ptr, None)
    ag.call("ag_stream_sync", None)
    assert out.get()[0] == want.value
    xu = x.view(np.uint64)
    wantu = C.c_uint64()
    getattr(ref, f"sum_uint64_{isa}")(ptr(xu), n, C.addressof(wantu))
    ru = C.c_uint64()
    ag.call("ag_sum_u64", ptr(xu), n, C.byref(ru))
    assert ru.value == wantu.value


def test_sum_100m_rows_properties(ag):
    """BASELINE config size (100M rows) through size-independent properties: data generated on
    the device, sum(int64) checked against the closed form of the generator's CPU twin on a
    window plus linearity: sum(x) over [0,n) == sum over [0,k) + sum over [k,n)."""
    n = 100_000_000
    d = Dev(nbytes=n * 8)
    ag.call("ag_generate_dev", 1, 0x94378165, -1000, 1000, d.ptr, n, None)
    out = Dev(np.zeros(3, dtype=np.int64))
    k = 33_333_334  # even split point keeps both halves 16-byte aligned or not — both paths are legal
    ag.call("ag_sum_i64_dev", d.ptr, n, out.ptr, None)
    ag.call("ag_sum_i64_dev", d.ptr, k, out.ptr + 8, None)
    ag.call("ag_sum_i64_dev", d.ptr + 8 * k, n - k, out.ptr + 16, None)
    ag.call("ag_stream_sync", None)
    tot, a, b = out.get()
    assert tot == a + b
    # float64 view of integer-valued data: exact in every order
    ag.call("ag_generate_dev", 3, 0x94378165, -(1 << 20), 1 << 20, d.ptr, n, None)
    outf = Dev(np.zeros(3))
    ag.call("ag_sum_f64_dev", d.ptr, n, outf.ptr, None)
    ag.call("ag_sum_f64_dev", d.ptr, k, outf.ptr + 8, None)
    ag.call("ag_sum_f64_dev", d.ptr + 8 * k, n - k, outf.ptr + 16, None)
    ag.call("ag_stream_sync", None)
    tot, a, b = outf.get()
    assert tot == a + b
    # a 1M-row window against the oracle's generator twin
    from oracle import oracle
    w = np.empty(1 << 20, dtype=np.float64)
    oracle.cpu().ref_generate(3, 0x94378165, -(1 << 20), 1 << 20, w.ctypes.data, w.size)
    got = d.buf.to_numpy(np.float64, w.size)
    assert got.tobytes() == w.tobytes()
