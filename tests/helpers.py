"""Test-side helpers: numpy containers, bitmap packing, ctypes glue around the oracle and the
C ABI.  No product logic lives here."""
import ctypes as C

import numpy as np

from arrow_go_b200 import _native as N

NP_OF = {
    N.UINT8: np.uint8, N.INT8: np.int8, N.UINT16: np.uint16, N.INT16: np.int16,
    N.UINT32: np.uint32, N.INT32: np.int32, N.UINT64: np.uint64, N.INT64: np.int64,
    N.FLOAT32: np.float32, N.FLOAT64: np.float64,
}
ALL_TYPES = list(NP_OF)
INT_TYPES = [t for t in ALL_TYPES if t not in (N.FLOAT32, N.FLOAT64)]
TYPE_NAME = {N.UINT8: "uint8", N.INT8: "int8", N.UINT16: "uint16", N.INT16: "int16", N.UINT32: "uint32",
             N.INT32: "int32", N.UINT64: "uint64", N.INT64: "int64", N.FLOAT32: "float32", N.FLOAT64: "float64"}


def ptr(a):
    return None if a is None else a.ctypes.data


def pack_bits(bools, offset=0, fill=0xA5, pad_bytes=2):
    """LSB-first bitmap holding `bools` starting at bit `offset`; every other bit comes from `fill`."""
    bools = np.asarray(bools, dtype=bool)
    nbytes = (offset + len(bools) + 7) // 8 + pad_bytes
    buf = np.full(nbytes, fill, dtype=np.uint8)
    bits = np.unpackbits(buf, bitorder="little")
    bits[offset:offset + len(bools)] = bools
    return np.packbits(bits, bitorder="little")


def unpack_bits(buf, offset, n):
    return np.unpackbits(np.asarray(buf, dtype=np.uint8), bitorder="little")[offset:offset + n].astype(bool)


def random_values(rng, type_id, n, small=False):
    dt = np.dtype(NP_OF[type_id])
    if dt.kind == "f":
        v = rng.standard_normal(n).astype(dt)
        if n > 8 and not small:
            v[rng.integers(0, n, 3)] = [np.nan, np.inf, -0.0]
        return v
    info = np.iinfo(dt)
    if small:
        lo, hi = max(info.min, -50), min(info.max, 50)
        return rng.integers(lo, hi + 1, n).astype(dt)
    return rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)


def cast_inputs(rng, itype, otype, n):
    """Inputs for a numeric cast whose converted value is representable in the output type —
    the domain on which the reference's AVX2 / SSE4 / scalar code agree (and the only one a
    safe cast accepts).  int -> anything and float -> float are defined on the whole input
    range; float -> int is restricted to truncations that fit."""
    idt, odt = np.dtype(NP_OF[itype]), np.dtype(NP_OF[otype])
    if idt.kind != "f":
        return random_values(rng, itype, n)
    if odt.kind == "f":
        v = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 30, n)).astype(idt)
        if n > 8:
            v[rng.integers(0, n, 4)] = [np.nan, np.inf, -np.inf, -0.0]
        return v
    info = np.iinfo(odt)
    # stay strictly inside the output range after rounding to the input float type
    shrink = 1.0 - 2.0 ** -20
    lo, hi = max(float(info.min), -2.0 ** 62) * shrink, min(float(info.max), 2.0 ** 62) * shrink
    v = rng.uniform(lo, hi, n)
    k = rng.integers(0, 4, n)
    v = np.where(k == 0, np.trunc(v), v)                    # whole numbers (pass the safe check)
    v = np.where(k == 1, rng.uniform(max(lo, -300.0), min(hi, 300.0), n), v)  # small magnitudes
    return v.astype(idt)


def same_bits(a, b):
    """Bit-exact equality (NaN payloads included)."""
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def same_float_class(a, b):
    """Bit-exact except that NaNs only have to be NaN on both sides (SURVEY §7 hard-part 7)."""
    a = np.asarray(a)
    b = np.asarray(b)
    na, nb = np.isnan(a), np.isnan(b)
    if not np.array_equal(na, nb):
        return False
    return a[~na].tobytes() == b[~nb].tobytes()


def misaligned(arr, elems=1):
    """A copy of arr that starts `elems` elements past a 64-byte boundary."""
    arr = np.ascontiguousarray(arr)
    raw = np.empty(arr.nbytes + 128 + elems * arr.itemsize, dtype=np.uint8)
    base = (-raw.ctypes.data) % 64 + elems * arr.itemsize
    view = raw[base:base + arr.nbytes].view(arr.dtype)
    view[...] = arr
    return view


class Dev:
    """Device copy of a numpy array for the *_dev entry points."""

    def __init__(self, arr=None, nbytes=None, byte_offset=0):
        from arrow_go_b200.device import DeviceBuffer
        self.byte_offset = byte_offset
        if arr is not None:
            arr = np.ascontiguousarray(arr)
            self.dtype = arr.dtype
            self.count = arr.size
            self.buf = DeviceBuffer(arr.nbytes + byte_offset + 64)
            if arr.nbytes:
                N.call("ag_upload", self.buf.ptr + byte_offset, arr.ctypes.data, arr.nbytes, None)
                N.call("ag_stream_sync", None)
        else:
            self.dtype = np.dtype(np.uint8)
            self.count = nbytes
            self.buf = DeviceBuffer(nbytes + byte_offset + 64)

    @property
    def ptr(self):
        return self.buf.ptr + self.byte_offset

    def get(self, dtype=None, count=None):
        dtype = np.dtype(dtype or self.dtype)
        count = self.count if count is None else count
        return self.buf.to_numpy(dtype, count, self.byte_offset)


def checksum64(words):
    """what ag_checksum64_dev gives for the uint64 `words`: sum of word i times a splitmix64 mix of i, modulo 2^64"""
    z = np.arange(words.size, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return int(((z ^ (z >> np.uint64(31))) * words).sum(dtype=np.uint64))


def dev_scalar_i64(value=0):
    return Dev(np.array([value], dtype=np.int64))


class CumsumOracleState(C.Structure):
    """oracle/cpu_ref.c ref_cumsum_state: the running value in the type's own bytes + the encountered-null flag."""
    _fields_ = [("cur", C.c_uint8 * 8), ("encountered_null", C.c_int64)]


def oracle_cumsum(cpu, chunks, valids=None, skip=False, start=None, voff=3):
    """ref_cumulative_sum over the chunks of one sequence (unchecked): (values, output validity, null count, final
    running value).  start None is zero."""
    dt = np.asarray(chunks[0]).dtype
    t = {v: k for k, v in NP_OF.items()}[dt.type]
    valids = valids if valids is not None else [None] * len(chunks)
    st = CumsumOracleState()
    raw = np.array([0 if start is None else start], dtype=dt).tobytes()
    for i, b in enumerate(raw):
        st.cur[i] = b
    total = sum(len(c) for c in chunks)
    out = np.zeros(total, dtype=dt)
    ovalid = np.zeros((total + 7) // 8 + 1, dtype=np.uint8)
    pos = nulls = 0
    for x, v in zip(chunks, valids):
        x = np.ascontiguousarray(x, dtype=dt)
        bm = pack_bits(v, offset=voff) if v is not None else None
        o = np.zeros(len(x), dtype=dt)
        nn, bad = C.c_int64(0), C.c_int64(0)
        rc = cpu.ref_cumulative_sum(t, ptr(x), ptr(bm), voff, len(x), int(skip), 0, ptr(o), ptr(ovalid), pos,
                                    C.byref(st), C.byref(nn), C.byref(bad))
        assert rc == 0
        out[pos:pos + len(x)] = o
        nulls += nn.value
        pos += len(x)
    cur = np.frombuffer(bytes(st.cur)[:dt.itemsize], dtype=dt)[0]
    return out, unpack_bits(ovalid, 0, total).astype(bool), nulls, cur
