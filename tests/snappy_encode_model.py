"""The exact parse of the device SNAPPY compressor (csrc/snappy_encode.cu, include/arrowgpu.h): 64 KiB fragments with
their own 4096-entry hash table, windows of 32 candidate positions, the first match of a window taken and extended byte
by byte, golang/snappy's element forms.  The device output is pinned to this byte for byte.  Not product code."""
import numpy as np

import snappy_ref as S

FRAGMENT = 1 << 16
WINDOW = 32
TABLE_BITS = 12


def _copy(off, n):
    out = bytearray()
    while n >= 68:
        out += S.copy(off, 64, 2)
        n -= 64
    if n > 64:
        out += S.copy(off, 60, 2)
        n -= 60
    return out + S.copy(off, n, 1 if n < 12 and off < 2048 else 2)


def _fragment(src, s, e, out):
    nc = e - s - 3                                                # candidates p: p + 4 <= e
    hashes = words = []
    if nc > 0:
        w = np.lib.stride_tricks.sliding_window_view(np.frombuffer(src[s:e], np.uint8), 4)[:nc].astype(np.uint32)
        words = (w[:, 0] | w[:, 1] << 8 | w[:, 2] << 16 | w[:, 3] << 24).astype(np.uint64)
        hashes = (((words * 0x1E35A7BD) & 0xFFFFFFFF) >> (32 - TABLE_BITS)).tolist()
        words = words.tolist()
    table, lit, cur = {}, 0, 0                                    # positions relative to s
    while cur < nc:
        hit = None
        for p in range(cur, min(cur + WINDOW, nc)):
            q = table.get(hashes[p])
            table[hashes[p]] = p
            if q is not None and words[q] == words[p]:
                hit = (p, q)
                break
        if hit is None:
            cur = min(cur + WINDOW, nc)
            continue
        p, q = hit
        n = 4
        while p + n + 64 <= e - s and src[s + q + n:s + q + n + 64] == src[s + p + n:s + p + n + 64]:
            n += 64
        while p + n < e - s and src[s + q + n] == src[s + p + n]:
            n += 1
        if p > lit:
            out += S.literal(src[s + lit:s + p])
        out += _copy(p - q, n)
        cur = lit = p + n
    if lit < e - s:
        out += S.literal(src[s + lit:e])


def compress(data):
    """the device's raw Snappy stream of one page"""
    data = bytes(data)
    out = bytearray(S.put_uvarint(len(data)))
    for s in range(0, len(data), FRAGMENT):
        _fragment(data, s, min(s + FRAGMENT, len(data)), out)
    return bytes(out)


def max_size(n):
    return 32 + n + n // 6


def corpora(rng, n):
    """{name: about n bytes} of the page bodies the compressor is measured on"""
    k = n // 8
    idx = rng.integers(0, 1 << 17, n * 8 // 17, dtype=np.uint64)
    bits = ((idx[:, None] >> np.arange(17, dtype=np.uint64)) & np.uint64(1)).astype(np.uint8).ravel()
    users = rng.zipf(1.3, n // 24) % 5000
    emails = b"".join(len(s).to_bytes(4, "little") + s for s in (f"user{u}@mail{u % 37}.example.com".encode() for u in users))
    return {
        "timestamps": (np.cumsum(rng.integers(0, 1000, k)) + (1 << 40)).astype(np.int64).tobytes(),
        "indices_17bit": np.packbits(bits, bitorder="little").tobytes()[:n],
        "prices": np.round(rng.lognormal(4, 1, k), 2).tobytes(),
        "categories": rng.integers(0, 50, n // 4).astype(np.int32).tobytes(),
        "emails": emails[:n],
        "zeros": bytes(n),
    }
