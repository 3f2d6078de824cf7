"""Test helper: a NumPy model of float32 / float64 cumulative_sum (arrow_go_b200/csrc/scan.cu,
cumsum_stream_kernel<float|double, *, false>) that fixes every bit of the outputs and of the carried state for any
input, non-finite ones included.  Not product code.

The kernel's association is fixed by (data, n) alone, so the model restates it operation by operation:
  * a tile is 32 KB (TILE_ROWS rows); warp w owns rows [w * SEG_ROWS, (w + 1) * SEG_ROWS) of it and lane l of the warp
    E contiguous rows (128 bytes) of that segment;
  * lane total: a left-to-right fold from zero() over the lane's counted rows (valid, below the first null unless nulls
    are skipped, below n);
  * warp scan: Hillis-Steele with d = 1, 2, 4, 8, 16 and incl = up + incl; lane_excl = incl of the lane before (zero
    for lane 0); the warp total is lane 31's incl; the tile total folds the 8 warp totals in warp order from zero, and
    warp_excl[w] is that fold stopped before warp w;
  * look-back of tile t (g = t / 128, qpos = t % 128, sg = g / 32, gq = g % 32): four 32-lane Hillis-Steele scans over
    the tile totals of group g below qpos (zero-padded), part = (((zero + x0[31]) + x1[31]) + x2[31]) + x3[31]; the
    group total (published by qpos == 127) is part + tile_total; gpart = lane 31 of a Hillis-Steele scan over the group
    totals of super-group sg below gq; base = the inclusive prefix of super-group sg - 1, or the start value for
    sg == 0; excl = (base + gpart) + part; the inclusive prefix of super-group sg (published by its last tile) is
    excl + tile_total;
  * finalize: run = warp_excl + lane_excl; for each counted row run = run + x and out = excl + run; null and dead rows
    are +0;
  * the state a call leaves is excl + tile_total of its last tile.  That is NOT always the bits of the last output:
    the last output associates as excl + ((warp_excl + lane_excl) + x ...), the state as excl + (the tile's warp-total
    fold); on general data they can differ in the last place.  The next chunk of a sequence starts from the state.

zero() is -0.0, the identity of IEEE addition (x + -0.0 == x for every x, -0.0 included), so every zero-padded lane,
entry and accumulator leaves the sum alone and a -0.0 start survives an all-(-0.0) prefix as the left-to-right loop
keeps it.  Every operation is one element-wise NumPy add in the value type (round to nearest, no FMA, subnormals
kept, as __fadd_rn / __dadd_rn); no np.cumsum, np.sum or add.reduce, whose orders are their own.

This module is the specification of the float scan: a change to the kernel's order changes this model with it."""
import numpy as np

# scan.cu constants
TILE_BYTES = 32768      # kScTileBytes
WARPS = 8               # kScWarps
VEC_ROWS = 8            # kScRows: 16-byte vectors per lane per tile
GROUP = 128             # kScGroup: tiles per look-back group
SUPER = 32              # kScSuper: groups per super-group
LANES = 32
LANE_BYTES = VEC_ROWS * 16


def geometry(dtype):
    """(TILE_ROWS, SEG_ROWS, E) for a value type: rows per tile, per warp segment, per lane."""
    w = np.dtype(dtype).itemsize
    tile = TILE_BYTES // w
    return tile, tile // WARPS, LANE_BYTES // w


def zero(dtype):
    """Pol<T, true>::zero()."""
    return np.dtype(dtype).type(-0.0)


def counted_rows(n, valid, skip):
    """Rows that accumulate: valid ones, and without skip only those before the first null."""
    if valid is None:
        return np.ones(n, dtype=bool)
    c = np.asarray(valid, dtype=bool).copy()
    if not skip:
        nulls = np.flatnonzero(~c)
        if nulls.size:
            c[nulls[0]:] = False
    return c


def hs_scan(v):
    """A 32-lane Hillis-Steele inclusive scan along the last axis: incl = up + incl for lanes >= d."""
    v = np.array(v, copy=True)
    with np.errstate(all="ignore"):
        for d in (1, 2, 4, 8, 16):
            v[..., d:] = v[..., :-d] + v[..., d:]
    return v


def tile_fold(x, counted):
    """Per tile: (tile_total[T], warp_excl[T, 8], lane_excl[T, 8, 32]); x, counted already tiled to [T, 8, 32, E]."""
    dt = x.dtype
    z = zero(dt)
    T = x.shape[0]
    with np.errstate(all="ignore"):
        tot = np.full(x.shape[:3], z, dtype=dt)
        for i in range(x.shape[3]):
            tot = np.where(counted[..., i], tot + x[..., i], tot)
        incl = hs_scan(tot)
        lane_excl = np.concatenate([np.full(incl.shape[:2] + (1,), z, dtype=dt), incl[..., :-1]], axis=-1)
        warp_excl = np.empty((T, WARPS), dtype=dt)
        acc = np.full(T, z, dtype=dt)
        for w in range(WARPS):
            warp_excl[:, w] = acc
            acc = acc + incl[:, w, LANES - 1]
    return acc, warp_excl, lane_excl


def lookback(tile_total, start):
    """The exclusive prefix of every tile (excl[T]) from the tile totals and the call's start value."""
    dt = tile_total.dtype
    z = zero(dt)
    T = tile_total.size
    n_groups = -(-T // GROUP)
    n_super = -(-n_groups // SUPER)
    t = np.arange(T)
    g, q = t // GROUP, t % GROUP
    padded = np.full(n_groups * GROUP, z, dtype=dt)
    padded[:T] = tile_total
    own = padded.reshape(n_groups, GROUP)
    with np.errstate(all="ignore"):
        a = np.where(np.arange(GROUP)[None, :] < q[:, None], own[g], z)         # [T, 128]: lane l of scan r = 32r + l
        s = hs_scan(a.reshape(T, GROUP // LANES, LANES))[..., LANES - 1]
        part = np.full(T, z, dtype=dt)
        for r in range(GROUP // LANES):
            part = part + s[:, r]
        gagg = np.full(n_super * SUPER, z, dtype=dt)                          # only complete groups are ever read
        last = np.arange(T // GROUP) * GROUP + GROUP - 1
        gagg[:last.size] = part[last] + tile_total[last]
        gg = np.arange(n_groups)
        b = np.where(np.arange(SUPER)[None, :] < (gg % SUPER)[:, None], gagg.reshape(n_super, SUPER)[gg // SUPER], z)
        gpart = hs_scan(b)[:, LANES - 1]
        excl = np.empty(T, dtype=dt)
        base = dt.type(start)
        for sg in range(n_super):
            lo, hi = sg * SUPER * GROUP, min(T, (sg + 1) * SUPER * GROUP)
            excl[lo:hi] = (base + gpart[g[lo:hi]]) + part[lo:hi]
            if hi == (sg + 1) * SUPER * GROUP:                                # the super-group is complete
                base = excl[hi - 1] + tile_total[hi - 1]
    return excl


def _tiled(a, T, fill, E):
    tile = WARPS * LANES * E
    buf = np.full(T * tile, fill, dtype=a.dtype)
    buf[:a.size] = a
    return buf.reshape(T, WARPS, LANES, E)


def scan_call(x, valid=None, skip=False, start=0.0):
    """One live call (the sequence is not dead): (out[n], state) for n >= 1."""
    x = np.ascontiguousarray(x)
    dt = x.dtype
    n = x.size
    assert n >= 1 and dt in (np.float32, np.float64)
    _, _, E = geometry(dt)
    T = -(-n // (WARPS * LANES * E))
    xt = _tiled(x, T, dt.type(0), E)
    ct = _tiled(counted_rows(n, valid, skip), T, False, E)
    tile_total, warp_excl, lane_excl = tile_fold(xt, ct)
    excl = lookback(tile_total, start)
    with np.errstate(all="ignore"):
        run = warp_excl[..., None] + lane_excl
        out = np.zeros_like(xt)
        ex = excl[:, None, None]
        for i in range(E):
            run = np.where(ct[..., i], run + xt[..., i], run)
            out[..., i] = np.where(ct[..., i], ex + run, dt.type(0))
        state = excl[-1] + tile_total[-1]
    return out.reshape(-1)[:n], dt.type(state)


def cumulative_sum(chunks, valids=None, skip=False, start=None):
    """A chunked sequence through one device state: (out of every chunk concatenated, final state).  start None is
    +0.0 (what ag_cumulative_sum_state_init_dev stores for no start).  Once a null was met without skip, later
    calls write 0 and leave the state alone."""
    chunks = [np.ascontiguousarray(c) for c in chunks]
    dt = chunks[0].dtype
    valids = valids if valids is not None else [None] * len(chunks)
    state = dt.type(0.0 if start is None else start)
    dead = False
    outs = []
    for x, v in zip(chunks, valids):
        if x.size == 0:
            outs.append(x.copy())
            continue
        if dead and not skip:
            outs.append(np.zeros_like(x))
            continue
        o, state = scan_call(x, v, skip, state)
        outs.append(o)
        if v is not None and not skip and not np.asarray(v, dtype=bool).all():
            dead = True
    return np.concatenate(outs), state
