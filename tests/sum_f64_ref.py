"""Test helper: a NumPy model of the default float64 Sum (arrow_go_b200/csrc/reduce.cu, sum_kernel<double, *>) that
fixes every bit of its result on any input, non-finite ones included.  Not product code.

The kernel's association order is fixed by (n) alone, so the model restates it step by step: the grid rule, the
tile -> thread -> load -> accumulator mapping, the accumulator merges, the block trees, the last block's fold of the
partials, the odd last element and the cross-rank fold of the global Sum.  Every modelled thread is one lane of a NumPy
array, and every TwoSum is written out operation by operation in IEEE double (NumPy adds and subtracts round to
nearest, and nothing here is contracted into an FMA, as the kernel's __dadd_rn / __dsub_rn are not).

This module is the specification of the default mode: a change to the kernel's order changes this model with it."""
import numpy as np

# reduce.cu constants
THREADS = 256                   # kSumThreads
LOADS = 8                       # kSumLoads: pair loads per thread per tile
ACC = 4                         # kSumAcc: accumulator pairs per thread, load k feeds k % 4
TILE_PAIRS = THREADS * LOADS    # kSumTilePairs: 2048 pairs = 32 KB
SMS = 132                       # kSumSMs
BLOCKS_PER_SM = 4               # sum_blocks_per_sm<double>()
MAX_BLOCKS = SMS * BLOCKS_PER_SM


def grid(n_pairs):
    """sum_grid<double>: one block per tile, at least one, at most 132 x 4."""
    want = (n_pairs + TILE_PAIRS - 1) // TILE_PAIRS
    return max(1, min(want, MAX_BLOCKS))


class Acc:
    """Acc<double>: (s, c) pairs, one per modelled thread.  s is the plain IEEE sum of the pair's chain, c the sum of
    the rounding errors TwoSum split off."""

    def __init__(self, s, c):
        self.s = np.asarray(s, dtype=np.float64)
        self.c = np.asarray(c, dtype=np.float64)

    @staticmethod
    def zeros(shape=()):
        return Acc(np.zeros(shape), np.zeros(shape))

    def add(self, x, mask=None):
        """Acc<double>::add; where `mask` is False the pair is left alone (a load the kernel does not make)."""
        with np.errstate(all="ignore"):
            t = self.s + x                          # t = s + x
            z = t - self.s                          # z = t - s
            e = (self.s - (t - z)) + (x - z)        # e = (s - (t - z)) + (x - z)
            c = self.c + e                          # c = c + e
        if mask is None:
            self.s, self.c = t, c
        else:
            self.s, self.c = np.where(mask, t, self.s), np.where(mask, c, self.c)

    def merge(self, o, mask=None):
        """Acc<double>::merge: add(o.s), then c = c + o.c."""
        self.add(o.s, mask)
        with np.errstate(all="ignore"):
            c = self.c + o.c
        self.c = c if mask is None else np.where(mask, c, self.c)

    def lanes(self, idx):
        """shfl_xor: the pairs of lanes `idx` along the last axis (a copy, taken before anyone merges)."""
        return Acc(self.s[..., idx], self.c[..., idx])

    def value(self):
        """Acc<double>::value: s + c while s is finite; a non-finite s (±inf, NaN) is the result as it stands."""
        with np.errstate(all="ignore"):
            return np.where(np.isfinite(self.s), self.s + self.c, self.s)


def block_tree(v):
    """block_tree_sum over the last axis (256 threads): xor-shuffle merges 16, 8, 4, 2, 1 inside every warp, then warp
    0 holds the 8 warp values in lanes 0..7 and merges xor 4, 2, 1.  Returns thread 0's pair."""
    lane = np.arange(32)
    w = Acc(v.s.reshape(v.s.shape[:-1] + (THREADS // 32, 32)), v.c.reshape(v.c.shape[:-1] + (THREADS // 32, 32)))
    for m in (16, 8, 4, 2, 1):
        w.merge(w.lanes(lane ^ m))
    r = Acc(w.s[..., 0], w.c[..., 0])               # smem[warp] = lane 0's pair; lanes 8..31 of warp 0 do not reach lane 0
    lane8 = np.arange(THREADS // 32)
    for m in (4, 2, 1):
        r.merge(r.lanes(lane8 ^ m))
    return Acc(r.s[..., 0], r.c[..., 0])


def local_pair(x):
    """The (s, c) pair one launch of sum_kernel<double> holds before value() (or the exchange), for n >= 1."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    n = x.size
    assert n >= 1
    n_pairs = n >> 1
    n_tiles = (n_pairs + TILE_PAIRS - 1) // TILE_PAIRS
    G = grid(n_pairs)
    xs, ys = x[0:2 * n_pairs:2], x[1:2 * n_pairs:2]   # pair j = (x[2j], x[2j+1])
    ax = [Acc.zeros((G, THREADS)) for _ in range(ACC)]
    ay = [Acc.zeros((G, THREADS)) for _ in range(ACC)]
    b = np.arange(G, dtype=np.int64)[:, None]
    t = np.arange(THREADS, dtype=np.int64)[None, :]
    # block b streams tiles b, b+G, ...; in a tile thread t owns pairs t + 256k, load k feeds accumulator pair k % 4
    for r in range((n_tiles + G - 1) // G):
        j0 = (r * G + b) * TILE_PAIRS + t
        for k in range(LOADS):
            jj = j0 + k * THREADS
            live = jj < n_pairs
            jc = np.where(live, jj, 0)
            ax[k % ACC].add(xs[jc], live)
            ay[k % ACC].add(ys[jc], live)
    # ((x0+y0)+(x1+y1)) + ((x2+y2)+(x3+y3))
    for k in range(ACC):
        ax[k].merge(ay[k])
    ax[0].merge(ax[1])
    ax[2].merge(ax[3])
    ax[0].merge(ax[2])
    v = block_tree(ax[0])                           # shape (G,): every block's thread-0 pair
    if G == 1:
        acc = Acc(v.s[0], v.c[0])
    else:
        # the last block: thread t folds partials t, t+256, ... in order, then the block tree
        acc = Acc.zeros(THREADS)
        tt = np.arange(THREADS)
        for i in range((G + THREADS - 1) // THREADS):
            idx = tt + i * THREADS
            live = idx < G
            acc.merge(v.lanes(np.where(live, idx, 0)), live)
        acc = block_tree(acc)
    if n & 1:
        acc.add(x[n - 1])                           # the odd last element, after the tree
    return acc


def sum_f64(x):
    """ag_sum_f64 / ag_sum_f64_dev (one rank): the result bits of the default mode."""
    x = np.asarray(x, dtype=np.float64)
    if x.size == 0:
        return np.float64(0.0)
    return np.float64(local_pair(x).value())


def global_sum_f64(shards):
    """ag_sum_f64_global_dev over len(shards) ranks: every rank folds the ranks' pairs in rank order into a zero pair
    (exchange_sum); a rank with n == 0 contributes a zero pair.  One rank does not exchange."""
    if len(shards) == 1:
        return sum_f64(shards[0])
    g = Acc.zeros()
    for x in shards:
        g.merge(local_pair(x) if len(x) else Acc.zeros())
    return np.float64(g.value())


# ---- the contract the model is held to, stated without its order ---------------------------------------------------
EPS = 2.0 ** -53                                    # unit roundoff of float64


def expected_class(x):
    """What any association of IEEE additions returns for x, where that does not depend on the association: "nan" if
    x holds a NaN or both infinities; otherwise, while the finite values' sum|x| stays below DBL_MAX, "+inf" / "-inf"
    if it holds infinities of one sign and "finite" if it holds none.  None where the class depends on the order
    (finite values whose partial sums may overflow)."""
    x = np.asarray(x, dtype=np.float64)
    if np.isnan(x).any() or (np.isposinf(x).any() and np.isneginf(x).any()):
        return "nan"
    fin = x[np.isfinite(x)]
    if float(np.sum(np.abs(fin), dtype=np.longdouble)) > np.finfo(np.float64).max * (1 - 2 * EPS):
        return None
    if np.isposinf(x).any():
        return "+inf"
    if np.isneginf(x).any():
        return "-inf"
    return "finite"


def float_class(v):
    v = float(v)
    if v != v:
        return "nan"
    if v == float("inf"):
        return "+inf"
    if v == float("-inf"):
        return "-inf"
    return "finite"


def sum2_error_bound(x, exact):
    """Ogita, Rump and Oishi's bound for TwoSum with the errors summed in floating point (Sum2), plus the final
    rounding of s + c: |res - S| <= 2 eps |S| + gamma_n^2 sum|x|, gamma_n = n eps / (1 - n eps).  `exact` is the
    correctly rounded sum (math.fsum); returned as a Fraction."""
    from fractions import Fraction
    import math
    n = len(x)
    gamma = Fraction(n) * Fraction(EPS) / (1 - Fraction(n) * Fraction(EPS))
    abs_sum = Fraction(math.fsum(np.abs(x))) * (1 + Fraction(EPS))     # fsum rounds sum|x| by at most eps
    return 2 * Fraction(EPS) * abs(Fraction(exact)) + gamma * gamma * abs_sum


def gensum(n, cond, seed):
    """An ill-conditioned float64 vector with sum|x| / |sum x| near `cond`, after Ogita, Rump and Oishi's GenSum: the
    first half has random signs and exponents spread over [0, log2(cond)]; the second half's exponents fall
    linearly to 0, each value minus the exact sum so far, so the running sum cancels down scale by scale; then a
    seeded shuffle.  Beyond 65536 values the extra ones are exactly cancelling pairs (y, -y) with exponents over the
    same range, shuffled in with the rest, which raises sum|x| but leaves the exact sum alone."""
    rng = np.random.default_rng(seed)
    b = float(np.log2(cond))
    m = min(n, 1 << 16)
    if m < 6:
        big = 2.0 ** round(b)
        core = np.array([big, 1.0 + rng.random(), -big, 0.5, -0.25][:m])
    else:
        h = m // 2
        e = np.rint(rng.random(h) * b)
        e[0], e[-1] = round(b), 0
        core = np.empty(m)
        core[:h] = (2 * rng.random(h) - 1) * 2.0 ** e
        scale = 1 << 80                             # every value is a multiple of 2^-53 times 2^e, e >= 0
        exact = 0
        for v in core[:h]:
            p, q = float(v).as_integer_ratio()
            exact += p * (scale // q)
        e2 = np.rint(np.linspace(b, 0, m - h))
        v2 = (2 * rng.random(m - h) - 1) * 2.0 ** e2
        for i, v in enumerate(v2):
            p, q = float(v).as_integer_ratio()
            xi = (p * (scale // q) - exact) / scale   # correctly rounded (int / int)
            core[h + i] = xi
            p, q = xi.as_integer_ratio()
            exact += p * (scale // q)
    if n == m:
        return core[rng.permutation(n)]
    k = (n - m) // 2
    y = (2 * rng.random(k) - 1) * 2.0 ** np.rint(rng.random(k) * b)
    rest = np.concatenate([y, -y, np.zeros(n - m - 2 * k)])
    return np.concatenate([core, rest])[rng.permutation(n)]
