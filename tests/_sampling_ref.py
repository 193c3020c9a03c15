"""Float64 restatement of the device sampler's rules (DESIGN.md section 3; sampling.cu) and Philox4x32-10 in numpy.

choose() gives the token the rules pick for one row of logits and draw u, with how far u lies from the edges of the
chosen token's interval (relative to W); decided() tells whether a choice holds for every logit vector within
+-3 bf16 ulps of the given one (the sampling analogue of the greedy near-tie rule)."""
import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def philox4x32_10(key, counter):
    """key (k0, k1), counter (c0, c1, c2, c3): uint32 scalars or broadcastable arrays -> the four output words"""
    k0, k1 = (np.asarray(k, dtype=np.uint64) for k in key)
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) for c in counter)
    for _ in range(10):
        p0 = np.uint64(M0) * c0
        p1 = np.uint64(M1) * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(MASK)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(MASK)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0 = (k0 + np.uint64(W0)) & np.uint64(MASK)
        k1 = (k1 + np.uint64(W1)) & np.uint64(MASK)
    return c0, c1, c2, c3


def uniform(seed, counter):
    """u of the row with 64-bit `seed` at Philox counter (counter, 0, 0, 0): (word0 >> 8) * 2^-24 (exact in fp64)"""
    seed = int(seed) % 2 ** 64
    w0 = philox4x32_10((seed & MASK, seed >> 32), (np.asarray(counter, dtype=np.uint64), 0, 0, 0))[0]
    return (w0 >> np.uint64(8)).astype(np.float64) * 2.0 ** -24


def argmax_rule(x):
    """argmax_kernel's token: lowest index of the largest non-NaN logit, 0 when none is above -inf"""
    x = np.asarray(x, dtype=np.float32)
    ok = ~np.isnan(x)
    if not ok.any() or np.nanmax(x) == -np.inf:
        return 0
    return int(np.flatnonzero(ok & (x == np.nanmax(x)))[0])


def kept_mask(x, T, k):
    """the kept tokens: z >= z of the k-th largest logit (z = fp32(x / T)); k = 0 or k >= V keeps all; NaN never"""
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(over="ignore"):
        z = x / np.float32(T)
    V = x.size
    if 0 < k < V:
        xs = np.sort(np.where(np.isnan(x), -np.inf, x))[::-1]
        return z >= np.float32(xs[k - 1]) / np.float32(T)
    return ~np.isnan(z)


def choose(x, T, k, u):
    """-> (token, margin): the rules' token for logits x (fp32, bf16-representable) and draw u, and the distance of
    u * W from the nearer edge of the token's interval over W (None for an arg-max row)"""
    x = np.asarray(x, dtype=np.float32)
    if T == 0:
        return argmax_rule(x), None
    with np.errstate(over="ignore"):
        z = x / np.float32(T)
    zmax = np.nanmax(z) if (~np.isnan(z)).any() else np.float32(np.nan)
    if not np.isfinite(zmax):
        return argmax_rule(x), None
    keep = kept_mask(x, T, k)
    w = np.where(keep, np.exp(z.astype(np.float64) - float(zmax)), 0.0)
    P = np.cumsum(w)
    W = P[-1]
    t = u * W
    over = np.flatnonzero(keep & (w > 0) & (P > t))
    j = int(over[0]) if over.size else int(np.flatnonzero(w > 0)[-1])     # rounding past the end: last nonzero w
    lo = P[j] - w[j]
    return j, min(t - lo, P[j] - t) / W


def bf16_ulp(x):
    """the bf16 unit in the last place at |x| (the smallest normal's for 0)"""
    a = np.maximum(np.abs(np.asarray(x, dtype=np.float64)), 2.0 ** -126)
    return 2.0 ** (np.floor(np.log2(a)) - 7)


def decided(x, T, k, u, j, ulps=3):
    """Whether every logit vector within +-ulps bf16 ulps of x picks token j for the draw u. The edges of j's
    interval move furthest when the kept logits before j go up and the rest down (lower edge), or the logits up to
    j go down and those after it up (upper edge); a k-th / (k+1)-th gap of at most 2 * ulps ulps may change the
    kept set and counts as undecided."""
    x = np.asarray(x, dtype=np.float64)
    if T == 0:
        return True
    V = x.size
    d = ulps * bf16_ulp(x)
    if 0 < k < V:
        xs = np.sort(x)[::-1]
        if xs[k - 1] - xs[k] <= 2 * ulps * bf16_ulp(xs[k - 1]):
            return False
    keep = kept_mask(x.astype(np.float32), T, k)
    if not keep[j]:
        return False
    c = x[keep].max()
    idx = np.arange(V)

    def frac(up, upto):
        xp = np.where(up, x + d, x - d)
        w = np.where(keep, np.exp((xp - c) / T), 0.0)
        return w[idx <= upto].sum() / w.sum() if upto >= 0 else 0.0
    lo_max = frac(idx < j, j - 1)          # the largest the lower edge can get
    hi_min = frac(idx > j, j)              # the smallest the upper edge can get
    return lo_max <= u < hi_min
