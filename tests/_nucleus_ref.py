"""Float64 restatement of the repetition penalty and top-p rules of the device sampler (DESIGN.md section 3;
sampling.cu, the 32-bit path), on top of _sampling_ref's temperature / top-k rules.

penalize() and scaled() are the fp32 operations themselves (bit-exact); top_p_keep() restates the fixed-point top-p
rule with float64 / integer arithmetic and reports, per tie group of z, how far its mass above lies from the
threshold, so that a test can tell the rows whose kept set does not depend on rounding at the boundary.

One difference from the device is stated, not modelled: the weights w = exp(z - z_max) are the correctly rounded fp32
values here, while the device's CUDA expf may differ by up to 2 ulps. A fixed-point mass then moves by at most
~2^-22 of its weight, so a kept set is exact only on rows whose tie groups lie outside a margin well above that
(the GPU tests use 1e-6 of W); inside it the helper's and the device's sets may differ at the boundary."""
import numpy as np

import _sampling_ref as R

MASS_SCALE = 2.0 ** 36          # fixed-point masses: q = rint(w * 2^36)


def penalize(x, r, tokens):
    """x' of one row: x fp32, r the penalty, tokens the token set (ids) -> fp32 copy with x < 0 ? x * r : x / r on the
    set (torch's where(score < 0, score * p, score / p) in fp32)"""
    x = np.asarray(x, dtype=np.float32).copy()
    if r == 1.0:
        return x
    r = np.float32(r)
    m = np.zeros(x.size, dtype=bool)
    ids = np.asarray(list(tokens), dtype=np.int64)
    m[ids[(ids >= 0) & (ids < x.size)]] = True
    with np.errstate(over="ignore", invalid="ignore"):
        x[m] = np.where(x[m] < 0, x[m] * r, x[m] / r)
    return x


def scaled(xp, T):
    """z = fp32(x' / T) (T = 0: T = 1, the greedy row's scores)"""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(xp, dtype=np.float32) / np.float32(T if T > 0 else 1.0)


def topk_keep(z, k):
    """top-k on z: z >= the k-th largest non-NaN z (ties kept); k = 0 or k >= V keeps every non-NaN token"""
    z = np.asarray(z, dtype=np.float32)
    ok = ~np.isnan(z)
    if 0 < k < z.size:
        zs = np.sort(np.where(ok, z, -np.inf))[::-1]
        return ok & (z >= zs[k - 1])
    return ok


def top_p_keep(z, keep, p):
    """-> (kept, margins): top-p over the top-k kept tokens `keep` of z. w = fp32 exp(z - z_max), q = rint(w * 2^36),
    Q = sum q, M(j) = sum of q over the kept tokens with z strictly above z_j; j stays iff z_j = z_max or
    M(j) < fp64(p) * Q. margins: per tie group of z (largest first) the pair (M / Q - p, (M + group mass - smallest w)
    / Q - p), the range HF's ascending sort can give its tokens' mass above."""
    z = np.asarray(z, dtype=np.float32)
    if p >= 1.0 or not keep.any():
        return keep.copy(), []
    zmax = z[keep].max()
    with np.errstate(invalid="ignore", over="ignore"):
        w = np.exp((z - zmax).astype(np.float64)).astype(np.float32)
    q = np.where(keep, np.rint(w.astype(np.float64) * MASS_SCALE), 0.0).astype(np.uint64)
    Q = int(q.sum())
    P = float(np.float32(p)) * float(Q)
    vals = np.unique(z[keep])[::-1]
    kept = np.zeros_like(keep)
    margins = []
    above = 0
    for v in vals:
        g = keep & (z == v)
        gm = int(q[g].sum())
        if v == zmax or float(above) < P:
            kept |= g
        if v != zmax:
            margins.append((above / Q - float(np.float32(p)), (above + gm - int(q[g].min())) / Q - float(np.float32(p))))
        above += gm
    return kept, margins


def decided(margins, eps):
    """whether no tie group's possible mass above lies within eps (relative to Q) of the threshold"""
    return all(hi < -eps or lo >= eps for lo, hi in margins)


def choose(x, T, k, p, r, tokens, u):
    """-> (token, kept, margin): the rules' token for logits x, the final kept set and the draw's margin (None for an
    arg-max row), as _sampling_ref.choose gives them with the penalty and top-p"""
    xp = penalize(x, r, tokens)
    if T == 0:
        return R.argmax_rule(xp), None, None
    z = scaled(xp, T)
    ok = ~np.isnan(z)
    zmax = z[ok].max() if ok.any() else np.float32(np.nan)
    if not np.isfinite(zmax):
        return R.argmax_rule(z), None, None
    keep, _ = top_p_keep(z, topk_keep(z, k), p)
    w = np.where(keep, np.exp(z.astype(np.float64) - float(zmax)), 0.0)
    Pc = np.cumsum(w)
    W = Pc[-1]
    t = u * W
    over = np.flatnonzero(keep & (w > 0) & (Pc > t))
    j = int(over[0]) if over.size else int(np.flatnonzero(w > 0)[-1])
    lo = Pc[j] - w[j]
    return j, keep, min(t - lo, Pc[j] - t) / W
