"""Float64 / integer restatement of the device's min-p, typical, epsilon and eta warpers (DESIGN.md section 3,
"Min-p, typical, epsilon and eta"; sampling.cu, warp_row), on top of _nucleus_ref's temperature / top-k / top-p.

Each warper acts on the set the stages before it kept, in HF's order, with w = fp32 exp(z - z_max), q = rint(w * 2^36),
Q = sum q and D = sum rint(q * (z_max - z)) over that set:
  min-p    keep iff w >= fp32(min_p)
  typical  c = D / Q, d = fp32(|(z_max - z) - c|); keep j iff the mass of the tokens with d < d_j is < fp32(p) * Q;
           z_max then becomes the largest kept z
  epsilon  keep iff q >= fp32(eps) * Q, or z = z_max
  eta      H = D / Q + log Q - 36 log 2, eta = min(e, sqrt(e) exp(-H)) with e = fp32(eta_cutoff); keep iff q >= eta * Q,
           or z = z_max
warp_keep also reports how far each decision lies from its boundary, so that a test can tell the rows whose kept set
does not depend on rounding: as in _nucleus_ref, w here is the correctly rounded fp32 exp while the device's expf may
differ by up to 2 ulps."""
import math

import numpy as np

import _nucleus_ref as N

OFF = (0.0, 1.0, 0.0, 0.0)      # min_p, typical_p, epsilon, eta


def _mass(z, kept, zmax):
    with np.errstate(invalid="ignore", over="ignore"):
        w = np.exp((z - zmax).astype(np.float64)).astype(np.float32)
    q = np.where(kept, np.rint(w.astype(np.float64) * N.MASS_SCALE), 0.0)
    return w, q


def _stats(z, kept, zmax):
    _, q = _mass(z, kept, zmax)
    dz = np.where(kept & (q > 0), float(zmax) - z.astype(np.float64), 0.0)
    return q, int(q.sum()), int(np.rint(q * dz).sum())


def warp_keep(z, keep, warpers):
    """-> (kept, zmax, margins): the warpers (min_p, typical_p, epsilon, eta; OFF: none) over the kept set `keep` of
    z (fp32). margins: a dict of the smallest relative distance of any decision to its threshold ("min_p", "eps",
    "eta"), and for typical the mass distances of the boundary's levels ("typ_mass") and the gap in d between the
    last kept and the first dropped level ("typ_gap")."""
    mp, ty, ep, et = (float(np.float32(v)) for v in warpers)
    z = np.asarray(z, dtype=np.float32)
    kept = keep.copy()
    zmax = np.float32(z[kept].max())
    m = {}
    if mp > 0:
        w, _ = _mass(z, kept, zmax)
        kept &= w >= np.float32(mp)
        dist = np.abs(w[keep & (z != zmax)].astype(np.float64) - mp) / mp   # (w = 1 exactly at zmax)
        m["min_p"] = float(dist.min()) if dist.size else 1.0
    if ty < 1:
        q, Q, D = _stats(z, kept, zmax)
        c = D / Q
        d = np.abs((float(zmax) - z.astype(np.float64)) - c).astype(np.float32)
        P = ty * Q
        levels = np.unique(d[kept])
        below, new = 0.0, np.zeros_like(kept)
        last_kept = first_drop = None
        for v in levels:
            g = kept & (d == v)
            if below < P:
                new |= g
                last_kept = (v, below)
            elif first_drop is None:
                first_drop = (v, below)
            below += float(q[g].sum())
        m["typ_mass"] = min([abs(t[1] - P) / Q for t in (last_kept, first_drop) if t is not None] + [1.0])
        m["typ_gap"] = float(first_drop[0] - last_kept[0]) if first_drop is not None else 1.0
        kept = new
        zmax = np.float32(z[kept].max())
    for name, e in (("eps", ep), ("eta", et)):
        if e <= 0:
            continue
        q, Q, D = _stats(z, kept, zmax)
        if name == "eps":
            thr = e * Q
        else:
            H = D / Q + math.log(Q) - 36.0 * math.log(2.0)
            thr = min(e, math.sqrt(e) * math.exp(-H)) * Q
        cand = kept & (z != zmax)
        dist = np.abs(q[cand] - thr) / thr
        m[name] = float(dist.min()) if dist.size else 1.0
        kept &= (q >= thr) | (z == zmax)
    return kept, zmax, m


def decided(margins, rel, gap):
    """whether every decision of warp_keep lies at least rel (relative) from its threshold, and typical's boundary
    levels at least `gap` apart in d"""
    return all(v >= (gap if k == "typ_gap" else rel) for k, v in margins.items())


def choose(x, T, k, p, warpers, u):
    """-> (token, kept, zmax, margins, draw margin): the rules' token for logits x (no penalty) with temperature T > 0,
    top-k k, top-p p and the warpers, the final kept set, its maximum, warp_keep's margins (plus "top_p": whether the
    top-p boundary is decided at 1e-6) and the draw's distance from its interval's edges relative to W"""
    z = N.scaled(x, T)
    keep, tm = N.top_p_keep(z, N.topk_keep(z, k), p)
    kept, zmax, m = warp_keep(z, keep, warpers)
    m["top_p"] = 1.0 if N.decided(tm, 1e-6) else 0.0
    w = np.where(kept, np.exp(z.astype(np.float64) - float(zmax)), 0.0)
    Pc = np.cumsum(w)
    W = Pc[-1]
    t = u * W
    over = np.flatnonzero(kept & (w > 0) & (Pc > t))
    j = int(over[0]) if over.size else int(np.flatnonzero(w > 0)[-1])
    return j, kept, zmax, m, min(t - (Pc[j] - w[j]), Pc[j] - t) / W


def logprob(z, kept, zmax, j):
    """the device's log-prob of token j over the final set, in float64: (z_j - zmax) - log W"""
    W = np.exp(z[kept].astype(np.float64) - float(zmax)).sum()
    return (float(z[j]) - float(zmax)) - math.log(W)

