"""float64 restatement of the log-prob rule of sampling.cu (DESIGN.md section 3), for one logits row.

x is the engine's row: bf16 values in fp32 storage. The processed scores s are HF's `scores`: x for a greedy row
(T = 0), fp32(x / T) over the tokens the top-k rule keeps (-inf elsewhere) for a sampled row; a NaN is never kept.
m = max s, W = sum of exp(s - m) over the kept tokens, lp(j) = (s_j - m) - log W. Here W and the logarithm are
float64; only s itself is the fp32 value the device computes.
"""
import numpy as np

import _sampling_ref as R

LOGPROBS_MAX = 20


def processed(x, T, k):
    """-> (s float64 [V] with -inf where not kept, kept mask)"""
    x = np.asarray(x, dtype=np.float32)
    if T > 0:
        kept = R.kept_mask(x, T, k)
        with np.errstate(over="ignore"):
            z = (x / np.float32(T)).astype(np.float32)
    else:
        kept = ~np.isnan(x)
        z = x
    s = np.where(kept, z.astype(np.float64), -np.inf)
    return s, kept


def logprobs(x, T, k, n, chosen):
    """-> (lp of token `chosen`, top ids [n], top lps [n]) by the rule; a row without a finite maximum gives NaN
    and id -1 at every place"""
    s, kept = processed(x, T, k)
    m = np.max(s) if kept.any() else -np.inf
    if not np.isfinite(m):
        return float("nan"), [-1] * n, [float("nan")] * n
    with np.errstate(under="ignore"):
        W = np.sum(np.exp(s[kept] - m))
    lp = (s - m) - np.log(W)
    idx = np.nonzero(kept)[0]
    order = idx[np.lexsort((idx, -s[idx]))][:n]       # s descending, then the lowest index
    ids = [int(i) for i in order] + [-1] * (n - len(order))
    lps = [float(lp[i]) for i in order] + [float("-inf")] * (n - len(order))
    return float(lp[chosen]), ids, lps


def close(got, want):
    """|got - want| <= 1e-5 + 2^-22 |want| (inf and NaN must match exactly)"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    same = (got == want) | (np.isnan(got) & np.isnan(want))
    fin = np.isfinite(want) & np.isfinite(got)
    diff = np.abs(np.where(fin, got - np.where(fin, want, 0), 0))
    ok = same | (fin & (diff <= 1e-5 + 2.0 ** -22 * np.abs(np.where(fin, want, 0))))
    return bool(ok.all())
