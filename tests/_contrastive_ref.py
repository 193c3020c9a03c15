"""Float64 restatement of contrastive search (transformers <= 4.55 _contrastive_search / _ranking_fast with
penalty_alpha = a and top_k = k; DESIGN.md section 3, "Contrastive search"), per prompt and step:
  p        softmax of the logits row z over its non-NaN entries
  c_1..k   the k most probable tokens, ties to the lower id
  s_j      max over the context rows h (the final-norm rows of the prompt's real columns so far) of cos(h, g_j)
  score_j  (1 - a) p_j - a s_j; j* the largest, ties to the lower j
HF masks left-padding columns with a large negative added to their cosines (cosine_matrix_mask); here they are simply
not context rows."""
import numpy as np
import torch


def probs(z):
    """p = softmax(z) in float64 over the non-NaN entries (NaN entries 0); a row without a finite maximum is NaN"""
    z = np.asarray(z, dtype=np.float64)
    ok = ~np.isnan(z)
    m = z[ok].max() if ok.any() else np.nan
    if not np.isfinite(m):
        return np.full(z.shape, np.nan)
    w = np.where(ok, np.exp(np.where(ok, z, -np.inf) - m), 0.0)
    return w / w.sum()


def candidates(z, k):
    """(tokens [k], p [k]): the k most probable tokens, best first, ties to the lower id"""
    p = probs(z)
    key = np.where(np.isnan(p), -1.0, p)
    order = np.lexsort((np.arange(len(p)), -key))[:k]
    return order, p[order]


def max_cos(ctx, g):
    """s [k]: the largest cosine of each candidate row g [k, D] against the context rows ctx [n, D] (float64)"""
    ctx = np.asarray(ctx, dtype=np.float64)
    g = np.asarray(g, dtype=np.float64)
    cos = (ctx @ g.T) / (np.linalg.norm(ctx, axis=1)[:, None] * np.linalg.norm(g, axis=1)[None, :])
    return cos.max(axis=0)


def rank(ctx, g, p, alpha):
    """(s [k], score [k], j*) of one prompt's step"""
    s = max_cos(ctx, g)
    score = (1.0 - alpha) * np.asarray(p, dtype=np.float64) - alpha * s
    return s, score, int(np.argmax(score))


def gap(a, b, rel=2e-3, abs_=1e-4):
    """the margin within which two float64 scores count as tied (the device computes in fp32 from bf16 rows)"""
    return abs_ + rel * max(abs(a), abs(b))


def decided(score, j, margin):
    """j's score beats every other candidate's by more than margin(a, b)"""
    return all(score[j] - score[i] > margin(score[j], score[i]) for i in range(len(score)) if i != j)


def generate(step, ctx0, z0, k, alpha, n, forced=None):
    """Contrastive search driven by `step(prefix_tokens, cand) -> (g [k, D], z [k, V])`, the candidates' final-norm
    rows and logits after the chosen tokens `prefix_tokens` so far. ctx0 [S_real, D]: the prompt's context rows; z0
    the prompt's last logits. forced [n]: take these tokens instead of the picks (teacher forcing; the rank is still
    reported). Returns a list of per-step dicts (cand, p, s, score, pick, token)."""
    ctx = np.asarray(ctx0, dtype=np.float64)
    z = z0
    out, chosen = [], []
    for t in range(n):
        cand, p = candidates(z, k)
        g, zs = step(chosen, cand)
        s, score, j = rank(ctx, g, p, alpha)
        out.append({"cand": cand, "p": p, "s": s, "score": score, "pick": j, "token": int(cand[j])})
        tok = int(cand[j]) if forced is None else int(forced[t])
        hit = np.nonzero(cand == tok)[0]
        if len(hit):
            g_t, z_t = g[hit[0]], zs[hit[0]]
        else:                           # a forced token outside this step's candidates (a near tie at the boundary)
            g1, z1 = step(chosen, np.array([tok]))
            g_t, z_t = g1[0], z1[0]
        chosen.append(tok)
        ctx = np.concatenate([ctx, np.asarray(g_t, dtype=np.float64)[None]], axis=0)
        z = z_t
    return out


def oracle_step_fn(sd, cfg, ids, feats):
    """step() of generate() for one prompt [1, S] on the oracle (oracle/vcl_oracle.py llm_forward): returns
    (step, ctx0, z0). Each call recomputes the prefix from the prompt, so it is slow but simple."""
    from oracle import vcl_oracle as O
    logits, hs, past = O.llm_forward(sd, cfg, ids, feats)
    ctx0 = hs[-1][0].double().cpu().numpy()
    z0 = logits[0, -1].double().cpu().numpy()
    cache = {(): past}

    def step(prefix, cand):
        key = tuple(prefix)
        if key not in cache:
            prev = cache[key[:-1]]
            _, _, p2 = O.llm_forward(sd, cfg, torch.tensor([[key[-1]]], device=ids.device), feats, prev)
            cache[key] = p2
        past_ = cache[key]
        gs, zs = [], []
        for c in cand:
            lg, h, _ = O.llm_forward(sd, cfg, torch.tensor([[int(c)]], device=ids.device), feats, past_)
            gs.append(h[-1][0, -1].double().cpu().numpy())
            zs.append(lg[0, -1].double().cpu().numpy())
        return np.stack(gs), zs

    return step, ctx0, z0
