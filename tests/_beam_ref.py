"""Reference rules of beam search (DESIGN.md section 3, "Beam search"), for the tests.

select(): steps 1-3 of transformers' _beam_search (do_sample=False) in float64 with our tie rule: per item, the
K = 2k best of lp + running score over its k * V candidates, ties to the lowest flat index beam * V + token; the hits
(EOS, or the max-length step); the k running picks, the best of score + hit * -1e9, ties to the lower index. lp is
the greedy log-prob of a row, log_softmax over its non-NaN logits.

hf_replay(): steps 4-6 on a sequence of records, computed by the installed transformers helpers themselves
(_update_finished_beams, _check_early_stop_heuristic, _beam_search_has_unfinished_sequences), the yardstick of the
host's fp32 replay."""
from types import SimpleNamespace

import numpy as np
import torch


def log_probs(x):
    """float64 greedy log-probs of one row x [V]: (x - max) - log(sum exp(x - max)) over the non-NaN tokens"""
    x = np.asarray(x, dtype=np.float64)
    ok = ~np.isnan(x)
    m = np.max(x[ok]) if ok.any() else np.nan
    if not np.isfinite(m):
        return np.full_like(x, np.nan)
    w = np.exp(np.where(ok, x - m, -np.inf)).sum()
    return (x - m) - np.log(w)


def select(logits, scores, k, eos=-1, last_step=False):
    """logits [B*k, V] (host), scores [B*k] -> per item (candidates [(score, beam, token)] * K best first, picks [k],
    hits [K], the score of the best candidate left out) in float64"""
    logits = np.asarray(logits, dtype=np.float64)
    Bk, V = logits.shape
    out = []
    for i in range(Bk // k):
        s = np.stack([log_probs(logits[i * k + j]) + float(scores[i * k + j]) for j in range(k)]).reshape(-1)
        s = np.where(np.isnan(s), -np.inf, s)
        order = np.lexsort((np.arange(k * V), -s))[:2 * k + 1]      # score descending, then flat index ascending
        top = [(float(s[o]), int(o // V), int(o % V)) for o in order[:2 * k]]
        nxt = float(s[order[2 * k]]) if len(order) > 2 * k else -np.inf
        hits = [last_step or (eos >= 0 and c[2] == eos) for c in top]
        masked = [c[0] - (1e9 if h else 0.0) for c, h in zip(top, hits)]
        picks = sorted(range(2 * k), key=lambda q: (-masked[q], q))[:k]
        out.append((top, picks, hits, nxt))
    return out


def gap(a, b):
    """the bound within which two candidate scores may swap places: 1e-5 + 2^-22 |s|"""
    return 1e-5 + 2.0 ** -22 * max(abs(a), abs(b))


def _hf():
    from transformers.generation.utils import GenerationMixin
    return GenerationMixin


def hf_replay(steps, B, k, S, n, eos, fill, length_penalty, early_stopping):
    """HF's own steps 4-6 over records: steps = [(score f32 [B, K], beam [B, K], token [B, K], pick [B, k]), ...].
    Returns (stop step, sequences [B, k, n], beam_scores [B, k], beam_indices [B, k, n], is_sent_finished) exactly as
    _beam_search holds them, the running beams taken from the picks."""
    G = _hf()
    me = SimpleNamespace(_gather_beams=G._gather_beams)
    K = 2 * k
    max_length = S + n
    running = torch.full((B, k, max_length), fill, dtype=torch.int64)
    sequences = running.clone()
    running_idx = torch.full((B, k, n), -1, dtype=torch.int32)
    beam_indices = running_idx.clone()
    beam_scores = torch.full((B, k), -1e9, dtype=torch.float32)
    is_fin = torch.zeros((B, k), dtype=torch.bool)
    unsat = torch.ones((B, 1), dtype=torch.bool)
    mask = torch.cat((torch.ones(k, dtype=torch.bool), torch.zeros(K - k, dtype=torch.bool)))
    cur_len = S
    for t, (score, beam, tok, pick) in enumerate(steps):
        topk_seq = G._gather_beams(running, beam)
        topk_seq[:, :, cur_len] = tok
        topk_idx = G._gather_beams(running_idx, beam)
        topk_idx[:, :, cur_len - S] = (beam + torch.arange(B)[:, None] * k).to(torch.int32)
        hit = torch.full((B, K), cur_len + 1 >= max_length)
        if eos is not None:
            hit = hit | (tok == eos)
        run_lp = score + hit.to(torch.float32) * -1.0e9
        running = G._gather_beams(topk_seq, pick)
        run_scores = G._gather_beams(run_lp, pick)
        running_idx = G._gather_beams(topk_idx, pick)
        sequences, beam_scores, beam_indices, is_fin = G._update_finished_beams(
            me, sequences, topk_seq, beam_scores, score.clone(), beam_indices, topk_idx, unsat, is_fin, hit, mask,
            k, cur_len, S, length_penalty, early_stopping)
        cur_len += 1
        unsat = G._check_early_stop_heuristic(unsat, run_scores, beam_scores, is_fin, cur_len, max_length, S,
                                              early_stopping, length_penalty)
        if not bool(G._beam_search_has_unfinished_sequences(unsat, is_fin, hit, early_stopping)):
            return t, sequences, beam_scores, beam_indices, is_fin
    return None, sequences, beam_scores, beam_indices, is_fin
