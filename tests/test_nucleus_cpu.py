"""CPU tests of top-p and the repetition penalty: the float64 restatement of the device rules (_nucleus_ref) against
the installed transformers processors, the host-side rejections, and the token sets generate_requests writes at
admission, preemption / resume, chunked prefill and continuation (with the fake engines of test_paged_kv_cpu.py)."""
import numpy as np
import pytest
import torch

import _nucleus_ref as N
import test_paged_kv_cpu as P
from test_paged_kv_cpu import EOS, REQ0, FakeEngine, _model

V = 32003
EPS = 1e-4          # a tie group whose mass above lies within EPS * W of p * W is undecided (fp32 cumsum in HF)


def _rows(rng, n):
    """bf16 logits rows with many exact ties, one row with -inf stretches, one with all but 3 tokens at -inf"""
    x = torch.randn(n, V, generator=rng) * 3
    x = x.to(torch.bfloat16).float()
    x[1, : V // 2] = float("-inf")
    x[2, 3:] = float("-inf")
    return x


def _hf(ids, scores, T, k, p, r):
    from transformers.generation.logits_process import (RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper,
                                                        TopKLogitsWarper, TopPLogitsWarper)
    s = scores.clone()
    if r != 1.0:
        s = RepetitionPenaltyLogitsProcessor(penalty=r)(ids, s)
    z = TemperatureLogitsWarper(T)(ids, s.clone())
    out = TopKLogitsWarper(top_k=k)(ids, z.clone()) if k else z.clone()
    if p < 1.0:
        out = TopPLogitsWarper(top_p=p)(ids, out)
    return z, out


@pytest.mark.parametrize("T", [0.2, 1.5])
@pytest.mark.parametrize("k", [0, 50])
@pytest.mark.parametrize("r", [1.0, 0.8, 1.3])
def test_rules_match_transformers(T, k, r):
    """Penalized z bit-identical to torch's; the kept sets equal on every decided row; few rows undecided"""
    rng = torch.Generator().manual_seed(int(T * 10) * 1000 + k * 10 + int(r * 10))
    x = _rows(rng, 12)
    ids = torch.randint(0, V, (12, 300), generator=rng)
    ids[3] = torch.arange(300)      # a row whose set holds the -inf-free head only
    undecided = 0
    for p in (0.0, 0.5, 0.9, 0.999, 1.0):
        z_hf, out_hf = _hf(ids, x, T, k, p, r)
        for b in range(x.shape[0]):
            z = N.scaled(N.penalize(x[b].numpy(), r, ids[b].tolist()), T)
            np.testing.assert_array_equal(z.view(np.uint32), z_hf[b].numpy().view(np.uint32))
            keep, margins = N.top_p_keep(z, N.topk_keep(z, k), p)
            if not N.decided(margins, EPS):
                undecided += 1
                continue
            hf_keep = torch.isfinite(out_hf[b]).numpy() | (out_hf[b].numpy() == np.inf)
            if p == 0.0:    # HF keeps one token of the largest tie group; the rule keeps the group whole
                assert keep[hf_keep].all() and (z[keep] == z[keep].max()).all()
                continue
            fin = np.isfinite(z)     # -inf tokens carry no mass: HF may keep them inside the cut, the rule too
            np.testing.assert_array_equal(keep & fin, hf_keep & fin)
    # at T = 1.5 over the whole vocabulary the boundary often falls inside a large group of equal bf16 logits, which
    # HF's sort splits in an arbitrary order: those rows are undecided by construction
    print(f"T={T} k={k} r={r}: {undecided} of 60 rows undecided")
    assert undecided <= (36 if k == 0 else 15), f"{undecided} undecided rows of 60"


def test_ties_at_the_boundary_kept_whole():
    z = np.array([3.0, 1.0, 1.0, 1.0, -2.0], dtype=np.float32)
    keep, _ = N.top_p_keep(z, np.ones(5, bool), 0.8)
    # w = 1, e^-2 x 3, e^-5: the mass above the tie group is 1 / W = 0.708 < 0.8, so all three ties stay; above the
    # last token it is 0.995
    assert keep.tolist() == [True, True, True, True, False]
    keep, _ = N.top_p_keep(z, np.ones(5, bool), 0.0)
    assert keep.tolist() == [True, False, False, False, False]


def test_penalty_rule_signs():
    x = np.array([-2.0, 2.0, 0.0, -0.5, 4.0], dtype=np.float32)
    xp = N.penalize(x, 2.0, [0, 1, 2])
    assert xp.tolist() == [-4.0, 1.0, 0.0, -0.5, 4.0]


# ---- host rejections ----------------------------------------------------------------------------------------------
def _fake_model(slots=4, kv_blocks=None, **kw):
    eng = TokenSetFake(640, slots, kv_blocks or 0, **kw)
    m = _model(eng, max_batch=slots, max_seq=640, kv_blocks=kv_blocks)
    m._SLOT_CHUNK = 8
    return m, eng


@pytest.mark.parametrize("kw", [dict(top_p=1.5), dict(top_p=-0.1), dict(top_p=float("nan")),
                                dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0),
                                dict(repetition_penalty=float("inf")), dict(repetition_penalty=float("nan"))])
def test_rejections(kw):
    m, eng = _fake_model()
    req = {"input_ids": torch.tensor([REQ0, 5, 6])}
    with pytest.raises(ValueError):
        m.generate_requests([req], max_new_tokens=4, **kw)
    with pytest.raises(ValueError):
        m.generate_requests([dict(req, **kw)], max_new_tokens=4)
    with pytest.raises(ValueError):
        m._nucleus_args(kw.get("top_p", 1.0), kw.get("repetition_penalty", 1.0))
    assert eng.calls == []


def test_vocabulary_limit():
    m, _ = _fake_model()
    m.config.vocab_size = 60000
    with pytest.raises(ValueError, match="vocabulary"):
        m._nucleus_args(0.9, 1.0)
    assert m._nucleus_args(1.0, 1.0) == (1.0, 1.0)


# ---- token sets in flight -----------------------------------------------------------------------------------------
class TokenSetFake(FakeEngine):
    """FakeEngine with the 32-bit sampler's table and token sets: it records every set_token_set and, as the device
    does, adds each token a penalized slot's prefill or decode step produces to that slot's set"""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.rep = [1.0] * self.n_slots
        self.sets = [set() for _ in range(self.n_slots)]
        self.writes = []                      # (slot, ids)

    def set_sampling(self, clips, temperature, top_k, seed):
        super().set_sampling(clips, temperature, top_k, seed)
        for s in clips:
            self.rep[s] = 1.0

    def set_sampling_ex(self, clips, temperature, top_k, seed, top_p, repetition_penalty):
        super().set_sampling(clips, temperature, top_k, seed)
        for s, r in zip(clips, repetition_penalty):
            self.rep[s] = r

    def set_token_set(self, entry, ids):
        ids = [int(t) for t in torch.as_tensor(ids).reshape(-1)]
        self.writes.append((entry, ids))
        self.sets[entry] = set(ids)

    def _mark(self, s, tok):
        if self.rep[s] != 1.0:
            self.sets[s].add(int(tok))

    def _prefill(self, s, ids):
        tok = super()._prefill(s, ids)
        self._mark(s, tok)
        return tok

    def slot_decode(self, first_tok, positions, n_new):
        out = super().slot_decode(first_tok, positions, n_new)
        for s in range(out.shape[0]):
            for t in out[s, 1:].tolist():
                self._mark(s, t)
        return out


def _requests(n, rng, long=False):
    reqs = []
    for i in range(n):
        S = int(torch.randint(600, 630, (1,), generator=rng)) if long and i % 3 == 0 else \
            int(torch.randint(5, 40, (1,), generator=rng))
        ids = torch.cat([torch.tensor([REQ0 + i]), torch.randint(1, 30000, (S - 1,), generator=rng)])
        reqs.append({"input_ids": ids, "max_new_tokens": int(torch.randint(3, 12, (1,), generator=rng)),
                     "repetition_penalty": 1.2 if i % 2 == 0 else 1.0})
    return reqs


def _check_sets(eng, outs, reqs):
    """every write of a penalized request's set is its prompt, or (at a resume) a prefix of its returned sequence"""
    by_first = {REQ0 + i: i for i in range(len(reqs))}
    n_resume = 0
    for s, ids in eng.writes:
        i = by_first[ids[0]]
        seq = outs[i][0].tolist()
        S = torch.as_tensor(reqs[i]["input_ids"]).numel()
        assert reqs[i]["repetition_penalty"] != 1.0
        assert len(ids) >= S and ids == seq[:len(ids)], (i, len(ids), S)
        n_resume += len(ids) > S
    assert {by_first[ids[0]] for _, ids in eng.writes} == {i for i, r in enumerate(reqs) if r["repetition_penalty"] != 1.0}
    return n_resume


@pytest.mark.parametrize("packed", [False, True])
def test_token_sets_contiguous(packed):
    rng = torch.Generator().manual_seed(1)
    reqs = _requests(10, rng)
    m, eng = _fake_model()
    outs = m.generate_requests(reqs, eos_token_id=EOS, packed_admission=packed)
    _check_sets(eng, outs, reqs)
    assert eng.rep == [1.0] * eng.n_slots      # every slot greedy, without penalty, after the call


@pytest.mark.parametrize("packed", [False, True])
def test_token_sets_paged_preemption(packed):
    rng = torch.Generator().manual_seed(2)
    reqs = _requests(10, rng)
    for r in reqs:
        r["max_new_tokens"], r["repetition_penalty"] = 200, 1.2
    m, eng = _fake_model(kv_blocks=6)
    eng.lens = {i: torch.as_tensor(r["input_ids"]).numel() + 200 for i, r in enumerate(reqs)}
    outs = m.generate_requests(reqs, eos_token_id=None, packed_admission=packed)
    assert m.last_kv_stats["preemptions"] > 0
    assert _check_sets(eng, outs, reqs) > 0     # resumed requests rebuilt their sets from prompt + tokens
    assert not eng.violations


def test_token_sets_chunked():
    rng = torch.Generator().manual_seed(3)
    reqs = _requests(6, rng, long=True)
    m, eng = _fake_model(kv_blocks=40)
    eng.lens = {i: torch.as_tensor(r["input_ids"]).numel() + r["max_new_tokens"] for i, r in enumerate(reqs)}
    eng.slots_prefill_chunk = lambda slots, starts, totals, ids_list, feats, vs: torch.tensor(
        [eng._chunk(s, st, tot, ids) for s, st, tot, ids in zip(slots, starts, totals, ids_list)], dtype=torch.int32)

    def chunk(s, start, total, ids):
        ids = [int(t) for t in torch.as_tensor(ids).reshape(-1)]
        for j, t in enumerate(ids):
            eng._write(s, start + j, t)
        if start == 0:
            eng.owner[s] = ids[0] - REQ0
        tok = P._tok(eng._read(s, start + len(ids)), start + len(ids) - 1, eng.seed[s])
        eng._mark(s, tok)
        return tok
    eng._chunk = chunk
    outs = m.generate_requests(reqs, eos_token_id=None, chunked_prefill=True)
    assert m.last_kv_stats["chunk_calls"] > 0
    _check_sets(eng, outs, reqs)
    # a chunked prompt's set is written before each of its chunk calls, so no discarded chunk token stays in it
    long = [i for i, r in enumerate(reqs) if torch.as_tensor(r["input_ids"]).numel() > 512 and i % 2 == 0]
    for i in long:
        assert sum(1 for _, ids in eng.writes if ids[0] == REQ0 + i) >= 2


# ---- continuations (sessions) -------------------------------------------------------------------------------------
@pytest.mark.parametrize("packed", [False, True])
def test_token_sets_of_continuations_are_the_whole_conversation(packed):
    """A "continues" request's set is the kept conversation, then its new text: the whole conversation, as
    generate_continue's; it is written once, before its tail prefill, and is a prefix of what the turn returns"""
    import test_sessions_cpu as SC

    class SessionSetFake(TokenSetFake, SC.SessionFake):
        pass

    eng = SessionSetFake(4, 12)
    m = _model(eng, max_batch=4, max_seq=SC.MAX_SEQ, kv_blocks=12)
    m._SLOT_CHUNK = 8
    eng.model = m
    convs = SC.conversations(5, 3, seed=4)
    res = SC.run_sessions(m, convs, 3, packed_admission=packed, repetition_penalty=1.2)
    assert not eng.violations
    for t in (1, 2):
        for c in range(len(convs)):
            conv = res[c][t - 1] + convs[c][t][0].tolist()       # the kept conversation and the new turn
            assert conv in [ids for _, ids in eng.writes], (t, c)
            assert res[c][t][:len(conv)] == conv, (t, c)
    # and no continuation's set is its new text alone
    for c in range(len(convs)):
        for t in (1, 2):
            assert convs[c][t][0].tolist() not in [ids for _, ids in eng.writes]


# ---- the unseeded stepwise path -----------------------------------------------------------------------------------
@pytest.mark.parametrize("T,k,p,r", [(0.7, 50, 0.9, 1.3), (1.5, 0, 0.5, 0.8), (0.2, 0, 0.999, 1.0),
                                     (1.0, 5, 1.0, 1.1), (0.7, 0, 0.0, 1.2)])
def test_host_processors_match_transformers(T, k, p, r):
    """The stepwise path's processors (_host_processors) against HF's four, on the same fp32 logits: bit for bit"""
    from video_chatgpt.model import VideoChatGPTLlamaForCausalLM as M
    rng = torch.Generator().manual_seed(int(T * 100) + k + int(p * 1000))
    x = _rows(rng, 6)
    ids = torch.randint(0, V, (6, 200), generator=rng)
    _, want = _hf(ids, x, T, k, p, r)
    got = M._host_processors(ids, x.clone(), True, T, k, p, r)
    assert torch.equal(got, want)
    # greedy: the penalty only
    from transformers.generation.logits_process import RepetitionPenaltyLogitsProcessor
    g = M._host_processors(ids, x.clone(), False, T, k, p, r)
    assert torch.equal(g, RepetitionPenaltyLogitsProcessor(penalty=r)(ids, x.clone()) if r != 1.0 else x)
