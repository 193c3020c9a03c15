"""Banned tokens on the host: the rules of _bans_ref.py against transformers' own processors, the stepwise path's
processors bit for bit, the argument checks, and (with fake engines) where generate_requests writes token histories and
ban tables: admission, chunked prefill, preemption / resume and session continuations."""
import pytest
import torch

import _bans_ref as BR
import test_paged_kv_cpu as P
from test_paged_kv_cpu import EOS, REQ0, _model
from test_nucleus_cpu import TokenSetFake

V = 32003


def _hf_banned(ids, ngram, words, eos, S, m):
    """the ids HF's three processors set to -inf, per row of ids [B, c]"""
    from transformers.generation.logits_process import (MinNewTokensLengthLogitsProcessor, NoBadWordsLogitsProcessor,
                                                         NoRepeatNGramLogitsProcessor)
    sc = torch.zeros(ids.shape[0], V)
    if ngram:
        sc = NoRepeatNGramLogitsProcessor(ngram)(ids, sc)
    if words is not None:
        sc = NoBadWordsLogitsProcessor(words, eos)(ids, sc)
    if eos is not None and m:
        sc = MinNewTokensLengthLogitsProcessor(S, m, eos)(ids, sc)
    return [set(torch.nonzero(torch.isinf(r))[:, 0].tolist()) for r in sc]


def _rows(rng, B, c, pads):
    """rows of c ids over a small alphabet (so n-grams repeat), left pads of 0 and runs of placeholder ids"""
    ids = torch.randint(3, 9, (B, c), generator=rng)
    for b in range(B):
        p = min(pads[b % len(pads)], c)
        ids[b, :p] = 0
        if c > p + 8:
            ids[b, p + 1:p + 6] = 32000
    return ids


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("c", [1, 2, 3, 4, 9, 40])
def test_rules_match_transformers(n, c):
    rng = torch.Generator().manual_seed(n * 100 + c)
    ids = _rows(rng, 6, c, [0, 2, 5])
    words = [[4], [5, 6], [3, 4, 5], [EOS], list(range(3, 3 + c + 1)), [6, 7, 8, 3]]   # one word longer than the row
    for eos in (EOS, None):
        S = max(c - 2, 0)
        want = _hf_banned(ids, n, words, eos, S, 3)
        for b in range(6):
            h = ids[b].tolist()
            assert BR.banned(h, n, words, eos, S, 3) == want[b], (b, eos)
    # each processor on its own
    for b, h in enumerate(ids.tolist()):
        assert BR.ngram_bans(h, n) == _hf_banned(ids, n, None, None, 0, 0)[b]
        assert BR.word_bans(h, [[EOS], [7]], EOS) == _hf_banned(ids, 0, [[EOS], [7]], EOS, 0, 0)[b] == {7}
        assert BR.word_bans(h, [[EOS]], None) == {EOS}
    assert BR.ngram_bans([5] * c, n) == ({5} if c >= n else set())   # (an n-gram needs c >= n ids)
    assert BR.ngram_bans([1, 2, 3][:max(n - 2, 0)], n) == set()          # c + 1 < n


def test_min_new_tokens_and_disabled_eos():
    ids = torch.tensor([[1, 5, 6, 7]])
    assert _hf_banned(ids, 0, None, EOS, 2, 3) == [{EOS}]               # 2 new < 3
    assert BR.eos_bans([1, 5, 6, 7], EOS, 2, 3) == {EOS}
    assert BR.eos_bans([1, 5, 6, 7, 8], EOS, 2, 3) == set()             # 3 new
    assert BR.eos_bans([1, 5, 6, 7], None, 2, 3) == set()


def _fake_model(slots=4, kv_blocks=None, **kw):
    eng = BanFake(640, slots, kv_blocks or 0, **kw)
    m = _model(eng, max_batch=slots, max_seq=640, kv_blocks=kv_blocks)
    m._SLOT_CHUNK = 8
    return m, eng


@pytest.mark.parametrize("T,k,p,r,bans", [
    (0.7, 50, 0.9, 1.3, dict(no_repeat_ngram_size=2)),
    (1.5, 0, 0.5, 0.8, dict(bad_words_ids=[[4], [5, 6], [EOS], [3, 4, 5]])),
    (0.2, 0, 1.0, 1.0, dict(min_new_tokens=6)),
    (1.0, 5, 1.0, 1.1, dict(no_repeat_ngram_size=1, bad_words_ids=[[6, 7]], min_new_tokens=2)),
    (0.7, 0, 0.9, 1.0, dict(no_repeat_ngram_size=3, bad_words_ids=[[EOS]], min_new_tokens=1))])
def test_host_processors_match_transformers(T, k, p, r, bans):
    """_host_processors with bans against HF's processor list, in HF's order, on the same fp32 logits: bit for bit"""
    from transformers.generation.logits_process import (LogitsProcessorList, MinNewTokensLengthLogitsProcessor,
                                                         NoBadWordsLogitsProcessor, NoRepeatNGramLogitsProcessor,
                                                         RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper,
                                                         TopKLogitsWarper, TopPLogitsWarper)
    m, _ = _fake_model()
    rng = torch.Generator().manual_seed(int(T * 10) + k)
    S = 12
    for c in (S, S + 3, S + 9):
        ids = _rows(rng, 3, c, [0, 3])
        x = (torch.randn(3, V, generator=rng) * 3).bfloat16().float()
        x[0, 7] = -0.0
        b = m._ban_args(bans.get("no_repeat_ngram_size"), bans.get("bad_words_ids"), bans.get("min_new_tokens"), EOS)
        hf = LogitsProcessorList()
        if r != 1.0:
            hf.append(RepetitionPenaltyLogitsProcessor(r))
        if bans.get("no_repeat_ngram_size"):
            hf.append(NoRepeatNGramLogitsProcessor(bans["no_repeat_ngram_size"]))
        if bans.get("bad_words_ids") is not None:
            hf.append(NoBadWordsLogitsProcessor(bans["bad_words_ids"], EOS))
        if bans.get("min_new_tokens"):
            hf.append(MinNewTokensLengthLogitsProcessor(S, bans["min_new_tokens"], EOS))
        for sampled in (False, True):
            lst = LogitsProcessorList(hf)
            if sampled:
                lst += [TemperatureLogitsWarper(T)]
                if k:
                    lst.append(TopKLogitsWarper(k))
                if p < 1.0:
                    lst.append(TopPLogitsWarper(p))
            want = lst(ids, x.clone())
            got = m._host_processors(ids, x.clone(), sampled, T, k, p, r, b, S)
            assert torch.equal(want.view(torch.int32), got.view(torch.int32)), (c, sampled)


@pytest.mark.parametrize("kw,msg", [
    (dict(no_repeat_ngram_size=-1), "`ngram_size` has to be a strictly positive integer"),
    (dict(no_repeat_ngram_size=2.0), "`ngram_size` has to be a strictly positive integer"),
    (dict(min_new_tokens=-2), "`min_new_tokens` has to be a positive integer"),
    (dict(min_new_tokens=1.5), "`min_new_tokens` has to be a positive integer"),
    (dict(bad_words_ids=[]), "`bad_words_ids` has to be a non-empty list"),
    (dict(bad_words_ids=[5, 6]), "`bad_words_ids` has to be a list of lists"),
    (dict(bad_words_ids=[[5, -1]]), "Each list in `bad_words_ids` has to be a list of positive integers"),
    (dict(bad_words_ids=[[5, "a"]]), "Each list in `bad_words_ids` has to be a list of positive integers"),
    (dict(bad_words_ids=[[]]), "non-empty list of token ids"),
    (dict(bad_words_ids=[[5, V]]), f"The model vocabulary size is {V}, but the following tokens were being biased"),
    (dict(bad_words_ids=[[5]] * 2 + [list(range(3, 1100))]), "more than 1024")])
def test_rejections(kw, msg):
    m, eng = _fake_model()
    req = {"input_ids": torch.tensor([REQ0, 5, 6])}
    with pytest.raises(ValueError, match=msg.replace("[", r"\[").replace("`", "`")):
        m.generate_requests([req], max_new_tokens=4, **kw)
    with pytest.raises(ValueError, match="request 0"):
        m.generate_requests([dict(req, **kw)], max_new_tokens=4)
    with pytest.raises(ValueError):
        m._ban_args(kw.get("no_repeat_ngram_size"), kw.get("bad_words_ids"), kw.get("min_new_tokens"), EOS)
    assert eng.calls == []


def test_off_settings_and_vocabulary_limit():
    m, _ = _fake_model()
    assert m._ban_args(None, None, None, EOS) is None
    assert m._ban_args(0, None, 0, EOS) is None
    assert m._ban_args(None, None, 5, None) is None             # no EOS: no MinNewTokens processor
    b = m._ban_args(None, [[EOS]], None, EOS)
    assert b is not None and b.words == []                      # HF keeps the processor, with nothing to ban
    assert m._ban_args(None, [[3, 4], [3, 4], [5]], None, EOS).words == [[3, 4], [5]]
    m.config.vocab_size = 60000
    with pytest.raises(ValueError, match="vocabulary"):
        m._ban_args(2, None, None, EOS)
    assert m._ban_args(2, None, None, EOS, device=False).ngram == 2


@pytest.mark.parametrize("kw", [dict(no_repeat_ngram_size=3), dict(bad_words_ids=[[5]]), dict(min_new_tokens=2)])
def test_beams_raise(kw):
    m, eng = _fake_model()
    with pytest.raises(NotImplementedError, match=list(kw)[0]):
        m.generate(torch.tensor([[REQ0, 5, 6]]), num_beams=2, max_new_tokens=4, **kw)
    assert eng.calls == []


# ---- histories and ban tables in flight -------------------------------------------------------------------------
class BanFake(TokenSetFake):
    """TokenSetFake with the ban table and token histories: it records every set_bans and set_token_history, writes
    each token a banning slot's prefill draws into its history, and checks at each prefill draw that the history
    holds the slot's cached ids"""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.bans = [None] * self.n_slots
        self.hist = [[] for _ in range(self.n_slots)]
        self.hwrites, self.bwrites, self.bad_draws = [], [], []

    def set_bans(self, clips, ngram, eos, eos_from_col, words):
        self.bwrites.append((list(clips), list(ngram), list(eos), list(eos_from_col), [list(w) for w in words]))
        for s, n, e, f, w in zip(clips, ngram, eos, eos_from_col, words):
            self.bans[s] = (n, e, f, w) if (n or e >= 0 or w) else None

    def set_token_history(self, entry, ids):
        ids = [int(t) for t in torch.as_tensor(ids).reshape(-1)]
        self.hwrites.append((entry, ids))
        self.hist[entry] = ids

    def _draw(self, s, c, tok):
        if self.bans[s] is None:
            return
        if self.hist[s][:c] != self._read(s, c):
            self.bad_draws.append((s, c))
        self.hist[s] = self.hist[s][:c] + [int(tok)]

    def _prefill(self, s, ids):
        tok = super()._prefill(s, ids)
        self._draw(s, len(ids.reshape(-1)), tok)
        return tok


def _requests(n, rng, long=False):
    reqs = []
    for i in range(n):
        S = int(torch.randint(600, 630, (1,), generator=rng)) if long and i % 3 == 0 else \
            int(torch.randint(5, 40, (1,), generator=rng))
        ids = torch.cat([torch.tensor([REQ0 + i]), torch.randint(1, 30000, (S - 1,), generator=rng)])
        r = {"input_ids": ids, "max_new_tokens": int(torch.randint(3, 12, (1,), generator=rng))}
        if i % 2 == 0:
            r.update(no_repeat_ngram_size=3, bad_words_ids=[[7, 8]], min_new_tokens=2)
        reqs.append(r)
    return reqs


def _check(eng, outs, reqs):
    """every history write of a banning request is its prompt, or (at a resume) a prefix of its returned sequence;
    every admission's ban-table write gives a banning request EOS from its prompt length + min_new_tokens; the table
    is all off after the call"""
    by_first = {REQ0 + i: i for i in range(len(reqs))}
    n_resume = 0
    for s, ids in eng.hwrites:
        i = by_first[ids[0]]
        seq = outs[i][0].tolist()
        S = torch.as_tensor(reqs[i]["input_ids"]).numel()
        assert "no_repeat_ngram_size" in reqs[i]
        assert len(ids) >= S and ids == seq[:len(ids)], (i, len(ids), S)
        n_resume += len(ids) > S
    assert {by_first[ids[0]] for _, ids in eng.hwrites} == {i for i, r in enumerate(reqs) if
                                                          "no_repeat_ngram_size" in r}
    assert eng.bwrites and eng.bans == [None] * eng.n_slots
    for clips, ngram, eos, frm, words in eng.bwrites[:-1]:
        for n, e, f, w in zip(ngram, eos, frm, words):
            assert (n, w) in ((3, [[7, 8]]), (0, [])) and e in ((EOS, -1) if n else (-1,))
            assert (n == 0) == (f == 0)
    assert not eng.bad_draws
    return n_resume


@pytest.mark.parametrize("packed", [False, True])
def test_histories_contiguous(packed):
    rng = torch.Generator().manual_seed(1)
    reqs = _requests(10, rng)
    m, eng = _fake_model()
    outs = m.generate_requests(reqs, eos_token_id=EOS, packed_admission=packed)
    _check(eng, outs, reqs)
    # EOS allowed from the prompt length + min_new_tokens
    firsts = {}
    for clips, ngram, eos, frm, words in eng.bwrites[:-1]:
        for s, n, f in zip(clips, ngram, frm):
            if n:
                firsts.setdefault(f, s)
    want = {torch.as_tensor(r["input_ids"]).numel() + 2 for r in reqs if "min_new_tokens" in r}
    assert set(firsts) == want


def test_no_ban_table_without_bans():
    rng = torch.Generator().manual_seed(5)
    reqs = _requests(6, rng)
    for r in reqs:
        for k in ("no_repeat_ngram_size", "bad_words_ids", "min_new_tokens"):
            r.pop(k, None)
    m, eng = _fake_model()
    m.generate_requests(reqs, eos_token_id=EOS)
    assert eng.bwrites == [] and eng.hwrites == []


@pytest.mark.parametrize("packed", [False, True])
def test_histories_paged_preemption(packed):
    rng = torch.Generator().manual_seed(2)
    reqs = _requests(10, rng)
    for r in reqs:
        r.update(max_new_tokens=200, no_repeat_ngram_size=3, bad_words_ids=[[7, 8]], min_new_tokens=2)
    m, eng = _fake_model(kv_blocks=6)
    eng.lens = {i: torch.as_tensor(r["input_ids"]).numel() + 200 for i, r in enumerate(reqs)}
    outs = m.generate_requests(reqs, eos_token_id=None, packed_admission=packed)
    assert m.last_kv_stats["preemptions"] > 0
    assert _check(eng, outs, reqs) > 0     # resumed requests rebuilt their histories from prompt + tokens


def test_histories_chunked():
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
        eng._draw(s, start + len(ids), tok)
        return tok
    eng._chunk = chunk
    outs = m.generate_requests(reqs, eos_token_id=None, chunked_prefill=True)
    assert m.last_kv_stats["chunk_calls"] > 0
    _check(eng, outs, reqs)
    # a chunked prompt's history is written before each of its chunk calls, so no discarded chunk token stays in it
    long = [i for i, r in enumerate(reqs) if torch.as_tensor(r["input_ids"]).numel() > 512 and i % 2 == 0]
    assert long
    for i in long:
        assert sum(1 for _, ids in eng.hwrites if ids[0] == REQ0 + i) >= 2


@pytest.mark.parametrize("packed", [False, True])
def test_histories_of_continuations_are_the_whole_conversation(packed):
    import test_sessions_cpu as SC

    class SessionBanFake(BanFake, SC.SessionFake):
        pass

    eng = SessionBanFake(4, 12)
    m = _model(eng, max_batch=4, max_seq=SC.MAX_SEQ, kv_blocks=12)
    m._SLOT_CHUNK = 8
    eng.model = m
    convs = SC.conversations(5, 3, seed=4)
    res = SC.run_sessions(m, convs, 3, packed_admission=packed, no_repeat_ngram_size=2, min_new_tokens=1)
    assert not eng.violations and not eng.bad_draws
    for t in (1, 2):
        for c in range(len(convs)):
            conv = res[c][t - 1] + convs[c][t][0].tolist()       # the kept conversation and the new turn
            assert conv in [ids for _, ids in eng.hwrites], (t, c)
            assert res[c][t][:len(conv)] == conv, (t, c)
            # min_new_tokens counts from the conversation's length (no EOS here: nothing to ban, and the column is it)
            assert any(len(conv) in frm for _, _, _, frm, _ in eng.bwrites)
