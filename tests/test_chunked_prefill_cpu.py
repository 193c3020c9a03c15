"""CPU tests of generate_requests(chunked_prefill=True) on a paged KV cache, driven by the fake engine of
test_paged_kv_cpu with a chunk entry point added. A chunk writes its rows at their absolute columns through the
block table and its token is a function of every column 0 .. its last row, so a chunk that runs before its blocks are
owned, skips rows, repeats rows or runs out of order changes the tokens or is recorded as a violation."""
import pytest
import torch

from test_paged_kv_cpu import C, REQ0, FakeEngine, _model, _tok

MAX_SEQ = 2048


class ChunkEngine(FakeEngine):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.done = {}                        # slot -> prompt rows written by chunks so far

    def _admitted(self):
        # the scheduler prefills the long prompts of an admission point before the short ones; its admission order
        # is queue order, so a request admitted at the same point with a higher index goes after this one
        run = self.running
        i = len(run) - 1
        while i > 0 and run[i - 1] > run[i]:
            run[i - 1], run[i] = run[i], run[i - 1]
            i -= 1

    def _prefill(self, s, ids):
        tok = super()._prefill(s, ids)
        self._admitted()
        return tok

    def slots_prefill_chunk(self, slots, starts, totals, ids_list, feats_list, vid_starts, tok_out=None):
        self.calls.append(("chunk", list(slots), list(starts), [len(i) for i in ids_list], list(totals)))
        toks = []
        for s, st, tot, ids in zip(slots, starts, totals, ids_list):
            ids = [int(t) for t in torch.as_tensor(ids).reshape(-1)]
            if st % 64 or not 1 <= len(ids) <= 512 or st + len(ids) > tot or tot > self.max_seq:
                self.violations.append(("bad chunk", s, st, len(ids), tot))
            if self.done.get(s, 0) != st:
                self.violations.append(("out of order", s, st, self.done.get(s, 0)))
            if st == 0:
                r = ids[0] - REQ0
                self.running.append(r)
                self._admitted()
                self.events.append(("admit", r))
                self.owner[s] = r
            for j, t in enumerate(ids):
                if self.table[s][(st + j) // C] == 0:
                    self.violations.append(("unowned", s, st + j))
                self._write(s, st + j, t)
            self.done[s] = st + len(ids) if st + len(ids) < tot else 0
            toks.append(_tok(self._read(s, st + len(ids)), st + len(ids) - 1, self.seed[s]))
        return torch.tensor(toks, dtype=torch.int32)


def _reqs(shape):
    return [dict(input_ids=torch.tensor([REQ0 + r] + [7 + (r * 13 + j) % 11 for j in range(S - 1)]),
                 max_new_tokens=n) for r, (S, n) in enumerate(shape)]


# prompts of 100 .. 1500 tokens: 513, 1024 and 1500 take 2 / 2 / 3 chunks, 577 ends one row past a 64-row tile
SHAPE = [(700, 60), (100, 30), (1500, 90), (513, 40), (300, 150), (1024, 8), (577, 200), (40, 20), (1200, 33),
         (128, 1)]


def _run(kv_blocks, shape=SHAPE, slots=4, packed=False, seed=None, chunked=True, max_seq=MAX_SEQ):
    lens = {r: S + n for r, (S, n) in enumerate(shape)}
    eng = ChunkEngine(max_seq, slots, kv_blocks, lens)
    m = _model(eng, max_batch=slots, max_seq=max_seq, kv_blocks=kv_blocks or None)
    kw = dict(do_sample=True, seed=seed, temperature=0.5) if seed is not None else {}
    if chunked is not None:
        kw["chunked_prefill"] = chunked
    outs = m.generate_requests(_reqs(shape), eos_token_id=None, packed_admission=packed, **kw)
    return [o[0].tolist() for o in outs], eng, m


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("seed", [None, 5])
def test_chunked_equals_contiguous_for_every_pool(packed, seed):
    ref, _, _ = _run(0, packed=packed, seed=seed)
    need = max(-(-(S + n) // C) for S, n in SHAPE)
    pre, long_swapped = [], False
    for kv in (need + 1, 18, 20, 24, 80):
        out, eng, m = _run(kv, packed=packed, seed=seed)
        long_swapped |= any(e[0] == "swap" and SHAPE[e[1]][0] > 512 for e in eng.events)
        assert out == ref, f"kv_blocks {kv}"
        assert eng.violations == [], eng.violations[:3]
        st = m.last_kv_stats
        assert st["chunked_prefills"] >= sum(S > 512 for S, _ in SHAPE)
        assert st["chunk_calls"] >= 1 and st["peak_blocks"] <= kv - 1
        pre.append(st["preemptions"])
    assert max(pre) > 0 and pre[-1] == 0 and long_swapped     # a long request is swapped out and resumes


def test_chunks_cover_each_prompt_once():
    out, eng, m = _run(80, packed=True)
    assert eng.violations == []
    long = sorted(S for S, _ in SHAPE if S > 512)
    seen = []
    for c in eng.calls:
        if c[0] == "chunk":
            for st, ln, tot in zip(c[2], c[3], c[4]):
                assert st % 64 == 0 and 1 <= ln <= 512 and st + ln <= tot
                if st == 0:
                    seen.append([tot, 0])
                cur = next(x for x in seen if x[0] == tot and x[1] == st)
                cur[1] += ln
    assert sorted(t for t, _ in seen) == long
    assert all(done == tot for tot, done in seen)            # 0 .. S-1 exactly once, in order
    st = m.last_kv_stats
    assert st["chunked_prefills"] == len(long)
    assert st["chunk_calls"] == sum(1 for c in eng.calls if c[0] == "chunk")


def test_packed_admission_packs_the_chunks_of_long_prompts():
    shape = [(1100, 10), (900, 10), (600, 10), (200, 10)]
    _, eng_p, _ = _run(80, shape=shape, packed=True)
    _, eng_s, _ = _run(80, shape=shape, packed=False)
    chunks_p = [c for c in eng_p.calls if c[0] == "chunk"]
    chunks_s = [c for c in eng_s.calls if c[0] == "chunk"]
    assert len(chunks_p) == 3 and len(chunks_p[0][1]) == 3           # rounds at 0 / 512 / 1024, three prompts first
    assert len(chunks_s) == 3 + 2 + 2 and all(len(c[1]) == 1 for c in chunks_s)
    assert eng_p.violations == eng_s.violations == []


def test_without_the_flag_nothing_changes():
    shape = [(S if S <= 512 else 400, n) for S, n in SHAPE]
    for packed in (False, True):
        _, eng0, m0 = _run(24, shape=shape, packed=packed, chunked=None)
        _, eng1, m1 = _run(24, shape=shape, packed=packed, chunked=False)
        _, eng2, m2 = _run(24, shape=shape, packed=packed, chunked=True)     # no long prompt: the same calls
        assert eng0.calls == eng1.calls == eng2.calls
        assert m0.last_kv_stats == m2.last_kv_stats and m0.last_kv_stats["chunk_calls"] == 0
    eng = ChunkEngine(MAX_SEQ, 4, 40, {0: 600})
    m = _model(eng, max_batch=4, max_seq=MAX_SEQ, kv_blocks=40)
    with pytest.raises(ValueError, match="512"):
        m.generate_requests([dict(input_ids=torch.tensor([REQ0] * 513), max_new_tokens=4)])
    with pytest.raises(ValueError, match="blocks"):       # 17 blocks > 15 usable, chunked or not
        m2 = _model(ChunkEngine(MAX_SEQ, 4, 16), max_batch=4, max_seq=MAX_SEQ, kv_blocks=16)
        m2.generate_requests([dict(input_ids=torch.tensor([REQ0] * 2000), max_new_tokens=40)], chunked_prefill=True)
    assert eng.calls == []


def test_contiguous_model_ignores_the_flag():
    out0, eng0, _ = _run(0, chunked=None)
    out1, eng1, _ = _run(0, chunked=True)
    assert out0 == out1 and eng0.calls == eng1.calls
    assert not any(c[0] == "chunk" for c in eng1.calls)
