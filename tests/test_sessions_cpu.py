"""CPU tests of conversation sessions in generate_requests ("session" / "continues" on a paged KV cache), driven by the
fake engine of test_paged_kv_cpu.py plus the continued prefill (slots_prefill_append). The fake's tokens are a function
of what the cache holds (read through the block table), the slot's sampling entry and the position, so a lost or
shared block, a wrong table row or a wrong restore changes them. The yardstick is the same fake with a contiguous cache
that is given each turn's whole conversation as a new prompt: its cache then holds the same values."""
import hashlib
import json
import os

import pytest
import torch

import test_paged_kv_cpu as P
from test_paged_kv_cpu import C, EOS, REQ0, FakeEngine, _model, _tok

MAX_SEQ = 640
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "paged_schedule.json")


class SessionFake(FakeEngine):
    """FakeEngine with the continued prefill. It checks, at every table write and decode, that no block of a kept
    conversation is in a slot's table row and that kept conversations share no block, and it classifies every copy
    out of the pool as a kept conversation's swap or a running request's preemption."""

    def __init__(self, n_slots, kv_blocks):
        super().__init__(MAX_SEQ, n_slots, kv_blocks)
        self.model = None
        self.continuing = set()               # keys the current call continues (set by the test)
        self.log = []                         # ("session swap", key, used) / ("preempt", block) / ("append", ...)

    def _write(self, s, c, v):                # coverage is checked against the contiguous result instead
        b, o = self._loc(s, c)
        self.pool[b][o] = v

    def _kept(self):
        return {k: ss.blocks for k, ss in self.model._sessions.items() if ss.blocks is not None}

    def _check_disjoint(self):
        kept = [b for bl in self._kept().values() for b in bl]
        if len(kept) != len(set(kept)):
            self.violations.append(("kept conversations share a block", kept))
        live = {b for r in self.table for b in r if b}
        if live & set(kept):
            self.violations.append(("a kept block is in a table row", sorted(live & set(kept))))

    def set_block_table(self, table):
        self.table = [list(map(int, r)) for r in table]
        live = [b for r in self.table for b in r if b]
        if len(live) != len(set(live)):
            self.violations.append(("shared block", live))
        self._check_disjoint()

    def _prefill(self, s, ids):
        ids = [int(t) for t in ids.reshape(-1)]
        for c, t in enumerate(ids):
            self._write(s, c, t)
        return _tok(self._read(s, len(ids)), len(ids) - 1, self.seed[s])

    def slot_decode(self, first_tok, positions, n_new):
        self._check_disjoint()
        return super().slot_decode(first_tok, positions, n_new)

    def slots_prefill_append(self, slots, starts, ids_list, tok_out=None):
        self.calls.append(("append", list(slots), list(starts), [int(torch.as_tensor(i).numel()) for i in ids_list]))
        out = []
        for s, st, ids in zip(slots, starts, ids_list):
            assert st >= 1
            ids = [int(t) for t in torch.as_tensor(ids).reshape(-1)]
            for j, t in enumerate(ids):
                self._write(s, st + j, t)
            out.append(_tok(self._read(s, st + len(ids)), st + len(ids) - 1, self.seed[s]))
        return torch.tensor(out, dtype=torch.int32)

    def kv_block_copy(self, block, buf, write=False):
        self.calls.append(("copy", block, write))
        if write:
            self.pool[block] = buf.tolist()
            return buf
        buf[:] = torch.tensor(self.pool[block], dtype=torch.int32)
        owners = [k for k, bl in self._kept().items() if block in bl]
        if owners:
            k = owners[0]
            ss = self.model._sessions[k]
            if block == ss.blocks[0]:         # the first block of a swap: the least recently used one goes
                others = [o.used for j, o in self.model._sessions.items()
                          if o.blocks is not None and j != k and j not in self.continuing]
                if others and ss.used > min(others):
                    self.violations.append(("not the least recently used", k))
                self.log.append(("session swap", k, ss.used))
        else:
            if self._kept():
                self.violations.append(("preempted while a kept conversation was resident", sorted(self._kept())))
            self.log.append(("preempt", block))
        return buf


def paged(slots=4, kv_blocks=12, chunk=8):
    eng = SessionFake(slots, kv_blocks)
    m = _model(eng, max_batch=slots, max_seq=MAX_SEQ, kv_blocks=kv_blocks)
    m._SLOT_CHUNK = chunk
    eng.model = m
    return m, eng


def contiguous(slots=4, chunk=8):
    eng = FakeEngine(MAX_SEQ, slots)
    m = _model(eng, max_batch=slots, max_seq=MAX_SEQ)
    m._SLOT_CHUNK = chunk
    return m


def conversations(n, turns, seed=0):
    """turn t of conversation c: (new ids, max_new_tokens); turn 0 starts with REQ0 + c"""
    g = torch.Generator().manual_seed(seed)
    out = []
    for c in range(n):
        conv = []
        for t in range(turns):
            S = int(torch.randint(60, 200, (1,), generator=g)) if t == 0 else int(torch.randint(3, 40, (1,), generator=g))
            ids = torch.randint(3, 30000, (S,), generator=g)
            if t == 0:
                ids[0] = REQ0 + c
            conv.append((ids, int(torch.randint(4, 60, (1,), generator=g))))
        out.append(conv)
    return out


def run_sessions(m, convs, turns, eos=None, **kw):
    """every conversation's turns through generate_requests with sessions; returns [conv][turn] token lists"""
    res = [[] for _ in convs]
    for t in range(turns):
        reqs = []
        for c, conv in enumerate(convs):
            ids, n = conv[t]
            reqs.append(dict(input_ids=ids, max_new_tokens=n, **({"session": c} if t == 0 else {"continues": c})))
        m._engine.continuing = set(range(len(convs))) if t else set()
        for c, o in enumerate(m.generate_requests(reqs, eos_token_id=eos, **kw)):
            res[c].append(o[0].tolist())
    return res


def run_reference(convs, turns, eos=None, **kw):
    """each turn's whole conversation re-submitted as a new prompt on the contiguous fake"""
    m = contiguous()
    res = [[] for _ in convs]
    prev = [None] * len(convs)
    for t in range(turns):
        reqs = []
        for c, conv in enumerate(convs):
            ids, n = conv[t]
            full = ids if prev[c] is None else torch.cat([torch.tensor(prev[c]), ids])
            reqs.append(dict(input_ids=full, max_new_tokens=n))
        for c, o in enumerate(m.generate_requests(reqs, eos_token_id=eos, **kw)):
            prev[c] = o[0].tolist()
            res[c].append(prev[c])
    return res


def check_kept(m, eng):
    """every resident kept conversation's blocks hold its tokens 0 .. L - 2 (the cache values of the fake)"""
    for k, ss in m._sessions.items():
        if ss.blocks is None:
            continue
        L = ss.ids.numel()
        vals = [eng.pool[ss.blocks[c // C]][c % C] for c in range(L - 1)]
        assert vals == ss.ids[:L - 1].tolist(), f"conversation {k}"


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("seed", [None, 9])
@pytest.mark.parametrize("kv_blocks", [40, 12, 6])
def test_sessions_equal_resubmitted_conversations(packed, seed, kv_blocks):
    convs = conversations(7, 3, seed=1)
    kw = dict(do_sample=True, seed=seed, temperature=0.5) if seed is not None else {}
    ref = run_reference(convs, 3, **kw)
    m, eng = paged(kv_blocks=kv_blocks)
    out = run_sessions(m, convs, 3, packed_admission=packed, **kw)
    assert out == ref
    assert eng.violations == [], eng.violations[:3]
    check_kept(m, eng)
    st = m.last_kv_stats
    assert st["continuations"] == 7 and st["sessions"] == 7
    assert st["sessions_resident"] + st["sessions_swapped"] == 7
    assert st["reused_rows"] == sum(len(r[1]) - 1 for r in ref)
    appends = [c for c in eng.calls if c[0] == "append"]
    if packed:
        assert any(len(c[1]) > 1 for c in appends)
    else:
        assert all(len(c[1]) == 1 for c in appends)
    if kv_blocks == 40:
        assert st["session_swaps"] == 0 and st["preemptions"] == 0
    if kv_blocks == 6:
        assert st["session_swaps"] > 0 and st["session_swapped_bytes"] > 0
    m.end_session()
    assert m._sessions == {}


def test_eviction_is_lru_and_precedes_preemption():
    convs = conversations(9, 3, seed=2)
    m, eng = paged(kv_blocks=6, chunk=4)
    ref = run_reference(convs, 3, eos=EOS)
    assert run_sessions(m, convs, 3, eos=EOS) == ref
    assert eng.violations == [], eng.violations[:3]
    # SessionFake flags a swap of a conversation that is not the least recently used one, and a preemption while
    # a kept conversation is resident
    assert any(e[0] == "session swap" for e in eng.log) and any(e[0] == "preempt" for e in eng.log)


def test_swapped_conversation_restores_exactly():
    convs = conversations(3, 2, seed=3)
    m, eng = paged(kv_blocks=6)
    out0 = m.generate_requests([dict(input_ids=c[0][0], max_new_tokens=c[0][1], session=i) for i, c in enumerate(convs)],
                               eos_token_id=None)
    kept = {k: (ss.ids.clone(), [list(eng.pool[b]) for b in ss.blocks]) for k, ss in m._sessions.items()}
    # a request that needs the whole pool swaps every kept conversation out
    big = dict(input_ids=torch.tensor([REQ0 + 50] + [5] * 499), max_new_tokens=139)     # 5 blocks: the pool
    m.generate_requests([big], eos_token_id=None)
    assert m.last_kv_stats["sessions_swapped"] == 3 and m.last_kv_stats["preemptions"] == 0
    saved = {k: [buf.tolist() for buf in ss.saved] for k, ss in m._sessions.items()}
    for k, (ids, blocks) in kept.items():
        assert torch.equal(m._sessions[k].ids, ids) and saved[k] == blocks
    out = m.generate_requests([dict(input_ids=c[1][0], max_new_tokens=c[1][1], continues=i)
                               for i, c in enumerate(convs)], eos_token_id=None)
    ref = run_reference(convs, 2)
    assert [o[0].tolist() for o in out0] == [r[0] for r in ref]
    assert [o[0].tolist() for o in out] == [r[1] for r in ref]
    assert eng.violations == []
    check_kept(m, eng)


def test_end_session_frees_everything():
    convs = conversations(4, 1, seed=4)
    m, eng = paged(kv_blocks=6)
    m.generate_requests([dict(input_ids=c[0][0], max_new_tokens=c[0][1], session=("chat", i))
                         for i, c in enumerate(convs)], eos_token_id=None)
    assert len(m._sessions) == 4
    m.end_session(("chat", 1))
    assert set(m._sessions) == {("chat", 0), ("chat", 2), ("chat", 3)}
    with pytest.raises(ValueError, match="no conversation"):
        m.end_session(("chat", 1))
    m.end_session()
    assert m._sessions == {}
    # the whole pool is free again: a request of kv_blocks - 1 blocks runs without any swap
    m.generate_requests([dict(input_ids=torch.tensor([REQ0 + 9] + [4] * 499), max_new_tokens=139)],
                        eos_token_id=None)
    st = m.last_kv_stats
    assert st["preemptions"] == 0 and st["session_swaps"] == 0 and st["sessions"] == 0


def test_rejections_before_any_device_call():
    m, eng = paged(kv_blocks=5)
    m.generate_requests([dict(input_ids=torch.tensor([REQ0, 5, 6]), max_new_tokens=4, session="a")],
                        eos_token_id=None)
    calls = list(eng.calls)
    tail = torch.tensor([7, 8])
    bad = [([dict(input_ids=tail, continues="zz")], "no conversation is kept"),
           ([dict(input_ids=torch.tensor([REQ0 + 1]), session="a")], "already kept"),
           ([dict(input_ids=torch.tensor([REQ0 + 1]), session="b"), dict(input_ids=tail, continues="b")],
            "same call"),
           ([dict(input_ids=torch.tensor([REQ0 + 1]), session="b"), dict(input_ids=torch.tensor([REQ0 + 2]),
                                                                          session="b")], "also started"),
           ([dict(input_ids=tail, continues="a"), dict(input_ids=tail, continues="a")], "also continued"),
           ([dict(input_ids=tail, continues="a", session="c")], "not both"),
           ([dict(input_ids=tail, continues="a", video_spatio_temporal_features=torch.zeros(356, 1024))], "text only"),
           ([dict(input_ids=torch.full((512,), 7), continues="a")], "513 rows"),
           ([dict(input_ids=torch.full((300,), 7), continues="a", max_new_tokens=334)], "max_seq"),
           ([dict(input_ids=torch.full((450,), 7), continues="a", max_new_tokens=100)], "5 blocks")]
    for reqs, msg in bad:
        with pytest.raises(ValueError, match=msg):
            m.generate_requests(reqs)
        assert eng.calls == calls, msg
    assert set(m._sessions) == {"a"}
    # the model still serves, and the kept conversation still continues
    out = m.generate_requests([dict(input_ids=tail, continues="a", max_new_tokens=3)], eos_token_id=None)
    assert out[0].shape == (1, 3 + 4 + 2 + 3)
    # sessions need a paged cache
    c = contiguous()
    for key in ("session", "continues"):
        with pytest.raises(ValueError, match="paged"):
            c.generate_requests([{"input_ids": tail, key: "a"}])
    assert c._engine.calls == []


def _record(kv, packed, seed, chunk, slots):
    """the paged schedule of test_paged_kv_cpu's workload: every engine call, every block table, the outputs and the
    counters of the parent scheduler (hashed in tests/golden/paged_schedule.json)"""
    lens = {r: S + n for r, (S, n) in enumerate(P.SHAPE)}
    eng = FakeEngine(640, slots, kv, lens)
    tables = []
    orig = eng.set_block_table

    def sbt(table):
        tables.append([list(map(int, r)) for r in table])
        return orig(table)
    eng.set_block_table = sbt
    m = _model(eng, max_batch=slots, kv_blocks=kv)
    m._SLOT_CHUNK = chunk
    kw = dict(do_sample=True, seed=seed, temperature=0.5) if seed is not None else {}
    outs = m.generate_requests(P._reqs(P.SHAPE), eos_token_id=None, packed_admission=packed, **kw)
    st = {k: m.last_kv_stats[k] for k in ("preemptions", "swapped_bytes", "peak_blocks")}
    body = dict(calls=[list(c) for c in eng.calls], tables=tables, outs=[o[0].tolist() for o in outs], stats=st)
    return len(eng.calls), hashlib.sha256(json.dumps(body, separators=(",", ":")).encode()).hexdigest()


def test_requests_without_sessions_schedule_as_before():
    """the golden hashes were recorded with the scheduler before sessions existed"""
    cases = json.load(open(GOLDEN))
    assert len(cases) == 12
    for c in cases:
        n, h = _record(c["kv"], c["packed"], c["seed"], c["chunk"], c["slots"])
        assert (n, h) == (c["n_calls"], c["sha256"]), c
