"""The in-flight scheduler's engine-call trace, pinned: generate_requests on a fake engine that combines the paged
cache, sessions, chunked prefill, token sets and log-probs of the other CPU tests, with every engine call logged by
name and arguments. Each case hashes that log with the outputs, last_logprobs, last_kv_stats and the kept
conversations; tests/golden/schedule_trace.json holds the hashes. A scheduler change that alters any engine call,
its order or its arguments, or any result, fails here. Regenerate with `python tests/test_schedule_trace_cpu.py`
only for an intended change of schedule."""
import hashlib
import itertools
import json
import os
import sys

import pytest
import torch

import test_paged_kv_cpu as P
import test_sessions_cpu as SC
from test_logprobs_cpu import LogprobMixin
from test_nucleus_cpu import TokenSetFake

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "schedule_trace.json")
METHODS = ("set_sampling", "set_sampling_ex", "set_token_set", "set_block_table", "slot_prefill", "slots_prefill",
           "slots_prefill_append", "slots_prefill_chunk", "slot_decode", "swap_buffer", "kv_block_copy",
           "set_logprobs", "read_logprobs")


class TraceFake(LogprobMixin, TokenSetFake, SC.SessionFake):
    """Every fake engine entry point in one class, on a contiguous (kv_blocks 0) or a paged cache"""

    def __init__(self, n_slots, kv_blocks):
        super().__init__(n_slots, kv_blocks)
        if not kv_blocks:
            self.table = []
        self._lp_init()

    def _write(self, s, c, v):
        if self.kv_blocks:
            return super()._write(s, c, v)
        self.cache[s][c] = v

    def slots_prefill_chunk(self, slots, starts, totals, ids_list, feats_list, vid_starts, tok_out=None):
        toks = []
        for s, st, ids in zip(slots, starts, ids_list):
            ids = [int(t) for t in torch.as_tensor(ids).reshape(-1)]
            for j, t in enumerate(ids):
                self._write(s, st + j, t)
            tok = P._tok(self._read(s, st + len(ids)), st + len(ids) - 1, self.seed[s])
            self._mark(s, tok)
            self._emit(s, tok, st + len(ids))
            toks.append(tok)
        return torch.tensor(toks, dtype=torch.int32)


def _plain(x):
    """a JSON form of an engine argument or a result"""
    if isinstance(x, torch.Tensor):
        return [str(x.dtype), list(x.shape), x.tolist()]
    if isinstance(x, (list, tuple)):
        return [_plain(v) for v in x]
    if isinstance(x, dict):
        return {str(k): _plain(v) for k, v in sorted(x.items(), key=lambda kv: str(kv[0]))}
    if isinstance(x, float):
        return repr(x)
    return x


def _traced(eng, log):
    """wrap every engine entry point: its name, positional and keyword arguments go to `log` before it runs; an
    output buffer (*_out) is logged by shape only, since its contents are not an input"""
    def wrap(name, fn):
        def call(*a, **kw):
            log.append([name, _plain(a), {k: (list(v.shape) if k.endswith("_out") else _plain(v))
                                          for k, v in sorted(kw.items())}])
            return fn(*a, **kw)
        return call
    for name in METHODS:
        setattr(eng, name, wrap(name, getattr(eng, name)))


def stop(ids, scores=None):
    """a stopping criterion: the newest token is a multiple of 29 (generate_requests calls it after each new token)"""
    return int(ids[0, -1]) % 29 == 0


def _samp(mode, i):
    """per-request keys of a sampling mode"""
    if mode != "mixed":
        return {}
    return [dict(do_sample=True, temperature=0.7, top_p=0.9), dict(repetition_penalty=1.2),
            dict(do_sample=True, seed=100 + i, top_k=20, repetition_penalty=1.1), {}][i % 4]


CALL_KW = {"greedy": {}, "seeded": dict(do_sample=True, seed=5, temperature=0.5), "mixed": dict(seed=7)}
LP = {2: 0, 3: 20, 5: None}                       # per-request logprobs keys of the "mixed" mode (others: the call's 3)


def _requests(work, mode, lps, stops, turn=0):
    if work == "base":
        reqs = P._reqs(P.SHAPE)
    elif work == "chunked":
        g = torch.Generator().manual_seed(3)
        reqs = []
        for i in range(8):
            lo, hi = (560, 620) if i % 3 == 0 else (5, 200)
            S = int(torch.randint(lo, hi, (1,), generator=g))
            ids = torch.cat([torch.tensor([P.REQ0 + i]), torch.randint(1, 30000, (S - 1,), generator=g)])
            n = int(torch.randint(1, min(90, SC.MAX_SEQ - S) + 1, (1,), generator=g))
            reqs.append(dict(input_ids=ids, max_new_tokens=n))
    else:
        reqs = [dict(input_ids=ids, max_new_tokens=n, **({"session": c} if turn == 0 else {"continues": c}))
                for c, (ids, n) in enumerate(conv[turn] for conv in SC.conversations(6, 3, seed=5))]
    for i, r in enumerate(reqs):
        r.update(_samp(mode, i))
        if lps == "mixed" and i in LP:
            r["logprobs"] = LP[i]
        if stops and i % 3 == 1:
            r["stopping_criteria"] = [stop]
    return reqs


_EOS = {}


def _eos(work, mode):
    """an EOS id that a request of the workload reaches mid-stream: without EOS, the middle new token of the first
    call's longest request among those without a stopping criterion"""
    if (work, mode) not in _EOS:
        outs, *_ = _run(work, 12, False, mode, "off", False, eos=None, traced=False)
        reqs = _requests(work, mode, "off", False)
        i = max((j for j in range(len(reqs)) if j % 3 != 1), key=lambda j: reqs[j]["max_new_tokens"])
        S = torch.as_tensor(reqs[i]["input_ids"]).numel()
        _EOS[(work, mode)] = outs[0][i][0, S + reqs[i]["max_new_tokens"] // 2].item()
    return _EOS[(work, mode)]


def _run(work, kv, packed, mode, lps, stops, eos="case", traced=True):
    eng = TraceFake(4, kv)
    m = P._model(eng, max_batch=4, max_seq=SC.MAX_SEQ, kv_blocks=kv or None)
    m._SLOT_CHUNK = 4 if kv == 6 else 8
    eng.model = m
    log = []
    if traced:
        _traced(eng, log)
    if eos == "case":
        eos = _eos(work, mode) if stops else None
    kw = dict(CALL_KW[mode], eos_token_id=eos, packed_admission=packed, logprobs=3 if lps == "mixed" else None,
              chunked_prefill=work == "chunked")
    outs, lp, stats = [], [], []
    for turn in range(3 if work == "sessions" else 1):
        if work == "sessions":
            eng.continuing = set(range(6)) if turn else set()
        outs.append(m.generate_requests(_requests(work, mode, lps, stops, turn), **kw))
        lp.append(m.last_logprobs)
        stats.append(m.last_kv_stats)
    kept = {str(k): dict(ids=ss.ids, blocks=ss.blocks, saved=None if ss.saved is None else len(ss.saved), used=ss.used)
            for k, ss in m._sessions.items()}
    return outs, lp, stats, kept, log


def _cases():
    cases = []
    for kv, packed, mode, lps, stops in itertools.product((0, 6, 12), (False, True), ("greedy", "seeded", "mixed"),
                                                          ("off", "mixed"), (False, True)):
        cases.append(("base", kv, packed, mode, lps, stops))
    for kv, packed, mode in itertools.product((0, 6, 12), (False, True), ("greedy", "mixed")):
        cases.append(("chunked", kv, packed, mode, "mixed" if mode == "mixed" else "off", mode == "mixed"))
    for kv, packed, mode in itertools.product((6, 12), (False, True), ("greedy", "mixed")):
        cases.append(("sessions", kv, packed, mode, "mixed" if mode == "mixed" else "off", mode == "mixed"))
    return cases


def _key(case):
    work, kv, packed, mode, lps, stops = case
    return f"{work}-kv{kv}-{'packed' if packed else 'single'}-{mode}-lp_{lps}-{'stops' if stops else 'nostops'}"


def record(case):
    """(number of engine calls, sha256 of the calls and the results) of one case, then its outputs, log-probs and
    counters of each call"""
    outs, lp, stats, kept, log = _run(*case)
    body = dict(calls=log, outs=_plain(outs), logprobs=_plain(lp), stats=_plain(stats), kept=_plain(kept))
    h = hashlib.sha256(json.dumps(body, separators=(",", ":")).encode()).hexdigest()
    return len(log), h, outs, lp, stats


@pytest.mark.parametrize("case", _cases(), ids=_key)
def test_schedule_trace(case):
    golden = json.load(open(GOLDEN))
    assert set(golden) == {_key(c) for c in _cases()}
    n, h, outs, lp, stats = record(case)
    assert [n, h] == golden[_key(case)]
    # each case reaches the branch it is there for
    work, kv, packed, mode, lps, stops = case
    st = stats[-1]
    if kv == 6 and work == "base":
        assert st["preemptions"] > 0
    if work == "chunked" and kv:
        assert st["chunk_calls"] > 0
    if work == "sessions":
        assert st["continuations"] > 0
        if kv == 6:
            assert st["session_swaps"] > 0
    if stops:
        reqs = _requests(work, mode, lps, stops, 0)
        eos = _eos(work, mode)
        new = [o[0, torch.as_tensor(r["input_ids"]).numel():] for o, r in zip(outs[0], reqs)]
        assert any(int(x[-1]) == eos and x.numel() < r["max_new_tokens"] for x, r in zip(new, reqs))
        assert any(int(x[-1]) % 29 == 0 and x.numel() < r["max_new_tokens"] and "stopping_criteria" in r
                   for x, r in zip(new, reqs))
    if lps == "mixed":
        assert any(e is not None and e["token_logprobs"].numel() for e in lp[0])


if __name__ == "__main__":
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "video-llava_b200"))
    out = {}
    for c in _cases():
        n, h, *_ = record(c)
        out[_key(c)] = [n, h]
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{len(out)} cases -> {GOLDEN}")
