"""CPU tests of log-probs of generated tokens: the float64 rule (_logprob_ref.py) pinned against the installed
transformers, generate_requests' host bookkeeping with a fake engine that stores a log-prob row per (entry,
position) as the device does, the rejections of the Python arguments, and the new C-ABI symbols."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import _logprob_ref as LR
import test_paged_kv_cpu as PK
import test_sessions_cpu as SC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------
def _hf_logprobs(x, T, k, cand):
    """HF: TemperatureLogitsWarper, TopKLogitsWarper (generate adds none for top_k 0), then
    compute_transition_scores(normalize_logits=True): the log-prob of each token of `cand`, as if generated"""
    from transformers import TemperatureLogitsWarper, TopKLogitsWarper
    from transformers.generation.utils import GenerationMixin
    V = x.numel()
    scores = x[None].clone()
    if T > 0:
        scores = TemperatureLogitsWarper(T)(None, scores)
        if k:
            scores = TopKLogitsWarper(k)(None, scores)
    me = SimpleNamespace(config=SimpleNamespace(get_text_config=lambda: SimpleNamespace(vocab_size=V)))
    seqs = torch.tensor(cand)[:, None]                  # one "sequence" per candidate: its transition score
    lp = GenerationMixin.compute_transition_scores(me, seqs, (scores.expand(len(cand), V),), normalize_logits=True)
    return dict(zip(cand, lp[:, 0].double().tolist()))


def _rows(V, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(6, V, generator=g) * 3).bfloat16().float()
    kth = torch.sort(x[1], descending=True).values[49]
    x[1, torch.randperm(V, generator=g)[:6]] = kth          # ties at the 50th value
    x[2, torch.randperm(V, generator=g)[:400]] = float("-inf")
    x[3] = float("-inf")                                    # no finite maximum
    top = x[4].max()
    x[4, torch.randperm(V, generator=g)[:3]] = top          # ties at the maximum
    return x


@pytest.mark.parametrize("T,k", [(0.0, 0), (0.2, 50), (1.5, 0), (1e-4, 1), (0.2, 32003 + 5), (1.0, 50)])
def test_rule_matches_transformers(T, k):
    V, n = 32003, 20
    x = _rows(V, seed=int(T * 1000) + k)
    for b in range(x.shape[0]):
        xb = x[b].numpy()
        if T > 0 and not np.isfinite(np.max(xb / np.float32(T))):
            continue
        s, kept = LR.processed(xb, T, k)
        # candidates: the 60 largest logits (ties by index), every 97th token, the -inf ones
        top = torch.sort(x[b], descending=True, stable=True).indices[:60].tolist()
        cand = sorted(set(top) | set(range(0, V, 97)) | set(np.nonzero(np.isneginf(xb))[0][:20].tolist()))
        hf = _hf_logprobs(x[b], T, k, cand)
        if not kept.any() or not np.isfinite(s.max()):
            assert all(np.isnan(v) for v in hf.values())
            lp, ids, lps = LR.logprobs(xb, T, k, n, 0)
            assert np.isnan(lp) and ids == [-1] * n and np.isnan(lps).all()
            continue
        for j, h in hf.items():
            lp, _, _ = LR.logprobs(xb, T, k, 0, j)
            assert lp == h or abs(lp - h) <= 1e-4 + 1e-6 * abs(h), (b, j, lp, h)
            assert kept[j] or h == -np.inf
        # the top n: HF's log-probs sorted (ties: the lowest index first); a token top-k drops is -1 / -inf
        _, ids, lps = LR.logprobs(xb, T, k, n, 0)
        order = sorted(top, key=lambda i: (-hf[i], i))[:n]
        want = [i if hf[i] > -np.inf or T == 0 else -1 for i in order]
        assert ids == want, (b, ids, want)
        for i, v in zip(ids, lps):
            assert (v == -np.inf) if i < 0 else (v == hf[i] or abs(v - hf[i]) <= 1e-4 + 1e-6 * abs(hf[i]))


def test_close_bound():
    assert LR.close([1.0, float("nan"), float("-inf")], [1.0 + 5e-6, float("nan"), float("-inf")])
    assert not LR.close([1.0], [1.0 + 3e-5])
    assert not LR.close([float("nan")], [0.0])


# ------------------------------------------------------------------------------------------
def _lp_row(tok, p):
    """the fake's log-prob row of token `tok` at position p: place q holds id tok + q and lp -(tok + p / 1e4)"""
    ids = torch.tensor([tok + q for q in range(LR.LOGPROBS_MAX + 1)], dtype=torch.int32)
    lps = torch.full((LR.LOGPROBS_MAX + 1,), -(tok + p / 1e4), dtype=torch.float32)
    return ids, lps


class LogprobMixin:
    """Stores a row per (entry, position) for every token an entry with top_n >= 0 produces, as the device does;
    nothing for an entry that is off (a read of it gives sentinels)"""

    def _lp_init(self):
        self.top_n = [-1] * self.n_slots
        self.lp = {}
        self.lp_calls = []

    def set_logprobs(self, clips, top_n):
        self.lp_calls.append((list(clips), list(top_n)))
        for b, k in zip(clips, top_n):
            assert -1 <= k <= LR.LOGPROBS_MAX
            self.top_n[b] = k

    def _emit(self, s, tok, p):
        if self.top_n[s] >= 0:
            self.lp[(s, p)] = _lp_row(int(tok), p)

    def read_logprobs(self, entry, first_pos, count, ids_out=None, lp_out=None):
        for j in range(count):
            ids, lps = self.lp.get((entry, first_pos + j), (torch.full((21,), -7, dtype=torch.int32),
                                                            torch.full((21,), float("nan"))))
            ids_out[j], lp_out[j] = ids, lps
        return ids_out, lp_out

    def slot_prefill(self, slot, ids, video_feats, vid_start, tok_out=None):
        out = super().slot_prefill(slot, ids, video_feats, vid_start, tok_out)
        self._emit(slot, out[0], ids.numel())
        return out

    def slots_prefill(self, slots, ids_list, feats_list, vid_starts, tok_out=None):
        out = super().slots_prefill(slots, ids_list, feats_list, vid_starts, tok_out)
        for s, ids, t in zip(slots, ids_list, out):
            self._emit(s, t, torch.as_tensor(ids).numel())
        return out

    def slots_prefill_append(self, slots, starts, ids_list, tok_out=None):
        out = super().slots_prefill_append(slots, starts, ids_list, tok_out)
        for s, st, ids, t in zip(slots, starts, ids_list, out):
            self._emit(s, t, st + torch.as_tensor(ids).numel())
        return out

    def slot_decode(self, first_tok, positions, n_new):
        out = super().slot_decode(first_tok, positions, n_new)
        for s in range(out.shape[0]):
            for j in range(1, n_new):
                self._emit(s, out[s, j], positions[s] + j)
        return out


class PagedLp(LogprobMixin, PK.FakeEngine):
    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self._lp_init()


class SessionLp(LogprobMixin, SC.SessionFake):
    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self._lp_init()


def _check_entries(m, outs, reqs, k):
    for i, (o, r) in enumerate(zip(outs, reqs)):
        e = m.last_logprobs[i]
        want_k = r.get("logprobs", k)
        if want_k is None:
            assert e is None
            continue
        new = o[0, -len(e["token_logprobs"]):].tolist()
        if not r.get("continues"):
            assert len(new) == o.shape[1] - r["input_ids"].numel()
        assert e["top_ids"].shape == (len(new), want_k) and e["top_ids"].dtype == torch.int64
        assert e["token_logprobs"].dtype == e["top_logprobs"].dtype == torch.float32
        p0 = o.shape[1] - len(new)
        for j, t in enumerate(new):
            ids, lps = _lp_row(t, p0 + j)
            assert e["token_logprobs"][j] == lps[0], (i, j)
            assert e["top_ids"][j].tolist() == ids[1:1 + want_k].tolist(), (i, j)


def _run(kv_blocks, slots=4, packed=False, k=5, per_req=None, chunk=8, seed=None):
    lens = {r: S + n for r, (S, n) in enumerate(PK.SHAPE)}
    eng = PagedLp(640, slots, kv_blocks, lens)
    m = PK._model(eng, max_batch=slots, kv_blocks=kv_blocks or None)
    m._SLOT_CHUNK = chunk
    reqs = PK._reqs(PK.SHAPE)
    for i, v in (per_req or {}).items():
        reqs[i]["logprobs"] = v
    kw = dict(do_sample=True, seed=seed, temperature=0.5) if seed is not None else {}
    outs = m.generate_requests(reqs, eos_token_id=None, packed_admission=packed, logprobs=k, **kw)
    return outs, reqs, m, eng


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("kv_blocks", [0, 5, 8, 40])
def test_requests_accumulate_across_chunks_and_preemption(packed, kv_blocks):
    ref, reqs, mref, _ = _run(0, packed=packed)
    outs, reqs, m, eng = _run(kv_blocks, packed=packed, chunk=4 if kv_blocks == 5 else 8)
    assert [o.tolist() for o in outs] == [o.tolist() for o in ref]
    _check_entries(m, outs, reqs, 5)
    if kv_blocks == 5:
        assert m.last_kv_stats["preemptions"] > 0
    # the values do not depend on paging or preemption
    for a, b in zip(m.last_logprobs, mref.last_logprobs):
        assert torch.equal(a["token_logprobs"], b["token_logprobs"]) and torch.equal(a["top_ids"], b["top_ids"])
    # every entry is off when the call returns
    assert eng.top_n == [-1] * eng.n_slots


def test_per_request_keys_and_requests_that_do_not_ask():
    per = {0: None, 2: 0, 3: 20}
    outs, reqs, m, eng = _run(8, per_req=per, k=None)
    for i in range(len(reqs)):
        if i in (2, 3):
            assert m.last_logprobs[i]["top_ids"].shape[1] == per[i]
        else:
            assert m.last_logprobs[i] is None
    _check_entries(m, outs, reqs, None)
    # only the asking requests' slots were ever turned on
    assert all(k in (-1, 0, 20) for _, ks in eng.lp_calls for k in ks)


def test_no_logprobs_no_calls():
    outs, reqs, m, eng = _run(8, k=None)
    assert m.last_logprobs is None and eng.lp_calls == [] and eng.lp == {}


def test_session_continuation_reports_its_new_tokens_only():
    eng = SessionLp(4, 24)
    m, _ = SC.paged(4, 24)
    m._engine = eng
    eng.model = m
    conv = [dict(input_ids=torch.tensor([PK.REQ0 + r] + [7] * (20 + r)), max_new_tokens=12, session=r)
            for r in range(3)]
    o1 = m.generate_requests(conv, eos_token_id=None, logprobs=3)
    _check_entries(m, o1, conv, 3)
    turn = [dict(input_ids=torch.tensor([9, 9, 9 + r]), max_new_tokens=10, continues=r) for r in range(3)]
    o2 = m.generate_requests(turn, eos_token_id=None, logprobs=3, packed_admission=True)
    for i, o in enumerate(o2):
        e = m.last_logprobs[i]
        assert len(e["token_logprobs"]) == 10
        p0 = o.shape[1] - 10
        for j, t in enumerate(o[0, p0:].tolist()):
            assert e["token_logprobs"][j] == _lp_row(t, p0 + j)[1][0]


# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [21, -1, True, 1.5, "3"])
def test_rejections_before_any_device_work(bad):
    eng = PagedLp(640, 4, 8, {})
    m = PK._model(eng, max_batch=4, kv_blocks=8)
    reqs = PK._reqs(PK.SHAPE[:3])
    with pytest.raises(ValueError, match="logprobs"):
        m.generate_requests(reqs, logprobs=bad)
    reqs[1]["logprobs"] = bad
    with pytest.raises(ValueError, match="request 1: logprobs"):
        m.generate_requests(reqs, logprobs=2)
    assert eng.calls == [] and eng.lp_calls == []
    from test_inflight_cpu import _model as contiguous_model
    mc = contiguous_model()
    ids = torch.tensor([[1, 5, 6]])
    with pytest.raises(ValueError, match="logprobs"):
        mc.generate(ids, logprobs=bad)
    mc._last_out = ids
    with pytest.raises(ValueError, match="logprobs"):
        mc.generate_continue(ids, logprobs=bad)
    assert mc._engine.calls == []


def test_unseeded_sampling_with_logprobs_names_seed():
    from test_inflight_cpu import _model as contiguous_model
    m = contiguous_model()
    with pytest.raises(NotImplementedError, match="seed="):
        m.generate(torch.tensor([[1, 5, 6]]), do_sample=True, logprobs=2)
    m._last_out = torch.tensor([[1, 5, 6]])
    with pytest.raises(NotImplementedError, match="seed="):
        m.generate_continue(torch.tensor([[7]]), do_sample=True, logprobs=0)
    assert m._engine.calls == []


def test_c_abi_symbols():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as G
    import vcl_native as vn
    new = {"vcl_llm_set_logprobs", "vcl_llm_read_logprobs", "vcl_op_sample_logprobs"}
    assert new <= set(G.declared_symbols())
    assert new <= set(vn.EXPORTED_SYMBOLS)
    assert vn.LOGPROBS_MAX == LR.LOGPROBS_MAX == 20 and vn.LOGPROB_PLACES == 21
    hdr = open(os.path.join(ROOT, "include", "vcl.h")).read()
    assert "#define VCL_LOGPROBS_MAX 20" in hdr
    assert hdr.count("compute_transition_scores") >= 2
