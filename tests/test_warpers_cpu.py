"""CPU tests of the min-p, typical, epsilon and eta warpers: the float64 restatement of the device rules
(_warpers_ref) against the installed transformers warpers composed with temperature / top-k / top-p, the stepwise
path's host warpers against HF's processor list bit for bit, the host-side rejections, and the warper entries
generate_requests writes at admission, packed admission, preemption / resume and chunked prefill (with the fake engines
of test_paged_kv_cpu.py)."""
import numpy as np
import pytest
import torch

import _nucleus_ref as N
import _warpers_ref as Wr
import test_paged_kv_cpu as P
from test_nucleus_cpu import REQ0, TokenSetFake, _model

V = 32003
REL, GAP = 1e-4, 1e-4     # a decision within REL (relative) of its threshold, or typical levels GAP apart, is undecided
SETTINGS = [(0.05, None, None, None), (1.0, None, None, None), (0.0, None, None, None), (None, 0.2, None, None),
            (None, 0.9, None, None), (None, 0.999, None, None), (None, None, 3e-4, None), (None, None, 3e-2, None),
            (None, None, None, 3e-4), (None, None, None, 3e-2), (0.05, 0.9, 3e-4, 3e-4)]


def _rows(rng, n, T):
    """bf16 logits rows: spread 6 T, and every third row near-flat with one token of probability ~0.3 (typical at a
    small mass drops its arg-max)"""
    x = torch.randn(n, V, generator=rng) * 6 * T
    for b in range(0, n, 3):
        x[b] = torch.randn(V, generator=rng) * 0.05 * T
        x[b, int(torch.randint(0, V, (1,), generator=rng))] = float(np.log(0.43 * V)) * T
    return x.to(torch.bfloat16).float()


def _hf_list(T, k, p, w):
    from transformers.generation.logits_process import (EpsilonLogitsWarper, EtaLogitsWarper, MinPLogitsWarper,
                                                        TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper,
                                                        TypicalLogitsWarper)
    mp, ty, ep, et = w
    procs = [TemperatureLogitsWarper(T)]
    if k:
        procs.append(TopKLogitsWarper(top_k=k))
    if p < 1.0:
        procs.append(TopPLogitsWarper(top_p=p))
    if mp is not None:
        procs.append(MinPLogitsWarper(min_p=mp))
    if ty is not None and ty < 1.0:
        procs.append(TypicalLogitsWarper(mass=ty))
    if ep is not None and 0.0 < ep < 1.0:
        procs.append(EpsilonLogitsWarper(epsilon=ep))
    if et is not None and 0.0 < et < 1.0:
        procs.append(EtaLogitsWarper(epsilon=et))
    return procs


def _table(w):
    mp, ty, ep, et = w
    return (0.0 if mp is None else mp, 1.0 if ty is None else ty, 0.0 if ep is None else ep,
            0.0 if et is None else et)


@pytest.mark.parametrize("T", [0.2, 0.7, 1.5])
@pytest.mark.parametrize("k,p", [(0, 1.0), (50, 1.0), (0, 0.9), (50, 0.9)])
def test_rules_match_transformers(T, k, p):
    """The kept sets of the float64 rule and of HF's warpers are equal on every row where no decision lies within the
    stated margin; few rows are undecided"""
    rng = torch.Generator().manual_seed(int(T * 10) * 100 + k + int(p * 10))
    x = _rows(rng, 6, T)
    ids = torch.zeros(6, 1, dtype=torch.long)
    undecided = total = 0
    for w in SETTINGS:
        out = x.clone()
        for proc in _hf_list(T, k, p, w):
            out = proc(ids, out)
        for b in range(x.shape[0]):
            total += 1
            z = N.scaled(x[b].numpy(), T)
            keep, tm = N.top_p_keep(z, N.topk_keep(z, k), p)
            kept, _, m = Wr.warp_keep(z, keep, _table(w))
            if not (N.decided(tm, REL) and Wr.decided(m, REL, GAP)):
                undecided += 1
                continue
            np.testing.assert_array_equal(kept, torch.isfinite(out[b]).numpy(), err_msg=f"{w} row {b}")
    print(f"T={T} k={k} p={p}: {undecided} of {total} rows undecided")
    # with top-p the boundary of a near-flat row (every third one) falls among many equal bf16 logits, which HF's sort
    # splits in an arbitrary order: those rows are undecided by construction
    assert undecided <= (total // 2 if p < 1.0 else total // 8), f"{undecided} undecided rows of {total}"


def test_typical_can_drop_the_argmax():
    from transformers.generation.logits_process import TypicalLogitsWarper
    rng = torch.Generator().manual_seed(3)
    x = _rows(rng, 1, 1.0)
    z = N.scaled(x[0].numpy(), 1.0)
    kept, zmax, m = Wr.warp_keep(z, np.ones(V, dtype=bool), _table((None, 0.2, None, None)))
    assert Wr.decided(m, REL, GAP) and not kept[int(np.argmax(z))] and zmax < z.max()
    hf = TypicalLogitsWarper(mass=0.2)(torch.zeros(1, 1, dtype=torch.long), x.clone())
    np.testing.assert_array_equal(kept, torch.isfinite(hf[0]).numpy())


@pytest.mark.parametrize("w", SETTINGS)
def test_host_warpers_match_transformers(w):
    """The stepwise path's processors (_host_processors with warpers) against HF's list, on the same fp32 logits: bit
    for bit"""
    from video_chatgpt.model import VideoChatGPTLlamaForCausalLM as M
    rng = torch.Generator().manual_seed(17)
    x = _rows(rng, 6, 0.7)
    ids = torch.randint(0, V, (6, 20), generator=rng)
    for T, k, p in ((0.7, 50, 0.9), (1.5, 0, 1.0)):
        want = x.clone()
        for proc in _hf_list(T, k, p, w):
            want = proc(ids, want)
        got = M._host_processors(ids, x.clone(), True, T, k, p, 1.0, warpers=_table(w))
        assert torch.equal(got, want), (w, T, k, p)


# ---- host rejections ----------------------------------------------------------------------------------------------
class WarpFake(TokenSetFake):
    """TokenSetFake with the warper entries of the sampling table: set_sampling / set_sampling_ex turn them off, as
    the device does. Every prefill and decode step checks that each slot holding a request has that request's
    warpers (expect: request -> _warper_args' value)."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.warp = [None] * self.n_slots
        self.expect, self.slot_req, self.bad = {}, {}, []
        self.checked = self.writes_w = 0

    def set_sampling(self, clips, temperature, top_k, seed):
        super().set_sampling(clips, temperature, top_k, seed)
        for s in clips:
            self.warp[s] = None

    def set_sampling_ex(self, clips, temperature, top_k, seed, top_p, repetition_penalty):
        super().set_sampling_ex(clips, temperature, top_k, seed, top_p, repetition_penalty)
        for s in clips:
            self.warp[s] = None

    def set_warpers(self, clips, min_p, typical_p, epsilon, eta):
        self.writes_w += 1
        for s, *w in zip(clips, min_p, typical_p, epsilon, eta):
            self.warp[s] = None if tuple(w) == Wr.OFF else tuple(w)

    def _check(self, s, r):
        self.checked += 1
        if self.warp[s] != self.expect.get(r):
            self.bad.append((s, r, self.warp[s], self.expect.get(r)))

    def _prefill(self, s, ids):
        r = int(torch.as_tensor(ids).reshape(-1)[0]) - REQ0
        self.slot_req[s] = r
        self._check(s, r)
        return super()._prefill(s, ids)

    def slot_decode(self, first_tok, positions, n_new):
        for s in range(first_tok.shape[0]):
            r = (self.owner if self.kv_blocks else self.slot_req).get(s)
            if r is not None:
                self._check(s, r)
        return super().slot_decode(first_tok, positions, n_new)


def _fake_model(slots=4, kv_blocks=None):
    eng = WarpFake(640, slots, kv_blocks or 0)
    m = _model(eng, max_batch=slots, max_seq=640, kv_blocks=kv_blocks)
    m._SLOT_CHUNK = 8
    return m, eng


KEYS = ("min_p", "typical_p", "epsilon_cutoff", "eta_cutoff")


@pytest.mark.parametrize("kw,msg", [(dict(min_p=1.5), "min_p"), (dict(min_p=-0.1), "min_p"),
                                    (dict(min_p=float("nan")), "min_p"), (dict(typical_p=0.0), "typical_p"),
                                    (dict(typical_p=-1.0), "typical_p")])
def test_rejections(kw, msg):
    m, eng = _fake_model()
    req = {"input_ids": torch.tensor([REQ0, 5, 6])}
    samp = dict(do_sample=True, seed=1)
    with pytest.raises(ValueError, match=msg):
        m.generate_requests([req], max_new_tokens=4, **samp, **kw)
    with pytest.raises(ValueError, match=msg):
        m.generate_requests([dict(req, **kw)], max_new_tokens=4, **samp)
    with pytest.raises(ValueError, match=msg):
        m._warper_args(*[kw.get(k) for k in KEYS])
    assert eng.calls == []


def test_off_values_and_greedy():
    m, _ = _fake_model()
    assert m._warper_args(None, None, None, None) is None
    assert m._warper_args(None, 1.0, 0.0, 0.0) is None
    assert m._warper_args(None, 1.5, 1.0, 2.0) is None             # HF adds none of them there
    assert m._warper_args(0.0, None, None, None) is None      # on in HF, but it removes nothing
    assert m._warper_args(0.1, 0.5, 3e-4, 0.2) == (0.1, 0.5, 3e-4, 0.2)
    assert m._warper_args(0.1, 0.5, 3e-4, 0.2, sampled=False) is None
    m.config.vocab_size = 60000
    with pytest.raises(ValueError, match="vocabulary"):
        m._warper_args(0.1, None, None, None)
    assert m._warper_args(0.1, None, None, None, device=False) == (0.1, 1.0, 0.0, 0.0)


@pytest.mark.parametrize("kw", [dict(num_beams=2), dict(penalty_alpha=0.6, top_k=4)])
@pytest.mark.parametrize("key", KEYS)
def test_beams_and_contrastive_reject_warpers(kw, key):
    m, eng = _fake_model()
    with pytest.raises(NotImplementedError, match=key):
        m.generate(torch.tensor([[REQ0, 5, 6]]), **kw, **{key: 0.5})
    assert eng.calls == []


@pytest.mark.parametrize("kw", [dict(num_beams=2), dict(penalty_alpha=0.6, top_k=4)])
def test_beams_and_contrastive_accept_off_values(kw):
    """HF GenerationConfig's defaults (typical_p 1.0, epsilon_cutoff 0.0, eta_cutoff 0.0) and min_p 0 turn nothing
    on, so they do not stop a beam or contrastive call (which fails later here only for want of a device)"""
    m, _ = _fake_model()
    for off in (dict(typical_p=1.0, epsilon_cutoff=0.0, eta_cutoff=0.0), dict(min_p=0.0), dict(typical_p=2.0)):
        try:
            m.generate(torch.tensor([[REQ0, 5, 6]]), **kw, **off)
        except NotImplementedError as e:
            raise AssertionError(f"{off} rejected: {e}")
        except Exception:   # noqa: BLE001  (the fake engine has no beam / contrastive entry points)
            pass


# ---- warper entries in flight -------------------------------------------------------------------------------------
OPTS = [dict(min_p=0.1), dict(), dict(typical_p=0.5, eta_cutoff=3e-2), dict(epsilon_cutoff=3e-4), dict(min_p=0.0)]


def _requests(n, rng, long=False, new=None):
    reqs = []
    for i in range(n):
        S = int(torch.randint(600, 630, (1,), generator=rng)) if long and i % 3 == 0 else \
            int(torch.randint(5, 40, (1,), generator=rng))
        ids = torch.cat([torch.tensor([REQ0 + i]), torch.randint(1, 30000, (S - 1,), generator=rng)])
        reqs.append(dict(input_ids=ids, max_new_tokens=new or int(torch.randint(3, 12, (1,), generator=rng)),
                         do_sample=i % 4 != 3, seed=7 * i, **OPTS[i % len(OPTS)]))
    return reqs


def _expect(m, eng, reqs):
    for i, r in enumerate(reqs):
        eng.expect[i] = m._warper_args(*[r.get(k) for k in KEYS], sampled=r["do_sample"])


@pytest.mark.parametrize("packed", [False, True])
def test_entries_contiguous(packed):
    rng = torch.Generator().manual_seed(1)
    reqs = _requests(10, rng)
    m, eng = _fake_model()
    _expect(m, eng, reqs)
    m.generate_requests(reqs, eos_token_id=None, packed_admission=packed)
    assert eng.checked > 0 and not eng.bad, eng.bad[:3]
    assert eng.writes_w > 0 and eng.warp == [None] * eng.n_slots     # every slot off after the call


@pytest.mark.parametrize("packed", [False, True])
def test_entries_paged_preemption(packed):
    rng = torch.Generator().manual_seed(2)
    reqs = _requests(10, rng, new=200)
    m, eng = _fake_model(kv_blocks=6)
    _expect(m, eng, reqs)
    eng.lens = {i: torch.as_tensor(r["input_ids"]).numel() + 200 for i, r in enumerate(reqs)}
    m.generate_requests(reqs, eos_token_id=None, packed_admission=packed)
    assert m.last_kv_stats["preemptions"] > 0
    assert eng.checked > 0 and not eng.bad, eng.bad[:3]
    assert not eng.violations


def test_entries_chunked():
    rng = torch.Generator().manual_seed(3)
    reqs = _requests(6, rng, long=True)
    m, eng = _fake_model(kv_blocks=40)
    _expect(m, eng, reqs)
    eng.lens = {i: torch.as_tensor(r["input_ids"]).numel() + r["max_new_tokens"] for i, r in enumerate(reqs)}

    def chunk(s, start, total, ids):
        ids = [int(t) for t in torch.as_tensor(ids).reshape(-1)]
        for j, t in enumerate(ids):
            eng._write(s, start + j, t)
        if start == 0:
            eng.owner[s] = ids[0] - REQ0
        eng._check(s, eng.owner[s])
        return P._tok(eng._read(s, start + len(ids)), start + len(ids) - 1, eng.seed[s])
    eng.slots_prefill_chunk = lambda slots, starts, totals, ids_list, feats, vs: torch.tensor(
        [chunk(s, st, tot, ids) for s, st, tot, ids in zip(slots, starts, totals, ids_list)], dtype=torch.int32)
    m.generate_requests(reqs, eos_token_id=None, chunked_prefill=True)
    assert m.last_kv_stats["chunk_calls"] > 0
    assert eng.checked > 0 and not eng.bad, eng.bad[:3]


@pytest.mark.parametrize("packed", [False, True])
def test_entries_of_continuations(packed):
    """A "continues" request's slot holds its own warpers when its tail is prefilled and at every decode step of the
    turn (the entry is written at its admission, before the tail prefill), for every turn of every conversation"""
    import test_sessions_cpu as SC

    class SessionWarpFake(WarpFake, SC.SessionFake):
        def set_block_table(self, table):     # which conversation (its first id) owns each slot
            super().set_block_table(table)
            self.owner = {s: self.pool[r[0]][0] - REQ0 for s, r in enumerate(self.table)
                          if r[0] != 0 and self.pool[r[0]][0] >= REQ0}

        def slots_prefill_append(self, slots, starts, ids_list, tok_out=None):
            for s in slots:
                self._check(s, self.owner.get(s))
            return super().slots_prefill_append(slots, starts, ids_list, tok_out)

    eng = SessionWarpFake(4, 12)
    m = _model(eng, max_batch=4, max_seq=SC.MAX_SEQ, kv_blocks=12)
    m._SLOT_CHUNK = 8
    eng.model = m
    convs = SC.conversations(5, 3, seed=4)
    w = dict(min_p=0.1, typical_p=0.7)
    eng.expect = {c: m._warper_args(0.1, 0.7, None, None) for c in range(len(convs))}
    SC.run_sessions(m, convs, 3, packed_admission=packed, do_sample=True, seed=3, **w)
    assert not eng.violations
    n_append = sum(1 for c in eng.calls if c[0] == "append")
    assert n_append > 0 and eng.checked > n_append and not eng.bad, eng.bad[:3]
