"""CPU tests of packed admission in the in-flight scheduler (generate_requests(packed_admission=True)), driven by the
fake engine of test_inflight_cpu.py with a slots_prefill: which requests one packed call admits and in which order,
prompts over the packed limit going alone, the activation bound, and that the flag off never packs."""
import torch

from test_inflight_cpu import EOS, FakeEngine, StopAfter, _model, _new, _req


class PackedFakeEngine(FakeEngine):
    def slots_prefill(self, slots, ids_list, feats_list, vid_starts, tok_out=None):
        rs = [int(ids.reshape(-1)[0]) - 100 for ids in ids_list]
        self.calls.append(("packed", list(slots), rs, [ids.numel() for ids in ids_list]))
        out = torch.zeros(len(slots), dtype=torch.int32)
        for j, (s, r) in enumerate(zip(slots, rs)):
            self.slot[s] = [r, 1]
            out[j] = self._tok(r, 0)
        return out


def _packed(calls):
    return [c for c in calls if c[0] == "packed"]


def test_first_fill_is_one_call_and_refills_follow_queue_order():
    m = _model(max_batch=4, eng=PackedFakeEngine())
    m._SLOT_CHUNK = 4
    eng = m._engine
    lens = [2, 9, 3, 12, 7, 4, 10, 6]
    outs = m.generate_requests([_req(r, max_new_tokens=n) for r, n in enumerate(lens)], eos_token_id=None,
                               packed_admission=True)
    for r, (o, n) in enumerate(zip(outs, lens)):
        assert _new(o) == [1000 * r + k + 1 for k in range(n)]
    packed = _packed(eng.calls)
    assert packed[0] == ("packed", [0, 1, 2, 3], [0, 1, 2, 3], [8] * 4)
    # the first chunk (the prefill's token + 4 steps) finishes requests 0 (2 tokens) and 2 (3 tokens): one call
    # refills slots 0 and 2 with the next two queued requests
    assert packed[1][1:3] == ([0, 2], [4, 5])
    assert [r for c in packed for r in c[2]] == list(range(len(lens)))
    assert not any(c[0] == "prefill" for c in eng.calls)


def test_same_results_as_one_at_a_time():
    """11 requests over 4 slots and 20 over 9, outputs of 1 to 40 tokens, EOS, a per-request stopping criterion and
    one prompt over the packed limit: every request gets what one-at-a-time admission gives it."""
    toks = {3: [11, EOS, 13], 6: [5, 6, EOS], 14: [7, 8, 9, EOS]}
    for n_slots, n_req in ((4, 11), (9, 20)):
        lens = [1 + (7 * r) % 40 for r in range(n_req)]
        got, seen = {}, {}
        for packed in (False, True):
            crit = StopAfter(1000 * 5 + 4)                   # request 5 stops at its 4th token
            reqs = [_req(r, S=6 + 3 * r, max_new_tokens=n) for r, n in enumerate(lens)]
            reqs[2] = _req(2, S=530, max_new_tokens=lens[2])
            reqs[5]["stopping_criteria"] = [crit]
            m = _model(max_batch=16, max_seq=600, eng=PackedFakeEngine(toks))
            got[packed] = [o.tolist() for o in m.generate_requests(reqs, slots=n_slots, packed_admission=packed)]
            seen[packed] = crit.seen
            calls = m._engine.calls
            assert bool(_packed(calls)) == packed
            if packed:   # only the 530-token prompt takes the single path
                assert [c[2] for c in calls if c[0] == "prefill"] == [2]
        assert got[True] == got[False], n_slots
        assert seen[True] == seen[False]
        assert _new(torch.tensor(got[True][5]), 6 + 15) == [5001, 5002, 5003, 5004]


def test_long_prompt_alone_the_rest_packed():
    m = _model(max_batch=4, max_seq=700, eng=PackedFakeEngine())
    eng = m._engine
    reqs = [_req(0, S=100, max_new_tokens=2), _req(1, S=600, max_new_tokens=2), _req(2, S=512, max_new_tokens=2),
            _req(3, S=513, max_new_tokens=2)]
    outs = m.generate_requests(reqs, eos_token_id=None, packed_admission=True)
    assert [o.shape[1] for o in outs] == [102, 602, 514, 515]
    admissions = [c for c in eng.calls if c[0] != "decode"]
    assert admissions == [("prefill", 1, 1, 600, False, -2 ** 31), ("prefill", 3, 3, 513, False, -2 ** 31),
                          ("packed", [0, 2], [0, 2], [100, 512])]


def test_full_slots_fit_the_activations():
    """Every slot refilled with the longest prompt max_seq allows still fits max_batch * max_seq tokens: one call."""
    m = _model(max_batch=4, max_seq=513, eng=PackedFakeEngine())
    eng = m._engine
    m.generate_requests([_req(r, S=512, max_new_tokens=1) for r in range(8)], eos_token_id=None, packed_admission=True)
    assert [(c[1], c[3]) for c in _packed(eng.calls)] == [([0, 1, 2, 3], [512] * 4)] * 2


def test_flag_off_never_packs():
    m = _model(max_batch=4, eng=PackedFakeEngine())
    eng = m._engine
    m.generate_requests([_req(r, max_new_tokens=3) for r in range(9)], eos_token_id=None)
    assert not _packed(eng.calls) and sum(c[0] == "prefill" for c in eng.calls) == 9
