"""CPU tests of score_candidates: the rejections, the round planner (candidates.plan), and the host code end to end
with a fake engine whose cache slots hold token ids and whose continuation runs a tiny HF LlamaForCausalLM on what the
slot holds. A fork one column short, a label shifted by a row, or a slot a round reuses too early changes the values
or trips the fake's checks. The yardstick: sum over t of log_softmax(model(prompt + option).logits)[S - 1 + t,
c_{t+1}] (0-based rows), within fp32 rounding."""
import pytest
import torch

from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
from video_chatgpt.model import candidates as C

V = 97
PATCH = 96               # the video placeholder id of these tests
NV = 4                   # video rows per clip of the fake engine


def _hf():
    from transformers import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    cfg = LlamaConfig(vocab_size=V, hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4,
                      max_position_embeddings=256)
    return LlamaForCausalLM(cfg).eval()


class FakeEngine:
    """Cache slots as lists of token ids. slots_score_append runs the HF model on slot[:start] + ids and scores its
    rows start .. against the labels. Every call enforces the preconditions its C entry checks (include/vcl.h)."""
    NV = NV

    def __init__(self, n_slots, hf=None, max_seq=128):
        self.hf = hf
        self.max_seq = max_seq
        self.slots = [None] * n_slots
        self.calls = []

    def _slots_ok(self, slots):
        assert 1 <= len(slots) <= len(self.slots) and len(slots) == len(set(slots))
        assert all(0 <= s < len(self.slots) for s in slots)

    def slots_prefill(self, slots, ids_list, feats_list, vid_starts, tok_out=None):
        self.calls.append(("prefill", list(slots), [int(torch.as_tensor(i).numel()) for i in ids_list]))
        self._slots_ok(slots)
        for s, ids in zip(slots, ids_list):
            assert 1 <= torch.as_tensor(ids).numel() <= min(C.PACKED_MAX_S, self.max_seq)
            self.slots[s] = [int(t) for t in torch.as_tensor(ids).reshape(-1)]
        return torch.zeros(len(slots), dtype=torch.int32)

    def slot_prefill(self, slot, ids, video_feats, vid_start, tok_out=None):
        self.calls.append(("slot_prefill", slot, int(ids.numel())))
        assert 0 <= slot < len(self.slots) and 1 <= ids.numel() <= self.max_seq
        self.slots[slot] = [int(t) for t in ids.reshape(-1)]
        return torch.zeros(1, dtype=torch.int32)

    def slots_fork(self, src, dst, cols):
        self.calls.append(("fork", list(src), list(dst), list(cols)))
        assert 0 <= len(src) <= len(self.slots) and not set(dst) & set(src) and len(dst) == len(set(dst))
        for s, d, c in zip(src, dst, cols):
            assert 0 <= s < len(self.slots) and 0 <= d < len(self.slots) and 0 <= c <= self.max_seq
            assert self.slots[s] is not None and len(self.slots[s]) >= c
            self.slots[d] = list(self.slots[s][:c])

    def slots_score_append(self, slots, starts, ids_list, labels_list):
        self.calls.append(("score", list(slots), list(starts), [int(i.numel()) for i in ids_list]))
        self._slots_ok(slots)
        assert sum(int(i.numel()) for i in ids_list) <= len(self.slots) * self.max_seq      # the activations
        lps, grs = [], []
        for s, st, ids, lab in zip(slots, starts, ids_list, labels_list):
            assert st >= 0 and 1 <= ids.numel() <= 512 and st + ids.numel() <= self.max_seq and lab.numel() == ids.numel()
            held = self.slots[s]
            assert held is not None and len(held) >= st, f"slot {s} holds {held and len(held)} columns, needs {st}"
            full = held[:st] + [int(t) for t in ids]
            self.slots[s] = full
            with torch.no_grad():
                logits = self.hf(torch.tensor([full])).logits[0, st:].float()
            lp = torch.log_softmax(logits, -1)
            lab = torch.as_tensor(lab)
            lps.append(lp[torch.arange(len(lab)), lab])
            grs.append((logits.argmax(-1) == lab).to(torch.uint8))
        return torch.cat(lps), torch.cat(grs)


def _model(eng, max_slots=4, max_seq=128, kv_blocks=None):
    cfg = VideoChatGPTConfig(hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4,
                             vocab_size=V)
    m = VideoChatGPTLlamaForCausalLM(cfg, clip_config={}, max_batch=max_slots, max_seq=max_seq, max_slots=max_slots,
                                     kv_blocks=kv_blocks)
    m.get_model().vision_config.vid_patch_token = PATCH
    m.device = torch.device("cpu")
    m._engine, m._llm_loaded = eng, True
    return m


def _prompt(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 90, (n,), generator=g)


def _options(lens, seed):
    return [_prompt(L, seed * 31 + j) for j, L in enumerate(lens)]


def _ref(hf, prompt, option):
    with torch.no_grad():
        logits = hf(torch.cat([prompt, option])[None]).logits[0].float()
    S, L = prompt.numel(), option.numel()
    lp = torch.log_softmax(logits, -1)[torch.arange(S - 1, S - 1 + L), option]
    greedy = bool((logits[S - 1:S - 1 + L].argmax(-1) == option).all())
    return lp, greedy


# ------------------------------------------------------------------------------------------------
# rejections
REJECT = [
    (lambda: ([_prompt(5, 1)], [[]]), None, "prompt 0: the option list is empty"),
    (lambda: ([_prompt(5, 1)], [[torch.tensor([], dtype=torch.int64)]]), None, "prompt 0 option 0 is empty"),
    (lambda: ([_prompt(5, 1), _prompt(6, 2)], [[torch.tensor([3])], [torch.tensor([4]), torch.tensor([1, V])]]), None,
     "prompt 1 option 1: token id 97 outside the vocabulary"),
    (lambda: ([_prompt(5, 1)], [[torch.tensor([-1])]]), None, "prompt 0 option 0: token id -1 outside"),
    (lambda: ([torch.tensor([1, 2, V + 3])], [[torch.tensor([1])]]), None, "prompt 0: token id 100 outside"),
    (lambda: ([_prompt(5, 1)], [[torch.tensor([3]), torch.tensor([4, PATCH])]]), None,
     "prompt 0 option 1: a video placeholder id"),
    (lambda: ([_prompt(100, 1)], [[torch.tensor([3] * 28), torch.tensor([4] * 29)]]), None,
     "prompt 0 option 1: prompt 100 \\+ option 29 tokens exceed max_seq 128"),
    (lambda: ([_prompt(5, 1)], [[torch.tensor([3])], [torch.tensor([3])]]), None, "candidates must be a list of 1"),
    (lambda: ([_prompt(5, 1), _prompt(5, 2)], [[torch.tensor([3])], [torch.tensor([3])]]), torch.zeros(1, NV, 1024),
     r"must be \[2, 4, 1024\]"),
    (lambda: ([_prompt(5, 1)], [[torch.tensor([3])]]), [torch.zeros(NV + 1, 1024)], r"prompt 0: .* must be \[4, 1024\]"),
    # the channel count of the vision tower (1024), checked before any device work
    (lambda: ([_prompt(5, 1), _prompt(5, 2)], [[torch.tensor([3])], [torch.tensor([3])]]),
     [None, torch.zeros(NV, 8)], r"prompt 1: .* must be \[4, 1024\], got \(4, 8\)"),
    (lambda: ([_prompt(5, 1)], [[torch.tensor([3])]]), torch.zeros(1, NV, 512), r"prompt 0: .* must be \[4, 1024\]"),
]


@pytest.mark.parametrize("case,feats,match", REJECT)
def test_rejections(case, feats, match):
    eng = FakeEngine(4)
    m = _model(eng)
    prompts, cands = case()
    with pytest.raises(ValueError, match=match):
        m.score_candidates(prompts, cands, video_spatio_temporal_features=feats)
    assert eng.calls == []


def test_rejects_an_option_over_512_tokens():
    eng = FakeEngine(4, max_seq=1024)
    m = _model(eng, max_seq=1024)
    with pytest.raises(ValueError, match="prompt 0 option 0: 513 tokens, more than 512"):
        m.score_candidates([_prompt(5, 1)], [[torch.ones(513, dtype=torch.int64)]])
    assert eng.calls == []


def test_paged_model_raises():
    m = _model(FakeEngine(4), kv_blocks=8)
    with pytest.raises(NotImplementedError, match="score_candidates"):
        m.score_candidates([_prompt(5, 1)], [[torch.tensor([3])]])


# ------------------------------------------------------------------------------------------------
# the planner
def _flat(rounds):
    return [(r.prefill, r.forks, [s for s in r.seqs]) for r in rounds]


def test_plan_packs_prompts_in_order():
    r = C.plan([10, 20, 5], [[3, 1], [2, 2, 2], [4]], n_slots=4, max_rows=1000)
    assert _flat(r) == [
        ([(0, 0)], [(0, 1, 9)], [(0, 0, 0, 9, 3), (0, 1, 1, 9, 1)]),
        # prompt 1's three options do not fit the two slots left: a new round, then prompt 2 joins it
        ([(1, 0), (2, 3)], [(0, 1, 19), (0, 2, 19)],
         [(1, 0, 0, 19, 2), (1, 1, 1, 19, 2), (1, 2, 2, 19, 2), (2, 0, 3, 4, 4)]),
    ]


def test_plan_row_budget():
    r = C.plan([10, 10], [[30, 30], [30]], n_slots=8, max_rows=80)
    assert [len(x.seqs) for x in r] == [2, 1]


def test_plan_splits_a_prompt_with_more_options_than_slots():
    r = C.plan([7, 9, 3], [[1], [2, 3, 4, 5, 6], [1]], n_slots=2, max_rows=1000)
    assert _flat(r) == [
        ([(0, 0)], [], [(0, 0, 0, 6, 1)]),
        # prompt 1 alone: slot 0 prefilled once, hosting an option only in the last round
        ([(1, 0)], [(0, 1, 8)], [(1, 0, 1, 8, 2)]),
        ([], [(0, 1, 8)], [(1, 1, 1, 8, 3)]),
        ([], [(0, 1, 8)], [(1, 2, 1, 8, 4)]),
        ([], [(0, 1, 8)], [(1, 3, 0, 8, 5), (1, 4, 1, 8, 6)]),
        ([(2, 0)], [], [(2, 0, 0, 2, 1)]),
    ]


def test_plan_single_slot_prefills_every_round():
    r = C.plan([4, 6], [[1, 2], [3]], n_slots=1, max_rows=1000)
    assert _flat(r) == [
        ([(0, 0)], [], [(0, 0, 0, 3, 1)]),
        ([(0, 0)], [], [(0, 1, 0, 3, 2)]),
        ([(1, 0)], [], [(1, 0, 0, 5, 3)]),
    ]


def test_plan_prompt_of_one_token():
    r = C.plan([1], [[2, 3]], n_slots=2, max_rows=100)
    assert _flat(r) == [([(0, 0)], [(0, 1, 0)], [(0, 0, 0, 0, 2), (0, 1, 1, 0, 3)])]


# ------------------------------------------------------------------------------------------------
# end to end through the host code
@pytest.fixture(scope="module")
def hf():
    return _hf()


def _check(out, hf, prompts, cands):
    assert len(out) == len(prompts)
    for b, (p, opts) in enumerate(zip(prompts, cands)):
        o = out[b]
        assert o["logprob"].dtype == torch.float64 and o["logprob"].shape == (len(opts),)
        assert o["greedy"].dtype == torch.bool and o["greedy"].shape == (len(opts),)
        for j, c in enumerate(opts):
            lp, greedy = _ref(hf, p, c)
            tl = o["token_logprobs"][j]
            assert tl.dtype == torch.float32 and tl.shape == (c.numel(),)
            torch.testing.assert_close(tl, lp, rtol=1e-5, atol=1e-5, msg=f"prompt {b} option {j}")
            assert abs(float(o["logprob"][j]) - float(lp.double().sum())) <= 1e-4 * max(1.0, abs(float(lp.sum())))
            assert float(o["logprob"][j]) == sum(float(x) for x in tl.tolist())
            assert bool(o["greedy"][j]) == greedy


@pytest.mark.parametrize("max_slots", [4, 2, 1])
def test_one_prompt(hf, max_slots):
    eng = FakeEngine(max_slots, hf)
    m = _model(eng, max_slots=max_slots)
    p = _prompt(20, 3)
    opts = _options([1, 5, 3, 1, 7], 3)
    _check(m.score_candidates([p], [opts]), hf, [p], [opts])


def test_three_left_padded_prompts(hf):
    eng = FakeEngine(4, hf)
    m = _model(eng)
    prompts = [_prompt(12, 5), _prompt(30, 6), _prompt(1, 7)]
    S = max(p.numel() for p in prompts)
    ids = torch.zeros(3, S, dtype=torch.int64)
    mask = torch.zeros(3, S, dtype=torch.int64)
    for b, p in enumerate(prompts):
        ids[b, S - p.numel():] = p
        mask[b, S - p.numel():] = 1
    cands = [_options([2, 1], 5), _options([1, 1, 4], 6), _options([6, 2, 1, 3, 2], 7)]
    out = m.score_candidates(ids, cands, attention_mask=mask)
    _check(out, hf, prompts, cands)
    # prompt 2 has more options than slots: its rounds run alone, and its slot is prefilled once
    assert sum(1 for c in eng.calls if c[0] == "prefill") == 3


def test_one_token_prompt(hf):
    """a BOS-only prompt: its options start at column 0 of their slots (a sequence new to its slot)"""
    eng = FakeEngine(4, hf)
    m = _model(eng)
    p, opts = torch.tensor([1]), _options([1, 4, 2], 9)
    _check(m.score_candidates([p], [opts]), hf, [p], [opts])
    assert [c for c in eng.calls if c[0] == "score"] == [("score", [0, 1, 2], [0, 0, 0], [1, 4, 2])]


def test_greedy_option(hf):
    """an option built from the model's own arg-max tokens is greedy; changing its last token makes it not"""
    p = _prompt(9, 11)
    seq = p.clone()
    with torch.no_grad():
        for _ in range(4):
            seq = torch.cat([seq, hf(seq[None]).logits[0, -1].argmax()[None]])
    good = seq[p.numel():]
    bad = good.clone()
    bad[-1] = (bad[-1] + 1) % 90
    out = _model(FakeEngine(4, hf)).score_candidates([p], [[good, bad]])
    assert out[0]["greedy"].tolist() == [True, False]


def test_state_after_the_call(hf):
    m = _model(FakeEngine(2, hf), max_slots=2)
    m._last_out, m._after_beams = torch.zeros(1, 3, dtype=torch.int64), True
    m.score_candidates([_prompt(4, 1)], [[torch.tensor([1])]])
    with pytest.raises(ValueError, match="no previous generate"):
        m.generate_continue(torch.tensor([[1, 2]]))
