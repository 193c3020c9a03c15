"""CPU tests of the in-flight scheduler (generate_requests) driven by a fake engine that emits scripted tokens:
admission order, refill of freed slots, the retirement rules (EOS, per-request max_new_tokens, stopping criteria
called token by token) and the host-side checks that run before any device work."""
import pytest
import torch

V = 32003
EOS = 31999                 # no scripted stream emits it unless told to


class FakeEngine:
    """Stands in for vcl_native.Engine: request r (told by its first prompt id, 100 + r) generates the tokens
    script[r] = 1000*r + 1, 1000*r + 2, ... unless `tokens` overrides them. Records every call."""

    NV = 356

    def __init__(self, tokens=None):
        self.tokens = tokens or {}
        self.calls = []
        self.slot = {}              # slot -> [request, tokens emitted so far]

    def _tok(self, r, k):
        seq = self.tokens.get(r)
        return seq[k] if seq is not None and k < len(seq) else 1000 * r + k + 1

    def slot_prefill(self, slot, ids, video_feats, vid_start, tok_out=None):
        r = int(ids.reshape(-1)[0]) - 100
        self.calls.append(("prefill", slot, r, ids.numel(), video_feats is not None, int(vid_start[0])))
        self.slot[slot] = [r, 1]
        tok_out[0] = self._tok(r, 0)
        return tok_out

    def slot_decode(self, first_tok, positions, n_new):
        self.calls.append(("decode", list(positions), n_new))
        out = torch.zeros(first_tok.shape[0], n_new, dtype=torch.int32)
        out[:, 0] = first_tok
        for s in range(first_tok.shape[0]):
            if s not in self.slot:
                assert positions[s] == 0, "an idle slot is parked at position 0"
                continue
            r, k = self.slot[s]
            for j in range(1, n_new):
                out[s, j] = self._tok(r, k + j - 1)
            self.slot[s][1] = k + n_new - 1
        return out


def _model(max_batch=4, max_seq=64, eng=None):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    cfg = VideoChatGPTConfig(hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4,
                             vocab_size=V, eos_token_id=EOS)
    m = VideoChatGPTLlamaForCausalLM(cfg, clip_config={}, max_batch=max_batch, max_seq=max_seq)
    vc = m.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = 32000, 32001, 32002, True
    m.device = torch.device("cpu")
    m._engine, m._llm_loaded = eng if eng is not None else FakeEngine(), True
    return m


def _req(r, S=8, **kw):
    return dict(input_ids=torch.tensor([100 + r] + [7] * (S - 1)), **kw)


def _new(out, S=8):
    return out[0, S:].tolist()


def test_admission_order_refill_and_lengths():
    m = _model(max_batch=2)
    m._SLOT_CHUNK = 4
    eng = m._engine
    lens = [3, 9, 2, 5, 1]
    outs = m.generate_requests([_req(r, max_new_tokens=n) for r, n in enumerate(lens)], eos_token_id=None)
    for r, (o, n) in enumerate(zip(outs, lens)):
        assert o.shape == (1, 8 + n) and o.dtype == torch.int64
        assert _new(o) == [1000 * r + k + 1 for k in range(n)]
        assert o[0, 0] == 100 + r
    prefills = [(c[1], c[2]) for c in eng.calls if c[0] == "prefill"]
    # requests enter in order; a freed slot takes the next queued request after the chunk that freed it
    assert [r for _, r in prefills] == [0, 1, 2, 3, 4]
    assert prefills[:2] == [(0, 0), (1, 1)]
    assert prefills[2] == (0, 2)                      # request 0 (3 tokens) left slot 0 after the first chunk
    decodes = [c for c in eng.calls if c[0] == "decode"]
    assert decodes[0] == ("decode", [8, 8], 5)        # both slots at their prompt length, chunk 4 (+ the fed token)
    assert all(d[2] == 5 for d in decodes)


def test_eos_ends_a_request_and_leaves_its_neighbours():
    toks = {1: [11, 12, EOS, 14, 15, 16]}
    m = _model(max_batch=3, eng=FakeEngine(toks))
    m._SLOT_CHUNK = 4
    outs = m.generate_requests([_req(r) for r in range(3)], max_new_tokens=6)
    assert _new(outs[1]) == [11, 12, EOS]
    for r in (0, 2):
        assert _new(outs[r]) == [1000 * r + k + 1 for k in range(6)]
    # eos_token_id=None decodes the full length
    m2 = _model(max_batch=3, eng=FakeEngine(toks))
    outs = m2.generate_requests([_req(1)], max_new_tokens=6, eos_token_id=None)
    assert _new(outs[0]) == toks[1]


def test_eos_at_the_first_token_and_one_token_requests():
    m = _model(max_batch=2, eng=FakeEngine({0: [EOS, 5, 6]}))
    outs = m.generate_requests([_req(0), _req(1, max_new_tokens=1), _req(2, max_new_tokens=2)], max_new_tokens=3)
    assert _new(outs[0]) == [EOS]
    assert _new(outs[1]) == [1001]
    assert _new(outs[2]) == [2001, 2002]


class StopAfter:
    """A per-prompt criterion like KeywordsStoppingCriteria: its first call only records the prompt length."""

    def __init__(self, token):
        self.token, self.start_len, self.seen = token, None, []

    def __call__(self, output_ids, scores=None):
        self.seen.append(output_ids.shape[1])
        if self.start_len is None:
            self.start_len = output_ids.shape[1]
            return False
        return int(output_ids[0, -1]) == self.token


def test_stopping_criteria_per_request_token_by_token():
    c0, c2 = StopAfter(3), StopAfter(99999)
    m = _model(max_batch=2)
    m._SLOT_CHUNK = 4
    outs = m.generate_requests([_req(0, stopping_criteria=[c0]), _req(1), _req(2, stopping_criteria=[c2])],
                               max_new_tokens=6, eos_token_id=None)
    assert _new(outs[0]) == [1, 2, 3]
    assert c0.seen == [9, 10, 11]                     # the prefix after every new token, as a stepwise generate
    assert _new(outs[1]) == [1001 + k for k in range(6)]
    assert c2.seen == [9, 10, 11, 12, 13, 14] and _new(outs[2]) == [2001 + k for k in range(6)]


def test_positions_near_max_seq_shorten_the_chunk():
    m = _model(max_batch=2, max_seq=20)
    m._SLOT_CHUNK = 8
    eng = m._engine
    outs = m.generate_requests([_req(0, S=14, max_new_tokens=6), _req(1, S=4, max_new_tokens=10)], eos_token_id=None)
    assert _new(outs[0], 14) == [1 + k for k in range(6)] and _new(outs[1], 4) == [1001 + k for k in range(10)]
    for c in eng.calls:
        if c[0] == "decode":
            assert max(c[1]) + c[2] - 1 <= 20


def test_video_request_is_checked_and_passed_on():
    m = _model(max_seq=400)
    eng = m._engine
    n_vid = eng.NV
    ids = torch.tensor([100, 7, 32001] + [32000] * n_vid + [32002, 7, 7])
    out = m.generate_requests([dict(input_ids=ids[None], video_spatio_temporal_features=torch.zeros(n_vid, 1024),
                                    max_new_tokens=2)], eos_token_id=None, slots=1)
    assert out[0].shape == (1, ids.numel() + 2)
    assert eng.calls[0] == ("prefill", 0, 0, ids.numel(), True, 2)


def test_errors_before_any_device_work():
    m = _model(max_batch=4, max_seq=32)
    eng = m._engine
    with pytest.raises(ValueError, match="slots"):
        m.generate_requests([_req(0)], slots=5)               # more than max_batch
    with pytest.raises(ValueError, match="slots"):
        m.generate_requests([_req(0)], slots=0)
    with pytest.raises(ValueError, match="slots"):
        _model(max_batch=20).generate_requests([_req(0)], slots=17)   # more than 16
    with pytest.raises(ValueError, match="max_seq"):
        m.generate_requests([_req(0, max_new_tokens=4), _req(1, S=30, max_new_tokens=3)])
    with pytest.raises(NotImplementedError, match="greedily"):
        m.generate_requests([_req(0)], do_sample=True)
    with pytest.raises(ValueError, match="input_ids"):
        m.generate_requests([dict(input_ids=torch.zeros(2, 4, dtype=torch.int64))])
    bad_span = torch.tensor([100, 32001, 32000, 32000, 7, 7])
    with pytest.raises(ValueError, match="video"):
        m.generate_requests([dict(input_ids=bad_span, video_spatio_temporal_features=torch.zeros(eng.NV, 1024),
                                 max_new_tokens=4)])
    assert eng.calls == []


def test_no_turn_to_continue_afterwards():
    m = _model()
    m._last_out = torch.zeros(1, 4, dtype=torch.int64)      # as left by an earlier generate
    m.generate_requests([_req(0, max_new_tokens=2)])
    with pytest.raises(ValueError, match="no previous generate"):
        m.generate_continue(torch.tensor([[5, 6]]))
