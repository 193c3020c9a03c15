"""CPU tests of beam search: the host's fp32 replay of _beam_search's steps 4-6 against the installed transformers
helpers on random records, generate(num_beams=k) end to end through the real host loop against HF's own beam search
on a tiny LlamaForCausalLM (a fake engine does the device's selection the way HF does and forks its cache), chunk
lengths, the rejections, and the new C-ABI symbols."""
import os
import sys

import pytest
import torch

import _beam_ref as BR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _records(B, k, n, V, eos, seed):
    """n steps of random records: K candidates per item with descending scores, EOS among them now and then, and
    picks taken as HF takes them (top k of score + hit * -1e9)"""
    g = torch.Generator().manual_seed(seed)
    K = 2 * k
    steps = []
    base = torch.zeros(B)
    for t in range(n):
        drop = torch.rand(B, K, generator=g) * 2.0
        score = (base[:, None] - drop.cumsum(dim=1)).to(torch.float32)
        beam = torch.randint(0, k, (B, K), generator=g)
        tok = torch.randint(0, V, (B, K), generator=g)
        if eos is not None:
            tok[torch.rand(B, K, generator=g) < 0.25] = eos
        hit = torch.full((B, K), t + 1 >= n)
        if eos is not None:
            hit = hit | (tok == eos)
        pick = torch.topk(score + hit.to(torch.float32) * -1.0e9, k)[1]
        steps.append((score, beam, tok, pick))
        base = score[:, 0].double() * 0.5
    return steps


@pytest.mark.parametrize("length_penalty", [-1.0, 0.0, 1.0, 2.0])
@pytest.mark.parametrize("early_stopping", [True, False, "never"])
@pytest.mark.parametrize("eos", [None, 7])
def test_replay_matches_transformers(length_penalty, early_stopping, eos):
    from video_chatgpt.model.video_chatgpt import _BeamReplay
    B, k, S, n, V = 3, 4, 5, 9, 50
    fill = eos if eos is not None else -1
    for seed in range(4):
        steps = _records(B, k, n, V, eos, seed * 31 + int(length_penalty * 7) + len(str(early_stopping)))
        stop, seqs, scores, idx, fin = BR.hf_replay(steps, B, k, S, n, eos, fill, length_penalty, early_stopping)
        r = _BeamReplay(B, k, S, n, eos, eos, length_penalty, early_stopping)
        mine = None
        for t, st in enumerate(steps):
            if r.step(*st):
                mine = t
                break
        assert mine == stop and stop is not None
        assert torch.equal(r.fin_score.view(torch.int32), scores.view(torch.int32)), (r.fin_score, scores)
        assert torch.equal(r.is_fin, fin)
        assert torch.equal(r.fin_seq, seqs[:, :, S:])
        assert torch.equal(r.fin_len, (idx >= 0).sum(dim=2))
        for m in (1, k):
            out, sc = r.result(m)
            L = int((idx[:, :m] >= 0).sum(dim=2).max())
            assert torch.equal(out, seqs[:, :m, S:S + L].reshape(B * m, L))
            assert torch.equal(sc, scores[:, :m].reshape(-1))


def test_select_tie_rule_and_hits():
    x = torch.full((4, 40), -5.0)
    x[0, 3] = x[0, 9] = 2.0              # a tie inside a row: the lower token first
    x[1, 3] = x[1, 20] = 2.0             # ... and across rows at equal scores: the lower beam first
    out = BR.select(x, [0.0, 0.0, 0.0, -1e9], 2, eos=9)
    (top, picks, hits, _), (top2, picks2, _, _) = out
    assert [(c[1], c[2]) for c in top[:3]] == [(0, 3), (0, 9), (1, 3)]
    assert hits[:3] == [False, True, False] and picks == [0, 2]
    assert all(c[1] == 0 for c in top2)   # beam 1 of item 1 is 1e9 behind
    _, _, hits, _ = BR.select(x, [0.0] * 4, 2, last_step=True)[0]
    assert all(hits)


# ------------------------------------------------------------------------------------------
V, HID = 96, 64


def _tiny_llama():
    from transformers import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    cfg = LlamaConfig(vocab_size=V, hidden_size=HID, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4, max_position_embeddings=256, bos_token_id=None, eos_token_id=None,
                      pad_token_id=None, initializer_range=0.2, attn_implementation="eager")
    model = LlamaForCausalLM(cfg).eval()
    model.generation_config.eos_token_id = None
    model.generation_config.pad_token_id = None
    model.generation_config.bos_token_id = None
    return model


class HFBeamEngine:
    """Stands in for vcl_native.Engine's beam entry points: runs the tiny LLaMA as HF's _beam_search does (k copies of
    each prompt, position ids from the mask, fp32 log_softmax + running scores, torch.topk for the K candidates and
    the running picks) and reorders its cache by the picks, the fake's fork. Records every call."""

    NV = 356

    def __init__(self, model):
        self.model = model
        self.calls = []

    def _select(self):
        lg = self.out.logits[:, -1, :].to(torch.float32)
        B, k = self.B, self.k
        acc = torch.log_softmax(lg, dim=-1).view(B, k, V) + self.scores[:, :, None]
        top, idx = torch.topk(acc.reshape(B, k * V), 2 * k)
        beam, tok = idx // V, idx % V
        hit = torch.full_like(tok, self.t + 1 >= self.n, dtype=torch.bool)
        if self.eos >= 0:
            hit = hit | (tok == self.eos)
        masked = top + hit.to(torch.float32) * -1.0e9
        pick = torch.topk(masked, k)[1]
        self.scores = torch.take_along_dim(masked, pick, dim=1)
        self.next = torch.take_along_dim(tok, pick, dim=1).reshape(-1, 1)
        parent = torch.take_along_dim(beam, pick, dim=1) + torch.arange(B)[:, None] * k
        self.out.past_key_values.reorder_cache(parent.reshape(-1))
        self.t += 1
        rec = torch.stack([top.view(torch.int32), beam.to(torch.int32), tok.to(torch.int32)], dim=-1)
        return rec[None], pick[None].to(torch.int32)

    @torch.no_grad()
    def beam_start(self, ids, video_feats, vid_start, num_beams, n_new, eos=-1, n_pad=None):
        self.calls.append(("start", tuple(ids.shape), num_beams, n_new, eos, n_pad))
        B, S = ids.shape
        self.B, self.k, self.n, self.eos, self.t = B, num_beams, n_new, eos, 0
        mask = torch.ones(B, S, dtype=torch.int64)
        for b, p in enumerate(n_pad or []):
            mask[b, :p] = 0
        self.mask = mask.repeat_interleave(num_beams, dim=0)
        pos = (self.mask.cumsum(-1) - 1).masked_fill(self.mask == 0, 0)
        self.pos = pos[:, -1:]
        self.out = self.model(input_ids=ids.repeat_interleave(num_beams, dim=0), attention_mask=self.mask,
                              position_ids=pos, use_cache=True)
        self.scores = torch.zeros(B, num_beams)
        self.scores[:, 1:] = -1e9
        return self._select()

    @torch.no_grad()
    def beam_decode(self, n_steps):
        self.calls.append(("decode", n_steps))
        assert self.t + n_steps <= self.n
        recs, picks = [], []
        for _ in range(n_steps):
            self.mask = torch.cat([self.mask, torch.ones(self.mask.shape[0], 1, dtype=torch.int64)], dim=1)
            self.pos = self.pos + 1
            self.out = self.model(input_ids=self.next, attention_mask=self.mask, position_ids=self.pos,
                                  past_key_values=self.out.past_key_values, use_cache=True)
            r, p = self._select()
            recs.append(r)
            picks.append(p)
        return torch.cat(recs), torch.cat(picks)


def _model(eng, eos, max_batch=32):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    cfg = VideoChatGPTConfig(hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4,
                             vocab_size=V, eos_token_id=eos)
    m = VideoChatGPTLlamaForCausalLM(cfg, clip_config={}, max_batch=max_batch, max_seq=128)
    vc = m.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = V + 1, V + 2, V + 3, True
    m.device = torch.device("cpu")
    m._engine, m._llm_loaded = eng, True
    return m


def _prompts(B, padded):
    g = torch.Generator().manual_seed(B * 7 + padded)
    S = 7
    ids = torch.randint(0, V, (B, S), generator=g)
    mask = torch.ones(B, S, dtype=torch.int64)
    if padded:
        for b in range(B):
            p = (2 * b + 1) % 4
            mask[b, :p] = 0
            ids[b, :p] = 0
    return ids, mask


_EOS = {}


def _eos_token(model):
    """a token the beams actually produce: the most frequent one of a short beam search without EOS"""
    if "eos" not in _EOS:
        ids, mask = _prompts(3, False)
        out = model.generate(ids, attention_mask=mask, num_beams=4, max_new_tokens=12, do_sample=False)
        _EOS["eos"] = int(torch.mode(out[:, 7:].reshape(-1)).values)
    return _EOS["eos"]


@pytest.mark.parametrize("B,padded", [(1, False), (3, False), (3, True)])
@pytest.mark.parametrize("k,m", [(2, 1), (4, 2), (8, 8)])
@pytest.mark.parametrize("use_eos", [False, True])
def test_generate_equals_hf_beam_search(B, padded, k, m, use_eos):
    model = _tiny_llama()
    eos = _eos_token(model) if use_eos else None
    ids, mask = _prompts(B, padded)
    n = 14
    for lp, es in ((1.0, False), (2.0, True), (-1.0, "never")):
        ref = model.generate(ids, attention_mask=mask, num_beams=k, num_return_sequences=m, max_new_tokens=n,
                             do_sample=False, eos_token_id=eos, pad_token_id=eos, length_penalty=lp,
                             early_stopping=es, return_dict_in_generate=True, output_scores=True)
        eng = HFBeamEngine(model)
        mine = _model(eng, eos)
        out = mine.generate(ids, attention_mask=mask if padded else None, num_beams=k, num_return_sequences=m,
                            max_new_tokens=n, eos_token_id=eos if use_eos else None, length_penalty=lp,
                            early_stopping=es)
        assert torch.equal(out, ref.sequences), (lp, es, out, ref.sequences)
        assert torch.equal(mine.last_beam_scores, ref.sequences_scores), (mine.last_beam_scores, ref.sequences_scores)
        assert eng.calls[0][0] == "start" and eng.calls[0][4] == (eos if use_eos else -1)
        assert eng.calls[0][5] == (None if not padded else [int((mask[b] == 0).sum()) for b in range(B)])


@pytest.mark.parametrize("use_eos", [False, True])
def test_chunk_lengths_give_identical_outputs(use_eos):
    model = _tiny_llama()
    eos = _eos_token(model) if use_eos else None
    ids, mask = _prompts(3, True)
    outs = []
    for chunk in (1, 3, 8, 32):
        eng = HFBeamEngine(model)
        m = _model(eng, eos)
        m._BEAM_CHUNK = chunk
        out = m.generate(ids, attention_mask=mask, num_beams=4, num_return_sequences=2, max_new_tokens=20,
                         eos_token_id=eos)
        outs.append((out, m.last_beam_scores))
        assert all(c[1] <= chunk for c in eng.calls[1:])
    for o, s in outs[1:]:
        assert torch.equal(o, outs[0][0]) and torch.equal(s, outs[0][1])


class NoDevice:
    NV = 356

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        return lambda *a, **k: self.calls.append(name)


@pytest.mark.parametrize("kw,exc,match", [
    (dict(num_beams=2, num_return_sequences=3), ValueError, "num_return_sequences"),
    (dict(num_beams=2, num_return_sequences=0), ValueError, "num_return_sequences"),
    (dict(num_beams=2, max_new_tokens=126), ValueError, "max_seq"),
    (dict(num_beams=9), ValueError, "num_beams"),
    (dict(num_beams=0), ValueError, "num_beams"),
    (dict(num_beams=2.0), ValueError, "num_beams"),
    (dict(num_beams=2, early_stopping="always"), ValueError, "early_stopping"),
    (dict(num_beams=2, do_sample=True), NotImplementedError, "do_sample"),
    (dict(num_beams=2, seed=3), NotImplementedError, "seed"),
    (dict(num_beams=2, logprobs=1), NotImplementedError, "logprobs"),
    (dict(num_beams=2, top_p=0.9), NotImplementedError, "top_p"),
    (dict(num_beams=2, repetition_penalty=1.2), NotImplementedError, "repetition_penalty"),
    (dict(num_beams=2, stopping_criteria=[lambda ids, s: False]), NotImplementedError, "stopping_criteria"),
    (dict(num_beams=8), ValueError, "max_batch"),
])
def test_rejections_before_any_device_work(kw, exc, match):
    eng = NoDevice()
    m = _model(eng, None, max_batch=4)
    with pytest.raises(exc, match=match):
        m.generate(torch.tensor([[1, 5, 6]]), **kw)
    assert eng.calls == []


def test_paged_model_rejects_beams():
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    cfg = VideoChatGPTConfig(hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4,
                             vocab_size=V)
    m = VideoChatGPTLlamaForCausalLM(cfg, clip_config={}, max_batch=4, max_seq=640, kv_blocks=8)
    m._engine, m._llm_loaded = NoDevice(), True
    with pytest.raises(NotImplementedError, match="paged"):
        m.generate(torch.tensor([[1, 5, 6]]), num_beams=2)
    assert m._engine.calls == []


class _Reached(Exception):
    pass


@pytest.mark.parametrize("kw", [dict(), dict(num_beams=1), dict(num_beams=1, num_return_sequences=1),
                                dict(do_sample=True, num_return_sequences=3), dict(num_return_sequences=2),
                                dict(num_return_sequences=0)])
def test_calls_without_beams_never_touch_the_beam_path(kw):
    """num_return_sequences without beams keeps its old treatment (ignored); the scores of an earlier beam call do not
    outlive the next call"""
    m = _model(NoDevice(), None)
    m.last_beam_scores, m._after_beams = torch.ones(2), True

    def beam(*a, **k):
        raise AssertionError("the beam path was taken")

    def engine(*a, **k):
        raise _Reached()

    m._beam_generate, m._ensure_engine = beam, engine
    with pytest.raises(_Reached):
        m.generate(torch.tensor([[1, 5, 6]]), **kw)
    assert m.last_beam_scores is None and not m._after_beams


def test_generate_continue_after_beams_raises():
    model = _tiny_llama()
    m = _model(HFBeamEngine(model), None)
    ids, _ = _prompts(1, False)
    m.generate(ids, num_beams=2, max_new_tokens=4)
    with pytest.raises(ValueError, match="beam search"):
        m.generate_continue(torch.tensor([[3, 4]]))


def test_c_abi_symbols():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as G
    import vcl_native as vn
    new = {"vcl_llm_beam_start", "vcl_llm_beam_decode", "vcl_op_beam_select"}
    assert new <= set(G.declared_symbols())
    assert new <= set(vn.EXPORTED_SYMBOLS)
    hdr = open(os.path.join(ROOT, "include", "vcl.h")).read()
    assert "#define VCL_BEAM_MAX 8" in hdr and vn.BEAM_MAX == 8
    rec = torch.tensor([[[0x3f800000, 2, 17]]], dtype=torch.int32)
    s, b, t = vn.beam_records(rec)
    assert s.item() == 1.0 and b.item() == 2 and t.item() == 17
