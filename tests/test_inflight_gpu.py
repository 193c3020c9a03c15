"""In-flight batching on the GPU: cache slots at their own positions (vcl_llm_slot_prefill / vcl_llm_slot_decode)
and the scheduler on top of them (generate_requests). Slot counts 3 and 9 cover both decode ring kernels
(gemv_tc for 1..4 clips, gemv_tcw for 5..16).

Bars: the slot decode is bit-identical to the shared-position loop on the same cache; a request's tokens do not
depend on its neighbours or on when it was admitted (every clip is its own MMA column and its own attention
cluster, so any difference is a cross-slot read or write); against the request run alone and the bf16 oracle the
margin rule of test_padded_batch_gpu.py holds (identical up to the oracle's first top-1/top-2 margin under 3 ulps).
"""
import time
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import make_engine, to_dev, vid_start_of  # noqa: E402
from test_padded_batch_gpu import first_near_tie, video_feats  # noqa: E402

DEV = "cuda"
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)


def prompt(cfg, seed, n_pre):
    return O.make_prompt_ids(cfg, 356, seed=seed, n_pre=n_pre)[0]


def text_prompt(seed, n):
    return torch.cat([torch.tensor([1]), torch.randint(3, 32000, (n - 1,), generator=torch.Generator().manual_seed(seed))])


def admit(eng, slot, ids, vf):
    """slot_prefill of one prompt (host ids [S]); returns its first token [1] int32 on the device"""
    ids = ids.to(DEV)[None]
    return eng.slot_prefill(slot, ids, vf, vid_start_of(ids, SMALL))


@pytest.fixture(scope="module")
def small_state():
    return to_dev(O.random_llm_state(SMALL, seed=21))


# ------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("NB", [3, 9])
def test_slot_decode_matches_the_shared_position_loop(NB, small_state):
    ids = O.make_prompt_ids(SMALL, 356, seed=30, batch=NB).to(DEV)
    S, k = ids.shape[1], 12
    vf = video_feats(NB, 31)
    eng = make_engine(llm=SMALL, max_batch=NB, max_seq=480)
    eng.load_llm(small_state)
    vs = vid_start_of(ids, SMALL)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        _, _, first = eng.prefill(ids, vf, vs)
        shared = eng.decode_loop(first, S, k)
        eng.prefill(ids, vf, vs)
        slots = eng.slot_decode(first, [S] * NB, k)
    st.synchronize()
    # the default stream cannot be captured: the same steps run eagerly
    eng.prefill(ids, vf, vs)
    eager = eng.slot_decode(first, [S] * NB, k)
    torch.cuda.synchronize()
    assert torch.equal(slots, shared), (slots.tolist(), shared.tolist())
    assert torch.equal(eager, shared)


@torch.no_grad()
def test_short_prompts_decode(small_state):
    """Text prompts of 31 and 201 tokens leave the last attention CTA of a head 15 and 9 keys (an odd count below
    16): the shared-position loop, the slot decode and single steps must agree there."""
    eng = make_engine(llm=SMALL, max_batch=2, max_seq=480)
    eng.load_llm(small_state)
    k = 6
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for S in (31, 201):
            ids = text_prompt(500 + S, S).to(DEV)[None]
            vs = vid_start_of(ids, SMALL)
            _, _, tok = eng.prefill(ids, None, vs)
            loop = eng.decode_loop(tok, S, k)
            steps = [tok]
            for i in range(1, k):
                steps.append(eng.decode_step(steps[-1], S + i - 1)[1])
            first = torch.cat([admit(eng, b, ids[0].cpu(), None) for b in range(2)])
            slots = eng.slot_decode(first, [S, S], k)
            st.synchronize()
            assert torch.equal(loop[0], torch.cat(steps)), S
            assert torch.equal(slots[0], loop[0]) and torch.equal(slots[1], loop[0]), S


@torch.no_grad()
@pytest.mark.parametrize("NB", [3, 9])
def test_slot_isolation(NB, small_state):
    """Request X in slot s: admitted at step 0 next to requests A, or admitted after request Y retired from slot s
    next to requests B of other lengths and positions -- bit-identical tokens."""
    s, k = NB // 2, 10
    eng = make_engine(llm=SMALL, max_batch=NB, max_seq=480)
    eng.load_llm(small_state)
    x = prompt(SMALL, 50, 40)
    vx = video_feats(1, 51)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        # run 1: everyone admitted at step 0
        first = torch.empty(NB, dtype=torch.int32, device=DEV)
        pos = []
        for b in range(NB):
            ids = x if b == s else prompt(SMALL, 60 + b, 20 + 3 * b)
            first[b:b + 1] = admit(eng, b, ids, vx if b == s else video_feats(1, 70 + b))
            pos.append(len(ids))
        run1 = eng.slot_decode(first, pos, k)[s].clone()
        # run 2: other neighbours (some text only) that have decoded a while, and request Y in slot s first
        first = torch.empty(NB, dtype=torch.int32, device=DEV)
        pos = []
        for b in range(NB):
            ids = prompt(SMALL, 80 + b, 10 + 5 * b) if b % 2 else text_prompt(90 + b, 30 + 7 * b)
            first[b:b + 1] = admit(eng, b, ids, video_feats(1, 100 + b) if b % 2 else None)
            pos.append(len(ids))
        for _ in range(2):
            out = eng.slot_decode(first, pos, 6)
            first = out[:, -1].contiguous()
            pos = [p + 5 for p in pos]
        first[s:s + 1] = admit(eng, s, x, vx)
        pos[s] = len(x)
        run2 = eng.slot_decode(first, pos, k)[s].clone()
    st.synchronize()
    assert torch.equal(run1, run2), (run1.tolist(), run2.tolist())


# ------------------------------------------------------------------------------------------
def _model(llm_cfg, max_batch):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    cfg = VideoChatGPTConfig(hidden_size=llm_cfg.hidden, intermediate_size=llm_cfg.inter,
                             num_hidden_layers=llm_cfg.layers, num_attention_heads=llm_cfg.heads,
                             vocab_size=llm_cfg.vocab, use_mm_proj=True, mm_hidden_size=1024)
    clip = dict(hidden_size=1024, intermediate_size=1024, num_hidden_layers=3, num_attention_heads=16)
    m = VideoChatGPTLlamaForCausalLM(cfg, clip_config=clip, max_batch=max_batch, max_seq=480)
    vc = m.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = 32000, 32001, 32002, True
    return m


def _requests(cfg, lens, text_only=()):
    reqs = []
    for i, n in enumerate(lens):
        if i in text_only:
            reqs.append(dict(input_ids=text_prompt(200 + i, 50 + i), max_new_tokens=n))
        else:
            reqs.append(dict(input_ids=prompt(cfg, 200 + i, 20 + 4 * i)[None],
                             video_spatio_temporal_features=video_feats(1, 300 + i)[0].half(), max_new_tokens=n))
    return reqs


@torch.no_grad()
def test_requests_match_each_request_alone_and_the_oracle():
    """Width 2560, 11 requests over 4 slots (slots are refilled), one text-only request: each request's tokens
    equal its own one-request generate and the bf16 oracle's up to the oracle's first near-tie."""
    cfg = O.LlmCfg(hidden=2560, inter=6912, heads=20, layers=2)
    lsd = O.random_llm_state(cfg, seed=5)
    m = _model(cfg, max_batch=4)
    m.load_state_dict(lsd)
    lens = [5, 9, 3, 12, 7, 4, 10, 6, 8, 2, 11]
    reqs = _requests(cfg, lens, text_only=(5,))
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        outs = m.generate_requests(reqs, eos_token_id=None)
    st.synchronize()
    sd_b = to_dev(lsd)
    for i, (r, n) in enumerate(zip(reqs, lens)):
        ids = torch.as_tensor(r["input_ids"]).reshape(1, -1).to(DEV)
        S = ids.shape[1]
        f = r.get("video_spatio_temporal_features")
        f = None if f is None else f[None]
        assert outs[i].shape == (1, S + n) and torch.equal(outs[i][:, :S], ids)
        own = m.generate(ids, video_spatio_temporal_features=f, max_new_tokens=n, eos_token_id=None)
        o_toks, o_logits = O.greedy_generate(sd_b, cfg, ids, None if f is None else f.to(DEV).bfloat16(), n)
        t = first_near_tie(o_logits)[0]
        new = outs[i][0, S:]
        assert torch.equal(new[:t], own[0, S:S + t]), (i, t, new.tolist(), own[0, S:].tolist())
        assert torch.equal(new[:t].cpu(), o_toks[0, :t].cpu()), (i, t, new.tolist(), o_toks[0].tolist())


class _Tok:
    """Tokenizer stand-in for KeywordsStoppingCriteria: keyword "t<id>." is the single token <id>"""

    def __call__(self, text):
        return SimpleNamespace(input_ids=[int(text[1:-1])])

    def batch_decode(self, ids, skip_special_tokens=True):
        return ["".join(f"t{int(i)}." for i in row) for row in ids]


@torch.no_grad()
def test_stopping_rules(small_state):
    """EOS, per-request max_new_tokens and a KeywordsStoppingCriteria per request end only their own request."""
    from video_chatgpt.model.utils import KeywordsStoppingCriteria
    m = _model(SMALL, max_batch=3)
    m.load_state_dict({k: v for k, v in small_state.items()})
    lens = [14, 6, 11, 9, 13]
    reqs = _requests(SMALL, lens, text_only=(3,))
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        free = [o[0, -n:].tolist() for o, n in zip(m.generate_requests(reqs, eos_token_id=None), lens)]
    st.synchronize()
    for o, n in zip(free, lens):
        assert len(o) == n

    def first_new(stream):
        """a step j >= 1 whose token does not occur before it"""
        return next(j for j in range(1, len(stream)) if stream[j] not in stream[:j])

    # EOS: the token request 2 produces at step j
    j = first_new(free[2])
    eos = free[2][j]
    with torch.cuda.stream(st):
        outs = m.generate_requests(reqs, eos_token_id=eos)
    st.synchronize()
    for i, (o, n) in enumerate(zip(outs, lens)):
        want = free[i][:free[i].index(eos) + 1] if eos in free[i] else free[i]
        assert o[0, -len(want):].tolist() == want and o.shape[1] == reqs_len(reqs[i]) + len(want), i
    assert outs[2].shape[1] == reqs_len(reqs[2]) + j + 1
    # a keyword criterion on request 0 (stateful, one per prompt as the reference builds it)
    j0 = first_new(free[0])
    crit = KeywordsStoppingCriteria([f"t{free[0][j0]}."], _Tok(), torch.as_tensor(reqs[0]["input_ids"]).reshape(1, -1))
    kreqs = [dict(r) for r in reqs]
    kreqs[0]["stopping_criteria"] = [crit]
    kreqs[4]["max_new_tokens"] = 4
    with torch.cuda.stream(st):
        outs = m.generate_requests(kreqs, eos_token_id=None)
    st.synchronize()
    assert outs[0][0, reqs_len(reqs[0]):].tolist() == free[0][:j0 + 1]
    assert outs[4][0, reqs_len(reqs[4]):].tolist() == free[4][:4]
    for i in (1, 2, 3):
        assert outs[i][0, reqs_len(reqs[i]):].tolist() == free[i], i
    # no turn to continue
    with pytest.raises(ValueError, match="no previous generate"):
        m.generate_continue(torch.tensor([[5, 6]]))


def reqs_len(r):
    return torch.as_tensor(r["input_ids"]).numel()


@torch.no_grad()
def test_errors_before_any_device_work(small_state):
    eng = make_engine(llm=SMALL, max_batch=3, max_seq=64)
    eng.load_llm(small_state)
    wide = make_engine(llm=SMALL, max_batch=17, max_seq=32)
    wide.load_llm(small_state)
    ids = text_prompt(7, 20).to(DEV)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        first = torch.cat([admit(eng, b, ids.cpu(), None) for b in range(3)])
        st.synchronize()
        n0 = vn.launch_count()
        with pytest.raises(vn.VclError, match="n_slots=4 outside 1..3"):
            eng.slot_decode(torch.zeros(4, dtype=torch.int32, device=DEV), [20] * 4, 4)   # more than max_batch
        with pytest.raises(vn.VclError, match="n_slots=17 outside 1..16"):
            wide.slot_decode(torch.zeros(17, dtype=torch.int32, device=DEV), [1] * 17, 2)  # more than 16
        with pytest.raises(vn.VclError, match="slot 3 outside"):
            admit(eng, 3, ids.cpu(), None)
        with pytest.raises(vn.VclError, match="exceeds max_seq"):
            eng.slot_decode(first, [20, 60, 20], 6)                                     # 60 + 5 > 64
        assert vn.launch_count() == n0
        # a padded cache is rejected until the slots are started again
        pad_ids = torch.cat([torch.zeros(3, 4, dtype=torch.int64, device=DEV), ids[None].expand(3, -1)], 1)
        vs = torch.full((3,), vn.NO_VIDEO, dtype=torch.int32, device=DEV)
        eng.prefill(pad_ids, None, vs, n_pad=[4, 0, 2])
        st.synchronize()
        n0 = vn.launch_count()
        with pytest.raises(vn.VclError, match="left-padded"):
            eng.slot_decode(first, [20] * 3, 4)
        assert vn.launch_count() == n0
        first = torch.cat([admit(eng, b, ids.cpu(), None) for b in range(3)])
        out = eng.slot_decode(first, [20] * 3, 4)
    st.synchronize()
    assert torch.equal(out[0], out[1]) and torch.equal(out[0], out[2])
    m = _model(SMALL, max_batch=2)
    m.load_state_dict(dict(small_state))
    with pytest.raises(NotImplementedError, match="greedily"):
        m.generate_requests([ids], do_sample=True)


@torch.no_grad()
def test_graph_is_reused_for_other_positions(small_state):
    """A second slot_decode with other positions, and then a decode_loop with the same (B, n_new), replay the graph
    the first call captured: the launch count grows by the same node count, each call is a replay (no capture or
    instantiation on the host), and its tokens are those of a fresh engine doing the same call."""
    NB, k = 3, 8
    eng = make_engine(llm=SMALL, max_batch=NB, max_seq=480)
    eng.load_llm(small_state)
    fresh = make_engine(llm=SMALL, max_batch=NB, max_seq=480)
    fresh.load_llm(small_state)
    rows = [text_prompt(400 + b, 30 + 11 * b) for b in range(NB)]
    S = len(rows[0]) - 9        # the shared position: every slot's columns below it hold its prompt in both engines
    st = torch.cuda.Stream()
    deltas, host_ms, outs = [], [], []
    with torch.cuda.stream(st):
        first = torch.cat([admit(eng, b, r, None) for b, r in enumerate(rows)])
        first_f = torch.cat([admit(fresh, b, r, None) for b, r in enumerate(rows)])
        st.synchronize()
        for call in (lambda: eng.slot_decode(first, [len(r) for r in rows], k),
                     lambda: eng.slot_decode(first, [len(r) - 9 for r in rows], k),
                     lambda: eng.decode_loop(first, S, k)):
            n0 = vn.launch_count()
            ev = torch.cuda.Event()
            t0 = time.perf_counter()
            outs.append(call())
            host_ms.append((time.perf_counter() - t0) * 1e3)
            ev.record(st)
            ev.synchronize()
            deltas.append(vn.launch_count() - n0)
        # the second call fed each slot at len - 9: a fresh engine whose slots hold the same prompts does the same
        ref = fresh.slot_decode(first_f, [len(r) - 9 for r in rows], k)
        ref_loop = fresh.decode_loop(first_f, S, k)
    st.synchronize()
    # decode_loop launches one kernel of its own before the graph: the fill of the shared position
    assert deltas[0] == deltas[1] == deltas[2] - 1 > (k - 1) * SMALL.layers, deltas
    assert host_ms[1] < 0.5 * host_ms[0] and host_ms[2] < 0.5 * host_ms[0], host_ms
    assert torch.equal(outs[1], ref)
    assert torch.equal(outs[2], ref_loop)
