"""Packed prefill into cache slots (vcl_llm_slots_prefill, Engine.slots_prefill) and the scheduler's packed admission
(generate_requests(packed_admission=True)).

Bar: bit identity with slot_prefill of each prompt alone -- first tokens and every layer's K / V cache. Each row of
a GEMM sums over K in the same order whatever rows sit next to it, and each (sequence, head, query tile) CTA of the
attention does the arithmetic of the same CTA of the single prefill, so nothing may differ. Every cache column a
call must not write keeps its bits (NaN sentinel or a live neighbour's sequence).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import make_engine, to_dev, vid_start_of  # noqa: E402
from test_padded_batch_gpu import video_feats  # noqa: E402

DEV = "cuda"
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)
WIDE = O.LlmCfg(hidden=2560, inter=6912, heads=20, layers=2)


def make_prompt(cfg, L, video, seed):
    """-> (ids [L] int64 on the host, video features [356, 1024] or None). A video prompt needs L >= 360."""
    if not video:
        g = torch.Generator().manual_seed(seed)
        return torch.cat([torch.tensor([1]), torch.randint(3, 32000, (L - 1,), generator=g)]), None
    n_post = min(26, L - 360)
    ids = O.make_prompt_ids(cfg, 356, seed=seed, n_pre=L - 359 - n_post, n_post=n_post)[0]
    assert ids.numel() == L
    return ids, video_feats(1, seed + 1)[0]


def vstart(cfg, ids, f):
    return int(vid_start_of(ids[None].to(DEV), cfg)[0]) if f is not None else vn.NO_VIDEO


def caches(eng, cfg):
    """every layer's (k, v) as int16 bit patterns"""
    out = []
    for l in range(cfg.layers):
        k, v = eng.kv_cache(l)
        out.append((k.view(torch.int16).clone(), v.view(torch.int16).clone()))
    return out


def fill_nan(eng, cfg):
    c = eng.cfg
    nan = torch.full((c.max_batch, c.llm_heads, c.max_seq, 128), float("nan"), dtype=torch.bfloat16, device=DEV)
    for l in range(cfg.layers):
        eng.set_kv_cache(l, nan, nan)


def singles(eng, cfg, slots, prompts):
    toks = []
    for s, (ids, f) in zip(slots, prompts):
        vs = torch.tensor([vstart(cfg, ids, f)], dtype=torch.int32, device=DEV)
        toks.append(eng.slot_prefill(s, ids.to(DEV)[None], f, vs))
    return torch.cat(toks)


def packed(eng, cfg, slots, prompts):
    return eng.slots_prefill(slots, [p[0] for p in prompts], [p[1] for p in prompts],
                             [vstart(cfg, ids, f) for ids, f in prompts])


@pytest.fixture(scope="module")
def small_state():
    return to_dev(O.random_llm_state(SMALL, seed=21))


# lengths straddle the attention's 64-query / 128-key tiles and the GEMM's 128-row tiles; "v" marks a video prompt
CASES = {
    1: ([3], ["448v"]),
    2: ([1, 0], [1, "512v"]),
    3: ([5, 0, 3], [31, "448v", 65]),
    9: ([8, 2, 6, 0, 15, 4, 11, 1, 7], [63, 64, "400v", 127, 128, 129, 200, "448v", 512]),
    16: ([9, 3, 14, 0, 7, 12, 1, 5, 15, 10, 2, 8, 13, 6, 11, 4],
         [1, 31, 63, 64, 65, 127, 128, 129, 200, "448v", 512, "512v", "400v", 448, 65, "448v"]),
}


def _prompts(cfg, lens, seed):
    return [make_prompt(cfg, int(str(L).rstrip("v")), str(L).endswith("v"), seed + 7 * j) for j, L in enumerate(lens)]


def _check_identity(eng, cfg, slots, prompts):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        fill_nan(eng, cfg)
        t_one = singles(eng, cfg, slots, prompts)
        c_one = caches(eng, cfg)
        fill_nan(eng, cfg)
        t_pack = packed(eng, cfg, slots, prompts)
        c_pack = caches(eng, cfg)
    st.synchronize()
    assert torch.equal(t_pack, t_one), (t_pack.tolist(), t_one.tolist())
    nan_bits = torch.tensor(float("nan"), dtype=torch.bfloat16).view(torch.int16).item()
    for l, ((k1, v1), (k2, v2)) in enumerate(zip(c_one, c_pack)):
        assert torch.equal(k1, k2) and torch.equal(v1, v2), l
        # outside columns 0 .. S_i-1 of the admitted slots: the sentinel
        written = torch.zeros(k2.shape[0], k2.shape[2], dtype=torch.bool, device=DEV)
        for s, (ids, _) in zip(slots, prompts):
            written[s, :ids.numel()] = True
        for x in (k2, v2):
            assert bool((x.permute(0, 2, 1, 3)[~written] == nan_bits).all()), l
            assert not bool((x.permute(0, 2, 1, 3)[written] == nan_bits).any()), l


@torch.no_grad()
@pytest.mark.parametrize("n", sorted(CASES))
def test_packed_equals_one_at_a_time(n, small_state):
    slots, lens = CASES[n]
    eng = make_engine(llm=SMALL, max_batch=16, max_seq=512)
    eng.load_llm(small_state)
    _check_identity(eng, SMALL, slots, _prompts(SMALL, lens, 100 + n))


@torch.no_grad()
def test_packed_equals_one_at_a_time_wide():
    eng = make_engine(llm=WIDE, max_batch=4, max_seq=512)
    eng.load_llm(to_dev(O.random_llm_state(WIDE, seed=5)))
    _check_identity(eng, WIDE, [2, 0, 3], _prompts(WIDE, [129, "448v", 63], 900))


@torch.no_grad()
def test_decode_continues_and_live_neighbours_keep_their_bits(small_state):
    """9 slots admitted packed and one at a time decode to the same tokens; a second wave into slots 7, 2, 4 with the
    others mid-sequence leaves the others' cache bits alone, and every slot keeps decoding identically."""
    NB = 9
    eng = make_engine(llm=SMALL, max_batch=NB, max_seq=512)
    eng.load_llm(small_state)
    lens = [65, "400v", 31, 128, 200, "448v", 1, 129, 64]
    first_wave = _prompts(SMALL, lens, 300)
    wave2_slots = [7, 2, 4]
    wave2 = _prompts(SMALL, [127, "448v", 90], 400)
    runs = {}
    st = torch.cuda.Stream()
    for mode in ("single", "packed"):
        admit = singles if mode == "single" else packed
        outs = []
        with torch.cuda.stream(st):
            fill_nan(eng, SMALL)                                # no columns left over from the other run
            first = admit(eng, SMALL, list(range(NB)), first_wave)
            pos = [p[0].numel() for p in first_wave]
            out = eng.slot_decode(first, pos, 7)
            outs.append(out.clone())
            first = out[:, -1].contiguous()
            pos = [p + 6 for p in pos]
            before = caches(eng, SMALL)
            t2 = admit(eng, SMALL, wave2_slots, wave2)
            after = caches(eng, SMALL)
            for j, s in enumerate(wave2_slots):
                first[s] = t2[j]
                pos[s] = wave2[j][0].numel()
            out = eng.slot_decode(first, pos, 9)
            outs.append(out.clone())
        st.synchronize()
        others = [s for s in range(NB) if s not in wave2_slots]
        for (k0, v0), (k1, v1) in zip(before, after):
            assert torch.equal(k0[others], k1[others]) and torch.equal(v0[others], v1[others]), mode
        runs[mode] = (outs, after)
    for a, b in zip(runs["single"][0], runs["packed"][0]):
        assert torch.equal(a, b), (a.tolist(), b.tolist())
    for (k0, v0), (k1, v1) in zip(runs["single"][1], runs["packed"][1]):
        assert torch.equal(k0, k1) and torch.equal(v0, v1)


@torch.no_grad()
def test_packed_admission_clears_padding(small_state):
    eng = make_engine(llm=SMALL, max_batch=3, max_seq=512)
    eng.load_llm(small_state)
    ref = make_engine(llm=SMALL, max_batch=3, max_seq=512)
    ref.load_llm(small_state)
    prompts = _prompts(SMALL, [40, 70, 20], 500)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        ids = torch.cat([torch.zeros(3, 4, dtype=torch.int64), prompts[0][0][None].expand(3, -1)], 1).to(DEV)
        eng.prefill(ids, None, torch.full((3,), vn.NO_VIDEO, dtype=torch.int32, device=DEV), n_pad=[4, 0, 2])
        first = packed(eng, SMALL, [0, 1, 2], prompts)
        out = eng.slot_decode(first, [p[0].numel() for p in prompts], 6)       # accepted: the cache is unpadded
        first_r = packed(ref, SMALL, [0, 1, 2], prompts)
        out_r = ref.slot_decode(first_r, [p[0].numel() for p in prompts], 6)
    st.synchronize()
    assert torch.equal(out, out_r)


@torch.no_grad()
def test_launches_do_not_grow_with_n(small_state):
    eng = make_engine(llm=SMALL, max_batch=16, max_seq=512)
    eng.load_llm(small_state)
    counts = {}
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for n in (1, 2, 3, 4, 5, 9, 16):
            prompts = _prompts(SMALL, ["448v", "400v"] * 8, 600)[:n]
            packed(eng, SMALL, list(range(n)), prompts)            # warm
            n0 = vn.launch_count()
            packed(eng, SMALL, list(range(n)), prompts)
            counts[n] = vn.launch_count() - n0
    st.synchronize()
    # the lm_head takes the 1..4-row decode kernel or the 5..16-row one (with its input re-laid out first)
    assert counts[1] == counts[2] == counts[3] == counts[4], counts
    assert counts[5] == counts[9] == counts[16], counts
    assert counts[16] - counts[1] <= 4, counts


@torch.no_grad()
def test_rejections_leave_the_cache_alone(small_state):
    eng = make_engine(llm=SMALL, max_batch=4, max_seq=300)
    eng.load_llm(small_state)
    wide = make_engine(llm=SMALL, max_batch=17, max_seq=8)
    wide.load_llm(small_state)
    big = make_engine(llm=SMALL, max_batch=2, max_seq=600)
    big.load_llm(small_state)
    fill_nan(eng, SMALL)
    torch.cuda.synchronize()
    snap = caches(eng, SMALL)
    p = _prompts(SMALL, [20, 30, 40, 50, 60], 700)
    n0 = vn.launch_count()
    with pytest.raises(vn.VclError, match="n=5 outside 1..4"):
        packed(eng, SMALL, [0, 1, 2, 3, 0], p)
    with pytest.raises(vn.VclError, match="n=0 outside"):
        eng.slots_prefill([], [], [], [])
    with pytest.raises(vn.VclError, match="n=17 outside 1..16"):
        packed(wide, SMALL, list(range(17)), _prompts(SMALL, [4] * 17, 750))
    with pytest.raises(vn.VclError, match="slot 4 outside"):
        packed(eng, SMALL, [0, 4], p[:2])
    with pytest.raises(vn.VclError, match="slot -1 outside"):
        packed(eng, SMALL, [-1, 0], p[:2])
    with pytest.raises(vn.VclError, match="slot 1 is given twice"):
        packed(eng, SMALL, [1, 0, 1], p[:3])
    with pytest.raises(vn.VclError, match="301 tokens, outside 1..300"):
        packed(eng, SMALL, [0, 1], [p[0], make_prompt(SMALL, 301, False, 1)])
    with pytest.raises(vn.VclError, match="0 tokens, outside"):
        packed(eng, SMALL, [0, 1], [p[0], (torch.zeros(0, dtype=torch.int64), None)])
    with pytest.raises(vn.VclError, match="513 tokens, outside 1..512"):
        packed(big, SMALL, [0], [make_prompt(SMALL, 513, False, 2)])
    assert vn.launch_count() == n0
    torch.cuda.synchronize()
    for (k0, v0), (k1, v1) in zip(snap, caches(eng, SMALL)):
        assert torch.equal(k0, k1) and torch.equal(v0, v1)


# ------------------------------------------------------------------------------------------
def _model(cfg, max_batch, max_seq=600):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    c = VideoChatGPTConfig(hidden_size=cfg.hidden, intermediate_size=cfg.inter, num_hidden_layers=cfg.layers,
                           num_attention_heads=cfg.heads, vocab_size=cfg.vocab, use_mm_proj=True, mm_hidden_size=1024)
    clip = dict(hidden_size=1024, intermediate_size=1024, num_hidden_layers=3, num_attention_heads=16)
    m = VideoChatGPTLlamaForCausalLM(c, clip_config=clip, max_batch=max_batch, max_seq=max_seq)
    vc = m.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = 32000, 32001, 32002, True
    return m


class _Tok:
    """Tokenizer stand-in for KeywordsStoppingCriteria: keyword "t<id>." is the single token <id>"""

    def __call__(self, text):
        from types import SimpleNamespace
        return SimpleNamespace(input_ids=[int(text[1:-1])])

    def batch_decode(self, ids, skip_special_tokens=True):
        return ["".join(f"t{int(i)}." for i in row) for row in ids]


@torch.no_grad()
@pytest.mark.parametrize("n_slots,n_req", [(4, 11), (9, 20)])
def test_scheduler_packed_equals_one_at_a_time(n_slots, n_req, small_state):
    from video_chatgpt.model.utils import KeywordsStoppingCriteria
    m = _model(SMALL, max_batch=n_slots)
    m.load_state_dict(dict(small_state))
    lens = [1 + (11 * r) % 40 for r in range(n_req)]
    reqs = []
    for r, n in enumerate(lens):
        L = [40, "448v", 129, "400v", 65, 200][r % 6]
        if r == 3:
            L = 540                                             # over the packed limit: admitted alone
        ids, f = make_prompt(SMALL, int(str(L).rstrip("v")), str(L).endswith("v"), 1000 + r)
        req = dict(input_ids=ids[None], max_new_tokens=n)
        if f is not None:
            req["video_spatio_temporal_features"] = f.half()
        reqs.append(req)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        free = [o[0, -n:].tolist() for o, n in zip(m.generate_requests(reqs, eos_token_id=None), lens)]
    st.synchronize()
    # EOS: a token request 1 produces; a keyword criterion on request 0 at a token of its own
    eos = free[1][min(5, len(free[1]) - 1)]
    kw = free[0][len(free[0]) // 2]
    out = {}
    for flag in (False, True):
        rq = [dict(r) for r in reqs]
        rq[0]["stopping_criteria"] = [KeywordsStoppingCriteria([f"t{kw}."], _Tok(), reqs[0]["input_ids"])]
        with torch.cuda.stream(st):
            out[flag] = [o.tolist() for o in m.generate_requests(rq, eos_token_id=eos, packed_admission=flag)]
        st.synchronize()
    assert out[True] == out[False]
    # the rules did fire: request 1 ends at its first EOS, request 0 at its keyword at the latest
    assert len(out[True][1][0]) == len(reqs[1]["input_ids"][0]) + free[1].index(eos) + 1
    assert len(out[True][0][0]) <= len(reqs[0]["input_ids"][0]) + free[0].index(kw) + 1
