"""The fp8 (E4M3) LLM weight format on the GPU. Everything is bit for bit:

- the load-time quantizer (vcl_op_quantize_fp8) equals the torch reference of tests/_fp8_ref.py: codes in the slot
  order, row scales, W~; the matrices include rows holding every finite code;
- the fp8 ring kernels (vcl_op_gemv_fp8) equal the bf16 ones (vcl_op_gemv) on W~ for every B in 1..16, with and
  without norm and residual, at the model's K and a ragged N;
- an engine loaded with W in fp8 equals a bf16 engine loaded with W~: prefill logits, token and every layer's KV
  cache, decode steps, generate at 1 / 3 / 5 / 9 / 16 / 17 clips (partial arg-max hand-off, both ring kernels, the
  GEMM path) and left-padded, generate_continue, seeded sampling, packed in-flight batching and vcl_llm_score;
  7B width with two layers and one 13B-width case;
- the decode graphs have as many kernel nodes in both formats, the fp8 engine holds at least 95 % of the computed
  saving less memory, and a non-finite weight fails the load with its name."""
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
import _fp8_ref as R  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import make_engine, to_dev, vid_start_of  # noqa: E402
from test_padded_batch_gpu import padded_batch, video_feats  # noqa: E402

DEV = "cuda"
W7B = O.LlmCfg(hidden=4096, inter=11008, heads=32, layers=2)
W13B = O.LlmCfg(hidden=5120, inter=13824, heads=40, layers=1)
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)


def _weights(N, K, seed):
    """rows of different magnitudes (row scales 2^-16 .. 2^2), a zero row, rows holding every finite code"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = torch.randn(N, K, device=DEV, generator=g) * torch.exp2(torch.randint(-16, 3, (N, 1), device=DEV, generator=g).float())
    codes = R.finite_codes().to(DEV)                            # K >= 254 below: each such row holds them all
    for i, r in enumerate(range(1, min(N, 40), 7)):
        row = codes[torch.randint(0, codes.numel(), (K,), device=DEV, generator=g)]
        row[torch.randperm(K, device=DEV, generator=g)[: codes.numel()]] = codes
        w[r] = row * 2.0 ** (i - 3)                              # row maximum 448 * 2^(i-3): e = i - 3
    w[0] = 0
    return w.bfloat16()


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,K", [(203, 2080), (128, 4096), (37, 14336)])
def test_quantizer_matches_the_reference(N, K):
    w = _weights(N, K, N + K)
    deq, codes, scales = vn.op_quantize_fp8(w)
    q, e, deq_ref = R.quantize(w)
    torch.cuda.synchronize()
    assert torch.equal(scales, R.pow2(e))
    assert torch.equal(codes, R.tiled_codes(q))
    assert torch.equal(deq.view(torch.int16), deq_ref.view(torch.int16))
    # in place, as the loader runs it
    w2 = w.clone()
    vn.lib().vcl_op_quantize_fp8(vn.ptr(w2), N, K, vn.ptr(w2), vn.ptr(codes), vn.ptr(scales), vn.cur_stream())
    torch.cuda.synchronize()
    assert torch.equal(w2.view(torch.int16), deq_ref.view(torch.int16))


def _combos(K):
    return [(False, False), (False, True)] + ([(True, False), (True, True)] if K <= 5120 else [])


@pytest.mark.parametrize("K", [4096, 5120, 11008, 13824, 14336])
def test_gemv_fp8_equals_bf16_on_dequantized_weights(K):
    N = 1000                                                   # ragged: 62.5 row groups
    w = _weights(N, K, K)
    deq = R.dequantized(w)
    g = torch.Generator(device=DEV).manual_seed(K)
    for B in range(1, 17):
        x = torch.randn(B, K, device=DEV, generator=g).bfloat16()
        for norm, res in _combos(K):
            nw = (1 + 0.1 * torch.randn(K, device=DEV, generator=g)).bfloat16() if norm else None
            r = torch.randn(B, N, device=DEV, generator=g).bfloat16() if res else None
            a = vn.op_gemv_fp8(x, w, r, nw, 1e-5)
            b = vn.op_gemv(x, deq, r, nw, 1e-5)
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), (B, norm, res)


@pytest.mark.parametrize("B", [1, 4, 5, 16])
def test_gemv_fp8_lm_head_shape(B):
    """vocab rows: more than 14 row groups per SM at 5..16 clips (consecutive launches over row slices)"""
    N, K = 32003, 4096
    w = _weights(N, K, 7)
    x = torch.randn(B, K, device=DEV).bfloat16()
    nw = (1 + 0.1 * torch.randn(K, device=DEV)).bfloat16()
    a = vn.op_gemv_fp8(x, w, None, nw, 1e-5)
    b = vn.op_gemv(x, R.dequantized(w), None, nw, 1e-5)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


# ------------------------------------------------------------------------------------------------
def _model(cfg, fmt, max_batch=17):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    c = VideoChatGPTConfig(hidden_size=cfg.hidden, intermediate_size=cfg.inter, num_hidden_layers=cfg.layers,
                           num_attention_heads=cfg.heads, vocab_size=cfg.vocab, use_mm_proj=True, mm_hidden_size=1024)
    clip = dict(hidden_size=1024, intermediate_size=1024, num_hidden_layers=3, num_attention_heads=16)
    m = VideoChatGPTLlamaForCausalLM(c, clip_config=clip, max_batch=max_batch, max_seq=480, llm_weight_format=fmt)
    vc = m.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = 32000, 32001, 32002, True
    return m


@pytest.fixture(scope="module")
def pair():
    """(fp8 model on W, bf16 model on W~), 7B width, two layers, 17 clips"""
    sd = to_dev(O.random_llm_state(W7B, seed=41))
    m8, mb = _model(W7B, "fp8_e4m3"), _model(W7B, "bf16")
    m8.load_state_dict(sd)
    mb.load_state_dict(R.dequantize_state(sd))
    m8._ensure_engine(need_llm=True)
    mb._ensure_engine(need_llm=True)
    yield m8, mb
    for m in (m8, mb):
        m._engine.close()


def _same(a, b, what):
    if a is None or b is None:
        assert a is None and b is None, what
        return
    a, b = a.reshape(-1).contiguous(), b.reshape(-1).contiguous()
    assert a.dtype == b.dtype and a.shape == b.shape, what
    assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)) if a.dtype.is_floating_point else torch.equal(a, b), what


def _prompt(cfg, B, seed):
    ids = O.make_prompt_ids(cfg, 356, seed=seed, batch=B).to(DEV)
    return ids, video_feats(B, seed + 1), vid_start_of(ids, cfg)


def test_prefill_cache_and_decode_steps(pair):
    m8, mb = pair
    ids, vf, vs = _prompt(W7B, 3, 50)
    S = ids.shape[1]
    outs = []
    for m in (m8, mb):
        eng = m._engine
        _, lg, tok = eng.prefill(ids, vf, vs, want_logits=True)
        caches = [eng.kv_cache(l) for l in range(W7B.layers)]
        steps = []
        t = tok
        for i in range(3):
            lgs, t = eng.decode_step(t, S + i, want_logits=True)
            steps.append((lgs, t))
        caches2 = [eng.kv_cache(l) for l in range(W7B.layers)]
        torch.cuda.synchronize()
        outs.append((lg, tok, caches, steps, caches2))
    (lg8, t8, c8, s8, d8), (lgb, tb, cb, sb, db) = outs
    _same(lg8, lgb, "prefill logits")
    _same(t8, tb, "prefill token")
    for l in range(W7B.layers):
        _same(c8[l][0], cb[l][0], f"K cache layer {l}")
        _same(c8[l][1], cb[l][1], f"V cache layer {l}")
        _same(d8[l][0], db[l][0], f"K cache after decode, layer {l}")
        _same(d8[l][1], db[l][1], f"V cache after decode, layer {l}")
    for i in range(3):
        _same(s8[i][0], sb[i][0], f"decode step {i} logits")
        _same(s8[i][1], sb[i][1], f"decode step {i} token")


@pytest.mark.parametrize("B", [1, 3, 5, 9, 16, 17])
def test_generate(pair, B):
    ids, vf, _ = _prompt(W7B, B, 60 + B)
    st = torch.cuda.Stream()
    outs, counts = [], []
    for m in pair:
        with torch.cuda.stream(st):
            m.generate(ids, video_spatio_temporal_features=vf, max_new_tokens=7, eos_token_id=None)   # captures
            c0 = vn.launch_count()
            outs.append(m.generate(ids, video_spatio_temporal_features=vf, max_new_tokens=7, eos_token_id=None))
            counts.append(vn.launch_count() - c0)
        st.synchronize()
    _same(outs[0], outs[1], f"generate B={B}")
    assert counts[0] == counts[1], counts                    # the same kernels, and graphs of as many nodes


def test_left_padded_generate_and_continue(pair):
    ids, n_pad, _ = padded_batch(W7B, [10, 40, 25], seed=70)
    vf = video_feats(3, 71)
    mask = torch.ones_like(ids)
    for b, p in enumerate(n_pad):
        mask[b, :p] = 0
    new = torch.randint(3, 32000, (3, 5), generator=torch.Generator().manual_seed(72)).to(DEV)
    outs = []
    st = torch.cuda.Stream()
    for m in pair:
        with torch.cuda.stream(st):
            a = m.generate(ids, video_spatio_temporal_features=vf, attention_mask=mask, max_new_tokens=6,
                           eos_token_id=None)
            c = m.generate_continue(new, max_new_tokens=5, eos_token_id=None)
        st.synchronize()
        outs.append((a, c))
    _same(outs[0][0], outs[1][0], "left-padded generate")
    _same(outs[0][1], outs[1][1], "generate_continue")


def test_seeded_sampling(pair):
    ids, vf, _ = _prompt(W7B, 5, 80)
    outs = []
    st = torch.cuda.Stream()
    for m in pair:
        with torch.cuda.stream(st):
            outs.append(m.generate(ids, video_spatio_temporal_features=vf, do_sample=True, temperature=0.7, top_k=50,
                                   seed=1234, max_new_tokens=9, eos_token_id=None))
        st.synchronize()
    _same(outs[0], outs[1], "seeded sampling")


def test_packed_inflight_requests(pair):
    lens = [5, 9, 3, 12, 7, 4, 10, 6, 8, 2, 11]
    reqs = []
    for i, n in enumerate(lens):
        if i == 5:
            ids = torch.cat([torch.tensor([1]), torch.randint(3, 32000, (49,), generator=torch.Generator().manual_seed(i))])
            reqs.append(dict(input_ids=ids, max_new_tokens=n))
        else:
            ids = O.make_prompt_ids(W7B, 356, seed=200 + i, n_pre=20 + 4 * i)
            reqs.append(dict(input_ids=ids, video_spatio_temporal_features=video_feats(1, 300 + i)[0].half(),
                             max_new_tokens=n))
    outs = []
    st = torch.cuda.Stream()
    for m in pair:
        with torch.cuda.stream(st):
            outs.append(m.generate_requests(reqs, eos_token_id=None, slots=4, packed_admission=True))
        st.synchronize()
    for i, (a, b) in enumerate(zip(*outs)):
        _same(a, b, f"request {i}")


def test_score(pair):
    ids, n_pad, _ = padded_batch(W7B, [10, 30], seed=90)
    vf = video_feats(2, 91)
    vs = vid_start_of(ids, W7B)
    labels = ids.clone()
    labels[:, :380] = -100
    outs = []
    for m in pair:
        outs.append(m._engine.score(ids, vf, vs, labels=labels, n_pad=n_pad, want_logits=True))
        torch.cuda.synchronize()
    for what, a, b in zip(("logits", "nll", "loss"), *outs):
        _same(a, b, f"score {what}")


def test_13b_width():
    sd = to_dev(O.random_llm_state(W13B, seed=43))
    m8, mb = _model(W13B, "fp8_e4m3", max_batch=16), _model(W13B, "bf16", max_batch=16)
    m8.load_state_dict(sd)
    mb.load_state_dict(R.dequantize_state(sd))
    st = torch.cuda.Stream()
    try:
        for B in (1, 4, 5, 16):                                 # gate|up at 5..16 clips: 14 row groups per SM
            ids, vf, vs = _prompt(W13B, B, 100 + B)
            outs = []
            for m in (m8, mb):
                with torch.cuda.stream(st):
                    _, lg, _ = m._ensure_engine(need_llm=True).prefill(ids, vf, vs, want_logits=True)
                    g = m.generate(ids, video_spatio_temporal_features=vf, max_new_tokens=5, eos_token_id=None)
                st.synchronize()
                outs.append((lg, g))
            _same(outs[0][0], outs[1][0], f"13B prefill logits B={B}")
            _same(outs[0][1], outs[1][1], f"13B generate B={B}")
    finally:
        for m in (m8, mb):
            if m._engine is not None:
                m._engine.close()


# ------------------------------------------------------------------------------------------------
def _saving_bytes(cfg):
    """bf16 decode copy minus (codes + row scales), per the loader's layouts"""
    D, F, V = cfg.hidden, cfg.inter, cfg.vocab
    mats = [(3 * D, D), (D, D), (2 * F, D), (D, F)] * cfg.layers + [(V, D)]
    return sum(vn.tiled_elems(N, K) * 2 - vn.tiled_elems(N, K) - 4 * N for N, K in mats)


def _resident(cfg, sd, fmt):
    gc.collect()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    eng = make_engine(llm=cfg, max_batch=4, max_seq=480)
    eng.load_llm(sd, weight_format=fmt)
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    eng.close()
    return used


def test_resident_memory_drops_by_the_computed_saving():
    cfg = O.LlmCfg(hidden=4096, inter=11008, heads=32, layers=4)
    sd = to_dev(O.random_llm_state(cfg, seed=3))
    bf, f8 = _resident(cfg, sd, "bf16"), _resident(cfg, sd, "fp8_e4m3")
    saving = _saving_bytes(cfg)
    print(f"[fp8] resident: bf16 {bf / 2**30:.3f} GiB, fp8 {f8 / 2**30:.3f} GiB, "
          f"computed saving {saving / 2**30:.3f} GiB, measured {(bf - f8) / 2**30:.3f} GiB")
    assert bf - f8 >= 0.95 * saving


def test_non_finite_weight_fails_the_load_with_its_name():
    sd = to_dev(O.random_llm_state(SMALL, seed=5))
    for name, row, val in (("model.layers.1.mlp.up_proj.weight", 5, float("nan")),
                           ("model.layers.0.self_attn.k_proj.weight", 130, float("inf")),
                           ("lm_head.weight", 31999, float("-inf"))):
        bad = dict(sd)
        bad[name] = sd[name].clone()
        bad[name][row, 7] = val
        eng = make_engine(llm=SMALL, max_batch=2, max_seq=480)
        with pytest.raises(vn.VclError, match=f"'{name}' has a non-finite value in row {row}"):
            eng.load_llm(bad, weight_format="fp8_e4m3")
        eng.close()
    eng = make_engine(llm=SMALL, max_batch=2, max_seq=480)
    with pytest.raises(ValueError):
        eng.load_llm(sd, weight_format="fp8")
    eng.load_llm(sd, weight_format="fp8_e4m3")                 # a rejected format leaves the handle loadable
    eng.close()
