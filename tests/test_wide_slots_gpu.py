"""Decode of 17..64 clips by the window kernel (gemv_tcw with 2 or 4 clip groups) and in-flight batching with up to
64 cache slots.

- the kernel (vcl_op_gemv) at B = 17, 24, 32, 33, 48, 64 against the fp64 reference and bounds of test_gemv, at the
  7B q|k|v, o_proj, down_proj and lm_head shapes; clip b's output does not depend on the other clips' inputs; the
  fp8 instance (vcl_op_gemv_fp8) equals the bf16 one on W~ bit for bit;
- a decode step and a slot decode at 24 and 64 clips write one cache column per clip (2-ulp bound of
  test_kv_cache_gpu.py) and nothing else, padded and unpadded;
- generate at 24 and 64 clips, and left-padded at 40, follows the bf16 oracle up to its first near-tie per clip;
- slots: slot decode equals the shared-position loop (graph and eager), slot isolation, graph replay for new
  positions, generate_requests(slots=64) against each request alone and the oracle, packed admission, seeded
  sampling independent of the admission order;
- an fp8 engine on W equals a bf16 engine on W~ at 7B and 13B width (generate at 17 / 33 / 64 clips, slot decode,
  packed in-flight batching) with equal launch counts;
- max_slots and slot counts above it are rejected before any device work;
- 65 clips still take the prefill-GEMM decode (rmsnorm, GEMM, rope_kv_prefill_kernel) and the chunked lm_head:
  cache writes and generate against the oracle there;
- at 7B width (B = 33: q|k|v in one launch, gate|up in two row slices) and 13B width (B = 48: q|k|v and gate|up in
  row slices), decode steps teacher-forced against the bf16 oracle follow the margin rule, which checks the RoPE and
  SwiGLU epilogues of the sliced launches against an independent reference; so do decode steps at 10240 width and
  5..16 clips (B = 8: q|k|v in row slices of one clip group)."""
import time
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
import _fp8_ref as R  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import relerr, teacher_forced_check, to_dev, vid_start_of  # noqa: E402
from test_padded_batch_gpu import first_near_tie, padded_batch, video_feats  # noqa: E402
from test_kv_cache_gpu import (_assert_kv, _assert_same, _caches, _check_step, _embed, _fill_sentinel, _ids,  # noqa: E402
                               _no_video, _ref_kv, _state)
from test_inflight_gpu import prompt, text_prompt  # noqa: E402

DEV = "cuda"
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)
W7B = O.LlmCfg(hidden=4096, inter=11008, heads=32, layers=2)
W13B = O.LlmCfg(hidden=5120, inter=13824, heads=40, layers=1)
W10K = O.LlmCfg(hidden=10240, inter=2048, heads=80, layers=1)   # q|k|v: 1920 row groups > 14 per SM x 132 SMs
WIDE_B = [17, 24, 32, 33, 48, 64]


def engine(llm, max_batch, max_seq, max_slots=0, sd=None, fmt="bf16"):
    clip = O.ClipCfg()
    c = vn.vcl_config()
    c.clip_layers, c.clip_hidden, c.clip_inter, c.clip_heads = clip.layers - 1, clip.hidden, clip.inter, clip.heads
    c.image_size, c.patch_size, c.clip_ln_eps = clip.image, clip.patch, clip.eps
    c.llm_layers, c.llm_hidden, c.llm_inter, c.llm_heads = llm.layers, llm.hidden, llm.inter, llm.heads
    c.vocab, c.rms_eps, c.rope_theta = llm.vocab, llm.rms_eps, llm.rope_theta
    c.proj_type = vn.PROJ_LINEAR if llm.proj_type == "linear" else vn.PROJ_MLP2X_GELU
    c.n_temporal = 100
    c.max_frames, c.max_batch, c.max_seq, c.max_slots = 1, max_batch, max_seq, max_slots
    eng = vn.Engine(c)
    if sd is not None:
        eng.load_llm(sd, weight_format=fmt)
    return eng


def model(cfg, max_batch, max_slots=None, fmt="bf16", max_seq=480):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    c = VideoChatGPTConfig(hidden_size=cfg.hidden, intermediate_size=cfg.inter, num_hidden_layers=cfg.layers,
                           num_attention_heads=cfg.heads, vocab_size=cfg.vocab, use_mm_proj=True, mm_hidden_size=1024)
    clip = dict(hidden_size=1024, intermediate_size=1024, num_hidden_layers=3, num_attention_heads=16)
    m = VideoChatGPTLlamaForCausalLM(c, clip_config=clip, max_batch=max_batch, max_seq=max_seq, llm_weight_format=fmt,
                                     max_slots=max_slots)
    vc = m.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = 32000, 32001, 32002, True
    return m


def same(a, b, what):
    a, b = a.reshape(-1).contiguous(), b.reshape(-1).contiguous()
    assert a.dtype == b.dtype and a.shape == b.shape, what
    ok = torch.equal(a.view(torch.uint8), b.view(torch.uint8)) if a.dtype.is_floating_point else torch.equal(a, b)
    assert ok, what


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("B", WIDE_B)
@pytest.mark.parametrize("N,K,norm,res", [(4096, 4096, False, True), (12288, 4096, True, False),
                                          (4096, 11008, False, True), (32003, 4096, False, False)])
def test_wide_gemv(B, N, K, norm, res):
    """the bounds of test_kernels_gpu.py::test_gemv"""
    torch.manual_seed(N + K + B)
    x = torch.randn(B, K, device=DEV).bfloat16()
    w = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
    nw = (1 + 0.1 * torch.randn(K, device=DEV)).bfloat16() if norm else None
    r = torch.randn(B, N, device=DEV).bfloat16() if res else None
    out = vn.op_gemv(x, w, r, nw, 1e-5)
    xf = x.float()
    if norm:
        xf = (nw.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5)).bfloat16().float()).bfloat16().float()
    ref = (xf.double() @ w.double().t()).float()
    mag = ref.abs()
    if res:
        ref = ref.bfloat16().float() + r.float()
    rel = ((out.float() - ref).norm() / ref.norm()).item()
    assert rel < 3e-3, rel
    mag = torch.maximum(mag, ref.abs())
    assert ((out.float() - ref).abs() <= 2.5 * mag.clamp_min(1e-2) * 2 ** -7).all()


@pytest.mark.parametrize("B", WIDE_B)
def test_wide_gemv_columns_are_isolated(B):
    """new inputs for every other clip leave clip b's outputs bit-identical (b in the first, a middle and the last
    clip group), at the lm_head shape (row slices) and a ragged one"""
    for N, K in ((32003, 4096), (1000, 5120)):
        g = torch.Generator(device=DEV).manual_seed(B * 7 + N)
        x = torch.randn(B, K, device=DEV, generator=g).bfloat16()
        w = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).bfloat16()
        out = vn.op_gemv(x, w)
        for b in sorted({0, B // 2, B - 1}):
            x2 = torch.randn(B, K, device=DEV, generator=g).bfloat16()
            x2[b] = x[b]
            out2 = vn.op_gemv(x2, w)
            same(out2[b], out[b], f"B={B} N={N} clip {b}")


@pytest.mark.parametrize("B", WIDE_B)
def test_wide_gemv_fp8_equals_bf16_on_dequantized_weights(B):
    from test_fp8_gpu import _weights
    for N, K, res in ((1000, 4096, True), (1000, 11008, False), (27648, 5120, False)):
        w = _weights(N, K, K + B)
        deq = R.dequantized(w)
        g = torch.Generator(device=DEV).manual_seed(B + K)
        x = torch.randn(B, K, device=DEV, generator=g).bfloat16()
        r = torch.randn(B, N, device=DEV, generator=g).bfloat16() if res else None
        same(vn.op_gemv_fp8(x, w, r), vn.op_gemv(x, deq, r), f"B={B} N={N} K={K}")


# ------------------------------------------------------------------------------------------------ KV cache
@pytest.fixture(scope="module")
def eng64():
    """width 512, 2 layers, 64 clips and 64 slots, 64 columns"""
    eng = engine(SMALL, 64, 64, max_slots=64, sd=_state(512))
    yield eng
    eng.close()


@torch.no_grad()
@pytest.mark.parametrize("B,padded", [(24, False), (24, True), (64, False), (64, True)])
def test_decode_step_writes_one_column(eng64, B, padded):
    S = 37
    pads = [(11 * b) % S for b in range(B)] if padded else None
    _fill_sentinel(eng64)
    eng64.prefill(_ids(B, S, 10 + B), None, _no_video(B), n_pad=pads)
    before = [(k.clone(), v.clone()) for k, v in _caches(eng64)]
    feed = torch.randint(3, 32000, (B,), generator=torch.Generator().manual_seed(B)).to(DEV, torch.int32)
    eng64.decode_step(feed, S)
    npad = pads or [0] * B
    _check_step(eng64, before, B, [S] * B, [S - npad[b] for b in range(B)], feed, f"B={B} padded={padded}")


@torch.no_grad()
@pytest.mark.parametrize("n_slots", [24, 64])
def test_slot_decode_writes_each_slots_column(eng64, n_slots):
    _fill_sentinel(eng64)
    lens = [5 + (7 * b) % 40 for b in range(n_slots)]
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for b, n in enumerate(lens):
            eng64.slot_prefill(b, _ids(1, n, 30 + b), None, _no_video(1))
        before = [(k.clone(), v.clone()) for k, v in _caches(eng64)]
        feed = torch.randint(3, 32000, (n_slots,), generator=torch.Generator().manual_seed(n_slots)).to(DEV, torch.int32)
        eng64.slot_decode(feed, lens, 2)
    st.synchronize()
    _check_step(eng64, before, n_slots, lens, lens, feed, f"{n_slots} slots")


# ------------------------------------------------------------------------------------------------ end to end
@pytest.fixture(scope="module")
def small_sd():
    return O.random_llm_state(SMALL, seed=21)


@torch.no_grad()
@pytest.mark.parametrize("B", [24, 64])
def test_generate_follows_the_oracle(B, small_sd, max_batch=64):
    m = model(SMALL, max_batch=max_batch)
    m.load_state_dict(dict(small_sd))
    ids = O.make_prompt_ids(SMALL, 356, seed=400 + B, batch=B).to(DEV)
    vf = video_feats(B, 401 + B)
    n = 8
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        out = m.generate(ids, video_spatio_temporal_features=vf, max_new_tokens=n, eos_token_id=None)
    st.synchronize()
    o_toks, o_logits = O.greedy_generate(to_dev(small_sd), SMALL, ids, vf.bfloat16(), n)
    ties = first_near_tie(o_logits)
    S = ids.shape[1]
    for b in range(B):
        t = ties[b]
        assert torch.equal(out[b, S:S + t].cpu(), o_toks[b, :t].cpu()), (b, t)
    m._engine.close()


@torch.no_grad()
def test_left_padded_generate_follows_the_oracle(small_sd):
    B = 40
    ids, pads, rows = padded_batch(SMALL, [63 - (7 * b) % 40 for b in range(B)], seed=40)
    vf = video_feats(B, 41)
    mask = torch.ones_like(ids)
    for b, p in enumerate(pads):
        mask[b, :p] = 0
    m = model(SMALL, max_batch=40)
    m.load_state_dict(dict(small_sd))
    n = 6
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        out = m.generate(ids, video_spatio_temporal_features=vf, attention_mask=mask, max_new_tokens=n,
                         eos_token_id=None)
    st.synchronize()
    sd_b, S = to_dev(small_sd), ids.shape[1]
    for b in range(B):
        row = rows[b].reshape(1, -1).to(DEV)
        o_toks, o_logits = O.greedy_generate(sd_b, SMALL, row, vf[b:b + 1].bfloat16(), n)
        t = first_near_tie(o_logits)[0]
        assert torch.equal(out[b, S:S + t].cpu(), o_toks[0, :t].cpu()), (b, t)
    m._engine.close()


# ------------------------------------------------------------------------------------------------ slots
@torch.no_grad()
@pytest.mark.parametrize("NB", [24, 64])
def test_slot_decode_matches_the_shared_position_loop(NB, small_sd):
    ids = O.make_prompt_ids(SMALL, 356, seed=30, batch=NB).to(DEV)
    S, k = ids.shape[1], 10
    vf = video_feats(NB, 31)
    eng = engine(SMALL, NB, 480, max_slots=NB, sd=to_dev(small_sd))
    vs = vid_start_of(ids, SMALL)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        _, _, first = eng.prefill(ids, vf, vs)
        shared = eng.decode_loop(first, S, k)
        eng.prefill(ids, vf, vs)
        slots = eng.slot_decode(first, [S] * NB, k)
    st.synchronize()
    eng.prefill(ids, vf, vs)
    eager = eng.slot_decode(first, [S] * NB, k)
    torch.cuda.synchronize()
    assert torch.equal(slots, shared)
    assert torch.equal(eager, shared)
    eng.close()


def _admit(eng, slot, ids, vf):
    ids = ids.to(DEV)[None]
    return eng.slot_prefill(slot, ids, vf, vid_start_of(ids, SMALL))


@torch.no_grad()
def test_slot_isolation_at_40_slots(small_sd):
    NB, s, k = 40, 23, 8
    eng = engine(SMALL, NB, 480, max_slots=NB, sd=to_dev(small_sd))
    x, vx = prompt(SMALL, 50, 40), video_feats(1, 51)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        first = torch.empty(NB, dtype=torch.int32, device=DEV)
        pos = []
        for b in range(NB):
            ids = x if b == s else prompt(SMALL, 60 + b, 20 + b)
            first[b:b + 1] = _admit(eng, b, ids, vx if b == s else video_feats(1, 70 + b))
            pos.append(len(ids))
        run1 = eng.slot_decode(first, pos, k)[s].clone()
        first = torch.empty(NB, dtype=torch.int32, device=DEV)
        pos = []
        for b in range(NB):
            ids = prompt(SMALL, 180 + b, 10 + b % 30) if b % 2 else text_prompt(190 + b, 30 + 3 * b)
            first[b:b + 1] = _admit(eng, b, ids, video_feats(1, 200 + b) if b % 2 else None)
            pos.append(len(ids))
        out = eng.slot_decode(first, pos, 6)
        first = out[:, -1].contiguous()
        pos = [p + 5 for p in pos]
        first[s:s + 1] = _admit(eng, s, x, vx)
        pos[s] = len(x)
        run2 = eng.slot_decode(first, pos, k)[s].clone()
    st.synchronize()
    assert torch.equal(run1, run2), (run1.tolist(), run2.tolist())
    eng.close()


@torch.no_grad()
def test_graph_is_replayed_for_new_positions(small_sd):
    NB, k = 33, 6
    sd = to_dev(small_sd)
    eng, fresh = engine(SMALL, NB, 480, NB, sd), engine(SMALL, NB, 480, NB, sd)
    rows = [text_prompt(400 + b, 30 + 3 * b) for b in range(NB)]
    st = torch.cuda.Stream()
    deltas, outs = [], []
    with torch.cuda.stream(st):
        first = torch.cat([_admit(eng, b, r, None) for b, r in enumerate(rows)])
        first_f = torch.cat([_admit(fresh, b, r, None) for b, r in enumerate(rows)])
        host_ms = []
        for shift in (0, 9):
            st.synchronize()
            n0 = vn.launch_count()
            t0 = time.perf_counter()
            outs.append(eng.slot_decode(first, [len(r) - shift for r in rows], k))
            host_ms.append((time.perf_counter() - t0) * 1e3)
            st.synchronize()
            deltas.append(vn.launch_count() - n0)
        ref = fresh.slot_decode(first_f, [len(r) - 9 for r in rows], k)
    st.synchronize()
    # a replay adds the graph's kernel nodes to the launch count and costs the host no capture / instantiation
    assert deltas[0] == deltas[1] > (k - 1) * SMALL.layers, deltas
    assert host_ms[1] < 0.5 * host_ms[0], host_ms
    assert torch.equal(outs[1], ref)
    eng.close()
    fresh.close()


def _requests(cfg, n, seed=0):
    reqs = []
    for i in range(n):
        k = 2 + (i * 5 + seed) % 9
        if i % 7 == 3:
            reqs.append(dict(input_ids=text_prompt(600 + i, 20 + i % 30), max_new_tokens=k))
        else:
            reqs.append(dict(input_ids=prompt(cfg, 700 + i, 10 + (3 * i) % 50)[None],
                             video_spatio_temporal_features=video_feats(1, 800 + i)[0].half(), max_new_tokens=k))
    return reqs


@torch.no_grad()
def test_requests_at_64_slots_match_each_request_alone_and_the_oracle(small_sd):
    m = model(SMALL, max_batch=64, max_slots=64)
    m.load_state_dict(dict(small_sd))
    reqs = _requests(SMALL, 100)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        outs = m.generate_requests(reqs, eos_token_id=None, slots=64)
        packed = m.generate_requests(reqs, eos_token_id=None, slots=64, packed_admission=True)
    st.synchronize()
    sd_b = to_dev(small_sd)
    for i, r in enumerate(reqs):
        same(packed[i], outs[i], f"request {i}: packed admission")
        ids = torch.as_tensor(r["input_ids"]).reshape(1, -1).to(DEV)
        S, n = ids.shape[1], r["max_new_tokens"]
        f = r.get("video_spatio_temporal_features")
        f = None if f is None else f[None]
        assert outs[i].shape == (1, S + n) and torch.equal(outs[i][:, :S], ids)
        own = m.generate(ids, video_spatio_temporal_features=f, max_new_tokens=n, eos_token_id=None)
        o_toks, o_logits = O.greedy_generate(sd_b, SMALL, ids, None if f is None else f.to(DEV).bfloat16(), n)
        t = first_near_tie(o_logits)[0]
        new = outs[i][0, S:]
        assert torch.equal(new[:t], own[0, S:S + t]), (i, t)
        assert torch.equal(new[:t].cpu(), o_toks[0, :t].cpu()), (i, t)
    m._engine.close()


@torch.no_grad()
def test_seeded_requests_do_not_depend_on_admission_order(small_sd):
    m = model(SMALL, max_batch=64, max_slots=64)
    m.load_state_dict(dict(small_sd))
    reqs = _requests(SMALL, 80, seed=3)
    for i, r in enumerate(reqs):
        r["seed"] = 1000 + i
    kw = dict(eos_token_id=None, do_sample=True, temperature=0.8, top_k=50)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        a = m.generate_requests(reqs, slots=64, **kw)
        b = m.generate_requests(reqs, slots=64, **kw)
        c = m.generate_requests(reqs[::-1], slots=40, packed_admission=True, **kw)[::-1]
    st.synchronize()
    for i in range(len(reqs)):
        same(a[i], b[i], f"request {i}: repeated")
        same(a[i], c[i], f"request {i}: reversed queue, packed, 40 slots")
    m._engine.close()


# ------------------------------------------------------------------------------------------------ fp8
def _fp8_pair(cfg, seed, max_batch=64):
    sd = to_dev(O.random_llm_state(cfg, seed=seed))
    m8, mb = model(cfg, max_batch, 64, "fp8_e4m3"), model(cfg, max_batch, 64, "bf16")
    m8.load_state_dict(sd)
    mb.load_state_dict(R.dequantize_state(sd))
    return m8, mb


@torch.no_grad()
@pytest.mark.parametrize("cfg", [W7B, W13B], ids=["7B", "13B"])
def test_fp8_equals_bf16_on_dequantized_weights(cfg):
    m8, mb = _fp8_pair(cfg, 47)
    st = torch.cuda.Stream()
    try:
        for B in (17, 33, 64):
            ids = O.make_prompt_ids(cfg, 356, seed=900 + B, batch=B).to(DEV)
            vf = video_feats(B, 901 + B)
            outs, counts = [], []
            for m in (m8, mb):
                with torch.cuda.stream(st):
                    m.generate(ids, video_spatio_temporal_features=vf, max_new_tokens=5, eos_token_id=None)
                    c0 = vn.launch_count()
                    outs.append(m.generate(ids, video_spatio_temporal_features=vf, max_new_tokens=5, eos_token_id=None))
                    counts.append(vn.launch_count() - c0)
                st.synchronize()
            same(outs[0], outs[1], f"generate B={B}")
            assert counts[0] == counts[1], counts
        # slot decode and packed in-flight batching
        reqs = _requests(cfg, 70, seed=5)
        outs = []
        for m in (m8, mb):
            with torch.cuda.stream(st):
                eng = m._ensure_engine(need_llm=True)
                rows = [text_prompt(950 + b, 20 + b) for b in range(48)]
                first = torch.cat([eng.slot_prefill(b, r.to(DEV)[None], None, _no_video(1)) for b, r in enumerate(rows)])
                sd_out = eng.slot_decode(first, [len(r) for r in rows], 4)
                rq = m.generate_requests(reqs, eos_token_id=None, slots=64, packed_admission=True)
            st.synchronize()
            outs.append((sd_out, rq))
        same(outs[0][0], outs[1][0], "slot decode at 48 slots")
        for i, (a, b) in enumerate(zip(outs[0][1], outs[1][1])):
            same(a, b, f"request {i}")
    finally:
        for m in (m8, mb):
            if m._engine is not None:
                m._engine.close()


# ------------------------------------------------------------------------------------------------ rejections
@torch.no_grad()
def test_rejections_before_any_device_work(small_sd):
    for mb, ms in ((8, 9), (80, 65), (8, -1)):
        n0 = vn.launch_count()
        with pytest.raises(vn.VclError, match=f"max_slots={ms} outside"):
            engine(SMALL, mb, 64, max_slots=ms)
        assert vn.launch_count() == n0
    for mb, ms in ((8, 9), (80, 65), (8, 0), (8, 2.5)):
        with pytest.raises(ValueError, match="max_slots"):
            model(SMALL, max_batch=mb, max_slots=ms)
    eng = engine(SMALL, 40, 64, max_slots=24, sd=to_dev(small_sd))
    ids = text_prompt(7, 20)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        first = torch.cat([_admit(eng, b, ids, None) for b in range(24)])
        st.synchronize()
        n0 = vn.launch_count()
        with pytest.raises(vn.VclError, match=r"n_slots=25 outside 1..24 \(max_slots 24\)"):
            eng.slot_decode(torch.zeros(25, dtype=torch.int32, device=DEV), [20] * 25, 2)
        with pytest.raises(vn.VclError, match=r"slot 24 outside 0..23 \(max_slots 24\)"):
            _admit(eng, 24, ids, None)
        with pytest.raises(vn.VclError, match=r"n=25 outside 1..24 \(max_slots 24\)"):
            eng.slots_prefill(list(range(25)), [ids] * 25, [None] * 25, [0] * 25)
        assert vn.launch_count() == n0
        out = eng.slot_decode(first, [20] * 24, 3)
    st.synchronize()
    assert (out == out[0]).all()
    eng.close()
    m = model(SMALL, max_batch=40, max_slots=24)
    m.load_state_dict(dict(small_sd))
    with pytest.raises(ValueError, match=r"slots=25 outside 1..24 \(max_slots 24\)"):
        m.generate_requests([ids], slots=25)


# ------------------------------------------------------------------------------------------------ 65 clips: the GEMM decode
@pytest.fixture(scope="module")
def eng65():
    eng = engine(SMALL, 65, 64, sd=_state(512))
    yield eng
    eng.close()


@torch.no_grad()
@pytest.mark.parametrize("padded", [False, True])
def test_decode_step_above_64_clips_writes_one_column(eng65, padded):
    B, S = 65, 37
    pads = [(11 * b) % S for b in range(B)] if padded else None
    _fill_sentinel(eng65)
    eng65.prefill(_ids(B, S, 77), None, _no_video(B), n_pad=pads)
    before = [(k.clone(), v.clone()) for k, v in _caches(eng65)]
    feed = torch.randint(3, 32000, (B,), generator=torch.Generator().manual_seed(65)).to(DEV, torch.int32)
    eng65.decode_step(feed, S)
    npad = pads or [0] * B
    # the GEMM decode normalises its rows with the engine's rmsnorm kernel, as the prefill does: the reference takes
    # those rows (prefill=True), so that a one-ulp flip of a normalised element is not counted against the cache
    after = _caches(eng65)
    rk, rv = _ref_kv(512, 0, _embed(feed), [S - npad[b] for b in range(B)], prefill=True)
    _assert_kv(after[0][0][:, :, S], rk, f"B=65 padded={padded}: layer 0 k")
    _assert_kv(after[0][1][:, :, S], rv, f"B=65 padded={padded}: layer 0 v")
    for l in range(SMALL.layers):
        for i, n in enumerate("kv"):
            a, b = after[l][i].clone(), before[l][i]
            assert torch.isfinite(a[:, :, S].float()).all(), (l, n)
            a[:, :, S] = b[:, :, S]
            _assert_same(a, b, f"B=65: layer {l} {n} outside the new column")


@torch.no_grad()
def test_generate_above_64_clips_follows_the_oracle(small_sd):
    test_generate_follows_the_oracle(65, small_sd, max_batch=65)


# ------------------------------------------------------------------------------------------------ 7B / 13B width
@torch.no_grad()
@pytest.mark.parametrize("cfg,B", [(W7B, 33), (W13B, 48)], ids=["7B-33", "13B-48"])
def test_wide_width_decode_teacher_forced_against_the_oracle(cfg, B):
    sd = O.random_llm_state(cfg, seed=61)
    sd_b = to_dev(sd)
    eng = engine(cfg, B, 480, sd=sd_b)
    ids = O.make_prompt_ids(cfg, 356, seed=620 + B, batch=B).to(DEV)
    vf = video_feats(B, 621 + B)
    teacher_forced_check(eng, sd_b, cfg, ids, vf, 4, f"{cfg.hidden} B={B}")
    eng.close()


@torch.no_grad()
def test_sliced_qkv_at_5_to_16_clips_decodes_like_the_oracle():
    """5..16 clips with q|k|v in row slices (width 10240: 1920 row groups, more than 14 per SM on 132 SMs) through the
    RoPE and KV-append epilogue. The prefill's RMSNorm takes widths up to 8192, so the engine decodes from an empty
    cache: steps at positions 0..3 on random tokens against the oracle's cached forward, with the margin rule."""
    cfg, B = W10K, 8
    sd_b = to_dev(O.random_llm_state(cfg, seed=61))
    eng = engine(cfg, B, 16, sd=sd_b)
    toks = torch.randint(3, 32000, (B, 4), generator=torch.Generator().manual_seed(628)).to(DEV)
    past = None
    for i in range(toks.shape[1]):
        o_logits, _, past = O.llm_forward(sd_b, cfg, toks[:, i:i + 1], None, past)
        o = o_logits[:, -1].float()
        lg, _ = eng.decode_step(toks[:, i].to(torch.int32).contiguous(), i, want_logits=True)
        e = relerr(lg, o)
        assert e < 3e-2, (i, e)
        top = torch.topk(o, 2, dim=-1)
        clear = (top.values[:, 0] - top.values[:, 1]) / (top.values[:, 0].abs().clamp_min(2 ** -6) * 2 ** -7) >= 3
        assert torch.equal(lg.argmax(-1)[clear], top.indices[clear, 0]), i
    eng.close()
