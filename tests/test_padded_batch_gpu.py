"""Left-padded batches of prompts of different lengths on the GPU (vcl_llm_prefill_padded /
vcl_llm_generate_padded, the padding carried on by appends and decode steps, and the attention_mask of
the Python drop-in): every clip of a padded batch must be computed as if it ran alone.

Tolerances are the ones the batch-path tests use (relerr < 1e-2 for a prefill, < 2e-2 for decode steps,
test_parity_gpu.py) and the teacher-forced margin rule against the bf16 oracle (_util.teacher_forced_check):
identical arg-max wherever the oracle's top-1/top-2 margin is >= 3 bf16 ulps, a tied candidate otherwise."""
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import make_engine, relerr, to_dev, vid_start_of  # noqa: E402

DEV = "cuda"
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)


def padded_batch(cfg, n_pres, seed, n_post=26, pad_id=0):
    """Rows of O.make_prompt_ids with n_pre = n_pres[b], left-padded with pad_id to the longest one.
    Returns (ids [B,S], n_pad list, the unpadded rows)."""
    rows = [O.make_prompt_ids(cfg, 356, seed=seed + b, n_pre=n, n_post=n_post)[0] for b, n in enumerate(n_pres)]
    S = max(len(r) for r in rows)
    ids = torch.full((len(rows), S), pad_id, dtype=torch.int64)
    for b, r in enumerate(rows):
        ids[b, S - len(r):] = r
    return ids.to(DEV), [S - len(r) for r in rows], [r[None].to(DEV) for r in rows]


def video_feats(B, seed):
    return (torch.randn(B, 356, 1024, generator=torch.Generator().manual_seed(seed)) * 0.5).half().float().to(DEV)


def margins_ulps(logits):
    """[B, V] -> the top-1/top-2 margin of every row in bf16 ulps of the top logit, and the top-1 values and ulps"""
    top = torch.topk(logits, 2, dim=-1)
    ulp = top.values[:, 0].abs().clamp_min(2 ** -6) * 2 ** -7
    return (top.values[:, 0] - top.values[:, 1]) / ulp, top.values[:, 0], ulp


def check_margin_rule(ours_tok, o_tok, o_logits, what):
    """the teacher-forced token rule of _util.teacher_forced_check for one step, every row"""
    margin, top, ulp = margins_ulps(o_logits)
    for b in range(o_logits.shape[0]):
        if margin[b] >= 3:
            assert int(ours_tok[b]) == int(o_tok[b]), (what, b, margin[b].item())
        else:
            gap = ((top[b] - o_logits[b, int(ours_tok[b])]) / ulp[b]).item()
            assert gap < 3, (what, b, "our token's oracle logit is %.2f ulps below the top" % gap)


def first_near_tie(o_logits):
    """[n_new, B, V] oracle logits -> per clip the first step whose margin is < 3 ulps (n_new if none)"""
    n, B = o_logits.shape[0], o_logits.shape[1]
    out = [n] * B
    for i in range(n):
        m, _, _ = margins_ulps(o_logits[i])
        for b in range(B):
            if out[b] == n and m[b] < 3:
                out[b] = i
    return out


def pads_for(NB):
    """n_pre per clip: pad counts from 0 to 39 columns, clip 0 unpadded"""
    return [63 - (7 * b) % 40 for b in range(NB)]


# ------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("NB", [3, 9, 17])
def test_padded_rows_match_clips_run_alone(NB):
    """1..4 clips: gemv_tc, 5..16: gemv_tcw, > 16: the GEMM decode with rope_kv_prefill_kernel. Per clip the
    padded batch must give the real rows' hidden states and the logits of the clip prefilled alone and unpadded,
    and two decode steps must follow it; every hidden state, pad rows included, must be finite."""
    ids, pads, rows = padded_batch(SMALL, pads_for(NB), seed=40)
    assert max(pads) > 0 and min(pads) == 0
    S = ids.shape[1]
    vf = video_feats(NB, 12)
    eng = make_engine(llm=SMALL, max_batch=NB, max_seq=480)
    eng.load_llm(to_dev(O.random_llm_state(SMALL, seed=21)))
    vs = vid_start_of(ids, SMALL)
    h, lg, _ = eng.prefill(ids, vf, vs, want_hidden=True, want_logits=True, n_pad=pads)
    assert torch.isfinite(h).all()
    tok = lg.argmax(-1).to(torch.int32)
    lgb, tokb = eng.decode_step(tok, S, want_logits=True)
    lgb2, _ = eng.decode_step(tokb, S + 1, want_logits=True)
    for b in sorted(set(range(0, NB, 4)) | {NB - 1}):
        n = rows[b].shape[1]
        h1, lg1, _ = eng.prefill(rows[b], vf[b:b + 1], vid_start_of(rows[b], SMALL), want_hidden=True, want_logits=True)
        assert relerr(h[b:b + 1, pads[b]:], h1) < 1e-2, (b, relerr(h[b:b + 1, pads[b]:], h1))
        assert relerr(lg[b:b + 1], lg1) < 1e-2, (b, relerr(lg[b:b + 1], lg1))
        l1, _ = eng.decode_step(tok[b:b + 1].contiguous(), n, want_logits=True)
        assert relerr(l1, lgb[b:b + 1]) < 2e-2, (b, relerr(l1, lgb[b:b + 1]))
        l2, _ = eng.decode_step(tokb[b:b + 1].contiguous(), n + 1, want_logits=True)
        assert relerr(l2, lgb2[b:b + 1]) < 2e-2, (b, relerr(l2, lgb2[b:b + 1]))


@torch.no_grad()
def test_padded_batch_vs_oracle_clips_alone():
    """Width 2560, 2 layers, 4 clips: the padded batch, teacher-forced with the bf16 oracle's tokens of each clip
    run alone, follows the margin rule; the free-running padded generate (CUDA graph) gives each clip's own
    tokens up to the oracle's first near-tie."""
    cfg = O.LlmCfg(hidden=2560, inter=6912, heads=20, layers=2)
    sd_b = to_dev(O.random_llm_state(cfg, seed=5))
    n_new = 6
    ids, pads, rows = padded_batch(cfg, [63, 41, 50, 22], seed=60)
    B, S = ids.shape
    vf = video_feats(B, 11)
    o_toks, o_logits = [], []
    for b in range(B):
        t, lgs = O.greedy_generate(sd_b, cfg, rows[b], vf[b:b + 1].bfloat16(), n_new)
        o_toks.append(t); o_logits.append(lgs)
    o_toks = torch.cat(o_toks, 0)                       # [B, n_new]
    o_logits = torch.cat(o_logits, 1)                   # [n_new, B, V]
    eng = make_engine(llm=cfg, max_batch=B, max_seq=480)
    eng.load_llm(sd_b)
    vs = vid_start_of(ids, cfg)
    _, lg, tok = eng.prefill(ids, vf, vs, want_logits=True, n_pad=pads)
    check_margin_rule(tok, o_toks[:, 0], o_logits[0], "padded prefill")
    assert relerr(lg, o_logits[0]) < 3e-2
    for i in range(1, n_new):
        lg, tok = eng.decode_step(o_toks[:, i - 1].to(torch.int32).contiguous(), S + i - 1, want_logits=True)
        check_margin_rule(tok, o_toks[:, i], o_logits[i], f"padded decode step {i}")
        assert relerr(lg, o_logits[i]) < 3e-2, (i, relerr(lg, o_logits[i]))
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        gen = eng.generate(ids, vf, vs, n_new, n_pad=pads).long()
        alone = [eng.generate(rows[b], vf[b:b + 1], vid_start_of(rows[b], cfg), n_new).long() for b in range(B)]
    st.synchronize()
    for b, t in enumerate(first_near_tie(o_logits)):
        assert torch.equal(gen[b, :t], alone[b][0, :t]), (b, t, gen[b].tolist(), alone[b].tolist())
        assert torch.equal(gen[b, :t], o_toks[b, :t]), (b, t, gen[b].tolist(), o_toks[b].tolist())


@torch.no_grad()
def test_long_padded_prompts_flash_kernel_and_append():
    """S > 512 (the flash prefill kernel): a padded prefill matches the clips alone, and prefill_append after it
    continues each clip's positions as a padded prefill of the concatenated rows does."""
    ids, pads, rows = padded_batch(SMALL, [183, 123], seed=70)            # S = 568, clip 1 padded by 60
    B, S = ids.shape
    assert S > 512 and pads == [0, 60]
    n_new = 24
    extra = torch.randint(3, 32000, (B, n_new), generator=torch.Generator().manual_seed(5)).to(DEV)
    full = torch.cat([ids, extra], 1)
    vf = video_feats(B, 14)
    eng = make_engine(llm=SMALL, max_batch=B, max_seq=S + n_new + 8)
    eng.load_llm(to_dev(O.random_llm_state(SMALL, seed=31)))
    vs = vid_start_of(ids, SMALL)
    h, lg, _ = eng.prefill(ids, vf, vs, want_hidden=True, want_logits=True, n_pad=pads)
    assert torch.isfinite(h).all()
    for b in range(B):
        h1, lg1, _ = eng.prefill(rows[b], vf[b:b + 1], vid_start_of(rows[b], SMALL), want_hidden=True, want_logits=True)
        assert relerr(h[b:b + 1, pads[b]:], h1) < 1e-2, (b, relerr(h[b:b + 1, pads[b]:], h1))
        assert relerr(lg[b:b + 1], lg1) < 1e-2, (b, relerr(lg[b:b + 1], lg1))
    S1 = full.shape[1]
    h_full, lg_full, tok_full = eng.prefill(full, vf, vs, want_hidden=True, want_logits=True, n_pad=pads)
    lg_full2, _ = eng.decode_step(tok_full, S1, want_logits=True)
    eng.prefill(ids, vf, vs, n_pad=pads)
    h_new, lg_new, _ = eng.prefill_append(full[:, S:], S, want_hidden=True, want_logits=True)
    assert relerr(h_new, h_full[:, S:]) < 1e-2, relerr(h_new, h_full[:, S:])
    assert relerr(lg_new, lg_full) < 1e-2, relerr(lg_new, lg_full)
    lg_new2, _ = eng.decode_step(tok_full, S1, want_logits=True)
    assert relerr(lg_new2, lg_full2) < 1e-2, relerr(lg_new2, lg_full2)
    with pytest.raises(vn.VclError, match="left padding"):
        eng.prefill_append(full[:, S:], 60)                                # inside clip 1's padding


@torch.no_grad()
def test_padded_prefill_flash_variant_at_short_prompts(monkeypatch):
    """VCL_PREFILL_ATTN_FLASH=1 (read per call) sends a <= 512-key padded prefill to the flash kernel; it must
    agree with the wgmma kernel."""
    ids, pads, _ = padded_batch(SMALL, [63, 30, 47], seed=80)
    vf = video_feats(3, 15)
    eng = make_engine(llm=SMALL, max_batch=3, max_seq=480)
    eng.load_llm(to_dev(O.random_llm_state(SMALL, seed=21)))
    vs = vid_start_of(ids, SMALL)
    h, lg, _ = eng.prefill(ids, vf, vs, want_hidden=True, want_logits=True, n_pad=pads)
    monkeypatch.setenv("VCL_PREFILL_ATTN_FLASH", "1")
    hf, lgf, _ = eng.prefill(ids, vf, vs, want_hidden=True, want_logits=True, n_pad=pads)
    monkeypatch.delenv("VCL_PREFILL_ATTN_FLASH")
    assert torch.isfinite(hf).all()
    for b in range(3):
        assert relerr(hf[b, pads[b]:], h[b, pads[b]:]) < 1e-2, b
    assert relerr(lgf, lg) < 1e-2


@torch.no_grad()
def test_padding_state_does_not_leak_into_plain_runs():
    """A padded generate, then a plain generate with the same (B, n_new) on the same engine: both replay one decode
    graph, which reads the pad counts from the device, so the plain run must find them cleared (and the padded run
    after it set again) -- its tokens equal a fresh engine's."""
    sd = to_dev(O.random_llm_state(SMALL, seed=21))
    ids_p, pads, _ = padded_batch(SMALL, [63, 35, 50], seed=90)
    ids_u = O.make_prompt_ids(SMALL, 356, seed=91, batch=3).to(DEV)
    vf = video_feats(3, 16)
    eng = make_engine(llm=SMALL, max_batch=3, max_seq=480)
    eng.load_llm(sd)
    fresh = make_engine(llm=SMALL, max_batch=3, max_seq=480)
    fresh.load_llm(sd)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        gp = eng.generate(ids_p, vf, vid_start_of(ids_p, SMALL), 8, n_pad=pads)
        gu = eng.generate(ids_u, vf, vid_start_of(ids_u, SMALL), 8)
        gp2 = eng.generate(ids_p, vf, vid_start_of(ids_p, SMALL), 8, n_pad=pads)
        ref_u = fresh.generate(ids_u, vf, vid_start_of(ids_u, SMALL), 8)
        ref_p = fresh.generate(ids_p, vf, vid_start_of(ids_p, SMALL), 8, n_pad=pads)
    st.synchronize()
    assert torch.equal(gu, ref_u)
    assert torch.equal(gp, gp2) and torch.equal(gp, ref_p)
    # all-zero pad counts are no padding: exactly the plain path
    with torch.cuda.stream(st):
        gz = eng.generate(ids_u, vf, vid_start_of(ids_u, SMALL), 8, n_pad=[0, 0, 0])
    st.synchronize()
    assert torch.equal(gz, ref_u)


def test_bad_pad_counts_raise():
    eng = make_engine(llm=O.LlmCfg(hidden=512, inter=1024, heads=4, layers=1), max_batch=2, max_seq=64)
    eng.load_llm(to_dev(O.random_llm_state(O.LlmCfg(hidden=512, inter=1024, heads=4, layers=1), seed=1)))
    ids = torch.randint(3, 1000, (2, 8), device=DEV)
    vs = torch.full((2,), vn.NO_VIDEO, dtype=torch.int32, device=DEV)
    with pytest.raises(vn.VclError, match="n_pad"):
        eng.prefill(ids, None, vs, n_pad=[0, 8])                          # n_pad >= S: no real token
    with pytest.raises(vn.VclError, match="n_pad"):
        eng.prefill(ids, None, vs, n_pad=[-1, 0])
    with pytest.raises(vn.VclError, match="n_pad"):
        eng.generate(ids, None, vs, 4, n_pad=[9, 0])
    with pytest.raises(vn.VclError, match="entries"):
        eng.prefill(ids, None, vs, n_pad=[1])


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


@torch.no_grad()
def test_dropin_generate_with_attention_mask():
    """m.generate(left-padded ids, attention_mask=...) as with HF's LLaMA: [B, S+n] with the prompt included,
    each row's new tokens are that clip's own up to the oracle's first near-tie, an all-ones mask is the same
    as none, sampling and a continued turn run on the padded cache, right padding is rejected."""
    lsd = O.random_llm_state(SMALL, seed=23)
    m = _model(SMALL, max_batch=3)
    m.load_state_dict(lsd)
    ids, pads, rows = padded_batch(SMALL, [63, 40, 55], seed=100)
    B, S = ids.shape
    mask = torch.ones(B, S, dtype=torch.int64)
    for b in range(B):
        mask[b, :pads[b]] = 0
    feats = video_feats(B, 17).half()
    n = 6
    out = m.generate(ids, video_spatio_temporal_features=feats, attention_mask=mask, do_sample=False,
                     max_new_tokens=n)                                   # EOS-chunked device path
    assert out.shape == (B, S + n) and torch.equal(out[:, :S], ids)
    out_fixed = m.generate(ids, video_spatio_temporal_features=feats, attention_mask=mask.bool(), do_sample=False,
                           max_new_tokens=n, eos_token_id=None)          # one device loop
    assert torch.equal(out_fixed, out)
    sd_b = to_dev(lsd)
    for b in range(B):
        own = m.generate(rows[b], video_spatio_temporal_features=feats[b:b + 1], do_sample=False, max_new_tokens=n)
        _, o_logits = O.greedy_generate(sd_b, SMALL, rows[b], feats[b:b + 1].bfloat16(), n)
        t = first_near_tie(o_logits)[0]
        assert torch.equal(out[b, S:S + t], own[0, -n:][:t]), (b, t, out[b, S:].tolist(), own[0, -n:].tolist())
    # an all-ones mask is exactly no mask
    plain = O.make_prompt_ids(SMALL, 356, seed=101, batch=B).to(DEV)
    a = m.generate(plain, video_spatio_temporal_features=feats, max_new_tokens=n)
    b_ = m.generate(plain, video_spatio_temporal_features=feats, max_new_tokens=n,
                    attention_mask=torch.ones(B, plain.shape[1], dtype=torch.int64))
    assert torch.equal(a, b_)
    # sampling (the stepwise path, decode steps on the padded cache)
    smp = m.generate(ids, video_spatio_temporal_features=feats, attention_mask=mask, do_sample=True, temperature=0.7,
                     max_new_tokens=4, eos_token_id=None)
    assert smp.shape == (B, S + 4) and torch.equal(smp[:, :S], ids)
    # a continued turn appends to the padded cache: its first token is the arg-max of the padded context
    # prefilled from scratch wherever that arg-max is decided by >= 3 ulps
    m.generate(ids, video_spatio_temporal_features=feats, attention_mask=mask, max_new_tokens=3, eos_token_id=None)
    q2 = torch.randint(3, 32000, (B, 9), generator=torch.Generator().manual_seed(8)).to(DEV)
    turn2 = m.generate_continue(q2, max_new_tokens=2, eos_token_id=None)
    L = S + 3 + 9
    assert turn2.shape == (B, L + 2) and torch.equal(turn2[:, S + 3:L], q2)
    ctx_mask = torch.cat([mask, torch.ones(B, L - S, dtype=torch.int64)], 1)
    lg = m(input_ids=turn2[:, :L], attention_mask=ctx_mask, video_spatio_temporal_features=feats).logits[:, 0].float()
    margin, _, _ = margins_ulps(lg)
    for b in range(B):
        if margin[b] >= 3:
            assert int(turn2[b, L]) == int(lg[b].argmax()), (b, margin[b].item())
    # malformed masks fail before any device work
    right = torch.ones(B, S, dtype=torch.int64); right[0, -3:] = 0
    with pytest.raises(ValueError, match="left padding"):
        m.generate(ids, video_spatio_temporal_features=feats, attention_mask=right, max_new_tokens=2)
    with pytest.raises(NotImplementedError, match="output_hidden_states"):
        m(input_ids=ids, attention_mask=mask, video_spatio_temporal_features=feats, output_hidden_states=True)
