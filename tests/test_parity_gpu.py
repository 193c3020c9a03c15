"""End-to-end parity on the GPU, through the C ABI (vcl_native -> libvcl.so):

  * against the committed golden fixtures (outputs of the reference itself, fp32 on CPU), and
  * against the oracle run on the same GPU in bf16 ("the reference's own PyTorch path on identical
    inputs") and in fp32 (gold).

Tolerances. The model dtype is bf16 (2^-8 spacing), so two correct bf16 implementations differ by
more than the north star's 1e-3 element-wise; parity is therefore graded norm-wise against the
fp32 gold, and the bar is: our error is no larger than the bf16 oracle's own error against the same
gold (x1.3 + 1e-3 slack). Token ids are checked teacher-forced against the bf16 oracle: identical
arg-max wherever the oracle's top-1/top-2 margin is >= 3 bf16 ulps, top-2 membership otherwise
(SURVEY.md section 7, "hard parts").
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import bar as _bar, make_engine, relerr, teacher_forced_check as _teacher_forced_check, to_dev, vid_start_of  # noqa: E402

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = "cuda"


# ------------------------------------------------------------------------------------------
# CLIP
# ------------------------------------------------------------------------------------------
@torch.no_grad()
def test_clip_tiny_vs_golden_and_oracle():
    g = np.load(os.path.join(G, "clip_tiny.npz"))
    cfg = O.ClipCfg(hidden=1024, inter=1024, heads=16, layers=3)
    sd = O.random_clip_state(cfg, seed=11)
    px = O.preprocess_frames(O.make_frames(7, 3)).to(DEV)
    eng = make_engine(clip=cfg, clip_run_layers=2, max_frames=4)
    eng.load_clip(to_dev(sd))
    gold = O.clip_hidden_states(to_dev(sd, torch.float32), cfg, px, 2)
    refb = O.clip_hidden_states(to_dev(sd), cfg, px.bfloat16(), 2)
    for i in range(3):
        h = eng.clip_encode(px.bfloat16(), n_layers=i)
        assert h.shape == (3, 257, 1024)
        # golden fixture (fp32 reference on CPU): slices and per-row norms
        e = relerr(h[:, :6, :96], torch.as_tensor(g[f"h{i}_slice"]))
        assert e < 2e-2, (i, e)
        en = relerr(h.float().norm(dim=-1), torch.as_tensor(g[f"h{i}_rownorm"]))
        assert en < 5e-3, (i, en)
        _bar(h, refb[i], gold[i], f"clip_tiny hidden_states[{i}]")


@torch.no_grad()
def test_clip_uint8_path_matches_bf16_path():
    """next-row (f1): raw uint8 NHWC frames normalised on device == CPU-preprocessed pixels, bit for bit (the
    device normalisation rounds to the same bf16 as preprocess_frames for every value and channel:
    test_vision_kernels_gpu.test_im2col)"""
    cfg = O.ClipCfg(hidden=1024, inter=1024, heads=16, layers=3)
    sd = O.random_clip_state(cfg, seed=11)
    frames = O.make_frames(3, 5)
    eng = make_engine(clip=cfg, clip_run_layers=2, max_frames=8)
    eng.load_clip(to_dev(sd))
    a = eng.clip_encode(O.preprocess_frames(frames).to(DEV).bfloat16())
    b = eng.clip_encode(torch.as_tensor(frames).to(DEV))
    assert torch.equal(b, a), relerr(b, a)


@torch.no_grad()
def test_config1_full_vit_pooled_vs_golden():
    """BASELINE config 1: 8 frames through the full 23-layer ViT-L/14 + pool -> [356,1024] fp16."""
    g = np.load(os.path.join(G, "config1.npz"))
    cfg = O.ClipCfg()
    sd = O.random_clip_state(cfg, seed=0, n_layers=23)
    frames = np.random.default_rng(0).integers(0, 256, (8, 224, 224, 3), dtype=np.uint8)
    px = O.preprocess_frames(frames).to(DEV)
    eng = make_engine(clip=cfg, max_frames=8)
    eng.load_clip(to_dev(sd))
    pooled = eng.clip_features(px.bfloat16(), torch.float16)
    assert pooled.shape == (356, 1024) and pooled.dtype == torch.float16
    assert (pooled[8:100] == 0).all()
    hid = eng.clip_encode(px.bfloat16())
    # pooling of our own hidden state through the stateless op == fused call (bit-exact)
    assert torch.equal(vn.st_pool(hid[:, 1:], 100, torch.float16), pooled)
    refb = O.clip_hidden_states(to_dev(sd), cfg, px.bfloat16())[-1]
    gold_pooled = torch.as_tensor(g["pooled"])
    _bar(pooled, O.st_pool_torch(refb[:, 1:]), gold_pooled, "config1 pooled features")
    e = relerr(hid.float().norm(dim=-1), torch.as_tensor(g["penult_rownorm"]))
    assert e < 1e-2, e


# ------------------------------------------------------------------------------------------
# LLM
# ------------------------------------------------------------------------------------------
@torch.no_grad()
def test_llm_tiny_vs_golden_and_oracle():
    g = np.load(os.path.join(G, "llm_tiny.npz"))
    cfg = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)
    sd = O.random_llm_state(cfg, seed=21)
    ids = O.make_prompt_ids(cfg, 356, seed=1, batch=2).to(DEV)
    gf = torch.Generator().manual_seed(9)
    vf = (torch.randn(2, 356, 1024, generator=gf) * 0.5).half().float().to(DEV)
    eng = make_engine(llm=cfg, max_batch=2, max_seq=480)
    eng.load_llm(to_dev(sd))
    sd_b, sd_f = to_dev(sd), to_dev(sd, torch.float32)
    _, gold_hs, _ = O.llm_forward(sd_f, cfg, ids, vf)
    _, refb_hs, _ = O.llm_forward(sd_b, cfg, ids, vf.bfloat16())
    vs = vid_start_of(ids, cfg)
    assert vs.tolist() == [64, 64]
    for nl in range(3):
        h, _, _ = eng.prefill(ids, vf, vs, n_layers=nl, want_hidden=True, want_token=False)
        if nl == 0:
            # spliced input embeddings: the video rows are mm_projector(features), the rest a gather
            assert relerr(h[:, 60:72], torch.as_tensor(g["h0_rows"])) < 4e-3
            assert torch.equal(h[:, :65], refb_hs[0][:, :65])            # pure gather: bit-exact
            assert torch.equal(h[:, 421:], refb_hs[0][:, 421:])
        if nl < 2:
            assert relerr(h.float().norm(dim=-1), torch.as_tensor(g[f"h{nl}_rownorm"])) < 5e-3
            _bar(h, refb_hs[nl], gold_hs[nl], f"llm_tiny hidden_states[{nl}]")
    _, lg, tok = eng.prefill(ids, vf, vs, want_logits=True)
    assert relerr(lg, torch.as_tensor(g["logits_last"])) < 2e-2
    _teacher_forced_check(eng, sd_b, cfg, ids, vf, 8, "llm_tiny")
    # full generate call (CUDA-graph decode loop) == step-by-step free-running decode
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        gen = eng.generate(ids, vf, vs, 8)
    st.synchronize()
    _, _, t = eng.prefill(ids, vf, vs)
    seq = [t.clone()]
    for i in range(1, 8):
        _, t = eng.decode_step(seq[-1], 448 + i - 1)
        seq.append(t.clone())
    assert torch.equal(gen, torch.stack(seq, 1))


@torch.no_grad()
def test_llm_7b_width_two_layers():
    """Vicuna-7B shapes (D 4096, F 11008, 32 heads, V 32003) at 2 layers, S = 448, B = 1."""
    cfg = O.LlmCfg(layers=2)
    sd = O.random_llm_state(cfg, seed=3)
    ids = O.make_prompt_ids(cfg, 356, seed=1, batch=1).to(DEV)
    gf = torch.Generator().manual_seed(10)
    vf = (torch.randn(1, 356, 1024, generator=gf) * 0.5).half().float().to(DEV)
    eng = make_engine(llm=cfg, max_batch=1, max_seq=480)
    sd_b = to_dev(sd)
    eng.load_llm(sd_b)
    sd_f = to_dev(sd, torch.float32)
    _, gold_hs, _ = O.llm_forward(sd_f, cfg, ids, vf)
    del sd_f
    _, refb_hs, _ = O.llm_forward(sd_b, cfg, ids, vf.bfloat16())
    vs = vid_start_of(ids, cfg)
    for nl in (0, 1, 2):
        h, _, _ = eng.prefill(ids, vf, vs, n_layers=nl, want_hidden=True, want_token=False)
        ref = refb_hs[nl] if nl < 2 else None
        if ref is not None:
            _bar(h, ref, gold_hs[nl], f"7B-width hidden_states[{nl}]")
    _teacher_forced_check(eng, sd_b, cfg, ids, vf, 8, "7B-width x2 layers")


@torch.no_grad()
@pytest.mark.parametrize("NB", [3, 9, 17])
def test_decode_batch_paths_agree(NB):
    """Batched decode (1..4 clips: gemv_tc, 5..16: gemv_tcw, > 16: wgmma GEMM with a narrow N tile; at this
    width every ring-kernel CTA owns a single row group) must reproduce, per clip, what the clip gets when
    decoded alone through the single-clip path (clips are independent)."""
    cfg = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)
    sd = O.random_llm_state(cfg, seed=21)
    ids = O.make_prompt_ids(cfg, 356, seed=4, batch=NB).to(DEV)
    gf = torch.Generator().manual_seed(12)
    vf = (torch.randn(NB, 356, 1024, generator=gf) * 0.5).half().float().to(DEV)
    eng = make_engine(llm=cfg, max_batch=NB, max_seq=480)
    eng.load_llm(to_dev(sd))
    vs = vid_start_of(ids, cfg)
    _, lg5, _ = eng.prefill(ids, vf, vs, want_logits=True)
    tok = lg5.argmax(-1).to(torch.int32)
    lg5b, _ = eng.decode_step(tok, 448, want_logits=True)
    for b in range(0, NB, 4):
        _, lg1, _ = eng.prefill(ids[b:b + 1], vf[b:b + 1], vs[b:b + 1], want_logits=True)
        assert relerr(lg1, lg5[b:b + 1]) < 1e-2
        lg1b, _ = eng.decode_step(tok[b:b + 1].contiguous(), 448, want_logits=True)
        assert relerr(lg1b, lg5b[b:b + 1]) < 2e-2


def test_error_behaviour():
    """Bad arguments fail loudly with a message (no silent fallback)."""
    cfg = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=1)
    eng = make_engine(llm=cfg, max_batch=1, max_seq=64)
    ids = torch.zeros(1, 8, dtype=torch.int64, device=DEV)
    vs = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    with pytest.raises(vn.VclError, match="not loaded"):
        eng.prefill(ids, None, vs)
    with pytest.raises(vn.VclError, match="T=101"):
        vn.st_pool(torch.zeros(101, 4, 8, device=DEV, dtype=torch.float16))
    with pytest.raises(vn.VclError, match="down_proj.*14336"):       # no decode kernel streams K > 14336
        make_engine(llm=O.LlmCfg(hidden=512, inter=16384, heads=4, layers=1), max_batch=1, max_seq=64)


@torch.no_grad()
def test_336px_mlp2x_variant_end_to_end():
    """SURVEY.md 8f row 2 (LLaVA-1.5 style checkpoints): 336-px tower (P = 576, S = 577, so the ViT
    attention takes the flash-style kernel), 676 video tokens, mlp2x_gelu projector."""
    ccfg = O.ClipCfg(hidden=1024, inter=1024, heads=16, layers=3, image=336)
    lcfg = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2, proj_type="mlp2x_gelu")
    csd, lsd = O.random_clip_state(ccfg, seed=5), O.random_llm_state(lcfg, seed=6)
    frames = O.make_frames(11, 4, size=336)
    px = O.preprocess_frames(frames).to(DEV)
    eng = make_engine(clip=ccfg, llm=lcfg, clip_run_layers=2, max_frames=4, max_batch=1, max_seq=800)
    eng.load_clip(to_dev(csd))
    eng.load_llm(to_dev(lsd))
    assert eng.P == 576 and eng.NV == 676
    hid = eng.clip_encode(px.bfloat16())
    assert hid.shape == (4, 577, 1024)
    gold = O.clip_hidden_states(to_dev(csd, torch.float32), ccfg, px, 2)[-1]
    refb = O.clip_hidden_states(to_dev(csd), ccfg, px.bfloat16(), 2)[-1]
    _bar(hid, refb, gold, "336px ViT hidden_states[2]")
    feats = eng.clip_features(torch.as_tensor(frames).to(DEV), torch.float16)      # uint8 path
    assert feats.shape == (676, 1024) and (feats[4:100] == 0).all()
    _bar(feats, O.st_pool_torch(refb[:, 1:]), O.st_pool_torch(gold[:, 1:]), "336px pooled features")
    ids = O.make_prompt_ids(lcfg, 676, seed=2).to(DEV)
    assert ids.shape == (1, 768)
    vf = feats[None].float()
    sd_b, sd_f = to_dev(lsd), to_dev(lsd, torch.float32)
    _, gold_hs, _ = O.llm_forward(sd_f, lcfg, ids, vf)
    _, refb_hs, _ = O.llm_forward(sd_b, lcfg, ids, vf.bfloat16())
    vs = vid_start_of(ids, lcfg)
    h0, _, _ = eng.prefill(ids, vf, vs, n_layers=0, want_hidden=True, want_token=False)
    _bar(h0[:, 65:741], refb_hs[0][:, 65:741], gold_hs[0][:, 65:741], "mlp2x_gelu projector rows")
    h1, _, _ = eng.prefill(ids, vf, vs, n_layers=1, want_hidden=True, want_token=False)
    _bar(h1, refb_hs[1], gold_hs[1], "336px llm hidden_states[1]")
    _teacher_forced_check(eng, sd_b, lcfg, ids, vf, 6, "336px / mlp2x_gelu")


@torch.no_grad()
def test_single_clip_decode_vs_oracle():
    """Single-clip decode at width 2560 (every CTA of the ring kernel owns several row groups), with the
    embedding gather fused into layer 0's q|k|v launch, teacher-forced against the bf16 oracle."""
    cfg = O.LlmCfg(hidden=2560, inter=6912, heads=20, layers=2)
    sd = O.random_llm_state(cfg, seed=5)
    ids = O.make_prompt_ids(cfg, 356, seed=2, batch=1).to(DEV)
    vf = (torch.randn(1, 356, 1024, generator=torch.Generator().manual_seed(11)) * 0.5).half().float().to(DEV)
    eng = make_engine(llm=cfg, max_batch=1, max_seq=480)
    sd_b = to_dev(sd)
    eng.load_llm(sd_b)
    _teacher_forced_check(eng, sd_b, cfg, ids, vf, 4, "width-2560 x2 layers B=1 (gemv_tc)")


@torch.no_grad()
@pytest.mark.parametrize("NB", [2, 4])
def test_decode_small_batch_ring_kernel(NB):
    """2..4 clips (width 2560) go through the multi-column gemv_tc kernel (activation vectors of all
    clips in shared memory, one MMA column per clip): per clip it must reproduce the single-clip
    decode (same weights, same summation order; the caches come from differently tiled prefills)."""
    cfg = O.LlmCfg(hidden=2560, inter=6912, heads=20, layers=2)   # every projection >= 132 row groups (one per SM): ring kernel
    sd = O.random_llm_state(cfg, seed=8)
    ids = O.make_prompt_ids(cfg, 356, seed=6, batch=NB).to(DEV)
    vf = (torch.randn(NB, 356, 1024, generator=torch.Generator().manual_seed(13)) * 0.5).half().float().to(DEV)
    eng = make_engine(llm=cfg, max_batch=NB, max_seq=480)
    eng.load_llm(to_dev(sd))
    vs = vid_start_of(ids, cfg)
    _, lg, _ = eng.prefill(ids, vf, vs, want_logits=True)
    tok = lg.argmax(-1).to(torch.int32)
    lgb, tokb = eng.decode_step(tok, 448, want_logits=True)
    lgb2, _ = eng.decode_step(tokb, 449, want_logits=True)
    for b in range(NB):
        eng.prefill(ids[b:b + 1], vf[b:b + 1], vs[b:b + 1])
        l1, t1 = eng.decode_step(tok[b:b + 1].contiguous(), 448, want_logits=True)
        assert relerr(l1, lgb[b:b + 1]) < 1e-2, (b, relerr(l1, lgb[b:b + 1]))
        l2, _ = eng.decode_step(tokb[b:b + 1].contiguous(), 449, want_logits=True)
        assert relerr(l2, lgb2[b:b + 1]) < 1e-2, (b, relerr(l2, lgb2[b:b + 1]))


@torch.no_grad()
@pytest.mark.parametrize("B,n_new", [(1, 24), (2, 70)])
def test_prefill_append_matches_full_prefill(B, n_new):
    """Multi-turn reuse of the KV cache (vcl_llm_prefill_append): prefilling a prompt and then appending
    n_new more tokens must give the hidden states / logits of prefilling everything at once (same
    arithmetic; the GEMM tiles differ, hence bf16 noise), and decoding continues identically."""
    cfg = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)
    sd = O.random_llm_state(cfg, seed=31)
    ids = O.make_prompt_ids(cfg, 356, seed=9, batch=B)
    extra = torch.randint(3, 32000, (B, n_new), generator=torch.Generator().manual_seed(5))
    full = torch.cat([ids, extra], 1).to(DEV)
    ids = ids.to(DEV)
    vf = (torch.randn(B, 356, 1024, generator=torch.Generator().manual_seed(14)) * 0.5).half().float().to(DEV)
    eng = make_engine(llm=cfg, max_batch=B, max_seq=448 + n_new + 8)
    eng.load_llm(to_dev(sd))
    vs = vid_start_of(ids, cfg)
    S0, S1 = ids.shape[1], full.shape[1]
    h_full, lg_full, tok_full = eng.prefill(full, vf, vs, want_hidden=True, want_logits=True)
    lg_full2, _ = eng.decode_step(tok_full, S1, want_logits=True)
    eng.prefill(ids, vf, vs)
    h_new, lg_new, tok_new = eng.prefill_append(full[:, S0:], S0, want_hidden=True, want_logits=True)
    assert relerr(h_new, h_full[:, S0:]) < 1e-2, relerr(h_new, h_full[:, S0:])
    assert relerr(lg_new, lg_full) < 1e-2, relerr(lg_new, lg_full)
    lg_new2, _ = eng.decode_step(tok_full, S1, want_logits=True)     # teacher-forced with the same token
    assert relerr(lg_new2, lg_full2) < 1e-2, relerr(lg_new2, lg_full2)
    with pytest.raises(vn.VclError):
        eng.prefill_append(full[:, S0:], 0)                           # a continuation needs a cache
    with pytest.raises(vn.VclError):
        eng.prefill_append(full[:, S0:], 448 + 9)                     # would run past max_seq


@torch.no_grad()
@pytest.mark.parametrize("NB", [5, 9, 16])
def test_decode_wide_ring_kernel(NB):
    """5..16 clips (width 2560) go through gemv_tcw (chunk-major walk over the slot-ordered weights, a warp
    per row group, clip b = MMA column b): per clip it must reproduce the single-clip ring-kernel decode
    (same weights, fp32 accumulation over the same products in another order -> bf16 noise), two steps deep."""
    cfg = O.LlmCfg(hidden=2560, inter=6912, heads=20, layers=2)
    sd = O.random_llm_state(cfg, seed=8)
    ids = O.make_prompt_ids(cfg, 356, seed=6, batch=NB).to(DEV)
    vf = (torch.randn(NB, 356, 1024, generator=torch.Generator().manual_seed(13)) * 0.5).half().float().to(DEV)
    eng = make_engine(llm=cfg, max_batch=NB, max_seq=480)
    sd_b = to_dev(sd)
    eng.load_llm(sd_b)
    vs = vid_start_of(ids, cfg)
    _, lg, _ = eng.prefill(ids, vf, vs, want_logits=True)
    tok = lg.argmax(-1).to(torch.int32)
    lgb, tokb = eng.decode_step(tok, 448, want_logits=True)
    lgb2, _ = eng.decode_step(tokb, 449, want_logits=True)
    assert torch.equal(tokb.long(), lgb.argmax(-1))
    for b in sorted({0, NB // 2, NB - 1}):
        eng.prefill(ids[b:b + 1], vf[b:b + 1], vs[b:b + 1])
        l1, t1 = eng.decode_step(tok[b:b + 1].contiguous(), 448, want_logits=True)
        assert relerr(l1, lgb[b:b + 1]) < 1e-2, (b, relerr(l1, lgb[b:b + 1]))
        l2, _ = eng.decode_step(tokb[b:b + 1].contiguous(), 449, want_logits=True)
        assert relerr(l2, lgb2[b:b + 1]) < 1e-2, (b, relerr(l2, lgb2[b:b + 1]))
    _teacher_forced_check(eng, sd_b, cfg, ids, vf, 6, f"width-2560 x2 layers B={NB} (gemv_tcw)")
