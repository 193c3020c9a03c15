"""Scoring on the GPU: the cross-entropy kernel (vcl_op_cross_entropy) against torch on the same bf16 logits, and
vcl_llm_score / forward(labels=...) end to end against the bf16 oracle's llm_forward(all_logits=True) + torch's
cross-entropy, with the suite's norm-wise bars (relerr < 3e-2 against the bf16 oracle, _util.bar against the fp32
gold). Labels are training style: -100 on the prompt and the video span, real ids on the 26-token answer."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import bar, make_engine, relerr, to_dev, vid_start_of  # noqa: E402

DEV = "cuda"
V = 32003
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)
N_ANSWER = 26


def bf16_ulp(x):
    """spacing of bf16 at |x| (fp32 tensor)"""
    a = x.abs().clamp_min(2 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def answer_labels(ids):
    """-100 everywhere but the last N_ANSWER columns, which carry the ids themselves"""
    lab = torch.full_like(ids, -100)
    lab[:, -N_ANSWER:] = ids[:, -N_ANSWER:]
    return lab


def video_feats(B, seed):
    return (torch.randn(B, 356, 1024, generator=torch.Generator().manual_seed(seed)) * 0.5).half().float().to(DEV)


def torch_nll(logits, labels):
    """the reference's loss path on bf16 logits [B,S,V]: shifted per-token NLL (bf16 -> fp32) and the mean"""
    lg = logits[:, :-1].reshape(-1, logits.shape[-1])
    t = labels[:, 1:].reshape(-1).to(lg.device)
    nll = F.cross_entropy(lg, t, reduction="none").float().view(labels.shape[0], -1)
    return nll, F.cross_entropy(lg, t)


# ------------------------------------------------------------------------------------------
@torch.no_grad()
def test_op_cross_entropy_matches_torch():
    rows, ld = 96, 32008
    g = torch.Generator(device=DEV).manual_seed(3)
    x = torch.randn(rows, ld, device=DEV, generator=g) * 3
    x[:8] = x[:8] * 25 + 60                          # logits of 60 and more in magnitude
    x[8:12] = -x[8:12].abs() * 25 - 60
    x[12, 17] = 90.0                                 # one dominant logit: probability ~1 at its label
    xb = x.to(torch.bfloat16)
    lab = torch.randint(0, V, (rows,), device=DEV, generator=g)
    lab[0], lab[1], lab[2], lab[12] = 0, V - 1, -100, 17
    lab[20:30] = -100
    nll, loss = vn.op_cross_entropy(xb, lab, V=V)
    torch.cuda.synchronize()
    xv = xb[:, :V]
    counted = lab != -100
    ref = -torch.log_softmax(xv.float(), -1).bfloat16().float()
    ref = ref.gather(1, lab.clamp_min(0)[:, None])[:, 0]
    tol = torch.maximum(bf16_ulp(ref), bf16_ulp(nll))
    assert ((nll - ref).abs()[counted] <= tol[counted]).all(), (nll - ref).abs()[counted].max().item()
    assert (nll[~counted] == 0).all()
    ref_loss = F.cross_entropy(xv, lab).float()
    assert (loss.bfloat16().float() - ref_loss).abs() <= bf16_ulp(ref_loss), (loss.item(), ref_loss.item())
    mean64 = nll.double()[counted].mean()
    assert abs(loss.double().item() - mean64.item()) <= 1e-6 * abs(mean64.item())
    # bit-identical from run to run
    nll2, loss2 = vn.op_cross_entropy(xb, lab, V=V)
    assert torch.equal(nll, nll2) and torch.equal(loss, loss2)
    # everything ignored: NaN loss, as torch; an out-of-range label: a NaN row, the others unchanged
    nll_i, loss_i = vn.op_cross_entropy(xb, torch.full_like(lab, -100), V=V)
    assert torch.isnan(loss_i) and (nll_i == 0).all()
    bad = lab.clone(); bad[5], bad[6], bad[7] = V, -5, 1 << 40
    nll_b, loss_b = vn.op_cross_entropy(xb, bad, V=V)
    assert torch.isnan(nll_b[5:8]).all() and torch.isnan(loss_b)
    keep = torch.ones(rows, dtype=torch.bool, device=DEV); keep[5:8] = False
    assert torch.equal(nll_b[keep], nll[keep])


def _score_vs_oracle(cfg, B, seed):
    sd = O.random_llm_state(cfg, seed=seed)
    sd_b, sd_f = to_dev(sd), to_dev(sd, torch.float32)
    ids = O.make_prompt_ids(cfg, 356, seed=seed, batch=B).to(DEV)
    lab = answer_labels(ids)
    vf = video_feats(B, seed)
    eng = make_engine(llm=cfg, max_batch=B, max_seq=480)
    eng.load_llm(sd_b)
    vs = vid_start_of(ids, cfg)
    logits, nll, loss = eng.score(ids, vf, vs, labels=lab, want_logits=True)
    o_logits, _, _ = O.llm_forward(sd_b, cfg, ids, vf.bfloat16(), all_logits=True)
    g_logits, _, _ = O.llm_forward(sd_f, cfg, ids, vf, all_logits=True)
    o_nll, o_loss = torch_nll(o_logits, lab)
    g_nll, g_loss = torch_nll(g_logits, lab)
    ans = lab[:, 1:] != -100
    assert logits.shape == (B, 448, V) and nll.shape == (B, 447) and loss.dim() == 0
    assert (nll[~ans] == 0).all()
    assert relerr(logits, o_logits) < 3e-2, relerr(logits, o_logits)
    bar(logits, o_logits, g_logits, f"width {cfg.hidden}: all-position logits")
    assert relerr(nll[ans], o_nll[ans]) < 3e-2, relerr(nll[ans], o_nll[ans])
    bar(nll[ans], o_nll[ans], g_nll[ans], f"width {cfg.hidden}: per-token NLL")
    assert relerr(loss, o_loss) < 3e-2, (loss.item(), o_loss.item())
    bar(loss.reshape(1), o_loss.reshape(1), g_loss.reshape(1), f"width {cfg.hidden}: loss")
    return eng, ids, vf, vs, lab, logits, nll, loss


@torch.no_grad()
def test_score_small_width_vs_oracle_and_consistency():
    """hidden 512: the lm_head chunks (45 rows at max_batch 2 x max_seq 480) do not divide B*S = 896"""
    eng, ids, vf, vs, lab, logits, nll, loss = _score_vs_oracle(SMALL, 2, seed=21)
    B, S = ids.shape
    assert (B * S) % 45 != 0
    # column S-1 against the prefill's last-position logits (GEMV path)
    _, last, _ = eng.prefill(ids, vf, vs, want_logits=True)
    col = logits[:, -1].float()
    assert relerr(col, last) < 1e-2, relerr(col, last)
    top = torch.topk(last, 2, dim=-1)
    margin = (top.values[:, 0] - top.values[:, 1]) / (top.values[:, 0].abs().clamp_min(2 ** -6) * 2 ** -7)
    for b in range(B):
        if margin[b] >= 3:
            assert int(col[b].argmax()) == int(last[b].argmax()), (b, margin[b].item())
    # the cache after a scoring call is the prefill's: the next decode step is identical
    tok = last.argmax(-1).to(torch.int32)
    after_prefill, _ = eng.decode_step(tok, S, want_logits=True)
    eng.score(ids, vf, vs, labels=lab)
    after_score, _ = eng.decode_step(tok, S, want_logits=True)
    assert torch.equal(after_score, after_prefill)
    # logits only (no labels), and the same call twice: bit-identical
    lg2, nll2, loss2 = eng.score(ids, vf, vs, want_logits=True)
    assert nll2 is None and loss2 is None and torch.equal(lg2, logits)
    _, nll3, loss3 = eng.score(ids, vf, vs, labels=lab)
    assert torch.equal(nll3, nll) and torch.equal(loss3, loss)


@torch.no_grad()
def test_score_width_2560_vs_oracle():
    _score_vs_oracle(O.LlmCfg(hidden=2560, inter=6912, heads=20, layers=2), 1, seed=5)


def padded_rows(cfg, n_pres, seed):
    rows = [O.make_prompt_ids(cfg, 356, seed=seed + b, n_pre=n)[0] for b, n in enumerate(n_pres)]
    return [r[None].to(DEV) for r in rows]


@torch.no_grad()
def test_left_padded_batch_matches_clips_scored_alone():
    rows = padded_rows(SMALL, [63, 40, 51], seed=50)
    S = max(r.shape[1] for r in rows)
    B = len(rows)
    pads = [S - r.shape[1] for r in rows]
    ids = torch.zeros(B, S, dtype=torch.int64, device=DEV)
    for b, r in enumerate(rows):
        ids[b, pads[b]:] = r[0]
    lab = answer_labels(ids)
    vf = video_feats(B, 13)
    eng = make_engine(llm=SMALL, max_batch=B, max_seq=480)
    eng.load_llm(to_dev(O.random_llm_state(SMALL, seed=21)))
    _, nll, loss = eng.score(ids, vf, vid_start_of(ids, SMALL), labels=lab, n_pad=pads)
    alone = []
    for b, r in enumerate(rows):
        _, n1, _ = eng.score(r, vf[b:b + 1], vid_start_of(r, SMALL), labels=answer_labels(r))
        assert relerr(nll[b:b + 1, pads[b]:], n1) < 1e-2, (b, relerr(nll[b:b + 1, pads[b]:], n1))
        alone.append(n1[0, -N_ANSWER:])
    assert relerr(loss, torch.cat(alone).double().mean()) < 1e-2


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
def test_dropin_forward_with_labels_and_collator_padding():
    """forward(labels=...) as the reference: a 0-d bf16 loss and [B,S,V] logits; logits_to_keep=0 gives the same
    logits without a loss; a right-padded, collator-style batch gives each row's own per-token NLL and loss; the
    default call still returns [B,1,V]."""
    lsd = O.random_llm_state(SMALL, seed=23)
    m = _model(SMALL, max_batch=3)
    m.load_state_dict(lsd)
    rows = padded_rows(SMALL, [63, 44, 55], seed=110)
    B, S = len(rows), max(r.shape[1] for r in rows)
    ids = torch.zeros(B, S, dtype=torch.int64)                   # pad_sequence(batch_first=True), pad id 0
    lab = torch.full((B, S), -100, dtype=torch.int64)
    for b, r in enumerate(rows):
        n = r.shape[1]
        ids[b, :n] = r[0].cpu()
        lab[b, n - N_ANSWER:n] = r[0, -N_ANSWER:].cpu()
    mask = ids.ne(0)
    feats = video_feats(B, 19).half()
    out = m(input_ids=ids, attention_mask=mask, labels=lab, video_spatio_temporal_features=feats)
    assert out.loss.dtype == torch.bfloat16 and out.loss.dim() == 0
    assert out.logits.shape == (B, S, V) and out.logits.dtype == torch.bfloat16
    # a right-padded mask with labels runs the unpadded batch; logits_to_keep=0 (no labels) accepts left padding
    # only, as forward without labels does, so it is compared on the same unpadded call
    keep0 = m(input_ids=ids, logits_to_keep=0, video_spatio_temporal_features=feats)
    assert keep0.loss is None and torch.equal(keep0.logits, out.logits)
    with pytest.raises(ValueError, match="left padding"):
        m(input_ids=ids, attention_mask=mask, logits_to_keep=0, video_spatio_temporal_features=feats)
    eng = m._ensure_engine(need_llm=True)
    ids_d = ids.to(DEV)
    _, nll, loss = eng.score(ids_d, feats, vid_start_of(ids_d, SMALL), labels=lab.to(DEV))
    assert torch.equal(out.loss, loss.to(torch.bfloat16))
    for b, r in enumerate(rows):
        n = r.shape[1]
        lab1 = lab[b:b + 1, :n].to(DEV)
        _, n1, _ = eng.score(r, feats[b:b + 1], vid_start_of(r, SMALL), labels=lab1)
        assert relerr(nll[b:b + 1, :n - 1], n1) < 1e-2, (b, relerr(nll[b:b + 1, :n - 1], n1))
        assert (nll[b, n - 1:] == 0).all()
    assert m(input_ids=ids, video_spatio_temporal_features=feats).logits.shape == (B, 1, V)
