"""Banned tokens on the GPU (sampling.cu's ban stage, vcl_llm_set_bans, token histories).

Bars:
- the kernel: vcl_op_sample_bans returns the tokens and log-probs vcl_op_sample_ex returns on the same rows with the
  banned ids of _bans_ref.py set to -inf on the host, bit for bit, over V, B, T, top-k, top-p, the penalty and every
  combination of the three settings (a row with every token banned included), and writes its token into the history;
- histories read back after generate (plain and left-padded), generate_continue, a session's two turns and a chunked
  prompt equal the returned sequence;
- end to end on bf16 and fp8 engines, greedy and seeded T = 0.7: no new token completes an n-gram seen earlier in its
  row or a bad word, and no EOS comes before min_new_tokens; greedy, teacher-forced on the engine's own scored logits
  with HF's processors applied on the host, picks HF's token at every step whose top-2 gap exceeds 3 bf16 ulps;
- in flight: a banning request returns what generate returns for it alone, across slots, admission modes, paging
  and preemption; a default call after a banning one equals a fresh engine's, with the same launch count.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
import _bans_ref as BR  # noqa: E402
import _sampling_ref as R  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import to_dev  # noqa: E402
from test_padded_batch_gpu import video_feats  # noqa: E402
from test_inflight_gpu import _requests  # noqa: E402
from test_nucleus_gpu import SMALL, _bits, _flat_model, _gen, _model_at, _run_requests  # noqa: E402

DEV = "cuda"
EOS = 2
WORDS = [[5], [7, 8], [9, 10, 11], [EOS], [3, 4, 5, 6]]


def _same(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


@torch.no_grad()
@pytest.mark.parametrize("V", [32003, 1000])
@pytest.mark.parametrize("B", [1, 16, 64])
def test_kernel_equals_sample_ex_on_banned_rows(V, B):
    rng = np.random.default_rng(V + B)
    g = torch.Generator().manual_seed(V * 7 + B)
    x = (torch.randn(B, V, generator=g) * torch.tensor(rng.choice([1.0, 4.0], B))[:, None].float()).bfloat16().float()
    hist_ld = 2049
    hist = np.zeros((B, hist_ld), dtype=np.int32)
    T, k, p, r, ng, eos, frm, words, cols = [], [], [], [], [], [], [], [], []
    for b in range(B):
        combo = b % 8                                    # every combination of the three settings
        c = int(rng.integers(1, hist_ld))
        alpha = int(rng.choice([6, 40, V]))
        h = rng.integers(0, alpha, c)
        hist[b, :c] = h
        T.append(float(rng.choice([0.0, 0.2, 1.5])))
        k.append(int(rng.choice([0, 50])))
        p.append(float(rng.choice([1.0, 0.9])))
        r.append(float(rng.choice([1.0, 1.3])))
        ng.append(int(rng.integers(1, 6)) if combo & 1 else 0)
        words.append(WORDS + [h[-3:].tolist()] if combo & 2 else [])
        eos.append(EOS if combo & 4 else -1)
        frm.append(c + int(rng.integers(-2, 3)) if combo & 4 else 0)
        cols.append(c)
    if V == 1000:                                        # every token banned: n = 1 over a history holding them all
        hist[0, :V] = rng.permutation(V)
        cols[0], ng[0], T[0] = V + 5, 1, 1.5
    # (the device bans the words it is given: dropping [eos] is the host's part)
    banned = [BR.ngram_bans(hist[b, :cols[b]].tolist(), ng[b]) | BR.word_bans(hist[b, :cols[b]].tolist(), words[b]) |
              BR.eos_bans(hist[b, :cols[b]].tolist(), EOS if eos[b] >= 0 else None, 0, frm[b]) for b in range(B)]
    if V == 1000:
        assert len(banned[0]) == V
    sets = [set(hist[b, :cols[b]].tolist()) for b in range(B)]
    xr = x.clone()
    for b in range(B):
        xr[b, sorted(banned[b])] = float("-inf")
    seeds = [int(s) for s in rng.integers(0, 2 ** 63, B)]
    top_n = [int(rng.choice([-1, 0, 5, 20])) for _ in range(B)]
    x, xr = x.to(DEV), xr.to(DEV)
    x0 = x.clone()
    hd = torch.from_numpy(hist).to(DEV)
    ts_a, ts_b = _bits(sets, V), _bits(sets, V)
    got = vn.op_sample_bans(x, T, k, seeds, cols, p, r, hd, ng, eos, frm, words, token_sets=ts_a, top_n=top_n)
    want = vn.op_sample_ex(xr, T, k, seeds, cols, p, r, token_sets=ts_b, top_n=top_n)
    torch.cuda.synchronize()
    for a, b in zip(got, want):
        assert _same(a, b)
    assert torch.equal(ts_a, ts_b)
    tok = got[0].cpu()
    hb = hd.cpu()
    for b in range(B):
        assert int(hb[b, cols[b]]) == int(tok[b])
        assert int(tok[b]) not in banned[b] or len(banned[b]) == V
    if V == 1000:
        assert int(tok[0]) == 0 and torch.isnan(got[2][0, 0])     # the arg-max fallback
    assert torch.equal(x, x0)                            # the logits were not written


def _completes(seq, S, n, words, eos, m):
    """(n-gram completions, bad-word completions, early EOS) among the new tokens seq[S:]"""
    bad = [0, 0, 0]
    for j in range(S, len(seq)):
        h = seq[:j]
        if n and seq[j] in BR.ngram_bans(h, n):
            bad[0] += 1
        if seq[j] in BR.word_bans(h, words, eos):
            bad[1] += 1
        if eos is not None and seq[j] == eos and j - S < m:
            bad[2] += 1
    return bad


BANS = dict(no_repeat_ngram_size=3, bad_words_ids=WORDS, min_new_tokens=6)


@torch.no_grad()
@pytest.mark.parametrize("fmt", ["bf16", "fp8_e4m3"])
def test_end_to_end_bans_hold_and_greedy_is_hf(fmt):
    state = to_dev(O.random_llm_state(SMALL, seed=21))
    m = _model_at(480, fmt=fmt)
    m.load_state_dict(dict(state))
    ids = O.make_prompt_ids(SMALL, 356, seed=3, batch=3).to(DEV)
    vf = video_feats(3, 4)
    S = ids.shape[1]
    checked = 0
    for kw in (dict(), dict(do_sample=True, temperature=0.7, top_k=0, seed=5)):
        out = _gen(m, ids, vf, 24, eos_token_id=EOS, **BANS, **kw)
        for b in range(3):
            seq = out[b].tolist()
            if EOS in seq[S:]:
                seq = seq[:S + seq[S:].index(EOS) + 1]
            assert _completes(seq, S, 3, WORDS, EOS, 6) == [0, 0, 0], (fmt, kw, b)
        if kw:
            continue
        # teacher-forced: the engine's scored logits, HF's processors on the host, outside near-ties
        bans = m._ban_args(3, WORDS, 6, EOS)
        logits = m(out, video_spatio_temporal_features=vf, logits_to_keep=0).logits.float().cpu()
        for b in range(3):
            for j in range(S, out.shape[1]):
                if EOS in out[b, S:j].tolist():
                    break
                xp = m._host_bans(out[b:b + 1, :j].cpu(), logits[b:b + 1, j - 1], bans, S)[0].numpy()
                top = np.sort(xp)[::-1][:2]
                if np.isfinite(top[1]) and top[0] - top[1] > 3 * R.bf16_ulp(top[0]):
                    checked += 1
                    assert int(out[b, j]) == int(np.argmax(xp)), (fmt, b, j)
    assert checked >= 20


@torch.no_grad()
def test_histories_follow_the_sequence():
    m = _flat_model()
    ids = O.make_prompt_ids(SMALL, 356, seed=3, batch=3).to(DEV)
    vf = video_feats(3, 4)
    out = _gen(m, ids, vf, 12, no_repeat_ngram_size=2, eos_token_id=None)
    eng = m._engine
    for b in range(3):
        assert eng.read_token_history(b, 0, out.shape[1]).tolist() == out[b].tolist()
    new = O.make_prompt_ids(SMALL, 0, seed=4, batch=3)[:, 1:9].to(DEV)
    out2 = m.generate_continue(new, max_new_tokens=8, bad_words_ids=WORDS, no_repeat_ngram_size=3, eos_token_id=None)
    for b in range(3):
        assert eng.read_token_history(b, 0, out2.shape[1]).tolist() == out2[b].tolist()
    mask = torch.ones_like(ids)
    mask[1, :5] = 0
    pids = ids.clone()
    pids[1, :5] = 0
    out3 = _gen(m, pids, vf, 12, attention_mask=mask, do_sample=True, temperature=0.7, seed=3, no_repeat_ngram_size=1,
                eos_token_id=None)
    for b in range(3):
        assert eng.read_token_history(b, 0, out3.shape[1]).tolist() == out3[b].tolist()
        assert len(set(out3[b, ids.shape[1]:].tolist()) & set(pids[b].tolist())) == 0    # n = 1: no id twice


@torch.no_grad()
def test_sessions_and_chunked_prompts_keep_their_histories():
    state = to_dev(O.random_llm_state(SMALL, seed=21))
    mp = _model_at(1024, kv_blocks=20)
    mp.load_state_dict(dict(state))
    mc = _model_at(1024)
    mc.load_state_dict(dict(state))
    samp = dict(do_sample=True, temperature=0.9, top_k=0, no_repeat_ngram_size=2, bad_words_ids=WORDS)
    g = torch.Generator().manual_seed(8)
    first = torch.cat([torch.tensor([1]), torch.randint(3, 32000, (39,), generator=g)])
    out1 = _run_requests(mp, [dict(input_ids=first, max_new_tokens=9, seed=3, session="a", **samp)], slots=1)[0][0]
    eng = mp._engine
    assert eng.read_token_history(0, 0, len(out1)).tolist() == out1
    turn = torch.randint(3, 32000, (10,), generator=g)
    out2 = _run_requests(mp, [dict(input_ids=turn, max_new_tokens=9, seed=4, continues="a", **samp)], slots=1)[0][0]
    assert out2[:len(out1) + 10] == out1 + turn.tolist()
    assert eng.read_token_history(0, 0, len(out2)).tolist() == out2
    mp.end_session()
    long = torch.cat([torch.tensor([1]), torch.randint(3, 32000, (699,), generator=g)])
    req = dict(input_ids=long, max_new_tokens=9, seed=5, **samp)
    got = _run_requests(mp, [req], slots=1, chunked_prefill=True)[0][0]
    assert mp.last_kv_stats["chunk_calls"] == 2
    assert eng.read_token_history(0, 0, len(got)).tolist() == got
    want = _gen(mc, long[None].to(DEV), None, 9, seed=5, eos_token_id=None, **samp)
    assert got == want.cpu().tolist()[0]


@torch.no_grad()
def test_requests_equal_generate_alone_across_slots_admission_and_paging():
    state = to_dev(O.random_llm_state(SMALL, seed=21))
    m = _model_at(480)
    m.load_state_dict(dict(state))
    reqs = _requests(SMALL, [20, 5, 12, 7, 3, 10, 6], text_only=(3,))
    for i, r in enumerate(reqs):
        r.update(do_sample=i % 3 != 2, temperature=0.9, top_k=0, seed=17 * i, repetition_penalty=[1.0, 1.2][i % 2],
                 no_repeat_ngram_size=[0, 1, 2, 3][i % 4], bad_words_ids=None if i % 3 == 0 else WORDS,
                 min_new_tokens=[0, 4][i % 2])
    base = _run_requests(m, reqs, slots=3)
    assert _run_requests(m, reqs, slots=1) == base
    assert _run_requests(m, reqs, slots=4, packed_admission=True) == base
    for i in (0, 1, 2, 5):
        r = reqs[i]
        kw = {k: r[k] for k in ("do_sample", "temperature", "top_k", "seed", "repetition_penalty",
                                "no_repeat_ngram_size", "bad_words_ids", "min_new_tokens")}
        ids = torch.as_tensor(r["input_ids"]).reshape(1, -1).to(DEV)
        vf = r.get("video_spatio_temporal_features")
        out = _gen(m, ids, None if vf is None else vf[None].to(DEV), r["max_new_tokens"], eos_token_id=None, **kw)
        assert out.cpu().tolist()[0] == base[i][0], i
    # paged, with preemption
    mp = _model_at(480, kv_blocks=7)
    mp.load_state_dict(dict(state))
    reqs = _requests(SMALL, [150] * 5, text_only=(0, 1, 2, 3, 4))
    for i, r in enumerate(reqs):
        r.update(do_sample=i != 1, temperature=1.0, top_k=0, seed=5 + i, no_repeat_ngram_size=2, bad_words_ids=WORDS,
                 min_new_tokens=3)
    want = _run_requests(m, reqs, slots=4)
    assert _run_requests(mp, reqs, slots=4) == want
    assert mp.last_kv_stats["preemptions"] > 0
    assert _run_requests(mp, reqs, slots=4, packed_admission=True) == want


@torch.no_grad()
def test_default_after_banning_equals_fresh_engine():
    ids = O.make_prompt_ids(SMALL, 356, seed=5, batch=2).to(DEV)
    vf = video_feats(2, 6)
    kw = dict(do_sample=True, temperature=0.7, top_k=50, seed=11, eos_token_id=None)
    fresh = _flat_model()
    a = _gen(fresh, ids, vf, 20, **kw)
    used = _flat_model()
    _gen(used, ids, vf, 20, **BANS, **kw)
    _gen(used, ids, vf, 20, no_repeat_ngram_size=2)        # greedy with bans
    _gen(used, ids, vf, 20, **kw)
    n0 = vn.launch_count()
    b = _gen(used, ids, vf, 20, **kw)
    lb = vn.launch_count() - n0
    n0 = vn.launch_count()
    _gen(fresh, ids, vf, 20, **kw)
    la = vn.launch_count() - n0
    assert torch.equal(a, b) and la == lb
    g1 = _gen(fresh, ids, vf, 20, eos_token_id=None)
    g2 = _gen(used, ids, vf, 20, eos_token_id=None)
    assert torch.equal(g1, g2)


def test_abi_rejections():
    m = _flat_model()
    eng = m._ensure_engine(need_llm=True)
    n0 = vn.launch_count()
    for args in ([[0], [-1], [-1], [0], [[]]], [[0], [0], [40000], [0], [[]]], [[0], [0], [-1], [-3], [[]]],
                 [[0], [0], [-1], [0], [[[5, 40000]]]], [[9], [2], [-1], [0], [[]]], [[1, 1], [2, 2], [-1, -1], [0, 0],
                                                                                  [[], []]]):
        with pytest.raises(vn.VclError):
            eng.set_bans(*args)
    with pytest.raises(vn.VclError):
        eng.set_token_history(0, [1] * 500)                 # max_seq + 1 = 481 columns
    with pytest.raises(vn.VclError):
        eng.set_token_history(9, [1, 2])
    with pytest.raises(vn.VclError):
        vn.op_sample_bans(torch.zeros(1, 100, device=DEV), [1.0], [0], [1], [10], [1.0], [1.0],
                          torch.zeros(1, 10, dtype=torch.int32, device=DEV), [2], [-1], [0], [[]])   # column 10 of 10
    assert vn.launch_count() == n0
