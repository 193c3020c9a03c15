"""GPU tests of beam search: vcl_op_beam_select against the float64 rule (_beam_ref.py) and against the sampler's
greedy log-probs, the engine's beam steps against its own eager decode steps (forks read back bit for bit, picks from
the logits decode_step gives), graph against eager, the fp8 engine against the bf16 one, a greedy call after a beam
call, and the rejections."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "video-llava_b200"))

import vcl_native as vn  # noqa: E402
import _beam_ref as BR  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import make_engine, to_dev, vid_start_of  # noqa: E402
from test_inflight_gpu import text_prompt  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)


def _rows(Bk, V, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(Bk, V, generator=g) * 3).bfloat16().float()
    for r in range(Bk):
        kind = r % 4
        if kind == 1:                                    # ties at the top of the row
            x[r, torch.randperm(V, generator=g)[:5]] = x[r].max()
        elif kind == 2:
            x[r, torch.randperm(V, generator=g)[:V // 3]] = float("-inf")
    return x


def _check_step(x, scores, k, eos, last, rec, picks):
    """records / picks of one step against _beam_ref.select, position by position: the candidate at place q must be
    the reference's wherever its score is apart from both neighbours (the next one left out, for the last place) by
    more than 1e-5 + 2^-22 |s|, or exactly tied with them (the tie rule orders both); the picks must be the
    reference's when every place is decided; every score within the bound. -> (decided places, places)"""
    score, beam, tok = vn.beam_records(rec.cpu())
    picks = picks.cpu()
    ref = BR.select(x.numpy(), scores.tolist(), k, eos, last)
    sep = lambda a, b: a == b or a - b > BR.gap(a, b)   # noqa: E731
    K = 2 * k
    decided = 0
    for i, (top, rpicks, hits, nxt) in enumerate(ref):
        vals = [np.inf] + [c[0] for c in top] + [nxt]
        all_ok = True
        for q in range(K):
            s = float(score[i, q])
            assert abs(s - top[q][0]) <= BR.gap(s, top[q][0]) or (np.isinf(top[q][0]) and s == top[q][0]), \
                (i, q, s, top[q])
            if sep(vals[q], vals[q + 1]) and sep(vals[q + 1], vals[q + 2]):
                decided += 1
                assert (int(beam[i, q]), int(tok[i, q])) == (top[q][1], top[q][2]), (i, q, top[q])
            else:
                all_ok = False
        if all_ok:
            assert picks[i].tolist() == rpicks, (i, picks[i], rpicks)
    return decided, K * len(ref)


@torch.no_grad()
@pytest.mark.parametrize("V", [32003, 1000])
@pytest.mark.parametrize("B,k", [(1, 2), (2, 2), (3, 8), (8, 8)])
def test_kernel_matches_fp64_rule(V, B, k):
    Bk = B * k
    x = _rows(Bk, V, seed=V + Bk)
    g = torch.Generator().manual_seed(Bk)
    scores = -(torch.rand(Bk, generator=g) * 4).float()
    eos = int(torch.argmax(x[0]))                        # EOS among the candidates
    decided = total = 0
    for last in (False, True):
        rec, picks = vn.op_beam_select(x.to(DEV), scores.to(DEV), k, eos=eos, last_step=last)
        d, t = _check_step(x, scores, k, eos, last, rec, picks)
        decided, total = decided + d, total + t
    print(f"[beam] V {V} B {B} k {k}: {decided} of {total} candidate places decided")
    assert decided >= 0.5 * total


@torch.no_grad()
def test_row_log_probs_are_the_samplers():
    """with running score 0 a candidate's score is the greedy log-prob vcl_op_sample_logprobs reports, bit for bit"""
    V, k = 32003, 2
    x = _rows(k, V, seed=3)
    x[1] = x[0]
    rec, _ = vn.op_beam_select(x.to(DEV), torch.zeros(k, device=DEV), k)
    score, beam, tok = vn.beam_records(rec.cpu())
    _, ids, lp = vn.op_sample_logprobs(x.to(DEV), [0.0] * k, [0] * k, [0] * k, [0] * k, [20] * k)
    ids, lp = ids.cpu(), lp.cpu()
    sampler = {int(i): float(v) for i, v in zip(ids[0, 1:], lp[0, 1:]) if i >= 0}
    for q in range(2 * k):
        t = int(tok[0, q])
        if t in sampler:
            assert torch.tensor(sampler[t]).view(torch.int32) == score[0, q].view(torch.int32), (t, sampler[t])


# ------------------------------------------------------------------------------------------
def _engine(max_batch, fmt="bf16", sd=None):
    eng = make_engine(llm=SMALL, max_batch=max_batch, max_seq=160)
    eng.load_llm(sd if sd is not None else to_dev(O.random_llm_state(SMALL, seed=21)), weight_format=fmt)
    return eng


def _prompts(B, padded):
    S = 24
    ids = torch.stack([text_prompt(700 + b, S) for b in range(B)]).to(DEV)
    pads = [(3 * b) % 7 for b in range(B)] if padded else None
    return ids, pads


def _run(eng, ids, pads, k, n, chunks, eos=-1):
    vs = vid_start_of(ids, SMALL)
    rec, picks = eng.beam_start(ids, None, vs, k, n, eos, n_pad=pads)
    recs, pks = [rec], [picks]
    t = 1
    for c in chunks:
        r, p = eng.beam_decode(c)
        recs.append(r)
        pks.append(p)
        t += c
    return torch.cat(recs).cpu(), torch.cat(pks).cpu(), t


def _clip_maps(rec, picks, B, k):
    """the beam -> clip map after each step, by the rule of beam_merge_kernel"""
    _, beam, _ = vn.beam_records(rec)
    m = [[i if j == 0 else B + i * (k - 1) + j - 1 for j in range(k)] for i in range(B)]
    maps, forks = [], []
    for t in range(rec.shape[0]):
        new, fk = [], []
        for i in range(B):
            par = [0 if t == 0 else int(beam[t, i, int(picks[t, i, r])]) for r in range(k)]
            used, nw = set(), [None] * k
            for r in range(k):
                if par[r] not in used:
                    used.add(par[r])
                    nw[r] = m[i][par[r]]
            free = [m[i][j] for j in range(k) if j not in used]
            for r in range(k):
                if nw[r] is None:
                    nw[r] = free.pop(0)
                    fk.append((m[i][par[r]], nw[r]))
            new.append(nw)
        m = new
        maps.append(m)
        forks.append(fk)
    return maps, forks


@torch.no_grad()
@pytest.mark.parametrize("B,k,padded", [(1, 2, False), (1, 4, True), (2, 4, False), (3, 8, True)])
def test_forks_and_picks_against_eager_decode_steps(B, k, padded):
    """Beams from the graph loop; then a fresh engine at the same B * k prefills every clip with the prompt and is
    teacher-forced with each clip's tokens through eager decode_step. Every step's records must be op_beam_select's on
    the logits decode_step gives, and the caches of the running beams must match bit for bit; columns no beam owns
    keep the NaN sentinel."""
    n, T = 40, 12
    sd = to_dev(O.random_llm_state(SMALL, seed=21))
    eng = _engine(B * k, sd=sd)
    ids, pads = _prompts(B, padded)
    S = ids.shape[1]
    nan = torch.full((B * k, SMALL.heads, 160, 128), float("nan"), dtype=torch.bfloat16, device=DEV)
    for l in range(SMALL.layers):
        eng.set_kv_cache(l, nan, nan)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        rec, picks, t = _run(eng, ids, pads, k, n, [5, 6])
    st.synchronize()
    assert t == T
    maps, _ = _clip_maps(rec, picks, B, k)
    score, beam, tok = vn.beam_records(rec)
    decided = total = 0

    # the reference: every clip holds its item's prompt; step s feeds each clip the token its beam picked at s - 1
    # (a first prefill of all B * k clips leaves every clip its item's padding; the B-prompt prefill then gives the
    # logits of step 0 and the prompt columns the forks copy)
    ref = _engine(B * k, sd=sd)
    item_of = [c if c < B else (c - B) // (k - 1) for c in range(B * k)]
    rids = ids[item_of]
    rp = None if pads is None else [pads[i] for i in item_of]
    ref.prefill(rids, None, vid_start_of(rids, SMALL), want_token=False, n_pad=rp)
    _, lg, _ = ref.prefill(ids, None, vid_start_of(ids, SMALL), want_logits=True, n_pad=pads)
    run_scores = torch.tensor([[0.0] + [-1e9] * (k - 1)] * B).reshape(-1)
    prev_map = [[i if j == 0 else B + i * (k - 1) + j - 1 for j in range(k)] for i in range(B)]
    for s in range(T):
        # beam r of item i reads the logits of its clip (step 0: the prompt's clip i)
        rows = [i if s == 0 else prev_map[i][j] for i in range(B) for j in range(k)]
        r2, p2 = vn.op_beam_select(lg[rows].contiguous(), run_scores.to(DEV), k, last_step=s + 1 >= n)
        assert torch.equal(r2.cpu(), rec[s]) and torch.equal(p2.cpu(), picks[s]), s
        # ... and the float64 rule on the same model logits, position by position
        d, tot = _check_step(lg[rows].float().cpu(), run_scores, k, -1, s + 1 >= n, rec[s], picks[s])
        decided, total = decided + d, total + tot
        pk = picks[s].to(torch.int64)
        run_scores = torch.take_along_dim(score[s], pk, dim=1).reshape(-1)
        nxt = torch.zeros(B * k, dtype=torch.int32)
        for i in range(B):
            for r in range(k):
                nxt[maps[s][i][r]] = int(tok[s, i, int(pk[i, r])])
        # the reference feeds each clip the token of the beam that now lives there, after copying the parent's cache
        # columns on the host (the fork)
        _, forks = _clip_maps(rec[:s + 1], picks[:s + 1], B, k)
        for src, dst in forks[s]:
            c0, c1 = (0, S) if s == 0 else (S, S + s)
            for l in range(SMALL.layers):
                kk, vv = ref.kv_cache(l)
                kk[dst, :, c0:c1] = kk[src, :, c0:c1]
                vv[dst, :, c0:c1] = vv[src, :, c0:c1]
                ref.set_kv_cache(l, kk, vv)
        prev_map = maps[s]
        if s + 1 < T:
            lg, _ = ref.decode_step(nxt.to(DEV), S + s, want_logits=True)
    torch.cuda.synchronize()
    print(f"[beam] forks {B}x{k}: {decided} of {total} candidate places decided against float64")
    assert decided >= 0.5 * total
    live = sorted(c for i in range(B) for c in maps[T - 1][i])
    for l in range(SMALL.layers):
        k0, v0 = eng.kv_cache(l)
        k1, v1 = ref.kv_cache(l)
        for c in live:
            lo = pads[item_of[c]] if pads else 0
            a, b = k0[c, :, lo:S + T - 1], k1[c, :, lo:S + T - 1]
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), (l, c)
            assert torch.equal(v0[c, :, lo:S + T - 1].view(torch.int16), v1[c, :, lo:S + T - 1].view(torch.int16))
            assert torch.isnan(k0[c, :, S + T - 1:].float()).all()


@torch.no_grad()
def test_graph_and_eager_runs_agree():
    B, k, n = 2, 4, 30
    eng = _engine(B * k)
    ids, pads = _prompts(B, True)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        g = _run(eng, ids, pads, k, n, [8, 8, 8])
    st.synchronize()
    e = _run(eng, ids, pads, k, n, [8, 8, 8])          # the legacy default stream cannot be captured: eager steps
    torch.cuda.synchronize()
    assert torch.equal(g[0], e[0]) and torch.equal(g[1], e[1])


@torch.no_grad()
def test_fp8_engine_equals_bf16_engine_on_dequantized_weights():
    B, k, n = 1, 4, 24
    sd = to_dev(O.random_llm_state(SMALL, seed=21))
    e8 = _engine(B * k, fmt="fp8_e4m3", sd=sd)
    deq = dict(sd)
    for name, w in sd.items():
        if name.endswith("proj.weight") or name == "lm_head.weight":
            deq[name] = vn.op_quantize_fp8(w)[0]
    e16 = _engine(B * k, sd=deq)
    ids, _ = _prompts(B, False)
    st = torch.cuda.Stream()
    out = []
    with torch.cuda.stream(st):
        for e in (e8, e16):
            st.synchronize()
            n0 = vn.launch_count()
            r = _run(e, ids, None, k, n, [7, 8])
            st.synchronize()
            out.append((r, vn.launch_count() - n0))
    assert torch.equal(out[0][0][0], out[1][0][0]) and torch.equal(out[0][0][1], out[1][0][1])
    assert out[0][1] == out[1][1]


@torch.no_grad()
def test_greedy_after_beams_is_a_fresh_engine():
    sd = to_dev(O.random_llm_state(SMALL, seed=21))
    eng, fresh = _engine(8, sd=sd), _engine(8, sd=sd)
    ids, _ = _prompts(3, False)
    vs = vid_start_of(ids, SMALL)
    st = torch.cuda.Stream()

    def counted(e, f):
        st.synchronize()
        n0 = vn.launch_count()
        out = f(e)
        st.synchronize()
        return out, vn.launch_count() - n0

    with torch.cuda.stream(st):
        _run(eng, ids[:2], [1, 0], 4, 20, [6])
        g0, n0 = counted(eng, lambda e: e.generate(ids, None, vs, 9))
        g1, n1 = counted(fresh, lambda e: e.generate(ids, None, vs, 9))
    st.synchronize()
    assert torch.equal(g0, g1) and n0 == n1


def test_rejections():
    eng = _engine(4)
    ids, _ = _prompts(1, False)
    vs = vid_start_of(ids, SMALL)
    n0 = vn.launch_count()
    for k, n, why in ((1, 8, "num_beams"), (9, 8, "num_beams"), (8, 8, "max_batch"), (2, 200, "max_seq")):
        with pytest.raises(vn.VclError, match=why):
            eng.beam_start(ids, None, vs, k, n)
    eng._beam_shape = (1, 2)
    with pytest.raises(vn.VclError, match="no beam search"):
        eng.beam_decode(1)
    with pytest.raises(vn.VclError, match="eos_token"):
        eng.beam_start(ids, None, vs, 2, 8, eos=SMALL.vocab)
    assert vn.launch_count() == n0
    eng.beam_start(ids, None, vs, 2, 4)
    with pytest.raises(vn.VclError, match="outside the call"):
        eng.beam_decode(4)
    eng.beam_start(ids, None, vs, 2, 8)
    eng.prefill(ids, None, vs)                          # a new sequence ends the beam search
    with pytest.raises(vn.VclError, match="no beam search"):
        eng.beam_decode(1)
    x = torch.zeros(4, 6, device=DEV)                   # V below 2k
    with pytest.raises(vn.VclError, match="V=6"):
        vn.op_beam_select(x, torch.zeros(4, device=DEV), 4)
    big = make_engine(llm=O.LlmCfg(hidden=512, inter=1024, heads=4, layers=0, vocab=60000), max_batch=2, max_seq=64)
    with pytest.raises(vn.VclError, match="vocabulary"):
        big.beam_start(ids[:, :8], None, vs, 2, 4)


# ---- end to end: model.generate(num_beams=k) against the bf16 oracle, teacher-forced with the engine's beams ---------
def _oracle_set(x, run, k, ulps=3):
    """HF's step 1-2 on oracle logits x [k, V] (fp32 log_softmax + the running scores, top 2k): the candidate set,
    and whether a move of every logit by `ulps` bf16 ulps cannot change it. A candidate's score moves by its own logit's
    move d_j and by its row's log-sum-exp; the latter is common to the candidates of one row and moves by at most
    sum_i p_i d_i (first order), so it counts only between candidates of different rows."""
    from _sampling_ref import bf16_ulp
    K, V = 2 * k, x.shape[1]
    lp = torch.log_softmax(x.double(), dim=-1)
    acc = (torch.log_softmax(x, dim=-1) + run[:, None]).double()
    d = torch.from_numpy(ulps * bf16_ulp(x.numpy()))
    E = (lp.exp() * d).sum(dim=1)
    idx = torch.topk(acc.reshape(-1), K).indices
    inside = torch.zeros(k * V, dtype=torch.bool)
    inside[idx] = True
    inside = inside.view(k, V)
    decided = True
    for r in range(k):
        if not inside[r].any():
            continue
        lo = (acc[r] - d[r])[inside[r]].min()
        for r2 in range(k):
            hi = (acc[r2] + d[r2])[~inside[r2]].max()
            decided = decided and bool(lo - (0.0 if r2 == r else E[r] + E[r2]) > hi)
    return {(int(i) // V, int(i) % V) for i in idx}, decided


@pytest.fixture(scope="module")
def oracle_tally():
    t = {2: [0, 0], 4: [0, 0]}
    yield t
    for k, (d, n) in t.items():
        print(f"[beam] generate(num_beams={k}) against the bf16 oracle: {d}/{n} steps decided")


@torch.no_grad()
@pytest.mark.parametrize("fmt", ["bf16", "fp8_e4m3"])
@pytest.mark.parametrize("k,n", [(2, 12), (4, 8)])
def test_generate_matches_oracle_candidate_sets_where_decided(fmt, k, n, oracle_tally):
    """model.generate(num_beams=4) on the sampling tests' peaked model, two prompts with video, the second left-padded.
    The engine's records are kept as the real host loop reads them. The output and sequences_scores are HF's own steps
    4-6 on those records; every step's candidate set is the one HF's log_softmax + topk give on the bf16 oracle's
    logits (run on each beam's unpadded prompt and tokens, W~ for fp8, with the engine's running scores) wherever a
    3-bf16-ulp move of the logits cannot change it."""
    from test_sampling_gpu import peaked_state
    from test_nucleus_gpu import _model_at
    from test_padded_batch_gpu import video_feats
    import _fp8_ref as F8
    B = 2
    sd = to_dev(peaked_state())
    osd = sd if fmt == "bf16" else F8.dequantize_state(sd)
    m = _model_at(480, fmt=fmt, max_batch=B * k)
    m.load_state_dict(dict(sd))
    rows = [O.make_prompt_ids(SMALL, 356, seed=61)[0], O.make_prompt_ids(SMALL, 356, seed=62, n_pre=57)[0]]
    S = max(r.numel() for r in rows)
    ids = torch.zeros(B, S, dtype=torch.int64)
    mask = torch.zeros(B, S, dtype=torch.int64)
    for b, r in enumerate(rows):
        ids[b, S - r.numel():], mask[b, S - r.numel():] = r, 1
    vf = video_feats(B, 62)
    eng = m._ensure_engine(need_llm=True)
    seen = []
    start, decode = eng.beam_start, eng.beam_decode
    eng.beam_start = lambda *a, **kw: seen.append(start(*a, **kw)) or seen[-1]        # noqa: E731
    eng.beam_decode = lambda *a, **kw: seen.append(decode(*a, **kw)) or seen[-1]      # noqa: E731
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        out = m.generate(ids.to(DEV), vf, attention_mask=mask.to(DEV), num_beams=k, num_return_sequences=k,
                         max_new_tokens=n, eos_token_id=None)
    st.synchronize()
    rec = torch.cat([r for r, _ in seen]).cpu()
    picks = torch.cat([p for _, p in seen]).cpu().to(torch.int64)
    score, beam, tok = vn.beam_records(rec)
    assert rec.shape[0] == n                           # EOS off, length penalty 1: every step runs
    # the output: HF's own steps 4-6 on the records
    _, seqs, scores, idx, _ = BR.hf_replay([(score[t], beam[t], tok[t], picks[t]) for t in range(n)], B, k, S, n,
                                           None, -1, 1.0, False)
    L = int((idx >= 0).sum(dim=2).max())
    assert torch.equal(out[:, S:].cpu(), seqs[:, :, S:S + L].reshape(B * k, L))
    assert torch.equal(out[:, :S].cpu(), ids.repeat_interleave(k, dim=0))
    assert torch.equal(m.last_beam_scores.view(torch.int32), scores.reshape(-1).view(torch.int32))
    # every step against the oracle
    hist = [[[] for _ in range(k)] for _ in range(B)]
    run = torch.tensor([[0.0] + [-1e9] * (k - 1)] * B)
    for t in range(n):
        for i in range(B):
            seq = torch.stack([torch.cat([rows[i], torch.tensor(h, dtype=torch.int64)]) for h in hist[i]]).to(DEV)
            lg, _, _ = O.llm_forward(osd, SMALL, seq, vf[i:i + 1].expand(k, -1, -1).bfloat16())
            cset, ok = _oracle_set(lg[:, -1].float().cpu(), run[i], k)
            oracle_tally[k][1] += 1
            if ok:
                oracle_tally[k][0] += 1
                got = {(int(beam[t, i, q]), int(tok[t, i, q])) for q in range(2 * k)}
                assert got == cset, (fmt, t, i, got ^ cset)
        for i in range(B):
            hist[i] = [hist[i][int(beam[t, i, q])] + [int(tok[t, i, q])] for q in picks[t, i].tolist()]
            run[i] = torch.take_along_dim(score[t, i], picks[t, i], dim=0)


def test_most_oracle_steps_are_decided(oracle_tally):
    """at least half the steps of the two-beam runs are decided. With four beams the set's boundary (candidates 8 and
    9) lies in the peaked model's dense tail, a few bf16 ulps apart, and only about a quarter are: that count is
    printed, and every decided step must still match"""
    d, n = oracle_tally[2]
    assert n > 0 and d >= 0.5 * n, oracle_tally
    assert oracle_tally[4][1] > 0
