"""Device sampling (sampling.cu, vcl_llm_set_sampling) on the GPU.

Bars:
- the kernel against the float64 rules of _sampling_ref.py: never a token outside the kept set; the fp64 choice
  wherever u * W lies at least 1e-5 W from the edges of the chosen interval (at least 99.9 % of draws); greedy rows
  equal the arg-max rule, also next to sampled rows;
- a chi-square test of 20 000 draws of one row against its exact probabilities (deterministic: so are the draws);
- end to end, the sampling analogue of the greedy near-tie rule: teacher-forced with the engine's tokens, the bf16
  oracle's choice for the same u equals the engine's at every step that every logit vector within +-3 bf16 ulps of
  the oracle's decides the same way, and at least 85 % of the steps are decided (at the reference's T = 0.2; 89 % are,
  see test_most_steps_are_decided). The model's lm_head scales 32 rows up, so that its logits single out a few
  candidates as a trained model's do (a random model's are flat: almost no draw among 32 000 near-equal tokens
  survives a 3-ulp perturbation). On such a model u rarely matters, so
- the counter rule is checked exactly on the flat model, against the engine's own logits: every token of a prefill
  (plain and left-padded), decode step, append, sampled graph, slot and packed prefill is the rules' choice for u at
  the position the token takes;
- bit-identical reproducibility (same call, shorter call, packed / one-at-a-time admission, queue order, a greedy
  request next to sampled ones); sampled graphs replayed for every setting; greedy calls unchanged afterwards.
"""
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
import _sampling_ref as R  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import make_engine, to_dev, vid_start_of  # noqa: E402
from test_padded_batch_gpu import padded_batch, video_feats  # noqa: E402
from test_inflight_gpu import _model, _requests, text_prompt  # noqa: E402

DEV = "cuda"
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)


def peaked_state():
    sd = O.random_llm_state(SMALL, seed=21)
    lm = sd["lm_head.weight"].clone()
    lm[1000:1032] *= 24.0
    sd["lm_head.weight"] = lm
    return sd


@pytest.fixture(scope="module")
def peaked():
    return to_dev(peaked_state())


@pytest.fixture(scope="module")
def model17(peaked):
    m = _model(SMALL, max_batch=17)
    m.load_state_dict(dict(peaked))
    return m


@pytest.fixture(scope="module")
def flat17():
    """the random model as it is: flat logits, so that every draw depends on its seed and position (the
    reproducibility tests below would not see a wrong seed or counter on a peaked model)"""
    m = _model(SMALL, max_batch=17)
    m.load_state_dict(to_dev(O.random_llm_state(SMALL, seed=21)))
    return m


def bf16_rows(B, V, seed, scale=2.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, V, generator=g) * scale).bfloat16().float()


# ------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("V", [32003, 1000])
@pytest.mark.parametrize("B", [1, 3, 5, 16, 17])
def test_kernel_matches_fp64_rules(V, B):
    rng = np.random.default_rng(1000 * B + V)
    temps = [0.2, 0.7, 1.0, 1.5, 1e-4, 0.0]
    ks = [0, 1, 50, 1000, V, V + 5]
    n_far = n_all = 0
    for rep in range(12):
        T = [float(rng.choice(temps)) for _ in range(B)]
        k = [int(rng.choice(ks)) for _ in range(B)]
        # logits spread 6 / T wide: a flat row over 32 000 tokens gives each token ~3e-5 of the mass, and most
        # draws would fall within 1e-5 W of an interval's edge
        scale = torch.tensor([6.0 * max(t, 0.2) for t in T])[:, None]
        x = (bf16_rows(B, V, seed=rep * 100 + B, scale=1.0) * scale).bfloat16().float()
        if B > 2:
            x[1, rng.choice(V, 40, replace=False)] = float("-inf")
            kth = torch.sort(x[2], descending=True).values[49]
            x[2, rng.choice(V, 5, replace=False)] = kth         # ties at the 50th value
        seed = [int(rng.integers(0, 2 ** 63)) * 2 + int(rng.integers(0, 2)) for _ in range(B)]
        ctr = [int(rng.integers(0, 2 ** 31)) for _ in range(B)]
        tok = vn.op_sample(x.to(DEV), T, k, seed, ctr).cpu().tolist()
        xn = x.numpy()
        for b in range(B):
            u = float(R.uniform(seed[b], ctr[b]))
            want, margin = R.choose(xn[b], T[b], k[b], u)
            if margin is None:
                assert tok[b] == want == int(torch.argmax(x[b])), (b, T[b], tok[b], want)
                continue
            assert R.kept_mask(xn[b], T[b], k[b])[tok[b]], (b, T[b], k[b], tok[b])
            n_all += 1
            if margin >= 1e-5:
                n_far += 1
                assert tok[b] == want, (b, T[b], k[b], u, tok[b], want, margin)
    assert n_all == 0 or n_far >= 0.999 * n_all - 1, (n_far, n_all)


@torch.no_grad()
def test_special_rows():
    V = 32003
    x = bf16_rows(5, V, seed=5)
    x[0, 77] = 3e38                                   # scaled maximum overflows at T = 1e-4: the arg-max
    x[1] = float("-inf")                              # nothing above -inf: token 0
    x[2, :] = 1.0                                     # all tied: top_k 1 keeps all of them
    x[3, 10] = float("nan")                           # a NaN is never drawn
    x[4] = float("-inf")                              # greedy: -0 and +0 compare equal, the lower index wins
    x[4, 5], x[4, 9] = -0.0, 0.0
    T, k = [1e-4, 0.5, 1.0, 1.0, 0.0], [0, 50, 1, 0, 0]
    ctr = [3, 4, 5, 6, 7]
    draws = set()
    for s in range(40):
        tok = vn.op_sample(x.to(DEV), T, k, [s] * 5, ctr).tolist()
        assert tok[0] == 77 and tok[1] == 0 and tok[3] != 10 and tok[4] == 5 == int(torch.argmax(x[4]))
        draws.add(tok[2])
        assert tok[2] == R.choose(x[2].numpy(), 1.0, 1, float(R.uniform(s, 5)))[0]
    assert len(draws) > 30


@torch.no_grad()
def test_distribution_chi_square():
    from scipy.stats import chisquare
    V, N = 257, 20000
    x = bf16_rows(1, V, seed=9, scale=1.5)
    T, k = 0.7, 20
    tok = vn.op_sample(x.expand(N, V).contiguous().to(DEV), [T] * N, [k] * N, [123] * N, list(range(N))).cpu()
    keep = R.kept_mask(x[0].numpy(), T, k)
    z = (x[0].numpy() / np.float32(T)).astype(np.float64)
    p = np.where(keep, np.exp(z - z[keep].max()), 0.0)
    p /= p.sum()
    counts = np.bincount(tok.numpy(), minlength=V)
    assert counts[~keep].sum() == 0
    big = p >= 5.0 / N
    obs = np.append(counts[big], counts[keep & ~big].sum())
    exp = np.append(p[big], p[keep & ~big].sum()) * N
    if exp[-1] == 0:
        obs, exp = obs[:-1], exp[:-1]
    stat, pval = chisquare(obs, exp)
    print(f"[sampling] chi-square over {len(obs)} bins: {stat:.1f}, p = {pval:.3f}")
    assert pval > 1e-3


# ------------------------------------------------------------------------------------------
# The counter rule, checked exactly against the engine's own logits: at T = 1 and top_k 50 on the flat random model,
# u decides among 50 tokens of ~2 % each, so a wrong counter or entry changes almost every token.
CT, CK = 1.0, 50
SEEDS = [11, 2 ** 64 - 22, 33, 44]


def _check_counter(logits, toks, counters, seeds, what, stats):
    """token b must be the rules' choice for logits[b] and u = uniform(seeds[b], counters[b]) wherever u * W lies at
    least 1e-5 W from an edge"""
    lg = logits.float().cpu().numpy()
    for b, t in enumerate(toks.tolist()):
        want, margin = R.choose(lg[b], CT, CK, float(R.uniform(seeds[b], counters[b])))
        stats[1] += 1
        if margin >= 1e-5:
            stats[0] += 1
            assert t == want, (what, b, t, want, counters[b])


@torch.no_grad()
def test_counter_is_the_position_the_token_takes():
    flat = to_dev(O.random_llm_state(SMALL, seed=21))
    eng = make_engine(llm=SMALL, max_batch=4, max_seq=480)
    eng.load_llm(flat)
    eng.set_sampling([0, 1, 2, 3], [CT] * 4, [CK] * 4, SEEDS)
    stats = [0, 0]
    B = 3
    rows = [text_prompt(900 + b, 40 + 9 * b) for b in range(B)]
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for pads in ([0] * B, [len(rows[-1]) - len(r) for r in rows]):
            S = len(rows[-1]) if any(pads) else len(rows[0])
            ids = torch.stack([torch.cat([torch.zeros(p, dtype=torch.int64), r[:S - p]]) for p, r in zip(pads, rows)])
            ids = ids.to(DEV)
            vs = torch.full((B,), vn.NO_VIDEO, dtype=torch.int32, device=DEV)
            tag = "padded" if any(pads) else "plain"
            # prefill: the first token takes position S - n_pad[b]
            _, lg, tok = eng.prefill(ids, None, vs, want_logits=True, n_pad=pads if any(pads) else None)
            _check_counter(lg, tok, [S - p for p in pads], SEEDS, f"{tag} prefill", stats)
            # decode steps feeding column q: position q + 1 - n_pad[b]
            for q in range(S, S + 3):
                lg, tok = eng.decode_step(tok, q, want_logits=True)
                _check_counter(lg, tok, [q + 1 - p for p in pads], SEEDS, f"{tag} step {q}", stats)
            # append of 4 tokens at start = S + 3: position start + 4 - n_pad[b]
            tail = torch.cat([tok[:, None].long(), torch.randint(3, 32000, (B, 3), device=DEV)], 1)
            _, lg, tok = eng.prefill_append(tail, S + 3, want_logits=True)
            _check_counter(lg, tok, [S + 7 - p for p in pads], SEEDS, f"{tag} append", stats)
            # the sampled graph (d_pos + i) draws what the eager steps draw, fed the same tokens
            first = tok.clone()
            loop = eng.decode_loop(first, S + 7, 6)
            prev = first
            for i in range(1, 6):
                lg, tok = eng.decode_step(prev, S + 6 + i, want_logits=True)
                _check_counter(lg, tok, [S + 7 + i - p for p in pads], SEEDS, f"{tag} loop step {i}", stats)
                assert torch.equal(tok, loop[:, i]), (tag, i)
                prev = loop[:, i].contiguous()
        # a slot prefill into slot 2 and a packed prefill into slots 3 and 1 use their slots' entries; each token
        # takes position S_i, and its logits are those of the prompt prefilled alone
        alone = []
        for r in rows:
            ids = r[None].to(DEV)
            _, lg, _ = eng.prefill(ids, None, torch.full((1,), vn.NO_VIDEO, dtype=torch.int32, device=DEV),
                                   want_logits=True)
            alone.append(lg.clone())
        t2 = eng.slot_prefill(2, rows[0].to(DEV), None, torch.full((1,), vn.NO_VIDEO, dtype=torch.int32, device=DEV))
        _check_counter(alone[0], t2, [len(rows[0])], [SEEDS[2]], "slot prefill", stats)
        tp = eng.slots_prefill([3, 1], [rows[1], rows[2]], [None, None], [0, 0])
        _check_counter(torch.cat([alone[1], alone[2]]), tp, [len(rows[1]), len(rows[2])], [SEEDS[3], SEEDS[1]],
                       "packed prefill", stats)
        eng.set_sampling([0, 1, 2, 3], [0.0] * 4, [0] * 4, [0] * 4)
    st.synchronize()
    print(f"[sampling] counter rule: {stats[0]}/{stats[1]} draws checked")
    assert stats[0] >= 0.95 * stats[1], stats


# ------------------------------------------------------------------------------------------
def _check_rule(toks, o_logits, seeds, counters0, T, k, what, tally):
    """toks [B, n] engine tokens, o_logits [n, B, V] the oracle teacher-forced with them; counter of step i of row b:
    counters0[b] + i"""
    B, n = toks.shape
    for b in range(B):
        for i in range(n):
            x = o_logits[i, b].float().cpu().numpy()
            u = float(R.uniform(seeds[b], counters0[b] + i))
            j, _ = R.choose(x, T, k, u)
            tally[1] += 1
            if R.decided(x, T, k, u, j):
                tally[0] += 1
                assert int(toks[b, i]) == j, (what, b, i, int(toks[b, i]), j, u)


@pytest.fixture(scope="module")
def tally():
    t = [0, 0]
    yield t
    print(f"[sampling] margin rule: {t[0]}/{t[1]} steps decided")


@torch.no_grad()
@pytest.mark.parametrize("B", [1, 3, 5, 9, 17])
def test_generate_matches_the_oracle_where_decided(B, model17, peaked, tally):
    ids = O.make_prompt_ids(SMALL, 356, seed=40 + B, batch=B).to(DEV)
    S, n, seed, T = ids.shape[1], 12, 1000 + B, 0.2
    vf = video_feats(B, 50 + B)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        out = model17.generate(ids, video_spatio_temporal_features=vf, do_sample=True, temperature=T, top_k=0,
                               seed=seed, max_new_tokens=n, eos_token_id=None)
    st.synchronize()
    toks = out[:, S:]
    _, o_logits = O.greedy_generate(peaked, SMALL, ids, vf.bfloat16(), n, forced=toks)
    _check_rule(toks, o_logits, [seed + b for b in range(B)], [S] * B, T, 0, f"B={B}", tally)


@torch.no_grad()
def test_padded_generate_matches_each_row_where_decided(model17, peaked, tally):
    ids, pads, rows = padded_batch(SMALL, [63, 40, 10, 55], seed=70)
    B, S = ids.shape
    mask = (torch.arange(S, device=DEV)[None] >= torch.tensor(pads, device=DEV)[:, None]).long()
    vf = video_feats(B, 80)
    n, seed, T = 12, 77, 0.2
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        out = model17.generate(ids, video_spatio_temporal_features=vf, attention_mask=mask, do_sample=True,
                               temperature=T, top_k=0, seed=seed, max_new_tokens=n, eos_token_id=None)
    st.synchronize()
    toks = out[:, S:]
    for b in range(B):   # the counter of a padded row: its own position, S - n_pad
        _, o_logits = O.greedy_generate(peaked, SMALL, rows[b], vf[b:b + 1].bfloat16(), n, forced=toks[b:b + 1])
        _check_rule(toks[b:b + 1], o_logits, [seed + b], [S - pads[b]], T, 0, f"padded row {b}", tally)


def test_most_steps_are_decided(tally):
    # Measured on an H100: 417 of the 468 steps of the two tests above (89 %) decided; with the in-flight test below,
    # which adds to the same tally, 483 of 542. The undecided ones are near-ties of the two best
    # candidates (within 6 bf16 ulps, which a 3-ulp shift of each can swap); they come with the bf16 spacing of
    # logits around 40, not with the sampler, and no scaling of this random model removes them
    assert tally[1] > 0 and tally[0] >= 0.85 * tally[1], tally


# ------------------------------------------------------------------------------------------
def _gen(m, ids, vf, n, **kw):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        out = m.generate(ids, video_spatio_temporal_features=vf, max_new_tokens=n, **kw)
    st.synchronize()
    return out


@torch.no_grad()
def test_reproducible_and_independent_of_chunking(flat17):
    ids = O.make_prompt_ids(SMALL, 356, seed=3, batch=3).to(DEV)
    vf = video_feats(3, 4)
    kw = dict(do_sample=True, temperature=1.0, top_k=0, seed=5, eos_token_id=None)
    a = _gen(flat17, ids, vf, 40, **kw)
    b = _gen(flat17, ids, vf, 40, **kw)
    c = _gen(flat17, ids, vf, 20, **kw)
    assert torch.equal(a, b)
    assert torch.equal(a[:, :c.shape[1]], c)
    # the chunked loop (EOS on, never met) gives the same stream as one loop
    d = _gen(flat17, ids, vf, 40, eos_token_id=31999, **{k: v for k, v in kw.items() if k != "eos_token_id"})
    if not (d[:, ids.shape[1]:] == 31999).any():
        assert torch.equal(a, d)
    # other seeds give other streams
    e = _gen(flat17, ids, vf, 40, **dict(kw, seed=6))
    assert not torch.equal(a, e)


def _sampled_reqs(seed0=0, T=0.2):
    # at 3 slots request 1 leaves slot 1 first while slot 0 keeps decoding: a packed admission into a slot other
    # than its row
    reqs = _requests(SMALL, [20, 5, 12, 7, 3, 10, 6], text_only=(3,))
    for i, r in enumerate(reqs):
        r.update(do_sample=True, temperature=T, top_k=0, seed=seed0 + 31 * i)
    return reqs


def _run_requests(m, reqs, **kw):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        outs = m.generate_requests(reqs, eos_token_id=None, **kw)
    st.synchronize()
    return [o.cpu() for o in outs]


@torch.no_grad()
def test_requests_are_independent_of_admission_order_and_neighbours(flat17):
    model17 = flat17
    reqs = _sampled_reqs(T=1.0)
    base = _run_requests(model17, reqs, slots=3)
    assert [o.tolist() for o in _run_requests(model17, reqs, slots=3)] == [o.tolist() for o in base]
    packed = _run_requests(model17, reqs, slots=3, packed_admission=True)
    assert all(torch.equal(x, y) for x, y in zip(base, packed))
    perm = [4, 0, 6, 2, 1, 5, 3]
    shuffled = _run_requests(model17, [reqs[i] for i in perm], slots=3)
    assert all(torch.equal(shuffled[j], base[i]) for j, i in enumerate(perm))
    # a greedy request among sampled ones gives its all-greedy tokens
    greedy = [dict(r, do_sample=False) for r in reqs]
    all_greedy = _run_requests(model17, greedy, slots=3)
    mixed = _run_requests(model17, [greedy[0]] + reqs[1:], slots=3)
    assert torch.equal(mixed[0], all_greedy[0])
    assert all(torch.equal(x, y) for x, y in zip(mixed[1:], base[1:]))


@torch.no_grad()
def test_request_in_flight_matches_generate_alone(model17, peaked, tally):
    """A sampled request in flight and the same request through generate(seed=...) alone (another kernel class for
    the decode, so not bit for bit): both satisfy the margin rule against the oracle."""
    reqs = _sampled_reqs(seed0=500)
    outs = _run_requests(model17, reqs, slots=4)
    for i in (0, 3, 5):
        r = reqs[i]
        ids = torch.as_tensor(r["input_ids"]).reshape(1, -1).to(DEV)
        S = ids.shape[1]
        f = r.get("video_spatio_temporal_features")
        f = None if f is None else f[None].to(DEV).float()
        alone = _gen(model17, ids, f, r["max_new_tokens"], do_sample=True, temperature=0.2, top_k=0, seed=r["seed"],
                     eos_token_id=None)
        for toks in (outs[i][:, S:].to(DEV), alone[:, S:]):
            _, o_logits = O.greedy_generate(peaked, SMALL, ids, None if f is None else f.bfloat16(), toks.shape[1],
                                            forced=toks)
            _check_rule(toks, o_logits, [r["seed"]], [S], 0.2, 0, f"request {i}", tally)


# ------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("NB", [3, 9])
def test_greedy_after_sampling_is_unchanged_and_graphs_replay(NB, peaked):
    k = 8
    rows = [text_prompt(600 + b, 30 + 7 * b) for b in range(NB)]
    S = min(len(r) for r in rows)
    ids = torch.stack([r[:S] for r in rows]).to(DEV)
    vs = vid_start_of(ids, SMALL)
    engs = [make_engine(llm=SMALL, max_batch=NB, max_seq=480) for _ in range(2)]
    for e in engs:
        e.load_llm(peaked)
    eng, fresh = engs
    st = torch.cuda.Stream()
    clips = list(range(NB))
    with torch.cuda.stream(st):
        def timed(call):
            st.synchronize()
            n0 = vn.launch_count()
            t0 = time.perf_counter()
            out = call()
            ms = (time.perf_counter() - t0) * 1e3
            st.synchronize()
            return out, vn.launch_count() - n0, ms

        _, _, first = eng.prefill(ids, None, vs)
        g0, d_greedy, _ = timed(lambda: eng.decode_loop(first, S, k))
        eng.set_sampling(clips, [1.0] * NB, [0] * NB, list(range(NB)))
        s1, d1, ms1 = timed(lambda: eng.decode_loop(first, S, k))               # captures the sampled graph
        # other settings and positions (past the prompt, so that the cache below S keeps the prompt) replay it
        eng.set_sampling(clips, [0.3 + 0.1 * b for b in clips], [5 * b for b in clips], [99 + b for b in clips])
        s2, d2, ms2 = timed(lambda: eng.decode_loop(first, S + 3, k))
        eng.set_sampling(clips, [0.0] + [1.0] * (NB - 1), [0] * NB, list(range(NB)))
        s3, d3, _ = timed(lambda: eng.decode_loop(first, S, k))
        eng.set_sampling(clips, [0.0] * NB, [0] * NB, [0] * NB)
        after, d_after, _ = timed(lambda: eng.decode_loop(first, S, k))
        _, _, ff = fresh.prefill(ids, None, vs)
        ref, d_fresh, _ = timed(lambda: fresh.decode_loop(ff, S, k))
    st.synchronize()
    # greedy calls afterwards: the same tokens and launches as on a fresh engine
    assert torch.equal(g0, ref) and torch.equal(after, ref) and d_after == d_fresh == d_greedy
    # one sampled graph per (B, n_new) for every setting. 1..4 clips: one sampler node per step more than greedy
    # (the partial arg-max hand-off is off), except the last step, where greedy runs the arg-max kernel too;
    # 5..16 clips: the sampler replaces the arg-max kernel
    assert d1 == d2 == d3
    extra = (k - 2) if NB <= 4 else 0
    assert d1 == d_greedy + extra, (d1, d_greedy)
    assert ms2 < 0.5 * ms1, (ms1, ms2)
    assert not torch.equal(s1, s2)
    # a greedy entry inside a sampled graph gives its arg-max
    assert torch.equal(s3[0], ref[0])


@torch.no_grad()
def test_stopping_rules_on_the_device_stream(model17):
    from video_chatgpt.model.utils import KeywordsStoppingCriteria
    from test_inflight_gpu import _Tok
    ids = O.make_prompt_ids(SMALL, 356, seed=11, batch=1, n_pre=10).to(DEV)
    S = ids.shape[1]
    vf = video_feats(1, 12)
    kw = dict(do_sample=True, temperature=1.0, top_k=0, seed=42)
    free = _gen(model17, ids, vf, 60, eos_token_id=None, **kw)[0, S:].tolist()
    j = max(i for i in range(1, 60) if free[i] not in free[:i])      # the last first occurrence
    out = _gen(model17, ids, vf, 60, eos_token_id=free[j], **kw)
    assert out[0, S:].tolist() == free[:j + 1] and model17._pos == out.shape[1] - 1
    crit = KeywordsStoppingCriteria([f"t{free[j]}."], _Tok(), ids.cpu())
    out = _gen(model17, ids, vf, 60, eos_token_id=None, stopping_criteria=[crit], **kw)
    assert out[0, S:].tolist() == free[:j + 1]
    # a continuation samples through prefill_append and the same loop
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        c1 = model17.generate_continue(torch.tensor([[5, 6, 7]]), max_new_tokens=10, eos_token_id=None, **kw)
    st.synchronize()
    assert c1.shape == (1, out.shape[1] + 3 + 10) and torch.equal(c1[:, :out.shape[1]], out)


@torch.no_grad()
def test_rejections_leave_everything_untouched(peaked):
    eng = make_engine(llm=SMALL, max_batch=3, max_seq=64)
    eng.load_llm(peaked)
    k0, v0 = eng.kv_cache(0)
    torch.cuda.synchronize()
    n0 = vn.launch_count()
    for args, msg in [(([0, 3], [1.0, 1.0], [0, 0], [1, 2]), "outside"),
                      (([1, 1], [1.0, 1.0], [0, 0], [1, 2]), "twice"),
                      (([0], [-1.0], [0], [1]), "temperature"),
                      (([0], [float("nan")], [0], [1]), "temperature"),
                      (([0], [float("inf")], [0], [1]), "temperature"),
                      (([0], [1.0], [-2], [1]), "top_k"),
                      (([0, 1, 2, 0], [1.0] * 4, [0] * 4, [1] * 4), "n=4")]:
        with pytest.raises(vn.VclError, match=msg):
            eng.set_sampling(*args)
    with pytest.raises(vn.VclError):
        vn.op_sample(torch.zeros(2, 100, device=DEV), [1.0, -1.0], [0, 0], [1, 1], [0, 0])
    torch.cuda.synchronize()
    assert vn.launch_count() == n0
    k1, v1 = eng.kv_cache(0)
    assert torch.equal(k0, k1) and torch.equal(v0, v1)
    # the table stayed greedy: a decode step launches the greedy kernels and gives the arg-max
    tok_in = torch.tensor([5, 6, 7], dtype=torch.int32, device=DEV)
    lg, tok = eng.decode_step(tok_in, 0, want_logits=True)
    assert torch.equal(tok.long(), lg.argmax(-1))


@torch.no_grad()
def test_video_chatgpt_infer_with_seed(tmp_path):
    from PIL import Image
    from _checkpoint import make_tiny_checkpoint
    from video_chatgpt.eval.model_utils import initialize_model
    from video_chatgpt.inference import video_chatgpt_infer
    ck = make_tiny_checkpoint(tmp_path)
    model, tower, tok, ip, vlen = initialize_model(ck["model_dir"], max_batch=1, max_seq=1024)
    frames = [Image.fromarray(f) for f in O.make_frames(21, 6)]
    args = (frames, "w10 w11 w12 w13", "pg-video-llava", model, tower, tok, ip, vlen)
    calls = []
    orig = model.generate

    def spy(input_ids, **kw):
        calls.append((input_ids, kw["video_spatio_temporal_features"]))
        return orig(input_ids, **kw)
    model.generate = spy
    video_chatgpt_infer(*args, do_sample=False, max_new_tokens=10)
    greedy = model._last_out[0].tolist()
    video_chatgpt_infer(*args, do_sample=True, temperature=1e-4, max_new_tokens=10, seed=3)
    cold = model._last_out[0].tolist()
    # At T = 1e-4 the draw is the arg-max wherever the maximum is unique. At an exact bf16 tie the tied tokens have
    # equal weight and u picks one of them, so the streams agree up to the first tie, and there the cold token is
    # one of the tied ones. The ties come from the engine's logits, teacher-forced with the cold stream.
    ids, feats = calls[-1]
    S = ids.shape[1]
    eng = model._engine
    vs = model._spans_dev(ids.cuda(), feats, eng.NV)
    _, lg, _ = eng.prefill(ids.cuda(), feats.cuda(), vs, want_logits=True)
    n = min(len(cold), len(greedy)) - S
    for j in range(n):
        top = torch.topk(lg[0], 2).values
        if top[0] == top[1]:
            assert lg[0, cold[S + j]] == top[0], (j, cold[S:], greedy[S:])
            break
        assert cold[S + j] == greedy[S + j], (j, cold[S:], greedy[S:])
        if j + 1 < n:
            lg, _ = eng.decode_step(torch.tensor([cold[S + j]], dtype=torch.int32, device=DEV), S + j, want_logits=True)
    a = video_chatgpt_infer(*args, do_sample=True, temperature=1.0, max_new_tokens=10, seed=4)
    b = video_chatgpt_infer(*args, do_sample=True, temperature=1.0, max_new_tokens=10, seed=4)
    assert isinstance(a, str) and a == b
