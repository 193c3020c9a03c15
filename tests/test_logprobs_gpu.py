"""Log-probs of generated tokens on the GPU (sample_kernel with top_n, vcl_llm_set_logprobs / _read_logprobs).

Bars:
- the kernel alone against the float64 rule of _logprob_ref.py: top ids exact (ties by index), every log-prob within
  1e-5 + 2^-22 |lp64|, and the chosen token bit for bit vcl_op_sample's;
- nothing changes: with log-probs on, every path returns the tokens (and leaves the cache bits) it returns with them
  off, and a greedy call afterwards runs the launches of a fresh engine;
- right logits at the right position: each step's rows equal vcl_op_sample_logprobs on the logits prefill /
  decode_step / prefill_append return for the same tokens (teacher-forced), bit for bit;
- a request's values do not depend on its slot, neighbours, queue order, admission mode, paging or preemption;
- the rejections.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
import _logprob_ref as LR  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import make_engine, to_dev, vid_start_of  # noqa: E402
from test_padded_batch_gpu import video_feats  # noqa: E402
from test_inflight_gpu import _model, _requests, text_prompt  # noqa: E402
from test_paged_kv_gpu import paged_model  # noqa: E402

DEV = "cuda"
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)


def bf16_rows(B, V, seed, scale):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, V, generator=g) * scale).bfloat16().float()


# ------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("V", [32003, 1000])
@pytest.mark.parametrize("B", [1, 3, 17, 64])
def test_kernel_matches_fp64_rule(V, B):
    rng = np.random.default_rng(7 * B + V)
    temps, ks, ns = [0.0, 1e-4, 0.2, 1.5], [0, 1, 50, V + 5], [0, 1, 5, 20]
    worst = 0.0
    for rep in range(4):
        T = [float(rng.choice(temps)) for _ in range(B)]
        k = [int(rng.choice(ks)) for _ in range(B)]
        n = [int(rng.choice(ns)) for _ in range(B)]
        x = bf16_rows(B, V, seed=rep * 1000 + B, scale=3.0)
        for b in range(B):
            kind = (b + rep) % 6
            if kind == 1:                                   # ties at the n-th and at the 50th value
                srt = torch.sort(x[b], descending=True).values
                x[b, rng.choice(V, 4, replace=False)] = srt[max(n[b], 1) - 1]
                x[b, rng.choice(V, 4, replace=False)] = srt[49]
            elif kind == 2:
                x[b, rng.choice(V, 50, replace=False)] = float("-inf")
            elif kind == 3:
                x[b, rng.choice(V, 7, replace=False)] = float("nan")
            elif kind == 4 and rep % 2:
                x[b] = float("-inf")                        # no finite maximum
        seed = [int(rng.integers(0, 2 ** 63)) for _ in range(B)]
        ctr = [int(rng.integers(0, 2 ** 31)) for _ in range(B)]
        xd = x.to(DEV)
        plain = vn.op_sample(xd, T, k, seed, ctr)
        tok, ids, lp = vn.Engine.sample_logprobs_op(xd, T, k, seed, ctr, n)
        assert torch.equal(tok, plain)
        tok, ids, lp = tok.cpu().tolist(), ids.cpu(), lp.cpu()
        for b in range(B):
            want, wids, wlps = LR.logprobs(x[b].numpy(), T[b], k[b], n[b], tok[b])
            assert ids[b, 0] == tok[b]
            assert ids[b, 1:1 + n[b]].tolist() == wids, (b, T[b], k[b], n[b])
            got = [float(lp[b, 0])] + lp[b, 1:1 + n[b]].tolist()
            ref = [want] + wlps
            assert LR.close(got, ref), (b, T[b], k[b], n[b], got, ref)
            fin = np.isfinite(ref) & np.isfinite(got)
            if fin.any():
                worst = max(worst, float(np.max(np.abs(np.subtract(got, ref))[fin] / (1e-5 + 2.0 ** -22 *
                                                                                      np.abs(ref)[fin]))))
    print(f"[logprobs] V {V} B {B}: worst error {worst:.3f} of the bound")


@torch.no_grad()
def test_special_rows():
    V = 32003
    x = bf16_rows(4, V, seed=5, scale=2.0)
    x[0, 77] = 3e38                                   # scaled maximum overflows at T = 1e-4: arg-max, NaN
    x[1] = float("-inf")                              # greedy, nothing above -inf: token 0, NaN
    x[2] = float("nan")
    x[3, :] = 1.0                                     # all tied: the lowest indices, lp = -log V
    tok, ids, lp = vn.Engine.sample_logprobs_op(x.to(DEV), [1e-4, 0.0, 0.3, 0.0], [0, 0, 5, 0], [1] * 4,
                                                [3] * 4, [3, 2, 1, 5])
    tok, ids, lp = tok.cpu(), ids.cpu(), lp.cpu()
    assert tok.tolist()[:2] == [77, 0]
    for b, n in ((0, 3), (1, 2), (2, 1)):
        assert ids[b, 0] == tok[b] and torch.isnan(lp[b, :1 + n]).all() and (ids[b, 1:1 + n] == -1).all()
    assert ids[3, :6].tolist() == [0, 0, 1, 2, 3, 4]
    assert torch.allclose(lp[3, :6].double(), torch.full((6,), -np.log(V), dtype=torch.float64), atol=1e-5)


# ------------------------------------------------------------------------------------------
def _check_rows(eng, logits, toks, entries, pos, T, k, seeds, top_n, what):
    """the engine's rows at (entries[b], pos[b]) equal the kernel alone on `logits`, bit for bit"""
    B = logits.shape[0]
    t, ids, lp = vn.Engine.sample_logprobs_op(logits, T, k, seeds, pos, top_n)
    assert torch.equal(t, toks.to(torch.int32)), what
    for b in range(B):
        gi, gl = eng.read_logprobs(entries[b], pos[b], 1)
        m = 1 + top_n[b]
        assert torch.equal(gi[0, :m], ids[b, :m]), (what, b)
        assert torch.equal(gl[0, :m].view(torch.int32), lp[b, :m].view(torch.int32)), (what, b)


@torch.no_grad()
@pytest.mark.parametrize("sampled", [False, True])
def test_rows_are_the_logits_at_their_positions(sampled):
    sd = to_dev(O.random_llm_state(SMALL, seed=21))
    eng = make_engine(llm=SMALL, max_batch=4, max_seq=480)
    eng.load_llm(sd)
    B = 3
    T = [0.7 if sampled else 0.0] * B
    K, seeds, top_n = [50, 0, 1000], [11, 12, 13], [5, 0, 20]
    eng.set_sampling(list(range(B)), T, K, seeds)
    eng.set_logprobs(list(range(B)), top_n)
    rows = [text_prompt(900 + b, 40 + 9 * b) for b in range(B)]
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for pads in ([0] * B, [len(rows[-1]) - len(r) for r in rows]):
            S = len(rows[-1]) if any(pads) else len(rows[0])
            ids = torch.stack([torch.cat([torch.zeros(p, dtype=torch.int64), r[:S - p]]) for p, r in zip(pads, rows)])
            ids = ids.to(DEV)
            vs = torch.full((B,), vn.NO_VIDEO, dtype=torch.int32, device=DEV)
            tag = "padded" if any(pads) else "plain"
            _, lg, tok = eng.prefill(ids, None, vs, want_logits=True, n_pad=pads if any(pads) else None)
            _check_rows(eng, lg, tok, [0, 1, 2], [S - p for p in pads], T, K, seeds, top_n, f"{tag} prefill")
            for q in range(S, S + 3):
                lg, tok = eng.decode_step(tok, q, want_logits=True)
                _check_rows(eng, lg, tok, [0, 1, 2], [q + 1 - p for p in pads], T, K, seeds, top_n, f"{tag} step {q}")
            tail = torch.cat([tok[:, None].long(), torch.randint(3, 32000, (B, 3), device=DEV)], 1)
            _, lg, tok = eng.prefill_append(tail, S + 3, want_logits=True)
            _check_rows(eng, lg, tok, [0, 1, 2], [S + 7 - p for p in pads], T, K, seeds, top_n, f"{tag} append")
            # the graph loop writes what the eager steps write, fed the same tokens
            loop = eng.decode_loop(tok.clone(), S + 7, 6)
            got = [eng.read_logprobs(b, S + 8 - pads[b], 5) for b in range(B)]
            prev = tok.clone()
            for i in range(1, 6):
                lg, t = eng.decode_step(prev, S + 6 + i, want_logits=True)
                assert torch.equal(t, loop[:, i]), (tag, i)
                _check_rows(eng, lg, t, [0, 1, 2], [S + 7 + i - p for p in pads], T, K, seeds, top_n, f"{tag} {i}")
                for b in range(B):
                    gi, gl = eng.read_logprobs(b, S + 7 + i - pads[b], 1)
                    assert torch.equal(gi[0], got[b][0][i - 1]) and torch.equal(gl[0], got[b][1][i - 1])
                prev = loop[:, i].contiguous()
    st.synchronize()


# ------------------------------------------------------------------------------------------
def _gen(m, ids, vf, n, **kw):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        out = m.generate(ids, video_spatio_temporal_features=vf, max_new_tokens=n, **kw)
    st.synchronize()
    return out


@pytest.fixture(scope="module")
def model17():
    m = _model(SMALL, max_batch=17)
    m.load_state_dict(to_dev(O.random_llm_state(SMALL, seed=21)))
    return m


def _greedy_consistent(out, S, lps, k, eos=None):
    for b, e in enumerate(lps):
        new = out[b, S:].cpu()
        ok = ~torch.isnan(e["token_logprobs"])
        assert e["top_ids"].shape == (len(new), k)
        if eos is not None and (new == eos).any():
            f = int((new == eos).nonzero()[0]) + 1
            assert not ok[f:].any() and (e["top_ids"][f:] == -1).all()
        assert ok.any() and (e["token_logprobs"][ok] <= 0).all()
        if k:   # a greedy token is the top alternative
            assert torch.equal(e["top_ids"][ok, 0], new[ok]) and torch.equal(e["top_logprobs"][ok, 0],
                                                                              e["token_logprobs"][ok])


@torch.no_grad()
@pytest.mark.parametrize("B", [1, 3, 5, 17])
def test_generate_tokens_unchanged(B, model17):
    ids = O.make_prompt_ids(SMALL, 356, seed=3, batch=B).to(DEV)
    vf = video_feats(B, 4)
    S = ids.shape[1]
    for kw in (dict(eos_token_id=None), dict(do_sample=True, temperature=0.7, top_k=50, seed=5, eos_token_id=None)):
        off = _gen(model17, ids, vf, 20, **kw)
        on = _gen(model17, ids, vf, 20, logprobs=5, **kw)
        assert torch.equal(on, off), kw
        assert len(model17.last_logprobs) == B
        if not kw.get("do_sample"):
            _greedy_consistent(on, S, model17.last_logprobs, 5)
        _gen(model17, ids, vf, 20, **kw)
        assert model17.last_logprobs is None


@torch.no_grad()
def test_generate_eos_criteria_padded_and_continue(model17):
    from test_padded_batch_gpu import padded_batch
    ids, pads, _ = padded_batch(SMALL, [10, 25, 3], seed=8)
    mask = torch.ones_like(ids)
    for b, p in enumerate(pads):
        mask[b, :p] = 0
    vf = video_feats(3, 4)
    S = ids.shape[1]
    off = _gen(model17, ids, vf, 24, attention_mask=mask, eos_token_id=None)
    eos = int(off[1, S + 4])                       # row 1 meets "EOS" early, the others keep going
    stop = [lambda o, s: o.shape[1] >= S + 19]
    for kw in (dict(eos_token_id=eos), dict(eos_token_id=eos, stopping_criteria=stop)):
        a = _gen(model17, ids, vf, 24, attention_mask=mask, **kw)
        b = _gen(model17, ids, vf, 24, attention_mask=mask, logprobs=3, **kw)
        assert torch.equal(a, b), kw
        _greedy_consistent(b, S, model17.last_logprobs, 3, eos)
        tail = torch.randint(3, 32000, (3, 5))
        c0 = model17.generate_continue(tail, max_new_tokens=12, eos_token_id=None)
        _gen(model17, ids, vf, 24, attention_mask=mask, **kw)
        c1 = model17.generate_continue(tail, max_new_tokens=12, eos_token_id=None, logprobs=4)
        torch.cuda.synchronize()
        # a stopping criterion's stepwise path feeds a finished row its padding, the device loops its own tokens:
        # the continuation of a row that met EOS may differ there, every other row's may not
        rows = [0, 2] if "stopping_criteria" in kw else [0, 1, 2]
        assert torch.equal(c0[rows], c1[rows]), kw
        _greedy_consistent(c1, c1.shape[1] - 12, model17.last_logprobs, 4)


@torch.no_grad()
def test_greedy_after_logprobs_is_a_fresh_engine():
    sd = to_dev(O.random_llm_state(SMALL, seed=21))
    engs = [make_engine(llm=SMALL, max_batch=3, max_seq=480) for _ in range(2)]
    for e in engs:
        e.load_llm(sd)
    eng, fresh = engs
    ids = torch.stack([text_prompt(600 + b, 30) for b in range(3)]).to(DEV)
    vs = vid_start_of(ids, SMALL)
    st = torch.cuda.Stream()

    def counted(e, f):
        st.synchronize()
        n0 = vn.launch_count()
        out = f(e)
        st.synchronize()
        return out, vn.launch_count() - n0

    with torch.cuda.stream(st):
        run = lambda e: e.generate(ids, None, vs, 9)   # noqa: E731
        g0, n_greedy = counted(eng, run)
        eng.set_logprobs([0, 1, 2], [2, -1, 20])
        g1, n_lp = counted(eng, run)
        eng.set_logprobs([0, 1, 2], [-1] * 3)
        g2, n_after = counted(eng, run)
        g3, n_fresh = counted(fresh, run)
        k0, v0 = eng.kv_cache(1)
        k1, v1 = fresh.kv_cache(1)
    st.synchronize()
    assert torch.equal(g0, g1) and torch.equal(g1, g2) and torch.equal(g2, g3)
    assert n_after == n_fresh == n_greedy and n_lp >= n_greedy
    assert torch.equal(k0.view(torch.int16), k1.view(torch.int16)) and torch.equal(v0.view(torch.int16),
                                                                                      v1.view(torch.int16))


# ------------------------------------------------------------------------------------------
def _run_requests(m, reqs, **kw):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        outs = m.generate_requests(reqs, eos_token_id=None, **kw)
    st.synchronize()
    return [o.cpu() for o in outs], m.last_logprobs


def _same(a, b):
    return all(torch.equal(x[f].view(torch.int32) if x[f].dtype == torch.float32 else x[f],
                           y[f].view(torch.int32) if y[f].dtype == torch.float32 else y[f])
               for x, y in zip(a, b) for f in ("token_logprobs", "top_ids", "top_logprobs"))


@torch.no_grad()
def test_requests_unchanged_and_invariant(model17):
    reqs = _requests(SMALL, [20, 5, 12, 7, 3, 10, 6], text_only=(3,))
    for i, r in enumerate(reqs):
        if i % 2:
            r.update(do_sample=True, temperature=0.7, top_k=50, seed=31 * i)
    base, _ = _run_requests(model17, reqs, slots=3)
    on, lps = _run_requests(model17, reqs, slots=3, logprobs=5)
    assert all(torch.equal(x, y) for x, y in zip(base, on))
    assert all(e["top_ids"].shape == (o.shape[1] - r["input_ids"].numel(), 5) for e, o, r in zip(lps, on, reqs))
    for kw in (dict(slots=1), dict(slots=3, packed_admission=True), dict(slots=7, packed_admission=True)):
        o2, l2 = _run_requests(model17, reqs, logprobs=5, **kw)
        assert all(torch.equal(x, y) for x, y in zip(base, o2)), kw
        assert _same(lps, l2), kw
    perm = [4, 0, 6, 2, 1, 5, 3]
    o3, l3 = _run_requests(model17, [reqs[i] for i in perm], slots=3, logprobs=5)
    assert _same([lps[i] for i in perm], l3)
    # per-request keys; the others report None
    mixed = [dict(r, logprobs=5) if i in (1, 4) else r for i, r in enumerate(reqs)]
    o4, l4 = _run_requests(model17, mixed, slots=3)
    assert [e is None for e in l4] == [i not in (1, 4) for i in range(len(reqs))]
    assert _same([lps[1], lps[4]], [l4[1], l4[4]])


@torch.no_grad()
@pytest.mark.parametrize("fmt", ["bf16", "fp8_e4m3"])
def test_paged_requests_with_preemption(fmt):
    sd = to_dev(O.random_llm_state(SMALL, seed=21))
    reqs = [dict(input_ids=text_prompt(300 + i, 60 + 37 * i), max_new_tokens=40 + 23 * i) for i in range(6)]
    for i, r in enumerate(reqs):
        if i % 3 == 1:
            r.update(do_sample=True, temperature=0.7, top_k=50, seed=7 * i)
    res = {}
    for kv in (0, 5, 40):
        if kv:
            m = paged_model(SMALL, 4, kv, max_seq=480)
        else:
            m = _model(SMALL, max_batch=4)
        m._llm_weight_format = fmt
        m.load_state_dict(dict(sd))
        off, _ = _run_requests(m, reqs, slots=4)
        on, lps = _run_requests(m, reqs, slots=4, logprobs=20, packed_admission=kv == 40)
        assert all(torch.equal(x, y) for x, y in zip(off, on)), kv
        if kv == 5:
            assert m.last_kv_stats["preemptions"] > 0
        res[kv] = (on, lps)
    for kv in (5, 40):
        assert all(torch.equal(x, y) for x, y in zip(res[0][0], res[kv][0]))
        assert _same(res[0][1], res[kv][1]), kv


# ------------------------------------------------------------------------------------------
def test_rejections():
    eng = make_engine(llm=SMALL, max_batch=4, max_seq=480)
    d = lambda n: torch.empty(n, vn.LOGPROB_PLACES, dtype=torch.int32, device=DEV)   # noqa: E731
    f = lambda n: torch.empty(n, vn.LOGPROB_PLACES, dtype=torch.float32, device=DEV)  # noqa: E731
    with pytest.raises(vn.VclError, match="ever turned on"):
        eng.read_logprobs(0, 1, 1, d(1), f(1))
    for clips, top_n, msg in (([4], [1], "outside 0..3"), ([0, 0], [1, 1], "given twice"), ([1], [21], "top_n 21"),
                              ([1], [-2], "top_n -2")):
        with pytest.raises(vn.VclError, match=msg):
            eng.set_logprobs(clips, top_n)
    with pytest.raises(vn.VclError, match="n=0"):
        vn.check(vn.lib().vcl_llm_set_logprobs(eng._h, 0, None, None, None))
    eng.set_logprobs([2], [3])
    for entry, p0, n, msg in ((4, 0, 1, "entry 4"), (0, 480, 2, "positions"), (0, -1, 1, "positions"),
                              (0, 0, 0, "positions")):
        with pytest.raises(vn.VclError, match=msg):
            vn.check(vn.lib().vcl_llm_read_logprobs(eng._h, entry, p0, n, vn.ptr(d(2)), vn.ptr(f(2)), None))
    eng.read_logprobs(3, 480, 1)                   # the last position a decode loop can reach
    x = torch.zeros(2, 100, device=DEV)
    with pytest.raises(vn.VclError, match="top_n 21"):
        vn.Engine.sample_logprobs_op(x, [0.0, 0.0], [0, 0], [0, 0], [0, 0], [0, 21])
