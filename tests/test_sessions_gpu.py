"""Conversation sessions on the paged KV cache (vcl_llm_slots_prefill_append, generate_requests with "session" /
"continues") against the contiguous engine's continued prefill (prefill_append, generate + generate_continue), two
engines with the same weights in one process, bit for bit (torch.equal):

- the append entry point at 7B width (2 layers) and 13B width (1 layer): slots prepared by a prompt and a few decode
  steps (copied into the contiguous engine's clip 0 before its prefill_append), then text tails of 1 / 37 / 65 / 512 rows at starts 1, 63, 64, 65, 200, 447 (wgmma kernel), 500, 577, 1000 and
  max_seq - len (flash kernel past 512 keys), both kernels in one launch, scrambled tables, NaN in every block no
  sequence owns: the next token, every cache column, and NaN past each end;
- the rejections of the entry point and of the model, after which both still serve;
- generate_requests over 3 turns of 6 conversations on 4 slots against the contiguous chain generate ->
  generate_continue -> generate_continue of each conversation alone: greedy with EOS and a KeywordsStoppingCriteria,
  and seeded sampling with per-request seeds; packed admission on and off; first turns over 512 tokens
  (chunked_prefill=True) and continuations whose context crosses column 512; a pool that keeps every conversation
  resident and one small enough that kept conversations are swapped out and running requests preempted; after every
  turn the kept blocks (or their host copies) equal the contiguous cache's columns 0 .. L - 2."""
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import to_dev  # noqa: E402
from test_inflight_gpu import text_prompt  # noqa: E402
from test_packed_prefill_gpu import _Tok  # noqa: E402
from test_padded_batch_gpu import video_feats  # noqa: E402
from test_wide_slots_gpu import model as _model, same  # noqa: E402
from test_paged_kv_gpu import (C, SMALL, W7B, W13B, engine, fill_nan, read_block, gather, scrambled_table,  # noqa: E402
                               paged_model)
from test_chunked_prefill_gpu import run_chunks  # noqa: E402

DEV = "cuda"
MAX_SEQ = 1536
DECODE = 3                     # decode steps between the prompt and the tail (the cache holds decode-written columns)


@pytest.fixture(scope="module", params=["7b", "13b"])
def width(request):
    cfg = W7B if request.param == "7b" else W13B
    return cfg, to_dev(O.random_llm_state(cfg, seed=31))


def cases():
    """(start, tail length, decode steps): the columns 0 .. start - 1 are a prompt of start - decode tokens and
    `decode` decoded ones"""
    wg = [(s, n, DECODE) for s in (63, 64, 65, 200, 447) for n in (1, 37, 65)]
    fl = [(s, n, DECODE) for s in (500, 577, 1000) for n in (1, 37, 65)] + [(MAX_SEQ - n, n, DECODE) for n in (1, 65)]
    return [(1, n, 0) for n in (1, 37, 65, 512)], wg + fl + [(64, 512, DECODE)]


def contiguous_append(contig, paged, row, start, tail):
    """the contiguous engine's continued prefill of one sequence (clip 0) on the columns 0 .. start - 1 the paged slot
    holds (its prompt and decode-written columns, copied over); returns the token after the tail and the K / V
    columns 0 .. start + len - 1 of every layer"""
    for layer in range(contig.cfg.llm_layers):
        k, v = contig.kv_cache(layer)
        pk, pv = gather(paged, row, start, layer)
        k[0, :, :start], v[0, :, :start] = pk, pv
        contig.set_kv_cache(layer, k, v)
    _, _, nxt = contig.prefill_append(tail.to(DEV)[None], start)
    end = start + tail.numel()
    kv = [tuple(t[0, :, :end].clone() for t in contig.kv_cache(layer)) for layer in range(contig.cfg.llm_layers)]
    return nxt, kv


@torch.no_grad()
def test_append_equals_contiguous_prefill_append(width):
    cfg, sd = width
    groups = cases()
    n = max(len(g) for g in groups)
    contig = engine(cfg, 1, MAX_SEQ, 1, sd=sd)
    for gi, group in enumerate(groups):
        need = [-(-(s + ln) // C) for s, ln, _ in group]
        paged = engine(cfg, n, MAX_SEQ, n, kv_blocks=sum(need) + 3, sd=sd)
        fill_nan(paged)
        table = scrambled_table(paged, need, seed=40 + gi)
        paged.set_block_table(table)
        slots = list(range(len(group)))
        prompts = [text_prompt(500 + 7 * i + gi, s - d) for i, (s, _, d) in enumerate(group)]
        tails = [text_prompt(900 + 5 * i + gi, ln + 1)[1:] for i, (_, ln, _) in enumerate(group)]
        first = run_chunks(paged, slots, [(p, None, 0) for p in prompts], [[512]] * len(group))
        d = group[0][2]
        if d:
            fed = torch.zeros(paged.n_slots, dtype=torch.int32, device=DEV)
            fed[:len(group)] = first
            pos = [p.numel() for p in prompts] + [0] * (paged.n_slots - len(group))
            paged.slot_decode(fed, pos, d + 1)
        nxt = paged.slots_prefill_append(slots, [s for s, _, _ in group], tails)
        torch.cuda.synchronize()
        assert any(s + ln > 512 for s, ln, _ in group) and any(s + ln <= 512 for s, ln, _ in group)
        for i, (s, ln, _) in enumerate(group):
            what = f"{cfg.hidden}: start {s}, tail {ln}"
            t_c, kv = contiguous_append(contig, paged, table[i], s, tails[i])
            torch.cuda.synchronize()
            same(nxt[i:i + 1], t_c, f"{what}: next token")
            for layer, (k, v) in enumerate(kv):
                pk, pv = gather(paged, table[i], s + ln, layer)
                same(pk, k, f"{what}: K, layer {layer}")
                same(pv, v, f"{what}: V, layer {layer}")
            if (s + ln) % C:
                assert torch.isnan(read_block(paged, table[i][need[i] - 1])[:, :, :, (s + ln) % C:]).all(), what
        owned = {b for r in table for b in r if b}
        for b in range(paged.kv_blocks):
            if b not in owned:
                assert torch.isnan(read_block(paged, b)).all(), f"block {b} owned by no table was written"
        paged.close()
    contig.close()


@torch.no_grad()
def test_rejections_leave_the_handle_and_the_model_working():
    sd = to_dev(O.random_llm_state(SMALL, seed=33))
    eng = engine(SMALL, 4, 1024, 4, kv_blocks=20, sd=sd)
    contig = engine(SMALL, 4, 1024, 4, sd=sd)
    t = text_prompt(3, 40)

    def app(e, slots, starts, lens):
        return e.slots_prefill_append(slots, starts, [t[:n] if n <= 40 else text_prompt(4, n) for n in lens])
    with pytest.raises(vn.VclError, match="contiguous"):
        app(contig, [0], [10], [5])
    bad = [(([0, 1, 2, 3, 0], [10] * 5, [5] * 5), "n=5 outside"),
           (([1, 1], [10, 10], [5, 5]), "twice"),
           (([4], [10], [5]), "slot 4 outside"),
           (([0], [0], [5]), "start >= 1"),
           (([0], [10], [513]), "outside 1..512"),
           (([0], [1000], [30]), "outside the cache")]
    for args, msg in bad:
        with pytest.raises(vn.VclError, match=msg):
            app(eng, *args)
    table = [[0] * eng.table_row for _ in range(4)]
    table[2][:2] = [7, 3]
    eng.set_block_table(table)
    p = text_prompt(5, 150)
    eng.slots_prefill([2], [p], [None], [0])
    t_p = app(eng, [2], [150], [40])
    contig.prefill(p.to(DEV)[None], None, torch.tensor([vn.NO_VIDEO], dtype=torch.int32, device=DEV))
    _, _, t_c = contig.prefill_append(t.to(DEV)[None], 150)
    torch.cuda.synchronize()
    same(t_p, t_c, "next token after the rejections")
    eng.close()
    contig.close()

    m = paged_model(SMALL, 4, 12, max_seq=1024)
    m.load_state_dict(O.random_llm_state(SMALL, seed=33))
    m.generate_requests([dict(input_ids=text_prompt(6, 100), max_new_tokens=5, session="a")], eos_token_id=None)
    tail = text_prompt(7, 20)
    for reqs, msg in [([dict(input_ids=tail, continues="b")], "no conversation"),
                      ([dict(input_ids=tail, session="a")], "already kept"),
                      ([dict(input_ids=tail, continues="a"), dict(input_ids=tail, continues="a")], "also continued"),
                      ([dict(input_ids=text_prompt(8, 600), continues="a")], "rows"),
                      ([dict(input_ids=tail, continues="a", max_new_tokens=920)], "max_seq")]:
        with pytest.raises(ValueError, match=msg):
            m.generate_requests(reqs)
    out = m.generate_requests([dict(input_ids=tail, continues="a", max_new_tokens=4)], eos_token_id=None)
    assert out[0].shape == (1, 100 + 5 + 20 + 4)
    m.end_session()
    c = _model(SMALL, 1, max_slots=1)
    with pytest.raises(ValueError, match="paged"):
        c.generate_requests([dict(input_ids=tail, session="x")])


N_CONV, TURNS = 6, 3


def conversations():
    """[conv][turn] -> (ids [S] host, feats or None, max_new_tokens); first turns of 200 .. 700 tokens, some with
    video, follow-ups of 16 .. 48 tokens"""
    g = torch.Generator().manual_seed(7)
    first = [(450, True), (700, False), (300, False), (620, True), (480, False), (200, False)]
    out = []
    for c, (S, vid) in enumerate(first):
        turns = []
        for t in range(TURNS):
            n = int(torch.randint(8, 48, (1,), generator=g))
            if t == 0 and vid:
                n_pre = 20 + c
                ids = O.make_prompt_ids(SMALL, 356, seed=300 + c, n_pre=n_pre, n_post=S - 359 - n_pre)[0]
                turns.append((ids, video_feats(1, 310 + c)[0].cpu(), n))
            elif t == 0:
                turns.append((text_prompt(320 + c, S), None, n))
            else:
                k = int(torch.randint(16, 49, (1,), generator=g))
                turns.append((text_prompt(330 + 10 * c + t, k + 1)[1:], None, n))
        out.append(turns)
    return out


def criteria(mode, ids, kw):
    from video_chatgpt.model.utils import KeywordsStoppingCriteria
    return [KeywordsStoppingCriteria([f"t{kw}."], _Tok(), ids[None])] if mode == "greedy" and kw is not None else None


def samp(mode, c, t):
    return dict(do_sample=True, seed=1000 + 10 * c + t, temperature=0.7, top_k=40) if mode == "seeded" else {}


def chain(ref, convs, mode, eos, kws):
    """each conversation alone on the contiguous model: generate, then generate_continue per turn. Returns the
    outputs [conv][turn] and the cache columns 0 .. L - 2 of every layer after every turn"""
    outs, caches = [], []
    for c, turns in enumerate(convs):
        o, kv = [], []
        for t, (ids, f, n) in enumerate(turns):
            kw = dict(max_new_tokens=n, eos_token_id=eos, stopping_criteria=criteria(mode, ids, kws[c][t]),
                      **samp(mode, c, t))
            if t == 0:
                r = ref.generate(ids[None], video_spatio_temporal_features=None if f is None else f[None].to(DEV), **kw)
            else:
                r = ref.generate_continue(ids[None].to(DEV), **kw)
            o.append(r.cpu())
            L = r.shape[1]
            kv.append([tuple(x[0, :, :L - 1].cpu() for x in ref._engine.kv_cache(layer))
                       for layer in range(SMALL.layers)])
        outs.append(o)
        caches.append(kv)
    return outs, caches


def check_kept(m, eng, caches, t, what):
    for c, ss in m._sessions.items():
        L = ss.ids.numel()
        for layer in range(SMALL.layers):
            k, v = caches[c][t][layer]
            if ss.blocks is not None:
                pk, pv = gather(eng, ss.blocks, L - 1, layer)
            else:
                pk = torch.cat([b[layer, 0] for b in ss.saved], 1)[:, :L - 1]
                pv = torch.cat([b[layer, 1] for b in ss.saved], 1)[:, :L - 1]
            same(pk.cpu(), k, f"{what}: conversation {c}, turn {t}, K layer {layer}")
            same(pv.cpu(), v, f"{what}: conversation {c}, turn {t}, V layer {layer}")


@torch.no_grad()
def test_generate_requests_sessions_equal_contiguous_chain():
    sd = O.random_llm_state(SMALL, seed=35)
    convs = conversations()
    ref = _model(SMALL, 1, max_slots=1, max_seq=2048)
    ref.load_state_dict(sd)
    # EOS: a token conversation 1 produces early in a free greedy run; a keyword on two conversations' later turns
    free, _ = chain(ref, convs, "greedy", None, [[None] * TURNS] * N_CONV)
    eos = int(free[1][0][0, -convs[1][0][2] + 3])
    kws = [[None] * TURNS for _ in range(N_CONV)]
    for c in (2, 4):
        a = free[c][1][0].tolist()
        kws[c][1] = a[len(a) - convs[c][1][2] // 2]
    refs = {mode: chain(ref, convs, mode, eos, kws) for mode in ("greedy", "seeded")}
    ref._engine.close()
    assert refs["greedy"][0][1][0].shape[1] < free[1][0].shape[1]                     # EOS fired
    assert any(convs[c][0][0].numel() > 512 for c in range(N_CONV))
    # a continuation whose tail starts below column 512 and ends past it (the flash kernel over the kept columns)
    spans = [(o[t - 1].shape[1] - 1, o[t - 1].shape[1] + convs[c][t][0].numel())
             for mode in refs for c, o in enumerate(refs[mode][0]) for t in range(1, TURNS)]
    assert any(a < 512 < b for a, b in spans), spans
    for kv_blocks, tight in ((100, False), (14, True)):
        m = paged_model(SMALL, 4, kv_blocks, max_seq=2048)
        m.load_state_dict(sd)
        preempted = 0
        for packed in (False, True):
            for mode in ("greedy", "seeded"):
                r_out, r_kv = refs[mode]
                what = f"kv_blocks {kv_blocks}, packed {packed}, {mode}"
                totals = dict(preemptions=0, session_swaps=0, reused_rows=0)
                for t in range(TURNS):
                    reqs = []
                    for c, turns in enumerate(convs):
                        ids, f, n = turns[t]
                        r = dict(input_ids=ids, max_new_tokens=n, stopping_criteria=criteria(mode, ids, kws[c][t]),
                                 **samp(mode, c, t))
                        if t == 0:
                            r["session"] = c
                            if f is not None:
                                r["video_spatio_temporal_features"] = f
                        else:
                            r["continues"] = c
                        reqs.append(r)
                    out = m.generate_requests(reqs, eos_token_id=eos, packed_admission=packed, chunked_prefill=True)
                    st = m.last_kv_stats
                    for k in totals:
                        totals[k] += st[k]
                    for c in range(N_CONV):
                        assert torch.equal(out[c].cpu(), r_out[c][t]), f"{what}: conversation {c}, turn {t}: {st}"
                    assert st["sessions"] == N_CONV, what
                    check_kept(m, m._engine, r_kv, t, what)
                assert totals["reused_rows"] == sum(r_out[c][t].shape[1] - 1 for c in range(N_CONV)
                                                    for t in range(TURNS - 1)), what
                if tight:
                    assert totals["session_swaps"] > 0, f"{what}: {totals}"
                else:
                    assert totals["preemptions"] == 0 and totals["session_swaps"] == 0, f"{what}: {totals}"
                preempted += totals["preemptions"]
                m.end_session()
        assert (preempted > 0) == tight, f"kv_blocks {kv_blocks}: {preempted} preemptions"
        m._engine.close()
