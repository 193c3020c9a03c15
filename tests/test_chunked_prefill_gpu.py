"""Chunked prefill on the paged KV cache (vcl_llm_slots_prefill_chunk, generate_requests(chunked_prefill=True))
against the contiguous engine's one-shot prefill of the whole prompt, two engines with the same weights in one
process, bit for bit (torch.equal):

- prompts of 513 / 577 / 640 / 1000 / 1471 / max_seq - 1 tokens, text only and with a video span (two of them
  straddling column 512), cut into chunks of 512 rows and into chunks of 64 / 192 / 448 rows: every owned cache
  column read back block by block and the first token, with NaN in every block no sequence owns and in the columns
  past each prompt, at 7B width (2 layers) and 13B width (1 layer);
- the packed flash attention with different starts in one launch (0, 512 and 960), next to a whole short prompt on
  the wgmma kernel in the same call;
- the rejections of the new entry point, after which the handle still works;
- generate_requests with prompts of 100 .. 1500 tokens against a contiguous model with max_seq 2048: greedy and
  seeded sampling, packed admission on and off, with a pool that never preempts and one that swaps out a long
  request."""
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import to_dev  # noqa: E402
from test_padded_batch_gpu import video_feats  # noqa: E402
from test_inflight_gpu import text_prompt  # noqa: E402
from test_wide_slots_gpu import model as _model, same  # noqa: E402
from test_paged_kv_gpu import (C, SMALL, W7B, W13B, engine, fill_nan, read_block, check_cache,  # noqa: E402
                               scrambled_table, paged_model)

DEV = "cuda"
MAX_SEQ = 1536
LONG = [513, 577, 640, 1000, 1471, MAX_SEQ - 1]


@pytest.fixture(scope="module", params=["7b", "13b"])
def width(request):
    cfg = W7B if request.param == "7b" else W13B
    return cfg, to_dev(O.random_llm_state(cfg, seed=5))


def long_prompt(cfg, S, seed, n_pre=None):
    """(ids [S] host, feats or None, vid_start): n_pre given -> a video span after n_pre + 1 tokens"""
    if n_pre is None:
        return text_prompt(seed, S), None, 0
    ids = O.make_prompt_ids(cfg, 356, seed=seed, n_pre=n_pre, n_post=S - 359 - n_pre)[0]
    return ids, video_feats(1, seed)[0], n_pre + 1


def run_chunks(eng, slots, prompts, cuts):
    """prefill every prompt (ids, feats, vs) into its slot through chunk calls: cuts[i] the chunk lengths of prompt
    i, cycled; round k packs chunk k of every prompt that has one. Returns the last chunk's token of each."""
    starts = [0] * len(prompts)
    first = [None] * len(prompts)
    k = 0
    while any(st < p[0].numel() for st, p in zip(starts, prompts)):
        live = [i for i, p in enumerate(prompts) if starts[i] < p[0].numel()]
        lens = [min(cuts[i][k % len(cuts[i])], prompts[i][0].numel() - starts[i]) for i in live]
        tok = eng.slots_prefill_chunk([slots[i] for i in live], [starts[i] for i in live],
                                      [prompts[i][0].numel() for i in live],
                                      [prompts[i][0][starts[i]:starts[i] + n] for i, n in zip(live, lens)],
                                      [prompts[i][1] for i in live], [prompts[i][2] for i in live])
        for j, (i, n) in enumerate(zip(live, lens)):
            starts[i] += n
            if starts[i] == prompts[i][0].numel():
                first[i] = tok[j:j + 1]
        k += 1
    return torch.cat(first)


def contiguous_first(contig, slots, prompts):
    out = []
    for s, (ids, f, vs) in zip(slots, prompts):
        out.append(contig.slot_prefill(s, ids.to(DEV)[None], f, torch.tensor([vs], dtype=torch.int32, device=DEV)))
    return torch.cat(out)


@torch.no_grad()
@pytest.mark.parametrize("cuts", ["512", "64-192-448"])
def test_chunked_prefill_equals_one_shot(width, cuts):
    cfg, sd = width
    # video spans: rows 202..557 of the 640-token prompt and 402..757 of the 1000-token one straddle column 512;
    # 1471 carries its span in its first chunk; 300 is a whole short prompt on the wgmma kernel in the same calls
    prompts = [long_prompt(cfg, 513, 1), long_prompt(cfg, 577, 2), long_prompt(cfg, 640, 3, n_pre=200),
               long_prompt(cfg, 1000, 4, n_pre=400), long_prompt(cfg, 1471, 5, n_pre=100),
               long_prompt(cfg, MAX_SEQ - 1, 6), long_prompt(cfg, 300, 7)]
    n = len(prompts)
    lens = [p[0].numel() for p in prompts]
    assert lens[:6] == LONG
    need = [-(-S // C) for S in lens]
    paged = engine(cfg, n, MAX_SEQ, n, kv_blocks=sum(need) + 4, sd=sd)
    contig = engine(cfg, n, MAX_SEQ, n, sd=sd)
    fill_nan(paged)
    table = scrambled_table(paged, need, seed=11)
    paged.set_block_table(table)
    slots = list(range(n))
    chunk = [[512]] * n if cuts == "512" else [[64, 192, 448], [448, 64], [192], [64, 448], [448], [192, 64], [300]]
    t_p = run_chunks(paged, slots, prompts, chunk)
    t_c = contiguous_first(contig, slots, prompts)
    torch.cuda.synchronize()
    same(t_p, t_c, f"first tokens, chunks {cuts}")
    check_cache(paged, contig, table, list(zip(slots, lens)), f"chunked prefill, chunks {cuts}")
    owned = {b for r in table for b in r if b}
    for s, S in enumerate(lens):
        if S % C:
            assert torch.isnan(read_block(paged, table[s][need[s] - 1])[:, :, :, S % C:]).all(), f"slot {s}"
    for b in range(paged.kv_blocks):
        if b not in owned:
            assert torch.isnan(read_block(paged, b)).all(), f"block {b} owned by no table was written"
    paged.close()
    contig.close()


@torch.no_grad()
def test_one_launch_with_starts_0_512_960(width):
    """three 1100-token prompts brought to different points, then one chunk call at starts 0 / 512 / 960"""
    cfg, sd = width
    prompts = [long_prompt(cfg, 1100, 20 + i, n_pre=(None, 600, None)[i]) for i in range(3)]
    need = [-(-1100 // C)] * 3
    paged = engine(cfg, 3, MAX_SEQ, 3, kv_blocks=sum(need) + 6, sd=sd)
    contig = engine(cfg, 3, MAX_SEQ, 3, sd=sd)
    fill_nan(paged)
    table = scrambled_table(paged, need, seed=12)
    paged.set_block_table(table)

    def call(items):
        return paged.slots_prefill_chunk([i for i, _, _ in items], [st for _, st, _ in items],
                                         [1100] * len(items), [prompts[i][0][st:st + n] for i, st, n in items],
                                         [prompts[i][1] for i, _, _ in items], [prompts[i][2] for i, _, _ in items])
    call([(1, 0, 512), (2, 0, 512)])
    call([(2, 512, 448)])
    tok_a = call([(0, 0, 512), (1, 512, 448), (2, 960, 140)])        # the launch under test
    tok_b = call([(0, 512, 512), (1, 960, 140)])
    tok_c = call([(0, 1024, 76)])
    first = torch.stack([tok_c[0], tok_b[1], tok_a[2]])
    t_c = contiguous_first(contig, [0, 1, 2], prompts)
    torch.cuda.synchronize()
    same(first, t_c, "first tokens")
    check_cache(paged, contig, table, [(s, 1100) for s in range(3)], "starts 0 / 512 / 960")
    owned = {b for r in table for b in r if b}
    for b in range(paged.kv_blocks):
        if b not in owned:
            assert torch.isnan(read_block(paged, b)).all(), f"block {b} owned by no table was written"
    paged.close()
    contig.close()


@torch.no_grad()
def test_chunk_rejections_leave_the_handle_working():
    sd = to_dev(O.random_llm_state(SMALL, seed=13))
    eng = engine(SMALL, 4, 1024, 4, kv_blocks=20, sd=sd)
    contig = engine(SMALL, 4, 1024, 4, sd=sd)
    ids = text_prompt(3, 700)

    def chunk(e, slots, starts, lens, totals):
        return e.slots_prefill_chunk(slots, starts, totals, [ids[st:st + n] for st, n in zip(starts, lens)],
                                     [None] * len(slots), [0] * len(slots))
    with pytest.raises(vn.VclError, match="contiguous"):
        chunk(contig, [0], [0], [512], [700])
    bad = [(dict(slots=[0, 1, 2, 3, 0], starts=[0] * 5, lens=[8] * 5, totals=[600] * 5), "n=5 outside"),
           (dict(slots=[0, 0], starts=[0, 0], lens=[8, 8], totals=[600, 600]), "twice"),
           (dict(slots=[4], starts=[0], lens=[8], totals=[600]), "slot 4 outside"),
           (dict(slots=[0], starts=[32], lens=[8], totals=[600]), "multiple of 64"),
           (dict(slots=[0], starts=[0], lens=[513], totals=[700]), "outside 1..512"),
           (dict(slots=[0], starts=[512], lens=[0], totals=[700]), "outside 1..512|null argument"),
           (dict(slots=[0], starts=[512], lens=[188], totals=[600]), "past its prompt"),
           (dict(slots=[0], starts=[0], lens=[512], totals=[1025]), "exceeds max_seq"),
           (dict(slots=[0], starts=[0], lens=[256], totals=[400]), "whole")]
    for kw, msg in bad:
        with pytest.raises(vn.VclError, match=msg):
            chunk(eng, **kw)
    with pytest.raises(vn.VclError, match="outside 1..512"):          # the packed prefill keeps its limit
        eng.slots_prefill([0], [text_prompt(1, 513)], [None], [0])
    # the handle still works
    table = [[0] * eng.table_row for _ in range(4)]
    table[1][:6] = [7, 3, 9, 12, 5, 14]
    eng.set_block_table(table)
    chunk(eng, [1], [0], [512], [700])
    t_p = chunk(eng, [1], [512], [188], [700])
    t_c = contig.slot_prefill(1, ids.to(DEV)[None], None, torch.tensor([0], dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    same(t_p, t_c, "first token after the rejections")
    check_cache(eng, contig, table, [(1, 700)], "after the rejections")
    m = paged_model(SMALL, 4, 20, max_seq=1024)
    m.load_state_dict(O.random_llm_state(SMALL, seed=13))
    with pytest.raises(ValueError, match="512"):
        m.generate_requests([dict(input_ids=text_prompt(2, 513), max_new_tokens=10)])


def _requests(cfg, n, seed):
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for i in range(n):
        nn = int(torch.randint(4, 60, (1,), generator=g))
        S = int(torch.randint(100, 1501, (1,), generator=g))
        if i % 3 == 1 and S >= 420:
            n_pre = int(torch.randint(10, S - 400, (1,), generator=g))
            ids = O.make_prompt_ids(cfg, 356, seed=800 + i, n_pre=n_pre, n_post=S - 359 - n_pre)
            reqs.append(dict(input_ids=ids, video_spatio_temporal_features=video_feats(1, 900 + i)[0].cpu(),
                             max_new_tokens=nn))
        else:
            reqs.append(dict(input_ids=text_prompt(700 + i, S), max_new_tokens=nn))
    return reqs


@torch.no_grad()
def test_generate_requests_chunked_equals_contiguous():
    sd = O.random_llm_state(SMALL, seed=14)
    reqs = _requests(SMALL, 24, seed=6)
    assert sum(r["input_ids"].numel() > 512 for r in reqs) >= 8
    ref_m = _model(SMALL, 8, max_slots=8, max_seq=2048)
    ref_m.load_state_dict(sd)
    samp = {0: {}, 11: dict(do_sample=True, seed=11, temperature=0.2, top_k=50)}
    ref = {s: ref_m.generate_requests(reqs, eos_token_id=None, **kw) for s, kw in samp.items()}
    ref_m._engine.close()
    for kv_blocks, preempts in ((120, False), (20, True)):
        m = paged_model(SMALL, 8, kv_blocks, max_seq=2048)
        m.load_state_dict(sd)
        for packed in (False, True):
            for s, kw in samp.items():
                out = m.generate_requests(reqs, eos_token_id=None, packed_admission=packed, chunked_prefill=True,
                                          **kw)
                st = m.last_kv_stats
                what = f"kv_blocks {kv_blocks}, packed {packed}, seed {s}: {st}"
                for i, (a, b) in enumerate(zip(out, ref[s])):
                    assert torch.equal(a.cpu(), b.cpu()), f"request {i}, {what}"
                assert (st["preemptions"] > 0) == preempts, what
                assert st["chunked_prefills"] >= sum(r["input_ids"].numel() > 512 for r in reqs), what
                assert st["chunk_calls"] >= 2 and st["peak_blocks"] <= kv_blocks - 1, what
        m._engine.close()
