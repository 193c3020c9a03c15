"""Paged KV cache (vcl_config.kv_blocks) against the contiguous cache, two engines with the same weights in one
process, at 7B width (2 layers) and 13B width (1 layer):

- packed prefill of prompts of 1 .. 512 tokens, with and without video, into scrambled block tables: every owned
  block equals the contiguous slot's columns bit for bit, the first tokens are equal, and no other column is written
  (NaN sentinel in every block beforehand);
- slot decode at 1 / 4 / 5 / 16 / 17 / 33 / 64 slots (gemv_tc, gemv_tcw with 1 / 2 / 4 clip groups, decode attention
  split 4 / 2 / 1) across block boundaries: tokens and every layer's cache bit-identical, equal launch counts, and a
  table rewritten (blocks moved) between replays of one graph;
- fp8 weights, paged against contiguous;
- generate_requests with 100 requests at 64 slots, video and text prompts, with a pool that never preempts and one
  that forces preemptions, packed admission on and off, greedy and seeded: identical to the contiguous model;
- rejections (static entry points, bad tables, long prompts, requests larger than the pool), after which the handle
  still works;
- the device memory a paged engine takes: the pool and the activations sized for min(max_seq, 512) rows."""
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import to_dev, vid_start_of  # noqa: E402
from test_padded_batch_gpu import video_feats  # noqa: E402
from test_inflight_gpu import text_prompt  # noqa: E402
from test_wide_slots_gpu import engine as _engine, model as _model, same  # noqa: E402

DEV = "cuda"
C = vn.KV_BLOCK_COLS
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)
W7B = O.LlmCfg(hidden=4096, inter=11008, heads=32, layers=2)
W13B = O.LlmCfg(hidden=5120, inter=13824, heads=40, layers=1)


def paged_model(cfg, max_batch, kv_blocks, max_seq=640):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    c = VideoChatGPTConfig(hidden_size=cfg.hidden, intermediate_size=cfg.inter, num_hidden_layers=cfg.layers,
                           num_attention_heads=cfg.heads, vocab_size=cfg.vocab, use_mm_proj=True, mm_hidden_size=1024)
    clip = dict(hidden_size=1024, intermediate_size=1024, num_hidden_layers=3, num_attention_heads=16)
    m = VideoChatGPTLlamaForCausalLM(c, clip_config=clip, max_batch=max_batch, max_seq=max_seq, max_slots=max_batch,
                                     kv_blocks=kv_blocks)
    vc = m.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = 32000, 32001, 32002, True
    return m


def engine(llm, max_batch, max_seq, max_slots, kv_blocks=0, sd=None, fmt="bf16"):
    c_eng = _engine(llm, max_batch, max_seq, max_slots)     # config template; replaced below when paged
    if not kv_blocks:
        if sd is not None:
            c_eng.load_llm(sd, weight_format=fmt)
        return c_eng
    cfg = c_eng.cfg
    c_eng.close()
    eng = vn.Engine(cfg, kv_blocks=kv_blocks)
    assert eng.cfg.kv_blocks == kv_blocks
    if sd is not None:
        eng.load_llm(sd, weight_format=fmt)
    return eng


@pytest.fixture(scope="module", params=["7b", "13b"])
def width(request):
    cfg = W7B if request.param == "7b" else W13B
    return cfg, to_dev(O.random_llm_state(cfg, seed=3))


def fill_nan(eng):
    buf = torch.full(eng.block_shape(), float("nan"), dtype=torch.bfloat16, device=DEV)
    for b in range(eng.kv_blocks):
        eng.kv_block_copy(b, buf, write=True)


def read_block(eng, b):
    return eng.kv_block_copy(b, torch.empty(eng.block_shape(), dtype=torch.bfloat16, device=DEV))


def gather(eng, table_row, n_cols, layer):
    """(k, v) [H, n_cols, 128] of one slot of a paged engine, read back block by block"""
    ks, vs = [], []
    for kb in range(-(-n_cols // C)):
        blk = read_block(eng, table_row[kb])
        ks.append(blk[layer, 0])
        vs.append(blk[layer, 1])
    return torch.cat(ks, 1)[:, :n_cols], torch.cat(vs, 1)[:, :n_cols]


def check_cache(paged, contig, table, slots_cols, what):
    for layer in range(contig.cfg.llm_layers):
        k, v = contig.kv_cache(layer)
        for s, n in slots_cols:
            pk, pv = gather(paged, table[s], n, layer)
            same(pk, k[s, :, :n], f"{what}: K of slot {s}, layer {layer}")
            same(pv, v[s, :, :n], f"{what}: V of slot {s}, layer {layer}")


def scrambled_table(eng, need, seed):
    """block rows for slots with need[s] blocks each, the blocks a random permutation of 1 .. kv_blocks-1"""
    perm = (torch.randperm(eng.kv_blocks - 1, generator=torch.Generator().manual_seed(seed)) + 1).tolist()
    table = [[0] * eng.table_row for _ in range(eng.n_slots)]
    for s, n in enumerate(need):
        table[s][:n] = [perm.pop() for _ in range(n)]
    return table


PREFILL_LENS = [1, 127, 128, 129, 300, 448, 512]


def prompts(cfg, lens, video=()):
    """prompt ids (host, [S]) and video features: prompts i in `video` carry a video span"""
    ids, feats, vs = [], [], []
    for i, S in enumerate(lens):
        if i in video:
            p = O.make_prompt_ids(cfg, 356, seed=40 + i, n_pre=S - 356 - 3 - 26)[0]
            ids.append(p)
            feats.append(video_feats(1, 50 + i)[0])
            vs.append(int(vid_start_of(p[None], cfg)[0]))
        else:
            ids.append(text_prompt(60 + i, S))
            feats.append(None)
            vs.append(0)
    return ids, feats, vs


@torch.no_grad()
def test_packed_prefill_into_scrambled_tables(width):
    cfg, sd = width
    lens = PREFILL_LENS + [448, 512]                         # 448 / 512 with and without video
    n = len(lens)
    need = [-(-S // C) for S in lens]
    paged = engine(cfg, n, 640, n, kv_blocks=sum(need) + 5, sd=sd)
    contig = engine(cfg, n, 640, n, sd=sd)
    fill_nan(paged)
    table = scrambled_table(paged, need, seed=1)
    paged.set_block_table(table)
    ids, feats, vs = prompts(cfg, lens, video={5, 8})              # 448 / 512 with video, and without
    assert sum(f is not None for f in feats) == 2
    slots = list(range(n))
    t_p = paged.slots_prefill(slots, ids, feats, vs)
    t_c = contig.slots_prefill(slots, ids, feats, vs)
    torch.cuda.synchronize()
    same(t_p, t_c, "first tokens")
    check_cache(paged, contig, table, list(zip(slots, lens)), "packed prefill")
    owned = {b for r in table for b in r if b}
    for s, S in enumerate(lens):              # the columns past S of a slot's last block are not written
        if S % C:
            assert torch.isnan(read_block(paged, table[s][need[s] - 1])[:, :, :, S % C:]).all(), f"slot {s}"
    for b in range(paged.kv_blocks):
        if b not in owned:
            assert torch.isnan(read_block(paged, b)).all(), f"block {b} owned by no table was written"
    # one prompt alone through slot_prefill (a packed prefill of one) into a fresh table row
    table2 = [[0] * paged.table_row for _ in range(n)]
    table2[3][:need[5]] = table[5][:need[5]]
    paged.set_block_table(table2)
    tok = paged.slot_prefill(3, ids[5].to(DEV)[None], feats[5], torch.tensor([vs[5]], dtype=torch.int32, device=DEV))
    same(tok, t_c[5:6], "slot_prefill on a paged engine")


DECODE_NB = [1, 4, 5, 16, 17, 33, 64]


@torch.no_grad()
@pytest.mark.parametrize("fmt", ["bf16", "fp8_e4m3"])
def test_slot_decode_across_blocks(width, fmt):
    cfg, sd = width
    if fmt == "fp8_e4m3" and cfg is W13B:
        pytest.skip("fp8 paged against contiguous is checked once, at 7B width")
    nb_list = DECODE_NB if fmt == "bf16" else [4, 33]
    NS, k = 64, 12
    lens = [110 + (7 * s) % 17 for s in range(NS)]                # decode crosses column 128 in every slot
    total = [S + (k - 1) * len(nb_list) + 1 for S in lens]
    need = [-(-t // C) for t in total]
    paged = engine(cfg, NS, 640, NS, kv_blocks=sum(need) + 8, sd=sd, fmt=fmt)
    contig = engine(cfg, NS, 640, NS, sd=sd, fmt=fmt)
    table = scrambled_table(paged, need, seed=2)
    paged.set_block_table(table)
    ids = [text_prompt(200 + s, S) for s, S in enumerate(lens)]
    first_p = paged.slots_prefill(list(range(NS)), ids, [None] * NS, [0] * NS)
    first_c = contig.slots_prefill(list(range(NS)), ids, [None] * NS, [0] * NS)
    same(first_p, first_c, "first tokens")
    pos = list(lens)
    for NB in nb_list:
        l0 = vn.launch_count()
        out_p = paged.slot_decode(first_p[:NB].contiguous(), pos[:NB], k)
        l1 = vn.launch_count()
        out_c = contig.slot_decode(first_c[:NB].contiguous(), pos[:NB], k)
        l2 = vn.launch_count()
        torch.cuda.synchronize()
        same(out_p, out_c, f"{fmt} tokens at {NB} slots")
        assert l1 - l0 == l2 - l1, f"launch counts at {NB} slots: {l1 - l0} vs {l2 - l1}"
        first_p[:NB] = out_p[:, -1]
        first_c[:NB] = out_c[:, -1]
        for s in range(NB):
            pos[s] += k - 1
        if NB == 17:
            # move every block of slots 0..16 to a free block and replay the same (17, k) graph with the new table
            owned = {b for r in table for b in r if b}
            spare = [b for b in range(1, paged.kv_blocks) if b not in owned]
            for s in range(2):
                for j in range(need[s]):
                    if spare:
                        nb_ = spare.pop()
                        paged.kv_block_copy(nb_, read_block(paged, table[s][j]), write=True)
                        table[s][j] = nb_
            paged.set_block_table(table)
            l0 = vn.launch_count()
            out_p = paged.slot_decode(first_p[:NB].contiguous(), pos[:NB], k)
            l1 = vn.launch_count()
            out_c = contig.slot_decode(first_c[:NB].contiguous(), pos[:NB], k)
            l2 = vn.launch_count()
            torch.cuda.synchronize()
            same(out_p, out_c, "tokens after the table was rewritten")
            assert l1 - l0 == l2 - l1
            first_p[:NB] = out_p[:, -1]
            first_c[:NB] = out_c[:, -1]
            for s in range(NB):
                pos[s] += k - 1
    check_cache(paged, contig, table, list(enumerate(pos)), f"{fmt} slot decode")


def _requests(cfg, n, seed):
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for i in range(n):
        nn = int(torch.randint(4, 72, (1,), generator=g))
        if i % 3 == 2:
            S = int(torch.randint(20, 300, (1,), generator=g))
            reqs.append(dict(input_ids=text_prompt(500 + i, S), max_new_tokens=nn))
        else:
            n_pre = int(torch.randint(14, 63, (1,), generator=g))        # 400 .. 448 tokens
            ids = O.make_prompt_ids(cfg, 356, seed=600 + i, n_pre=n_pre)
            reqs.append(dict(input_ids=ids, video_spatio_temporal_features=video_feats(1, 700 + i)[0].cpu(),
                             max_new_tokens=nn))
    return reqs


@torch.no_grad()
def test_generate_requests_paged_equals_contiguous():
    sd = O.random_llm_state(SMALL, seed=9)
    reqs = _requests(SMALL, 100, seed=4)
    ref_m = _model(SMALL, 64, max_slots=64, max_seq=640)
    ref_m.load_state_dict(sd)
    ref = {s: ref_m.generate_requests(reqs, eos_token_id=None, packed_admission=True,
                                      **(dict(do_sample=True, seed=s, temperature=0.7, top_k=20) if s else {}))
           for s in (0, 11)}
    for kv_blocks, preempts in ((400, False), (24, True)):
        m = paged_model(SMALL, 64, kv_blocks)
        m.load_state_dict(sd)
        for packed in (False, True):
            for s in (0, 11):
                out = m.generate_requests(reqs, eos_token_id=None, packed_admission=packed,
                                          **(dict(do_sample=True, seed=s, temperature=0.7, top_k=20) if s else {}))
                st = m.last_kv_stats
                what = f"kv_blocks {kv_blocks}, packed {packed}, seed {s}: {st}"
                assert len(out) == len(reqs)
                for i, (a, b) in enumerate(zip(out, ref[s])):
                    assert torch.equal(a.cpu(), b.cpu()), f"request {i}, {what}"
                assert (st["preemptions"] > 0) == preempts, what
                assert st["peak_blocks"] <= kv_blocks - 1
        m._engine.close()


@torch.no_grad()
def test_rejections_leave_the_handle_working():
    sd = to_dev(O.random_llm_state(SMALL, seed=12))
    eng = engine(SMALL, 4, 640, 4, kv_blocks=12, sd=sd)
    ids = O.make_prompt_ids(SMALL, 356, seed=1).to(DEV)
    vs = vid_start_of(ids, SMALL)
    tok1 = torch.zeros(1, dtype=torch.int32, device=DEV)
    calls = [lambda: eng.prefill(ids, None, vs), lambda: eng.prefill(ids, None, vs, n_pad=[0]),
             lambda: eng.prefill_states(ids, None, vs), lambda: eng.prefill_append(ids, 5),
             lambda: eng.decode_step(tok1, 3), lambda: eng.decode_loop(tok1, 3, 4),
             lambda: eng.generate(ids, None, vs, 4), lambda: eng.generate(ids, None, vs, 4, n_pad=[0]),
             lambda: eng.score(ids, None, vs), lambda: eng.kv_cache(0)]
    for f in calls:
        with pytest.raises(vn.VclError, match="generate_requests|vcl_kv_block_copy"):
            f()
    ok = [[0] * eng.table_row for _ in range(4)]
    ok[0][:4] = [3, 4, 5, 6]
    bad_range = [r[:] for r in ok]
    bad_range[1][0] = 12
    dup = [r[:] for r in ok]
    dup[2][0] = 4
    for t, msg in ((bad_range, "outside"), (dup, "twice")):
        with pytest.raises(vn.VclError, match=msg):
            eng.set_block_table(t)
    with pytest.raises(vn.VclError, match="outside 1..512"):
        eng.slots_prefill([0], [text_prompt(1, 513)], [None], [0])
    with pytest.raises(vn.VclError, match="block"):
        eng.kv_block_copy(12, torch.empty(eng.block_shape(), dtype=torch.bfloat16, device=DEV))
    m = paged_model(SMALL, 4, 3)
    m.load_state_dict(O.random_llm_state(SMALL, seed=12))
    with pytest.raises(ValueError, match="blocks"):
        m.generate_requests([dict(input_ids=text_prompt(2, 300), max_new_tokens=10)])     # 3 blocks > 2
    with pytest.raises(ValueError, match="512"):
        m.generate_requests([dict(input_ids=text_prompt(2, 513), max_new_tokens=10)])
    assert m._engine is None or m.last_kv_stats is None
    # the handle still works: the table that was rejected never reached it
    contig = engine(SMALL, 4, 640, 4, sd=sd)
    eng.set_block_table(ok)
    t_p = eng.slots_prefill([0], [ids[0].cpu()], [None], [0])
    t_c = contig.slots_prefill([0], [ids[0].cpu()], [None], [0])
    o_p = eng.slot_decode(t_p.repeat(4).contiguous(), [ids.shape[1], 0, 0, 0], 6)
    o_c = contig.slot_decode(t_c.repeat(4).contiguous(), [ids.shape[1], 0, 0, 0], 6)
    same(o_p[0], o_c[0], "tokens after the rejections")


def test_memory_is_pool_plus_activations():
    cfg, max_batch, max_seq, kv_blocks = W7B, 16, 1472, 40
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    contig = engine(cfg, max_batch, max_seq, max_batch)
    free1 = torch.cuda.mem_get_info()[0]
    contig.close()
    torch.cuda.synchronize()
    free2 = torch.cuda.mem_get_info()[0]
    paged = engine(cfg, max_batch, max_seq, max_batch, kv_blocks=kv_blocks)
    free3 = torch.cuda.mem_get_info()[0]
    paged.close()
    used_c, used_p = free0 - free1, free2 - free3
    D, F, L, H = cfg.hidden, cfg.inter, cfg.layers, cfg.heads
    cache_c = 2 * L * max_batch * H * max_seq * 128 * 2
    pool = kv_blocks * vn.kv_block_bytes(L, H)
    act_row = (6 * D + F) * 2 + 2 * 4               # l_h, l_x, l_qkv (3D), l_attn, l_act (F); the pack map
    rows_saved = max_batch * (max_seq - 512)
    want = used_c - cache_c + pool - rows_saved * act_row
    print(f"[paged] contiguous engine {used_c / 2**20:.1f} MiB, paged {used_p / 2**20:.1f} MiB, computed {want / 2**20:.1f} MiB")
    assert abs(used_p - want) <= 0.01 * want + 32 * 2 ** 20
