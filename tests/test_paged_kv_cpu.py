"""CPU tests of generate_requests on a paged KV cache, driven by a fake engine that models the block pool, the block
table and the swap copies. Its tokens are a function of what the cache holds (read through the table), the slot's
sampling entry and the position, so a wrong table, a lost block or a wrong restore changes them. The same fake with
a contiguous cache is the yardstick."""
import ctypes

import pytest
import torch

V = 32003
EOS = 31999
C = 128                       # columns per block
REQ0 = 40000                  # request r's prompt starts with REQ0 + r; generated tokens stay below 30002


def _tok(vals, col, seed):
    """the token at column col + 1, from the cache columns 0 .. col"""
    h = seed * 7919 + col
    for j, v in enumerate(vals):
        h = (h * 31 + (j + 1) * v) % 1000003
    return h % 30000 + 1


class FakeEngine:
    NV = 356

    def __init__(self, max_seq, n_slots, kv_blocks=0, lens=None):
        self.max_seq, self.n_slots, self.kv_blocks = max_seq, n_slots, kv_blocks
        self.table_row = -(-max_seq // C)
        self.block_bytes = C * 4
        self.lens = lens or {}                # request -> S + n: the columns it may read
        self.calls, self.events, self.violations = [], [], []
        self.seed = [0] * n_slots
        if kv_blocks:
            self.pool = [[0] * C for _ in range(kv_blocks)]
            self.table = [[0] * self.table_row for _ in range(n_slots)]
        else:
            self.cache = [[0] * max_seq for _ in range(n_slots)]
        self.running = []                     # requests in admission order (paged)
        self.owner = {}                       # slot -> request, from the table (paged)

    # ---- cache access ----
    def _loc(self, s, c):
        return self.table[s][c // C], c % C

    def _write(self, s, c, v):
        if not self.kv_blocks:
            self.cache[s][c] = v
            return
        b, o = self._loc(s, c)
        if b == 0 and s in self.owner and c < self.lens[self.owner[s]]:
            self.violations.append(("uncovered", s, self.owner[s], c))
        self.pool[b][o] = v

    def _read(self, s, n):
        if not self.kv_blocks:
            return self.cache[s][:n]
        return [self.pool[self._loc(s, c)[0]][c % C] for c in range(n)]

    # ---- engine interface ----
    def set_sampling(self, clips, temperature, top_k, seed):
        for s, t, sd in zip(clips, temperature, seed):
            self.seed[s] = sd if t > 0 else 0

    def set_block_table(self, table):
        assert self.kv_blocks
        rows = [list(map(int, r)) for r in table]
        assert len(rows) == self.n_slots and all(len(r) == self.table_row for r in rows)
        live = [b for r in rows for b in r if b != 0]
        if len(live) != len(set(live)):
            self.violations.append(("shared block", live))
        assert all(0 <= b < self.kv_blocks for b in live)
        self.table = rows
        owner = {}
        for s, r in enumerate(rows):
            if r[0] != 0 and self.pool[r[0]][0] >= REQ0:
                owner[s] = self.pool[r[0]][0] - REQ0
        for s, r in self.owner.items():            # a request that left its slot without a swap has finished
            if owner.get(s) != r and r in self.running:
                self.running.remove(r)
                self.events.append(("finish", r))
        self.owner = owner

    def _prefill(self, s, ids):
        ids = [int(t) for t in ids.reshape(-1)]
        for c, t in enumerate(ids):
            self._write(s, c, t)
        r = ids[0] - REQ0
        self.running.append(r)
        self.events.append(("admit", r))
        if self.kv_blocks:
            self.owner[s] = r
        return _tok(self._read(s, len(ids)), len(ids) - 1, self.seed[s])

    def slot_prefill(self, slot, ids, video_feats, vid_start, tok_out=None):
        self.calls.append(("prefill", slot))
        tok_out[0] = self._prefill(slot, ids)
        return tok_out

    def slots_prefill(self, slots, ids_list, feats_list, vid_starts, tok_out=None):
        self.calls.append(("packed", list(slots)))
        return torch.tensor([self._prefill(s, torch.as_tensor(i)) for s, i in zip(slots, ids_list)], dtype=torch.int32)

    def slot_decode(self, first_tok, positions, n_new):
        self.calls.append(("decode", list(positions), n_new))
        out = torch.zeros(first_tok.shape[0], n_new, dtype=torch.int32)
        out[:, 0] = first_tok
        for s in range(first_tok.shape[0]):
            p = positions[s]
            for j in range(1, n_new):
                self._write(s, p + j - 1, int(out[s, j - 1]))
                out[s, j] = _tok(self._read(s, p + j), p + j - 1, self.seed[s])
        return out

    def swap_buffer(self):
        return torch.zeros(C, dtype=torch.int32)

    def kv_block_copy(self, block, buf, write=False):
        self.calls.append(("copy", block, write))
        if write:
            self.pool[block] = buf.tolist()
            if buf[0] >= REQ0:                      # a request's first block: it resumes
                r = int(buf[0]) - REQ0
                self.running.append(r)
                self.events.append(("resume", r))
        else:
            buf[:] = torch.tensor(self.pool[block], dtype=torch.int32)
            if self.pool[block][0] >= REQ0 and any(t[0] == block for t in self.table):
                r = self.pool[block][0] - REQ0
                if not self.running or self.running[-1] != r:
                    self.violations.append(("not the latest admission", r, list(self.running)))
                self.running.remove(r)
                self.events.append(("swap", r))
        return buf


def _model(eng, max_batch=4, max_seq=640, kv_blocks=None):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    cfg = VideoChatGPTConfig(hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4,
                             vocab_size=V, eos_token_id=EOS)
    m = VideoChatGPTLlamaForCausalLM(cfg, clip_config={}, max_batch=max_batch, max_seq=max_seq, max_slots=max_batch,
                                     kv_blocks=kv_blocks)
    m.device = torch.device("cpu")
    m._engine, m._llm_loaded = eng, True
    return m


def _reqs(shape):
    return [dict(input_ids=torch.tensor([REQ0 + r] + [7 + r % 5] * (S - 1)), max_new_tokens=n)
            for r, (S, n) in enumerate(shape)]


SHAPE = [(100, 60), (300, 150), (40, 200), (250, 30), (128, 128), (1, 5), (200, 240), (60, 100), (127, 1), (129, 90)]


def _run(kv_blocks, shape=SHAPE, slots=4, packed=False, seed=None, chunk=8):
    lens = {r: S + n for r, (S, n) in enumerate(shape)}
    eng = FakeEngine(640, slots, kv_blocks, lens)
    m = _model(eng, max_batch=slots, kv_blocks=kv_blocks or None)
    m._SLOT_CHUNK = chunk
    kw = dict(do_sample=True, seed=seed, temperature=0.5) if seed is not None else {}
    outs = m.generate_requests(_reqs(shape), eos_token_id=None, packed_admission=packed, **kw)
    return [o[0].tolist() for o in outs], eng, m


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("seed", [None, 5])
def test_paged_equals_contiguous_for_every_pool(packed, seed):
    ref, _, _ = _run(0, packed=packed, seed=seed)
    need = max(-(-(S + n) // C) for S, n in SHAPE)          # the largest request alone
    pre = []
    for kv in (need + 1, need + 2, 8, 12, 40):
        out, eng, m = _run(kv, packed=packed, seed=seed)
        assert out == ref, f"kv_blocks {kv}"
        assert eng.violations == [], eng.violations[:3]
        st = m.last_kv_stats
        assert 1 <= st["peak_blocks"] <= kv - 1
        pre.append(st["preemptions"])
        if st["preemptions"]:
            assert st["swapped_bytes"] > 0
    assert pre[0] > 0 and pre[-1] == 0          # just large enough for one request preempts; 40 blocks never do


def test_swapped_requests_resume_first_with_their_state():
    out, eng, m = _run(5, chunk=4)
    ref, _, _ = _run(0, chunk=4)
    assert out == ref and eng.violations == []
    ev = eng.events
    assert any(e[0] == "swap" for e in ev)
    waiting = set()
    for e in ev:
        if e[0] == "swap":
            waiting.add(e[1])
        elif e[0] == "resume":
            waiting.discard(e[1])
        elif e[0] == "admit":
            assert not waiting, f"request {e[1]} admitted while {waiting} waited in host memory"
    admits = [e[1] for e in ev if e[0] == "admit"]
    assert admits == sorted(admits) == list(range(len(SHAPE)))        # queue order, no overtaking


def test_chunks_cover_their_columns_and_idle_slots_park():
    out, eng, _ = _run(6, slots=4)
    assert eng.violations == []
    # after the run every slot is parked: its table row points at block 0 only
    assert all(b == 0 for r in eng.table for b in r)
    for c in eng.calls:
        if c[0] == "decode":
            assert max(c[1]) + c[2] - 1 <= 640


def test_rejections_before_any_device_call():
    eng = FakeEngine(640, 4, 4)
    m = _model(eng, kv_blocks=4)
    with pytest.raises(ValueError, match="512"):
        m.generate_requests([dict(input_ids=torch.tensor([REQ0] * 513), max_new_tokens=4)])
    with pytest.raises(ValueError, match="blocks"):
        m.generate_requests([dict(input_ids=torch.tensor([REQ0] * 300), max_new_tokens=200)])    # 4 blocks > 3
    assert eng.calls == [] and eng.events == []
    with pytest.raises(NotImplementedError, match="generate_requests"):
        m.generate(torch.tensor([[1, 2, 3]]))
    with pytest.raises(NotImplementedError, match="generate_requests"):
        m(torch.tensor([[1, 2, 3]]))
    m._last_out = torch.zeros(1, 4, dtype=torch.int64)
    with pytest.raises(NotImplementedError, match="generate_requests"):
        m.generate_continue(torch.tensor([[5, 6]]))
    for bad in (1, 0, -3, 2.5, True):
        with pytest.raises(ValueError, match="kv_blocks"):
            _model(FakeEngine(640, 4), kv_blocks=bad)


def test_config_has_kv_blocks_last():
    import vcl_native as vn
    # vcl_config keeps its 20 fields; vcl_config_ex, the struct Engine hands to vcl_create, appends kv_blocks
    assert [f[0] for f in vn.vcl_config._fields_][-1] == "max_slots" and ctypes.sizeof(vn.vcl_config) == 20 * 4
    assert issubclass(vn.vcl_config_ex, vn.vcl_config)
    assert [f[0] for f in vn.vcl_config_ex._fields_] == ["kv_blocks"]
    assert vn.vcl_config_ex.kv_blocks.offset == vn.vcl_config.max_slots.offset + 4 == 20 * 4
    assert ctypes.sizeof(vn.vcl_config_ex) == 21 * 4
    c = vn.vcl_config_ex()
    assert c.max_slots == 0 and c.kv_blocks == 0     # zero-initialised: the default slot count, a contiguous cache
    # the header declares the field right after max_slots, last
    import __graft_entry__ as entry
    import os
    import re
    hdr = open(os.path.join(os.path.dirname(entry.__file__), "include", "vcl.h")).read()
    body = re.search(r"typedef struct vcl_config \{(.*?)\} vcl_config;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"\b(?:int32_t|float)\s+(\w+);", body)
    assert fields[-2:] == ["max_slots", "kv_blocks"] and len(fields) == 21
    assert vn.kv_block_bytes(32, 32) == 64 * 2 ** 20 and vn.kv_block_bytes(40, 40) == 100 * 2 ** 20
    assert {"vcl_llm_set_block_table", "vcl_kv_block_copy"} <= set(vn.EXPORTED_SYMBOLS)


def test_model_passes_kv_blocks_to_the_engine(monkeypatch):
    import vcl_native as vn
    seen = []

    class Recorder:
        def __init__(self, cfg, **kw):
            seen.append((type(cfg), dict(kw)))
            self.NV = 356

    monkeypatch.setattr(vn, "Engine", Recorder)
    for kv, want in ((None, {}), (9, {"kv_blocks": 9})):
        m = _model(None, kv_blocks=kv)
        m._engine = None
        m._ensure_engine()
        assert seen[-1] == (vn.vcl_config, want)

    # Engine copies a plain vcl_config into the full struct, kv_blocks last
    c = vn.vcl_config()
    c.max_seq, c.max_slots = 640, 8
    ex = vn.vcl_config_ex()
    ctypes.memmove(ctypes.addressof(ex), ctypes.addressof(c), ctypes.sizeof(c))
    ex.kv_blocks = 9
    assert (ex.max_seq, ex.max_slots, ex.kv_blocks) == (640, 8, 9)
