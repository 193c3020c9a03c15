"""Decode attention (decode_attn_cluster_kernel<SPLIT, PAGED>, decode_attention.cu) one launch at a time, against the
float64 reference of tests/_attn_ref.py, at the lengths and clip counts the engine decodes at, on the contiguous
cache (vcl_op_decode_attention) and on a paged pool (vcl_op_decode_attention_paged).

A decode row is (clip b, pos = kv_len - 1 + pos_dev[b], kmin = n_pad[b]): the query attends keys n_pad[b] .. pos.
The keys are split over a cluster of SPLIT CTAs (4, 2 or 1 by B * H against the SM count); CTA r owns `per` keys
from n_pad[b] + r * per, per = ceil(n / SPLIT) rounded up to 16.

Input kinds:
  - count: q = 0 and v[j] one-hot at (7 j + 3 h) % 128. Every key weighs exactly p = bf16(fp32(1 / n)) and the
    kernel sums exact multiples of p, so element d is bf16(c_d * p) (R.equal_weight_ref): bar bit-identity.
  - probe: q = 0, v zero except at up to 128 probe keys per (clip, head), each one-hot on its own dimension. An
    element is 0, bf16(p) or bf16(2 p): the probe was skipped, read once or read twice, and a read from the wrong
    address lights the wrong dimension. Every attended key of every clip is a probe in some launch (R.probe_plan:
    neighbouring keys in different launches or heads): bar bit-identity. This is the exact check at long lengths,
    where bf16 no longer tells c_d from c_d + 1.
  - random: q, k, v ~ N(0, 1).
  - rising / falling: the scores grow (fall) by ~0.5 per 64 keys along the clip, so the row maximum sits in the
    last (first) CTA.
  - spike: one key per (clip, head) scores far above the rest; the CTA holding it turns with the clip and head, so
    every CTA of a cluster holds the maximum somewhere. Even heads score 181 above the rest, so every other CTA's
    exponentials underflow to 0; odd heads 45 above.
  Bars of the last four: relative L2 error per (clip, head) < 1e-2 and over the output < 4e-3.

Poisoning: the columns below n_pad[b] and from a clip's last key on are NaN, as are the k | v columns of a q | k | v
row, and (paged) every block a clip does not own and the other layer of each block. The output starts as a NaN
sentinel, so every element must be written and finite. Each paged launch must equal the contiguous launch on the
same logical cache bit for bit: the arithmetic is the same, only the addresses differ."""
import gc
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
import _attn_ref as R  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402

DEV = "cuda"
SENTINEL = 0x7FC1          # a bf16 NaN bit pattern no kernel produces
NAN = float("nan")
SMEM_MAX = 48 * 1024


@pytest.fixture(autouse=True)
def _hand_back_memory():
    """a case holds a few GB at a time through torch's caching allocator, in blocks of sizes no other case reuses;
    hand them back to the device after each test, since engines allocate outside torch"""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _split(B, H):
    """decode_attention.cu: CTAs per (clip, head)"""
    return 4 if B * H <= 2 * _sms() else (2 if B * H <= 3 * _sms() else 1)


def _per(n, split):
    return ((n + split - 1) // split + 15) // 16 * 16


def _cta_counts(n, split):
    """keys of each CTA of a clip attending n keys"""
    per = _per(n, split)
    return [max(0, min(n - r * per, per)) for r in range(split)]


def _fits(split, s_max, paged):
    """the launcher's shared memory with pos_dev: scores of per(s_max) keys, 16 x 128 + 128 partial outputs, 10
    floats of statistics and scratch, and (paged) the table row"""
    return (_per(s_max, split) + 16 * 128 + 128 + 2 + 8 + (paged and (s_max + 127) // 128)) * 4 <= SMEM_MAX


def _limit(split, paged):
    s = 1
    while _fits(split, s + 1, paged):
        s += 1
    return s


class Case:
    """B clips of H heads; clip b attends keys pads[b] .. ends[b] - 1, launched as kv_len plus pos_dev[b] =
    ends[b] - kv_len; q_heads = 3: q inside q | k | v rows (q_ld = 3 H 128); s_max columns per clip"""

    def __init__(self, H, ends, pads, kv_len=1, q_heads=1, s_max=None, name=""):
        self.B, self.H = len(ends), H
        self.ends, self.pads, self.kv_len, self.q_heads = list(ends), list(pads), kv_len, q_heads
        assert all(0 <= p < e for p, e in zip(pads, ends)) and kv_len <= min(ends)
        self.s_max = s_max or max(ends) + 70
        self.name = name or f"B={self.B} H={H}"
        self.split = _split(self.B, H)

    def rows(self):
        return (torch.arange(self.B), torch.tensor([e - 1 for e in self.ends]), torch.tensor(self.pads))

    def n(self, b):
        return self.ends[b] - self.pads[b]

    def device_args(self):
        pos = torch.tensor([e - self.kv_len for e in self.ends], dtype=torch.int32, device=DEV)
        return torch.tensor(self.pads, dtype=torch.int32, device=DEV), pos


def _poison(c, q, k, v):
    for b in range(c.B):
        for t in (k, v):
            t[b, :, :c.pads[b]] = NAN
            t[b, :, c.ends[b]:] = NAN
    if c.q_heads > 1:
        q[:, c.H * 128:] = NAN
    return q, k, v


def _inputs(c, kind, seed):
    """q [B, q_heads H 128] and the logical caches k / v [B, H, s_max, 128] bf16, poisoned"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    B, H, S = c.B, c.H, c.s_max
    q = torch.randn(B, H, 128, device=DEV, generator=g)
    k = torch.randn(B, H, S, 128, device=DEV, generator=g, dtype=torch.bfloat16)
    v = torch.randn(B, H, S, 128, device=DEV, generator=g, dtype=torch.bfloat16)
    if kind == "count":
        q.zero_()
        v = R.counting_values(B, H, S, device=DEV)
    elif kind in ("rising", "falling"):
        u = torch.randn(B, H, 128, device=DEV, generator=g)
        u = u / u.norm(dim=-1, keepdim=True)
        q = 8 * (u + 0.1 * q)
        j = torch.arange(S, device=DEV, dtype=torch.float32)
        for b in range(B):                                # clip by clip: no fp32 copy of the whole cache
            beta = 0.011 * ((j - c.pads[b]) if kind == "rising" else (c.ends[b] - j))
            k[b] = (beta[None, :, None] * u[b][:, None, :] + 0.3 * k[b].float()).bfloat16()
    elif kind == "spike":
        for b in range(B):
            cnt, per = _cta_counts(c.n(b), c.split), _per(c.n(b), c.split)
            for h in range(H):
                r = (b + h) % c.split
                r = r if cnt[r] else 0
                j = c.pads[b] + r * per + (7 * b + 13 * h) % cnt[r]
                k[b, h, j] = ((16 if h % 2 == 0 else 4) * q[b, h]).bfloat16()
    q = torch.cat([q.reshape(B, H * 128), torch.zeros(B, (c.q_heads - 1) * H * 128, device=DEV)], 1)
    return _poison(c, q.bfloat16(), k, v)


def _probe_launches(c):
    """[launch][b][h] -> the probe set of (clip b, head h) in that launch: every attended key of every clip once"""
    plans = [R.probe_plan(range(c.pads[b], c.ends[b])) for b in range(c.B)]
    n = max((len(p) + c.H - 1) // c.H for p in plans)
    return [[[p[t * c.H + h] if t * c.H + h < len(p) else None for h in range(c.H)] for p in plans]
            for t in range(n)]


def _probe_inputs(c, sets):
    q = torch.zeros(c.B, c.q_heads * c.H * 128, dtype=torch.bfloat16, device=DEV)
    k = torch.zeros(c.B, c.H, c.s_max, 128, dtype=torch.bfloat16, device=DEV)
    return _poison(c, q, k, R.probe_values(c.B, c.H, c.s_max, sets, device=DEV))


def _pool(c, k, v, order, seed):
    """the logical caches in a pool [n_blocks][2 layers][K | V][H][128][128] at layer 1, through a scrambled table
    or one that gives each clip's blocks in descending order; unowned blocks and layer 0 are NaN"""
    row = (c.s_max + 127) // 128
    need = [(e + 127) // 128 for e in c.ends]
    n_own = sum(need)
    n_blocks = n_own + 3
    ids = (torch.randperm(n_blocks, generator=torch.Generator().manual_seed(seed)).tolist() if order == "scrambled"
           else list(range(n_blocks))[::-1])
    own, spare = ids[:n_own], ids[n_own:]
    pool = torch.full((n_blocks, 2, 2, c.H, 128, 128), NAN, dtype=torch.bfloat16, device=DEV)
    table = [[spare[(b + kb) % len(spare)] for kb in range(row)] for b in range(c.B)]
    i = 0
    for b in range(c.B):
        for kb in range(need[b]):
            blk = table[b][kb] = own[i]
            i += 1
            w = min(128, c.s_max - kb * 128)
            pool[blk, 1, 0, :, :w] = k[b, :, kb * 128:kb * 128 + w]
            pool[blk, 1, 1, :, :w] = v[b, :, kb * 128:kb * 128 + w]
    return pool, table


def _sentinel(B, H):
    return torch.full((B, H * 128), SENTINEL, dtype=torch.int16, device=DEV).view(torch.bfloat16)


def _launch(c, q, k, v, pool=None, xwin=False):
    npd, pos = c.device_args()
    if xwin:
        out = torch.full(((c.H * 128 + vn.XWIN_KC - 1) // vn.XWIN_KC * c.B * vn.XWIN_PITCH,), SENTINEL,
                         dtype=torch.int16, device=DEV).view(torch.bfloat16)
    else:
        out = _sentinel(c.B, c.H)
    n0 = vn.launch_count()
    if pool is None:
        o = vn.op_decode_attention(q, k, v, c.kv_len, npd, pos, R.SCALE, o_xwin=xwin, out=out)
    else:
        p, table = pool
        o = vn.op_decode_attention(q, p[0, 1, 0], p[0, 1, 1], c.kv_len, npd, pos, R.SCALE, o_xwin=xwin, table=table,
                                   n_blocks=p.shape[0], blk=p[0].numel(), s_max=c.s_max, out=out)
    torch.cuda.synchronize()
    assert vn.launch_count() - n0 == 1
    return o


def _exact(c, o, v, what):
    assert torch.isfinite(o.float()).all(), f"{what}: an element is unwritten (sentinel) or not finite"
    got = o.view(c.B, c.H, 128).double()
    want = R.equal_weight_ref(v, *c.rows())
    bad = got != want
    if bad.any():
        where = bad.nonzero()[:6].tolist()
        info = [(b, h, d, c.pads[b], c.ends[b], got[b, h, d].item(), want[b, h, d].item()) for b, h, d in where]
        raise AssertionError(f"{what}: {int(bad.sum())} elements differ from bf16(c_d p); (clip, head, d, n_pad, "
                             f"end, got, want): {info}")


def _bars(c, o, q, k, v, what):
    assert torch.isfinite(o.float()).all(), f"{what}: an element is unwritten (sentinel) or not finite"
    got = o.view(c.B, c.H, 128).double()
    ref = R.attn_ref(q, k, v, *c.rows())
    per = (got - ref).norm(dim=-1) / ref.norm(dim=-1).clamp_min(1e-30)
    tot = ((got - ref).norm() / ref.norm()).item()
    worst = divmod(per.argmax().item(), c.H)
    print(f"[decode-attn] {what}: max per-(clip, head) {per.max().item():.3e} at {worst}, total {tot:.3e}")
    assert per.max().item() < 1e-2 and tot < 4e-3, (what, per.max().item(), worst, tot)


def _xwin_equal(c, ox, o, what):
    idx = torch.tensor([[vn.xwin_offset(b, d, c.B) for d in range(c.H * 128)] for b in range(c.B)], device=DEV)
    assert torch.equal(ox.view(torch.int16)[idx], o.view(torch.int16)), f"{what}: the xwin store differs"


def _run(c, kind, seed, order="scrambled", xwin=False, twice=True):
    """one input kind on the contiguous cache (bars of the kind, determinism, o_xwin) and on a pool (bit-identity
    with the contiguous launch); probe: as many launches as its plan takes"""
    what = f"{c.name} split={c.split} [{kind}]"
    if kind == "probe":
        todo = [_probe_inputs(c, sets) for sets in _probe_launches(c)]
    else:
        todo = [_inputs(c, kind, seed)]
    for i, (q, k, v) in enumerate(todo):
        w = f"{what} launch {i}" if kind == "probe" else what
        o = _launch(c, q, k, v)
        if kind in ("count", "probe"):
            _exact(c, o, v, w)
        else:
            _bars(c, o, q, k, v, w)
        if twice:
            assert torch.equal(_launch(c, q, k, v).view(torch.int16), o.view(torch.int16)), f"{w}: not deterministic"
        if xwin:
            _xwin_equal(c, _launch(c, q, k, v, xwin=True), o, w)
        pool = _pool(c, k, v, order, seed + i)
        op = _launch(c, q, k, v, pool=pool)
        assert torch.equal(op.view(torch.int16), o.view(torch.int16)), f"{w}: the {order} pool differs from the cache"
        del pool


# ------------------------------------------------------------------------------------------
# split x remainder sweep: the last CTA's key count takes every value mod 128
def _sweep_lengths(split, n_max=4096):
    need, out = set(range(1, 128)), []
    for n in range(1, n_max):
        got = {x % 128 for x in _cta_counts(n, split) if x % 128}
        if got & need:
            out.append(n)
            need -= got
        if not need:
            return out
    raise AssertionError(f"split {split}: residues {sorted(need)} not reached")


def _sweep_case(split):
    """H = 2 and B just above the threshold of the split, one length per clip (the lengths of _sweep_lengths, then
    repeated), left padding 0 .. 149 and a shared kv_len below every clip's end"""
    sms = _sms()
    B = {4: 2 * sms // 2, 2: 2 * sms // 2 + 1, 1: 3 * sms // 2 + 1}[split]
    lens = _sweep_lengths(split)
    assert len(lens) <= B, (split, len(lens), B)
    lens = [lens[b % len(lens)] for b in range(B)]
    pads = [(37 * b) % 150 for b in range(B)]
    ends = [p + n for p, n in zip(pads, lens)]
    return Case(2, ends, pads, kv_len=min(ends), name=f"sweep B={B} H=2")


@torch.no_grad()
@pytest.mark.parametrize("split", [4, 2, 1])
def test_split_remainder_sweep(split):
    """every CTA key count mod 128 in 1 .. 127, odd counts below 16 included (the old stall): count and probe bit
    for bit, random against the bars, on the cache and on a scrambled pool"""
    c = _sweep_case(split)
    assert c.split == split, f"{_sms()} SMs: B={c.B} H={c.H} runs split {c.split}"
    seen = {x % 128 for b in range(c.B) for x in _cta_counts(c.n(b), split)}
    assert set(range(1, 128)) <= seen
    for i, kind in enumerate(("count", "probe", "random")):
        _run(c, kind, seed=split * 10 + i)


def _long_case(split):
    """two clips past 1024 keys per CTA (1 100 and 1 033 + 16 per CTA, odd last CTAs), H just above the split's
    threshold at B = 2 (a head stride of up to 200 heads)"""
    H = {4: 2, 2: _sms() + 1, 1: 3 * _sms() // 2 + 1}[split]
    ends = [1100 * split - 3 + 5, 1049 * split + 200]
    pads = [5, 200]
    return Case(H, ends, pads, kv_len=min(ends), name=f"long B=2 H={H}")


@torch.no_grad()
@pytest.mark.parametrize("split", [4, 2, 1])
def test_past_1024_keys_per_cta(split):
    c = _long_case(split)
    assert c.split == split and all(min(_cta_counts(c.n(b), split)) > 1024 for b in range(2))
    for i, kind in enumerate(("count", "probe", "random", "spike", "rising", "falling")):
        _run(c, kind, seed=split * 100 + i, order="reversed" if i % 2 else "scrambled")


# ------------------------------------------------------------------------------------------
# engine shapes: the 7B (H = 32) and 13B (H = 40) heads at every clip-count regime of the decode
ENGINE_B = [1, 4, 5, 8, 9, 12, 13, 16, 17, 33, 64, 65]
XWIN_B = {5, 8, 13, 17, 33, 64}


def _engine_case(B, H):
    """a 356-token video prompt plus 0 .. 744 answer tokens per clip, one clip at 2 048 keys; left padding up to 99
    on every third clip; B = 65 is the GEMM decode (q inside the q | k | v row), up to 64 the ring path (q_ld = D)"""
    ends = [356 + (b * 337) % 745 for b in range(B)]
    ends[B // 2] = 2048
    pads = [(b * 53) % 100 if b % 3 == 1 else 0 for b in range(B)]
    return Case(H, ends, pads, kv_len=356, q_heads=3 if B > 64 else 1, name=f"engine B={B} H={H}")


@torch.no_grad()
@pytest.mark.parametrize("H", [32, 40])
@pytest.mark.parametrize("B", ENGINE_B)
def test_engine_shapes(B, H):
    c = _engine_case(B, H)
    want = 4 if B * H <= 2 * 132 else (2 if B * H <= 3 * 132 else 1)
    assert _sms() != 132 or c.split == want
    kinds = ("count", "probe", "random", "spike") + (("rising", "falling") if B in (1, 9, 17, 65) else ())
    for i, kind in enumerate(kinds):
        _run(c, kind, seed=B * 1000 + H * 10 + i, order="reversed" if (B + i) % 2 else "scrambled",
             xwin=B in XWIN_B and kind in ("random", "probe"))


# ------------------------------------------------------------------------------------------
# the shared-memory limit of each split with pos_dev, contiguous and paged
def _limit_shape(split):
    sms = _sms()
    return {4: (2, 16), 2: (4, (2 * sms + 4) // 4), 1: (4, (3 * sms + 4) // 4)}[split]


@torch.no_grad()
@pytest.mark.parametrize("paged", [False, True], ids=["contiguous", "paged"])
@pytest.mark.parametrize("split", [4, 2, 1])
def test_shared_memory_limit(split, paged):
    """the largest s_max that fits (with pos_dev, smem is sized for s_max keys) runs the probe input over every key
    of a clip attending all s_max columns; one column more is refused before any launch"""
    B, H = _limit_shape(split)
    s_max = _limit(split, paged)
    if _sms() == 132:
        assert s_max == {(4, False): 40384, (2, False): 20192, (1, False): 10096,
                         (4, True): 39168, (2, True): 19872, (1, True): 10016}[split, paged]
    ends = [s_max, 300, 1, 5000][:B]
    pads = [0, 17, 0, 4999][:B]
    c = Case(H, ends, pads, kv_len=1, s_max=s_max, name=f"limit {'paged' if paged else 'contiguous'} s_max={s_max}")
    assert c.split == split
    t0 = time.time()
    for i, sets in enumerate(_probe_launches(c)):
        q, k, v = _probe_inputs(c, sets)
        o = _launch(c, q, k, v)
        _exact(c, o, v, f"{c.name} launch {i}")
        if paged:
            op = _launch(c, q, k, v, pool=_pool(c, k, v, "scrambled" if i % 2 else "reversed", i))
            assert torch.equal(op.view(torch.int16), o.view(torch.int16)), f"{c.name} launch {i}: pool differs"
        del q, k, v
    print(f"[decode-attn] {c.name}: {i + 1} probe launches, {time.time() - t0:.1f} s")
    # one column more: refused by the launcher before any launch (buffers of one head suffice)
    s1 = s_max + 1
    q = torch.zeros(B, H * 128, dtype=torch.bfloat16, device=DEV)
    kv = torch.zeros(H, 128, 128, dtype=torch.bfloat16, device=DEV)
    z = torch.zeros(B, dtype=torch.int32, device=DEV)
    o = torch.empty(B, H * 128, dtype=torch.bfloat16, device=DEV)
    n0 = vn.launch_count()
    with pytest.raises(vn.VclError, match=f"s_max {s1} too long"):
        if paged:
            row = (s1 + 127) // 128
            vn.op_decode_attention(q, kv, kv, 1, z, z, table=[[0] * row] * B, n_blocks=1, blk=kv.numel(), s_max=s1,
                                   out=o)
        else:
            vn.check(vn.lib().vcl_op_decode_attention(vn.ptr(q), H * 128, vn.ptr(kv), vn.ptr(kv), vn.ptr(o), B, H, s1,
                                                      1, vn.ptr(z), vn.ptr(z), R.SCALE, 0, vn.cur_stream()))
    assert vn.launch_count() == n0


# ------------------------------------------------------------------------------------------
# argument checks of the paged entry
PAGED_BAD = [
    (dict(table=[[0, 1], [1, 3]]), r"table\[1\]\[1\] = 3 outside the pool"),
    (dict(table=[[0, -1], [1, 0]]), r"table\[0\]\[1\] = -1"),
    (dict(blk=128 * 128), "blk=16384"),                 # below H * 128 * 128
    (dict(n_blocks=0), "n_blocks=0"),
]


@torch.no_grad()
@pytest.mark.parametrize("bad,match", PAGED_BAD)
def test_paged_rejects(bad, match):
    H, s_max = 2, 200
    pool = torch.zeros(3, 2, 2, H, 128, 128, dtype=torch.bfloat16, device=DEV)
    q = torch.zeros(2, H * 128, dtype=torch.bfloat16, device=DEV)
    z = torch.zeros(2, dtype=torch.int32, device=DEV)
    args = dict(table=[[0, 1], [1, 2]], n_blocks=3, blk=pool[0].numel())
    n0 = vn.launch_count()
    with pytest.raises(vn.VclError, match=match):
        vn.op_decode_attention(q, pool[0, 1, 0], pool[0, 1, 1], 1, z, z, s_max=s_max, **dict(args, **bad))
    assert vn.launch_count() == n0
    o = vn.op_decode_attention(q, pool[0, 1, 0], pool[0, 1, 1], 1, z, z, s_max=s_max, **args)
    torch.cuda.synchronize()
    assert vn.launch_count() == n0 + 1 and torch.equal(o, torch.zeros_like(o))


# ------------------------------------------------------------------------------------------
# vcl_create refuses a max_seq decode attention cannot hold at some clip count
TINY = O.LlmCfg(hidden=1024, inter=1024, heads=8, layers=1)   # H = 8: split 1 from 50 clips on (132 SMs)


def _tiny(max_seq, kv_blocks=None, max_batch=64):
    clip = O.ClipCfg()
    cfg = vn.vcl_config()
    cfg.clip_layers, cfg.clip_hidden, cfg.clip_inter, cfg.clip_heads = 0, clip.hidden, clip.inter, clip.heads
    cfg.image_size, cfg.patch_size, cfg.clip_ln_eps = clip.image, clip.patch, clip.eps
    cfg.llm_layers, cfg.llm_hidden, cfg.llm_inter, cfg.llm_heads = TINY.layers, TINY.hidden, TINY.inter, TINY.heads
    cfg.vocab, cfg.rms_eps, cfg.rope_theta = TINY.vocab, TINY.rms_eps, TINY.rope_theta
    cfg.proj_type = vn.PROJ_LINEAR
    cfg.n_temporal = 100
    cfg.max_frames, cfg.max_batch, cfg.max_seq, cfg.max_slots = 1, max_batch, max_seq, max_batch
    return vn.Engine(cfg, kv_blocks=kv_blocks)


@torch.no_grad()
def test_create_refuses_a_max_seq_decode_attention_cannot_hold():
    """64 slots of 8 heads reach split 1 (at 50 clips on 132 SMs): the first max_seq past its limit is refused at
    create, naming the clip count and the largest max_seq that fits; the paged limit itself is accepted, and its
    slot decode runs at 64 clips at positions up to max_seq - 1, where the graph sizes decode attention's shared
    memory for max_seq keys (slots fed the same token over the same keys agree)"""
    B1 = next(B for B in range(1, 65) if _split(B, TINY.heads) == 1)
    for paged, blocks in ((False, None), (True, 200)):
        lim = _limit(1, paged)
        match = (rf"max_seq {lim + 1} is too long for decode attention at {B1} clips x 8 heads"
                 rf"{' [(]paged[)]' if paged else ''}: .* at most max_seq {lim}")
        with pytest.raises(vn.VclError, match=match):
            _tiny(lim + 1, blocks)
    lim = _limit(1, True)
    row = (lim + 127) // 128
    eng = _tiny(lim, 1 + 64 * row)                    # block 0 parks; slot s owns blocks 1 + s * row ..
    eng.load_llm({k: t.to(DEV, torch.bfloat16) for k, t in O.random_llm_state(TINY, seed=8).items()})
    g = torch.Generator(device=DEV).manual_seed(8)
    for kb in range(row):                             # slot s + 32 holds slot s's keys
        for s in range(32):
            buf = torch.randn(eng.block_shape(), generator=g, device=DEV).bfloat16()
            eng.kv_block_copy(1 + s * row + kb, buf, write=True)
            eng.kv_block_copy(1 + (s + 32) * row + kb, buf, write=True)
    eng.set_block_table([[1 + s * row + kb for kb in range(row)] for s in range(64)])
    pos = [(row - 1) * 128 + s % 32 for s in range(64)]
    assert max(pos) == lim - 1
    feed = torch.randint(3, 32000, (32,), generator=torch.Generator().manual_seed(9)).repeat(2).to(DEV, torch.int32)
    try:
        out = eng.slot_decode(feed, pos, 2)
        torch.cuda.synchronize()
    finally:
        eng.close()
    assert ((out >= 0) & (out < TINY.vocab)).all()
    assert torch.equal(out[:32], out[32:]), "slots over the same keys decode different tokens"
