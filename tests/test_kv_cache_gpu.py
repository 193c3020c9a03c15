"""The KV cache itself, read back on the GPU: what the RoPE / cache writers store, which columns they touch, what
decode attention reads out of it, and the arg-max tie rule of every path that picks a token.

Writers (Engine.kv_cache reads a layer's whole cache; Engine.set_kv_cache fills it with a NaN sentinel first):
  - the ACT_ROPE epilogue of the prefill q|k|v GEMM (gemm_tc.cu), 128- and 256-wide tiles;
  - rope_kv_prefill_kernel (elementwise.cu): VCL_PREFILL_ROPE_SEPARATE=1 and the decode path beyond 16 clips;
  - the GEMV_QKV epilogue of the decode ring kernels (decode_gemv.cu), 1..4 and 5..16 clips.
The expected cache is computed from the engine's own input to the layer (the hidden state a prefill with
n_layers = l returns, or the embedding row of the fed token): k = bf16(rmsnorm(x) . Wk^T) with fp64 products
(rmsnorm: see _ref_kv), then
the reference's RoPE rounding (oracle: _rope_cos_sin, _rotate_half: every product rounded to bf16, then the sum) at
the angle of max(column - n_pad[b], 0) (kernels.h: decode positions), v = bf16(rmsnorm(x) . Wv^T). The only
difference left is the fp32 accumulation order before the one bf16 rounding of k / v, so an element may differ by
at most 2 bf16 ulps of the larger magnitude of its RoPE pair (d, d + 64), at least 99 % of the elements are
bit-identical, and everything a call must not touch keeps its bits.

Reader: decode_attn_cluster_kernel (decode_attention.cu) against an fp64 evaluation with the reference's rounding
points, the pad keys and every column past a clip's last key poisoned with NaN."""
import json
import os
import subprocess
import sys
from functools import lru_cache

import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import make_engine, to_dev  # noqa: E402
from _attn_ref import attn_ref  # noqa: E402

DEV = "cuda"
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)
WIDE = O.LlmCfg(hidden=2560, inter=6912, heads=20, layers=2)
CFGS = {512: SMALL, 2560: WIDE}
SENTINEL = 0x7FC1          # a bf16 NaN bit pattern no kernel produces


@lru_cache(maxsize=None)
def _state(width, seed=21):
    return to_dev(O.random_llm_state(CFGS[width], seed=seed))


def _engine(width, max_batch, max_seq, lm_head=None):
    sd = _state(width)
    if lm_head is not None:
        sd = dict(sd, **{"lm_head.weight": lm_head})
    eng = make_engine(llm=CFGS[width], max_batch=max_batch, max_seq=max_seq)
    eng.load_llm(sd)
    return eng


def _ids(B, S, seed):
    return torch.randint(3, 32000, (B, S), generator=torch.Generator().manual_seed(seed)).to(DEV)


def _no_video(B):
    return torch.full((B,), vn.NO_VIDEO, dtype=torch.int32, device=DEV)


def _bits(t):
    return t.contiguous().view(torch.int16)


def _fill_sentinel(eng):
    c = eng.cfg
    s = torch.full((c.max_batch, c.llm_heads, c.max_seq, 128), SENTINEL, dtype=torch.int16, device=DEV)
    s = s.view(torch.bfloat16)
    for l in range(c.llm_layers):
        eng.set_kv_cache(l, s, s)


def _caches(eng):
    return [eng.kv_cache(l) for l in range(eng.cfg.llm_layers)]


def _ref_kv(width, layer, x, angles, prefill=True):
    """x [N, D] bf16 (the layer's input rows), angles [N] (RoPE positions) -> (k, v) [N, H, 128] bf16.
    prefill: the normalised rows are those of the engine's rmsnorm kernel (vn.op_rmsnorm, pinned to LlamaRMSNorm by
    test_kernels_gpu.py), bit for bit the rows the prefill's q|k|v GEMM reads. A one-ulp flip of bf16(x * rsqrt) in
    one large element of a deep layer's input moves k by many ulps, and that rounding is not what is under test.
    Otherwise (decode steps, which normalise inside the projection kernels) the rows are normalised here in fp64."""
    cfg = CFGS[width]
    sd = _state(width)
    lp = f"model.layers.{layer}."
    N, D, H = x.shape[0], cfg.hidden, cfg.heads
    w = sd[lp + "input_layernorm.weight"]
    if prefill:
        y = vn.op_rmsnorm(x.contiguous(), w, cfg.rms_eps).double()
    else:
        xd = x.double()
        xn = (xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + cfg.rms_eps)).bfloat16()
        y = (w * xn).double()                                              # LlamaRMSNorm: w * bf16(x_normed)
    k = (y @ sd[lp + "self_attn.k_proj.weight"].double().t()).bfloat16().view(N, H, 128)
    v = (y @ sd[lp + "self_attn.v_proj.weight"].double().t()).bfloat16().view(N, H, 128)
    cos, sin = O._rope_cos_sin(cfg, torch.as_tensor(angles).cpu(), torch.bfloat16, x.device)
    k = k * cos[:, None] + O._rotate_half(k) * sin[:, None]
    return k, v


def _assert_kv(got, ref, what):
    """got / ref [..., 128] bf16: within 2 bf16 ulps of the pair's larger magnitude, >= 99 % bit-identical"""
    g, r = got.float(), ref.float()
    assert torch.isfinite(g).all(), f"{what}: non-finite values (sentinel left or NaN written)"
    m = torch.maximum(r[..., :64].abs(), r[..., 64:].abs())
    ulp = torch.exp2(torch.floor(torch.log2(torch.cat([m, m], -1).clamp_min(1e-30))) - 7)
    bad = (g - r).abs() > 2 * ulp
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} elements off by more than 2 ulps, first at "
                           f"{bad.nonzero()[:4].tolist()}: got {g[bad][:4].tolist()} want {r[bad][:4].tolist()}")
    same = (_bits(got) == _bits(ref)).float().mean().item()
    assert same >= 0.99, f"{what}: only {same:.4f} of the elements bit-identical"


def _assert_sentinel(t, what):
    n = int((_bits(t) != SENTINEL).sum())
    assert n == 0, f"{what}: {n} elements written where nothing may be"


def _assert_same(a, b, what):
    n = int((_bits(a) != _bits(b)).sum())
    assert n == 0, f"{what}: {n} elements changed"


# ------------------------------------------------------------------------------------------
# 1, 2. prefill writers
def _prefill_case(width, B, S, pads, seed=3):
    """A prefill of B text-only rows of S tokens (left padding pads or none) into a cache of max_batch = B + 1 clips
    and max_seq = S + 16 columns, filled with the sentinel first. Every layer's columns [0, S) of clips 0 .. B-1 must
    match the reference; everything else must keep the sentinel. Returns the launches of the checked prefill."""
    cfg = CFGS[width]
    eng = _engine(width, B + 1, S + 16)
    ids = _ids(B, S, seed)
    vs = _no_video(B)
    xs = [eng.prefill(ids, None, vs, n_layers=l, want_hidden=True, want_token=False, n_pad=pads)[0]
          for l in range(cfg.layers)]
    _fill_sentinel(eng)
    n0 = vn.launch_count()
    eng.prefill(ids, None, vs, n_pad=pads)
    launches = vn.launch_count() - n0
    npad = pads or [0] * B
    angles = [max(c - npad[b], 0) for b in range(B) for c in range(S)]
    for l, (k, v) in enumerate(_caches(eng)):
        rk, rv = _ref_kv(width, l, xs[l].view(B * S, cfg.hidden), angles)
        rk, rv = [t.view(B, S, cfg.heads, 128).transpose(1, 2) for t in (rk, rv)]
        _assert_kv(k[:B, :, :S], rk, f"layer {l} k")
        _assert_kv(v[:B, :, :S], rv, f"layer {l} v")
        for t, n in ((k, "k"), (v, "v")):
            _assert_sentinel(t[:, :, S:], f"layer {l} {n} columns >= S")
            _assert_sentinel(t[B:], f"layer {l} {n} clips >= B")
    return launches


PREFILL_CASES = [
    # width, B, S, pads. S = 77: B * S is no multiple of the 128-row tile
    (512, 1, 77, None),                      # one M tile
    (512, 3, 77, None),
    (512, 3, 77, [0, 76, 30]),               # pad counts 0 and S - 1
    (2560, 7, 77, None),                     # 539 rows: 256-wide tiles (checked below)
    (2560, 7, 77, [0, 76, 5, 40, 0, 11, 60]),
]


@torch.no_grad()
@pytest.mark.parametrize("width,B,S,pads", PREFILL_CASES)
def test_prefill_writes_the_reference_cache(width, B, S, pads):
    """The ACT_ROPE epilogue of the prefill q|k|v GEMM. gemm_tc.cu picks the tile width from the shape: 2 x 6
    (B = 3) or 1 x 6 tiles of 256 columns at width 512 are fewer than the SMs, so 128-wide tiles run; at width
    2560, 539 rows give 5 x 30 tiles of 256 columns, at least one per SM, so 256-wide tiles run."""
    cfg = CFGS[width]
    M, N = B * S, 3 * cfg.hidden
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    wide_tiles = (M + 127) // 128 > 1 and (M + 127) // 128 * (N // 256) >= sms
    assert wide_tiles == (width == 2560), "the case no longer runs the tile width it is meant for"
    _prefill_case(width, B, S, pads)


@torch.no_grad()
def test_separate_rope_kernel_writes_the_same_cache():
    """VCL_PREFILL_ROPE_SEPARATE=1 (plain GEMM + rope_kv_prefill_kernel) must meet the same checks. The variable is
    read once per process, so the cases run in a child process; that child's prefill launches one kernel more per
    layer, which shows the separate kernel ran."""
    cases = [(512, 3, 77, [0, 76, 30]), (512, 1, 77, None)]
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    script = ("import json, sys; sys.path[:0] = %r; import test_kv_cache_gpu as t; "
              "print(json.dumps([t._prefill_case(*c) for c in %r]))" % ([root, os.path.join(root, "video-llava_b200"),
                                                                         here], cases))
    env = dict(os.environ, VCL_PREFILL_ROPE_SEPARATE="1")
    r = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    separate = json.loads(r.stdout.strip().splitlines()[-1])
    fused = [_prefill_case(*c) for c in cases]
    assert separate == [f + SMALL.layers for f in fused], (separate, fused)


# ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng17():
    """width 512, 2 layers, 17 clips (every decode path), 64 columns"""
    return _engine(512, 17, 64)


def _embed(tok):
    return _state(512)["model.embed_tokens.weight"][tok.long()]


# 3. continuation
@torch.no_grad()
@pytest.mark.parametrize("pads", [None, [0, 17]])
def test_prefill_append_writes_only_its_columns(eng17, pads):
    """prefill_append at start_pos = 40 writes columns [40, 63) at those angles (minus the clip's padding) and leaves
    [0, 40) of every layer, the columns after it and the other clips bit-identical."""
    S0, S1, B = 40, 23, 2
    _fill_sentinel(eng17)
    eng17.prefill(_ids(B, S0, 5), None, _no_video(B), n_pad=pads)
    before = [(k.clone(), v.clone()) for k, v in _caches(eng17)]
    new = _ids(B, S1, 6)
    eng17.prefill_append(new, S0)
    after = _caches(eng17)
    npad = pads or [0] * B
    rk, rv = _ref_kv(512, 0, _embed(new).view(B * S1, -1), [S0 + j - npad[b] for b in range(B) for j in range(S1)])
    rk, rv = [t.view(B, S1, SMALL.heads, 128).transpose(1, 2) for t in (rk, rv)]
    _assert_kv(after[0][0][:B, :, S0:S0 + S1], rk, "layer 0 k")
    _assert_kv(after[0][1][:B, :, S0:S0 + S1], rv, "layer 0 v")
    for l in range(SMALL.layers):
        for i, n in enumerate("kv"):
            a, b = after[l][i], before[l][i]
            assert torch.isfinite(a[:B, :, S0:S0 + S1].float()).all(), (l, n)
            _assert_same(a[:B, :, :S0], b[:B, :, :S0], f"layer {l} {n} columns < start_pos")
            _assert_same(a[:, :, S0 + S1:], b[:, :, S0 + S1:], f"layer {l} {n} columns after the append")
            _assert_same(a[B:], b[B:], f"layer {l} {n} other clips")


# 4. decode writes
def _check_step(eng, before, B, cols, angles, feed, what):
    """after one decode step that fed `feed` [B] at cache column cols[b]: layer 0 column cols[b] of clip b matches the
    reference at angles[b]; every other element of every layer kept its bits; the written columns are finite."""
    after = _caches(eng)
    rk, rv = _ref_kv(512, 0, _embed(feed), angles, prefill=False)
    bi = torch.arange(B, device=DEV)
    ci = torch.as_tensor(cols, device=DEV)
    _assert_kv(after[0][0][bi, :, ci], rk, f"{what}: layer 0 k")
    _assert_kv(after[0][1][bi, :, ci], rv, f"{what}: layer 0 v")
    for l in range(eng.cfg.llm_layers):
        for i, n in enumerate("kv"):
            a, b = after[l][i].clone(), before[l][i]
            assert torch.isfinite(a[bi, :, ci].float()).all(), (what, l, n)
            a[bi, :, ci] = b[bi, :, ci]
            _assert_same(a, b, f"{what}: layer {l} {n} outside the new columns")


@torch.no_grad()
@pytest.mark.parametrize("B,padded", [(1, False), (3, False), (3, True), (5, False), (9, True), (16, False),
                                      (17, False), (17, True)])
def test_decode_step_writes_one_column(eng17, B, padded):
    """1..4 clips: the fused-embedding ring kernel; 5..16: the wide ring kernel; 17: GEMM + rope_kv_prefill_kernel.
    One step after a prefill of S = 37 writes column 37 of every clip at the angle 37 - n_pad[b], nothing else."""
    S = 37
    pads = [(11 * b) % S for b in range(B)] if padded else None
    _fill_sentinel(eng17)
    eng17.prefill(_ids(B, S, 10 + B), None, _no_video(B), n_pad=pads)
    before = [(k.clone(), v.clone()) for k, v in _caches(eng17)]
    feed = torch.randint(3, 32000, (B,), generator=torch.Generator().manual_seed(B)).to(DEV, torch.int32)
    eng17.decode_step(feed, S)
    npad = pads or [0] * B
    _check_step(eng17, before, B, [S] * B, [S - npad[b] for b in range(B)], feed, f"B={B} padded={padded}")


@torch.no_grad()
@pytest.mark.parametrize("n_slots", [3, 9])
def test_slot_decode_writes_each_slots_column(eng17, n_slots):
    """slot_decode (the graph loop) with a different position per slot: slot b's step writes column pos[b] at angle
    pos[b] and nothing else."""
    _fill_sentinel(eng17)
    lens = [5 + (7 * b) % 40 for b in range(n_slots)]
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for b, n in enumerate(lens):
            eng17.slot_prefill(b, _ids(1, n, 30 + b), None, _no_video(1))
        before = [(k.clone(), v.clone()) for k, v in _caches(eng17)]
        feed = torch.randint(3, 32000, (n_slots,), generator=torch.Generator().manual_seed(n_slots)).to(DEV, torch.int32)
        eng17.slot_decode(feed, lens, 2)
    st.synchronize()
    _check_step(eng17, before, n_slots, lens, lens, feed, f"{n_slots} slots")


# 5. slot isolation
@torch.no_grad()
def test_slot_prefill_touches_only_its_slot(eng17):
    """slot_prefill into slot 2 writes columns [0, S) of slot 2 (layer 0 against the reference) and leaves every
    other slot, and the rest of slot 2, bit-identical in all layers."""
    _fill_sentinel(eng17)
    for b, n in enumerate([30, 12, 50, 21]):
        eng17.slot_prefill(b, _ids(1, n, 50 + b), None, _no_video(1))
    before = [(k.clone(), v.clone()) for k, v in _caches(eng17)]
    S = 19
    ids = _ids(1, S, 60)
    eng17.slot_prefill(2, ids, None, _no_video(1))
    after = _caches(eng17)
    rk, rv = _ref_kv(512, 0, _embed(ids[0]), list(range(S)))
    _assert_kv(after[0][0][2, :, :S], rk.transpose(0, 1), "slot 2 layer 0 k")
    _assert_kv(after[0][1][2, :, :S], rv.transpose(0, 1), "slot 2 layer 0 v")
    for l in range(SMALL.layers):
        for i, n in enumerate("kv"):
            a, b = after[l][i], before[l][i]
            assert torch.isfinite(a[2, :, :S].float()).all(), (l, n)
            _assert_same(torch.cat([a[:2], a[3:]]), torch.cat([b[:2], b[3:]]), f"layer {l} {n} other slots")
            _assert_same(a[2, :, S:], b[2, :, S:], f"layer {l} {n} slot 2 columns >= S")


# ------------------------------------------------------------------------------------------
# 6. decode attention against fp64
def _attn_ref(q, k, v, kv_len, n_pad, pos, scale):
    """[B, H, 128] fp64 (tests/_attn_ref.py): clip b's query at column c_b = kv_len - 1 + pos[b] attends keys
    n_pad[b] .. c_b"""
    B = k.shape[0]
    return attn_ref(q, k, v, list(range(B)), [kv_len - 1 + pos[b] for b in range(B)], list(n_pad), scale)


def _attn_case(B, H, s_max, kv_len, n_pad, pos, kind="random", q_ld_heads=1, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    scale = 128 ** -0.5
    q = torch.randn(B, q_ld_heads * H * 128, device=DEV, generator=g).bfloat16()
    k = torch.randn(B, H, s_max, 128, device=DEV, generator=g).bfloat16()
    v = torch.randn(B, H, s_max, 128, device=DEV, generator=g).bfloat16()
    posl = pos or [0] * B
    for b in range(B):
        c = kv_len - 1 + posl[b]
        if kind == "one_high":            # one key far above the rest: p = 1 there, ~0 elsewhere
            j = n_pad[b] + (c - n_pad[b]) // 3
            k[b, :, j] = (4 * q[b, :H * 128].float().view(H, 128)).bfloat16()
        elif kind == "all_equal":         # q = 0: every score 0, p = 1 / n_keys
            q[b] = 0
        k[b, :, :n_pad[b]] = float("nan"); v[b, :, :n_pad[b]] = float("nan")
        k[b, :, c + 1:] = float("nan"); v[b, :, c + 1:] = float("nan")
    npd = torch.tensor(n_pad, dtype=torch.int32, device=DEV)
    pdv = torch.tensor(pos, dtype=torch.int32, device=DEV) if pos is not None else None
    o = vn.op_decode_attention(q, k, v, kv_len, npd, pdv, scale)
    ox = vn.op_decode_attention(q, k, v, kv_len, npd, pdv, scale, o_xwin=True)
    torch.cuda.synchronize()
    assert torch.isfinite(o.float()).all(), "non-finite output: a pad key or a column past the last key was read"
    ref = _attn_ref(q, k, v, kv_len, n_pad, posl, scale)
    got = o.view(B, H, 128).double()
    per = ((got - ref).norm(dim=-1) / ref.norm(dim=-1).clamp_min(1e-30))
    tot = ((got - ref).norm() / ref.norm()).item()
    assert per.max().item() < 1e-2 and tot < 4e-3, (per.max().item(), per.argmax().item(), tot)
    # the xwin store: same kernel, only the address differs -> bit-identical
    idx = torch.tensor([[vn.xwin_offset(b, c, B) for c in range(H * 128)] for b in range(B)], device=DEV)
    assert torch.equal(_bits(ox)[idx], _bits(o)), "xwin output differs from the row-major one"


@torch.no_grad()
@pytest.mark.parametrize("kv_len,n_pad", [(1, [0, 0]), (15, [0, 3]), (16, [0, 15]), (17, [0, 1]), (63, [0, 30]),
                                          (65, [0, 0]), (40, [39, 12])])
def test_decode_attention_lengths(kv_len, n_pad):
    """4-CTA split at lengths where some CTAs own no key (1, 15, 16, 17), at 63 / 65 keys, and kv_len - n_pad = 1."""
    _attn_case(2, 3, 80, kv_len, n_pad, None, seed=kv_len)


@torch.no_grad()
@pytest.mark.parametrize("kind", ["random", "one_high", "all_equal"])
def test_decode_attention_per_clip_positions(kind):
    """different pos_dev[b] in one launch (a single key, a few, many), q inside a q|k|v row (q_ld = 3 * H * 128)"""
    _attn_case(4, 2, 200, 1, [0, 0, 3, 40], [0, 5, 17, 150], kind=kind, q_ld_heads=3, seed=7)


@torch.no_grad()
@pytest.mark.parametrize("B", [1, 9, 16])
def test_decode_attention_split_thresholds(B):
    """B * H up to 2 x SMs: clusters of 4 CTAs, up to 3 x SMs: 2, beyond: 1 (132 SMs, H = 32: B = 1, 9, 16)"""
    H = 32
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    split = 4 if B * H <= 2 * sms else (2 if B * H <= 3 * sms else 1)
    assert split == {1: 4, 9: 2, 16: 1}[B], f"{sms} SMs: B = {B} no longer runs the split it is meant for"
    n_pad = [(7 * b) % 20 for b in range(B)]
    pos = [(b % 5) * 6 for b in range(B)]
    _attn_case(B, H, 100, 70, n_pad, pos, q_ld_heads=3, seed=B)


@torch.no_grad()
def test_decode_attention_at_the_shared_memory_limit():
    """With pos_dev, shared memory holds a quarter of s_max scores: s_max = 40384 is the largest that fits 48 KB
    (10096 keys per CTA); clip 0 attends all of them. One column more is refused before any launch."""
    _attn_case(2, 2, 40384, 1, [0, 999], [40383, 1000], seed=3)
    k = torch.zeros(1, 1, 40385, 128, dtype=torch.bfloat16, device=DEV)
    z = torch.zeros(1, dtype=torch.int32, device=DEV)
    with pytest.raises(vn.VclError, match="smem"):
        vn.op_decode_attention(torch.zeros(1, 128, dtype=torch.bfloat16, device=DEV), k, k, 1, z, z)


# ------------------------------------------------------------------------------------------
# 7. arg-max ties
P_ROWS = [1000, 1001, 3048, 17000, 31000]     # lm_head rows +e_K (1000 / 3048 and 700 / 2748: one arg-max thread,
N_ROWS = [700, 2748, 9000, 25000]             # 1024 apart x 2; the rest in different CTAs of gemv_grid(vocab))
K_DIM = 5


def _one_hot_head():
    w = torch.zeros(SMALL.vocab, SMALL.hidden)
    w[P_ROWS, K_DIM] = 1.0
    w[N_ROWS, K_DIM] = -1.0
    return w.to(DEV, torch.bfloat16)


@pytest.fixture(scope="module", params=["zero", "one_hot"])
def tie_engine(request):
    head = torch.zeros(SMALL.vocab, SMALL.hidden, dtype=torch.bfloat16, device=DEV) if request.param == "zero" \
        else _one_hot_head()
    return request.param, _engine(512, 17, 64, lm_head=head)


def _allowed(kind):
    # a one-hot row's logit is exact, so the maximum is tied exactly: +e_K rows, -e_K rows, or every row (x_K = 0)
    return {0} if kind == "zero" else {0, P_ROWS[0], N_ROWS[0]}


def _check_ties(kind, lg, tok, what):
    lg = lg.float()
    top = lg.max(-1, keepdim=True).values
    assert ((lg == top).sum(-1) >= 2).all(), f"{what}: no tie to break"
    assert torch.equal(tok.long().cpu(), lg.argmax(-1).cpu()), (what, tok.tolist(), lg.argmax(-1).tolist())
    assert set(tok.tolist()) <= _allowed(kind), (what, tok.tolist())


@torch.no_grad()
@pytest.mark.parametrize("B", [1, 3, 9, 17])
def test_argmax_ties_take_the_first_index(tie_engine, B):
    """Tokens follow torch.argmax (the first maximum) through the prefill's argmax_kernel and decode_step, at every
    clip count (lm_head of 1..4 clips, 5..16, and more than 16 in chunks)."""
    kind, eng = tie_engine
    S = 21
    _, lg, tok = eng.prefill(_ids(B, S, 70 + B), None, _no_video(B), want_logits=True)
    _check_ties(kind, lg, tok, f"prefill B={B}")
    lg, tok = eng.decode_step(tok, S, want_logits=True)
    _check_ties(kind, lg, tok, f"decode_step B={B}")


@torch.no_grad()
@pytest.mark.parametrize("B", [2, 9, 17])
def test_argmax_ties_in_the_graph_loop(tie_engine, B):
    """The CUDA-graph decode loop: at B <= 4 the per-CTA partial arg-max is reduced inside the next q|k|v kernel;
    5..16 and 17 clips run argmax_kernel. Later tokens have no returned logits, so they are checked against the
    rule: an all-zero head gives token 0 at every step, a one-hot head the first row of the tied group."""
    kind, eng = tie_engine
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        out = eng.generate(_ids(B, 21, 80 + B), None, _no_video(B), 6)
    st.synchronize()
    assert set(out.flatten().tolist()) <= _allowed(kind), out.tolist()
