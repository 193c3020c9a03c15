"""The prefill attention kernels over the KV cache, one launch at a time, against the float64 reference of
tests/_attn_ref.py: attn_prefill_tc_kernel (wgmma, up to 512 keys, attention_prefill_tc.cu) and attn_fwd_kernel
(flash, attention.cu), in every form the engine launches them (prefill_attn_args in vcl_api.cu):
  - cached (vcl_op_attention_cached): a prefill (start 0) or a continuation (prefill_append: start > 0) of B clips,
    with or without left padding;
  - packed (vcl_op_attention_packed): up to 64 sequences in scrambled slots of a contiguous cache, or of a paged pool
    through a block table, wgmma and flash sequences in one launch (vcl_llm_slots_prefill / _chunk / _append).

Input kinds (each case runs the first two):
  - count: q = 0, so every score is exactly 0 and every attended key weighs 1 / n; v[j] is one-hot at
    (7 j + 3 h) % 128. Output element d is then (attended keys in class d) / n, which both kernels compute exactly
    up to the final bf16 rounding: bar 1 bf16 ulp per element. One key too many or too few moves some element by
    1 / n against c / n (c <= ceil(n / 128)).
  - random: q, k, v ~ N(0, 1).
  - rising / falling: q scaled by 8 and aligned with a direction the keys follow more (less) and more along the
    cache, so the row maximum grows on every key tile (the flash kernel rescales on every tile) or is set by the first.
  - spike: the key at a row's own position, or at its key floor, scores far above the rest (p ~ 1 on the mask edge).
  Bars of the last three: relative L2 error per (row, head) < 1e-2 and over the whole output < 4e-3 (the decode
  attention bars of test_kv_cache_gpu.py).

Poisoning: every cache column at or past a sequence's last key is NaN, as are the cache slots and pool blocks no
sequence owns, the other layer of every pool block, and the k | v columns of the q | k | v rows; pad columns are
finite (magnitude 100), because pad queries read them. The output is filled with a NaN sentinel first, so every
row must be written and finite."""
import contextlib
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
import _attn_ref as R  # noqa: E402

DEV = "cuda"
SENTINEL = 0x7FC1          # a bf16 NaN bit pattern no kernel produces
NAN = float("nan")
KINDS = ("count", "random")


@contextlib.contextmanager
def _flash_env(on):
    """VCL_PREFILL_ATTN_FLASH=1 (read per call): the flash kernel for every cached case"""
    if not on:
        yield
        return
    os.environ["VCL_PREFILL_ATTN_FLASH"] = "1"
    try:
        yield
    finally:
        del os.environ["VCL_PREFILL_ATTN_FLASH"]


def _sentinel(rows, H):
    return torch.full((rows, H * 128), SENTINEL, dtype=torch.int16, device=DEV).view(torch.bfloat16)


def _inputs(kind, C, H, cols, rows, pads, seed):
    """q [R, 3 H 128] (q | NaN | NaN, the engine's q | k | v rows) and logical caches k / v [C, H, cols, 128] bf16
    for the rows (clip, pos, kmin); pads: C pad counts or None"""
    clip, pos, kmin = rows
    g = torch.Generator(device=DEV).manual_seed(seed)
    n = len(clip)
    cl, ps, km = (t.to(DEV) for t in (clip, pos, kmin))
    q = torch.randn(n, H, 128, device=DEV, generator=g)
    k = torch.randn(C, H, cols, 128, device=DEV, generator=g)
    v = torch.randn(C, H, cols, 128, device=DEV, generator=g)
    npd = torch.tensor(pads or [0] * C, device=DEV)
    pad_row = ps < npd[cl]
    if kind == "count":
        q.zero_()
        v = R.counting_values(C, H, cols, pads, device=DEV).float()
    elif kind in ("rising", "falling"):
        # score_j ~ 0.5 per 64 keys along the cache (+ noise of ~0.3): ~128 keys carry a row's weight
        u = torch.randn(C, H, 128, device=DEV, generator=g)
        u = u / u.norm(dim=-1, keepdim=True)
        q = 8 * (u[cl] + 0.1 * q)
        j = torch.arange(cols, device=DEV, dtype=torch.float32)
        beta = 0.011 * (j if kind == "rising" else cols - j)
        k = beta[None, None, :, None] * u[:, :, None, :] + 0.3 * k
    for c, p in enumerate(pads or []):   # pad columns: finite, magnitude 100
        k[c, :, :p] *= 100
        if kind != "count":
            v[c, :, :p] *= 100
    if kind != "count":
        q[pad_row] *= 0.01               # pad queries read the pad keys: keep their scores O(1)
    if kind == "spike":
        # real rows: own key (the last row and the middle one of each clip), and one row's key floor
        for c in torch.unique(cl).tolist():
            r_c = (cl == c).nonzero()[:, 0]
            real = r_c[~pad_row[r_c]]
            if len(real) == 0:
                continue
            for r in (real[-1], real[len(real) // 2]):
                k[c, :, ps[r]] = 4 * q[r]
            r = real[len(real) // 3]
            k[c, :, km[r]] = 4 * q[r]
    q = torch.cat([q.reshape(n, H * 128), torch.full((n, 2 * H * 128), NAN, device=DEV)], 1)
    return q.bfloat16(), k.bfloat16(), v.bfloat16()


def _poison(k, v, ends):
    """NaN in every column at or past clip c's last key (ends[c]; None: the whole clip)"""
    for c, e in enumerate(ends):
        k[c, :, e or 0:] = NAN
        v[c, :, e or 0:] = NAN


def _check(o, q, k, v, rows, kind, what):
    """o [R, H * 128] against the reference; returns (max per-(row, head) error, whole-tensor error) or None (count)"""
    H = k.shape[1]
    assert torch.isfinite(o.float()).all(), f"{what} [{kind}]: a row is unwritten (sentinel) or not finite"
    got = o.view(-1, H, 128).double()
    if kind == "count":
        want = R.mean_ref(v, *rows)
        bad = (got - want).abs() > R.bf16_ulp(want)
        assert not bad.any(), (f"{what} [count]: {int(bad.sum())} elements off by more than 1 bf16 ulp, first (row, "
                               f"head, d) {bad.nonzero()[:4].tolist()}: got {got[bad][:4].tolist()} want "
                               f"{want[bad][:4].tolist()}")
        return None
    ref = R.attn_ref(q, k, v, *rows)
    per = (got - ref).norm(dim=-1) / ref.norm(dim=-1).clamp_min(1e-30)
    tot = ((got - ref).norm() / ref.norm()).item()
    worst = divmod(per.argmax().item(), H)
    print(f"[prefill-attn] {what} [{kind}]: max per-(row, head) {per.max().item():.3e} at {worst}, total {tot:.3e}")
    assert per.max().item() < 1e-2 and tot < 4e-3, (what, kind, per.max().item(), worst, tot)
    return per.max().item(), tot


def _launches(fn, want):
    n0 = vn.launch_count()
    out = fn()
    torch.cuda.synchronize()
    assert vn.launch_count() - n0 == want, f"{vn.launch_count() - n0} launches, expected {want}"
    return out


def _cached(q, k, v, start, pads, flash=False):
    B, H = k.shape[:2]
    with _flash_env(flash):
        return _launches(lambda: vn.op_attention_cached(q, k, v, start, pads, out=_sentinel(q.shape[0], H)), 1)


def _cached_case(B, H, start, S, pads, kinds, seed, flash=False):
    """runs each kind on B clips of S queries at start (pads or none); returns {kind: (q, k, v, o)}"""
    cols = start + S + 70
    rows = R.cached_rows(B, start, S, pads)
    out = {}
    for i, kind in enumerate(kinds):
        q, k, v = _inputs(kind, B, H, cols, rows, pads, seed + i)
        _poison(k, v, [start + S] * B)
        o = _cached(q, k, v, start, pads, flash)
        _check(o, q, k, v, rows, kind, f"cached B={B} H={H} start={start} S={S} pads={pads} flash={flash}")
        out[kind] = (q, k, v, o)
    return out


def _both_kernels(B, H, start, S, pads, kinds, seed):
    """a case of at most 512 keys: the wgmma kernel (default), then the flash kernel (VCL_PREFILL_ATTN_FLASH=1) on
    the same inputs; both meet the bars. With S > 16 queries over more than 64 keys their random outputs differ
    somewhere, which shows that two kernels ran: the flash kernel rounds P against the running maximum of each
    64-key tile, the wgmma kernel against the row's final one. Over at most 64 keys (one key tile) the running
    maximum is the final one, and the two kernels agree bit for bit on H100."""
    assert start + S <= 512
    tc = _cached_case(B, H, start, S, pads, kinds, seed)
    fl = _cached_case(B, H, start, S, pads, kinds, seed, flash=True)
    if start + S <= 64:
        assert torch.equal(tc["random"][3], fl["random"][3]), "one key tile: the wgmma and flash runs differ"
    elif S > 16:
        assert not torch.equal(tc["random"][3], fl["random"][3]), "the wgmma and flash runs are bit-identical"


# ------------------------------------------------------------------------------------------
# cached, at most 512 keys: wgmma by default, flash under VCL_PREFILL_ATTN_FLASH=1
WGMMA_CASES = [
    # start, S, extra kinds                 the edge it is for
    (0, 1, ()),                             # one query, one key
    (0, 64, ("spike",)),                    # one full 64-query tile
    (0, 65, ("spike",)),                    # a second query tile holding one row
    (1, 1, ()),                             # continuation by one query over one cached key
    (1, 63, ("spike",)),                    # continuation whose last query sits at key 63 (64-key tile edge)
    (63, 1, ()),                            # single query at the end of the first 64-key tile
    (63, 65, ("spike", "rising")),          # queries straddle the 64- and 128-key edges
    (64, 64, ("spike",)),                   # continuation tile starting exactly on a 64-key edge
    (127, 129, ("spike", "rising")),        # last key 255: queries cross the 128-key block edge twice
    (200, 37, ("falling",)),                # mid-block start, short tail
    (384, 128, ("spike", "rising")),        # ends exactly at 512: four key blocks
    (447, 65, ("spike",)),                  # ends at 512 from a start one below a 64-key edge
    (511, 1, ("spike",)),                   # one query on key 511
]


@torch.no_grad()
@pytest.mark.parametrize("start,S,extra", WGMMA_CASES)
def test_cached_up_to_512_keys(start, S, extra):
    """attn_prefill_tc_kernel<false, false> (key blocks n_kb from last_key, mask key > qpos) and, under
    VCL_PREFILL_ATTN_FLASH, attn_fwd_kernel<128, true> (tiles n_tiles, mask kidx > qrow + q_off), B = 2, H = 2"""
    _both_kernels(2, 2, start, S, None, KINDS + extra, seed=start * 7 + S)


@torch.no_grad()
def test_cached_32_heads():
    """H = 32 (the 7B model's heads): the head stride of q, the cache and o"""
    _both_kernels(1, 32, 127, 129, None, KINDS + ("spike",), seed=32)


FLASH_CASES = [
    # start, S, extra kinds                 the edge it is for (attn_fwd_kernel<128, true>: more than 512 keys)
    (512, 1, ()),                           # one query on key 512, the first beyond the wgmma kernel
    (500, 37, ("spike", "rising")),         # queries cross 512
    (577, 64, ("spike",)),                  # a 64-query tile that is not 64-key aligned
    (960, 64, ("rising",)),                 # aligned tile ending at 1024: 16 key tiles
    (640, 384, ("spike", "rising", "falling")),   # six query tiles, ending at 1024
    (1000, 24, ("spike",)),                 # short tail deep in the cache
]


@torch.no_grad()
@pytest.mark.parametrize("start,S,extra", FLASH_CASES)
def test_cached_past_512_keys(start, S, extra):
    _cached_case(2, 2, start, S, None, KINDS + extra, seed=start * 7 + S)


# ------------------------------------------------------------------------------------------
# left padding, B = 3 (PAD kernels: kmin of the rows, kb0 = k_pad / 128 and jt0 = k_pad / 64 skips)
PAD_CASES = [
    # start, S, pads                        the edge it is for
    (0, 200, [0, 63, 129]),                 # new sequence: pad queries inside the first tiles (causal from key 0)
    (0, 200, [1, 64, 199]),                 # one pad; a 64-key edge; S - 1 pads (one real query)
    (0, 200, [127, 128, 0]),                # the 128-key block edge from both sides
    (300, 100, [129, 0, 64]),               # continuation ending below 512 keys (wgmma, kb0 > 0)
    (600, 64, [128, 63, 129]),              # continuation past 512 keys (flash, jt0 > 0)
    (0, 700, [0, 127, 699]),                # new sequence past 512 keys: flash with pad queries over 11 tiles
]


@torch.no_grad()
@pytest.mark.parametrize("start,S,pads", PAD_CASES)
def test_cached_left_padding(start, S, pads):
    """attn_prefill_tc_kernel<true, false> up to 512 keys (and the flash kernel under VCL_PREFILL_ATTN_FLASH),
    attn_fwd_kernel<128, true, true> beyond"""
    kinds = KINDS + ("spike", "rising")
    if start + S <= 512:
        _both_kernels(3, 2, start, S, pads, kinds, seed=start + S + sum(pads))
    else:
        _cached_case(3, 2, start, S, pads, kinds, seed=start + S + sum(pads))


# ------------------------------------------------------------------------------------------
# packed
def _pool(k, v, slots, ends, layers, layer, seed):
    """the logical caches k / v [C, H, cols, 128] laid out in a paged pool [n_blocks][layers][K | V][H][128][128]
    through a scrambled table; blocks no sequence owns and every other layer are NaN. Returns (pool, table)."""
    C, H, cols = k.shape[:3]
    row = (cols + 127) // 128
    need = {s: (e + 127) // 128 for s, e in zip(slots, ends)}
    n_blocks = sum(need.values()) + 3
    g = torch.Generator().manual_seed(seed)
    ids = torch.randperm(n_blocks, generator=g).tolist()
    spare = ids[sum(need.values()):]
    pool = torch.full((n_blocks, layers, 2, H, 128, 128), NAN, dtype=torch.bfloat16, device=DEV)
    table = [[spare[(s + kb) % len(spare)] for kb in range(row)] for s in range(C)]
    for s, nb in need.items():
        for kb in range(nb):
            b = ids.pop(0)
            table[s][kb] = b
            w = min(128, cols - kb * 128)
            pool[b, layer, 0, :, :w] = k[s, :, kb * 128:kb * 128 + w]
            pool[b, layer, 1, :, :w] = v[s, :, kb * 128:kb * 128 + w]
    return pool, table


def _packed_run(q, k, v, seqs, paged, layers=2, layer=1, seed=0, check_launches=True):
    """seqs: [(slot, start, len, flash)]; k / v the logical caches. Runs vcl_op_attention_packed on the contiguous
    cache or (paged) on a pool holding them at layer `layer`."""
    slots, starts, lens, flash = (list(t) for t in zip(*seqs))
    H = k.shape[1]
    kinds = 1 + (any(flash) and not all(flash))
    out = _sentinel(sum(lens), H)
    if not paged:
        fn = lambda: vn.op_attention_packed(q, k, v, slots, starts, lens, flash, out=out)   # noqa: E731
    else:
        pool, table = _pool(k, v, slots, [a + n for a, n in zip(starts, lens)], layers, layer, seed)
        blk = pool[0].numel()
        fn = lambda: vn.op_attention_packed(q, pool[0, layer, 0], pool[0, layer, 1], slots, starts, lens,  # noqa: E731
                                            flash, table=table, n_blocks=pool.shape[0], blk=blk,
                                            s_max=k.shape[2], out=out)
    return _launches(fn, kinds) if check_launches else fn()


def _packed_case(seqs, n_slots, H, paged, kinds, seed):
    """each kind: the packed launch against the reference; then (random kind) every sequence bit for bit against
    the cached kernel in a clip of its own at the same start (the flash kernel for flash sequences, under
    VCL_PREFILL_ATTN_FLASH when they end at or below 512 keys), and on a pool the wgmma sequences against the same
    sequences packed on the contiguous cache"""
    slots = [s[0] for s in seqs]
    ends = {s: a + n for s, a, n, _ in seqs}
    cols = (max(ends.values()) + 127) // 128 * 128 + 128
    rows = R.packed_rows(slots, [s[1] for s in seqs], [s[2] for s in seqs])
    what = f"packed {'paged' if paged else 'contiguous'} n={len(seqs)}"
    for i, kind in enumerate(kinds):
        q, k, v = _inputs(kind, n_slots, H, cols, rows, None, seed + i)
        _poison(k, v, [ends.get(c) for c in range(n_slots)])
        o = _packed_run(q, k, v, seqs, paged, seed=seed)
        _check(o, q, k, v, rows, kind, what)
        if kind != "random":
            continue
        off = 0
        for slot, start, n, fl in seqs:
            alone = _cached(q[off:off + n], k[slot:slot + 1], v[slot:slot + 1], start, None,
                            flash=fl and start + n <= 512)
            assert torch.equal(alone, o[off:off + n]), f"{what}: sequence at slot {slot} start {start} len {n}"
            off += n
        tc = [s for s in seqs if not s[3]]
        if paged and tc:
            qi = torch.cat([q[r] for r in _seq_rows(seqs, tc)])
            oc = _packed_run(qi, k, v, tc, False)
            assert torch.equal(oc, torch.cat([o[r] for r in _seq_rows(seqs, tc)])), f"{what}: pool vs contiguous"


def _seq_rows(seqs, sub):
    offs, off = {}, 0
    for s in seqs:
        offs[s] = slice(off, off + s[2])
        off += s[2]
    return [offs[s] for s in sub]


def _scrambled(lens, n_slots, seed, starts=None):
    g = torch.Generator().manual_seed(seed)
    slots = torch.randperm(n_slots, generator=g)[:len(lens)].tolist()
    return [(s, (starts or [0] * len(lens))[i], n, False) for i, (s, n) in enumerate(zip(slots, lens))]


def _lens64():
    g = torch.Generator().manual_seed(64)
    lens = torch.randint(1, 97, (64,), generator=g).tolist()
    lens[17] = 512
    return lens


PACKED_CONTIGUOUS = {
    # attn_prefill_tc_kernel<false, true>: blockIdx.z is the sequence, its keys clip slot_i
    "one": ([512], 3, None),                                      # a single whole 512-token prompt
    "five": ([512, 1, 65, 200, 129], 8, None),                    # lens across the tile edges, three unused slots
    "sixty_four": (_lens64(), 70, None),                          # PACK_SEQ_MAX sequences, one of 512
    "tails": ([37, 65, 1, 256], 6, [100, 447, 1, 256]),           # continuations (start > 0), ending at <= 512 keys
}


@torch.no_grad()
@pytest.mark.parametrize("name", list(PACKED_CONTIGUOUS))
def test_packed_contiguous(name):
    lens, n_slots, starts = PACKED_CONTIGUOUS[name]
    seqs = _scrambled(lens, n_slots, seed=len(lens) + n_slots, starts=starts)
    _packed_case(seqs, n_slots, 2, False, KINDS + ("spike",), seed=n_slots)


PACKED_PAGED = {
    # (slot, start, len, flash): attn_prefill_tc_kernel<false, true, true> and attn_fwd_kernel<128, true, false,
    # true, true> (key tile jt at (jt & 1) * 64 of block table[slot][jt / 2]) in one launch each
    "chunks": [(5, 0, 128, False),       # a whole prompt ending on a block boundary
               (0, 512, 128, True),      # a chunk of a long prompt ending on a block boundary (640)
               (3, 0, 256, True),        # the first chunk of a long prompt, on the flash kernel
               (7, 256, 256, False),     # wgmma, ending at 512
               (2, 64, 65, True),        # a chunk at a 64-multiple start ending one past a block (129)
               (6, 448, 65, True)],      # ending at 513, one past the wgmma limit
    "tails": [(1, 500, 37, True),        # appended tails past 512 keys (vcl_llm_slots_prefill_append)
              (4, 577, 64, True),
              (0, 1000, 24, True),
              (6, 128, 128, False),      # a wgmma tail ending at 256
              (2, 0, 129, False)],       # a whole prompt ending one past a block
}


@torch.no_grad()
@pytest.mark.parametrize("name", list(PACKED_PAGED))
def test_packed_paged(name):
    """wgmma and flash sequences in one packed launch on a paged pool of 2 layers, read at layer 1 (a block or
    layer stride mistake reads NaN)"""
    _packed_case(PACKED_PAGED[name], 9, 2, True, KINDS + ("spike", "rising"), seed=len(name))


# ------------------------------------------------------------------------------------------
# rejections
def _valid_cached():
    q = torch.zeros(2 * 8, 3 * 2 * 128, dtype=torch.bfloat16, device=DEV)
    k = torch.zeros(2, 2, 32, 128, dtype=torch.bfloat16, device=DEV)
    return q, k


CACHED_BAD = [
    # (what, q_ld, B, H, s_max, start, S, pads)                match
    (dict(q_ld=200), "q_ld"),                                   # below H * 128
    (dict(q_ld=3 * 2 * 128 - 4), "q_ld"),                       # not a multiple of 8
    (dict(H=0), "H=0"),
    (dict(start=20, S=13), "outside the cache"),                # start + S > s_max
    (dict(S=0), "outside the cache"),
    (dict(pads=[0, -1]), r"n_pad\[1\]"),
    (dict(pads=[8, 0]), r"n_pad\[0\]"),                          # n_pad >= start + S at start 0
    (dict(start=4, pads=[4, 0]), "start_pos 4 lies inside"),    # a continuation inside the padding
]


def _call_cached(q, k, q_ld=3 * 2 * 128, B=2, H=2, s_max=32, start=0, S=8, pads=None, o=None):
    o = o if o is not None else torch.zeros(B * S if S > 0 else 1, max(H, 1) * 128, dtype=torch.bfloat16, device=DEV)
    p = None if pads is None else (vn.c_int32 * len(pads))(*pads)
    vn.check(vn.lib().vcl_op_attention_cached(vn.ptr(q), q_ld, vn.ptr(k), vn.ptr(k), vn.ptr(o), B, H, s_max, start, S,
                                              p, vn.cur_stream()))
    return o


@torch.no_grad()
@pytest.mark.parametrize("bad,match", CACHED_BAD)
def test_cached_rejects(bad, match):
    """every invalid argument is named and refused before any launch; a valid call afterwards still runs"""
    q, k = _valid_cached()
    n0 = vn.launch_count()
    with pytest.raises(vn.VclError, match=match):
        _call_cached(q, k, **bad)
    assert vn.launch_count() == n0
    _launches(lambda: _call_cached(q, k, pads=[3, 0]), 1)


def _valid_packed():
    H, L, n_blocks = 2, 2, 6
    pool = torch.zeros(n_blocks, L, 2, H, 128, 128, dtype=torch.bfloat16, device=DEV)
    q = torch.zeros(700, 3 * H * 128, dtype=torch.bfloat16, device=DEV)
    return q, pool


def _call_packed(q, pool, seqs=((0, 0, 8, 0), (1, 600, 8, 1)), table=((1, 2, 3, 4, 5, 0, 0, 0), (2, 3, 4, 5, 1, 0, 0, 0)),
                 n=None, q_ld=768, s_max=1024, n_blocks=None, paged=True, k=None):
    slots, starts, lens, flash = (list(t) for t in zip(*seqs)) if seqs else ([], [], [], [])
    n = len(seqs) if n is None else n
    rows = max(sum(lens), 1)
    o = torch.zeros(rows, 256, dtype=torch.bfloat16, device=DEV)
    ints = lambda v: (vn.c_int32 * max(len(v), 1))(*v)   # noqa: E731
    n_slots = len(table)
    if paged:
        kp, vp = pool[0, 1, 0], pool[0, 1, 1]
        tab, row = ints([b for r in table for b in r]), len(table[0])
    else:
        kp = vp = k
        tab, row = None, 0
    vn.check(vn.lib().vcl_op_attention_packed(
        vn.ptr(q), q_ld, vn.c_void_p(kp.data_ptr()), vn.c_void_p(vp.data_ptr()), vn.ptr(o), 2, s_max, n_slots, n,
        ints(slots), ints(starts), ints(lens), ints(flash), tab, row, pool.shape[0] if n_blocks is None else n_blocks,
        pool[0].numel(), vn.cur_stream()))
    return o


PACKED_BAD = [
    (dict(n=0, seqs=()), "n=0"),
    (dict(seqs=tuple((i % 2, 0, 1, 0) for i in range(65))), "n=65"),
    (dict(seqs=((0, 0, 0, 0),)), "sequence 0 has 0 rows"),
    (dict(seqs=((0, 0, 513, 1),)), "sequence 0 has 513 rows"),
    (dict(seqs=((0, 0, 8, 0), (1, 500, 13, 0))), "sequence 1 ends at 513 keys"),     # wgmma past 512 keys
    (dict(seqs=((0, 1020, 8, 1),)), "outside the cache"),                             # start + len > s_max
    (dict(seqs=((2, 0, 8, 0),)), "slot 2 outside"),
    (dict(q_ld=200), "q_ld"),
    (dict(table=((1, 2, 3, 4, 5, 0, 0, 0), (2, 3, 4, 5, 6, 0, 0, 0))), r"table\[1\]\[4\] = 6"),   # past the pool
    (dict(table=((1, 2, 3, 4, 5, 0, 0, 0), (2, 3, -1, 5, 1, 0, 0, 0))), r"table\[1\]\[2\] = -1"),
    (dict(table=((1, 2, 3, 4, 5, 0, 0), (2, 3, 4, 5, 1, 0, 0))), "table_row=7"),   # too short for s_max 1024
]


@torch.no_grad()
@pytest.mark.parametrize("bad,match", PACKED_BAD)
def test_packed_rejects(bad, match):
    q, pool = _valid_packed()
    n0 = vn.launch_count()
    with pytest.raises(vn.VclError, match=match):
        _call_packed(q, pool, **bad)
    assert vn.launch_count() == n0
    _launches(lambda: _call_packed(q, pool), 2)                  # one wgmma and one flash sequence


@torch.no_grad()
def test_packed_rejects_flash_on_a_contiguous_cache():
    q, pool = _valid_packed()
    k = torch.zeros(2, 2, 1024, 128, dtype=torch.bfloat16, device=DEV)
    n0 = vn.launch_count()
    with pytest.raises(vn.VclError, match="sequence 1 is on the flash kernel"):
        _call_packed(q, pool, paged=False, k=k)
    assert vn.launch_count() == n0
    _launches(lambda: _call_packed(q, pool, seqs=((0, 0, 8, 0), (1, 100, 8, 0)), paged=False, k=k), 1)
