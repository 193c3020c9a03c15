"""The float64 attention reference of tests/_attn_ref.py on the CPU: its masks against dense boolean masks built
independently from the rules of kernels.h (left padding, continuations, packed sequences), and the counting input of
tests/test_prefill_attention_gpu.py against its closed form."""
import pytest
import torch

import _attn_ref as R


def _dense_cached(B, start, S, n_pad, n_keys):
    """[B * S, B, n_keys]: kernels.h, positions in the KV cache. Clip b's query j sits at column c = start + j; a real
    query (c >= n_pad[b]) attends keys n_pad[b] .. c, a pad query attends causally from key 0; no other clip."""
    m = torch.zeros(B * S, B, n_keys, dtype=torch.bool)
    for b in range(B):
        for j in range(S):
            c = start + j
            lo = n_pad[b] if c >= n_pad[b] else 0
            for key in range(lo, c + 1):
                m[b * S + j, b, key] = True
    return m


def _dense_packed(slots, starts, lens, n_slots, n_keys):
    """[sum lens, n_slots, n_keys]: kernels.h, packed prefill. Sequence i's rows follow sequence i - 1's; its row j
    sits at position start_i + j and attends keys 0 .. start_i + j of slot_i only."""
    m = torch.zeros(sum(lens), n_slots, n_keys, dtype=torch.bool)
    r = 0
    for s, a, n in zip(slots, starts, lens):
        for j in range(n):
            m[r, s, :a + j + 1] = True
            r += 1
    return m


def _from_rows(clip, pos, kmin, C, n_keys):
    """the reference's mask spread over every clip: row r's mask sits in clip[r]"""
    m = torch.zeros(len(clip), C, n_keys, dtype=torch.bool)
    rm = R.ref_mask(pos, kmin, n_keys)
    m[torch.arange(len(clip)), clip] = rm
    return m


@pytest.mark.parametrize("B,start,S,n_pad", [
    (1, 0, 77, None), (3, 0, 130, [0, 64, 129]), (3, 0, 130, [1, 63, 128]), (2, 200, 37, [127, 0]),
    (3, 512, 64, [0, 129, 511]), (2, 1, 1, None), (3, 0, 5, [4, 0, 1])])
def test_cached_masks(B, start, S, n_pad):
    """prefill / continuation / left padding: the rows cached_rows describes attend exactly the keys of the rules"""
    n_keys = start + S + 3
    clip, pos, kmin = R.cached_rows(B, start, S, n_pad)
    want = _dense_cached(B, start, S, n_pad or [0] * B, n_keys)
    assert torch.equal(_from_rows(clip, pos, kmin, B, n_keys), want)


@pytest.mark.parametrize("slots,starts,lens", [
    ([0], [0], [512]), ([3, 0, 6, 1], [0, 0, 100, 577], [65, 1, 37, 64]), ([2, 1], [1000, 448], [24, 65])])
def test_packed_masks(slots, starts, lens):
    n_slots, n_keys = max(slots) + 2, max(a + n for a, n in zip(starts, lens)) + 5
    clip, pos, kmin = R.packed_rows(slots, starts, lens)
    want = _dense_packed(slots, starts, lens, n_slots, n_keys)
    assert torch.equal(_from_rows(clip, pos, kmin, n_slots, n_keys), want)


def test_decode_rows_are_real_queries():
    """a decode query at column c >= n_pad takes the floor n_pad, as decode_attention.cu's keys n_pad .. c"""
    for c, npd in [(0, 0), (39, 39), (40, 12), (5, 0)]:
        assert R.key_floor(c, npd) == npd
    assert R.key_floor(3, 4) == 0


def _rand(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g, dtype=torch.float64) * scale).bfloat16()


@pytest.mark.parametrize("B,start,S,n_pad", [(3, 0, 130, [0, 64, 129]), (2, 200, 37, [127, 0])])
def test_counting_input_closed_form(B, start, S, n_pad):
    """q = 0 and one-hot values (counting_values): every score is 0, so the reference's p is bf16(1 / n) (n the
    attended keys) and its output is that times the attended values' sum per class; mean_ref gives the exact
    (sum in class d) / n. Both are checked against a count taken over the dense mask of the rules, and the pad
    columns (value 100) count 100 times."""
    H, cols = 2, start + S + 7
    g = torch.Generator().manual_seed(B + S)
    clip, pos, kmin = R.cached_rows(B, start, S, n_pad)
    q = torch.zeros(B * S, 3 * H * 128, dtype=torch.bfloat16)
    k = _rand((B, H, cols, 128), g)
    v = R.counting_values(B, H, cols, n_pad)
    dense = _dense_cached(B, start, S, n_pad, cols)                               # [R, B, cols]
    want = torch.zeros(B * S, H, 128, dtype=torch.float64)
    n = torch.zeros(B * S, dtype=torch.float64)
    for r in range(B * S):
        b = int(clip[r])
        keys = dense[r, b].nonzero()[:, 0].tolist()
        n[r] = len(keys)
        for h in range(H):
            for j in keys:
                want[r, h, (7 * j + 3 * h) % 128] += 100.0 if j < n_pad[b] else 1.0
    exact = R.mean_ref(v, clip, pos, kmin)
    assert torch.equal(exact, want / n[:, None, None])
    p = (1.0 / n).float().bfloat16().double()                                       # fp32 softmax of n zeros
    assert torch.equal(R.attn_ref(q, k, v, clip, pos, kmin), want * p[:, None, None])


def test_reference_ignores_poisoned_columns_and_rejects_attended_ones():
    """NaN outside the attended keys leaves the output finite and unchanged; NaN in an attended key is an error of
    the test's construction, so the reference refuses it"""
    g = torch.Generator().manual_seed(5)
    B, H, S, cols = 2, 2, 40, 64
    clip, pos, kmin = R.cached_rows(B, 0, S, [3, 0])
    q = _rand((B * S, H * 128), g)
    k, v = _rand((B, H, cols, 128), g), _rand((B, H, cols, 128), g)
    clean = R.attn_ref(q, k, v, clip, pos, kmin)
    kp, vp = k.clone(), v.clone()
    kp[:, :, S:] = float("nan"); vp[:, :, S:] = float("nan")
    assert torch.equal(R.attn_ref(q, kp, vp, clip, pos, kmin), clean)
    kp[0, :, 1] = float("nan")                                                    # a pad key clip 0's pad rows read
    with pytest.raises(AssertionError, match="attended"):
        R.attn_ref(q, kp, vp, clip, pos, kmin)


def test_reference_matches_a_direct_evaluation():
    """attn_ref against a row-by-row evaluation of the same rounding points over explicit key lists"""
    g = torch.Generator().manual_seed(9)
    B, H, start, S, cols = 2, 3, 20, 9, 40
    n_pad = [0, 7]
    clip, pos, kmin = R.cached_rows(B, start, S, n_pad)
    q = _rand((B * S, 3 * H * 128), g)
    k, v = _rand((B, H, cols, 128), g), _rand((B, H, cols, 128), g, 4.0)
    got = R.attn_ref(q, k, v, clip, pos, kmin)
    sc = torch.tensor(R.SCALE, dtype=torch.float32)
    for r in range(B * S):
        b, c = int(clip[r]), int(pos[r])
        lo = n_pad[b] if c >= n_pad[b] else 0
        for h in range(H):
            qh = q[r, h * 128:(h + 1) * 128].double()
            s = torch.stack([(qh * k[b, h, j].double()).sum() for j in range(lo, c + 1)]).bfloat16().float()
            p = torch.softmax((s * sc).bfloat16().float(), 0).bfloat16().double()
            want = (p[:, None] * v[b, h, lo:c + 1].double()).sum(0)
            assert torch.allclose(got[r, h], want, rtol=0, atol=1e-12), (r, h)


def test_bf16_ulp():
    x = torch.tensor([1.0, 1.5, 0.75, 3.0e-3, 0.0, -2.0], dtype=torch.float64)
    want = torch.tensor([2 ** -7, 2 ** -7, 2 ** -8, 2.0 ** -16, 2.0 ** -133, 2 ** -6], dtype=torch.float64)
    assert torch.equal(R.bf16_ulp(x), want)


def _bf16_p(n):
    """the decode kernel's weight of one of n equal keys: bf16(fp32(1) / fp32(n))"""
    return float(torch.tensor(1.0, dtype=torch.float32).div(torch.tensor(float(n), dtype=torch.float32)).bfloat16())


def _decode_rows(kv_len, pos, n_pad):
    """decode rows (clip b, pos = kv_len - 1 + pos[b], kmin = n_pad[b]) as test_decode_attention_gpu.py builds them"""
    B = len(pos)
    return (torch.arange(B), torch.tensor([kv_len - 1 + p for p in pos]), torch.tensor(n_pad))


@pytest.mark.parametrize("kv_len,pos,n_pad", [(1, [0, 0], [0, 0]), (30, [0, 170, 3], [0, 29, 5]),
                                              (300, [0, 77], [128, 1])])
def test_equal_weight_closed_form_counts(kv_len, pos, n_pad):
    """counting input, pad and out-of-range columns NaN: equal_weight_ref against a key-by-key count of the classes
    (7 j + 3 h) % 128 over keys n_pad .. c and the rounding bf16(c_d * bf16(fp32(1 / n)))"""
    H = 3
    clip, p, kmin = _decode_rows(kv_len, pos, n_pad)
    cols = int(p.max()) + 5
    v = R.counting_values(len(pos), H, cols)
    for b in range(len(pos)):
        v[b, :, :n_pad[b]] = float("nan")
        v[b, :, int(p[b]) + 1:] = float("nan")
    got = R.equal_weight_ref(v, clip, p, kmin)
    for b in range(len(pos)):
        keys = range(n_pad[b], int(p[b]) + 1)
        pb = _bf16_p(len(keys))
        for h in range(H):
            cnt = [0] * 128
            for j in keys:
                cnt[(7 * j + 3 * h) % 128] += 1
            want = torch.tensor([c * pb for c in cnt], dtype=torch.float64).bfloat16().double()
            assert torch.equal(got[b, h], want), (b, h)


def test_probe_plan_covers_every_key_once_with_neighbours_apart():
    for keys in ([5], [0, 1], list(range(3, 260)), list(range(1000, 1000 + 128 * 9 + 1)), [7, 9, 130, 131, 4000]):
        plan = R.probe_plan(keys)
        got = sorted(j for s in plan for j, _ in s)
        assert got == sorted(keys)
        where = {j: i for i, s in enumerate(plan) for j, _ in s}
        for s in plan:
            assert len(s) <= 128 and len({d for _, d in s}) == len(s)
        for a, b in zip(sorted(keys), sorted(keys)[1:]):
            assert where[a] != where[b], (a, b)


def test_probe_closed_form():
    """probe input: an attended probe gives bf16(p) at its dimension, an unattended one (below the floor, past the
    last key) nothing; a probe read twice would give bf16(2 p), which is a different bf16 number"""
    B, H, kv_len, pos, n_pad = 2, 2, 200, [0, 57], [10, 0]
    clip, p, kmin = _decode_rows(kv_len, pos, n_pad)
    cols = 300
    sets = [[[(3, 0), (10, 1), (11, 2), (199, 3), (200, 4)], [(150, 127)]],
            [[(0, 5), (256, 6), (257, 7)], None]]
    v = R.probe_values(B, H, cols, sets)
    got = R.equal_weight_ref(v, clip, p, kmin)
    for b in range(B):
        lo, hi = n_pad[b], int(p[b])
        pb = _bf16_p(hi - lo + 1)
        for h in range(H):
            want = torch.zeros(128, dtype=torch.float64)
            for j, d in sets[b][h] or []:
                if lo <= j <= hi:
                    want[d] += pb
            assert torch.equal(got[b, h], want), (b, h)
        assert float(torch.tensor(2 * pb).bfloat16()) != pb
