"""The GEMM's exact reference (tests/_gemm_ref.py) checked on the host before any GPU run: the exactness bound holds
for every summation order, bf16_rn rounds integers once with ties to even, the residual is rounded after the GEMM
output as the store warps' bf16x2 add does, and the poisoned views have the pitches, alignment and sentinel margins
the GPU tests rely on."""
import pytest
import torch

import _gemm_ref as G
from _act_ref import bf16_rn


def _rn_int(n, bits=8):
    """round the integer n to `bits` significant bits, ties to even, with integer arithmetic"""
    s = max(abs(n).bit_length() - bits, 0)
    if s == 0:
        return n
    q, r = divmod(abs(n), 1 << s)
    half = 1 << (s - 1)
    if r > half or (r == half and q % 2 == 1):
        q += 1
    return (q << s) * (1 if n >= 0 else -1)


@pytest.mark.parametrize("K", [64, 640, 4096, 13824])
def test_exact_bound_every_order(K):
    """the bound is below 2^24 at the engine's largest K, and fp32 sums of the products in any order equal the
    float64 sum: random operands in shuffled K orders, and the worst case, where every product is the largest"""
    assert G.exact_bound(K) == K * 2 + 8 < 2 ** 24
    a, w, b, _ = G.operands(4, 6, K, seed=K, bias=True)
    y = G.gemm_exact(a, w, b)
    assert torch.equal(y, y.round()) and y.abs().max() <= G.exact_bound(K)
    prods = a.float()[:, None, :] * w.float()[None, :, :]                 # [M, N, K], exact in fp32
    for seed in range(4):
        perm = torch.randperm(K, generator=torch.Generator().manual_seed(seed))
        acc = torch.zeros(4, 6, dtype=torch.float32)
        for k in perm.tolist():                                           # one fp32 rounding per addition
            acc += prods[:, :, k]
        assert torch.equal((acc + b.float()).double(), y)
    worst = torch.full((K,), 2.0 * 1.0)
    acc = torch.zeros((), dtype=torch.float32)
    for p in worst:
        acc += p
    assert float(acc) + 8 == G.exact_bound(K)


def test_exact_bound_refuses():
    with pytest.raises(AssertionError):
        G.exact_bound(2 ** 23)
    with pytest.raises(AssertionError):
        G.operands(1, 1, 2 ** 23, seed=0)


def test_operands_are_exact_integers():
    a, w, b, r = G.operands(33, 40, 128, seed=3, bias=True, res_cols=40)
    for t, lim in ((a, G.A_MAX), (w, G.W_MAX), (b, G.BIAS_MAX), (r, G.RES_MAX)):
        v = t.double()
        assert torch.equal(v, v.round()) and v.abs().max() == lim and v.min() == -lim
    _, ws, bs, _ = G.operands(33, 40, 128, seed=3, bias=True, w_exp=-3)
    assert torch.equal(ws.double(), w.double() / 8) and torch.equal(bs.double(), b.double() / 8)


def test_bf16_rn_integers():
    """every integer 2^8 ... 2^24 class: ties (halfway between two bf16 values) round to the even mantissa, the
    integers next to a tie round to the nearer value, and torch's fp64 -> bf16 conversion would differ on some"""
    ns = []
    for s in range(1, 17):                                # integers in [2^(s+7), 2^(s+8)): bf16 spacing 2^s
        for q in (128, 129, 130, 200, 254, 255):
            base = q << s
            ns += [base, base + (1 << (s - 1)), base + (1 << (s - 1)) - 1, base + (1 << (s - 1)) + 1, base + 1]
    ns += [2 ** 8, 2 ** 24, 2 ** 24 - 1, 2 ** 24 - 2 ** 15, 2 ** 24 - 2 ** 15 - 1]
    ns += torch.randint(2 ** 8, 2 ** 24, (20000,), generator=torch.Generator().manual_seed(1)).tolist()
    ns += [-n for n in ns]
    got = bf16_rn(torch.tensor(ns, dtype=torch.float64)).double().tolist()
    want = [float(_rn_int(n)) for n in ns]
    assert got == want
    # within fp32's 24 bits there is no double rounding: bf16_rn agrees with torch's conversion through fp32
    t = torch.tensor(ns, dtype=torch.float64)
    assert torch.equal(bf16_rn(t).view(torch.int16), t.float().bfloat16().view(torch.int16))


def test_residual_rounds_after_the_gemm_output():
    """bf16(bf16(y) + res), not bf16(y + res): 513 rounds to 512 (spacing 4), + 2 = 514 is a tie that goes to 512,
    while 515 rounds to 516; and the rule is torch's eager bf16 add of the rounded GEMM output and the residual"""
    y = torch.tensor([513.0, 259.0, -513.0], dtype=torch.float64)
    res = torch.tensor([2.0, 1.0, -2.0]).bfloat16()
    assert G.plain_out(y, res).double().tolist() == [512.0, 260.0, -512.0]
    assert bf16_rn(y + res.double()).double().tolist() == [516.0, 260.0, -516.0]
    a, w, _, r = G.operands(64, 96, 4096, seed=9, res_cols=96)
    y = G.gemm_exact(a, w)
    assert torch.equal(G.plain_out(y, r).view(torch.int16), (bf16_rn(y) + r).view(torch.int16))
    assert not torch.equal(G.plain_out(y, r), bf16_rn(y + r.double()))   # the two rules differ at these sizes


def test_padded_views():
    buf, v = G.padded(5, 24, top=2, bottom=3, pad_cols=16, fill=G.SENTINEL)
    assert buf.shape == (10, 40) and v.shape == (5, 24) and v.stride() == (40, 1)
    assert G.view_origin(buf, v) == (2, 0)
    assert (v.stride(0) * v.element_size()) % 16 == 0 and (v.data_ptr() - buf.data_ptr()) % 16 == 0
    assert (buf.view(torch.int16) == G.SENTINEL).all() and torch.isnan(buf.float()).all()
    bufa, va = G.padded(3, 64, top=1, bottom=1, pad_cols=8)
    assert torch.isnan(bufa.float()).all() and va.stride(0) == 72
    with pytest.raises(AssertionError):
        G.padded(3, 64, pad_cols=4)
    # buffer_check: a written view passes; one margin write and one unwritten element are both seen
    ref = torch.arange(120, dtype=torch.float32).view(5, 24).bfloat16()
    v.copy_(ref)
    assert [int(x) for x in G.buffer_check(buf, v, ref)] == [0, 0]
    buf[7, 0] = 1.0                                       # the row below the view
    buf[3, 24] = 1.0                                      # a pad column
    v[4, 23] = float("nan")
    v[0, 0] = -0.0                                        # ref is +0 there: the sign of zero is folded
    assert [int(x) for x in G.buffer_check(buf, v, ref)] == [1, 2]
    fresh_buf, fresh = G.padded(5, 24, top=2, bottom=3, pad_cols=16, fill=G.SENTINEL)
    assert int(G.buffer_check(fresh_buf, fresh, ref)[0]) == 120     # an unwritten view fails everywhere


@pytest.mark.parametrize("K", [64, 1024, 4096])
def test_probe_codes(K):
    """the one-hot columns cover every k; the codes are exact bf16 values, distinct along k for every row, and
    decode back to their column"""
    i = torch.arange(K)
    assert torch.equal(torch.sort(G.probe_k(i, K)).values, i)
    for j in (0, 1, 77, 4099):
        codes = G.probe_code(torch.full((K,), j), i, K)
        assert torch.isfinite(codes.float()).all() and (codes.float() > 0).all()
        assert torch.unique(codes.view(torch.int16)).numel() == K
        assert torch.equal(G.probe_decode(codes, j, K), i)
    bad = torch.tensor([float("nan"), 0.0, -1.0, 1e-30, 2.0 ** 30]).bfloat16()
    assert (G.probe_decode(bad, 0, K) == -1).all()
