"""The references of tests/_act_ref.py checked on the host, before any GPU run: every finite bf16 value through the
fp64 activations and through torch's CPU eager bf16 ops, and the mirrors of the decode projections' row split and
xwin layout.

torch's fp32 eager ops must meet the bar the GPU kernels are held to (_act_ref.check_activation) wherever fp32
arithmetic can: away from the inputs where its exp overflows (silu, the quick-GELU sigmoid) or 1 + erf cancels (GELU,
x < -3), its output is bf16(u * s') for s' the bf16-rounded fp64 activation or a neighbour, and at least 99 % of its
outputs are the fp64 reference's bits. (torch's vectorized CPU GELU also flushes subnormal results to 0.)"""
import math

import numpy as np
import pytest
import torch

import vcl_native as vn
import _act_ref as R

EXP_MAX = float(np.log(np.finfo(np.float32).max))    # 88.72: exp(x) overflows fp32 beyond


def test_every_finite_bf16_value_once():
    v = R.all_finite_bf16()
    assert v.numel() == R.N_FINITE_BF16 == 65280
    assert torch.isfinite(v.float()).all()
    assert torch.unique(v.view(torch.int16)).numel() == v.numel()
    assert v.float().max().item() == torch.finfo(torch.bfloat16).max


def test_bf16_rn_rounds_once():
    x = torch.randn(100000, dtype=torch.float64) * torch.exp2(torch.randint(-140, 120, (100000,)).double())
    x = x.float()                                        # fp32 inputs: torch's conversion rounds once
    assert torch.equal(R.bf16_rn(x.double()).view(torch.int16), x.bfloat16().view(torch.int16))
    # just above a tie of the 8-bit grid: fp64 -> fp32 lands on the tie, and a second rounding goes to even
    t = torch.tensor([1 + 2 ** -8 + 2 ** -30, -(1 + 2 ** -8 + 2 ** -30), 1 + 3 * 2 ** -8 - 2 ** -40], dtype=torch.float64)
    assert t.bfloat16().tolist() != R.bf16_rn(t).tolist()
    assert R.bf16_rn(t).double().tolist() == [1 + 2 ** -7, -(1 + 2 ** -7), 1 + 2 ** -7]
    assert R.bf16_rn(torch.tensor([1e39, -1e39, 3.39e38], dtype=torch.float64)).float().tolist() == \
        [math.inf, -math.inf, torch.finfo(torch.bfloat16).max]


def test_bf16_neighbours():
    v = R.all_finite_bf16()
    dn, up = R.bf16_neighbours(v)
    vf, df, uf = v.double(), dn.double(), up.double()
    assert (df < vf).all() and (uf > vf).all()
    # nothing in between: the neighbours of each value are the adjacent values of the sorted finite set
    s = torch.unique(vf)                                 # +0 and -0 collapse
    i = torch.searchsorted(s, vf)
    inner = (i > 0) & (i < s.numel() - 1)
    assert torch.equal(df[inner], s[i[inner] - 1]) and torch.equal(uf[inner], s[i[inner] + 1])


def _sweep(kind, u_kind="one"):
    x = R.all_finite_bf16()
    if kind == "swiglu":
        u = torch.ones_like(x) if u_kind == "one" else \
            torch.randn(x.numel(), generator=torch.Generator().manual_seed(5)).bfloat16()
        _, s64, ref = R.swiglu_ref(x, u)
        return x, u, s64, ref, R.eager(kind, x, u), -x.float()
    if kind == "qgelu":
        u, s64, ref = R.qgelu_ref(x)
        return x, u, s64, ref, R.eager(kind, x), -R.qgelu_t(x).float()
    u, s64, ref = R.gelu_ref(x)
    return x, u, s64, ref, R.eager(kind, x), None


@pytest.mark.parametrize("kind,u_kind", [("swiglu", "one"), ("swiglu", "random"), ("qgelu", "one"), ("gelu", "one")])
def test_torch_cpu_eager_meets_the_bar(kind, u_kind):
    x, u, s64, ref, eager, exp_arg = _sweep(kind, u_kind)
    inside = R.in_neighbourhood(eager, u, s64)
    outside = ~inside
    if exp_arg is not None:
        # only where fp32 exp overflows, and there the quotient is 0
        overflow = exp_arg > EXP_MAX
        assert not (outside & ~overflow).any(), x[outside & ~overflow][:8].tolist()
        assert (eager[outside].float() == 0).all()
    else:
        # 1 + erf(x / sqrt 2) cancels in fp32 below x = -4; torch's vectorized CPU gelu flushes results below the
        # smallest normal fp32 number to 0, and its x * (1 + erf) overflows from x = 2^127 on
        tiny = torch.finfo(torch.float32).tiny
        allowed = (x.float() < -4) | ((eager.float() == 0) & (s64.float().abs() <= tiny)) | \
                  ((x.float() >= 2.0 ** 127) & (eager.float() == float("inf")))
        assert not (outside & ~allowed).any(), x[outside & ~allowed][:8].tolist()
    # (the subnormal results torch's vectorized CPU code flushes to 0 are not counted: torch on the GPU keeps them)
    kept = ~((eager.float() == 0) & (ref.float() != 0) & (ref.float().abs() <= torch.finfo(torch.float32).tiny))
    same = (eager.view(torch.int16) == ref.view(torch.int16))[kept].float().mean().item()
    print(f"{kind} (up {u_kind}): torch CPU eager outside the fp64 neighbourhood {int(outside.sum())}, "
          f"bit-identical to fp64 {same:.5f}")
    assert same >= 0.99
    masks = R.check_activation(eager, u, s64, eager)
    assert masks["exact"].all() and not masks["bad"].any()


def test_the_fdividef_zone_is_covered():
    """The inputs where __fdividef(x, 1 + e^-x) returns 0 (2^126 < 1 + e^-x < 2^128) are finite bf16 values with a
    normal, nonzero silu that torch's eager op gets right."""
    x = R.all_finite_bf16()
    d = 1.0 + torch.exp(-x.double())
    zone = (d > 2.0 ** 126) & (d < 2.0 ** 128)
    assert sorted(x[zone].float().tolist()) == [-88.5, -88.0, -87.5]
    _, s64, ref = R.swiglu_ref(x[zone], torch.ones(3, dtype=torch.bfloat16))
    assert (ref.float().abs() > torch.finfo(torch.float32).tiny).all()
    assert torch.equal(R.eager("swiglu", x[zone], torch.ones(3, dtype=torch.bfloat16)).view(torch.int16),
                       ref.view(torch.int16))


@pytest.mark.parametrize("N,grid", [(32003, 132), (32003, 114), (2000, 125), (16, 1), (22016, 132), (17, 2)])
def test_cta_row_groups(N, grid):
    parts = R.cta_row_groups(N, grid)
    assert len(parts) == grid
    rows = torch.cat([torch.arange(r0, r0 + n) for r0, n in parts])
    assert torch.equal(rows, torch.arange(N))
    sizes = [n for _, n in parts[:-1]]                   # the last CTA may own a ragged group
    assert all(n > 0 for _, n in parts) and max(sizes, default=16) - min(sizes, default=16) <= 16
    assert all(r0 % 16 == 0 for r0, _ in parts)


@pytest.mark.parametrize("B,K", [(5, 512), (17, 1000), (64, 11008), (33, 1)])
def test_xwin_unpack(B, K):
    n = R.xwin_elems(B, K)
    idx = R.xwin_index(B, K)
    assert idx.shape == (B, K) and idx.min() >= 0 and idx.max() < n
    assert torch.unique(idx).numel() == B * K
    assert idx[B - 1, K - 1].item() == vn.xwin_offset(B - 1, K - 1, B)
    buf = torch.full((n,), -1.0)
    want = torch.arange(B * K, dtype=torch.float32).view(B, K)
    buf[idx.flatten()] = want.flatten()
    got, unused = R.xwin_unpack(buf, B, K)
    assert torch.equal(got, want)
    assert (buf[unused] == -1).all() and int(unused.sum()) == n - B * K
