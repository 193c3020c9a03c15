"""Per-kernel parity on the GPU: every CUDA kernel of libvcl against a plain PyTorch fp32
evaluation of the same operator on the same bf16 inputs (tolerances stated per test).
The end-to-end parity against the oracle lives in test_parity_gpu.py."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402


def _dev():
    return torch.device("cuda:0")


def _rel(a, b):
    a = a.float(); b = b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-20)).item()


def _describe(out, ref):
    """Where are the wrong elements? (helps to tell a descriptor bug from a pipeline bug)"""
    d = (out.float() - ref.float()).abs()
    tol = 0.02 * ref.float().abs().max().item() + 1e-3
    bad = d > tol
    msg = [f"bad={bad.float().mean().item():.4f} maxerr={d.max().item():.4g} refmax={ref.float().abs().max().item():.4g}"]
    if bad.any():
        rows = bad.any(1).nonzero().flatten()
        cols = bad.any(0).nonzero().flatten()
        msg.append(f"bad rows: n={rows.numel()} first={rows[:8].tolist()} last={rows[-4:].tolist()}")
        msg.append(f"bad cols: n={cols.numel()} first={cols[:8].tolist()} last={cols[-4:].tolist()}")
        msg.append(f"row%8 hist={torch.bincount(rows % 8, minlength=8).tolist()} "
                   f"row//32%4 hist={torch.bincount((rows // 32) % 4, minlength=4).tolist()}")
        msg.append(f"out[:2,:6]={out[:2, :6].float().tolist()} ref[:2,:6]={ref[:2, :6].float().tolist()}")
    return " | ".join(msg)


def _gemm_ref(a, w, bias, res, act):
    """Returns (reference, magnitude of the largest bf16 intermediate feeding each output)."""
    y = a.float() @ w.float().t()
    if bias is not None:
        y = y + bias.float()
    mag = y.abs()
    if act == vn.ACT_SWIGLU:
        g = y[:, 0::2].bfloat16().float()
        u = y[:, 1::2].bfloat16().float()
        out = torch.nn.functional.silu(g).bfloat16().float() * u
        return out, torch.maximum(out.abs(), (g.abs() + 1) * u.abs())
    if act == vn.ACT_QGELU:
        x = y.bfloat16().float()
        y = x * torch.sigmoid((1.702 * x).bfloat16().float()).bfloat16().float()
    elif act == vn.ACT_GELU:
        y = torch.nn.functional.gelu(y.bfloat16().float())
    if res is not None:
        y = y.bfloat16().float() + res.float()
    return y, torch.maximum(mag, y.abs())


GEMM_CASES = [
    # M, N, K, block_n, bias, res, act
    (128, 256, 64, 256, False, False, vn.ACT_NONE),
    (128, 256, 256, 256, False, False, vn.ACT_NONE),
    (128, 128, 512, 128, False, False, vn.ACT_NONE),
    (256, 512, 1024, 64, False, False, vn.ACT_NONE),
    (256, 512, 1024, 32, False, False, vn.ACT_NONE),
    (300, 1024, 1024, 256, True, False, vn.ACT_NONE),
    (300, 1024, 1024, 128, True, True, vn.ACT_NONE),
    (515, 4096, 1024, 0, True, False, vn.ACT_QGELU),
    (515, 1024, 4096, 0, True, True, vn.ACT_NONE),
    (448, 2048, 512, 0, False, False, vn.ACT_SWIGLU),
    (356, 512, 1024, 0, True, False, vn.ACT_GELU),
    (16, 12288, 4096, 0, False, False, vn.ACT_NONE),
    (25700, 3072, 1024, 256, True, False, vn.ACT_NONE),
    (25700, 1024, 4096, 256, True, True, vn.ACT_NONE),
    (448, 22016, 4096, 0, False, False, vn.ACT_SWIGLU),
]


@pytest.mark.parametrize("M,N,K,bn,has_bias,has_res,act", GEMM_CASES)
def test_gemm_tcgen05(M, N, K, bn, has_bias, has_res, act):
    torch.manual_seed(M * 7 + N * 3 + K + bn)
    dev = _dev()
    a = torch.randn(M, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=dev).bfloat16() if has_bias else None
    n_out = N // 2 if act == vn.ACT_SWIGLU else N
    res = torch.randn(M, n_out, device=dev).bfloat16() if has_res else None
    ref, mag = _gemm_ref(a, w, bias, res, act)
    out = res.clone() if has_res else None  # residual is updated in place on the hot path
    out = vn.op_gemm(a, w, bias, out if has_res else None, act, bn, out=out)
    torch.cuda.synchronize()
    rel = _rel(out, ref)
    # bf16 output: one rounding of an fp32 accumulation -> 2^-9 rms; allow 3e-3 norm-wise
    assert rel < 3e-3, f"rel={rel:.3e} " + _describe(out, ref)
    # element-wise: a couple of bf16 ulps of the largest intermediate (the reference rounds the
    # nn.Linear output to bf16 before the activation / residual, and so does the kernel)
    ulp = mag.clamp_min(1e-2) * 2 ** -7
    assert ((out.float() - ref).abs() <= 2.5 * ulp).all(), _describe(out, ref)


@pytest.mark.parametrize("rows,D", [(7, 1024), (25700, 1024), (448, 4096), (33, 5120)])
def test_layernorm_rmsnorm(rows, D):
    torch.manual_seed(rows + D)
    dev = _dev()
    x = (torch.randn(rows, D, device=dev) * 3 + 0.5).bfloat16()
    w = (1 + 0.1 * torch.randn(D, device=dev)).bfloat16()
    b = (0.1 * torch.randn(D, device=dev)).bfloat16()
    y = vn.op_layernorm(x, w, b, 1e-5)
    ref = torch.nn.functional.layer_norm(x.float(), (D,), w.float(), b.float(), 1e-5)
    assert _rel(y, ref) < 3e-3
    assert ((y.float() - ref).abs() <= ref.abs().clamp_min(1e-2) * 2 ** -7).all()
    y2 = vn.op_rmsnorm(x, w, 1e-5)
    xf = x.float()
    ref2 = w.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5)).bfloat16().float()
    assert _rel(y2, ref2) < 3e-3
    # same rounding order as LlamaRMSNorm: expect (nearly) bit-identical output
    frac = (y2 == ref2.bfloat16()).float().mean().item()
    assert frac > 0.999, frac


@pytest.mark.parametrize("rows,D", [(7, 1024), (25700, 1024), (300, 768)])
def test_layernorm_offset_and_outlier_rows(rows, D):
    """LayerNorm of rows on a large common offset and of rows with a few outlier channels (magnitude ~1000), as
    CLIP's residual stream carries them into layer_norm1 / 2: a one-pass variance E[x^2] - E[x]^2 loses them. At
    D = 1024 this is the warp-per-row kernel of the encoder's layer norms, at 768 the block kernel. Bar as for the
    CLIP pre-LN (_vit_ref.ln_check): 1 bf16 ulp of the fp64 value, at least 99 % bit-identical."""
    import _vit_ref as V
    g = torch.Generator(device=_dev()).manual_seed(rows + D)
    x = torch.randn(rows, D, device=_dev(), generator=g)
    r = torch.arange(rows, device=_dev())
    x[r % 4 == 0] = 700 + 8 * x[r % 4 == 0]
    x[r % 4 == 2] = 1000 + 3 * x[r % 4 == 2]
    ch = torch.randint(0, D, (rows, 4), device=_dev(), generator=g)
    odd = (r % 3 == 1).nonzero()[:, 0]
    x[odd[:, None], ch[odd]] = -1000 + 100 * torch.rand(len(odd), 4, device=_dev(), generator=g)
    x = x.bfloat16()
    w = (1 + 0.05 * torch.randn(D, device=_dev(), generator=g)).bfloat16()
    b = (0.02 * torch.randn(D, device=_dev(), generator=g)).bfloat16()
    y = vn.op_layernorm(x, w, b, 1e-5)
    torch.cuda.synchronize()
    V.ln_check(y, x, w, b, 1e-5, f"layernorm rows={rows} D={D}")


@pytest.mark.parametrize("B,S,H,hd,causal", [(3, 257, 16, 64, False), (2, 448, 4, 128, True),
                                             (1, 64, 2, 128, True), (5, 577, 2, 64, False),
                                             (1, 100, 3, 128, True),
                                             # causal hd 128 up to 512 keys: the wgmma prefill kernel (1..4 key blocks,
                                             # ragged last tile, a single head / clip); 640 keys: the mma.sync kernel
                                             (1, 512, 2, 128, True), (2, 129, 3, 128, True), (1, 300, 1, 128, True),
                                             (3, 448, 32, 128, True), (1, 640, 2, 128, True)])
def test_attention(B, S, H, hd, causal):
    torch.manual_seed(S + hd)
    dev = _dev()
    q, k, v = [torch.randn(B, S, H, hd, device=dev).bfloat16() for _ in range(3)]
    scale = hd ** -0.5
    o = vn.op_attention(q, k, v, scale, causal)
    qf, kf, vf = [t.float().permute(0, 2, 1, 3) for t in (q, k, v)]
    s = (qf @ kf.transpose(-1, -2)).bfloat16().float() * scale
    s = s.bfloat16().float()
    if causal:
        s = s.masked_fill(torch.ones(S, S, device=dev, dtype=torch.bool).triu(1), float("-inf"))
    p = torch.softmax(s, -1).bfloat16().float()
    ref = (p @ vf).permute(0, 2, 1, 3)
    rel = _rel(o, ref)
    assert rel < 6e-3, rel  # P is rounded un-normalised (flash form) vs normalised in eager


@pytest.mark.parametrize("B,S,H", [(1, 448, 32), (2, 77, 5), (3, 129, 3), (1, 511, 1), (2, 512, 4), (1, 16, 2)])
def test_attention_prefill_tcgen05_vs_mma_sync(B, S, H):
    """The wgmma prefill kernel against the flash-style mma.sync kernel, same inputs, one process
    (VCL_PREFILL_ATTN_FLASH is read per call): they differ only in where P is rounded (relative to the final row
    maximum vs the running one) and in summation order, so they agree far inside the tolerance either has against
    the eager reference."""
    import os
    torch.manual_seed(B * 1000 + S + H)
    dev = _dev()
    q, k, v = [torch.randn(B, S, H, 128, device=dev).bfloat16() for _ in range(3)]
    o_tc = vn.op_attention(q, k, v, 128 ** -0.5, True)
    os.environ["VCL_PREFILL_ATTN_FLASH"] = "1"
    try:
        o_mma = vn.op_attention(q, k, v, 128 ** -0.5, True)
    finally:
        del os.environ["VCL_PREFILL_ATTN_FLASH"]
    assert torch.isfinite(o_tc.float()).all()
    rel = _rel(o_tc, o_mma)
    per_row = (o_tc.float() - o_mma.float()).flatten(2).norm(dim=2) / o_mma.float().flatten(2).norm(dim=2)
    assert rel < 4e-3 and per_row.max().item() < 2e-2, (rel, per_row.max().item())
    assert not torch.equal(o_tc, o_mma) or S <= 16      # two different kernels did run


@pytest.mark.parametrize("B,N,K,norm,res", [(1, 4096, 4096, False, True), (1, 12288, 4096, True, False),
                                            (4, 4096, 11008, False, True), (3, 1000, 5120, True, True),
                                            (2, 32003, 4096, True, False), (16, 32003, 4096, False, False),
                                            (8, 1000, 5120, True, True)])
def test_gemv(B, N, K, norm, res):
    torch.manual_seed(N + K + B)
    dev = _dev()
    x = torch.randn(B, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    nw = (1 + 0.1 * torch.randn(K, device=dev)).bfloat16() if norm else None
    r = torch.randn(B, N, device=dev).bfloat16() if res else None
    out = vn.op_gemv(x, w, r, nw, 1e-5)
    xf = x.float()
    if norm:
        xf = (nw.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5)).bfloat16().float()).bfloat16().float()
    ref = (xf.double() @ w.double().t()).float()     # exact products: the reference does not depend on the GPU's BLAS
    mag = ref.abs()
    if res:
        ref = ref.bfloat16().float() + r.float()
    assert _rel(out, ref) < 3e-3, _rel(out, ref)
    # element-wise: as in test_gemm_tcgen05, a couple of bf16 ulps of the largest intermediate (the projection is
    # rounded to bf16 before the residual add; a sum on a rounding boundary may round either way)
    mag = torch.maximum(mag, ref.abs())
    assert ((out.float() - ref).abs() <= 2.5 * mag.clamp_min(1e-2) * 2 ** -7).all()


@pytest.mark.parametrize("T,P,C,dt_in,dt_out", [(100, 256, 1024, torch.bfloat16, torch.float16),
                                                (8, 256, 1024, torch.float16, torch.float16),
                                                (100, 576, 1024, torch.bfloat16, torch.bfloat16),
                                                (1, 4, 64, torch.float16, torch.bfloat16),
                                                (37, 256, 1024, torch.bfloat16, torch.float16)])
def test_st_pool(T, P, C, dt_in, dt_out):
    torch.manual_seed(T * P)
    dev = _dev()
    hid = torch.randn(T, P + 1, C, device=dev).to(dt_in)   # pooled in place behind the CLS row
    feats = hid[:, 1:]
    out = vn.st_pool(feats, 100, dt_out)
    f32 = feats.float()
    temporal = f32.mean(1).to(dt_in)
    spatial = f32.mean(0).to(dt_in)
    pad = torch.zeros(100 - T, C, device=dev)
    ref = torch.cat([temporal.float(), pad, spatial.float()], 0).to(dt_out)
    assert out.shape == (100 + P, C)
    assert (out[T:100] == 0).all()
    diff = (out.float() - ref.float()).abs()
    # fp32 accumulation order differs from torch's reduction tree: allow 1 ulp of the output type
    ulp = ref.float().abs().clamp_min(2 ** -14) * (2 ** -7 if torch.bfloat16 in (dt_in, dt_out) else 2 ** -10)
    assert (diff <= ulp).all(), diff.max().item()
    assert (out == ref).float().mean().item() > 0.98


@pytest.mark.parametrize("M,N,K,bn,cl,act", [(448, 1024, 512, 256, 2, vn.ACT_NONE), (448, 1024, 512, 256, 4, vn.ACT_NONE),
                                             (300, 512, 256, 128, 4, vn.ACT_NONE), (1000, 2048, 1024, 256, 2, vn.ACT_QGELU),
                                             (448, 22016, 4096, 256, 4, vn.ACT_SWIGLU), (25700, 3072, 1024, 256, 2, vn.ACT_NONE),
                                             (129, 256, 64, 128, 2, vn.ACT_NONE)])
def test_gemm_cluster_multicast(M, N, K, bn, cl, act):
    """TMA-multicast clusters along M (weight tile shared by 2 / 4 CTAs) give the same result."""
    torch.manual_seed(M + N + K + cl)
    dev = _dev()
    a = torch.randn(M, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=dev).bfloat16()
    ref, mag = _gemm_ref(a, w, bias, None, act)
    out = vn.op_gemm(a, w, bias, None, act, bn, cluster=cl)
    base = vn.op_gemm(a, w, bias, None, act, bn, cluster=1)
    torch.cuda.synchronize()
    assert _rel(out, ref) < 3e-3, _describe(out, ref)
    assert torch.equal(out, base), _describe(out, base.float())   # same tiles, same order: bit-identical


@pytest.mark.parametrize("M,N,K,bn,has_bias,has_res,act", [
    (256, 256, 64, 256, False, False, vn.ACT_NONE),
    (256, 512, 512, 256, True, False, vn.ACT_NONE),
    (300, 1024, 1024, 256, True, True, vn.ACT_NONE),
    (515, 4096, 1024, 256, True, False, vn.ACT_QGELU),
    (515, 1024, 4096, 128, True, True, vn.ACT_NONE),
    (448, 2048, 512, 128, False, False, vn.ACT_SWIGLU),
    (448, 12288, 4096, 128, False, False, vn.ACT_NONE),
    (25700, 3072, 1024, 256, True, False, vn.ACT_NONE),
    (25700, 1024, 4096, 256, True, True, vn.ACT_NONE),
])
def test_gemm_cta_pair(M, N, K, bn, has_bias, has_res, act):
    """cluster = -2, CTA pairs: two CTAs of a cluster share one 256-row tile, each fetching half of the weight
    tile. Same tiles and the same accumulation order as the single-CTA kernel -> bit-identical results."""
    torch.manual_seed(M + N + K + bn)
    dev = _dev()
    a = torch.randn(M, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=dev).bfloat16() if has_bias else None
    n_out = N // 2 if act == vn.ACT_SWIGLU else N
    res = torch.randn(M, n_out, device=dev).bfloat16() if has_res else None
    ref, mag = _gemm_ref(a, w, bias, res, act)
    out = vn.op_gemm(a, w, bias, res.clone() if has_res else None, act, bn, cluster=-2)
    base = vn.op_gemm(a, w, bias, res.clone() if has_res else None, act, bn, cluster=1)
    torch.cuda.synchronize()
    assert _rel(out, ref) < 3e-3, _describe(out, ref)
    assert torch.equal(out, base), _describe(out, base.float())
