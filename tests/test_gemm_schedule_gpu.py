"""The wgmma GEMM's tile schedule does not change its results.

The consumer warpgroups hand each staged output tile to the store warps and start the next tile at once, so a
persistent CTA that runs many tiles keeps one staging block per consumer warpgroup in flight across all of them.
At shapes where every CTA runs many tiles and the last M tile is ragged, every (block_n, cluster) the launcher
accepts must give the automatic choice's output bit for bit: each output element gets the same k16 wgmma
accumulations in the same K order whichever tile covers it. The automatic choice is checked against the fp32
reference with the tolerance of test_kernels_gpu.py."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
from test_kernels_gpu import _describe, _gemm_ref, _rel  # noqa: E402

TILES = [(bn, cl) for bn in (256, 128) for cl in (1, 2, 4, -2)] + [(64, 1), (32, 1)]

CASES = [
    # name, M, N, K, act, bias, residual (updated in place, C aliasing it, as on the hot path)
    ("vit_out", 25700, 1024, 1024, vn.ACT_NONE, True, True),
    ("vit_fc1", 25700, 4096, 1024, vn.ACT_QGELU, True, False),
    ("vit_gelu", 25700, 1024, 1024, vn.ACT_GELU, True, False),
    ("pre448_gu", 448, 22016, 4096, vn.ACT_SWIGLU, False, False),
    ("pre448_down", 448, 4096, 11008, vn.ACT_NONE, False, True),
    ("pre7168_gu", 7168, 22016, 4096, vn.ACT_SWIGLU, False, False),
    ("pre7168_o", 7168, 4096, 4096, vn.ACT_NONE, False, True),
]


@pytest.mark.parametrize("name,M,N,K,act,has_bias,has_res", CASES, ids=[c[0] for c in CASES])
def test_gemm_every_tile_matches_auto(name, M, N, K, act, has_bias, has_res):
    torch.manual_seed(M + N + K + act)
    dev = torch.device("cuda:0")
    a = torch.randn(M, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=dev).bfloat16() if has_bias else None
    n_out = N // 2 if act == vn.ACT_SWIGLU else N
    res = torch.randn(M, n_out, device=dev).bfloat16() if has_res else None

    def run(bn, cl):
        out = res.clone() if has_res else torch.full((M, n_out), float("nan"), device=dev, dtype=torch.bfloat16)
        return vn.op_gemm(a, w, bias, out if has_res else None, act, bn, out=out, cluster=cl)

    auto = run(0, 0)
    torch.cuda.synchronize()
    ref, mag = _gemm_ref(a, w, bias, res, act)
    assert _rel(auto, ref) < 3e-3, _describe(auto, ref)
    ulp = mag.clamp_min(1e-2) * 2 ** -7
    assert ((auto.float() - ref).abs() <= 2.5 * ulp).all(), _describe(auto, ref)
    del ref, mag
    for bn, cl in TILES:
        out = run(bn, cl)
        torch.cuda.synchronize()
        assert torch.equal(out, auto), f"block_n={bn} cluster={cl}: " + _describe(out, auto.float())
