"""Kernel micro-benchmarks on one GPU (CUDA events, L2 flushed between timed launches).
Prints achieved TFLOP/s for the wgmma GEMM on the hot-path shapes and GB/s for the HBM-bound
kernels. Development tool, not the contract bench (bench.py)."""
import math
import os
import sys

import torch

os.environ.setdefault("VCL_OP_GEMV_CACHE", "1")   # keep the slot-ordered weight copy between timed calls

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "video-llava_b200"))
import vcl_native as vn  # noqa: E402

dev = torch.device("cuda:0")
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        s = torch.cuda.Event(enable_timing=True); e = torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record(); torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def gemm_case(M, N, K, bn, act=vn.ACT_NONE, bias=True, res=False):
    a = torch.randn(M, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    b = torch.randn(N, device=dev).bfloat16() if bias else None
    n_out = N // 2 if act == vn.ACT_SWIGLU else N
    out = torch.zeros(M, n_out, device=dev, dtype=torch.bfloat16)
    r = out if res else None
    ms = timeit(lambda: vn.op_gemm(a, w, b, r, act, bn, out=out))
    tf = 2.0 * M * N * K / ms / 1e9
    ms_t = timeit(lambda: torch.matmul(a, w.t()))
    print(f"gemm M={M} N={N} K={K} bn={bn} act={act} res={res}: {ms:.3f} ms {tf:.0f} TFLOP/s | torch {ms_t:.3f} ms {2.0*M*N*K/ms_t/1e9:.0f} TFLOP/s", flush=True)


def gemv_case(B, N, K, norm):
    if only == "gemv16" and B < 5:
        return
    x = torch.randn(B, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    nw = torch.ones(K, device=dev).bfloat16() if norm else None
    ms = timeit(lambda: vn.op_gemv(x, w, None, nw, 1e-5))
    print(f"gemv B={B} N={N} K={K} norm={norm}: {ms*1e3:.1f} us {N*K*2/ms/1e6:.0f} GB/s", flush=True)


def pool_case(T, P, C):
    hid = torch.randn(T, P + 1, C, device=dev).bfloat16()
    ms = timeit(lambda: vn.st_pool(hid[:, 1:], 100, torch.float16))
    print(f"st_pool T={T} P={P}: {ms*1e3:.1f} us {(T*P*C*2 + (100+P)*C*2)/ms/1e6:.0f} GB/s", flush=True)


only = sys.argv[1] if len(sys.argv) > 1 else "all"
if __name__ == "__main__":
    print(torch.cuda.get_device_name(0))
    for bn in ((256, 128) if only in ("all", "gemm") else ()):
        gemm_case(25700, 3072, 1024, bn)
        gemm_case(25700, 1024, 1024, bn, res=True)
        gemm_case(25700, 4096, 1024, bn, act=vn.ACT_QGELU)
        gemm_case(25700, 1024, 4096, bn, res=True)
    if only in ("all", "gemm"):
        gemm_case(8192, 8192, 8192, 256, bias=False)
        gemm_case(448, 12288, 4096, 0, bias=False)
        gemm_case(448, 22016, 4096, 0, act=vn.ACT_SWIGLU, bias=False)
        gemm_case(448, 4096, 11008, 0, bias=False, res=True)
        gemm_case(7168, 12288, 4096, 256, bias=False)
        gemm_case(16, 12288, 4096, 0, bias=False)
    gemv_case(1, 12288, 4096, True)
    gemv_case(1, 4096, 4096, False)
    gemv_case(1, 22016, 4096, True)
    gemv_case(1, 4096, 11008, False)
    gemv_case(4, 12288, 4096, True)
    gemv_case(1, 32003, 4096, True)
    if only in ("all", "gemv16"):
        for nb in (16, 8):
            gemv_case(nb, 12288, 4096, False)
            gemv_case(nb, 4096, 4096, False)
            gemv_case(nb, 22016, 4096, False)
            gemv_case(nb, 4096, 11008, False)
            gemv_case(nb, 32003, 4096, False)
    pool_case(100, 256, 1024)
    pool_case(100, 576, 1024)


def attn_case(n, S, H):
    """The ViT attention: the wgmma kernel and the mma.sync flash kernel (VCL_VIT_ATTN_FLASH, read per call)."""
    qkv = torch.randn(n * S, 3 * H * 64, device=dev).bfloat16()
    fl = n * H * 4.0 * S * S * 64
    outs = {}
    for name, flash in (("wgmma", False), ("flash mma.sync", True)):
        if flash:
            os.environ["VCL_VIT_ATTN_FLASH"] = "1"
        try:
            ms = timeit(lambda: vn.op_attention_vit(qkv, n, S, H))
            outs[name] = vn.op_attention_vit(qkv, n, S, H).float()
        finally:
            os.environ.pop("VCL_VIT_ATTN_FLASH", None)
        print(f"attn_vit {name} n={n} S={S} H={H}: {ms*1e3:.1f} us {fl/ms/1e9:.0f} TFLOP/s", flush=True)
    a, b = outs.values()
    print(f"attn_vit wgmma vs flash: rel {((a - b).norm() / b.norm()).item():.2e}", flush=True)


if __name__ == "__main__" and (len(sys.argv) < 2 or sys.argv[1] in ("all", "attn")):
    attn_case(100, 257, 16)
