"""Sweep block_n x cluster for the GEMM shapes of the hot path (one GPU)."""
import math, os, sys
import torch
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "video-llava_b200"))
import vcl_native as vn
dev = torch.device("cuda:0")
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
def timeit(fn, iters=8, warm=2):
    for _ in range(warm): fn()
    ts = []
    for _ in range(iters):
        if not os.environ.get("SWEEP_NOFLUSH"): flush.zero_()      # SWEEP_NOFLUSH=1: operands stay in L2 between runs
        s = torch.cuda.Event(enable_timing=True); e = torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record(); torch.cuda.synchronize(); ts.append(s.elapsed_time(e))
    ts.sort(); return ts[len(ts) // 2]
SHAPES = [("vit_qkv", 25700, 3072, 1024, vn.ACT_NONE), ("vit_out", 25700, 1024, 1024, vn.ACT_NONE),
          ("vit_fc1", 25700, 4096, 1024, vn.ACT_QGELU), ("vit_fc2", 25700, 1024, 4096, vn.ACT_NONE),
          ("pre_qkv", 448, 12288, 4096, vn.ACT_NONE), ("pre_o", 448, 4096, 4096, vn.ACT_NONE),
          ("pre_gu", 448, 22016, 4096, vn.ACT_SWIGLU), ("pre_down", 448, 4096, 11008, vn.ACT_NONE),
          ("pre16_qkv", 7168, 12288, 4096, vn.ACT_NONE)]
only = os.environ.get("SWEEP_SHAPES")        # name prefix filter, e.g. SWEEP_SHAPES=pre
for name, M, N, K, act in SHAPES:
    if only and not name.startswith(only): continue
    a = torch.randn(M, K, device=dev).bfloat16(); w = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    out = torch.zeros(M, N // 2 if act == vn.ACT_SWIGLU else N, device=dev, dtype=torch.bfloat16)
    res = []
    for bn in (256, 128, 64):
        for cl in ((1, 2, 4) if bn >= 128 else (1,)):
            if N % bn: continue
            ms = timeit(lambda: vn.op_gemm(a, w, None, None, act, bn, out=out, cluster=cl))
            res.append((ms, bn, cl))
    best = min(res)
    print(name, " ".join(f"bn{bn}/cl{cl}:{ms*1e3:.0f}us" for ms, bn, cl in res), f"| best bn{best[1]}/cl{best[2]} {2.0*M*N*K/best[0]/1e9:.0f} TF/s", flush=True)
