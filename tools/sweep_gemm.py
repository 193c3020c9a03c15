"""Sweep block_n x cluster of the wgmma GEMM on every GEMM shape bench.py runs (one GPU), with torch.matmul on the
same shape as a same-card yardstick. Epilogues as on the hot path: bias on the ViT / projector GEMMs, the residual
added in place (C aliasing it) on out / fc2 / o / down. `auto` is the launcher's own choice (block_n = 0).

    python tools/sweep_gemm.py [--json FILE]      (SWEEP_SHAPES=<prefix> filters, SWEEP_NOFLUSH=1 keeps L2 warm)
"""
import argparse, json, math, os, subprocess, sys
import torch
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "video-llava_b200"))
import vcl_native as vn
dev = torch.device("cuda:0")
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10, warm=3):
    for _ in range(warm): fn()
    ts = []
    for _ in range(iters):
        if not os.environ.get("SWEEP_NOFLUSH"): flush.zero_()      # operands come from HBM, as in the model
        s = torch.cuda.Event(enable_timing=True); e = torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record(); torch.cuda.synchronize(); ts.append(s.elapsed_time(e))
    ts.sort(); return ts[len(ts) // 2]


# name, M, N, K, act, bias, residual
SHAPES = [("vit_patch", 25600, 1024, 640, vn.ACT_NONE, False, False),
          ("vit_qkv", 25700, 3072, 1024, vn.ACT_NONE, True, False), ("vit_out", 25700, 1024, 1024, vn.ACT_NONE, True, True),
          ("vit_fc1", 25700, 4096, 1024, vn.ACT_QGELU, True, False), ("vit_fc2", 25700, 1024, 4096, vn.ACT_NONE, True, True),
          ("vit_out_nores", 25700, 1024, 1024, vn.ACT_NONE, True, False),    # what the residual costs the store warps
          ("vit_fc2_nores", 25700, 1024, 4096, vn.ACT_NONE, True, False),
          ("proj", 356, 4096, 1024, vn.ACT_NONE, True, False)]
for M in (448, 7168):   # config 2 (one clip, S_p = 448) and config 3 (16 clips); q|k|v runs ACT_ROPE, same tiles
    SHAPES += [(f"pre{M}_qkv", M, 12288, 4096, vn.ACT_NONE, False, False), (f"pre{M}_o", M, 4096, 4096, vn.ACT_NONE, False, True),
               (f"pre{M}_gu", M, 22016, 4096, vn.ACT_SWIGLU, False, False), (f"pre{M}_down", M, 4096, 11008, vn.ACT_NONE, False, True)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:   # the query is informational; the sweep still runs
        q = f"{torch.cuda.get_device_name(0)} (nvidia-smi: {ex})"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    only = os.environ.get("SWEEP_SHAPES")
    print("card:", card(), flush=True)
    rows = []
    for name, M, N, K, act, has_bias, has_res in SHAPES:
        if only and not name.startswith(only): continue
        torch.manual_seed(0)
        a = torch.randn(M, K, device=dev).bfloat16(); w = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
        bias = torch.randn(N, device=dev).bfloat16() if has_bias else None
        out = torch.randn(M, N // 2 if act == vn.ACT_SWIGLU else N, device=dev).bfloat16()
        res = out if has_res else None
        cfgs = [(0, 0)] + [(bn, cl) for bn in (256, 128, 64, 32) for cl in ((1, 2, 4) if bn >= 128 else (1,)) if N % bn == 0]
        us = {}
        for bn, cl in cfgs:
            us[f"bn{bn}/cl{cl}" if bn else "auto"] = 1e3 * timeit(lambda: vn.op_gemm(a, w, bias, res, act, bn, out=out, cluster=cl))
        us["torch"] = 1e3 * timeit(lambda: torch.matmul(a, w.t()))
        best = min((v, k) for k, v in us.items() if k not in ("auto", "torch"))
        fl = 2.0 * M * N * K
        print(f"{name} M={M} N={N} K={K}: " + " ".join(f"{k}:{v:.0f}" for k, v in us.items())
              + f" us | best {best[1]} {fl / best[0] / 1e6:.0f} TF/s, auto {fl / us['auto'] / 1e6:.0f} TF/s,"
              f" torch {fl / us['torch'] / 1e6:.0f} TF/s", flush=True)
        rows.append({"name": name, "M": M, "N": N, "K": K, "us": us})
        del a, w, out
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
