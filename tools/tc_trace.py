"""Timeline of the per-matrix decode kernels (gemv_tc.cu) over one eager decode step (VCL_TC_TRACE)."""
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "video-llava_b200"))
os.environ["VCL_TC_TRACE"] = "1"
import bench  # noqa: E402
import vcl_native as vn  # noqa: E402

L = int(os.environ.get("PROF_LLM_LAYERS", "8"))
bench.MODELS["7b"]["layers"] = L
dev = torch.device("cuda:0")
c = vn.vcl_config()
c.clip_layers, c.clip_hidden, c.clip_inter, c.clip_heads = 1, 1024, 4096, 16
c.image_size, c.patch_size, c.clip_ln_eps = 224, 14, 1e-5
c.llm_layers, c.llm_hidden, c.llm_inter, c.llm_heads = L, 4096, 11008, 32
c.vocab, c.rms_eps, c.rope_theta = 32003, 1e-5, 10000.0
c.proj_type, c.n_temporal = vn.PROJ_LINEAR, 100
c.max_frames, c.max_batch, c.max_seq = 100, 1, 480
eng = vn.Engine(c)
_, llm_sd = bench.device_weights("7b", dev)
eng.load_llm(llm_sd)
del llm_sd
ids = torch.randint(3, 32000, (1, 448), device=dev); ids[:, 64] = 32001; ids[:, 65:421] = 32000; ids[:, 421] = 32002
vs = torch.full((1,), 64, dtype=torch.int32, device=dev)
feats = torch.randn(1, 356, 1024, device=dev).to(torch.bfloat16)
_, _, tok = eng.prefill(ids, feats, vs)
for i in range(6):
    _, tok = eng.decode_step(tok, 448 + i)
torch.cuda.synchronize()
path = os.path.join(ROOT, "gpurun_out", "tc_trace.bin")
lib = vn.lib()
lib.vcl_debug_tc_trace_dump.argtypes = [ctypes.c_char_p]
print("dump rc", lib.vcl_debug_tc_trace_dump(path.encode()))
raw = np.fromfile(path, dtype=np.uint64)
n_rec, G = int(raw[0]), int(raw[1])
t = raw[2:].reshape(-1, G, 8).astype(np.int64)     # [launch][CTA][8 stamps]
per_step = 4 * L + 1
recs = t[n_rec - per_step:n_rec]
names = {2: "qkv", 0: "res", 1: "swiglu", 3: "logits"}
# stamps: 0 kernel start, 1 dependency wait returned, 2 activation vector staged, 3 main loop done, 4 epilogue done,
#         5 / 6 producer first / last copy issued, 7 = (mode << 32) | N
print("step span us", (recs[-1][:, 4].max() - recs[0][:, 0].min()) / 1e3, "launches", per_step)
agg = {}
for k in range(4, per_step - 1):          # skip layer 0 and the head
    r = recs[k]
    mode = int(r[0, 7] >> 32); N = int(r[0, 7] & 0xffffffff)
    key = names.get(mode, str(mode)) + f"_N{N}"
    prev_end = recs[k - 1][:, 4].max()
    d = dict(gap=(r[:, 1].min() - prev_end) / 1e3, x_stage=(r[:, 2] - r[:, 1]).mean() / 1e3,
             stream=(r[:, 3] - r[:, 2]).mean() / 1e3, stream_max=(r[:, 3].max() - r[:, 2].min()) / 1e3,
             epi=(r[:, 4] - r[:, 3]).mean() / 1e3, total=(r[:, 4].max() - prev_end) / 1e3)
    agg.setdefault(key, []).append(d)
for key, ds in agg.items():
    print(key, {f: round(float(np.mean([d[f] for d in ds])), 2) for f in ds[0]})
