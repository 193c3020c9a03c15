"""Float64 references of the CLIP vision tower's own kernels, with the reference's rounding points:
  - im2col_ref      the patch gather (im2col_kernel, elementwise.cu): the patch embedding Conv2d (stride = kernel =
                    patch) as a GEMM over a [n P, KP] matrix whose pad columns are zero;
  - embed_ln_ref    CLS / patch row + position row (embed_sum_ref), then pre_layrnorm (clip_embed_ln_kernel, elementwise.cu):
                    transformers/models/clip/modeling_clip.py:138-218 and 677, the embeddings a bf16 tensor;
  - layernorm_ref   that LayerNorm in fp64; also the encoder's layer_norm1 / 2 (rownorm_warp_kernel at D = 1024);
  - attn_ref        the eager ViT attention over the fused q | k | v rows (attn_vit_tc_kernel, attention_tc.cu, and
                    attn_fwd_kernel<64, false>, attention.cu): modeling_clip.py:261-279 eager, as in
                    oracle.vcl_oracle.clip_hidden_states. The scores are bf16(bf16(q . k) * 0.125) with the q . k
                    products exact (fp64 sums of bf16 products), the softmax runs in fp32, p is rounded to bf16 and
                    p . v is accumulated in fp64;
  - mean_ref        the exact output of that attention when every score is equal (q = 0) and the values are one-hot
                    (counting_values): (keys of the frame in class d) / S.

Rows are the engine's: frame n's S tokens are rows n S .. n S + S - 1 of the activations, head h at columns
h * 64 .. h * 64 + 63."""
import torch

from _attn_ref import bf16_ulp  # noqa: F401  (the tests' ulp, one definition)

HD = 64
SCALE = HD ** -0.5               # 0.125, exact in fp32 and bf16


def im2col_ref(pixels, patch, KP):
    """pixels [n, 3, I, I] (any float dtype: the values are taken as given) -> [n (I / patch)^2, KP] fp64. Row
    n P + py G + px is patch (py, px) of frame n, column c patch^2 + i patch + j its pixel (c, py patch + i,
    px patch + j); columns 3 patch^2 .. KP - 1 are +0.0."""
    n, ch, image, _ = pixels.shape
    assert ch == 3 and image % patch == 0 and KP >= 3 * patch * patch
    G = image // patch
    x = pixels.double().reshape(n, 3, G, patch, G, patch).permute(0, 2, 4, 1, 3, 5).reshape(n * G * G, -1)
    out = torch.zeros(n * G * G, KP, dtype=torch.float64, device=pixels.device)
    out[:, :x.shape[1]] = x
    return out


def embed_sum_ref(patch_out, cls, pos, n_frames, round_sum=True):
    """patch_out [n P, D], cls [D], pos [P + 1, D] -> the embeddings [n (P + 1), D] fp64: row n (P + 1) + t is
    src + pos[t], src = cls for t = 0 and patch row n P + t - 1 otherwise. round_sum: rounded to bf16 (the embeddings
    tensor of a bf16 model)."""
    D = cls.shape[-1]
    P = pos.shape[0] - 1
    src = torch.cat([cls.double().reshape(1, 1, D).expand(n_frames, 1, D),
                     patch_out.double().reshape(n_frames, P, D)], 1)
    v = (src + pos.double()[None]).reshape(n_frames * (P + 1), D)
    return v.bfloat16().double() if round_sum else v


def embed_ln_ref(patch_out, cls, pos, w, b, n_frames, eps=1e-5, round_sum=True):
    """LayerNorm of embed_sum_ref's rows in fp64, not rounded [n (P + 1), D]"""
    return layernorm_ref(embed_sum_ref(patch_out, cls, pos, n_frames, round_sum), w, b, eps)


def layernorm_ref(x, w, b, eps=1e-5):
    """LayerNorm over the last dimension in fp64 (biased variance, as nn.LayerNorm), not rounded"""
    x = x.double()
    mean = x.mean(-1, keepdim=True)
    var = (x - mean).pow(2).mean(-1, keepdim=True)
    return (x - mean) / torch.sqrt(var + eps) * w.double() + b.double()


def split_qkv(qkv, n, S, H):
    """the fused rows [>= n S, 3 H 64] -> q, k, v [n, H, S, 64] fp64"""
    C = H * HD
    x = qkv[:n * S].double()
    return [x[:, i * C:(i + 1) * C].reshape(n, S, H, HD).permute(0, 2, 1, 3) for i in range(3)]


def attn_ref(qkv, n, S, H, frames_per_step=8):
    """qkv [>= n S, 3 H 64] bf16 -> o [n S, H, 64] fp64 with the rounding points above (frames in groups, so that a
    hundred frames of 257 tokens fit)"""
    out = torch.empty(n * S, H, HD, dtype=torch.float64, device=qkv.device)
    sc = torch.tensor(SCALE, dtype=torch.float32)
    for f0 in range(0, n, frames_per_step):
        f1 = min(n, f0 + frames_per_step)
        q, k, v = split_qkv(qkv[f0 * S:f1 * S], f1 - f0, S, H)
        s = (q @ k.transpose(-1, -2)).bfloat16().float()                        # exact q . k, one rounding
        s = (s * sc).bfloat16().float()
        p = torch.softmax(s, -1).bfloat16().double()
        out[f0 * S:f1 * S] = (p @ v).permute(0, 2, 1, 3).reshape(-1, H, HD)
    return out


def counting_values(n, S, H, device="cpu"):
    """v [n S, H 64] bf16 for the counting input: key j (token j of its frame) of head h is one-hot at
    d = (7 j + 3 h) % 64, of value 1. With q = 0 every key of the frame weighs exactly 1 / S."""
    j = torch.arange(S)
    h = torch.arange(H)
    d = (7 * j[:, None] + 3 * h[None, :]) % HD                                  # [S, H]
    v = torch.zeros(S, H, HD)
    v.scatter_(2, d[:, :, None], 1.0)
    return v.reshape(1, S, H * HD).expand(n, S, H * HD).reshape(n * S, H * HD).to(device=device, dtype=torch.bfloat16)


def mean_ref(v, n, S, H):
    """the exact mean of each frame's values, v [>= n S, H 64] -> [n S, H, 64] fp64: the output of the attention when
    all scores are equal (q = 0), up to the final bf16 rounding"""
    m = v[:n * S].double().reshape(n, S, H, HD).mean(1, keepdim=True)
    return m.expand(n, S, H, HD).reshape(n * S, H, HD)



# The LayerNorm bar: 1 bf16 ulp of the fp64 value, where the ulp is taken at |value| >= a floor of the row. A correct
# fp32 kernel errs in two places a bf16 rounding does not cover:
#   - x_hat * w + b where the two terms cancel: ~1e-8 absolute, more than 1 ulp of a result below ~2^-17. LN_FLOOR
#     = 2^-12 leaves a margin of ~100 and is still 1 ulp for 99.98 % of N(0, 1) outputs.
#   - the fp32 mean of a row on a large common offset: its rounding (~2^-24 |mean|) moves every x_hat by ~2^-24 |mean|
#     / std. On rows of 500 + N(0, 64) at D = 768 (mean / 768 is not exact) that was measured at up to 1.8 ulp of
#     results near 3e-4; at D = 1024 (exact division) 0.5 ulp. The floor of such a row is 2^-13 |w| |mean| / std,
#     which covers four times that error, and is still far below the 2^-8 relative error a one-pass variance
#     E[x^2] - E[x]^2 makes on a row of 1000 + N(0, 9).
LN_FLOOR = 2.0 ** -12


def ln_check(got, x, w, b, eps, what, min_identical=0.99):
    """got [rows, D] bf16 against layernorm_ref(x, w, b, eps): every element within 1 bf16 ulp (at the floors above),
    and at least min_identical of them equal to the bf16 of the fp64 value. Prints the fraction and the worst error
    in ulps; returns the fraction."""
    ref = layernorm_ref(x, w, b, eps)
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    std = (xd - mean).pow(2).mean(-1, keepdim=True).add(eps).sqrt()
    floor = torch.maximum(torch.full_like(ref, LN_FLOOR), 2.0 ** -13 * w.double().abs() * mean.abs() / std)
    g = got.double()
    err = (g - ref).abs() / bf16_ulp(torch.maximum(ref.abs(), floor))
    bad = ~(err <= 1)                                        # NaN (an unwritten sentinel) counts as bad
    same = (got.view(torch.int16) == ref.bfloat16().view(torch.int16)).double().mean().item()
    print(f"[layernorm] {what}: bit-identical {same:.6f}, worst {err.nan_to_num(float('inf')).max().item():.3f} ulp")
    assert not bad.any(), (f"{what}: {int(bad.sum())} elements off by more than 1 bf16 ulp, first (row, col) "
                           f"{bad.nonzero()[:4].tolist()}: got {g[bad][:4].tolist()} want {ref[bad][:4].tolist()}")
    assert same >= min_identical, (what, same)
    return same
