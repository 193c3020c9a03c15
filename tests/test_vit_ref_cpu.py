"""The float64 references of tests/_vit_ref.py on the CPU: the patch gather against the patch embedding Conv2d, the
embedding + pre-LN against the oracle's hidden_states[0], the attention against the oracle's eager bf16 form, and the
counting input against its closed form."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _vit_ref as V
from oracle import vcl_oracle as O


def _kp(patch):
    """the engine's padded im2col width (vcl_create: 3 patch^2 up to a multiple of 64)"""
    return (3 * patch * patch + 63) // 64 * 64


@pytest.mark.parametrize("image,n", [(224, 2), (336, 1)])
def test_im2col_times_weight_is_the_patch_conv(image, n):
    """im2col_ref(x) W_pad^T (W zero-padded to KP columns, as vcl_load_clip_weights lays it out) equals
    Conv2d(x, W, stride = patch), the patch embedding, in fp64; the pad columns are +0.0"""
    g = torch.Generator().manual_seed(image + n)
    patch, C = 14, 16
    x = torch.randn(n, 3, image, image, generator=g, dtype=torch.float64)
    w = torch.randn(C, 3, patch, patch, generator=g, dtype=torch.float64)
    KP = _kp(patch)
    cols = V.im2col_ref(x, patch, KP)
    P = (image // patch) ** 2
    assert cols.shape == (n * P, KP)
    pad = cols[:, 3 * patch * patch:]
    assert torch.equal(pad, torch.zeros_like(pad)) and not torch.signbit(pad).any()
    w_pad = torch.zeros(C, KP, dtype=torch.float64)
    w_pad[:, :3 * patch * patch] = w.reshape(C, -1)
    want = F.conv2d(x, w, stride=patch).flatten(2).transpose(1, 2).reshape(n * P, C)
    torch.testing.assert_close(cols @ w_pad.t(), want, rtol=1e-12, atol=1e-12)


def test_im2col_row_and_column_order():
    """element (row n P + py G + px, column c patch^2 + i patch + j) is pixel (n, c, py patch + i, px patch + j)"""
    n, image, patch = 2, 42, 14
    x = torch.arange(n * 3 * image * image, dtype=torch.float64).reshape(n, 3, image, image)
    cols = V.im2col_ref(x, patch, _kp(patch))
    G = image // patch
    for (f, py, px, c, i, j) in [(0, 0, 0, 0, 0, 0), (1, 2, 1, 2, 13, 5), (0, 1, 2, 1, 7, 13), (1, 0, 2, 0, 3, 0)]:
        assert cols[f * G * G + py * G + px, c * patch * patch + i * patch + j] == x[f, c, py * patch + i, px * patch + j]


@pytest.mark.parametrize("image", [224, 336])
def test_embed_ln_ref_is_the_oracles_first_hidden_state(image):
    """with the embedding sum left unrounded, embed_ln_ref of the patch GEMM equals O.clip_hidden_states(...)[0], the
    post-pre_layrnorm embeddings, in fp64"""
    cfg = O.ClipCfg(hidden=64, inter=64, heads=1, layers=1, image=image)
    sd = O.random_clip_state(cfg, seed=3, dtype=torch.float64, n_layers=0)
    frames = O.make_frames(2, 2, size=image)
    px = O.preprocess_frames(frames).double()
    want = O.clip_hidden_states(sd, cfg, px, 0)[0]
    p = "vision_model."
    KP = _kp(cfg.patch)
    w_pad = torch.zeros(cfg.hidden, KP, dtype=torch.float64)
    w_pad[:, :3 * cfg.patch ** 2] = sd[p + "embeddings.patch_embedding.weight"].reshape(cfg.hidden, -1)
    patch_out = V.im2col_ref(px, cfg.patch, KP) @ w_pad.t()
    got = V.embed_ln_ref(patch_out, sd[p + "embeddings.class_embedding"], sd[p + "embeddings.position_embedding.weight"],
                         sd[p + "pre_layrnorm.weight"], sd[p + "pre_layrnorm.bias"], 2, cfg.eps, round_sum=False)
    torch.testing.assert_close(got, want.reshape(got.shape), rtol=1e-10, atol=1e-10)


def test_embed_ln_ref_rounds_the_sum_to_bf16():
    """round_sum: the LayerNorm sees bf16(src + pos), the embeddings tensor of a bf16 model"""
    g = torch.Generator().manual_seed(4)
    D, P = 32, 4
    po, cls, pos = (torch.randn(s, generator=g, dtype=torch.float64).bfloat16() for s in ((P, D), (D,), (P + 1, D)))
    w, b = torch.ones(D), torch.zeros(D)
    got = V.embed_ln_ref(po, cls, pos, w, b, 1, 1e-5)
    v = torch.cat([cls[None], po]).double() + pos.double()
    want = F.layer_norm(v.bfloat16().double(), (D,), eps=1e-5)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


def _eager_bf16(qkv, n, S, H):
    """the oracle's eager attention (clip_hidden_states, modeling_clip.py:261-279) on bf16 tensors"""
    q, k, v = [t.bfloat16() for t in V.split_qkv(qkv, n, S, H)]
    w = torch.matmul(q, k.transpose(-1, -2)) * V.SCALE
    w = F.softmax(w, dim=-1, dtype=torch.float32).to(q.dtype)
    return torch.matmul(w, v).permute(0, 2, 1, 3).reshape(n * S, H, V.HD)


@pytest.mark.parametrize("n,S,H", [(2, 17, 2), (1, 65, 3), (3, 130, 1)])
def test_attn_ref_agrees_with_the_eager_bf16_attention(n, S, H):
    g = torch.Generator().manual_seed(n * S + H)
    qkv = torch.randn(n * S, 3 * H * V.HD, generator=g).bfloat16()
    ref = V.attn_ref(qkv, n, S, H)
    eager = _eager_bf16(qkv, n, S, H).double()
    rel = ((eager - ref).norm() / ref.norm()).item()
    assert rel < 4e-3, rel
    per = (eager - ref).norm(dim=-1) / ref.norm(dim=-1)
    assert per.max().item() < 1.5e-2, per.max().item()


def test_attn_ref_matches_a_direct_evaluation():
    """attn_ref against a row-by-row evaluation of the same rounding points; frames do not see each other's keys"""
    g = torch.Generator().manual_seed(8)
    n, S, H = 3, 11, 2
    qkv = (torch.randn(n * S, 3 * H * V.HD, generator=g) * 2).bfloat16()
    got = V.attn_ref(qkv, n, S, H, frames_per_step=2)
    C = H * V.HD
    sc = torch.tensor(V.SCALE, dtype=torch.float32)
    for f in range(n):
        rows = slice(f * S, (f + 1) * S)
        for h in range(H):
            k = qkv[rows, C + h * V.HD:C + (h + 1) * V.HD].double()
            v = qkv[rows, 2 * C + h * V.HD:2 * C + (h + 1) * V.HD].double()
            for t in range(S):
                q = qkv[f * S + t, h * V.HD:(h + 1) * V.HD].double()
                s = torch.stack([(q * k[j]).sum() for j in range(S)]).bfloat16().float()
                p = torch.softmax((s * sc).bfloat16().float(), 0).bfloat16().double()
                want = (p[:, None] * v).sum(0)
                assert torch.allclose(got[f * S + t, h], want, rtol=0, atol=1e-12), (f, h, t)


@pytest.mark.parametrize("n,S,H", [(2, 257, 2), (1, 65, 16), (3, 1, 1)])
def test_counting_input_closed_form(n, S, H):
    """q = 0 and one-hot values: every score is 0, so attn_ref's p is bf16(1 / S) and its output is that times the
    count of the frame's keys in class d; mean_ref is the exact count / S. Both against a count taken key by key."""
    v = V.counting_values(n, S, H)
    count = np.zeros((H, V.HD))
    for j in range(S):
        for h in range(H):
            count[h, (7 * j + 3 * h) % V.HD] += 1
    want = torch.tensor(count, dtype=torch.float64)[None].expand(n * S, H, V.HD)
    assert torch.equal(V.mean_ref(v, n, S, H), want / S)
    k = torch.randn(n * S, H * V.HD, generator=torch.Generator().manual_seed(S)).bfloat16()
    qkv = torch.cat([torch.zeros(n * S, H * V.HD, dtype=torch.bfloat16), k, v], 1)
    p = torch.tensor(1.0 / S, dtype=torch.float32).bfloat16().double()
    assert torch.equal(V.attn_ref(qkv, n, S, H), want * p)
