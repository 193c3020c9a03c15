"""The vision tower's own kernels, one launch at a time, against the float64 references of tests/_vit_ref.py:
  - im2col_kernel (vcl_op_im2col): both pixel formats, 224 and 336 px, 1 / 8 / 100 frames. Bar: bit-identical,
    pad columns +0.0. The uint8 frames hold every value 0..255 in every channel, so every (value, channel) pair of
    the CLIP normalisation is checked; the kernel's fp32 (x * (1 / 255) - mean) / std rounds to the bf16 of the
    oracle's preprocess_frames for all 768 of them, with or without a contracted multiply-add.
  - clip_embed_ln_kernel (vcl_op_clip_embed_ln): P 256 / 576, 1 / 100 frames, D 1024 / 768, with rows on a large
    common offset and outlier channels of magnitude ~1000. Bar: _vit_ref.ln_check (1 bf16 ulp, >= 99 % identical).
  - the ViT attention (vcl_op_attention_vit): attn_vit_tc_kernel (wgmma, 129 <= S <= 257) and attn_fwd_kernel<64,
    false> (mma.sync, flash form, every other S and, under VCL_VIT_ATTN_FLASH=1, read per call, those too).
  - the engine's front end: vcl_clip_encode at 0 layers is these two kernels around the patch GEMM, bit for bit.

Attention input kinds:
  - count: q = 0, so every score is exactly 0 and each key of the frame weighs 1 / S; v[j] is one-hot at
    (7 j + 3 h) % 64. Output element d is (the frame's keys in class d) / S, which both kernels compute exactly up
    to the final bf16 rounding: bar 1 bf16 ulp. One key too many moves an element by about 1 / S of itself.
  - random: q, k, v ~ N(0, 1).
  - peaked: q * 4, so about ten keys carry a row.
  - spike: query t is 3 k[j] for j one of the keys 0, 63, 64, 255, 256 (the N32 tail block at S = 257) and S - 1
    that S has, so key j scores far above the rest of the row.
  - rising: q and the keys follow a direction of the (frame, head) more and more along the frame, so the row
    maximum grows on every 64-key tile (the mma.sync kernel rescales on every tile).
  - border (two frames or more): the first 64 keys of frame f + 1 follow frame f's queries, ~15 above the scores of
    frame f's own keys, so a key read past S - 1 takes over the row.
  Bars of the last five: relative L2 error per (row, head) < 1e-2 and over the whole output < 4e-3 (the prefill
  attention bars of test_prefill_attention_gpu.py).

Poisoning: the q | k | v rows are a view into a buffer whose rows before and after the launch are NaN, and the output
is a view into a buffer of a NaN sentinel with margin rows: every row must be written and finite, and the margins
must keep the sentinel."""
import contextlib
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
import _vit_ref as V  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import make_engine, to_dev  # noqa: E402

DEV = "cuda"
SENTINEL = 0x7FC1          # a bf16 NaN bit pattern no kernel produces
NAN = float("nan")
MARGIN = 3                 # sentinel rows before and after an output
PATCH = 14
KP = 640                   # the engine's im2col width at patch 14: 3 * 14 * 14 = 588 up to a multiple of 64


def _sentinel(rows, cols):
    return torch.full((rows, cols), SENTINEL, dtype=torch.int16, device=DEV).view(torch.bfloat16)


def _framed(rows, cols):
    """(buffer, view): `rows` rows of a sentinel buffer with MARGIN sentinel rows on each side"""
    buf = _sentinel(rows + 2 * MARGIN, cols)
    return buf, buf[MARGIN:MARGIN + rows]


def _margins_kept(buf, what):
    bits = buf.view(torch.int16)
    assert (bits[:MARGIN] == SENTINEL).all() and (bits[-MARGIN:] == SENTINEL).all(), f"{what}: wrote past its rows"


def _launches(fn, want=1):
    n0 = vn.launch_count()
    out = fn()
    torch.cuda.synchronize()
    assert vn.launch_count() - n0 == want, f"{vn.launch_count() - n0} launches, expected {want}"
    return out


# ------------------------------------------------------------------------------------------
# im2col
def _frames_u8(n, image):
    """[n, image, image, 3] uint8: pixel (y, x) of channel c in frame f is (y image + x + 85 c + 7 f) % 256, so every
    frame holds every value in every channel"""
    y = torch.arange(image)[:, None]
    x = torch.arange(image)[None, :]
    c = torch.arange(3)
    f = torch.arange(n)
    v = ((y * image + x)[None, :, :, None] + 85 * c + 7 * f[:, None, None, None]) % 256
    return v.to(torch.uint8).numpy()


@torch.no_grad()
@pytest.mark.parametrize("n", [1, 8, 100])
@pytest.mark.parametrize("image", [224, 336])
@pytest.mark.parametrize("fmt", [vn.PIXELS_BF16_NCHW, vn.PIXELS_U8_NHWC])
def test_im2col(fmt, image, n):
    P = (image // PATCH) ** 2
    if fmt == vn.PIXELS_U8_NHWC:
        frames = _frames_u8(n, image)
        pixels = torch.as_tensor(frames).to(DEV)
        values = O.preprocess_frames(frames).bfloat16().to(DEV)         # the oracle's normalisation, rounded
    else:
        g = torch.Generator(device=DEV).manual_seed(image + n)
        pixels = (2 * torch.randn(n, 3, image, image, device=DEV, generator=g)).bfloat16()
        pixels[:, :, ::7, ::5] = -0.0                                  # the sign of a zero must survive the copy
        values = pixels
    want = V.im2col_ref(values, PATCH, KP).bfloat16().view(torch.int16)
    buf, out = _framed(n * P, KP)
    _launches(lambda: vn.op_im2col(pixels, fmt, KP, PATCH, out=out))
    _margins_kept(buf, "im2col")
    got = out.view(torch.int16)
    pad = got[:, 3 * PATCH * PATCH:]
    assert (pad == 0).all(), f"pad columns not +0.0 in {int((pad != 0).any(1).sum())} rows"
    bad = got != want
    assert not bad.any(), (f"{int(bad.sum())} elements differ, first (row, col) {bad.nonzero()[:4].tolist()}: got "
                           f"{out[bad][:4].tolist()} want {want.view(torch.bfloat16)[bad][:4].tolist()}")


@torch.no_grad()
def test_im2col_rejects():
    px = torch.zeros(1, 3, 224, 224, dtype=torch.bfloat16, device=DEV)
    n0 = vn.launch_count()
    with pytest.raises(vn.VclError, match="bad geometry"):
        vn.op_im2col(px, vn.PIXELS_BF16_NCHW, 584)                      # KP below 3 * 14 * 14
    with pytest.raises(vn.VclError, match="mode must be"):
        vn.op_im2col(px, 2, KP)
    out = torch.zeros(256, KP, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(vn.VclError, match="patch=0"):
        vn.check(vn.lib().vcl_op_im2col(vn.ptr(px), vn.PIXELS_BF16_NCHW, vn.ptr(out), 1, 224, 0, KP, vn.cur_stream()))
    assert vn.launch_count() == n0


# ------------------------------------------------------------------------------------------
# CLIP embedding + pre-LN
def _embed_inputs(n, P, D, seed):
    """patch rows ~ N(0, 1), every fifth 500 + N(0, 64) and every seventh 1000 + N(0, 9) (a large common offset: the
    latter breaks a one-pass variance), every third with three outlier
    channels of magnitude ~1000, a CLS row with two outliers, position rows
    ~ N(0, 0.5) (one row off moves every element by many ulps), LayerNorm weight ~ 1 + N(0, 0.05) and bias
    ~ N(0, 0.02) as in random_clip_state"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    po = torch.randn(n * P, D, device=DEV, generator=g)
    r = torch.arange(n * P, device=DEV)
    po[r % 5 == 1] = 500 + 8 * po[r % 5 == 1]
    po[r % 7 == 2] = 1000 + 3 * po[r % 7 == 2]
    out_ch = torch.randint(0, D, (n * P, 3), device=DEV, generator=g)
    sign = torch.randint(0, 2, (n * P, 3), device=DEV, generator=g) * 2 - 1
    rows = (r % 3 == 0).nonzero()[:, 0]
    po[rows[:, None], out_ch[rows]] = (1000 + 50 * torch.rand(len(rows), 3, device=DEV, generator=g)) * sign[rows]
    cls = torch.randn(D, device=DEV, generator=g)
    cls[:2] = torch.tensor([900.0, -1100.0])
    pos = 0.5 * torch.randn(P + 1, D, device=DEV, generator=g)
    w = 1 + 0.05 * torch.randn(D, device=DEV, generator=g)
    b = 0.02 * torch.randn(D, device=DEV, generator=g)
    return [t.bfloat16() for t in (po, cls, pos, w, b)]


@torch.no_grad()
@pytest.mark.parametrize("D", [1024, 768])
@pytest.mark.parametrize("n", [1, 100])
@pytest.mark.parametrize("P", [256, 576])
def test_clip_embed_ln(P, n, D):
    po, cls, pos, w, b = _embed_inputs(n, P, D, seed=P + n + D)
    buf, out = _framed(n * (P + 1), D)
    _launches(lambda: vn.op_clip_embed_ln(po, cls, pos, w, b, n, 1e-5, out=out))
    _margins_kept(buf, "clip_embed_ln")
    V.ln_check(out, V.embed_sum_ref(po, cls, pos, n), w, b, 1e-5, f"clip_embed_ln P={P} n={n} D={D}")


# ------------------------------------------------------------------------------------------
# ViT attention
@contextlib.contextmanager
def _flash_env(on):
    """VCL_VIT_ATTN_FLASH=1 (read per call): the mma.sync kernel at every S"""
    if not on:
        yield
        return
    os.environ["VCL_VIT_ATTN_FLASH"] = "1"
    try:
        yield
    finally:
        del os.environ["VCL_VIT_ATTN_FLASH"]


def _spike_keys(S):
    return sorted({j for j in (0, 63, 64, 255, 256, S - 1) if j < S})


def _attn_inputs(kind, n, S, H, seed):
    """q | k | v rows [n S, 3 H 64] bf16, a view into a buffer with MARGIN NaN rows before and 64 after"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    q, k, v = (torch.randn(n, S, H, V.HD, device=DEV, generator=g) for _ in range(3))
    if kind == "count":
        q.zero_()
        v = V.counting_values(n, S, H, device=DEV).float().view(n, S, H, V.HD)
    elif kind == "peaked":
        q *= 4
    elif kind == "spike":
        j = torch.tensor([_spike_keys(S)[t % len(_spike_keys(S))] for t in range(S)], device=DEV)
        q = 3 * k[:, j]
    elif kind in ("rising", "border"):
        u = torch.randn(n, 1, H, V.HD, device=DEV, generator=g)
        u = u / u.norm(dim=-1, keepdim=True)
        if kind == "rising":
            # score_j ~ j / 128 (0.5 more per 64 keys) + noise of ~0.3
            q = 8 * (u + 0.1 * q)
            beta = torch.arange(S, device=DEV, dtype=torch.float32) / 128
            k = beta[None, :, None, None] * u + 0.3 * k
        else:
            # frame f's queries score ~15 on the first 64 keys of frame f + 1 and O(1) on their own
            q = 0.5 * q + 3 * u
            k[1:, :64] = 40 * u[:-1] + 0.3 * k[1:, :64]
    # q and k on a grid of 1/8: every q . k is exact in fp32 whatever the summation order, so the kernels' bf16
    # scores are the reference's bit for bit. A real-valued q . k within fp32 rounding of a bf16 tie may round the
    # other way, which moves that key's weight by 2^-8 of its score (1.6 % at a score of 4) and its row by ~1e-2
    # (measured before the grid: up to 1.04e-2 per row on random inputs, 3.6e-2 on peaked ones).
    q, k = torch.round(q * 8) / 8, torch.round(k * 8) / 8
    rows = n * S
    buf = torch.full((MARGIN + rows + 64, 3 * H * V.HD), NAN, device=DEV, dtype=torch.bfloat16)
    qkv = buf[MARGIN:MARGIN + rows]
    qkv.copy_(torch.cat([t.reshape(rows, H * V.HD) for t in (q, k, v)], 1))
    return qkv


def _attend(qkv, n, S, H, flash):
    buf, out = _framed(n * S, H * V.HD)
    with _flash_env(flash):
        _launches(lambda: vn.op_attention_vit(qkv, n, S, H, out=out))
    _margins_kept(buf, "attention_vit")
    return out


def _check(o, qkv, n, S, H, kind, what):
    assert torch.isfinite(o.float()).all(), f"{what} [{kind}]: a row is unwritten (sentinel) or not finite"
    got = o.view(-1, H, V.HD).double()
    if kind == "count":
        want = V.mean_ref(qkv[:, 2 * H * V.HD:], n, S, H)
        bad = (got - want).abs() > V.bf16_ulp(want)
        assert not bad.any(), (f"{what} [count]: {int(bad.sum())} elements off by more than 1 bf16 ulp, first (row, "
                               f"head, d) {bad.nonzero()[:4].tolist()}: got {got[bad][:4].tolist()} want "
                               f"{want[bad][:4].tolist()}")
        return
    ref = V.attn_ref(qkv, n, S, H)
    per = (got - ref).norm(dim=-1) / ref.norm(dim=-1).clamp_min(1e-30)
    tot = ((got - ref).norm() / ref.norm()).item()
    worst = divmod(per.argmax().item(), H)
    print(f"[vit-attn] {what} [{kind}]: max per-(row, head) {per.max().item():.3e} at (row, head) {worst} "
          f"(token {worst[0] % S}), total {tot:.3e}")
    assert per.max().item() < 1e-2 and tot < 4e-3, (what, kind, per.max().item(), worst, tot)


def _case(n, S, H):
    """every kind on the kernel the engine takes; at 129 <= S <= 257 also on the mma.sync kernel, which must give a
    different random output (two kernels ran: it rounds P against the running maximum of each 64-key tile, the
    wgmma kernel against the row's final one)"""
    kinds = ("count", "random", "peaked", "spike", "rising") + (("border",) if n >= 2 else ())
    both = 129 <= S <= 257
    random_out = {}
    for i, kind in enumerate(kinds):
        qkv = _attn_inputs(kind, n, S, H, seed=1000 * n + 10 * S + H + i)
        for flash in ((False, True) if both else (False,)):
            o = _attend(qkv, n, S, H, flash)
            _check(o, qkv, n, S, H, kind, f"n={n} S={S} H={H} {'mma.sync' if flash or not both else 'wgmma'}")
            if kind == "random":
                random_out[flash] = o
    if both:
        assert not torch.equal(random_out[False], random_out[True]), "the wgmma and mma.sync runs are bit-identical"


S_CASES = [1, 2, 63, 64, 65, 128, 129, 192, 255, 256, 257, 258, 320, 577]


@torch.no_grad()
@pytest.mark.parametrize("H", [1, 2, 16])
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("S", S_CASES)
def test_attention_vit(S, n, H):
    _case(n, S, H)


@torch.no_grad()
@pytest.mark.parametrize("n,S,H", [(3, 257, 16), (2, 257, 2), (4, 200, 3), (2, 129, 1), (2, 256, 2),
                                   (100, 257, 16)])     # the last: bench config 5's 100 frames of 224 px
def test_attention_vit_engine_shapes(n, S, H):
    _case(n, S, H)


# ------------------------------------------------------------------------------------------
# the engine's front end
@torch.no_grad()
@pytest.mark.parametrize("image,n", [(224, 3), (336, 2)])
@pytest.mark.parametrize("fmt", [vn.PIXELS_BF16_NCHW, vn.PIXELS_U8_NHWC])
def test_clip_encode_front_end_is_these_kernels(fmt, image, n):
    """vcl_clip_encode at n_layers = 0 equals op_im2col -> op_gemm (the engine's automatic tile) -> op_clip_embed_ln
    bit for bit, the patch weight zero-padded to KP columns as vcl_load_clip_weights lays it out"""
    cfg = O.ClipCfg(hidden=1024, inter=1024, heads=16, layers=2, image=image)
    sd = to_dev(O.random_clip_state(cfg, seed=image + n))
    eng = make_engine(clip=cfg, clip_run_layers=1, max_frames=n)
    eng.load_clip(sd)
    frames = O.make_frames(5, n, size=image)
    pixels = (O.preprocess_frames(frames).bfloat16() if fmt == vn.PIXELS_BF16_NCHW else torch.as_tensor(frames)).to(DEV)
    got = eng.clip_encode(pixels, n_layers=0)
    p = "vision_model."
    C = cfg.hidden
    w_pad = torch.zeros(C, KP, dtype=torch.bfloat16, device=DEV)
    w_pad[:, :3 * PATCH * PATCH] = sd[p + "embeddings.patch_embedding.weight"].reshape(C, -1)
    cols = vn.op_im2col(pixels, fmt, KP)
    patch_out = vn.op_gemm(cols, w_pad, None, None, vn.ACT_NONE, 0)
    want = vn.op_clip_embed_ln(patch_out, sd[p + "embeddings.class_embedding"],
                               sd[p + "embeddings.position_embedding.weight"], sd[p + "pre_layrnorm.weight"],
                               sd[p + "pre_layrnorm.bias"], n, cfg.eps)
    torch.cuda.synchronize()
    assert torch.equal(got.view(n * (eng.P + 1), C), want)
