"""The NumPy mirror of vcl_resize_frames (tests/_resize_ref.py) against its oracles: torch's nearest interpolate for
load_video's resize, PIL's BICUBIC resize for the image processor's, and the processor's 2023 size and crop rules for
video_chatgpt.preprocess.processor_plan."""
import types

import numpy as np
import pytest
import torch
from PIL import Image

import _resize_ref as R


def _pil(frames, out_h, out_w):
    return np.stack([np.asarray(Image.fromarray(f).resize((out_w, out_h), Image.BICUBIC)) for f in frames])


def _torch_nearest(frames, out_h, out_w):
    """load_video's resize (video_chatgpt/eval/model_utils.py)."""
    t = torch.from_numpy(frames).permute(0, 3, 1, 2).float()
    return torch.nn.functional.interpolate(t, size=(out_h, out_w)).permute(0, 2, 3, 1).to(torch.uint8).numpy()


def test_nearest_index_rule_matches_torch_for_every_size():
    for n_out in (224, 336, 7, 1):
        outs = []
        for n_in in range(1, 2201):
            src = torch.arange(n_in, dtype=torch.float32).view(1, 1, 1, n_in)
            got = torch.nn.functional.interpolate(src, size=(1, n_out)).view(-1).long().numpy()
            outs.append((n_in, got))
        bad = [n_in for n_in, got in outs if not np.array_equal(got, R.nearest_index(n_in, n_out))]
        assert not bad, (n_out, bad[:10])


@pytest.mark.parametrize("shape", [(720, 1280, 224, 224), (1080, 1920, 336, 336), (360, 640, 224, 224),
                                   (37, 53, 224, 336), (224, 224, 224, 224)])
def test_nearest_frames_match_load_video(shape):
    H, W, oh, ow = shape
    frames = np.random.default_rng(H * W).integers(0, 256, (2, H, W, 3), dtype=np.uint8)
    assert np.array_equal(R.nearest_ref(frames, oh, ow), _torch_nearest(frames, oh, ow))


def _inputs(H, W, n, seed):
    """random frames, a diagonal gradient, and saturated 0 / 255 blocks next to each other."""
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    f[0] = ((yy * 255 // max(H - 1, 1) + xx * 255 // max(W - 1, 1)) // 2)[..., None].astype(np.uint8)
    if n > 1:
        f[1, : H // 2] = 255
        f[1, H // 2:] = 0
        f[1, :, : W // 3] = 255 - f[1, :, : W // 3]
    return f


# (in_h, in_w, out_h, out_w): 4K, 1080p, 720p and 480p down to the 224 / 336 towers' shortest-edge sizes, portrait,
# odd sizes, one pixel in and out, upscales
BICUBIC_GRID = [(2160, 3840, 224, 398), (1080, 1920, 336, 597), (720, 1280, 224, 398), (480, 640, 336, 448),
                (1280, 720, 398, 224), (37, 53, 11, 7), (1, 1, 224, 224), (224, 224, 1, 1), (224, 224, 336, 336),
                (360, 640, 224, 398), (5, 9, 13, 3), (300, 301, 300, 224), (301, 300, 224, 300)]


@pytest.mark.parametrize("shape", BICUBIC_GRID)
def test_bicubic_mirror_matches_pil(shape):
    H, W, oh, ow = shape
    frames = _inputs(H, W, 1 if H * W > 1e6 else 3, seed=H + W)
    assert np.array_equal(R.bicubic_ref(frames, oh, ow), _pil(frames, oh, ow))


def test_bicubic_saturated_blocks_need_the_clamp():
    """The fixed-point sum leaves 0..255 next to saturated edges, so the mirror's clamp is exercised."""
    H, W, oh, ow = 64, 64, 200, 200
    f = np.zeros((1, H, W, 3), np.uint8)
    f[0, :, ::2] = 255
    bounds, kk = R.bicubic_coeffs(W, ow)
    acc = (1 << 21) + 255 * np.where(kk > 0, kk, 0).sum(1)
    assert (acc >> 22).max() > 255                             # the positive lobe alone overshoots
    assert np.array_equal(R.bicubic_ref(f, oh, ow), _pil(f, oh, ow))


def _processor(**kw):
    from video_chatgpt.preprocess import CLIP_MEAN, CLIP_STD
    d = dict(do_resize=True, size={"shortest_edge": 224}, resample=3, do_center_crop=True,
             crop_size={"height": 224, "width": 224}, do_rescale=True, rescale_factor=1 / 255, do_normalize=True,
             image_mean=list(CLIP_MEAN), image_std=list(CLIP_STD))
    d.update(kw)
    return types.SimpleNamespace(**d)


def test_processor_plan_follows_the_2023_size_and_crop_rules():
    from video_chatgpt.preprocess import processor_plan
    for size in (224, 336):
        ip = _processor(size={"shortest_edge": size}, crop_size={"height": size, "width": size})
        for H, W in [(720, 1280), (1080, 1920), (2160, 3840), (480, 640), (1280, 720), (size, size), (size, 1000),
                     (999, size), (301, 300), (1, 1), (225, 8192), (7, 13)]:
            (oh, ow), (top, left, ch, cw) = processor_plan(ip, H, W, size)
            assert (oh, ow) == R.shortest_edge_size(H, W, size)
            assert (top, left) == R.center_crop_offsets(oh, ow, size, size) and (ch, cw) == (size, size)
            assert 0 <= top and top + ch <= oh and 0 <= left and left + cw <= ow
    # int(size * long / short) truncates: 224 * 1280 / 720 = 398.2
    assert processor_plan(_processor(), 720, 1280, 224)[0] == (224, 398)


def test_processor_plan_matches_the_installed_processor_settings():
    """The processor the checkpoints ship (CLIPImageProcessor with shortest_edge and a square crop) is accepted."""
    from transformers import CLIPImageProcessor
    from video_chatgpt.preprocess import processor_plan
    ip = CLIPImageProcessor(size={"shortest_edge": 336}, crop_size={"height": 336, "width": 336})
    assert processor_plan(ip, 480, 640, 336) == ((336, 448), (0, 56, 336, 336))


@pytest.mark.parametrize("kw, what", [
    (dict(do_resize=False), "do_resize"),
    (dict(size={"height": 224, "width": 224}), "size"),
    (dict(resample=2), "resample"),
    (dict(do_center_crop=False), "center crop"),
    (dict(crop_size={"height": 224, "width": 200}), "center crop"),
    (dict(size={"shortest_edge": 200}), "shortest_edge=200"),
    (dict(rescale_factor=1 / 256), "rescale"),
    (dict(do_rescale=False), "rescale"),
    (dict(image_mean=[0.5, 0.5, 0.5]), "normalisation"),
    (dict(do_normalize=False), "normalisation"),
])
def test_processor_plan_rejects_settings_it_cannot_reproduce(kw, what):
    from video_chatgpt.preprocess import processor_plan
    with pytest.raises(ValueError, match=what):
        processor_plan(_processor(**kw), 720, 1280, 224)
