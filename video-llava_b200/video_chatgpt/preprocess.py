"""CLIPImageProcessor's resize and center crop on the device, for raw uint8 frames.

The reference runs `image_processor.preprocess(frames)` on the CPU (inference.py:86): with transformers as the
reference pins it, a PIL bicubic resize of the shortest edge to `size["shortest_edge"]`, a center crop to
`crop_size`, then x / 255 and CLIP's mean / std. `processor_resize` does the resize and the crop with
vcl_resize_frames, bit for bit, and leaves uint8 frames the tower normalises itself (its uint8 path applies the same
rescale and mean / std). Settings it cannot reproduce raise; there is no CPU fallback.
"""
import torch

import vcl_native as vn

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)   # the constants the tower's uint8 path applies (im2col)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
PIL_BICUBIC = 3


def _field(d, key):
    """`key` of a size dict: a plain dict in older transformers, a SizeDict with attributes in newer ones."""
    if d is None:
        return None
    return d.get(key) if isinstance(d, dict) else getattr(d, key, None)


def processor_plan(image_processor, frame_h: int, frame_w: int, image_size: int):
    """-> ((out_h, out_w), (top, left, crop_h, crop_w)): the processor's resize of a frame_h x frame_w frame and the
    crop it then takes, for a tower of image_size px. Raises ValueError on any setting it cannot reproduce."""
    ip = image_processor

    def need(ok, what):
        if not ok:
            raise ValueError(f"the image processor's {what} cannot be reproduced on the device")

    need(getattr(ip, "do_resize", False), "do_resize=False")
    size = getattr(ip, "size", None)
    short = _field(size, "shortest_edge")
    need(short is not None and _field(size, "height") is None and _field(size, "width") is None,
         f"size={size!r} (only shortest_edge)")
    resample = getattr(ip, "resample", None)
    need(resample is not None and int(resample) == PIL_BICUBIC, f"resample={resample!r} (only BICUBIC)")
    crop = getattr(ip, "crop_size", None)
    need(getattr(ip, "do_center_crop", False) and _field(crop, "height") == image_size
         and _field(crop, "width") == image_size, f"center crop {crop!r} (only {image_size}x{image_size}, the tower's)")
    need(short >= image_size, f"shortest_edge={short} below the {image_size}-px crop (the crop would pad)")
    need(getattr(ip, "do_rescale", False) and float(ip.rescale_factor) == 1 / 255,
         f"rescale (do_rescale={getattr(ip, 'do_rescale', None)}, factor {getattr(ip, 'rescale_factor', None)})")
    need(getattr(ip, "do_normalize", False) and tuple(map(float, ip.image_mean)) == CLIP_MEAN
         and tuple(map(float, ip.image_std)) == CLIP_STD, "normalisation (only CLIP's mean / std)")

    # transformers' get_resize_output_image_size(default_to_square=False): the short side becomes `short`
    lo, hi = (frame_w, frame_h) if frame_w <= frame_h else (frame_h, frame_w)
    if lo == short:
        out_h, out_w = frame_h, frame_w
    else:
        new_long = int(short * hi / lo)
        out_h, out_w = (new_long, short) if frame_w <= frame_h else (short, new_long)
    return (out_h, out_w), ((out_h - image_size) // 2, (out_w - image_size) // 2, image_size, image_size)


def processor_resize(frames: torch.Tensor, image_processor, image_size: int) -> torch.Tensor:
    """uint8 [T,H,W,3] frames -> uint8 [T, image_size, image_size, 3] CUDA frames: the processor's resize and crop,
    equal to its output before the rescale and normalisation. Frames the processor leaves as they are (no resize,
    the crop the whole frame) are returned without a launch."""
    if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
        raise ValueError("frames must be a uint8 [T,H,W,3] tensor, got "
                         f"{getattr(frames, 'dtype', type(frames))} {tuple(getattr(frames, 'shape', ()))}")
    frames = frames.cuda()
    size, crop = processor_plan(image_processor, frames.shape[1], frames.shape[2], image_size)
    if size == (image_size, image_size) == tuple(frames.shape[1:3]):
        return frames
    return vn.resize_frames(frames, size, "bicubic", crop)

