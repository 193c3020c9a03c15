"""NumPy restatement of the two frame resizes `vcl_resize_frames` reproduces (csrc/frame_resize.cu), and of the
image processor's resize / crop geometry.

nearest_ref  torch.nn.functional.interpolate(mode="nearest") on CPU tensors, which load_video runs on frames:
             s = fp32(in) / fp32(out), src = min(floor(fp32(dst) * s), in - 1).
bicubic_ref  PIL.Image.resize(..., BICUBIC) on RGB uint8 frames (CLIPImageProcessor.resize before transformers
             moved to torchvision): two separable passes, horizontal then vertical, each rounding to uint8 and
             skipped when its size does not change; per output index xx, in double arithmetic,
                 scale = in / out, fs = max(scale, 1), support = 2 fs, center = (xx + 0.5) scale,
                 xmin = max(int(center - support + 0.5), 0), n = min(int(center + support + 0.5), in) - xmin,
                 w_x = cubic((x + xmin - center + 0.5) * (1 / fs)), a = -0.5, then w_x / sum(w),
             to fixed point with 22 fraction bits (round half away from zero); a pixel is
             clamp((2^21 + sum(p k)) >> 22, 0, 255) in int32.
resize_plan  CLIPImageProcessor's shortest-edge size rule and center-crop offsets (transformers 2023):
             the short side becomes `size`, the long side int(size * long / short); top = (H - crop) // 2.
"""
import numpy as np

PRECISION_BITS = 22


def nearest_index(n_in: int, n_out: int) -> np.ndarray:
    s = np.float32(n_in) / np.float32(n_out)
    dst = np.arange(n_out, dtype=np.float32)
    return np.minimum(np.floor(dst * s).astype(np.int64), n_in - 1)


def nearest_ref(frames: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """frames [..., H, W, C] uint8 -> [..., out_h, out_w, C]."""
    H, W = frames.shape[-3], frames.shape[-2]
    return frames[..., nearest_index(H, out_h)[:, None], nearest_index(W, out_w)[None, :], :]


def _cubic(x: float) -> float:
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def bicubic_window(n_in: int, n_out: int, xx: int):
    """(xmin, n) of output index xx: the source span its filter covers."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support = 2.0 * fs
    center = (xx + 0.5) * scale
    xmin = max(int(center - support + 0.5), 0)
    return xmin, min(int(center + support + 0.5), n_in) - xmin


def bicubic_coeffs(n_in: int, n_out: int):
    """-> bounds [n_out, 2] (xmin, n) and int32 weights [n_out, kmax] (zero past n)."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    ss = 1.0 / fs
    rows = []
    bounds = np.zeros((n_out, 2), np.int64)
    for xx in range(n_out):
        center = (xx + 0.5) * scale
        xmin, n = bicubic_window(n_in, n_out, xx)
        w = [_cubic((x + xmin - center + 0.5) * ss) for x in range(n)]
        ww = 0.0
        for v in w:
            ww += v
        k = [(v / ww if ww != 0.0 else v) for v in w]
        k = [int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS)) for v in k]
        bounds[xx] = (xmin, n)
        rows.append(k)
    kmax = max(len(r) for r in rows)
    kk = np.zeros((n_out, kmax), np.int64)
    for xx, r in enumerate(rows):
        kk[xx, :len(r)] = r
    return bounds, kk


def _pass(frames: np.ndarray, n_out: int, axis: int) -> np.ndarray:
    """One bicubic pass along `axis` of an int64 array, rounded to uint8 values."""
    n_in = frames.shape[axis]
    bounds, kk = bicubic_coeffs(n_in, n_out)
    x = np.moveaxis(frames.astype(np.int64), axis, -1)
    out = np.empty(x.shape[:-1] + (n_out,), np.int64)
    for xx in range(n_out):
        xmin, n = bounds[xx]
        acc = (1 << (PRECISION_BITS - 1)) + x[..., xmin:xmin + n] @ kk[xx, :n]
        out[..., xx] = np.clip(acc >> PRECISION_BITS, 0, 255)
    return np.moveaxis(out, -1, axis).astype(np.uint8)


def bicubic_ref(frames: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """frames [..., H, W, C] uint8 -> [..., out_h, out_w, C]; bit for bit PIL's BICUBIC resize."""
    H, W = frames.shape[-3], frames.shape[-2]
    x = frames
    if out_w != W:
        x = _pass(x, out_w, x.ndim - 2)
    if out_h != H:
        x = _pass(x, out_h, x.ndim - 3)
    return np.ascontiguousarray(x)


def shortest_edge_size(h: int, w: int, size: int):
    """(out_h, out_w) of transformers' get_resize_output_image_size(size=shortest_edge, default_to_square=False)."""
    short, long = (w, h) if w <= h else (h, w)
    if short == size:
        return h, w
    new_short, new_long = size, int(size * long / short)
    return (new_long, new_short) if w <= h else (new_short, new_long)


def center_crop_offsets(h: int, w: int, crop_h: int, crop_w: int):
    """(top, left) of transformers' center_crop when the crop fits inside the image."""
    return (h - crop_h) // 2, (w - crop_w) // 2
