"""vcl_resize_frames on the H100: bit-identical to the NumPy mirror (tests/_resize_ref.py), to torch's nearest
interpolate (load_video) and to PIL's BICUBIC resize (the image processor), memory-safe, and wired through
load_video(device=), video_chatgpt_infer and the offline extractor with unchanged results."""
import ctypes
import importlib.util
import os
import pickle
import sys
import types

import numpy as np
import pytest
import torch
from PIL import Image

import _resize_ref as R

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _vn():
    import vcl_native as vn
    return vn


def _pil(frames, out_h, out_w):
    return np.stack([np.asarray(Image.fromarray(f).resize((out_w, out_h), Image.BICUBIC)) for f in frames])


def _torch_nearest(frames, out_h, out_w):
    t = torch.from_numpy(frames).permute(0, 3, 1, 2).float()
    return torch.nn.functional.interpolate(t, size=(out_h, out_w)).permute(0, 2, 3, 1).to(torch.uint8).numpy()


def _frames(n, H, W, seed):
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    f[0, : H // 3, : W // 3] = 255                      # saturated blocks: the clamp
    f[0, H // 2:, W // 2:] = 0
    return f


def _center(oh, ow, c):
    return ((oh - c) // 2, (ow - c) // 2, c, c)


GRID = [(2160, 3840, 224, 398), (1080, 1920, 336, 597), (720, 1280, 224, 398), (480, 640, 336, 448),
        (1280, 720, 398, 224), (37, 53, 11, 7), (1, 1, 224, 224), (224, 224, 1, 1), (224, 224, 336, 336),
        (360, 640, 224, 398), (300, 301, 300, 224), (301, 300, 224, 300), (224, 224, 224, 224)]


@pytest.mark.parametrize("shape", GRID)
def test_bicubic_matches_mirror_and_pil(shape):
    vn = _vn()
    H, W, oh, ow = shape
    n = 1 if H * W > 2e6 else 3
    f = _frames(n, H, W, H * 7 + W)
    want = _pil(f, oh, ow)
    assert np.array_equal(R.bicubic_ref(f, oh, ow), want)
    got = vn.resize_frames(torch.from_numpy(f).cuda(), (oh, ow), "bicubic").cpu().numpy()
    assert got.shape == want.shape and np.array_equal(got, want)
    c = min(oh, ow)
    if c < max(oh, ow) or c > 2:                          # a crop: the center one, and one off center
        for crop in (_center(oh, ow, c), (oh - c, ow - c, c, c), (oh // 3, ow // 4, max(oh // 2, 1), max(ow // 3, 1))):
            t, l, ch, cw = crop
            got = vn.resize_frames(torch.from_numpy(f).cuda(), (oh, ow), "bicubic", crop).cpu().numpy()
            assert np.array_equal(got, want[:, t:t + ch, l:l + cw]), crop


@pytest.mark.parametrize("shape", [(2160, 3840, 224, 224), (1080, 1920, 336, 336), (720, 1280, 224, 224),
                                   (360, 640, 224, 224), (37, 53, 224, 336), (1, 1, 7, 1), (224, 224, 224, 224)])
def test_nearest_matches_load_video_rule(shape):
    vn = _vn()
    H, W, oh, ow = shape
    f = _frames(2, H, W, H + W)
    want = _torch_nearest(f, oh, ow)
    assert np.array_equal(R.nearest_ref(f, oh, ow), want)
    got = vn.resize_frames(torch.from_numpy(f).cuda(), (oh, ow), "nearest").cpu().numpy()
    assert np.array_equal(got, want)
    crop = (oh // 4, ow // 5, max(oh // 2, 1), max(ow // 2, 1))
    got = vn.resize_frames(torch.from_numpy(f).cuda(), (oh, ow), "nearest", crop).cpu().numpy()
    t, l, ch, cw = crop
    assert np.array_equal(got, want[:, t:t + ch, l:l + cw])


@pytest.mark.parametrize("n", [1, 8, 100])
def test_frame_counts(n):
    """Every frame gets its own pixels: 720p through the processor's 224 resize + crop and load_video's nearest."""
    vn = _vn()
    f = _frames(n, 720, 1280, n)
    x = torch.from_numpy(f).cuda()
    got = vn.resize_frames(x, (224, 398), "bicubic", _center(224, 398, 224)).cpu().numpy()
    assert np.array_equal(got, _pil(f, 224, 398)[:, :, 87:311])
    assert np.array_equal(vn.resize_frames(x, (224, 224), "nearest").cpu().numpy(), _torch_nearest(f, 224, 224))


def test_nearest_then_bicubic_composite():
    """load_video(shape=224) meeting a 336-px processor: nearest to 224, then the processor's upscale to 336."""
    vn = _vn()
    from video_chatgpt.preprocess import processor_resize
    from transformers import CLIPImageProcessor
    ip = CLIPImageProcessor(size={"shortest_edge": 336}, crop_size={"height": 336, "width": 336})
    f = _frames(4, 720, 1280, 5)
    cpu = _pil(_torch_nearest(f, 224, 224), 336, 336)
    dev = processor_resize(vn.resize_frames(torch.from_numpy(f).cuda(), (224, 224), "nearest"), ip, 336)
    assert np.array_equal(dev.cpu().numpy(), cpu)
    # native frames straight into the processor: shortest edge 336, then the center crop
    want = _pil(f, 336, 597)[:, :, 130:466]
    assert np.array_equal(processor_resize(torch.from_numpy(f), ip, 336).cpu().numpy(), want)


def test_canaries_around_output_and_workspace_stay_untouched():
    vn = _vn()
    l = vn.lib()
    f = torch.from_numpy(_frames(3, 480, 640, 9)).cuda()
    pad = 4096
    for mode, (oh, ow), crop in [(1, (336, 448), (0, 56, 336, 336)), (1, (336, 640), (0, 100, 300, 336)),
                                 (1, (480, 300), (20, 10, 400, 224)), (0, (224, 224), (1, 2, 200, 201))]:
        geo = (3, 480, 640, mode, oh, ow, *crop)
        ws_bytes = l.vcl_resize_frames_workspace_bytes(*geo)
        out_bytes = 3 * crop[2] * crop[3] * 3
        buf = torch.full((pad + out_bytes + pad,), 0xA5, dtype=torch.uint8, device="cuda")
        ws = torch.full((pad + ws_bytes + pad,), 0x5A, dtype=torch.uint8, device="cuda")
        vn.check(l.vcl_resize_frames(vn.ptr(f), *geo, ctypes.c_void_p(buf.data_ptr() + pad),
                                     ctypes.c_void_p(ws.data_ptr() + pad), ws_bytes, vn.cur_stream()))
        torch.cuda.synchronize()
        assert (buf[:pad] == 0xA5).all() and (buf[pad + out_bytes:] == 0xA5).all(), geo
        assert (ws[:pad] == 0x5A).all() and (ws[pad + ws_bytes:] == 0x5A).all(), geo
        t, lft, ch, cw = crop
        ref = (_pil if mode else _torch_nearest)(f.cpu().numpy(), oh, ow)[:, t:t + ch, lft:lft + cw]
        assert np.array_equal(buf[pad:pad + out_bytes].view(3, ch, cw, 3).cpu().numpy(), ref), geo


def test_rejections_name_the_argument():
    vn = _vn()
    l = vn.lib()
    x = torch.zeros(2, 100, 120, 3, dtype=torch.uint8, device="cuda")
    for kw, what in [(dict(mode="area"), "unknown mode"), (dict(size=(0, 224)), "out_h x out_w"),
                     (dict(size=(224, 8193)), "out_h x out_w"), (dict(crop=(0, 0, 0, 5)), "crop_h x crop_w"),
                     (dict(crop=(1, 0, 224, 224)), "crop"), (dict(crop=(0, -1, 10, 10)), "crop"),
                     (dict(crop=(0, 220, 10, 10)), "outside")]:
        with pytest.raises(vn.VclError, match=what):
            vn.resize_frames(x, kw.get("size", (224, 224)), kw.get("mode", "bicubic"), kw.get("crop"))
    geo = [2, 100, 120, 1, 224, 224, 0, 0, 224, 224]
    ws_bytes = l.vcl_resize_frames_workspace_bytes(*geo)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    out = torch.empty(2, 224, 224, 3, dtype=torch.uint8, device="cuda")

    def call(geo=geo, inp=vn.ptr(x), outp=vn.ptr(out), wsp=vn.ptr(ws), nb=ws_bytes):
        return l.vcl_resize_frames(inp, *geo, outp, wsp, nb, vn.cur_stream())

    for i, what in [(0, "n=0"), (1, "in_h x in_w"), (2, "in_h x in_w"), (3, "unknown mode")]:
        g = list(geo); g[i] = 0 if i < 3 else 9
        assert call(g) == -1 and what in l.vcl_last_error().decode()
        assert l.vcl_resize_frames_workspace_bytes(*g) == ctypes.c_size_t(-1).value
    g = list(geo); g[1] = 8193
    assert call(g) == -1 and "in_h x in_w" in l.vcl_last_error().decode()
    g = list(geo); g[0] = 8193
    assert call(g) == -1 and "n=8193" in l.vcl_last_error().decode()
    assert call(nb=ws_bytes - 1) == -1 and "ws_bytes" in l.vcl_last_error().decode()
    assert call(wsp=ctypes.c_void_p(0)) == -1 and "null ws" in l.vcl_last_error().decode()
    assert call(inp=ctypes.c_void_p(0)) == -1 and "null argument (in)" in l.vcl_last_error().decode()
    assert call(outp=ctypes.c_void_p(0)) == -1 and "null argument (out)" in l.vcl_last_error().decode()
    with pytest.raises(vn.VclError, match="uint8"):
        vn.resize_frames(x.float(), (224, 224), "bicubic")
    assert call() == 0


@pytest.mark.parametrize("image", [224, 336])
@torch.no_grad()
def test_tower_and_features_from_native_frames_match_the_cpu_resize(tmp_path, image):
    """Native frames through the device resize give the tower hidden_states[-2] and clip_features of the
    CPU-resized (PIL + crop) frames bit for bit, for the 224 / linear and 336 / mlp2x checkpoints."""
    from _checkpoint import make_tiny_checkpoint
    from video_chatgpt.eval.model_utils import initialize_model
    from video_chatgpt.preprocess import processor_resize
    ck = make_tiny_checkpoint(tmp_path, image=image)
    model, tower, tok, ip, vlen = initialize_model(ck["model_dir"], max_seq=1024)
    f = _frames(5, 360, 640, image)
    oh, ow = image, int(image * 640 / 360)
    cpu = torch.from_numpy(_pil(f, oh, ow)[:, :, (ow - image) // 2:(ow - image) // 2 + image].copy()).cuda()
    dev = processor_resize(torch.from_numpy(f), ip, image)
    assert torch.equal(dev, cpu)
    assert torch.equal(tower(dev).hidden_states[-2], tower(cpu).hidden_states[-2])
    eng = model._ensure_engine(need_clip=True)
    assert torch.equal(eng.clip_features(dev), eng.clip_features(cpu))


class _Reader:
    """decord.VideoReader over .npy "videos" of native 360x640 frames."""
    def __init__(self, path, ctx=None):
        self.arr = np.load(path)
    def __len__(self): return len(self.arr)
    def get_batch(self, idx): return types.SimpleNamespace(asnumpy=lambda: self.arr[list(idx)])


def _stub_decord(monkeypatch):
    monkeypatch.setitem(sys.modules, "decord", types.SimpleNamespace(VideoReader=_Reader, cpu=lambda i: None))


def test_load_video_on_the_device_equals_the_cpu_path(tmp_path, monkeypatch):
    _stub_decord(monkeypatch)
    from video_chatgpt.eval.model_utils import load_video
    vn = _vn()
    np.save(tmp_path / "v.npy", _frames(130, 360, 640, 3))
    for shape in [(224, 224), (336, 336), (360, 640)]:
        cpu = np.stack([np.asarray(im) for im in load_video(str(tmp_path / "v.npy"), shape=shape)])
        n0 = vn.launch_count()
        dev = load_video(str(tmp_path / "v.npy"), shape=shape, device="cuda")
        assert vn.launch_count() - n0 == (0 if shape == (360, 640) else 1)
        assert dev.is_cuda and dev.dtype == torch.uint8 and np.array_equal(dev.cpu().numpy(), cpu), shape
        assert cpu.shape[0] == 100


@torch.no_grad()
def test_video_chatgpt_infer_from_native_frames(tmp_path, monkeypatch):
    """A frame tensor gives the text of the PIL list: from load_video(device="cuda") against load_video(), and
    native 360x640 frames against their PIL resize + crop. The PIL path launches what it did before."""
    _stub_decord(monkeypatch)
    from _checkpoint import make_tiny_checkpoint
    from video_chatgpt.eval.model_utils import initialize_model, load_video
    from video_chatgpt.inference import video_chatgpt_infer
    vn = _vn()
    ck = make_tiny_checkpoint(tmp_path)
    model, tower, tok, ip, vlen = initialize_model(ck["model_dir"], max_batch=1, max_seq=1024)
    native = _frames(6, 360, 640, 17)
    np.save(tmp_path / "v.npy", native)
    args = ("w10 w11 w12", "pg-video-llava", model, tower, tok, ip, vlen)
    kw = dict(do_sample=False, max_new_tokens=8)

    pil_list = load_video(str(tmp_path / "v.npy"))
    video_chatgpt_infer(pil_list, *args, **kw)             # first call: the decode graphs are captured
    n0 = vn.launch_count()
    a = video_chatgpt_infer(pil_list, *args, **kw)
    n_pil = vn.launch_count() - n0
    t224 = load_video(str(tmp_path / "v.npy"), device="cuda")
    n0 = vn.launch_count()
    b = video_chatgpt_infer(t224, *args, **kw)
    assert vn.launch_count() - n0 == n_pil                 # 224-px frames: no resize launch
    assert a == b, (a, b)

    crop = _pil(native, 224, 398)[:, :, 87:311]
    c = video_chatgpt_infer([Image.fromarray(x) for x in crop], *args, **kw)
    n0 = vn.launch_count()
    d = video_chatgpt_infer(torch.from_numpy(native), *args, **kw)
    assert vn.launch_count() - n0 == n_pil + 3             # coefficient tables, horizontal and vertical pass
    print(f"[frame_resize] infer: {a!r} / {b!r}; native {c!r} / {d!r}")
    assert c == d, (c, d)


def test_offline_extractor_pickles_are_byte_identical(tmp_path, monkeypatch):
    _stub_decord(monkeypatch)
    from _checkpoint import make_tiny_checkpoint
    from video_chatgpt.eval.model_utils import load_video
    ck = make_tiny_checkpoint(tmp_path)
    vids, outd = tmp_path / "videos", tmp_path / "feats"
    vids.mkdir()
    for i in range(3):
        np.save(vids / f"clip{i}.npy", _frames(5 + 3 * i, 360, 640, 40 + i))
    spec = importlib.util.spec_from_file_location(
        "vcl_save_feats_resize", os.path.join(HERE, "..", "video-llava_b200", "scripts",
                                              "save_spatio_temporal_clip_features.py"))
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    monkeypatch.setattr(sys, "argv", ["x", "--llava", "1.1", "--video_dir_path", str(vids), "--clip_feat_path", str(outd),
                                      "--clip_dir", ck["clip_dir"]])
    mod.main()
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    from video_chatgpt.eval.model_utils import _load_weight_files
    owner = VideoChatGPTLlamaForCausalLM(VideoChatGPTConfig(num_hidden_layers=0, hidden_size=512, intermediate_size=1024,
                                                            num_attention_heads=4, vocab_size=8),
                                         clip_config=ck["clip_dir"], max_seq=8)
    owner.get_vision_tower().load_state_dict(_load_weight_files(ck["clip_dir"]))
    engine = owner._ensure_engine(need_clip=True)
    for i in range(3):
        frames = np.stack([np.asarray(im) for im in load_video(str(vids / f"clip{i}.npy"), shape=(224, 224))])
        want = pickle.dumps(mod.extract_video(engine, frames))          # the CPU resize, as before
        assert (outd / f"clip{i}.pkl").read_bytes() == want, i
