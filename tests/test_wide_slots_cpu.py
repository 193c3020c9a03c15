"""The slot capacity (max_slots) on the host: the config field, the Python rule and its rejections, which all come
before any engine exists. The device side is tests/test_wide_slots_gpu.py."""
import ctypes
import inspect

import numpy as np
import pytest

import vcl_native as vn


def test_config_has_a_trailing_max_slots_field():
    names = [f[0] for f in vn.vcl_config._fields_]
    assert names[-1] == "max_slots" and names[-2] == "max_seq"
    assert ctypes.sizeof(vn.vcl_config) == 20 * 4
    assert vn.vcl_config().max_slots == 0          # zero-initialised: the default slot count


@pytest.mark.parametrize("max_batch,max_slots,want", [(1, None, 1), (9, None, 9), (17, None, 16), (200, None, 16),
                                                      (64, 64, 64), (200, 64, 64), (40, 17, 17), (3, 1, 1)])
def test_slot_capacity(max_batch, max_slots, want):
    assert vn.slot_capacity(max_batch, max_slots) == want


@pytest.mark.parametrize("max_batch,max_slots", [(8, 9), (80, 65), (8, 0), (8, -1), (8, 2.5), (8, True), (8, "4")])
def test_slot_capacity_rejects(max_batch, max_slots):
    with pytest.raises(ValueError, match="max_slots"):
        vn.slot_capacity(max_batch, max_slots)


def _model(**kw):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    c = VideoChatGPTConfig(hidden_size=512, intermediate_size=1024, num_hidden_layers=1, num_attention_heads=4,
                           vocab_size=32003, use_mm_proj=True, mm_hidden_size=1024)
    clip = dict(hidden_size=1024, intermediate_size=1024, num_hidden_layers=3, num_attention_heads=16)
    return VideoChatGPTLlamaForCausalLM(c, clip_config=clip, max_seq=480, **kw)


def test_model_rejects_a_bad_max_slots_before_an_engine_exists():
    for mb, ms in ((8, 9), (80, 65), (8, 0)):
        with pytest.raises(ValueError, match="max_slots"):
            _model(max_batch=mb, max_slots=ms)
    m = _model(max_batch=80, max_slots=64)
    assert m._engine is None and m._n_slots == 64 and m._max_slots == 64
    assert _model(max_batch=80)._n_slots == 16 and _model(max_batch=80)._max_slots == 0


def test_generate_requests_is_capped_by_the_slot_count():
    m = _model(max_batch=40, max_slots=24)
    with pytest.raises(ValueError, match=r"slots=25 outside 1..24 \(max_slots 24\)"):
        m.generate_requests([[1, 2, 3]], slots=25)
    d = _model(max_batch=40)
    with pytest.raises(ValueError, match=r"slots=17 outside 1..16 \(at most 16 and at most max_batch 40\)"):
        d.generate_requests([[1, 2, 3]], slots=17)
    assert m._engine is None and d._engine is None


def test_max_slots_reaches_the_engine_config_and_initialize_model(monkeypatch):
    from video_chatgpt.eval.model_utils import initialize_model
    from video_chatgpt.model import VideoChatGPTLlamaForCausalLM
    assert inspect.signature(initialize_model).parameters["max_slots"].default is None
    assert inspect.signature(VideoChatGPTLlamaForCausalLM.__init__).parameters["max_slots"].default is None
    seen = []

    class FakeEngine:
        def __init__(self, cfg):
            seen.append((cfg.max_batch, cfg.max_slots))

    monkeypatch.setattr(vn, "Engine", FakeEngine)
    _model(max_batch=80, max_slots=40)._ensure_engine()
    _model(max_batch=80, max_slots=np.int64(64))._ensure_engine()
    _model(max_batch=80)._ensure_engine()
    assert seen == [(80, 40), (80, 64), (80, 0)]


def test_slot_capacity_takes_numpy_integers():
    assert vn.slot_capacity(64, np.int64(48)) == 48 and type(vn.slot_capacity(64, np.int32(2))) is int
    with pytest.raises(ValueError):
        vn.slot_capacity(64, np.float32(4))
