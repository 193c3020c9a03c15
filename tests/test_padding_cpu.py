"""CPU tests of left-padded batching on the host side: the attention_mask parser (left padding only,
bool or integer masks, all-ones = no padding) and the check that a video span lies inside the real
tokens of its row."""
import pytest
import torch

from oracle import vcl_oracle as O
from video_chatgpt.model.video_chatgpt import left_padding


def _mask(rows):
    return torch.tensor(rows, dtype=torch.int64)


def test_left_padding_is_accepted():
    m = _mask([[0, 0, 1, 1, 1], [1, 1, 1, 1, 1], [0, 0, 0, 0, 1]])
    assert left_padding(m, (3, 5)) == [2, 0, 4]


@pytest.mark.parametrize("dtype", [torch.bool, torch.int32, torch.int64, torch.uint8])
def test_bool_and_int_masks_agree(dtype):
    m = _mask([[0, 1, 1, 1], [0, 0, 0, 1]]).to(dtype)
    assert left_padding(m, (2, 4)) == [1, 3]


def test_all_ones_mask_means_no_padding():
    assert left_padding(torch.ones(3, 7, dtype=torch.int64), (3, 7)) is None
    assert left_padding(torch.ones(1, 7, dtype=torch.bool), (1, 7)) is None
    assert left_padding(None, (2, 7)) is None


@pytest.mark.parametrize("rows, match", [
    ([[1, 1, 1, 0]], "not left padding"),           # right padding
    ([[1, 1, 1, 1], [1, 1, 0, 0]], "row 1 is not left padding"),
    ([[0, 1, 0, 1]], "not left padding"),           # a hole after the padding
    ([[1, 0, 1, 1]], "not left padding"),           # a hole inside the real tokens
    ([[0, 0, 0, 0]], "no real token"),              # an empty row
    ([[0, 2, 1, 1]], "0/1"),                        # not a mask
])
def test_malformed_masks_are_rejected(rows, match):
    m = _mask(rows)
    with pytest.raises(ValueError, match=match):
        left_padding(m, tuple(m.shape))


def test_mask_shape_must_match_the_ids():
    with pytest.raises(ValueError, match="shape"):
        left_padding(torch.ones(2, 5, dtype=torch.int64), (2, 6))
    with pytest.raises(ValueError, match="0/1"):
        left_padding(torch.ones(1, 5), (1, 5))          # a float mask


def test_video_span_must_not_overlap_the_padding():
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    cfg = VideoChatGPTConfig(hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4,
                             vocab_size=32003, use_mm_proj=True, mm_hidden_size=1024)
    m = VideoChatGPTLlamaForCausalLM(cfg, clip_config={})
    vc = m.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = 32000, 32001, 32002, True
    lcfg = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)
    # row 0: 6 pad ids then a prompt with 57 ids before <vid_start> (at column 6 + 58 = 64); row 1 unpadded
    short = O.make_prompt_ids(lcfg, 356, seed=1, n_pre=57)
    ids = torch.cat([torch.cat([torch.zeros(1, 6, dtype=torch.int64), short], 1),
                     O.make_prompt_ids(lcfg, 356, seed=2)], 0)
    assert m._video_spans(ids, 356, [6, 0]) == [64, 64]
    with pytest.raises(ValueError, match="inside the left padding"):
        m._video_spans(ids, 356, [65, 0])
    vc.use_vid_start_end = False                          # the patch tokens themselves start the span (column 65)
    assert m._video_spans(ids, 356, [65, 0]) == [64, 64]
    with pytest.raises(ValueError, match="inside the left padding"):
        m._video_spans(ids, 356, [66, 0])
