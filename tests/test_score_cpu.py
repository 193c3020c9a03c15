"""CPU tests of forward(labels=...) on the host side: the labels / attention_mask checks run before any device
work (left and right padding accepted with labels, malformed labels rejected), and the unsupported argument
combinations raise NotImplementedError."""
import pytest
import torch

from video_chatgpt.model.video_chatgpt import score_padding

V = 32003


def _t(rows):
    return torch.tensor(rows, dtype=torch.int64)


def test_no_mask_and_all_ones_mask_run_unpadded():
    lab = _t([[-100, 5, 6, 7], [-100, -100, 0, V - 1]])
    assert score_padding(None, lab, (2, 4), V) is None
    assert score_padding(torch.ones(2, 4, dtype=torch.bool), lab, (2, 4), V) is None


def test_left_padding_gives_the_pad_counts():
    mask = _t([[0, 0, 1, 1, 1], [1, 1, 1, 1, 1]])
    lab = _t([[-100, -100, -100, 8, 9], [-100, 4, 5, 6, 7]])
    assert score_padding(mask, lab, (2, 5), V) == [2, 0]


def test_right_padding_collator_layout_runs_unpadded():
    # train.py's collator: pad_sequence(batch_first=True), labels padded with -100, mask = ids != pad
    mask = _t([[1, 1, 1, 0, 0], [1, 1, 1, 1, 1]])
    lab = _t([[-100, 4, 5, -100, -100], [-100, -100, 6, 7, 8]])
    assert score_padding(mask, lab, (2, 5), V) is None
    assert score_padding(mask.bool(), lab, (2, 5), V) is None


@pytest.mark.parametrize("lab, match", [
    ([[-100, 5, V]], "neither a token id"),                      # one past the vocabulary
    ([[-100, -1, 5]], "neither a token id"),                     # negative, not -100
    ([[-100, 5, -101]], "neither a token id"),
])
def test_out_of_range_labels_are_rejected(lab, match):
    with pytest.raises(ValueError, match=match):
        score_padding(None, _t(lab), (1, 3), V)


def test_labels_shape_and_dtype():
    with pytest.raises(ValueError, match="shape"):
        score_padding(None, _t([[1, 2, 3]]), (1, 4), V)
    with pytest.raises(ValueError, match="integer"):
        score_padding(None, torch.zeros(1, 3), (1, 3), V)


@pytest.mark.parametrize("mask, lab, match", [
    ([[0, 1, 1, 1]], [[5, -100, 6, 7]], "pad column"),            # a pad column with a real label
    ([[0, 1, 1, 1]], [[-100, 5, 6, 7]], "first real token"),      # the first real token after left padding
    ([[1, 1, 1, 0]], [[-100, 5, 6, 7]], "pad column"),            # right padding with a real label
    ([[1, 0, 1, 1]], [[-100, -100, 6, 7]], "holes"),
    ([[0, 1, 1, 1], [1, 1, 1, 0]], [[-100, -100, 6, 7], [-100, 5, 6, -100]], "mixes"),
    ([[0, 0, 0, 0]], [[-100, -100, -100, -100]], "no real token"),
    ([[0, 2, 1, 1]], [[-100, -100, 6, 7]], "0/1"),
])
def test_malformed_masks_and_pad_labels_are_rejected(mask, lab, match):
    m = _t(mask)
    with pytest.raises(ValueError, match=match):
        score_padding(m, _t(lab), tuple(m.shape), V)


def _model():
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    cfg = VideoChatGPTConfig(hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4,
                             vocab_size=V, use_mm_proj=True, mm_hidden_size=1024)
    return VideoChatGPTLlamaForCausalLM(cfg, clip_config={})


def test_forward_validates_on_the_host_before_any_device_work():
    """Without a GPU the engine cannot be created, so a ValueError / NotImplementedError here proves the check
    ran first."""
    m = _model()
    ids = torch.randint(3, 1000, (2, 6))
    with pytest.raises(ValueError, match="neither a token id"):
        m(input_ids=ids, labels=torch.full((2, 6), V))
    with pytest.raises(ValueError, match="shape"):
        m(input_ids=ids, labels=torch.full((2, 5), -100))
    mask = torch.ones(2, 6, dtype=torch.int64); mask[1, -2:] = 0
    lab = torch.full((2, 6), -100); lab[1, -1] = 9
    with pytest.raises(ValueError, match="pad column"):
        m(input_ids=ids, attention_mask=mask, labels=lab)
    with pytest.raises(NotImplementedError, match="logits_to_keep"):
        m(input_ids=ids, logits_to_keep=2)
    with pytest.raises(NotImplementedError, match="output_hidden_states"):
        m(input_ids=ids, labels=torch.full((2, 6), -100), output_hidden_states=True)
    with pytest.raises(NotImplementedError, match="cached"):
        m(input_ids=ids[:, :1], labels=torch.full((2, 1), -100), past_key_values=6)
