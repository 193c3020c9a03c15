"""Classifier-free guidance restated in torch (transformers' UnbatchedClassifierFreeGuidanceLogitsProcessor): the
scores of a row become g * (log_softmax(cond) - log_softmax(uncond)) + log_softmax(uncond), in fp32, where uncond are
the logits of the row's unconditional sequence (its negative prompt; by default the prompt's last token alone)."""
import torch


def guide(cond, uncond, g):
    """cond / uncond [B, V] logits -> the guided scores [B, V] fp32"""
    lc = torch.log_softmax(cond.float(), dim=-1)
    lu = torch.log_softmax(uncond.float(), dim=-1)
    return g * (lc - lu) + lu


def default_negative(input_ids):
    """HF's unconditional context without negative_prompt_ids: each row's last prompt token, at position 0"""
    return input_ids[:, -1:]
