"""Host-side mirror of the reference's `video_chatgpt` package for the inference hot path only.

Same import paths, names, argument meaning and error behaviour as the reference modules named in
each file's docstring; the device work behind them is libvcl.so (hand-written sm_90a CUDA through
the C ABI in include/vcl.h). Nothing here falls back to PyTorch modules or to the CPU.
"""
from .model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM  # noqa: F401
