"""mm_projector factory (reference: video_chatgpt/model/multimodal_projector/builder.py:33-51).

In this build the projector is not an nn.Module: its GEMM(s) run inside libvcl.so (wgmma GEMM with
bias / erf-GELU epilogues, written straight into the rows that get spliced into the prompt). The
factory therefore returns a ProjectorSpec that names the state_dict keys and the C-ABI proj_type.
"""
import re
from dataclasses import dataclass


@dataclass(frozen=True)
class ProjectorSpec:
    kind: str          # 'linear' | 'mlp2x_gelu' | 'identity'
    in_features: int
    out_features: int

    @property
    def state_keys(self):
        if self.kind == "linear":
            return ["weight", "bias"]
        if self.kind == "mlp2x_gelu":
            return ["0.weight", "0.bias", "2.weight", "2.bias"]
        return []


def build_vision_projector(config, delay_load=False, **kwargs):
    kind = getattr(config, "mm_projector_type", "linear")
    if kind == "linear":
        return ProjectorSpec("linear", config.mm_hidden_size, config.hidden_size)
    m = re.match(r"^mlp(\d+)x_gelu$", kind)
    if m:
        if int(m.group(1)) != 2:
            raise ValueError(f"libvcl implements mlp2x_gelu only (got {kind})")
        return ProjectorSpec("mlp2x_gelu", config.mm_hidden_size, config.hidden_size)
    if kind == "identity":
        raise ValueError("identity projector: mm_hidden_size must equal hidden_size; not supported by libvcl")
    raise ValueError(f"Unknown projector type: {kind}")
