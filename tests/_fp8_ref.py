"""Torch restatement of the fp8 (E4M3) weight format of vcl_load_llm_weights_ex (include/vcl.h):

    a_r = max_k |W[r,k]|,  e_r = the smallest integer with a_r <= 448 * 2^e_r (0 for an all-zero row),
    q[r,k] = E4M3(W[r,k] * 2^-e_r)  (round to nearest even, subnormals included),
    W~[r,k] = q[r,k] * 2^e_r        (exactly a bf16 number),

and the slot order in which the decode kernels read the codes. Works on any device."""
import torch

E4M3_MAX = 448.0


def row_exponents(w: torch.Tensor) -> torch.Tensor:
    """e_r of every row of w [N, K] (int64): 448 = 0.875 * 2^9, a_r = m * 2^x with 0.5 <= m < 1"""
    a = w.float().abs().amax(1)
    m, x = torch.frexp(a)
    e = torch.where(m <= 0.875, x - 9, x - 8).long()
    return torch.where(a > 0, e, torch.zeros_like(e))


def pow2(e: torch.Tensor) -> torch.Tensor:
    """2^e exactly, fp32"""
    return torch.ldexp(torch.ones(e.shape, dtype=torch.float32, device=e.device), e.to(torch.int32))


def quantize(w: torch.Tensor):
    """w [N, K] bf16 -> (codes [N, K] float8_e4m3fn, e [N] int64, W~ [N, K] bf16)"""
    e = row_exponents(w)
    q = (w.float() * pow2(-e)[:, None]).to(torch.float8_e4m3fn)
    deq = (q.float() * pow2(e)[:, None]).to(torch.bfloat16)
    return q, e, deq


def dequantized(w: torch.Tensor) -> torch.Tensor:
    return quantize(w)[2]


def finite_codes() -> torch.Tensor:
    """every finite E4M3 value (254 of them: 0x7f / 0xff are NaN), as float32, in code order"""
    c = torch.arange(256, dtype=torch.uint8)
    c = c[(c & 0x7F) != 0x7F]
    return c.view(torch.float8_e4m3fn).float()


def slot_offsets(N: int, K: int, device="cpu") -> torch.Tensor:
    """byte offset of code (r, k) in the slot-ordered copy: [16-row group][512-k chunk][32-k block][row half]
    [lane = (r % 8) * 4 + k % 32 / 8][k % 8]"""
    r = torch.arange(N, device=device)[:, None]
    k = torch.arange(K, device=device)[None, :]
    return ((r // 16) * 16 * K + (k // 512) * 8192 + (k % 512 // 32) * 512 + (r % 16 // 8) * 256
            + ((r % 8) * 4 + k % 32 // 8) * 8 + k % 8)


def tiled_codes(q: torch.Tensor) -> torch.Tensor:
    """codes [N, K] float8_e4m3fn -> the flat uint8 copy the decode kernels read (rows past N zero)"""
    N, K = q.shape
    out = torch.zeros((N + 15) // 16 * 16 * K, dtype=torch.uint8, device=q.device)
    out[slot_offsets(N, K, q.device).reshape(-1)] = q.view(torch.uint8).reshape(-1)
    return out


def dequantize_state(sd: dict) -> dict:
    """A state dict whose five streamed matrices per layer (q, k, v, o, gate, up, down) and lm_head are replaced by
    W~. The quantization is per row, so quantizing each tensor alone equals quantizing the loader's fused q|k|v
    and interleaved gate|up."""
    out = {}
    for k, v in sd.items():
        streamed = k == "lm_head.weight" or (k.startswith("model.layers.") and k.endswith("_proj.weight"))
        out[k] = dequantized(v.to(torch.bfloat16)) if streamed else v
    return out
