"""fp64 references of the activation epilogues, with the reference's bf16 rounding points, and host mirrors of how the
decode projections lay out their rows and outputs.

Activations (transformers: LlamaMLP silu(gate) * up, CLIP quick_gelu x * sigmoid(1.702 x), GELU(erf)):
  swiglu  s = bf16(silu(g)), out = bf16(s * u)               g, u bf16 (the projection outputs, rounded)
  qgelu   t = bf16(fp32(1.702 x)), s = bf16(sigmoid(t)), out = bf16(x * s)   (three bf16 tensors)
  gelu    out = bf16(0.5 x (1 + erf(x / sqrt 2)))
Every rounding of an fp64 value to bf16 is one correct rounding (bf16_rn).

The bar the kernels are held to over every finite bf16 input (check_activation): an output must be bf16(u * s')
for some s' in {s64 and its two bf16 neighbours}, s64 the bf16-rounded fp64 activation (the kernels use __expf and
__fdividef, a few fp32 ulps off, which may move s by one bf16 step next to a rounding boundary); otherwise it must
equal torch's eager op on the same bf16 input bit for bit. The second rule covers x <= -88.7, where torch's own fp32
exp overflows and both give -0 while s64 is a normal number."""
import math

import numpy as np
import torch

import vcl_native as vn

N_FINITE_BF16 = 65280     # 2^16 bit patterns less the 256 infinities and NaNs


def all_finite_bf16():
    """every finite bf16 value once, [65280] bf16 (CPU), ascending bit pattern"""
    v = torch.from_numpy(np.arange(65536, dtype=np.uint16).view(np.int16).copy()).view(torch.bfloat16)
    return v[torch.isfinite(v.float())]


def bf16_rn(x):
    """fp64 -> bf16 rounded once to nearest even. torch rounds fp64 through fp32, a double rounding; rounding to odd
    into fp32 first keeps the information a second rounding to 8 bits needs."""
    x = x.double()
    f = x.float()
    over = f.double().abs() > x.abs()                       # rounded away from zero: take the truncation
    f = torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f)
    sticky = (f.double() != x).to(torch.int32)
    return (f.view(torch.int32) | sticky).view(torch.float32).bfloat16()


def bf16_neighbours(s):
    """(next below, next above) of bf16 values s, by value (the neighbours of +-0 are the smallest subnormals)"""
    b = s.view(torch.int16).to(torch.int32)
    neg = b < 0
    mag = b & 0x7FFF
    up_mag = torch.where(neg, mag - 1, mag + 1)             # toward +inf
    dn_mag = torch.where(neg, mag + 1, mag - 1)             # toward -inf
    zero = mag == 0
    up = torch.where(zero, torch.full_like(b, 0x0001), torch.where(neg & (mag == 1), torch.zeros_like(b),
                                                                   (b & ~0x7FFF) | up_mag))
    dn = torch.where(zero, torch.full_like(b, 0x8001 - 65536), torch.where(~neg & (mag == 1), torch.zeros_like(b),
                                                                           (b & ~0x7FFF) | dn_mag))
    to16 = lambda t: t.to(torch.int16).view(torch.bfloat16)
    return to16(dn), to16(up)


def silu64(g):
    g = g.double()
    return g / (1.0 + torch.exp(-g))


def sigmoid64(t):
    return 1.0 / (1.0 + torch.exp(-t.double()))


def gelu64(x):
    x = x.double()
    return 0.5 * x * (1.0 + torch.special.erf(x / math.sqrt(2.0)))


def qgelu_t(x):
    """the first bf16 tensor of quick_gelu, 1.702 * x as an eager bf16 op computes it (fp32 product, then bf16)"""
    return (x.float() * np.float32(1.702)).bfloat16()


def swiglu_ref(g, u):
    """(u, s64, out) of silu(g) * u, g / u bf16"""
    s = bf16_rn(silu64(g))
    return u, s, bf16_rn(s.double() * u.double())


def qgelu_ref(x):
    s = bf16_rn(sigmoid64(qgelu_t(x)))
    return x, s, bf16_rn(s.double() * x.double())


def gelu_ref(x):
    s = bf16_rn(gelu64(x))
    return torch.ones_like(x), s, s


def eager(kind, x, u=None):
    """torch's eager bf16 ops of an activation on the device of x"""
    F = torch.nn.functional
    if kind == "swiglu":
        return F.silu(x) * u
    if kind == "qgelu":
        return x * torch.sigmoid(1.702 * x)
    return F.gelu(x)


def in_neighbourhood(out, u, s64):
    """out == bf16(u * s') for some s' in {s64 and its two bf16 neighbours}, compared by value (+0 == -0)"""
    u, s64 = u.to(out.device), s64.to(out.device)
    dn, up = bf16_neighbours(s64)
    of = out.float()
    near = torch.zeros_like(of, dtype=torch.bool)
    for s in (dn, s64, up):
        near |= of == bf16_rn(s.double() * u.double()).float()
    return near


def check_activation(out, u, s64, torch_out):
    """The bar above, element-wise over flat bf16 tensors (any device). Returns a dict of boolean masks:
    exact (bit-identical to torch), near (not torch's bits but bf16(u * s') for a neighbour s'), torch_only (torch's
    bits, outside the fp64 neighbourhood), bad (neither)."""
    near = in_neighbourhood(out, u, s64)
    exact = out.view(torch.int16) == torch_out.to(out.device).view(torch.int16)
    return {"exact": exact, "near": near & ~exact, "torch_only": exact & ~near, "bad": ~near & ~exact}


def describe_mismatches(masks, x, out, torch_out, ref, what, n=6):
    """one printable line per kind of mismatch: count and the first few (x, out, torch, fp64 reference)"""
    lines = []
    for kind in ("near", "torch_only", "bad"):
        idx = masks[kind].nonzero().flatten()[:n].cpu()
        items = [(float(x.flatten()[i]), float(out.flatten()[i]), float(torch_out.flatten()[i]),
                  float(ref.flatten()[i])) for i in idx.tolist()]
        lines.append(f"{what}: {kind} {int(masks[kind].sum())}: (x, kernel, torch, fp64) {items}")
    return lines


# ---- the decode projections' layout (decode_gemv.cu, kernels.h) ----
def cta_row_groups(N, grid):
    """[(first row, rows)] of each CTA of a projection over N rows on `grid` CTAs: contiguous blocks of 16-row groups,
    sizes differing by at most one group (decode_gemv.cu: cta_row_groups)"""
    groups = (N + 15) // 16
    out = []
    for c in range(grid):
        g0, g1 = c * groups // grid, (c + 1) * groups // grid
        out.append((16 * g0, min(16 * g1, N) - 16 * g0))
    return out


def xwin_elems(B, K):
    return (K + vn.XWIN_KC - 1) // vn.XWIN_KC * B * vn.XWIN_PITCH


def xwin_index(B, K, device="cpu"):
    """[B, K] flat indices of the elements (b, k) in an xwin buffer (vn.xwin_offset)"""
    b = torch.arange(B, device=device)[:, None]
    k = torch.arange(K, device=device)[None, :]
    return vn.xwin_offset(b, k, B)


def xwin_unpack(buf, B, K):
    """the [B, K] rows of an xwin buffer, and the mask of the buffer's elements that belong to no (b, k)"""
    idx = xwin_index(B, K, buf.device)
    unused = torch.ones(buf.numel(), dtype=torch.bool, device=buf.device)
    unused[idx.flatten()] = False
    return buf[idx], unused
