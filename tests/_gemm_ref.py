"""Exact-integer operands, the float64 reference and poisoned views for the wgmma GEMM (gemm_tc.cu).

Exactness. A holds integers in [-2, 2], W integers in [-1, 1], the bias integers in [-8, 8] and the residual
integers in [-64, 64], all exact in bf16. W and the bias may share a power-of-two scale 2^w_exp (the activation
tests use one so that pre-activations land where the activations bend); that moves every value by the same
exponent and changes nothing below. Every product A[m, k] W[n, k] is then an integer multiple of 2^w_exp, and
every partial sum of K products plus the bias is bounded by

    K * max|A| * max|W| + max|bias|       (in units of 2^w_exp, exact_bound)

which exact_bound asserts is below 2^24: fp32 holds every such partial sum exactly, so the accumulator value does
not depend on the K order, the tile, the cluster or the schedule, and the reference is the exact sum.

Reference (gemm_exact / plain_out):
  y   = A . W^T + bias                         float64 (exact, the operands are integers)
  out = bf16_rn(y)                             one rounding (_act_ref.bf16_rn: .bfloat16() on float64 rounds
                                               twice, through fp32)
  out = bf16_rn(bf16_rn(y) + res)              with a residual: the store warps' packed bf16x2 add of the rounded
                                               GEMM output and the residual, rounded once more
An exact zero may come out as +0 or -0 depending on how signed zero products meet in the sum, so outputs are
compared with the sign of zero folded (same_bits); every other value must match bit for bit.

Poisoned views (padded): an operand or output lives in a larger backing buffer, at a row pitch of cols + pad_cols
(a multiple of 8, so every row starts 16-byte aligned), with `top` rows above and `bottom` rows below it. A and W are
filled with NaN outside the view, so an element read past column K or outside the rows turns outputs into NaN.
Outputs and residuals sit in a buffer of SENTINEL, a NaN bit pattern no kernel writes: the margins must keep it bit
for bit, and an element inside the view that the kernel never wrote keeps it too and fails the comparison."""
import torch

from _act_ref import bf16_rn

A_MAX, W_MAX, BIAS_MAX, RES_MAX = 2, 1, 8, 64
EXACT_LIMIT = 2 ** 24        # every integer of magnitude up to 2^24 is an fp32 value
SENTINEL = 0x7FA5            # a bf16 NaN bit pattern no kernel produces


def exact_bound(K, a_max=A_MAX, w_max=W_MAX, bias_max=BIAS_MAX):
    """the largest magnitude a partial sum of K products plus the bias can reach (in units of the W / bias scale);
    asserts that fp32 holds every such sum exactly"""
    b = K * a_max * w_max + bias_max
    assert b < EXACT_LIMIT, f"K={K}: partial sums up to {b} are not all exact in fp32"
    return b


def ints(shape, lim, gen, device="cpu", exp=0):
    """bf16 integers uniform in [-lim, lim], times 2^exp"""
    v = torch.randint(-lim, lim + 1, shape, generator=gen, dtype=torch.int32).double()
    return (v * 2.0 ** exp).to(device=device, dtype=torch.bfloat16)


def operands(M, N, K, seed, device="cpu", bias=False, res_cols=0, w_exp=0):
    """(A [M, K], W [N, K], bias [N] or None, residual [M, res_cols] or None): exact integers as above"""
    exact_bound(K)
    g = torch.Generator().manual_seed(seed)
    a = ints((M, K), A_MAX, g, device)
    w = ints((N, K), W_MAX, g, device, w_exp)
    b = ints((N,), BIAS_MAX, g, device, w_exp) if bias else None
    r = ints((M, res_cols), RES_MAX, g, device) if res_cols else None
    return a, w, b, r


def gemm_exact(a, w, bias=None):
    """y = A . W^T (+ bias) in float64, on the operands' device: exact for the operands above (and for any bf16
    operands whose products and partial sums fit float64's 53 bits)"""
    y = a.double() @ w.double().t()
    if bias is not None:
        y += bias.double()
    return y


def plain_out(y, res=None):
    """the kernel's output without an activation: bf16_rn(y), then bf16_rn(that + res) with a residual"""
    o = bf16_rn(y)
    if res is not None:
        o = bf16_rn(o.double() + res.double())
    return o


def padded(rows, cols, top=0, bottom=0, pad_cols=0, fill=float("nan"), device="cpu"):
    """(buffer, view): view is [rows, cols] at row `top` of a [top + rows + bottom, cols + pad_cols] bf16 buffer.
    fill: a float (A, W: NaN) or an int bf16 bit pattern (outputs: SENTINEL) for the whole buffer."""
    assert pad_cols % 8 == 0 and pad_cols >= 0, "pitches stay multiples of 8 elements (16 bytes)"
    shape = (top + rows + bottom, cols + pad_cols)
    if isinstance(fill, int):
        buf = torch.full(shape, fill, dtype=torch.int16, device=device).view(torch.bfloat16)
    else:
        buf = torch.full(shape, fill, dtype=torch.bfloat16, device=device)
    return buf, buf[top:top + rows, :cols]


def view_origin(buf, view):
    """(row, column) of view's first element inside buf"""
    assert view.stride() == buf.stride() and view.untyped_storage().data_ptr() == buf.untyped_storage().data_ptr()
    return divmod(view.storage_offset() - buf.storage_offset(), buf.stride(0))


def fold_zero(bits):
    """int16 bf16 bit patterns with -0 mapped to +0"""
    return torch.where(bits == -32768, torch.zeros_like(bits), bits)


def same_bits(out, ref):
    """element-wise: bit-identical with the sign of zero folded"""
    return fold_zero(out.view(torch.int16)) == fold_zero(ref.view(torch.int16))


def buffer_check(buf, view, ref, fill=SENTINEL):
    """(wrong elements inside the view, changed margin elements) of an output buffer, as 0-d int64 tensors on the
    buffer's device (no host synchronisation): inside, same_bits with ref; outside, the bit pattern `fill`"""
    r0, c0 = view_origin(buf, view)
    rows, cols = view.shape
    bits = buf.view(torch.int16)
    inside = torch.zeros(bits.shape, dtype=torch.bool, device=bits.device)
    inside[r0:r0 + rows, c0:c0 + cols] = True
    margin_bad = ((bits != fill) & ~inside).sum()
    return (~same_bits(view, ref)).sum(), margin_bad


# ---- the K-addressing probe ----
def probe_k(i, K):
    """the K column one-hot row i of the probe operand selects: (37 i + 5) mod K, a bijection on K consecutive i"""
    return (37 * i + 5) % K


def probe_code(j, k, K):
    """an exact bf16 value that names column k of row j of the coded operand: with c = (k + 13 j) mod K < 4096,
    (128 + c % 128) * 2^(c // 128 - 16), i.e. c's low 7 bits are the mantissa and its high 5 bits the exponent
    (positive, normal, from 2^-9 to just under 2^23: one product with 1, plus products with 0, is exact)"""
    assert K <= 4096
    c = (k + 13 * j) % K
    return ((128 + c % 128).double() * torch.exp2((c // 128 - 16).double())).bfloat16()


def probe_decode(v, j, K):
    """the column k whose code probe_code(j, k, K) is the bf16 value v (int64 tensor; -1 where v is no code: NaN,
    zero, negative or a subnormal)"""
    bits = v.view(torch.int16).to(torch.int64) & 0xFFFF
    e = (bits >> 7) & 0xFF                                # v = 2^(e - 127) (1 + mantissa / 128) = 2^(h - 9) (128 + ...)
    h = e - 127 + 9
    c = (h << 7) | (bits & 0x7F)
    ok = (bits < 0x7F80) & (h >= 0) & (c < K)
    return torch.where(ok, (c - 13 * j) % K, torch.full_like(c, -1))
