"""The wgmma GEMM (gemm_tc.cu, vcl_op_gemm_ex) against its exact reference (tests/_gemm_ref.py).

The operands are small integers, so every partial sum is exact in fp32 and the accumulator holds the exact A . W^T
whatever the K order, tile, cluster or schedule: every (block_n, cluster) must give the reference's bits (the sign
of an exact zero aside), not merely the automatic choice's. Every launch runs on poisoned views: A and W inside
NaN-filled buffers at a pitch wider than K (a column read past K, or a row outside the operand, turns outputs into
NaN), bias followed by NaN, outputs and separate residuals inside a buffer of a NaN sentinel whose margins must keep
their bits (a store past row M or past the last column changes them; an element never stored keeps the sentinel
and fails the comparison).

  - edge sweep: per (block_n, cluster), every M in EDGE_M (ragged last 64-row block, clusters with CTAs whose whole
    M tile is past M), N below the TMA box, ragged N tiles and multicast slices past N, K at the operand ring's
    depth boundaries (K / 64 = STAGES - 1, STAGES, STAGES + 1), with the four epilogues: plain, bias, bias and a
    residual updated in place (C aliasing it, as the engine does), and a separate residual at a wider pitch than C
  - K-addressing probe: one operand one-hot, the other a code that names its column, so a wrong value names the
    column k it came from: a neighbouring k is a swizzle / descriptor bug, k +- 64 s a ring-stage bug
  - the activations (QGELU, GELU, SwiGLU) at ragged M and N on exact pre-activations: _act_ref.check_activation
  - the engine's call sites at the pitches vcl_api.cu passes, with the automatic tile and with every tile of
    test_gemm_schedule_gpu.TILES
  - the launcher's refusals: named in the error, no launch, and the next valid call still runs"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
import _act_ref as R  # noqa: E402
import _gemm_ref as G  # noqa: E402
from test_gemm_schedule_gpu import TILES  # noqa: E402

DEV = torch.device("cuda:0")
NAN = float("nan")
ACT_ROPE = 4                                   # kernels.h: the prefill's q|k|v epilogue, not reachable here
STAGES = {256: 3, 128: 5, 64: 8, 32: 8}        # GemmCfg<BLOCK_N>::STAGES
SWEEP = [(bn, cl) for bn in (256, 128, 64, 32) for cl in (1, 2, 4, -2)]
EDGE_M = (1, 63, 64, 65, 127, 128, 129, 200, 383, 513)
SHOW = 6                                       # failures reported per test


def edge_n(bn):
    return sorted({n for n in (32, bn - 32, bn, bn + 32, 3 * bn - 32) if n > 0 and n % 32 == 0})


def edge_k(bn):
    s = STAGES[bn]
    return [64 * x for x in sorted({1, s - 1, s, s + 1, 2 * s + 1})]


def _p(t):
    if t is None:
        return ctypes.c_void_p(0)
    assert t.is_cuda and t.dtype == torch.bfloat16 and (t.dim() == 1 or t.stride(1) == 1)
    return ctypes.c_void_p(t.data_ptr())


def launch(a, w, c, bias=None, res=None, act=vn.ACT_NONE, bn=0, cl=0, M=None, N=None, K=None, lda=None,
           ldw=None, ldc=None, ldr=None):
    """vcl_op_gemm_ex on row-strided views (pitches from the views unless given)"""
    M = a.shape[0] if M is None else M
    K = a.shape[1] if K is None else K
    N = w.shape[0] if N is None else N
    lda = a.stride(0) if lda is None else lda
    ldw = w.stride(0) if ldw is None else ldw
    ldc = c.stride(0) if ldc is None else ldc
    ldr = (res.stride(0) if res is not None else 0) if ldr is None else ldr
    vn.check(vn.lib().vcl_op_gemm_ex(_p(a), lda, _p(w), ldw, _p(c), ldc, _p(bias), _p(res), ldr, M, N, K, act,
                                     bn, cl, vn.cur_stream()))


def nan_view(t, top=1, bottom=2, pad_cols=24):
    """t copied into a NaN buffer (the A / W poisoning)"""
    buf, v = G.padded(t.shape[0], t.shape[1], top, bottom, pad_cols, NAN, DEV)
    v.copy_(t)
    return buf, v


def nan_bias(b, pad=16):
    buf = torch.full((b.numel() + pad,), NAN, dtype=torch.bfloat16, device=DEV)
    buf[:b.numel()] = b
    return buf[:b.numel()]


def out_view(M, n_out, pad_cols=8, top=2, bottom=2, init=None):
    """a C (or residual) view inside a SENTINEL buffer, holding `init` if given"""
    buf, v = G.padded(M, n_out, top, bottom, pad_cols, G.SENTINEL, DEV)
    if init is not None:
        v.copy_(init)
    return buf, v


def _pool(rows, cols, lim, seed, exp=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    v = torch.randint(-lim, lim + 1, (rows, cols), generator=g, device=DEV, dtype=torch.int32).double()
    return (v * 2.0 ** exp).bfloat16()


class Failures:
    """per-launch 0-d count tensors (wrong elements, changed margin elements[, changed residual elements]), read back
    once at the end (no host synchronisation per launch)"""

    def __init__(self):
        self.items = []

    def add(self, what, counts):
        self.items.append((what, torch.stack([c.reshape(()) for c in counts])))

    def check(self, title):
        if not self.items:
            return
        counts = torch.stack([c for _, c in self.items]).cpu().tolist()
        bad = [(what, c) for (what, _), c in zip(self.items, counts) if any(c)]
        msg = [f"{what}: {c}" for what, c in bad[:SHOW]]
        assert not bad, f"{title}: {len(bad)} of {len(counts)} launches wrong; first: " + " | ".join(msg)


# ------------------------------------------------------------------------------------------------
# the edge sweep
@pytest.mark.parametrize("bn,cl", SWEEP, ids=[f"bn{bn}-cl{cl}" for bn, cl in SWEEP])
def test_gemm_edges_exact(bn, cl):
    ns, ks = edge_n(bn), edge_k(bn)
    Mx, Nx, Kx = max(EDGE_M), max(ns), max(ks)
    for K in ks:
        G.exact_bound(K)
    A = _pool(Mx, Kx, G.A_MAX, seed=bn + cl)
    W = _pool(Nx, Kx, G.W_MAX, seed=bn * 3 + cl)
    B = _pool(1, Nx, G.BIAS_MAX, seed=bn * 5 + cl)[0]
    RES = _pool(Mx, Nx, G.RES_MAX, seed=bn * 7 + cl)
    fails, refused = Failures(), []
    z = torch.zeros((), dtype=torch.int64, device=DEV)
    for K in ks:
        for N in ns:
            w_buf, w = nan_view(W[:N, :K], top=2, bottom=1, pad_cols=40)
            bias = nan_bias(B[:N])
            for M in EDGE_M:
                a_buf, a = nan_view(A[:M, :K], top=1, bottom=2, pad_cols=24)
                res = RES[:M, :N]
                y = G.gemm_exact(a, w)
                yb = y + bias.double()
                tag = f"M={M} N={N} K={K}"
                try:
                    c_buf, c = out_view(M, N)
                    launch(a, w, c, bn=bn, cl=cl)
                    fails.add(f"{tag} plain", (*G.buffer_check(c_buf, c, G.plain_out(y)), z))
                    c_buf, c = out_view(M, N, pad_cols=16)
                    launch(a, w, c, bias, bn=bn, cl=cl)
                    fails.add(f"{tag} bias", (*G.buffer_check(c_buf, c, G.plain_out(yb)), z))
                    c_buf, c = out_view(M, N, init=res)                       # residual updated in place
                    launch(a, w, c, bias, res=c, bn=bn, cl=cl)
                    fails.add(f"{tag} bias+residual in place", (*G.buffer_check(c_buf, c, G.plain_out(yb, res)), z))
                    r_buf, r = out_view(M, N, pad_cols=40, top=1, bottom=1, init=res)   # ldr = ldc + 32
                    c_buf, c = out_view(M, N)
                    launch(a, w, c, res=r, bn=bn, cl=cl)
                    fails.add(f"{tag} separate residual", (*G.buffer_check(c_buf, c, G.plain_out(y, res)),
                                                           sum(G.buffer_check(r_buf, r, res))))
                except vn.VclError as e:
                    refused.append(f"{tag}: {e}")
    assert not refused, f"bn={bn} cl={cl}: {len(refused)} shapes refused; first: {refused[:SHOW]}"
    fails.check(f"bn={bn} cl={cl}")


@pytest.mark.parametrize("bn,cl", SWEEP, ids=[f"bn{bn}-cl{cl}" for bn, cl in SWEEP])
def test_gemm_views_match_contiguous(bn, cl):
    """the pitch does not change the arithmetic: a ragged case through poisoned views and through contiguous
    tensors (vn.op_gemm) gives the same bits, and both are exact"""
    M, N, K = 383, 3 * bn - 32, 64 * (STAGES[bn] + 1)
    a, w, b, r = G.operands(M, N, K, seed=bn + 11 * cl, device=DEV, bias=True, res_cols=N)
    ref = G.plain_out(G.gemm_exact(a, w, b), r)
    contiguous = vn.op_gemm(a, w, b, r.clone(), vn.ACT_NONE, bn, out=r.clone(), cluster=cl)
    _, av = nan_view(a)
    _, wv = nan_view(w, top=3, bottom=0, pad_cols=64)
    rbuf, rv = out_view(M, N, pad_cols=24, init=r)
    cbuf, cv = out_view(M, N)
    launch(av, wv, cv, nan_bias(b), res=rv, bn=bn, cl=cl)
    torch.cuda.synchronize()
    assert torch.equal(cv.view(torch.int16), contiguous.view(torch.int16))
    assert int(G.same_bits(contiguous, ref).logical_not().sum()) == 0
    assert [int(x) for x in G.buffer_check(cbuf, cv, ref)] == [0, 0]
    assert [int(x) for x in G.buffer_check(rbuf, rv, r)] == [0, 0]


# ------------------------------------------------------------------------------------------------
# the K-addressing probe
def _probe_report(out, exp_k, j_of, K, what):
    """the first wrong elements, each with the column its value is the code of"""
    bad = (~G.same_bits(out, exp_k[1])).nonzero()
    if bad.numel() == 0:
        return None
    items = []
    for m, n in bad[:SHOW].tolist():
        j = j_of(m, n)
        got = int(G.probe_decode(out[m, n].reshape(1), j, K)[0])
        want = int(exp_k[0][m, n])
        items.append(f"(m={m}, n={n}) k={want} got {'no code' if got < 0 else f'k={got} (k{got - want:+d})'}")
    return f"{what}: {bad.shape[0]} wrong: " + ", ".join(items)


@pytest.mark.parametrize("bn,cl", SWEEP, ids=[f"bn{bn}-cl{cl}" for bn, cl in SWEEP])
def test_gemm_k_addressing_probe(bn, cl):
    """A's row m one-hot at k(m) = (37 m + 5) mod K, M >= K (every K column, every position of the 64-column swizzle
    span and every k16 step), W[n, k] = probe_code(n, k): C[m, n] = W[n, k(m)] exactly. Transposed: W's row n
    one-hot at k(n), A[m, k] = probe_code(m, k), C[m, n] = A[m, k(n)]."""
    msgs = []
    for K in (64, 1024, 4096):
        kk = torch.arange(K, device=DEV)
        # direct
        M, N = K + 65, 3 * bn - 32
        km = G.probe_k(torch.arange(M, device=DEV), K)
        a = torch.zeros(M, K, dtype=torch.bfloat16, device=DEV)
        a[torch.arange(M, device=DEV), km] = 1.0
        w = G.probe_code(torch.arange(N, device=DEV)[:, None], kk[None, :], K)
        _, av = nan_view(a)
        _, wv = nan_view(w, pad_cols=64)
        cbuf, cv = out_view(M, N)
        launch(av, wv, cv, bn=bn, cl=cl)
        ref = w.t()[km]                                              # [M, N] = W[n, k(m)]
        rep = _probe_report(cv, (km[:, None].expand(M, N), ref), lambda m, n: n, K, f"K={K} A one-hot")
        margin = int(G.buffer_check(cbuf, cv, ref)[1])
        msgs += [rep] if rep else []
        msgs += [f"K={K} A one-hot: {margin} margin elements changed"] if margin else []
        # transposed
        M, N = 200, K + 96
        kn = G.probe_k(torch.arange(N, device=DEV), K)
        w = torch.zeros(N, K, dtype=torch.bfloat16, device=DEV)
        w[torch.arange(N, device=DEV), kn] = 1.0
        a = G.probe_code(torch.arange(M, device=DEV)[:, None], kk[None, :], K)
        _, av = nan_view(a)
        _, wv = nan_view(w, pad_cols=64)
        cbuf, cv = out_view(M, N)
        launch(av, wv, cv, bn=bn, cl=cl)
        ref = a[:, kn]                                               # [M, N] = A[m, k(n)]
        rep = _probe_report(cv, (kn[None, :].expand(M, N), ref), lambda m, n: m, K, f"K={K} W one-hot")
        margin = int(G.buffer_check(cbuf, cv, ref)[1])
        msgs += [rep] if rep else []
        msgs += [f"K={K} W one-hot: {margin} margin elements changed"] if margin else []
    assert not msgs, f"bn={bn} cl={cl}: " + " || ".join(msgs)


# ------------------------------------------------------------------------------------------------
# activations on exact pre-activations
def act_reference(kind, y):
    """(x, u, s64, ref, torch_out) of the activation on the exact pre-activation y (float64)"""
    if kind == "swiglu":
        g, u = R.bf16_rn(y[:, 0::2]), R.bf16_rn(y[:, 1::2])
        _, s64, ref = R.swiglu_ref(g, u)
        return g, u, s64, ref, R.eager("swiglu", g, u)
    x = R.bf16_rn(y)
    u, s64, ref = (R.qgelu_ref if kind == "qgelu" else R.gelu_ref)(x)
    return x, u, s64, ref, R.eager(kind, x)


class ActTally:
    """check_activation over many launches: no output outside the bar, margins intact, and at least 99 % of all
    outputs bit-identical to torch's eager op (the bar of test_decode_epilogues_gpu.test_gemm_activation_every_input)"""

    def __init__(self):
        self.exact = self.total = 0
        self.msgs = []

    def add(self, what, c_buf, c, x, u, s64, ref, torch_out):
        m = R.check_activation(c.flatten(), u.flatten(), s64.flatten(), torch_out.flatten())
        margin = int(G.buffer_check(c_buf, c, ref)[1])
        n_bad = int(m["bad"].sum())
        if n_bad or margin:
            lines = R.describe_mismatches(m, x.flatten(), c.flatten(), torch_out.flatten(), ref.flatten(), what, n=4)
            self.msgs.append(f"{what}: {n_bad} outside the bar, {margin} margin elements changed; {lines[-1]}")
        self.exact += int(m["exact"].sum())
        self.total += c.numel()

    def check(self, title):
        assert not self.msgs, f"{title}: " + " || ".join(self.msgs[:SHOW])
        assert self.exact >= 0.99 * self.total, f"{title}: only {self.exact}/{self.total} bit-identical to torch"


ACT_KINDS = {"qgelu": vn.ACT_QGELU, "gelu": vn.ACT_GELU, "swiglu": vn.ACT_SWIGLU}


@pytest.mark.parametrize("bn", [256, 128, 64, 32])
def test_gemm_activations_at_edges(bn):
    """QGELU and GELU with bias at ragged M and N, SwiGLU (n_out = N / 2) at ragged N. W and the bias carry a scale of
    2^-3, so the exact pre-activations spread over the activations' curved range."""
    tally = ActTally()
    for kind, act in ACT_KINDS.items():
        for M in (1, 65, 200):
            for N in sorted({bn + 32, 3 * bn - 32}):
                K = 64 * (STAGES[bn] + 1)
                a, w, b, _ = G.operands(M, N, K, seed=M + N + act, device=DEV, bias=kind != "swiglu", w_exp=-3)
                y = G.gemm_exact(a, w, b)
                x, u, s64, ref, torch_out = act_reference(kind, y)
                _, av = nan_view(a)
                _, wv = nan_view(w)
                c_buf, c = out_view(M, ref.shape[1])
                launch(av, wv, c, nan_bias(b) if b is not None else None, act=act, bn=bn, cl=1)
                tally.add(f"{kind} M={M} N={N} K={K}", c_buf, c, x, u, s64, ref, torch_out)
    tally.check(f"bn={bn}")


# ------------------------------------------------------------------------------------------------
# the engine's call sites (vcl_api.cu), at its pitches: A [M, K] at pitch K, W [N, K] at pitch K, C at pitch
# n_out, the residual = C (updated in place)
def _vit(px, frames):
    P = (px // 14) ** 2
    M = frames * (P + 1)
    t = f"vit{px}x{frames}"
    return [(f"{t}_qkv", M, 3072, 1024, "bias"), (f"{t}_out", M, 1024, 1024, "bias+res"),
            (f"{t}_fc1", M, 4096, 1024, "bias+qgelu"), (f"{t}_fc2", M, 1024, 4096, "bias+res"),
            (f"{t}_patch", frames * P, 1024, 640, "patch")]


def _llm(width, M):
    D, F = {"7b": (4096, 11008), "13b": (5120, 13824)}[width]
    t = f"{width}m{M}"
    return [(f"{t}_qkv", M, 3 * D, D, ""), (f"{t}_o", M, D, D, "res"), (f"{t}_gateup", M, 2 * F, D, "swiglu"),
            (f"{t}_down", M, D, F, "res")]


SITES = (_vit(224, 1) + _vit(224, 8) + _vit(336, 1) + _vit(336, 8)
         + [(f"proj_linear_m{M}", M, 4096, 1024, "bias") for M in (356, 712)]
         + [(f"proj_mlp2x_fc{i}_m{M}", M, 4096, 1024 if i == 0 else 4096, "bias+gelu" if i == 0 else "bias")
            for M in (356, 712) for i in (0, 1)]
         + _llm("7b", 448) + _llm("7b", 709) + _llm("13b", 448) + _llm("13b", 709)
         + [(f"decode_m{M}_{n.split('_', 1)[1]}", M, N, K, e) for M in (65, 70) for n, _, N, K, e in _llm("7b", M)]
         + [("lm_head_chunk", 768, 32256, 4096, "lm_head:0"), ("lm_head_last", 200, 32256, 4096, "lm_head:768")])


def _site_operands(M, N, K, epi, seed):
    """(A view, W view, bias, residual, act): A and W at pitch K with NaN rows around them"""
    a = _pool(M, K, G.A_MAX, seed)
    w = _pool(N, K, G.W_MAX, seed + 1, exp=-3 if "gelu" in epi or "swiglu" in epi else 0)
    bias = _pool(1, N, G.BIAS_MAX, seed + 2, exp=-3 if "gelu" in epi else 0)[0] if "bias" in epi else None
    act = next((v for k, v in ACT_KINDS.items() if k in epi), vn.ACT_NONE)
    n_out = N // 2 if act == vn.ACT_SWIGLU else N
    res = _pool(M, n_out, G.RES_MAX, seed + 3) if "res" in epi else None
    if epi == "patch":                         # im2col: 3 * 14 * 14 = 588 real columns, KP = 640, zero pads
        a[:, 588:] = 0
        w[:, 588:] = 0
    _, av = nan_view(a, pad_cols=0)
    if epi.startswith("lm_head"):              # vocabulary rows 32000.. of the padded lm_head are zero; the chunk's
        w[32000:] = 0                          # A starts at row r0 of the final-norm rows
        r0 = int(epi.split(":")[1])
        prev = _pool(r0, K, G.A_MAX, seed + 4)
        _, full = nan_view(torch.cat([prev, a]), pad_cols=0)
        av = full[r0:]
    _, wv = nan_view(w, top=2, bottom=2, pad_cols=0)
    return av, wv, bias, res, act


@pytest.mark.parametrize("name,M,N,K,epi", SITES, ids=[s[0] for s in SITES])
def test_gemm_engine_call_sites(name, M, N, K, epi):
    G.exact_bound(K)
    av, wv, bias, res, act = _site_operands(M, N, K, epi, seed=M * 3 + N + K)
    y = G.gemm_exact(av, wv, bias)
    kind = next((k for k, v in ACT_KINDS.items() if v == act), None)
    if kind is None:
        ref = G.plain_out(y, res)
    else:
        x, u, s64, ref, torch_out = act_reference(kind, y)
    del y
    n_out = ref.shape[1]

    def run(bn, cl):
        c_buf, c = out_view(M, n_out, pad_cols=0, init=res)
        launch(av, wv, c, bias, res=c if res is not None else None, act=act, bn=bn, cl=cl)
        return c_buf, c

    c_buf, auto = run(0, 0)
    if kind is None:
        wrong, margin = (int(v) for v in G.buffer_check(c_buf, auto, ref))
        assert wrong == 0 and margin == 0, f"{name} auto: {wrong} wrong, {margin} margin elements changed"
    else:
        tally = ActTally()
        tally.add(f"{name} auto", c_buf, auto, x, u, s64, ref, torch_out)
        tally.check(name)
        ref = auto                                    # exact pre-activations: every tile gives these bits
    fails = Failures()
    for bn, cl in TILES:
        c_buf, c = run(bn, cl)
        fails.add(f"block_n={bn} cluster={cl}", G.buffer_check(c_buf, c, ref))
    fails.check(name)


# ------------------------------------------------------------------------------------------------
# refusals
VM, VN, VK = 130, 96, 128          # the valid call every refusal test varies


def _valid():
    """(a, w, bias, residual, C, wide): a valid problem, and a zero buffer to cut misaligned views from"""
    a, w, b, r = G.operands(VM, VN, VK, seed=5, device=DEV, bias=True, res_cols=VN)
    wide = torch.zeros(VM + 1, 2 * VK + 64, dtype=torch.bfloat16, device=DEV)
    return a, w, b, r, torch.empty(VM, VN, dtype=torch.bfloat16, device=DEV), wide


# name, the error's words, the arguments that differ from the valid call (from _valid's tensors t)
REFUSALS = [
    ("empty", "empty problem", lambda t: dict(M=0)),
    ("k_not_x64", "multiple of 64", lambda t: dict(K=96)),
    ("n_not_x32", "multiple of 32", lambda t: dict(N=48)),
    ("lda_not_x8", "pitches must be x8", lambda t: dict(lda=VK + 4)),
    ("ldc_not_x8", "pitches must be x8", lambda t: dict(ldc=VN + 2)),
    ("lda_below_k", "pitches must cover a row", lambda t: dict(lda=VK - 64)),
    ("ldc_below_n", "pitches must cover a row", lambda t: dict(ldc=VN - 32)),
    ("ldr_below_n", "pitches must cover a row", lambda t: dict(res=t[3], ldr=VN - 32)),
    ("a_misaligned", "16-byte aligned", lambda t: dict(a=t[5][:VM, 1:VK + 1])),
    ("c_misaligned", "16-byte aligned", lambda t: dict(c=t[5].view(-1)[4:4 + VM * VN].view(VM, VN))),
    ("res_misaligned", "residual must be 16-byte aligned",
     lambda t: dict(res=t[5].view(-1)[2:2 + VM * VN].view(VM, VN))),
    ("res_ld_not_x8", "residual must be 16-byte aligned", lambda t: dict(res=t[3], ldr=VN + 4)),
    ("bias_misaligned", "bias alignment", lambda t: dict(bias=t[5][0, 2:2 + VN])),
    ("swiglu_residual", "swiglu takes no residual",
     lambda t: dict(act=vn.ACT_SWIGLU, c=t[4][:, :VN // 2], res=t[3])),
    ("cluster_3", "cluster must be 1, 2 or 4", lambda t: dict(cl=3)),
    ("cluster_8", "cluster must be 1, 2 or 4", lambda t: dict(cl=8, bn=128)),
    ("block_n_96", "unsupported block_n", lambda t: dict(bn=96)),
    ("unknown_act", "unknown activation", lambda t: dict(act=7, bn=128)),
    ("rope_without_tables", "ACT_ROPE needs the RoPE tables", lambda t: dict(act=ACT_ROPE, bn=128)),
]


@pytest.mark.parametrize("which,msg,change", REFUSALS, ids=[x[0] for x in REFUSALS])
def test_gemm_refusals(which, msg, change):
    """each refusal of launch_gemm_bf16_tn names its cause and launches nothing; a valid call afterwards runs and is
    exact. (ACT_ROPE's tile-width refusal needs the RoPE tables, which only the engine passes.)"""
    t = _valid()
    a, w, b, _, c, _ = t
    args = dict(a=a, w=w, c=c, bias=b, res=None, act=vn.ACT_NONE, bn=0, cl=0)
    args.update(change(t))
    n0 = vn.launch_count()
    with pytest.raises(vn.VclError, match=msg):
        launch(**args)
    assert vn.launch_count() == n0, f"{which}: a refused call launched a kernel"
    out = torch.full_like(c, NAN)
    launch(a, w, out, b)
    torch.cuda.synchronize()
    assert vn.launch_count() == n0 + 1
    assert int(G.same_bits(out, G.plain_out(G.gemm_exact(a, w, b))).logical_not().sum()) == 0
