"""The SwiGLU and logits epilogues of the decode projections (decode_gemv.cu, through vcl_op_gemv_ex), and the
activation epilogues over every finite bf16 input.

- SwiGLU against fp64 at 1..64 clips: row-major out at 1..4 clips, the xwin layout at 5..64 (pre-filled with a NaN
  sentinel that every element outside the B x N/2 outputs must keep), row slices at 17..64 clips on the 7B / 13B
  gate|up shapes. Inputs normalised as the engine does: the fused RMSNorm at 1..4 clips, xwin_norm above. The
  normalised operand is checked against fp64 (_operand), the projection and its epilogue against fp64 on that
  operand, with every bf16 rounding point of the reference.
  Bars: 2.5 bf16 ulps of max(|ref|, (|g| + 1) |u|) (test_kernels_gpu._gemm_ref), >= 99 % bit-identical.
- Logits against fp64 (N = 32003: a last 16-row group of 3 rows), within 2.5 ulps and >= 99 % bit-identical; at
  1..4 clips every per-CTA arg-max partial is the (value, lowest row) maximum of the kernel's own logits over that
  CTA's rows, the partials reduce to the first arg-max, and a partials-only launch gives the same partials.
- Exact ties: one-hot activations make every logit exactly one weight; the lowest tied row must win everywhere.
- fp8 weights: SwiGLU and logits equal the bf16 launch on W~ bit for bit (partials included).
- Every finite bf16 gate through the GEMV SwiGLU epilogue, and every finite bf16 input through the GEMM's SwiGLU,
  quick-GELU and GELU epilogues, against the fp64 references of _act_ref.py (the bar is written there).
- A 0-layer engine's decode step (embedding -> final norm -> lm_head) at 1..70 clips, and the GEMM at decode widths
  above 64 clips (every tile / cluster bit-identical to the automatic choice)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
import _act_ref as R  # noqa: E402
from _util import make_engine  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from test_gemm_schedule_gpu import TILES  # noqa: E402
from test_kernels_gpu import _describe, _gemm_ref, _rel  # noqa: E402

DEV = "cuda"
EPS = 1e-5
SENTINEL = 0x7FC1          # a bf16 NaN bit pattern no kernel produces
SWIGLU_B = [1, 2, 3, 4, 5, 9, 16, 17, 32, 33, 48, 64]
SWIGLU_SHAPES = [(2048, 512), (13824, 2560), (22016, 4096), (27648, 5120), (2000, 1024)]
LOGIT_B = [1, 2, 3, 4, 5, 16, 17, 33, 64]
VOCAB = 32003


def _bits(t):
    return t.contiguous().view(torch.int16)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, seed, std=1.0):
    return (torch.randn(*shape, generator=_gen(seed), device=DEV) * std).bfloat16()


def _operand(x, nw, chunks=None):
    """The normalised rows the projection kernels read, taken from the kernels themselves (a RES launch on the
    identity matrix returns its operand exactly), checked against the fp64 normalisation w * bf16(x * rstd): equal,
    but for a few elements whose bf16(x * rstd) is a neighbour of the fp64 one. rstd is an fp32 number in the kernels
    (LlamaRMSNorm computes it in fp32 too), so x * rstd may round the other way next to a rounding boundary, and one
    such element of a large x moves every output of its row by many of the small outputs' ulps. The projection is
    then checked on the operand it read. chunks: the row blocks launched together (the engine's split above 64
    clips)."""
    B, K = x.shape
    eye = torch.eye(K, device=DEV).bfloat16()
    chunks = chunks or [(0, B)]
    got = torch.cat([vn.op_gemv_ex(x[b0:b1].contiguous(), eye, vn.GEMV_RES, norm_w=nw, eps=EPS) for b0, b1 in chunks])
    xd = x.double()
    xn = R.bf16_rn(xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + EPS))
    want = R.bf16_rn(nw.double() * xn.double())
    off = got.view(torch.int16) != want.view(torch.int16)
    flipped = torch.zeros_like(off)
    for c in R.bf16_neighbours(xn):
        flipped |= got.view(torch.int16) == R.bf16_rn(nw.double() * c.double()).view(torch.int16)
    assert not (off & ~flipped).any(), f"normalised rows: {int((off & ~flipped).sum())} elements off the fp64 ones"
    assert off.float().mean().item() <= 1e-3, f"normalised rows: {int(off.sum())} elements rounded the other way"
    return got


def _assert_close(out, ref, mag, what):
    """out / ref bf16 values (any float dtype): within 2.5 bf16 ulps of mag, >= 99 % bit-identical"""
    o, r = out.float(), ref.float()
    assert torch.isfinite(o).all(), f"{what}: non-finite outputs"
    ulp = mag.float().clamp_min(1e-2) * 2 ** -7
    bad = (o - r).abs() > 2.5 * ulp
    assert not bad.any(), (f"{what}: {int(bad.sum())} outputs beyond 2.5 ulps, first at {bad.nonzero()[:4].tolist()}: "
                           f"got {o[bad][:4].tolist()} want {r[bad][:4].tolist()}")
    same = (o == r).float().mean().item()
    print(f"[epilogues] {what}: bit-identical {same:.5f}")
    assert same >= 0.99, f"{what}: only {same:.4f} bit-identical"


def _swiglu_out(out, B, F):
    """the [B, F] outputs of a SwiGLU launch; at 5..64 clips the xwin buffer must keep the sentinel elsewhere"""
    if B <= 4:
        return out
    rows, unused = R.xwin_unpack(out, B, F)
    n = int((_bits(out)[unused] != SENTINEL).sum())
    assert n == 0, f"B={B} F={F}: {n} xwin elements written outside the outputs"
    return rows


def _swiglu_launch(x, w, B, N, fp8=False, norm_w=None):
    F = N // 2
    out = None
    if B > 4:
        out = torch.full((R.xwin_elems(B, F),), SENTINEL, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    out = vn.op_gemv_ex(x, w, vn.GEMV_SWIGLU, fp8=fp8, norm_w=norm_w, eps=EPS, out=out)
    return _swiglu_out(out, B, F)


# ------------------------------------------------------------------------------------------------
# SwiGLU against fp64
@pytest.mark.parametrize("N,K", SWIGLU_SHAPES)
def test_swiglu_epilogue(N, K):
    w = _randn(N, K, seed=N + K, std=K ** -0.5)
    nw = (1 + 0.1 * torch.randn(K, generator=_gen(K), device=DEV)).bfloat16()
    wd = w.double()
    for B in SWIGLU_B:
        x = _randn(B, K, seed=B * 1000 + K, std=2.0)
        out = _swiglu_launch(x, w, B, N, norm_w=nw)
        y = _operand(x, nw).double() @ wd.t()
        g, u = R.bf16_rn(y[:, 0::2]), R.bf16_rn(y[:, 1::2])
        _, s, ref = R.swiglu_ref(g, u)
        mag = torch.maximum(ref.double().abs(), (g.double().abs() + 1) * u.double().abs())
        _assert_close(out, ref, mag, f"swiglu B={B} N={N} K={K}")


# ------------------------------------------------------------------------------------------------
# logits and the per-CTA arg-max partials
def _partials_of(logits):
    """per-CTA (value, lowest row) maxima of [B, N] logits, [grid, B] each"""
    B, N = logits.shape
    vals, idxs = [], []
    for r0, n in R.cta_row_groups(N, vn.gemv_grid(N)):
        seg = logits[:, r0:r0 + n]
        m = seg.max(dim=1).values
        first = (seg == m[:, None]).int().argmax(dim=1) + r0       # argmax of a 0/1 row: its first 1
        vals.append(m)
        idxs.append(first)
    return torch.stack(vals), torch.stack(idxs).int()


def _check_partials(lg, pt, what):
    """pt [grid, B, 2] int32 (value bits, row) of the kernel against the kernel's own logits lg [B, N]"""
    v, i = _partials_of(lg)
    got_v = pt[..., 0].contiguous().view(torch.float32)
    assert torch.equal(got_v.view(torch.int32), v.contiguous().view(torch.int32)) and torch.equal(pt[..., 1], i), \
        f"{what}: partials differ from the per-CTA maxima of the logits"
    # the reduction the next step's q|k|v kernel does: largest value, lowest row among equals
    best = got_v.max(dim=0).values
    tok = torch.where(got_v == best, pt[..., 1], torch.full_like(pt[..., 1], 2 ** 31 - 1)).min(dim=0).values
    assert torch.equal(tok.long(), lg.argmax(dim=1)), f"{what}: reduced partials {tok.tolist()} != first arg-max"
    return tok


def _logits_launch(x, w, B, fp8=False, norm_w=None):
    lg, pt = vn.op_gemv_ex(x, w, vn.GEMV_LOGITS, fp8=fp8, norm_w=norm_w, eps=EPS, partials=B <= 4)
    return lg, pt


@pytest.mark.parametrize("K", [4096, 5120])
def test_logits_epilogue(K):
    w = _randn(VOCAB, K, seed=K, std=K ** -0.5)
    nw = (1 + 0.1 * torch.randn(K, generator=_gen(K + 1), device=DEV)).bfloat16()
    wd = w.double()
    for B in LOGIT_B:
        x = _randn(B, K, seed=B * 7 + K)
        lg, pt = _logits_launch(x, w, B, norm_w=nw)
        assert torch.equal(lg, lg.bfloat16().float()), "logits must be bf16 values"
        y = _operand(x, nw).double() @ wd.t()
        _assert_close(lg, R.bf16_rn(y), y.abs(), f"logits B={B} K={K}")
        if B <= 4:
            _check_partials(lg, pt, f"B={B} K={K}")
            _, pt2 = vn.op_gemv_ex(x, w, vn.GEMV_LOGITS, norm_w=nw, eps=EPS, logits=False, partials=True)
            assert torch.equal(pt, pt2), f"B={B} K={K}: a partials-only launch gives other partials"


# ------------------------------------------------------------------------------------------------
# exact ties: x_b = e_{k_b} (no norm), so logit n of clip b is exactly W[n, k_b]
def _tie_rows(kind):
    """rows holding the tied maximum of one placement (None: every row)"""
    parts = R.cta_row_groups(VOCAB, vn.gemv_grid(VOCAB))
    r0, n = parts[5]
    return {"group": [16 * 40 + 11, 16 * 40 + 3],          # one 16-row group, both halves
            "warps": [r0 + 40, r0 + 5],                    # one CTA, warps 1 and 0 of its arg-max loop
            "ctas": [parts[9][0] + 7, parts[3][0] + 2],    # two CTAs
            "ends": [VOCAB - 1, 0],
            "all": None}[kind]


TIE_KINDS = ["group", "warps", "ctas", "ends", "all"]


@pytest.mark.parametrize("B", [1, 2, 3, 4, 5, 17])
def test_logit_ties_take_the_lowest_row(B):
    K = 4096
    w = _randn(VOCAB, K, seed=99, std=0.05)
    cols = [7 + 61 * j for j in range(len(TIE_KINDS))]
    for j, kind in enumerate(TIE_KINDS):
        rows = _tie_rows(kind)
        if rows is None:
            w[:, cols[j]] = 0.5
        else:
            w[rows, cols[j]] = 1.0
    for shift in range(len(TIE_KINDS) if B < len(TIE_KINDS) else 1):
        which = [(b + shift) % len(TIE_KINDS) for b in range(B)]
        x = torch.zeros(B, K, dtype=torch.bfloat16, device=DEV)
        x[torch.arange(B), torch.tensor([cols[j] for j in which])] = 1.0
        lg, pt = _logits_launch(x, w, B)
        want = w[:, [cols[j] for j in which]].t().float()
        assert torch.equal(lg, want), f"B={B} {[TIE_KINDS[j] for j in which]}: one-hot logits are not exact"
        first = [0 if _tie_rows(TIE_KINDS[j]) is None else min(_tie_rows(TIE_KINDS[j])) for j in which]
        assert lg.argmax(dim=1).tolist() == first
        if B <= 4:
            assert _check_partials(lg, pt, f"ties B={B}").tolist() == first


# ------------------------------------------------------------------------------------------------
# fp8 weights: bit for bit the bf16 launch on W~
@pytest.mark.parametrize("mode", ["swiglu", "logits"])
def test_fp8_equals_bf16_on_dequantized_weights(mode):
    N, K = (22016, 4096) if mode == "swiglu" else (VOCAB, 4096)
    w = _randn(N, K, seed=N, std=K ** -0.5)
    deq = vn.op_quantize_fp8(w)[0]
    nw = (1 + 0.1 * torch.randn(K, generator=_gen(3), device=DEV)).bfloat16()
    for B in [1, 4, 5, 17, 33, 64]:
        x = _randn(B, K, seed=B + 5)
        if mode == "swiglu":
            a, b = _swiglu_launch(x, w, B, N, fp8=True, norm_w=nw), _swiglu_launch(x, deq, B, N, norm_w=nw)
            assert torch.equal(_bits(a), _bits(b)), f"swiglu B={B}: fp8 != bf16 on W~"
        else:
            (la, pa), (lb, pb) = _logits_launch(x, w, B, fp8=True, norm_w=nw), _logits_launch(x, deq, B, norm_w=nw)
            assert torch.equal(la.view(torch.int32), lb.view(torch.int32)), f"logits B={B}: fp8 != bf16 on W~"
            if B <= 4:
                assert torch.equal(pa, pb), f"partials B={B}: fp8 != bf16 on W~"


# ------------------------------------------------------------------------------------------------
# every finite bf16 input through the activation epilogues
def _assert_activation(out, x, u, s64, ref, torch_out, what):
    m = R.check_activation(out, u, s64, torch_out)
    for line in R.describe_mismatches(m, x, out, torch_out, ref, what):
        print("[epilogues]", line)
    same = m["exact"].float().mean().item()
    print(f"[epilogues] {what}: bit-identical to torch's eager op {same:.5f}")
    assert not m["bad"].any(), f"{what}: {int(m['bad'].sum())} outputs outside the bar"
    assert same >= 0.99, f"{what}: only {same:.4f} bit-identical to torch"


# (B, F): the 1..4-clip kernel, and the 5..64-clip kernel with 1, 2 and 4 clip groups; the last is row-sliced
SWEEP_LAUNCHES = [(2, 32640), (16, 4080), (32, 2040), (64, 8192)]


@pytest.mark.parametrize("up", ["one", "random"])
@pytest.mark.parametrize("B,F", SWEEP_LAUNCHES)
def test_gemv_swiglu_every_gate(B, F, up):
    """x_b = e_{k_b} and W[2j, k_b] = g: the projection is exact, so every finite bf16 gate reaches the epilogue
    as it is; clip b, output j takes gate number b * F + j (cycled when B * F > 65280)."""
    K = 256
    if B == 64 and F == 8192:
        assert 2 * F // 16 > 6 * torch.cuda.get_device_properties(0).multi_processor_count, "not row-sliced"
    vals = R.all_finite_bf16().to(DEV)
    n = B * F
    assert n >= vals.numel()
    gates = vals[torch.arange(n, device=DEV) % vals.numel()].view(B, F)
    ups = torch.ones_like(gates) if up == "one" else _randn(B, F, seed=B + F)
    cols = torch.arange(B, device=DEV) * 3 + 1
    w = torch.zeros(2 * F, K, dtype=torch.bfloat16, device=DEV)
    for b in range(B):
        w[0::2, cols[b]] = gates[b]
        w[1::2, cols[b]] = ups[b]
    x = torch.zeros(B, K, dtype=torch.bfloat16, device=DEV)
    x[torch.arange(B, device=DEV), cols] = 1.0
    out = _swiglu_launch(x, w, B, 2 * F).flatten()
    g, u = gates.flatten(), ups.flatten()
    _, s64, ref = R.swiglu_ref(g, u)
    _assert_activation(out, g, u, s64, ref, R.eager("swiglu", g, u), f"gemv swiglu B={B} F={F} up={up}")


@pytest.mark.parametrize("kind", ["swiglu", "swiglu_up", "qgelu", "gelu"])
def test_gemm_activation_every_input(kind):
    """A = I_128 (M = K = 128), so y = W^T exactly: y[m, n] = W[n, m] covers every finite bf16 value"""
    vals = R.all_finite_bf16().to(DEV)
    eye = torch.eye(128, device=DEV).bfloat16()
    n_out = 512
    xs = vals[torch.arange(128 * n_out, device=DEV) % vals.numel()].view(128, n_out)    # [m, output column]
    if kind.startswith("swiglu"):
        ups = torch.ones_like(xs) if kind == "swiglu" else _randn(128, n_out, seed=77)
        w = torch.empty(2 * n_out, 128, dtype=torch.bfloat16, device=DEV)
        w[0::2] = xs.t()
        w[1::2] = ups.t()
        out = vn.op_gemm(eye, w, None, None, vn.ACT_SWIGLU)
        x, u = xs.flatten(), ups.flatten()
        _, s64, ref = R.swiglu_ref(x, u)
        torch_out = R.eager("swiglu", x, u)
    else:
        out = vn.op_gemm(eye, xs.t().contiguous(), None, None, vn.ACT_QGELU if kind == "qgelu" else vn.ACT_GELU)
        x = xs.flatten()
        u, s64, ref = (R.qgelu_ref if kind == "qgelu" else R.gelu_ref)(x)
        torch_out = R.eager(kind, x)
    torch.cuda.synchronize()
    _assert_activation(out.flatten(), x, u, s64, ref, torch_out, f"gemm {kind}")


# ------------------------------------------------------------------------------------------------
# a 0-layer engine's decode step: embedding -> final norm -> lm_head
@pytest.fixture(scope="module")
def eng0():
    cfg = O.LlmCfg(hidden=4096, inter=11008, heads=32, layers=0)
    g = _gen(4)
    sd = {"model.embed_tokens.weight": torch.randn(VOCAB, 4096, generator=g, device=DEV).bfloat16(),
          "model.norm.weight": (1 + 0.05 * torch.randn(4096, generator=g, device=DEV)).bfloat16(),
          "lm_head.weight": (torch.randn(VOCAB, 4096, generator=g, device=DEV) * 4096 ** -0.5).bfloat16(),
          "model.mm_projector.weight": (torch.randn(4096, 1024, generator=g, device=DEV) / 32).bfloat16(),
          "model.mm_projector.bias": torch.zeros(4096, device=DEV).bfloat16()}
    eng = make_engine(llm=cfg, max_batch=70, max_seq=64)
    eng.load_llm(sd)
    return eng, sd


@pytest.mark.parametrize("B", [1, 4, 5, 64, 65, 70])
def test_decode_step_logits(eng0, B):
    eng, sd = eng0
    tok = torch.randint(0, VOCAB, (B,), generator=_gen(B), device=DEV, dtype=torch.int32)
    lg, out_tok = eng.decode_step(tok, 3, want_logits=True)
    torch.cuda.synchronize()
    n = (B + 15) // 16                                   # lm_head_argmax: chunks of the 5..16-clip kernel above 64
    chunks = [(B * i // n, B * (i + 1) // n) for i in range(n)] if B > 64 else None
    y = _operand(sd["model.embed_tokens.weight"][tok.long()], sd["model.norm.weight"], chunks).double() @ \
        sd["lm_head.weight"].double().t()
    _assert_close(lg, R.bf16_rn(y), y.abs(), f"decode step B={B}")
    assert torch.equal(out_tok.long(), lg.argmax(dim=1)), f"B={B}: the token is not the first arg-max"


# ------------------------------------------------------------------------------------------------
# the GEMM at decode widths above 64 clips
GEMM_CASES = [("gate_up", 22016, 4096, vn.ACT_SWIGLU, False), ("down", 4096, 11008, vn.ACT_NONE, True),
              ("qkv", 12288, 4096, vn.ACT_NONE, False)]


@pytest.mark.parametrize("M", [65, 100, 128])
@pytest.mark.parametrize("name,N,K,act,has_res", GEMM_CASES, ids=[c[0] for c in GEMM_CASES])
def test_gemm_above_64_clips(name, N, K, act, has_res, M):
    a = _randn(M, K, seed=M + N)
    w = _randn(N, K, seed=N + K, std=K ** -0.5)
    n_out = N // 2 if act == vn.ACT_SWIGLU else N
    res = _randn(M, n_out, seed=M) if has_res else None

    def run(bn, cl):
        out = res.clone() if has_res else torch.full((M, n_out), float("nan"), device=DEV, dtype=torch.bfloat16)
        return vn.op_gemm(a, w, None, out if has_res else None, act, bn, out=out, cluster=cl)

    auto = run(0, 0)
    torch.cuda.synchronize()
    ref, mag = _gemm_ref(a, w, None, res, act)
    assert _rel(auto, ref) < 3e-3, _describe(auto, ref)
    assert ((auto.float() - ref).abs() <= 2.5 * mag.clamp_min(1e-2) * 2 ** -7).all(), _describe(auto, ref)
    for bn, cl in TILES:
        out = run(bn, cl)
        torch.cuda.synchronize()
        assert torch.equal(out, auto), f"{name} M={M} block_n={bn} cluster={cl}: " + _describe(out, auto.float())
