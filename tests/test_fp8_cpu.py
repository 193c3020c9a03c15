"""CPU tests of the fp8 (E4M3) LLM weight format: the torch reference quantizer (tests/_fp8_ref.py) against the rule
of include/vcl.h (exponent choice, ties to even, subnormal codes, the 448 ceiling, the zero row, W~ exact in bf16)
and the slot order, and the Python plumbing of the option with a fake engine (every rejection before any engine
exists)."""
import ctypes

import pytest
import torch

import _fp8_ref as R
import vcl_native as vn


def _row(*vals, K=32):
    w = torch.zeros(1, K)
    w[0, :len(vals)] = torch.tensor(vals)
    return w.to(torch.bfloat16)


def test_exponent_is_the_smallest_that_fits():
    for e in (-12, -7, 0, 3):
        s = 2.0 ** e
        assert R.row_exponents(_row(448 * s)).item() == e            # exactly at the ceiling: no headroom lost
        assert R.row_exponents(_row(450 * s)).item() == e + 1        # just above (the next bf16): the next power
        assert R.row_exponents(_row(-224 * s)).item() == e - 1       # 224 * 2^e = 448 * 2^(e-1)
        assert R.row_exponents(_row(225 * s)).item() == e            # lands in (224, 448]
    torch.manual_seed(1)
    w = (torch.randn(64, 256) * torch.exp2(torch.randint(-14, 2, (64, 1)).float())).bfloat16()
    q, e, _ = R.quantize(w)
    scaled = w.float().abs().amax(1) * R.pow2(-e)                        # exact
    assert (scaled > 224).all() and (scaled <= 448).all()
    amax = q.float().abs().amax(1)                                       # E4M3 rounds (224, 232) down to 224
    assert (amax >= 224).all() and (amax <= 448).all()
    # against the definition: a <= 448 * 2^e and a > 448 * 2^(e-1)
    a = w.float().abs().amax(1).double()
    assert (a <= 448 * 2.0 ** e.double()).all() and (a > 448 * 2.0 ** (e.double() - 1)).all()


def test_round_to_nearest_even_and_subnormals():
    # e = 0 (row maximum 448): E4M3 spacing is 2 in [16, 32), 2^-9 among the subnormals
    w = _row(448, 17, 19, -17, 2 ** -10, 3 * 2 ** -10, 5 * 2 ** -10, 2 ** -9, 7 * 2 ** -9, 2 ** -6, 2 ** -11)
    q, e, _ = R.quantize(w)
    assert e.item() == 0
    got = q.float()[0, :11].tolist()
    want = [448, 16, 20, -16, 0, 2 ** -8, 2 ** -8, 2 ** -9, 7 * 2 ** -9, 2 ** -6, 0]
    assert got == want
    # the scaling is exact, so a power-of-two shift of the whole row shifts the codes' exponents only
    for s in (-20, -5, 9):
        q2, e2, _ = R.quantize((w.float() * 2.0 ** s).bfloat16())
        assert e2.item() == s and torch.equal(q2.view(torch.uint8), q.view(torch.uint8))


def test_never_above_448_and_no_nan_codes():
    w = _row(447, 447.5, -448, 440, 100)
    q, e, _ = R.quantize(w)
    assert e.item() == 0 and q.float()[0, :5].tolist() == [448, 448, -448, 448, 96]
    w = torch.randn(256, 512).bfloat16()
    q, _, _ = R.quantize(w)
    assert ((q.view(torch.uint8) & 0x7F) != 0x7F).all()


def test_zero_row_and_signed_zero():
    w = torch.zeros(3, 64, dtype=torch.bfloat16)
    w[1, 5] = -0.0
    w[2, 7] = 3.0
    q, e, deq = R.quantize(w)
    assert e.tolist()[:2] == [0, 0] and (q.float()[:2] == 0).all() and (deq[:2] == 0).all()
    assert q.view(torch.uint8)[1, 5].item() == 0x80                      # -0 keeps its sign


def test_dequantized_weights_are_exact_bf16_and_close():
    torch.manual_seed(0)
    w = (torch.randn(4096, 4096) * 0.02).bfloat16()
    q, e, deq = R.quantize(w)
    exact = q.double() * torch.exp2(e.double())[:, None]
    assert torch.equal(deq.double(), exact)                              # q * 2^e is a bf16 number: nothing rounded
    rel = ((deq.float() - w.float()).norm() / w.float().norm()).item()
    print(f"[fp8] W~ relative error, Gaussian 4096 x 4096: {rel:.4f}")
    assert 0.02 < rel < 0.03


def test_every_finite_code_round_trips():
    vals = R.finite_codes()
    assert vals.numel() == 254 and vals.abs().max() == 448
    w = vals[None].bfloat16()                                            # every E4M3 value is a bf16 value
    q, e, deq = R.quantize(w)
    assert e.item() == 0 and torch.equal(q.float()[0], vals) and torch.equal(deq.float()[0], vals)


def test_slot_order():
    N, K = 37, 1056                                                      # ragged rows, a 32-k tail chunk
    off = R.slot_offsets(N, K)
    assert off.unique().numel() == N * K and off.max() < (N + 15) // 16 * 16 * K
    assert off[0, :8].tolist() == list(range(8))                         # lane 0: k 0..7 of row 0
    assert off[0, 8].item() == 8 and off[1, 0].item() == 32              # lane 1 = k 8.., lane 4 = row 1
    assert off[8, 0].item() == 256 and off[0, 32].item() == 512          # row half, next 32-k block
    assert off[0, 512].item() == 8192 and off[16, 0].item() == 16 * K    # next chunk, next row group
    q = R.quantize(torch.randn(N, K).bfloat16())[0]
    t = R.tiled_codes(q)
    assert torch.equal(t[off.reshape(-1)], q.view(torch.uint8).reshape(-1))
    unused = torch.ones(t.numel(), dtype=torch.bool)
    unused[off.reshape(-1)] = False
    assert t.numel() == 48 * K and unused.sum() == (48 - N) * K and (t[unused] == 0).all()   # rows past N: zero


def test_dequantize_state_touches_the_streamed_matrices_only():
    sd = {"model.embed_tokens.weight": torch.randn(8, 32), "model.norm.weight": torch.randn(32),
          "lm_head.weight": torch.randn(8, 32), "model.layers.0.self_attn.q_proj.weight": torch.randn(32, 32),
          "model.layers.0.mlp.down_proj.weight": torch.randn(32, 64), "model.mm_projector.weight": torch.randn(32, 16),
          "model.layers.0.input_layernorm.weight": torch.randn(32)}
    out = R.dequantize_state({k: v.bfloat16() for k, v in sd.items()})
    for k, v in out.items():
        changed = not torch.equal(v, sd[k].bfloat16())
        assert changed == (k == "lm_head.weight" or k.endswith("_proj.weight") and k.startswith("model.layers.")), k


# ---------------------------------------------------------------------------------------------
# Python plumbing
# ---------------------------------------------------------------------------------------------
def test_weight_format_codes():
    assert vn.weight_format_code("bf16") == vn.WEIGHTS_BF16 == 0
    assert vn.weight_format_code("fp8_e4m3") == vn.WEIGHTS_FP8_E4M3 == 1
    for bad in ("fp8", "FP8_E4M3", "e4m3", None, 1, "bf16 "):
        with pytest.raises(ValueError, match="unknown LLM weight format"):
            vn.weight_format_code(bad)


class _LibSpy:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append(name)
            return 0
        return fn


def test_engine_load_llm_dispatch_and_rejection(monkeypatch):
    spy = _LibSpy()
    monkeypatch.setattr(vn, "lib", lambda: spy)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda: None)
    eng = vn.Engine.__new__(vn.Engine)
    eng._h = ctypes.c_void_p()
    state = {"lm_head.weight": torch.zeros(2, 2, dtype=torch.bfloat16)}
    monkeypatch.setattr(vn, "_tensor_array", lambda st, keep: (vn.vcl_tensor * len(st))())
    eng.load_llm(state)
    eng.load_llm(state, weight_format="fp8_e4m3")
    assert spy.calls == ["vcl_load_llm_weights", "vcl_load_llm_weights_ex"]
    with pytest.raises(ValueError):
        eng.load_llm(state, weight_format="int8")
    assert len(spy.calls) == 2                                           # nothing reached the library


class _FakeEngine:
    made = []

    def __init__(self, cfg):
        self.cfg = cfg
        self.loads = []
        _FakeEngine.made.append(self)

    def load_llm(self, state, weight_format="bf16"):
        self.loads.append(weight_format)


def _model(**kw):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    cfg = VideoChatGPTConfig(hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4,
                             vocab_size=32003)
    return VideoChatGPTLlamaForCausalLM(cfg, clip_config={}, **kw)


@pytest.mark.parametrize("fmt", ["bf16", "fp8_e4m3", None])
def test_model_passes_the_format_to_the_engine(monkeypatch, fmt):
    monkeypatch.setattr(vn, "Engine", _FakeEngine)
    _FakeEngine.made.clear()
    m = _model() if fmt is None else _model(llm_weight_format=fmt)
    m._ensure_engine(need_llm=True)
    assert [e.loads for e in _FakeEngine.made] == [[fmt or "bf16"]]


def test_bad_model_format_raises_before_an_engine(monkeypatch):
    monkeypatch.setattr(vn, "Engine", _FakeEngine)
    _FakeEngine.made.clear()
    for bad in ("fp16", "int4", ""):
        with pytest.raises(ValueError, match="unknown LLM weight format"):
            _model(llm_weight_format=bad)
    assert _FakeEngine.made == []


def test_from_pretrained_and_initialize_model_pass_the_format(monkeypatch, tmp_path):
    from _checkpoint import make_tiny_checkpoint
    from video_chatgpt.eval.model_utils import initialize_model
    from video_chatgpt.model import VideoChatGPTLlamaForCausalLM
    ck = make_tiny_checkpoint(tmp_path)
    m = VideoChatGPTLlamaForCausalLM.from_pretrained(ck["model_dir"], llm_weight_format="fp8_e4m3")
    assert m._llm_weight_format == "fp8_e4m3"
    with pytest.raises(ValueError):
        VideoChatGPTLlamaForCausalLM.from_pretrained(ck["model_dir"], llm_weight_format="fp4")
    monkeypatch.setattr(vn, "Engine", _FakeEngine)
    _FakeEngine.made.clear()
    model = initialize_model(ck["model_dir"], llm_weight_format="fp8_e4m3")[0]
    assert model._llm_weight_format == "fp8_e4m3" and _FakeEngine.made == []   # the engine comes at first use
    model._ensure_engine(need_llm=True)
    assert _FakeEngine.made[-1].loads == ["fp8_e4m3"]
    with pytest.raises(ValueError):
        initialize_model(ck["model_dir"], llm_weight_format="bf8")
    assert initialize_model(ck["model_dir"])[0]._llm_weight_format == "bf16"
