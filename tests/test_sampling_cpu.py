"""CPU tests of device sampling: the Philox4x32-10 reference against its published known-answer vectors, the float64
rules on hand-made rows, and the host side of generate / generate_requests with a fake engine: the sampling-table
writes per admission, the per-request seeds, restoring greedy entries, and every rejection before any device work."""
import math

import numpy as np
import pytest
import torch

import _sampling_ref as R
from test_inflight_cpu import EOS, FakeEngine, _model, _new, _req


def test_philox_known_answers():
    words = R.philox4x32_10((0, 0), (0, 0, 0, 0))
    assert [int(w) for w in words] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    m = 0xFFFFFFFF
    words = R.philox4x32_10((m, m), (m, m, m, m))
    assert [int(w) for w in words] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    # u from word 0: 24 bits, in [0, 1)
    u = R.uniform(2 ** 64 - 1, np.arange(1000))
    assert u.min() >= 0 and u.max() < 1 and np.all(u * 2 ** 24 == np.floor(u * 2 ** 24))


def test_rules_on_small_rows():
    x = np.array([1.0, 3.0, 3.0, 2.0, -np.inf], dtype=np.float32)
    assert R.choose(x, 0.0, 0, 0.5)[0] == 1                      # greedy: the first of the tied maxima
    # top_k 1 keeps both tied maxima (HF's `scores < kth` rule), with equal weights
    assert R.kept_mask(x, 1.0, 1).tolist() == [False, True, True, False, False]
    assert R.choose(x, 1.0, 1, 0.49)[0] == 1 and R.choose(x, 1.0, 1, 0.51)[0] == 2
    # top_k 0 and top_k >= V keep every number; -inf keeps weight 0
    assert R.kept_mask(x, 1.0, 0).tolist() == R.kept_mask(x, 1.0, 7).tolist() == [True] * 5
    assert R.choose(x, 1.0, 0, 0.999999)[0] == 3
    # a non-finite scaled maximum falls back to the arg-max
    big = np.array([1.0, 3e38, 2.0], dtype=np.float32)
    assert R.choose(big, 1e-4, 0, 0.0) == (1, None)
    assert R.choose(np.full(4, -np.inf, dtype=np.float32), 0.5, 0, 0.3) == (0, None)
    assert R.argmax_rule(np.array([np.nan, 1.0, 1.0], dtype=np.float32)) == 1


class SamplingEngine(FakeEngine):
    """FakeEngine that also records the sampling-table writes"""

    def __init__(self, tokens=None):
        super().__init__(tokens)
        self.table = {}

    def set_sampling(self, clips, temperature, top_k, seed):
        self.calls.append(("sampling", list(clips), list(temperature), list(top_k), list(seed)))
        for b, t, k, s in zip(clips, temperature, top_k, seed):
            self.table[b] = (t, k, s)


def test_greedy_requests_never_touch_the_table():
    m = _model(max_batch=2, eng=SamplingEngine())
    m.generate_requests([_req(r, max_new_tokens=3) for r in range(3)], eos_token_id=None)
    assert not [c for c in m._engine.calls if c[0] == "sampling"]
    m.generate_requests([_req(0, max_new_tokens=3)], eos_token_id=None, seed=5)      # a seed alone samples nothing
    assert not [c for c in m._engine.calls if c[0] == "sampling"]


@pytest.mark.parametrize("packed", [False, True])
def test_admission_writes_the_admitted_slots_entries(packed):
    eng = SamplingEngine()
    if packed:
        def slots_prefill(slots, ids_list, feats_list, vid_starts, tok_out=None):
            eng.calls.append(("packed", list(slots)))
            out = []
            for s, ids in zip(slots, ids_list):
                r = int(torch.as_tensor(ids).reshape(-1)[0]) - 100
                eng.slot[s] = [r, 1]
                out.append(eng._tok(r, 0))
            return torch.tensor(out, dtype=torch.int32)
        eng.slots_prefill = slots_prefill
    m = _model(max_batch=2, eng=eng)
    m._SLOT_CHUNK = 4
    reqs = [_req(0, max_new_tokens=3), _req(1, max_new_tokens=6, do_sample=False),
            _req(2, max_new_tokens=2, seed=77, temperature=0.5, top_k=7), _req(3, max_new_tokens=2)]
    outs = m.generate_requests(reqs, eos_token_id=None, do_sample=True, temperature=0.2, top_k=50, seed=1000,
                               packed_admission=packed)
    assert [_new(o) for o in outs] == [[1000 * r + k + 1 for k in range(n)] for r, n in enumerate([3, 6, 2, 2])]
    writes = [c for c in eng.calls if c[0] == "sampling"]
    # first admission: slots 0, 1 <- requests 0 (sampled, seed 1000 + 0) and 1 (greedy)
    assert writes[0] == ("sampling", [0, 1], [0.2, 0.0], [50, 0], [1000, 0])
    # request 0 leaves slot 0 after the first chunk: request 2 (its own settings) enters
    assert writes[1] == ("sampling", [0], [0.5], [7], [77])
    # then request 3 (seed 1000 + 3)
    assert writes[2] == ("sampling", [0], [0.2], [50], [1003])
    # every write precedes its admission's prefill, and the call ends with every slot greedy
    kinds = [c[0] for c in eng.calls]
    for i, k in enumerate(kinds):
        if k == "sampling" and i + 1 < len(kinds):
            assert kinds[i + 1] in ("prefill", "packed", "sampling")
    assert writes[-1] == ("sampling", [0, 1], [0.0, 0.0], [0, 0], [0, 0])
    assert eng.table == {0: (0.0, 0, 0), 1: (0.0, 0, 0)}


def test_table_is_restored_when_a_call_fails():
    class Failing(SamplingEngine):
        def slot_decode(self, first_tok, positions, n_new):
            raise RuntimeError("device error")
    eng = Failing()
    m = _model(max_batch=2, eng=eng)
    with pytest.raises(RuntimeError, match="device error"):
        m.generate_requests([_req(0), _req(1)], do_sample=True, seed=3, eos_token_id=None)
    assert eng.calls[-1] == ("sampling", [0, 1], [0.0, 0.0], [0, 0], [0, 0])


def test_seeds_wrap_and_temperature_zero_is_greedy():
    eng = SamplingEngine()
    m = _model(max_batch=2, eng=eng)
    m.generate_requests([_req(0, max_new_tokens=1), _req(1, max_new_tokens=1, temperature=0.0)], do_sample=True,
                        seed=2 ** 64 - 1, eos_token_id=None)
    assert eng.calls[0] == ("sampling", [0, 1], [1.0, 0.0], [50, 0], [2 ** 64 - 1, 0])


def test_rejections_before_any_device_work():
    eng = SamplingEngine()
    m = _model(max_batch=4, max_seq=32, eng=eng)
    with pytest.raises(NotImplementedError, match="greedily"):
        m.generate_requests([_req(0)], do_sample=True)
    with pytest.raises(NotImplementedError, match="greedily"):
        m.generate_requests([_req(0, seed=1), _req(1, do_sample=True)])
    for bad in (dict(temperature=-0.1), dict(temperature=math.inf), dict(temperature=math.nan), dict(top_k=-1),
                dict(top_k=2.5), dict(seed="7"), dict(seed=1.5)):
        kw = dict(do_sample=True, seed=1, max_new_tokens=4)
        kw.update(bad)
        with pytest.raises(ValueError):
            m.generate_requests([_req(0, max_new_tokens=4)], **kw)
        with pytest.raises(ValueError):
            m.generate(torch.tensor([[1, 5, 6]]), **kw)
    assert eng.calls == []


def test_chunks_stop_on_the_host_like_the_stepwise_path():
    """The seeded generate applies EOS, padding and stopping criteria token by token to the device's stream
    (_host_stops): a fake engine with scripted tokens shows the truncation, the tokens fed to the next chunk and
    their positions."""
    script = [[11, 12, EOS, 14, 15, 16, 17, 18], [21, 22, 23, 24, 25, 26, 27, 28]]

    class LoopEngine(SamplingEngine):
        k = 3

        def decode_loop(self, first, S, n_new):
            self.calls.append(("loop", first.tolist(), S, n_new))
            out = torch.tensor([[f] + row[self.k:self.k + n_new - 1] for f, row in zip(first.tolist(), script)],
                               dtype=torch.int32)
            self.k += n_new - 1
            return out

    m = _model(max_batch=2, max_seq=64)
    m._GREEDY_CHUNK = 3
    ctx = torch.tensor([[1, 5, 6], [1, 7, 8]])
    first = torch.tensor([row[:3] for row in script], dtype=torch.int32)
    eng = LoopEngine()
    out = m._host_stops(eng, ctx, first, 8, None, EOS, 0)
    # row 0 finishes at its EOS (step 2); from then on it is padded, and fed the pad token
    assert out[:, 3:].tolist() == [[11, 12, EOS, 0, 0, 0, 0, 0], script[1]]
    assert eng.calls == [("loop", [EOS, 23], 5, 4), ("loop", [0, 26], 8, 3)]
    assert m._pos == out.shape[1] - 1
    # a stopping criterion ends the call at the token where it fires, inside a chunk
    seen = []

    def crit(seq, scores):
        seen.append(seq.shape[1])
        return int(seq[1, -1]) == 25
    eng = LoopEngine()
    out = m._host_stops(eng, ctx, first, 8, [crit], None, 0)
    assert out[1, 3:].tolist() == [21, 22, 23, 24, 25] and seen == [4, 5, 6, 7, 8]
    assert m._pos == 7
    # every row at EOS: the call ends there, inside the first chunk
    eng = LoopEngine()
    out = m._host_stops(eng, ctx, torch.tensor([[11, EOS, 5], [EOS, 7, 8]], dtype=torch.int32), 8, None, EOS, 0)
    assert out[:, 3:].tolist() == [[11, EOS], [EOS, 0]] and eng.calls == [] and m._pos == 4
