"""Float64 reference of the attention kernels over the KV cache (prefill: attention_prefill_tc.cu, attention.cu;
decode: decode_attention.cu), with the reference's rounding points.

A query row is described by (clip, pos, kmin): it sits at absolute position pos of cache clip (or slot) `clip` and
attends keys kmin .. pos of that clip. kernels.h's rules give kmin: a clip with n_pad pad columns gives a real query
(pos >= n_pad) the floor n_pad and a pad query the floor 0 (causal from key 0); packed sequences and decode queries
of an unpadded clip have floor 0.

Rounding points (transformers' eager LLaMA attention, modeling_llama.py:199-222): the scores are
bf16(bf16(q . k) * scale) with scale an fp32 number and the q . k products exact (fp64 sums of bf16 products), the
softmax runs in fp32, p is rounded to bf16 and p . v is accumulated in fp64."""
import torch

SCALE = 128 ** -0.5


def key_floor(pos, n_pad):
    """kmin of a query at column pos of a clip with n_pad pad columns (kernels.h: positions in the KV cache)"""
    return n_pad if pos >= n_pad else 0


def cached_rows(B, start, S, n_pad=None):
    """The rows of a prefill of B clips of S queries at positions start .. start + S - 1 (row b * S + j: clip b,
    position start + j), n_pad None or B pad counts -> (clip, pos, kmin), int64 tensors [B * S]"""
    pads = list(n_pad) if n_pad is not None else [0] * B
    clip = torch.arange(B).repeat_interleave(S)
    pos = torch.arange(start, start + S).repeat(B)
    npd = torch.tensor(pads, dtype=torch.int64)[clip]
    kmin = torch.where(pos >= npd, npd, torch.zeros_like(npd))
    return clip, pos, kmin


def packed_rows(slots, starts, lens):
    """The rows of packed sequences (kernels.h: sequence i's len_i rows follow sequence i - 1's and sit at positions
    start_i .. of slot_i, attending keys 0 .. their own position) -> (clip, pos, kmin)"""
    clip = torch.cat([torch.full((int(n),), int(s), dtype=torch.int64) for s, n in zip(slots, lens)])
    pos = torch.cat([torch.arange(int(a), int(a) + int(n)) for a, n in zip(starts, lens)])
    return clip, pos, torch.zeros_like(pos)


def ref_mask(pos, kmin, n_keys):
    """[R, n_keys] bool: row r attends key j when kmin[r] <= j <= pos[r]"""
    j = torch.arange(n_keys, device=pos.device)
    return (j[None] >= kmin[:, None]) & (j[None] <= pos[:, None])


def _groups(clip, pos, kmin, device):
    clip, pos, kmin = (torch.as_tensor(t, dtype=torch.int64).to(device) for t in (clip, pos, kmin))
    for c in torch.unique(clip).tolist():
        rows = (clip == c).nonzero()[:, 0]
        n = int(pos[rows].max()) + 1
        yield c, rows, n, ref_mask(pos[rows], kmin[rows], n)


def _attended(t, c, n, used, what):
    """columns 0 .. n - 1 of clip c of a cache [C, H, cols, 128] in fp64; the attended ones must be finite (the tests
    poison every column no query may read), the others are zeroed so that p = 0 meets no NaN"""
    x = t[c, :, :n].double()
    assert torch.isfinite(x[:, used]).all(), f"{what}: an attended column of clip {c} is not finite"
    return torch.where(used[None, :, None], x, torch.zeros((), dtype=x.dtype, device=x.device))


def attn_ref(q, k, v, clip, pos, kmin, scale=SCALE):
    """q [R, >= H * 128] bf16 (head h at columns h * 128 ..), k / v [C, H, cols, 128] bf16, the rows' (clip, pos,
    kmin) -> o [R, H, 128] fp64 with the rounding points above"""
    H = k.shape[1]
    out = torch.empty(q.shape[0], H, 128, dtype=torch.float64, device=q.device)
    sc = torch.tensor(scale, dtype=torch.float32)
    for c, rows, n, m in _groups(clip, pos, kmin, q.device):
        used = m.any(0)
        kk, vv = _attended(k, c, n, used, "k"), _attended(v, c, n, used, "v")
        qq = q[rows, :H * 128].double().view(-1, H, 128).transpose(0, 1)          # [H, r, 128]
        s = (qq @ kk.transpose(1, 2)).bfloat16().float()                          # exact q . k, one rounding
        s = (s * sc).bfloat16().float()
        s = s.masked_fill(~m[None], float("-inf"))
        p = torch.softmax(s, -1).bfloat16().double()
        out[rows] = (p @ vv).transpose(0, 1)
    return out


def mean_ref(v, clip, pos, kmin):
    """The exact mean of the attended values, [R, H, 128] fp64: the output of every attention kernel when all scores
    are equal (q = 0), up to the final bf16 rounding"""
    H = v.shape[1]
    out = torch.empty(len(clip), H, 128, dtype=torch.float64, device=v.device)
    for c, rows, n, m in _groups(clip, pos, kmin, v.device):
        vv = _attended(v, c, n, m.any(0), "v")
        out[rows] = torch.einsum("rn,hnd->rhd", m.double(), vv) / m.sum(1).double()[:, None, None]
    return out


def equal_weight_ref(v, clip, pos, kmin):
    """The decode kernel's exact output when all scores are equal (q = 0) and v holds small integers (the counting
    and probe inputs), [R, H, 128] fp64 holding bf16 values. Every key then weighs e = exp(0) = 1, the fp32 sum is
    n, p = bf16(fp32(1 / n)), and the fp32 accumulator holds c_d * p exactly (c_d the sum of the attended keys'
    values at d, below 2^16), so element d is bf16(c_d * p)."""
    H = v.shape[1]
    out = torch.empty(len(clip), H, 128, dtype=torch.float64, device=v.device)
    for c, rows, n, m in _groups(clip, pos, kmin, v.device):
        vv = _attended(v, c, n, m.any(0), "v")
        cnt = torch.einsum("rn,hnd->rhd", m.double(), vv)
        assert cnt.abs().max() < 2 ** 16 and torch.equal(cnt, cnt.round()), "not an exact input"
        p = (torch.ones((), dtype=torch.float32, device=v.device) / m.sum(1).float()).bfloat16().double()
        out[rows] = (cnt * p[:, None, None]).bfloat16().double()
    return out


def probe_plan(keys, n_sets=None):
    """The probe input's schedule for one (clip, head): the sorted keys to probe are dealt round robin over
    n_sets >= 2 sets (default: as few as hold 128 each), so that neighbouring keys never share a set. Returns
    [[(key, dimension), ...] per set]; key i of the list is set i % n_sets, dimension i // n_sets."""
    keys = sorted(set(int(j) for j in keys))
    n = max(2, (len(keys) + 127) // 128) if n_sets is None else n_sets
    assert n >= 2 and len(keys) <= 128 * n
    return [[(j, i // n) for i, j in enumerate(keys) if i % n == s] for s in range(n)]


def probe_values(C, H, cols, sets, device="cpu"):
    """v [C, H, cols, 128] bf16 for the probe input: zero, except key j of clip c, head h is one-hot at dimension d
    for each (j, d) in sets[c][h] (None or missing: no probe). With q = 0 an output element is then 0, bf16(p) or
    bf16(2 p): its probe was skipped, read once or read twice, and a read from the wrong address lights the wrong
    dimension (equal_weight_ref gives the expected output)."""
    v = torch.zeros(C, H, cols, 128, dtype=torch.bfloat16, device=device)
    for c, per_head in enumerate(sets):
        for h, s in enumerate(per_head):
            if s:
                j, d = (torch.tensor(t, device=device) for t in zip(*s))
                v[c, h, j, d] = 1.0
    return v


def counting_values(C, H, cols, n_pad=None, pad_value=100.0, device="cpu"):
    """v [C, H, cols, 128] bf16 for the counting input: column j of head h is one-hot at d = (7 j + 3 h) % 128, of
    value 1 (pad_value in clip c's first n_pad[c] columns). With q = 0 every attended key weighs exactly 1 / n, so
    output element d is (sum of the attended keys' values in class d) / n."""
    j = torch.arange(cols)
    h = torch.arange(H)
    d = (7 * j[None, :] + 3 * h[:, None]) % 128                                    # [H, cols]
    v = torch.zeros(C, H, cols, 128, dtype=torch.bfloat16, device=device)
    v.scatter_(3, d.to(device)[None, :, :, None].expand(C, H, cols, 1), 1.0)
    for c, npd in enumerate(n_pad or []):
        v[c, :, :npd] *= pad_value
    return v


def bf16_ulp(x):
    """the spacing of bf16 numbers at |x| (fp64; the smallest normal spacing for 0)"""
    a = x.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)
