"""Candidate scoring for score_candidates: the host-side checks of the prompts and their options, the plan of the
device rounds, and the rounds themselves.

Each prompt is prefilled once into a cache slot. Its options are scored as continuations of that prompt: columns
0 .. S - 2 of the prompt's slot are copied into the slots of its other options (Engine.slots_fork), and every option of
a round is one packed continuation (Engine.slots_score_append). Option c_1 .. c_L of a prompt p_1 .. p_S is the
sequence p_S, c_1 .. c_{L-1} at start S - 1 of its slot, so its row t predicts c_{t+1}: every option has exactly L
rows, and the prompt's own prefill needs no logits."""
from types import SimpleNamespace

import torch

import vcl_native as vn

PACKED_MAX_S = 512      # prompts up to this many tokens share one packed prefill (Engine.slots_prefill)
MAX_OPTION = 512        # rows of one packed continuation (vcl_llm_slots_score_append)


def _ids_1d(x, what):
    t = torch.as_tensor(x).detach().cpu()
    if t.dim() == 2 and t.shape[0] == 1:
        t = t[0]
    if t.dim() != 1 or t.dtype.is_floating_point or t.dtype == torch.bool:
        raise ValueError(f"{what} must be a 1-D sequence of token ids, got shape {tuple(t.shape)} ({t.dtype})")
    return t.to(torch.int64)


def check(model, input_ids, candidates, feats, attention_mask, n_vid):
    """-> SimpleNamespace(prompts [B] int64 1-D tensors, options [B][n_b] int64 1-D tensors, feats [B] ([n_vid, C]
    or None), vid_start [B] ints). Raises ValueError naming the prompt and option; no device work."""
    from .video_chatgpt import left_padding
    if isinstance(input_ids, torch.Tensor) and input_ids.dim() == 2:
        ids = input_ids.detach().cpu().to(torch.int64)
        B, S = ids.shape
        pads = left_padding(attention_mask, (B, S)) or [0] * B
        prompts = [ids[b, pads[b]:] for b in range(B)]
    else:
        if attention_mask is not None:
            raise ValueError("score_candidates: attention_mask goes with a [B, S] input_ids tensor; a list of prompts "
                             "carries no padding")
        prompts = [_ids_1d(p, f"prompt {b}") for b, p in enumerate(input_ids)]
    B = len(prompts)
    if B == 0:
        raise ValueError("score_candidates: no prompt")
    if not isinstance(candidates, (list, tuple)) or len(candidates) != B:
        raise ValueError(f"score_candidates: candidates must be a list of {B} option lists, one per prompt")
    V, max_seq, C = model.config.vocab_size, model._max_seq, model.clip_config.hidden_size
    vc = model.get_model().vision_config
    video_ids = {vc.vid_patch_token}
    if vc.use_vid_start_end:
        video_ids |= {vc.vid_start_token, vc.vid_end_token}
    video_ids.discard(None)
    options = []
    for b, p in enumerate(prompts):
        if p.numel() == 0:
            raise ValueError(f"prompt {b} is empty")
        if bool(((p < 0) | (p >= V)).any()):
            raise ValueError(f"prompt {b}: token id {int(p[(p < 0) | (p >= V)][0])} outside the vocabulary 0..{V - 1}")
        opts = candidates[b]
        if isinstance(opts, torch.Tensor) or not isinstance(opts, (list, tuple)) or len(opts) == 0:
            raise ValueError(f"prompt {b}: the option list is empty or not a list")
        row = []
        for j, o in enumerate(opts):
            c = _ids_1d(o, f"prompt {b} option {j}")
            if c.numel() == 0:
                raise ValueError(f"prompt {b} option {j} is empty")
            bad = (c < 0) | (c >= V)
            if bool(bad.any()):
                raise ValueError(f"prompt {b} option {j}: token id {int(c[bad][0])} outside the vocabulary 0..{V - 1}")
            if any(int(t) in video_ids for t in c):
                raise ValueError(f"prompt {b} option {j}: a video placeholder id is inside the option (options are "
                                 "text only)")
            if c.numel() > MAX_OPTION:
                raise ValueError(f"prompt {b} option {j}: {c.numel()} tokens, more than {MAX_OPTION}")
            if p.numel() + c.numel() > max_seq:
                raise ValueError(f"prompt {b} option {j}: prompt {p.numel()} + option {c.numel()} tokens exceed "
                                 f"max_seq {max_seq}")
            row.append(c)
        options.append(row)
    fl = [None] * B
    if feats is not None:
        if isinstance(feats, torch.Tensor):
            if feats.dim() != 3 or feats.shape[0] != B:
                raise ValueError(f"video_spatio_temporal_features must be [{B}, {n_vid}, {C}] for {B} prompts, got "
                                 f"{tuple(feats.shape)}")
            fl = list(feats)
        else:
            fl = list(feats)
            if len(fl) != B:
                raise ValueError(f"video_spatio_temporal_features has {len(fl)} entries for {B} prompts")
    vs = []
    for b, f in enumerate(fl):
        if f is None:
            vs.append(vn.NO_VIDEO)
            continue
        if f.dim() == 3 and f.shape[0] == 1:
            f = fl[b] = f[0]
        if f.dim() != 2 or f.shape[0] != n_vid or f.shape[1] != C:
            raise ValueError(f"prompt {b}: video_spatio_temporal_features must be [{n_vid}, {C}], got {tuple(f.shape)}")
        vs.append(model._video_spans(prompts[b][None], n_vid)[0])
    return SimpleNamespace(prompts=prompts, options=options, feats=fl, vid_start=vs)


def plan(prompt_lens, option_lens, n_slots, max_rows):
    """The rounds of one call, each SimpleNamespace(prefill [(prompt, slot)], forks [(src, dst, cols)], seqs [(prompt,
    option, slot, start, len)]). A round holds at most n_slots sequences and max_rows continuation rows. Prompts are
    taken in order; a prompt whose options do not fit the rest of a round starts the next one. A prompt with more
    options than slots runs alone over several rounds: its slot 0 is prefilled in the first and hosts an option only in
    the last, so columns 0 .. S - 2 stay intact for the forks of the later rounds (with a single slot, every round
    prefills the prompt again and scores one option there)."""
    rounds = []
    cur = None

    def new_round():
        nonlocal cur
        cur = SimpleNamespace(prefill=[], forks=[], seqs=[], rows=0)
        rounds.append(cur)

    def place(b, js, slot0, prefill, own):
        """options js of prompt b in the current round, the prompt in slot slot0 (prefilled there when `prefill`);
        the first option takes slot0 itself when `own`"""
        S = prompt_lens[b]
        if prefill:
            cur.prefill.append((b, slot0))
        nxt = slot0 + 1
        for k, j in enumerate(js):
            L = option_lens[b][j]
            if own and k == 0:
                slot = slot0
            else:
                slot, nxt = nxt, nxt + 1
                cur.forks.append((slot0, slot, S - 1))
            cur.seqs.append((b, j, slot, S - 1, L))
            cur.rows += L

    for b, S in enumerate(prompt_lens):
        n_b = len(option_lens[b])
        rows = sum(option_lens[b])
        if n_b <= n_slots:
            if cur is None or len(cur.seqs) + n_b > n_slots or cur.rows + rows > max_rows:
                new_round()
            place(b, list(range(n_b)), len(cur.seqs), True, True)
            continue
        # more options than slots: alone, over several rounds
        js = list(range(n_b))
        if n_slots == 1:
            for j in js:
                new_round()
                place(b, [j], 0, True, True)
            cur = None
            continue
        first = True
        while js:
            new_round()
            last = len(js) <= n_slots
            take = js if last else js[:n_slots - 1]
            js = [] if last else js[n_slots - 1:]
            place(b, take, 0, first, last)
            first = False
        cur = None
    return rounds


def score(model, eng, q):
    """Run the rounds of the checked call q (check) on the engine; returns score_candidates' list."""
    n_slots = model._n_slots
    max_rows = model._max_batch * model._max_seq
    P = q.prompts
    rounds = plan([p.numel() for p in P], [[c.numel() for c in row] for row in q.options], n_slots, max_rows)
    parts = []   # (round's seqs, lp, greedy) on the device
    for rd in rounds:
        short = [(b, s) for b, s in rd.prefill if P[b].numel() <= PACKED_MAX_S]
        if short:
            eng.slots_prefill([s for _, s in short], [P[b] for b, _ in short], [q.feats[b] for b, _ in short],
                              [q.vid_start[b] for b, _ in short])
        for b, s in rd.prefill:
            if P[b].numel() > PACKED_MAX_S:
                vs = torch.tensor([q.vid_start[b]], dtype=torch.int32, device=model.device)
                eng.slot_prefill(s, P[b].to(model.device), q.feats[b], vs)
        if rd.forks:
            eng.slots_fork([f[0] for f in rd.forks], [f[1] for f in rd.forks], [f[2] for f in rd.forks])
        ids, labels = [], []
        for b, j, _, _, _ in rd.seqs:
            c = q.options[b][j]
            ids.append(torch.cat([P[b][-1:], c[:-1]]))
            labels.append(c)
        lp, greedy = eng.slots_score_append([s[2] for s in rd.seqs], [s[3] for s in rd.seqs], ids, labels)
        parts.append((rd.seqs, lp, greedy))
    out = [dict(logprob=None, greedy=None, token_logprobs=[None] * len(row)) for row in q.options]
    gr = [[False] * len(row) for row in q.options]
    for seqs, lp, greedy in parts:
        lp, greedy = lp.cpu(), greedy.cpu().bool()
        r = 0
        for b, j, _, _, L in seqs:
            out[b]["token_logprobs"][j] = lp[r:r + L].clone()
            gr[b][j] = bool(greedy[r:r + L].all())
            r += L
    for b, o in enumerate(out):
        tl = o["token_logprobs"]
        o["logprob"] = torch.tensor([sum(float(x) for x in t.tolist()) for t in tl], dtype=torch.float64)
        o["greedy"] = torch.tensor(gr[b], dtype=torch.bool)
    return out
