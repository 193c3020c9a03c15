"""In-flight batching for generate_requests: the host-side checks of the requests, one admission / decode loop
(schedule) for the contiguous (Slots) and the paged (PagedSlots) KV cache, and the log-probs the requests collect."""
import collections
from types import SimpleNamespace

import torch

import vcl_native as vn


def request(model, i, r, max_new_tokens, stopping_criteria, n_vid, samp):
    """One request of generate_requests, checked on the host -> (ids [S] int64 on the host, S, n, feats,
    vid_start, criteria, its sampling-table entry: temperature (0: greedy), top_k, seed, top_p, penalty, warp
    (model._warper_args; None: none), and its bans (model._ban_args; None: none))"""
    if isinstance(r, torch.Tensor):
        r = {"input_ids": r}
    ids = torch.as_tensor(r["input_ids"]).detach().cpu().to(torch.int64)
    if ids.dim() == 2 and ids.shape[0] == 1:
        ids = ids[0]
    if ids.dim() != 1 or ids.numel() == 0:
        raise ValueError(f"request {i}: input_ids must be [S] or [1, S], got shape {tuple(ids.shape)}")
    S, n = ids.numel(), int(r.get("max_new_tokens", max_new_tokens))
    if n < 1 or S + n > model._max_seq:
        raise ValueError(f"request {i}: prompt length {S} + max_new_tokens {n} does not fit max_seq {model._max_seq}")
    feats, vs = r.get("video_spatio_temporal_features"), vn.NO_VIDEO
    if feats is not None and r.get("continues") is not None:
        raise ValueError(f"request {i}: a continuation carries text only (its video is in the kept cache)")
    if feats is not None:
        if feats.dim() == 3 and feats.shape[0] == 1:
            feats = feats[0]
        if feats.dim() != 2 or feats.shape[0] != n_vid:
            raise ValueError(f"request {i}: video_spatio_temporal_features must be [{n_vid}, C], got "
                             f"{tuple(feats.shape)}")
        vs = model._video_spans(ids[None], n_vid)[0]
    crit = r.get("stopping_criteria", stopping_criteria)
    T, k, seed = 0.0, 0, 0
    top_p, penalty = model._nucleus_args(r.get("top_p", samp.get("top_p", 1.0)),
                                         r.get("repetition_penalty", samp.get("repetition_penalty", 1.0)),
                                         f"request {i}", r.get("do_sample", samp["do_sample"]))
    if r.get("do_sample", samp["do_sample"]):
        own = r.get("seed") is not None       # a seed is there (generate_requests checks it first)
        T, k, seed = model._sampling_args(r.get("temperature", samp["temperature"]), r.get("top_k", samp["top_k"]),
                                          r["seed"] if own else samp["seed"], f"request {i}")
        seed = seed if own else (seed + i) % 2 ** 64
        if T == 0:
            k, seed = 0, 0
    warp = model._warper_args(r.get("min_p", samp.get("min_p")), r.get("typical_p", samp.get("typical_p")),
                              r.get("epsilon_cutoff", samp.get("epsilon_cutoff")),
                              r.get("eta_cutoff", samp.get("eta_cutoff")), f"request {i}", T > 0)
    if T == 0:
        top_p = 1.0                           # HF adds no warpers when greedy
    bans = model._ban_args(r.get("no_repeat_ngram_size", samp.get("no_repeat_ngram_size")),
                           r.get("bad_words_ids", samp.get("bad_words_ids")),
                           r.get("min_new_tokens", samp.get("min_new_tokens")), samp.get("eos"), f"request {i}")
    return SimpleNamespace(ids=ids, S=S, n=n, feats=feats, vid_start=vs, criteria=list(crit or []),
                           temperature=T, top_k=k, seed=seed, top_p=top_p, penalty=penalty, bans=bans, warp=warp,
                           session=r.get("session"),
                           continues=r.get("continues"), start=0, lp=r.get("logprobs", samp.get("logprobs")))


def bind_sessions(model, reqs):
    """The "session" / "continues" keys of generate_requests' requests, checked on the host before any device
    work. A continuation's ids become the whole conversation (the kept tokens, then its new turn), its S their
    length and its start the first column its tail prefill writes: the kept position L - 1, where
    generate_continue would start."""
    started, continued = {}, {}
    for i, r in enumerate(reqs):
        if r.session is not None and r.continues is not None:
            raise ValueError(f"request {i}: a request starts a conversation (\"session\") or continues one "
                             "(\"continues\"), not both")
        if r.session is not None:
            if r.session in model._sessions:
                raise ValueError(f"request {i}: a conversation is already kept under session key {r.session!r} "
                                 "(continue it, or end_session it first)")
            if r.session in started:
                raise ValueError(f"request {i}: session key {r.session!r} is also started by request "
                                 f"{started[r.session]}")
            started[r.session] = i
        if r.continues is not None:
            if r.continues in continued:
                raise ValueError(f"request {i}: conversation {r.continues!r} is also continued by request "
                                 f"{continued[r.continues]}; one turn per conversation and call")
            continued[r.continues] = i
    for key, i in continued.items():
        r = reqs[i]
        if key in started:
            raise ValueError(f"request {i}: conversation {key!r} is started by request {started[key]} in the same "
                             "call; a turn's text depends on the previous answer, so continue it in a later call")
        if key not in model._sessions:
            raise ValueError(f"request {i}: no conversation is kept under key {key!r}")
        if r.S + 1 > model._PACKED_MAX_S:
            raise ValueError(f"request {i}: the continuation's tail (the last kept token and {r.S} new tokens) "
                             f"has {r.S + 1} rows, more than {model._PACKED_MAX_S}")
        conv = model._sessions[key].ids
        L = conv.numel()
        if L + r.S + r.n > model._max_seq:
            raise ValueError(f"request {i}: conversation of {L} tokens + {r.S} new + max_new_tokens {r.n} does not "
                             f"fit max_seq {model._max_seq}")
        r.ids, r.start = torch.cat([conv, r.ids]), L - 1
        r.S = r.ids.numel()


def check_paged(model, reqs, chunked):
    """The requests a paged cache takes, checked on the host before any device work: a prompt of at most
    min(512, max_seq) tokens (a paged engine prefills packed) unless `chunked` (any prompt `request` accepts), and
    at most kv_blocks - 1 blocks for the prompt and every new token, so that a request alone always fits the pool
    and the scheduler always makes progress."""
    C, usable = vn.KV_BLOCK_COLS, model._kv_blocks - 1
    s_lim = min(model._PACKED_MAX_S, model._max_seq)
    for i, r in enumerate(reqs):
        if r.start == 0 and r.S > s_lim and not chunked:
            raise ValueError(f"request {i}: prompt of {r.S} tokens; a paged KV cache takes prompts of at most "
                             f"{s_lim} tokens (the packed prefill); chunked_prefill=True takes longer ones")
        need = -(-(r.S + r.n) // C)
        if need > usable:
            what = f"conversation of {r.S} tokens" if r.start > 0 else f"prompt {r.S}"
            raise ValueError(f"request {i}: {what} + max_new_tokens {r.n} needs {need} blocks of {C} columns, more "
                             f"than the pool's {usable} (kv_blocks {model._kv_blocks}, block 0 is the park block)")


def request_done(r, gen, eos):
    """Whether the request ends with its newest token gen[-1]: EOS, then the stopping criteria, then the
    length limit, in the order of _stepwise"""
    if eos is not None and gen[-1] == eos:
        return True
    if r.criteria:
        seq = torch.cat([r.ids, torch.tensor(gen, dtype=torch.int64)])[None]
        if any(c(seq, None) for c in r.criteria):
            return True
    return len(gen) >= r.n


def admit_sampling(model, eng, group, resumed, banning=False, eos=None):
    """The sampling-table entries of the (slot, request) pairs admitted at one point, in one write, and the token
    set of each penalized one: its ids; for a (slot, request, tokens) of `resumed`, its ids then those tokens. Under
    `banning` (some request of the call bans) also the ban-table entries of every pair, in one write (EOS allowed
    from column S + min_new_tokens), and the token history of each banning one, from the same ids."""
    rows = list(group) + [(s, r) for s, r, _ in resumed]
    model._set_entries(eng, [s for s, _ in rows], [r.temperature for _, r in rows], [r.top_k for _, r in rows],
                       [r.seed for _, r in rows], [r.top_p for _, r in rows], [r.penalty for _, r in rows],
                       [r.warp for _, r in rows])
    ids = [(s, r, r.ids) for s, r in group]
    ids += [(s, r, torch.cat([r.ids, torch.tensor(toks, dtype=torch.int64)])) for s, r, toks in resumed]
    model._token_sets(eng, [(s, t) for s, r, t in ids if r.penalty != 1.0])
    if banning:
        model._set_bans(eng, [s for s, _ in rows], [r.bans for _, r in rows], eos,
                        [r.S + r.bans.min_new if r.bans else 0 for _, r in rows])
        model._histories(eng, [(s, t) for s, r, t in ids if r.bans is not None])


def prefill(model, eng, group, first, packed):
    """Prefill the (slot, request) pairs of one admission point, each slot's first token into first[slot]: one at a
    time (slot_prefill), or under `packed` all prompts of at most _PACKED_MAX_S tokens in one slots_prefill, which
    always fits the activations (max_batch * max_seq tokens: at most max_batch prompts, each shorter than max_seq)."""
    dev = first.device
    for s, r in group:
        if not packed or r.S > model._PACKED_MAX_S:
            feats = None if r.feats is None else r.feats.to(dev)
            vs = torch.tensor([r.vid_start], dtype=torch.int32, device=dev)
            eng.slot_prefill(s, r.ids.to(dev), feats, vs, tok_out=first[s:s + 1])
    group = [(s, r) for s, r in group if packed and r.S <= model._PACKED_MAX_S]
    if group:
        slots = [s for s, _ in group]
        tok = eng.slots_prefill(slots, [r.ids for _, r in group],
                                [None if r.feats is None else r.feats.to(dev) for _, r in group],
                                [r.vid_start for _, r in group])
        first[torch.tensor(slots, device=dev)] = tok


def prefill_chunked(model, eng, group, first, packed, sampling, stats):
    """Prefill the (slot, request) pairs of one admission point whose prompts are longer than _PACKED_MAX_S on a
    paged engine: each prompt runs as consecutive chunks of _PACKED_MAX_S rows (Engine.slots_prefill_chunk),
    every chunk attending the columns its earlier chunks left in the slot's blocks. packed: chunk k of every
    prompt of the group goes into one call (at most n_slots * 512 rows, which the activations hold); otherwise
    each prompt runs alone. A slot's first token (first[slot]) is the one its last chunk gives; stats counts the
    prompts and the calls. Every chunk call also draws a token for each of its prompts (only the last one's is
    kept), which a penalized slot adds to its token set and a banning one writes into its history: so both are
    written again before each later call."""
    dev, L = first.device, model._PACKED_MAX_S
    stats["chunked_prefills"] += len(group)
    for batch in ([group] if packed else [[g] for g in group]):
        for start in range(0, max(r.S for _, r in batch), L):
            live = [(s, r) for s, r in batch if start < r.S]
            if sampling and start > 0:   # (chunk 0 follows the admission's write)
                model._token_sets(eng, [(s, r.ids) for s, r in live if r.penalty != 1.0])
                model._histories(eng, [(s, r.ids) for s, r in live if r.bans is not None])
            tok = eng.slots_prefill_chunk([s for s, _ in live], [start] * len(live), [r.S for _, r in live],
                                          [r.ids[start:start + L] for _, r in live],
                                          [None if r.feats is None else r.feats.to(dev) for _, r in live],
                                          [r.vid_start for _, r in live])
            stats["chunk_calls"] += 1
            for j, (s, r) in enumerate(live):
                if start + L >= r.S:
                    first[s] = tok[j]


def schedule(model, eng, reqs, n_slots, packed, sampling, eos, chunked, lps):
    """The admission / decode loop of generate_requests on either cache (Slots, PagedSlots): seat requests in idle
    slots, write their sampling and log-prob entries, prefill them, decode a chunk of _SLOT_CHUNK steps (fewer only
    when a slot nears max_seq) and take each slot's new tokens up to its request's end. Returns the results."""
    slots = (PagedSlots if model._kv_blocks else Slots)(model, eng, reqs, n_slots, lps)
    owner, pos, unseen = slots.owner, slots.pos, slots.unseen
    dev, K, L = model.device, model._SLOT_CHUNK, model._PACKED_MAX_S
    results = [None] * len(reqs)
    queue = collections.deque(range(len(reqs)))
    gen = {}                            # request -> its new tokens so far
    banning = any(r.bans is not None for r in reqs)
    while True:
        admitted, resumed, tails = slots.admit(queue)
        for _, i in admitted + tails:
            gen[i] = []
        if sampling and (admitted or resumed or tails):
            # a resumed request's token set: its prompt and its tokens, the pending one too when the host has
            # not seen it yet (its prefill's token)
            admit_sampling(model, eng, [(s, reqs[i]) for s, i in admitted + tails],
                           [(s, reqs[i], gen[i] + ([int(slots.first[s])] if unseen[s] else [])) for s, i in resumed],
                           banning, eos)
        lps.sync(owner)
        # continuations: the tails admitted here in one call under packed admission, one call each otherwise
        for group in ([tails] if packed and tails else [[t] for t in tails]):
            tok = eng.slots_prefill_append([s for s, _ in group], [reqs[i].start for _, i in group],
                                           [reqs[i].ids[reqs[i].start:] for _, i in group])
            slots.first[torch.tensor([s for s, _ in group], device=dev)] = tok
        if chunked and admitted:
            long = [(s, reqs[i]) for s, i in admitted if reqs[i].S > L]
            admitted = [(s, i) for s, i in admitted if reqs[i].S <= L]
            if long:
                prefill_chunked(model, eng, long, slots.first, packed, sampling, slots.stats)
        prefill(model, eng, [(s, reqs[i]) for s, i in admitted], slots.first, packed)
        active = [s for s in range(n_slots) if owner[s] is not None]
        if not active:
            slots.close()
            return results
        m = min([K] + [model._max_seq - pos[s] for s in active])
        slots.grow(m)
        running = [(s, owner[s]) for s in active if owner[s] is not None]
        out = eng.slot_decode(slots.first, pos, m + 1)
        slots.first = out[:, m].contiguous()
        host = out.tolist()
        for s, i in running:
            r = reqs[i]
            pos[s] += m
            for t in (host[s] if unseen[s] else host[s][1:]):
                gen[i].append(t)
                if request_done(r, gen[i], eos):
                    seq = torch.cat([r.ids, torch.tensor(gen[i], dtype=torch.int64)])
                    results[i] = seq[None].to(dev)
                    slots.finish(s, r, seq)
                    break
            unseen[s] = False
        lps.collect([(s, i, len(gen[i])) for s, i in running])


class Slots:
    """The slots of one generate_requests call on a contiguous KV cache: each slot's request (owner), its cached tokens
    (pos; 0 when idle), whether the host has not seen its prefill's token yet (unseen) and the token it is fed next
    (first). A slot holds max_seq columns, so every idle slot takes the queue head, and nothing grows or swaps."""

    def __init__(self, model, eng, reqs, n_slots, lps):
        self.eng, self.reqs, self.lps = eng, reqs, lps
        self.owner = [None] * n_slots
        self.pos = [0] * n_slots
        self.unseen = [False] * n_slots
        self.first = torch.zeros(n_slots, dtype=torch.int32, device=model.device)

    def admit(self, queue):
        """-> (admitted, resumed, tails): (slot, request) pairs of new prompts, resumed requests and continuations"""
        admitted = []
        for s in range(len(self.owner)):
            if self.owner[s] is None and queue:
                i = queue.popleft()
                self.owner[s], self.pos[s], self.unseen[s] = i, self.reqs[i].S, True
                admitted.append((s, i))
        return admitted, [], []

    def grow(self, m):
        """Room for the next decode chunk of m steps in every running slot"""

    def finish(self, s, r, seq):
        """Request r in slot s has ended with the tokens seq: the slot is idle"""
        self.owner[s], self.pos[s] = None, 0

    def close(self):
        """The call's last request has ended"""


class PagedSlots(Slots):
    """The cache slots on a paged KV cache. The host keeps a free list and each slot's row of the block table (block 0,
    the park block, wherever no request owns a block), and writes the whole table to the engine before every prefill
    and every decode chunk.
    - Blocks. A running request at position pos, decoding a chunk of m steps, owns the blocks of columns
      0 .. min(pos + m, S + n) - 1: every column the chunk writes that the request can still read (past S + n - 1
      the request has all its tokens; those columns of a chunk land in the park block or in its own last block).
    - Admission. Swapped-out requests resume first, oldest admission first, then queued requests in queue order
      (none overtakes another): each into a free slot when the free list covers its blocks for one chunk.
    - Preemption. When a chunk's growth is not covered, the most recently admitted running request is swapped out
      (its written blocks copied to pinned host memory, its blocks freed, its slot parked) until it is. Its
      position, pending token and sampling entry stay on the host; it resumes into any free slot and free blocks,
      restored exactly, and its tokens depend on its seed and positions only.
    - Chunked prefill. A prompt over _PACKED_MAX_S tokens is admitted by the same rule (its prompt's blocks plus one
      chunk's growth) and prefilled at its admission point by prefill_chunked, before the next decode chunk; so a
      request that is swapped out always holds its whole prompt.
    - Sessions. A request with a "session" or "continues" key keeps its conversation when it ends (model._sessions):
      its tokens [L] and the blocks of columns 0 .. L - 2, which stay out of the free list, also across calls;
      its other blocks are freed. A continuation is admitted by the same rule with its conversation's blocks in
      its slot's row (copied back into fresh blocks first if they were swapped out) and prefills its tail, the
      columns L - 1 .. S - 1, through Engine.slots_prefill_append.
    - Eviction. Kept conversations are idle: when an admission, a resume or a chunk's growth is short of blocks,
      the least recently used one that is resident is swapped to pinned host memory (its blocks freed) before
      anything waits or any running request is preempted.
    - Log-probs. A request swapped out before its first token reached the host takes that token's row along (it
      lives in its old slot's entry); every other row is read after the chunk that produced it.
    check_paged guarantees that the oldest running request alone always fits. model.last_kv_stats holds the
    counters when the call returns."""

    def __init__(self, model, eng, reqs, n_slots, lps):
        super().__init__(model, eng, reqs, n_slots, lps)
        self.model, self.K, self.C = model, model._SLOT_CHUNK, vn.KV_BLOCK_COLS
        self.sessions = model._sessions
        self.table = [[0] * eng.table_row for _ in range(eng.n_slots)]    # every slot of the engine, parked
        kept = {b for ss in self.sessions.values() if ss.blocks is not None for b in ss.blocks}
        self.free = [b for b in range(eng.kv_blocks - 1, 0, -1) if b not in kept]   # pop() takes the lowest block
        self.blocks = [[] for _ in range(n_slots)]
        self.order = [0] * n_slots          # admission stamp of the slot's request (the latest is preempted first)
        self.stamp = 0
        self.swapped = {}                   # request -> (pos, pending token, unseen, host copies of its blocks)
        self.released = []                  # host buffers whose copy back may still be in flight
        self.stats = dict(preemptions=0, swapped_bytes=0, peak_blocks=0, kv_blocks=eng.kv_blocks, chunked_prefills=0,
                          chunk_calls=0, continuations=0, reused_rows=0, session_swaps=0, session_swapped_bytes=0)

    def seat(self, s, i, p, unseen):
        self.stamp += 1
        self.owner[s], self.pos[s], self.unseen[s], self.order[s] = i, p, unseen, self.stamp

    def cover(self, i, p, m):               # blocks of columns 0 .. min(p + m, S + n) - 1
        r = self.reqs[i]
        return -(-min(p + m, r.S + r.n) // self.C)

    def take(self, s, want):
        while len(self.blocks[s]) < want:
            self.blocks[s].append(self.free.pop())
        self.table[s][:len(self.blocks[s])] = self.blocks[s]
        self.stats["peak_blocks"] = max(self.stats["peak_blocks"], self.eng.kv_blocks - 1 - len(self.free))

    def release(self, s, keep=0):           # the first `keep` blocks stay with a kept conversation
        self.free.extend(reversed(self.blocks[s][keep:]))
        self.blocks[s], self.table[s] = [], [0] * self.eng.table_row
        self.owner[s], self.pos[s] = None, 0

    def copy_out(self, blocks):             # each block's pinned host copy
        saved = []
        for b in blocks:
            buf = self.eng.swap_buffer()
            self.eng.kv_block_copy(b, buf)
            saved.append(buf)
        return saved

    def copy_back(self, s, saved):          # host copies into the slot's first blocks
        for b, buf in zip(self.blocks[s], saved):
            self.eng.kv_block_copy(b, buf, write=True)
        self.released.extend(saved)

    def room(self, need, spare=None):
        """whether `need` blocks are free, after swapping resident kept conversations (not `spare`) to host memory,
        least recently used first, while they are not"""
        while len(self.free) < need:
            keys = [k for k, ss in self.sessions.items() if ss.blocks is not None and k != spare]
            if not keys:
                return False
            ss = self.sessions[min(keys, key=lambda k: self.sessions[k].used)]
            ss.saved = self.copy_out(ss.blocks)
            self.free.extend(reversed(ss.blocks))
            ss.blocks = None
            self.stats["session_swaps"] += 1
            self.stats["session_swapped_bytes"] += len(ss.saved) * self.eng.block_bytes
        return True

    def swap_out(self, s):
        i = self.owner[s]
        if self.unseen[s]:
            self.lps.collect([(s, i, 1)])
        saved = self.copy_out(self.blocks[s][:-(-self.pos[s] // self.C)])   # the blocks that hold written columns
        self.swapped[i] = (self.pos[s], int(self.first[s]), self.unseen[s], saved)
        self.stats["preemptions"] += 1
        self.stats["swapped_bytes"] += len(saved) * self.eng.block_bytes
        self.release(s)

    def admit(self, queue):
        self.released.clear()               # the last decode chunk's tokens reached the host after every copy back
        sessions, K = self.sessions, self.K
        idle = [s for s in range(len(self.owner)) if self.owner[s] is None]
        admitted, resumed, tails = [], [], []
        while self.swapped and idle:
            i = min(self.swapped)           # requests are first admitted in queue (= index) order
            p, tok, uns, saved = self.swapped[i]
            if not self.room(self.cover(i, p, K)):
                break
            del self.swapped[i]
            s = idle.pop(0)
            self.seat(s, i, p, uns)
            self.take(s, self.cover(i, p, K))
            self.copy_back(s, saved)
            self.first[s] = tok
            resumed.append((s, i))
        while not self.swapped and idle and queue:
            i = queue[0]
            r = self.reqs[i]
            ss = sessions[r.continues] if r.continues is not None else None
            own = ss.blocks if ss is not None and ss.blocks is not None else []
            if not self.room(self.cover(i, r.S, K) - len(own), spare=r.continues):
                break
            queue.popleft()
            s = idle.pop(0)
            self.seat(s, i, r.S, True)
            self.blocks[s] = list(own)
            self.take(s, self.cover(i, r.S, K))
            if ss is None:
                admitted.append((s, i))
                continue
            del sessions[r.continues]
            if ss.saved is not None:        # swapped out: copied back into the slot's first blocks
                self.copy_back(s, ss.saved)
            tails.append((s, i))
            self.stats["continuations"] += 1
            self.stats["reused_rows"] += r.start
        if admitted or resumed or tails:
            self.eng.set_block_table(self.table)
        return admitted, resumed, tails

    def grow(self, m):
        # oldest admission first; while the free list falls short, swap out a kept conversation, else preempt the
        # latest running request
        owner = self.owner
        for s in sorted((s for s in range(len(owner)) if owner[s] is not None), key=lambda t: self.order[t]):
            while owner[s] is not None and not self.room(self.cover(owner[s], self.pos[s], m) - len(self.blocks[s])):
                self.swap_out(max((t for t in range(len(owner)) if owner[t] is not None), key=lambda t: self.order[t]))
            if owner[s] is not None:
                self.take(s, self.cover(owner[s], self.pos[s], m))
        self.eng.set_block_table(self.table)
        self.lps.sync(owner)

    def finish(self, s, r, seq):
        key = r.continues if r.continues is not None else r.session
        keep = 0
        if key is not None:                 # kept: columns 0 .. L - 2, generate_continue's cache
            keep = -(-(seq.numel() - 1) // self.C)
            self.model._session_clock += 1
            self.sessions[key] = SimpleNamespace(ids=seq, blocks=self.blocks[s][:keep], saved=None,
                                                 used=self.model._session_clock)
        self.release(s, keep)

    def close(self):
        self.eng.set_block_table(self.table)        # every slot parked again
        self.stats["sessions"] = len(self.sessions)
        self.stats["sessions_resident"] = sum(ss.blocks is not None for ss in self.sessions.values())
        self.stats["sessions_swapped"] = self.stats["sessions"] - self.stats["sessions_resident"]
        self.model.last_kv_stats = self.stats


class RequestLogprobs:
    """The log-probs of one generate_requests call: the slots' entries as the engine holds them, and each request's
    rows read so far (blocks of rows, one row per new token, in order). Request i's k-th new token took position
    reqs[i].S + k of its slot's entry."""

    def __init__(self, model, eng, reqs, n_slots):
        self.model, self.eng, self.reqs, self.dev = model, eng, reqs, model.device
        self.on = any(r.lp is not None for r in reqs)
        self.written = [-1] * n_slots
        self.rows = {i: [] for i, r in enumerate(reqs) if r.lp is not None}
        self.have = {i: 0 for i in self.rows}

    def sync(self, owner):
        """One set_logprobs call for the slots whose entry changed: the top_n of the slot's request, -1 without one"""
        if not self.on:
            return
        want = [-1 if i is None or self.reqs[i].lp is None else self.reqs[i].lp for i in owner]
        changed = [s for s, w in enumerate(want) if w != self.written[s]]
        if changed:
            self.eng.set_logprobs(changed, [want[s] for s in changed])
            for s in changed:
                self.written[s] = want[s]

    def collect(self, running):
        """(slot, request, its new tokens so far): read the rows the host does not hold yet, all in one copy"""
        reads = [(s, i, self.have[i], n - self.have[i]) for s, i, n in running if i in self.rows and n > self.have[i]]
        if not reads:
            return
        total = sum(c for *_, c in reads)
        ids = torch.empty(total, vn.LOGPROB_PLACES, dtype=torch.int32, device=self.dev)
        lp = torch.empty(total, vn.LOGPROB_PLACES, dtype=torch.float32, device=self.dev)
        o = 0
        for s, i, had, c in reads:
            self.eng.read_logprobs(s, self.reqs[i].S + had, c, ids_out=ids[o:o + c], lp_out=lp[o:o + c])
            o += c
        ids, lp = ids.cpu(), lp.cpu()
        o = 0
        for s, i, had, c in reads:
            self.rows[i].append((ids[o:o + c], lp[o:o + c]))
            self.have[i] += c
            o += c

    def result(self):
        out = [None] * len(self.reqs)
        for i, rows in self.rows.items():
            ids = torch.cat([a for a, _ in rows])
            lp = torch.cat([b for _, b in rows])
            out[i] = self.model._logprob_entry(ids, lp, self.reqs[i].lp)
        return out
