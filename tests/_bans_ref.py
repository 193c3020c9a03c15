"""The banned-token rules of DESIGN.md section 3 ("Banned tokens") restated in plain Python: HF's
NoRepeatNGramLogitsProcessor, NoBadWordsLogitsProcessor and MinNewTokensLengthLogitsProcessor as sets of token ids.

A draw at cache column c sees the row's ids h[0 .. c) (HF's input_ids: left padding, video placeholders, prompt and
every token so far)."""


def ngram_bans(h, n):
    """no_repeat_ngram_size n (0: off): if c + 1 >= n, h[i + n - 1] for every i in 0 .. c - n whose n - 1 ids equal
    the last n - 1 ids of the row"""
    c = len(h)
    if n <= 0 or c + 1 < n:
        return set()
    key = list(h[c - n + 1:c])
    return {h[i + n - 1] for i in range(c - n + 1) if list(h[i:i + n - 1]) == key}


def word_bans(h, words, eos=None):
    """bad_words_ids (None: off): a word equal to [eos] is dropped; a one-id word is always banned; a longer word w
    bans w[-1] when len(w) <= c and the row ends with w[:-1]"""
    if words is None:
        return set()
    c = len(h)
    out = set()
    for w in words:
        if eos is not None and list(w) == [eos]:
            continue
        if len(w) == 1:
            out.add(w[0])
        elif len(w) <= c and list(h[c - len(w) + 1:]) == list(w[:-1]):
            out.add(w[-1])
    return out


def eos_bans(h, eos, S, m):
    """min_new_tokens m: EOS while c < S + m (S the first new token's column); nothing when EOS is disabled"""
    if eos is None or not m or len(h) >= S + m:
        return set()
    return {eos}


def banned(h, ngram=0, words=None, eos=None, S=0, min_new=0):
    """every id a draw after h bans"""
    return ngram_bans(h, ngram) | word_bans(h, words, eos) | eos_bans(h, eos, S, min_new)
