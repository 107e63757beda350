"""Generation several tokens per decoder step, from n-gram drafts, with the ids of one token per step.

A verify step feeds [pending input | d1 | ... | dk] as k + 1 segments (`Engine.step(..., segments=...)`): every segment
computes the bits a step of its own computes, so decision j is the one-token loop's decision j as long as d1 .. dj
were that loop's ids.  The loop keeps the decisions up to the first wrong draft plus the model's own token there, and
cuts the stream back to the inputs that produced them: the ids and the KV cache are those of the one-token loop.

The drafts come from prompt lookup over the session's own token ids (`NgramDrafter`): no second model.  How often they
are accepted depends on the text; the cost of a rejected draft is the verify step's extra cost over a one-token step.

Sampled responses keep this exactness: the device draws a row's id from its logits, its KV position and the seed only
(vlo_sample), and segment j of a verify step gets the position and penalty ids the one-token loop has at that token.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Tuple

from .engine import SampleRow

SEP = -1   # a history entry that is not a token id (a frame row): no n-gram spans it and no draft continues past it


class NgramDrafter:
    """Prompt-lookup drafts over one session's ids, one history entry per KV position (frame rows are SEP).

    An index maps every n-gram (n <= max_ngram, no SEP inside) to the positions where its occurrences end, in order, so
    appending or removing an entry costs O(max_ngram).  `propose` takes the longest suffix of the history that occurred
    before and returns the ids that followed its most recent earlier occurrence."""

    def __init__(self, max_ngram: int = 4):
        self.max_ngram = max_ngram
        self.ids: List[int] = []
        self._ends: Dict[Tuple[int, ...], List[int]] = {}

    def __len__(self) -> int:
        return len(self.ids)

    def extend(self, ids: Sequence[int]):
        ids_, ends = self.ids, self._ends
        for t in ids:
            t = int(t)
            ids_.append(t if t >= 0 else SEP)
            end = len(ids_)
            for n in range(1, min(self.max_ngram, end) + 1):
                if ids_[end - n] == SEP:
                    break
                ends.setdefault(tuple(ids_[end - n:end]), []).append(end)

    def truncate(self, n: int):
        ids_, ends = self.ids, self._ends
        while len(ids_) > n:
            end = len(ids_)
            for k in range(1, min(self.max_ngram, end) + 1):
                if ids_[end - k] == SEP:
                    break
                key = tuple(ids_[end - k:end])
                occ = ends[key]
                occ.pop()            # the last occurrence of every n-gram ending here is this one
                if not occ:
                    del ends[key]
            ids_.pop()

    def drop(self, start: int, n: int):
        """Remove history entries [start, start + n), as a context window drops those cache positions: the index is
        rebuilt from the kept entries (cheap: frame rows are SEP and index nothing)."""
        kept = self.ids[:start] + self.ids[start + n:]
        self.ids, self._ends = [], {}
        self.extend(kept)

    def keep(self, spans: Sequence[Tuple[int, int]]):
        """Keep only history entries [first, first + n) of every (first, n) in spans (sorted), as a context window that
        keeps the conversation compacts the cache to them: the index is rebuilt from the kept entries."""
        kept = [t for f, n in spans for t in self.ids[f:f + n]]
        self.ids, self._ends = [], {}
        self.extend(kept)

    def sync(self, n: int):
        """Make the history n entries long: cut it back, or pad it with SEP for KV rows it never saw (a cache filled
        or copied in from elsewhere)."""
        if len(self.ids) > n:
            self.truncate(n)
        elif len(self.ids) < n:
            self.extend([SEP] * (n - len(self.ids)))

    def propose(self, max_k: int) -> List[int]:
        ids_, end = self.ids, len(self.ids)
        if max_k <= 0:
            return []
        for n in range(min(self.max_ngram, end), 0, -1):
            # a suffix without SEP is indexed, its last occurrence is itself; one with a SEP inside is not indexed
            occ = self._ends.get(tuple(ids_[end - n:]))
            if not occ or len(occ) < 2:
                continue
            draft = []
            for t in ids_[occ[-2]:occ[-2] + max_k]:
                if t == SEP:
                    break
                draft.append(t)
            if draft:
                return draft
        return []


def token_tile(rows: int) -> int:
    """Token rows the decoder's weight-streaming GEMMs process for a step of `rows` tokens (bf16 instances, gemm.cu):
    one 16 / 32 / 64 / 96 / 128-row tile, 128-row tiles beyond.  A step moves the same weight bytes for any row count up
    to its tile."""
    for t in (16, 32, 64, 96):
        if rows <= t:
            return t
    return (rows + 127) // 128 * 128


def draft_cap(eng, sid: int, n_prefix: int, remaining: int) -> int:
    """Most drafts the next step of stream `sid` may carry behind a pending input of n_prefix rows, with `remaining`
    ids still wanted: the step keeps the token tile of the pending input alone, leaves room for the model's own token
    after the last draft, stays within max_step_tokens and max_kv_tokens, and gets its pages from the pool (fewer
    drafts, or none, when the pool is short; a step that fails changes no stream)."""
    kv = eng.kv_len(sid)
    k = min(token_tile(n_prefix) - n_prefix, remaining - 1, eng.max_step_tokens - n_prefix,
            eng.max_kv_tokens - kv - n_prefix)
    if k <= 0:
        return 0
    info = eng.kv_pool_info()
    page, free = info["page_tokens"], info["free_pages"]
    held = -(-kv // page)   # a stream holds ceil(kv_len / page) pages
    while k > 0 and -(-(kv + n_prefix + k) // page) - held > free:
        k -= 1
    return k


def sample_rows(sampling, position0: int, history: List[int], n_history: int, n_drafts: int) -> List[SampleRow]:
    """The SampleRow of each segment of a step [pending | d1 .. dk] (k = n_drafts): segment j's token sits at KV
    position position0 + j, and its penalty set is history[:n_history + j] with history = the response's prompt ids,
    the ids generated so far, then d1 .. dk.  These are the position and the ids the one-token loop has at that token,
    so segment j draws the id a step of its own would draw."""
    s = sampling
    return [SampleRow(s.seed, position0 + j, s.temperature, s.top_k, s.top_p, s.repetition_penalty, history,
                      n_history + j) for j in range(n_drafts + 1)]


def generate_ids(eng, sid: int, step: Callable[..., None], n_first: int, max_new: int, eos_token_id: int, *,
                 first_ids: Optional[Sequence[int]] = None, drafter=None, consume: Optional[Callable] = None,
                 base: int = 0, sampling=None, position_base: int = 0) -> List[int]:
    """Ids of stream `sid` until EOS or max_new ids, verifying the drafter's proposals on the way: the argmax, or with
    `sampling` (a SamplingConfig with do_sample) the ids the device draws.

    step(ids, drafts) enqueues one decoder step of the stream over the pending input ids, then the drafts as one-token
    segments (segments [[len(ids), 1, ...]]; no drafts: an ordinary step).  When sampling it is called as
    step(ids, drafts, rows) and passes rows (one SampleRow per segment, `sample_rows`) on as Engine.step(sample=rows).
    The first step's input is n_first rows: ids = first_ids, or None when they are not token ids (the caller feeds its
    own embeddings).  After it, ids is [previous id].  consume(decision) -> decision sees every decision the one-token
    loop would act on, in order, and no other; the loop takes its `sampled_id` when sampling, else its `argmax_id`.
    The drafter's history is the stream's KV from position `base` on (sync / extend / propose).  The penalty set of a
    sampled response is first_ids and the ids generated so far.  position_base is added to the KV positions the samples
    are drawn at: a session under a context window passes the positions it dropped, so no position repeats."""
    if sampling is not None and not sampling.do_sample:
        sampling = None
    out: List[int] = []
    prompt = list(first_ids) if first_ids is not None else []
    pending: Optional[List[int]] = list(first_ids) if first_ids is not None else None
    n_pending = n_first
    pend_ids = pending if pending is not None else [SEP] * n_first
    while len(out) < max_new:
        kv0 = eng.kv_len(sid)
        drafts: List[int] = []
        if drafter is not None:
            drafter.sync(kv0 - base)
            drafter.extend(pend_ids)
            k = draft_cap(eng, sid, n_pending, max_new - len(out)) if pending is not None else 0
            drafts = [int(t) for t in drafter.propose(k)[:k]] if k > 0 else []
            drafter.extend(drafts)
        try:
            if sampling is None:
                step(pending, drafts)
            else:
                step(pending, drafts, sample_rows(sampling, position_base + kv0 + n_pending - 1, prompt + out + drafts,
                                                  len(prompt) + len(out), len(drafts)))
        except Exception:
            if drafter is not None:
                drafter.sync(kv0 - base)
            raise
        decs = eng.read_decisions(1 + len(drafts))
        j = 0
        for j, dec in enumerate(decs):
            if consume is not None:
                dec = consume(dec)
            new_id = dec.argmax_id if sampling is None else dec.sampled_id
            out.append(new_id)
            if new_id == eos_token_id or len(out) == max_new or j == len(drafts) or drafts[j] != new_id:
                break
        if j < len(drafts):   # drafts j .. k - 1 were not the loop's inputs: drop them
            eng.kv_truncate(sid, kv0 + n_pending + j)
            if drafter is not None:
                drafter.sync(kv0 + n_pending + j - base)
        if out[-1] == eos_token_id:
            break
        pending = pend_ids = [out[-1]]
        n_pending = 1
    return out


greedy_generate = generate_ids   # the loop without `sampling`
