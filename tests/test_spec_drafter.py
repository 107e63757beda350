"""The n-gram drafter and the draft caps of speculative greedy generation, on the host (no GPU)."""
import pytest

from videollm_online_b200.speculative import SEP, NgramDrafter, draft_cap, greedy_generate, token_tile


def test_proposes_what_followed_the_last_earlier_occurrence():
    d = NgramDrafter()
    d.extend([5, 6, 7, 8, 9, 1, 5, 6])
    assert d.propose(3) == [7, 8, 9]
    assert d.propose(10) == [7, 8, 9, 1, 5, 6]   # an occurrence may run into the suffix itself
    d.extend([2, 5, 6])
    assert d.propose(2) == [2, 5]                # the most recent earlier occurrence wins


def test_longest_matching_suffix_wins():
    d = NgramDrafter(max_ngram=3)
    d.extend([1, 2, 3, 10, 9, 2, 3, 20, 1, 2, 3])
    assert d.propose(1) == [10]                  # [1, 2, 3] matched, not the later [2, 3] -> 20
    d2 = NgramDrafter(max_ngram=3)
    d2.extend([4, 2, 3, 10, 9, 2, 3, 20, 1, 2, 3])
    assert d2.propose(1) == [20]                 # only [2, 3] matches: its last earlier occurrence


def test_no_match_no_draft():
    d = NgramDrafter()
    assert d.propose(4) == []
    d.extend([1, 2, 3])
    assert d.propose(4) == []
    assert d.propose(0) == []


def test_separators_break_ngrams_and_drafts():
    d = NgramDrafter()
    d.extend([7, 8, SEP, 9, 7, 8])
    assert d.propose(4) == []                    # what followed [7, 8] is a frame row
    d.extend([SEP, 3])
    assert d.propose(4) == []                    # [.., SEP, 3]: no earlier 3
    e = NgramDrafter()
    e.extend([1, SEP, 2, 3, 1])
    assert e.propose(4) == []                    # [SEP, 1] is not an n-gram, and 1 was followed by a frame row
    e.extend([-5])                               # any negative id is a separator
    assert e.ids[-1] == SEP


def test_truncate_restores_the_index():
    d = NgramDrafter()
    d.extend([1, 2, 3, 4, 1, 2])
    assert d.propose(2) == [3, 4]
    d.extend([9, 9, 1, 2])
    assert d.propose(2) == [9, 9]
    d.truncate(6)                                # back to [1, 2, 3, 4, 1, 2]
    assert d.ids == [1, 2, 3, 4, 1, 2] and d.propose(2) == [3, 4]
    fresh = NgramDrafter()
    fresh.extend([1, 2, 3, 4, 1, 2])
    assert d._ends == fresh._ends
    d.truncate(0)
    assert d.ids == [] and d._ends == {}


def test_sync_pads_with_separators():
    d = NgramDrafter()
    d.extend([1, 2])
    d.sync(5)
    assert d.ids == [1, 2, SEP, SEP, SEP]
    d.sync(1)
    assert d.ids == [1]


def test_token_tile():
    assert [token_tile(t) for t in (1, 16, 17, 32, 33, 64, 65, 96, 97, 128, 129)] == \
        [16, 16, 32, 32, 64, 64, 96, 96, 128, 128, 256]


class FakeEngine:
    """kv lengths, a page pool and scripted decisions: enough of Engine for the generation loop"""

    def __init__(self, kv=0, max_step_tokens=128, max_kv_tokens=4096, free_pages=1000, page=64, script=()):
        self.kv, self.max_step_tokens, self.max_kv_tokens = kv, max_step_tokens, max_kv_tokens
        self.free, self.page = free_pages, page
        self.script = list(script)      # the model's greedy ids, one per input position after the prompt
        self.steps = []

    def kv_len(self, sid):
        return self.kv

    def kv_pool_info(self):
        return {"page_tokens": self.page, "total_pages": 10 ** 6, "free_pages": self.free}

    def kv_truncate(self, sid, n):
        assert n <= self.kv
        self.kv = n

    def read_decisions(self, n):
        return self._decs[:n]


class Dec:
    def __init__(self, i):
        self.argmax_id = i


def test_draft_caps():
    e = FakeEngine(kv=100)
    assert draft_cap(e, 0, 1, 100) == 15          # the one-token step keeps its 16-row tile
    assert draft_cap(e, 0, 20, 100) == 12         # a 20-token prompt keeps its 32-row tile
    assert draft_cap(e, 0, 1, 4) == 3             # room for the model's own token after the last draft
    assert draft_cap(e, 0, 1, 1) == 0
    assert draft_cap(e, 0, 200, 100) == 0         # a chunked prompt carries none
    assert draft_cap(FakeEngine(kv=100, max_step_tokens=8), 0, 1, 100) == 7
    assert draft_cap(FakeEngine(kv=4090, max_kv_tokens=4096), 0, 1, 100) == 5
    # kv 120 holds 2 pages; 0 free pages leave room up to 128 tokens: 7 drafts after the pending token
    assert draft_cap(FakeEngine(kv=120, free_pages=0), 0, 1, 100) == 7
    assert draft_cap(FakeEngine(kv=128, free_pages=0), 0, 1, 100) == 0


def _run_loop(script, drafts_of, max_new=100, eos=2, kv=50, **kw):
    """the loop over a fake model whose greedy id at response position i is script[i]; drafts_of(i) proposes"""
    e = FakeEngine(kv=kv, script=script, **kw)
    consumed = []

    class Drafter:
        def __init__(self):
            self.pos = 0

        def sync(self, n):
            pass

        def extend(self, ids):
            pass

        def propose(self, k):
            return drafts_of(len(out_so_far))[:k]

    out_so_far = []

    def step(ids, drafts):
        e.steps.append((None if ids is None else list(ids), list(drafts)))
        i = len(out_so_far)
        e._decs = [Dec(script[min(i + j, len(script) - 1)]) for j in range(len(drafts) + 1)]
        e.kv += (len(ids) if ids is not None else 3) + len(drafts)

    def consume(d):
        consumed.append(d.argmax_id)
        out_so_far.append(d.argmax_id)
        return d
    out = greedy_generate(e, 0, step, 3, max_new, eos, first_ids=[7, 7, 7], drafter=Drafter(), consume=consume)
    return out, consumed, e


def test_loop_accepts_the_matching_prefix_and_cuts_the_rest():
    script = [10, 11, 12, 13, 2]
    out, consumed, e = _run_loop(script, lambda i: script[i:i + 3][:2] + [99])
    assert out == script and consumed == script
    assert e.kv == 50 + 3 + 4          # prompt + every id but the EOS, as one token per step leaves it
    out, consumed, e = _run_loop(script, lambda i: [])
    assert out == script and len(e.steps) == 5 and e.kv == 57


def test_loop_stops_at_the_buffer_end_inside_a_run():
    script = list(range(10, 30))
    out, consumed, e = _run_loop(script, lambda i: script[i:i + 15], max_new=6)
    assert out == script[:6] and consumed == out
    assert e.kv == 50 + 3 + 5
    assert all(len(d) <= 6 - 1 for _, d in e.steps[:1])


def test_loop_with_wrong_drafts_at_every_position():
    script = [10, 11, 12, 13, 14, 2]
    for bad in range(4):
        def drafts_of(i, bad=bad):
            d = script[i:i + 4]
            return [x + 1000 if j == bad else x for j, x in enumerate(d)]
        out, consumed, e = _run_loop(script, drafts_of)
        assert out == script and consumed == script and e.kv == 50 + 3 + 5


def test_loop_without_a_drafter_is_one_token_per_step():
    e = FakeEngine(kv=0)
    script = [5, 6, 2]
    seen = []

    def step(ids, drafts):
        assert drafts == []
        seen.append(ids)
        e._decs = [Dec(script[len(seen) - 1])]
        e.kv += 1
    assert greedy_generate(e, 0, step, 1, 100, 2, first_ids=[1]) == script
    assert seen == [[1], [5], [6]]


@pytest.mark.parametrize("max_ngram", [1, 2, 4])
def test_drafter_over_a_repeating_text(max_ngram):
    text = [3, 4, 5, 6] * 5
    d = NgramDrafter(max_ngram=max_ngram)
    d.extend(text[:8])
    assert d.propose(4) == [3, 4, 5, 6]
