"""A context window that keeps the conversation, host side (no GPU): the retention policy (`engine.retain_spans`) on
scripted histories and on rendered conversations (the kept ids are what the chat template renders for the same
conversation with some frames and turns deleted), the window's validation, the drafter's multi-span drop and the
--context_keep_turns flag."""
import random

import pytest

from videollm_online_b200 import VloError, tiny_config
from videollm_online_b200.config import parse_args
from videollm_online_b200.engine import check_context_window_turns, kept_rows, retain_spans
from videollm_online_b200.speculative import SEP, NgramDrafter
from videollm_online_b200.tokenization_live import ByteTokenizer

I = 11          # interval id
FNT = 10        # rows per frame
F = [-1] * FNT  # one frame's rows


def _dropped(spans, n):
    kept = {p for f, k in spans for p in range(f, f + k)}
    return [p for p in range(n) if p not in kept]


def _stream(n_frames, interval=True):
    out = []
    for j in range(n_frames):
        out += ([I] if j and interval else []) + F
    return out


PROMPT = [1, 50, 51, 52, 40, 41]   # bos, system text, "\n["


def test_nothing_goes_while_the_step_fits():
    h = PROMPT + _stream(5)
    assert retain_spans(h, 10, len(h) + 10, len(PROMPT), I, FNT) == []


def test_the_oldest_frames_go_first_whole_with_their_interval_row():
    h = PROMPT + _stream(40)                         # 6 + 40 * 10 + 39 = 445 rows
    window = 448
    spans = retain_spans(h, 11, window, len(PROMPT), I, FNT)
    gone = _dropped(spans, len(h))
    assert spans[0] == (0, len(PROMPT))              # the prompt stays exactly
    # window / 8 = 56 tokens: 6 frame units of 11 rows (66 >= 56), the oldest ones
    assert gone == list(range(len(PROMPT), len(PROMPT) + 6 * (FNT + 1)))
    assert len(gone) >= window // 8 and len(h) - len(gone) + 11 <= window


def _turn(text_len):
    # "]\n" then text, ending with "\n[" (the text run between two stream messages)
    return [933] + [100 + k % 50 for k in range(text_len - 3)] + [40, 41]


def test_turns_stay_under_the_budget_and_the_oldest_goes_past_it():
    # messages of 4 frames separated by turns of 30 rows
    h, turn_at = list(PROMPT), []
    for m in range(8):
        h += _stream(4)
        if m < 7:
            turn_at.append(len(h))
            h += _turn(30)
    window = 400
    spans = retain_spans(h, 11, window, len(PROMPT), I, FNT)
    gone = set(_dropped(spans, len(h)))
    # 7 turns x 30 = 210 text rows > 200 = window / 2: the oldest turn goes with the frame before it
    t0 = turn_at[0]
    assert set(range(t0 - FNT, t0 + 30)) <= gone
    assert all(not set(range(t, t + 30)) & gone for t in turn_at[1:])     # every other turn stays whole
    # the rest are the oldest frames; never the last frame of a message alone
    for t in turn_at[1:]:
        assert not set(range(t - FNT, t)) & gone
    assert len(gone) >= window // 8 and len(h) - len(gone) + 11 <= window
    # no partial frame anywhere
    runs, cur = [], []
    for p in range(len(h)):
        if h[p] == -1:
            cur.append(p)
        elif cur:
            runs.append(cur)
            cur = []
    runs.append(cur)
    for r in runs:
        for k in range(0, len(r), FNT):
            fr = set(r[k:k + FNT])
            assert fr <= gone or not fr & gone


def test_every_turn_is_kept_under_the_budget_even_when_frames_run_short():
    h = list(PROMPT)
    for m in range(5):
        h += _stream(6)
        if m < 4:
            h += _turn(20)
    spans = retain_spans(h, 11, 300, len(PROMPT), I, FNT)
    kept = kept_rows(h, spans)
    assert kept.count(933) == 4                          # every turn stays
    assert len(kept) + 11 <= 300


def test_it_raises_when_nothing_that_may_go_is_enough():
    h = PROMPT + _stream(1) + _turn(100)                  # one frame, then a long trailing turn: nothing may go
    with pytest.raises(VloError, match="do not fit"):
        retain_spans(h, 11, len(h), len(PROMPT), I, FNT)
    with pytest.raises(VloError, match="whole frames"):
        retain_spans(PROMPT + [-1] * 7, 100, 50, len(PROMPT), I, FNT)


# ------------------------------------------------------------------------------------------------ the template
def _conversation(rng, n_msgs):
    """[(n_frames, turn messages or None)] : stream messages, each followed by a turn (the last one stays open)"""
    conv = []
    for m in range(n_msgs):
        turn = None
        if m < n_msgs - 1:
            q = "".join(rng.choice("abcdefgh") for _ in range(rng.randint(3, 25)))
            r = " " + "".join(rng.choice("xyz ") for _ in range(rng.randint(2, 30)))
            turn = [{"role": "user", "content": q}, {"role": "assistant", "content": r}] if rng.random() < 0.6 \
                else [{"role": "assistant", "content": r}]
        conv.append((rng.randint(1, 9), turn))
    return conv


def _render(tok, cfg, conv):
    """ids of the system prompt and the conversation as LiveInfer feeds it: frame rows -1, the last message open"""
    msgs = [{"role": "system", "content": "sys prompt"}]
    for n, turn in conv:
        if n:
            msgs.append({"role": "stream", "num_frames": n})
        msgs += turn or []
    ids = tok.apply_chat_template(msgs)
    assert ids[-1] == tok.encode("]")[0]
    return [-1 if t == cfg.v_placeholder_id else t for t in ids[:-1]]


@pytest.mark.parametrize("version", ["live1+", "live1"])
def test_kept_ids_are_the_template_of_a_shorter_conversation(version):
    over = {} if version == "live1+" else dict(frame_token_pooled=None, frame_num_tokens=1, frame_token_interval="")
    cfg = tiny_config(**over)
    tok = ByteTokenizer(cfg)
    iid = cfg.frame_token_interval_id if cfg.frame_token_interval else None
    prompt = tok.apply_chat_template([{"role": "system", "content": "sys prompt"}], add_stream_prompt=True)
    rng = random.Random(0 if iid else 1)
    checked = turns_dropped = 0
    for trial in range(40):
        conv = _conversation(rng, rng.randint(3, 14))
        full = _render(tok, cfg, conv)
        assert full[:len(prompt)] == prompt
        # positions -> (message, frame of it) or (turn index); built from the conversation
        p = len(prompt)
        pos_frame, pos_turn = [None] * len(full), [None] * len(full)
        for m, (n, turn) in enumerate(conv):
            for j in range(n):
                for _ in range(cfg.frame_num_tokens):
                    pos_frame[p] = (m, j)
                    p += 1
                if j < n - 1 and iid is not None:
                    pos_frame[p] = (m, j)
                    p += 1
            if turn is not None:
                while p < len(full) and full[p] != -1:
                    pos_turn[p] = m
                    p += 1
        assert p == len(full)
        window = rng.choice([200, 260, 400])
        need = rng.randint(1, 20)
        try:
            spans = retain_spans(full, need, window, len(prompt), iid, cfg.frame_num_tokens)
        except VloError:
            continue
        if not spans:
            continue
        kept_ids = kept_rows(full, spans)
        assert len(kept_ids) + need <= window
        keep = set(p for f, n in spans for p in range(f, f + n))
        # the shorter conversation: kept frames per message; a dropped turn merges its two messages
        frames_kept = [0] * len(conv)
        for q in keep:
            if pos_frame[q] is not None and full[q] == -1:
                frames_kept[pos_frame[q][0]] += 1
        turn_kept = [conv[m][1] is not None and all(q in keep for q in range(len(full)) if pos_turn[q] == m)
                     for m in range(len(conv))]
        for m in range(len(conv)):           # a turn goes whole or not at all
            rows = [q for q in range(len(full)) if pos_turn[q] == m]
            assert all(q in keep for q in rows) or not any(q in keep for q in rows)
        short, acc = [], 0
        for m, (n, turn) in enumerate(conv):
            acc += frames_kept[m] // cfg.frame_num_tokens
            if turn is None:
                short.append((acc, None))
            elif turn_kept[m]:
                assert acc > 0                # a message that stays keeps a frame
                short.append((acc, turn))
                acc = 0
        assert kept_ids == _render(tok, cfg, short), trial
        checked += 1
        turns_dropped += sum(conv[m][1] is not None and not turn_kept[m] for m in range(len(conv)))
        # the turn budget holds whenever a turn went
        text_rows = sum(1 for q in keep if q >= len(prompt) and pos_turn[q] is not None)
        if not all(turn_kept[m] for m in range(len(conv)) if conv[m][1] is not None):
            assert text_rows <= window // 2 or len(kept_ids) + need > window - window // 8
    assert checked >= 10 and turns_dropped > 0


def test_repeated_evictions_keep_the_template_and_every_recent_turn():
    """Feed a long rendered conversation in steps, evicting before each; the kept ids stay a rendering throughout."""
    cfg = tiny_config()
    tok = ByteTokenizer(cfg)
    iid = cfg.frame_token_interval_id
    prompt = tok.apply_chat_template([{"role": "system", "content": "sys prompt"}], add_stream_prompt=True)
    rng = random.Random(3)
    conv = _conversation(rng, 60)
    full = _render(tok, cfg, conv)
    window = 512
    hist, n_evict = list(full[:len(prompt)]), 0
    p = len(prompt)
    while p < len(full):
        q = p + 1
        while q < len(full) and not (full[q] == -1 and full[q - 1] != -1):
            q += 1
        step = full[p:q]
        spans = retain_spans(hist, len(step), window, len(prompt), iid, cfg.frame_num_tokens)
        if spans:
            n_evict += 1
            dropped = len(hist) - sum(n for _, n in spans)
            assert dropped >= window // 8
            hist = kept_rows(hist, spans)
        hist += step
        assert len(hist) <= window
        p = q
    assert n_evict > 5
    assert hist[:len(prompt)] == prompt
    # the most recent turns are all there, in order
    last_turns = [t for _, t in conv if t is not None][-3:]
    txt = tok.decode([t for t in hist if t >= 0], skip_special_tokens=False)
    for t in last_turns:
        for m in t:
            assert m["content"] in txt


# ------------------------------------------------------------------------------------------------ validation, drafter, flag
def test_window_validation():
    check_context_window_turns(1024, 2048, 30, 110)
    with pytest.raises(ValueError, match="positive"):
        check_context_window_turns(0, 2048, 30, 110)
    with pytest.raises(ValueError, match="max_kv_tokens"):
        check_context_window_turns(4096, 2048, 30, 110)
    # prompt + window / 2 + window / 8 + step: 30 + 200 + 50 + 110 = 390 <= 400; 30 + 185 + 47 + 110 = 372 > 370
    check_context_window_turns(400, 2048, 30, 110)
    with pytest.raises(ValueError, match="turn budget"):
        check_context_window_turns(370, 2048, 30, 110)


def test_drafter_multi_span_drop_equals_a_rebuild():
    rng = random.Random(5)
    for _ in range(20):
        ids = [rng.choice([SEP, 3, 4, 5, 6, 7]) for _ in range(rng.randint(20, 200))]
        d = NgramDrafter()
        d.extend(ids)
        cuts = sorted(rng.sample(range(len(ids) + 1), 6))
        spans = [(cuts[k], cuts[k + 1] - cuts[k]) for k in (0, 2, 4) if cuts[k + 1] > cuts[k]]
        d.keep(spans)
        ref = NgramDrafter()
        ref.extend(kept_rows(ids, spans))
        assert d.ids == ref.ids and d._ends == ref._ends
        for k in range(1, 6):
            assert d.propose(k) == ref.propose(k)


def test_flag():
    assert parse_args([]).context_keep_turns is False
    assert parse_args(["--context_window", "4096", "--context_keep_turns"]).context_keep_turns is True
