"""The context window's host side (no GPU): the eviction policy, the drafter's history under an eviction, the window's
validation, the --context_window flag and the rotation vlo_kv_evict is given."""
import math
import random

import pytest
import torch

from videollm_online_b200 import VloError, tiny_config
from videollm_online_b200 import weights as W
from videollm_online_b200.config import parse_args
from videollm_online_b200.engine import check_context_window, evict_span, sink_tokens
from videollm_online_b200.speculative import SEP, NgramDrafter

P = 64


def test_no_eviction_while_the_step_fits():
    assert evict_span(1000, 24, 1024, 30, P) == (0, 0)
    assert evict_span(0, 1024, 1024, 30, P) == (0, 0)


def test_the_sink_stays_and_the_floor_is_window_over_8_in_pages():
    # window 1024: floor 128 tokens = 2 pages; one token over needs 1 page, the floor makes it 2
    assert evict_span(1024, 1, 1024, 30, P) == (64, 128)
    # the sink is ceil(keep / 64) pages
    assert evict_span(1024, 1, 1024, 64, P) == (64, 128)
    assert evict_span(1024, 1, 1024, 65, P) == (128, 128)
    assert evict_span(1024, 1, 1024, 0, P) == (0, 128)
    # window 1000: floor ceil(125 / 64) = 2 pages
    assert evict_span(990, 11, 1000, 30, P) == (64, 128)


def test_the_fewest_pages_above_the_floor():
    # 300 tokens over a 1024 window: ceil(300 / 64) = 5 pages > the 2-page floor
    assert evict_span(1000, 324, 1024, 30, P) == (64, 5 * 64)
    # exactly 3 pages over
    assert evict_span(1024, 192, 1024, 30, P) == (64, 192)


def test_the_floor_is_clipped_to_the_full_pages_there_are():
    # 200 cached: pages [64, 128) and [128, 192) are full after the sink; 200 + 100 > 250 needs 1 page, the floor
    # (ceil(31.25 / 64) = 1 page) asks for 1, so 1
    assert evict_span(200, 100, 250, 30, P) == (64, 64)
    # window 4096 (floor 8 pages), 4 full pages after the sink, 1 needed: all 4 go
    assert evict_span(320, 3800, 4096, 30, P) == (64, 256)


def test_impossible_room_raises():
    with pytest.raises(VloError, match="do not fit"):
        evict_span(200, 200, 250, 30, P)          # even both full pages after the sink leave 72 + 200 > 250
    with pytest.raises(VloError):
        evict_span(100, 200, 250, 30, P)


def test_random_policy_properties():
    rng = random.Random(0)
    for _ in range(3000):
        window = rng.randrange(256, 20000)
        keep = rng.randrange(0, 200)
        kv = rng.randrange(0, window + 1)
        need = rng.randrange(1, 400)
        try:
            first, n = evict_span(kv, need, window, keep, P)
        except VloError:
            assert kv + need > window
            assert sink_tokens(keep, P) + kv % P + need > window or kv < sink_tokens(keep, P) + P
            continue
        if kv + need <= window:
            assert n == 0
            continue
        assert first == sink_tokens(keep, P) and first % P == 0 and n % P == 0 and n > 0
        assert first + n <= kv // P * P                       # whole, full pages
        assert kv - n + need <= window                        # room made
        least = -(-(kv + need - window) // P) * P
        floor = -(-window // (8 * P)) * P
        assert n == min(kv // P * P - first, max(least, floor))


def _rebuilt(ids):
    d = NgramDrafter()
    d.extend(ids)
    return d


def test_drafter_drop_equals_a_drafter_of_the_kept_ids():
    rng = random.Random(1)
    for _ in range(200):
        ids = [rng.choice([SEP, SEP, 3, 4, 5, 6, 7]) for _ in range(rng.randrange(0, 300))]
        d = _rebuilt(ids)
        start = rng.randrange(0, len(ids) + 1)
        n = rng.randrange(0, len(ids) - start + 1)
        d.drop(start, n)
        want = _rebuilt(ids[:start] + ids[start + n:])
        assert d.ids == want.ids and d._ends == want._ends
        for k in (1, 3, 8):
            assert d.propose(k) == want.propose(k)


def test_window_validation():
    check_context_window(1024, 2048, 30, 110, P)
    with pytest.raises(ValueError, match="max_kv_tokens"):
        check_context_window(4096, 2048, 30, 110, P)
    with pytest.raises(ValueError, match="must be >="):
        check_context_window(256, 2048, 30, 200, P)   # 64 sink + 64 chunk + 200 > 256
    check_context_window(328, 2048, 30, 200, P)
    for bad in (0, -64, 1.5, True, None):
        with pytest.raises(ValueError):
            check_context_window(bad, 2048, 30, 110, P)


def test_context_window_flag():
    assert parse_args([]).context_window == 0
    assert parse_args(["--context_window", "13312"]).context_window == 13312


def test_rotation_uses_the_tables_frequencies():
    cfg = tiny_config()
    inv = W.rope_inv_freq(cfg)
    assert inv.dtype == torch.float32 and inv.numel() == cfg.head_dim // 2
    d = cfg.head_dim
    old = 1.0 / (cfg.rope_theta ** (torch.arange(0, d, 2, dtype=torch.int64).to(dtype=torch.float) / d))
    assert torch.equal(inv, old)
    cos, _ = W.rope_tables(cfg, 300, "cpu")
    assert torch.equal(cos, (torch.arange(300, dtype=torch.float32)[:, None] * old[None, :]).cos().to(torch.bfloat16))
    for delta in (64, 1664, 8320):
        c, s = W.rope_rotation(cfg, delta)
        assert c.dtype == torch.float32 and c.shape == (d // 2,)
        for j in (0, 1, 17, 63):
            ang = float(inv[j]) * delta           # fp64 from the fp32 frequency
            assert float(c[j]) == float(torch.tensor(math.cos(ang), dtype=torch.float32))
            assert float(s[j]) == float(torch.tensor(math.sin(ang), dtype=torch.float32))


def test_old_session_states_load_with_no_evictions():
    from videollm_online_b200.inference import SessionState
    st = SessionState(kv=None, last_ids=torch.zeros(1, 1), video_time=0.0, last_frame_idx=-1, query_queue=[],
                      frame_embeds_queue=[], drafter_ids=None, n_calls=0, started=False)
    assert st.evicted_tokens == 0
