"""Response sampling on the host side: SamplingConfig validation, the CLI flags, the SampleRow of every segment of a
verify step, the SessionState round trip with a sampling config, and the NumPy Philox restatement the GPU tests use."""
import io

import numpy as np
import pytest
import torch

from sampling_reference import gumbel, philox4x32_10


def test_sampling_config_validation():
    from videollm_online_b200.config import SamplingConfig
    c = SamplingConfig()
    assert (c.do_sample, c.temperature, c.top_k, c.top_p, c.repetition_penalty, c.seed) == (False, 1.0, 50, 1.0, 1.0, 0)
    SamplingConfig(do_sample=True, temperature=0.6, top_p=0.9, top_k=0, repetition_penalty=1.2, seed=2 ** 64 - 1)
    for bad in (dict(temperature=0.0), dict(temperature=-1.0), dict(temperature=float("inf")),
                dict(temperature=float("nan")), dict(top_k=-1), dict(top_k=2.5), dict(top_p=0.0), dict(top_p=1.5),
                dict(top_p=float("nan")), dict(repetition_penalty=0.0), dict(seed=-1), dict(seed=2 ** 64)):
        with pytest.raises(ValueError):
            SamplingConfig(do_sample=True, **bad)
    with pytest.raises(ValueError, match="do_sample"):
        SamplingConfig(repetition_penalty=1.3)      # a penalty on a greedy response would be ignored


def test_cli_flags():
    from videollm_online_b200.config import SamplingConfig, parse_args
    a = parse_args([])
    assert SamplingConfig.from_args(a) is None and a.seed == 0
    a = parse_args(["--do_sample", "--temperature", "0.6", "--top_p", "0.9", "--top_k", "0", "--repetition_penalty",
                    "1.1", "--sample_seed", "7", "--seed", "3", "--synthetic_weights", "true"])
    assert a.synthetic_weights is True and a.seed == 3
    assert SamplingConfig.from_args(a) == SamplingConfig(True, 0.6, 0, 0.9, 1.1, 7)
    assert SamplingConfig.from_args(parse_args(["--do_sample", "false", "--temperature", "0.5"])) is None
    with pytest.raises(ValueError):
        SamplingConfig.from_args(parse_args(["--do_sample", "--top_p", "0"]))


def test_verify_step_rows_match_one_token_loop():
    """Segment j of [pending | d1 .. dk] gets the KV position and the penalty ids the one-token loop has at that token"""
    from videollm_online_b200.config import SamplingConfig
    from videollm_online_b200.speculative import sample_rows
    cfg = SamplingConfig(do_sample=True, temperature=0.7, top_k=20, top_p=0.9, repetition_penalty=1.2, seed=99)
    prompt, out, drafts = [5, 6, 7], [40, 41], [42, 43, 44]
    kv0, n_pending = 500, 1
    hist = prompt + out + drafts
    rows = sample_rows(cfg, kv0 + n_pending - 1, hist, len(prompt) + len(out), len(drafts))
    assert len(rows) == 4
    for j, r in enumerate(rows):
        assert r.position == kv0 + j                      # the one-token loop's step j reads its logits here
        assert list(r.penalty_ids[:r.n_penalty]) == prompt + out + drafts[:j]
        assert (r.seed, r.temperature, r.top_k, r.top_p, r.repetition_penalty) == (99, 0.7, 20, 0.9, 1.2)
    assert all(r.penalty_ids is hist for r in rows)       # one list: the engine uploads it once


def test_session_state_round_trip_with_sampling():
    from videollm_online_b200.config import SamplingConfig
    from videollm_online_b200.engine import KvImage
    from videollm_online_b200.inference import SessionState
    img = KvImage(torch.zeros(2 * 2 * 2 * 64 * 128 * 2, dtype=torch.uint8), 40, (2, 2, 128, 64))
    cfg = SamplingConfig(do_sample=True, temperature=0.6, top_p=0.9, seed=12345678901234)
    st = SessionState(kv=img, last_ids=torch.tensor([[11]]), video_time=1.0, last_frame_idx=2, query_queue=[],
                      frame_embeds_queue=[], drafter_ids=None, n_calls=3, started=True, sampling=cfg)
    buf = io.BytesIO()
    torch.save(st, buf)
    buf.seek(0)
    got = torch.load(buf)
    assert got.sampling == cfg and isinstance(got.sampling, SamplingConfig)
    old = SessionState(kv=img, last_ids=torch.tensor([[11]]), video_time=1.0, last_frame_idx=2, query_queue=[],
                       frame_embeds_queue=[], drafter_ids=None, n_calls=3, started=True)
    assert old.sampling is None


def test_philox_known_answers():
    """Random123's known-answer vectors for philox4x32_10"""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
             ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
             ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
              (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in cases:
        got = philox4x32_10([np.array([c]) for c in ctr], key)
        assert tuple(int(w[0]) for w in got) == want


def test_gumbel_noise_layout():
    g = gumbel(0x1234_5678_9ABC_DEF0, 77, 1024)
    assert g.shape == (1024,) and np.isfinite(g).all()
    w = philox4x32_10([np.array([5]), np.array([77]), np.array([0]), np.array([0])], (0x9ABCDEF0, 0x12345678))
    u = ((int(w[2][0]) >> 8) + 0.5) * 2.0 ** -24     # id 22 = word 2 of counter 5
    assert g[22] == -np.log(-np.log(u))
    assert not np.array_equal(g, gumbel(0x1234_5678_9ABC_DEF0, 78, 1024))
