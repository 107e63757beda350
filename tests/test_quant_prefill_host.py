"""quantized_prefill on the host: the flag rules of build_live / build_model_and_tokenizer, LiveArguments and the CLI,
and session states, which do not record the flag: a state saved on a prefilling quantized engine resumes on one that
chunks, and the other way round (both compute the same bits)."""
import dataclasses
import threading

import pytest
import torch

import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import tiny_config


def test_flag_needs_a_quantized_layer_form():
    from videollm_online_b200.modeling_live import build_live, build_model_and_tokenizer
    cfg = tiny_config()
    for build in (build_live, build_model_and_tokenizer):
        with pytest.raises(ValueError, match="quantized_prefill"):
            build(config=cfg, quantized_prefill=True, synthetic_weights=True, device="cpu")
        with pytest.raises(ValueError, match="quantized_prefill"):
            build(config=cfg, quantized_prefill=True, fp8_activations=False, quantize_vocab=False, synthetic_weights=True,
                  device="cpu")


def test_liveinfer_arguments_reach_build_live(monkeypatch):
    """LiveInfer hands every LiveArguments field to build_model_and_tokenizer, quantized_prefill included"""
    from videollm_online_b200 import inference
    from videollm_online_b200.config import LiveArguments
    seen = {}

    def fake_build(**kw):
        seen.update(kw)
        raise RuntimeError("stop")
    monkeypatch.setattr(inference, "build_model_and_tokenizer", fake_build)
    with pytest.raises(RuntimeError, match="stop"):
        inference.LiveInfer(LiveArguments(int4_weights=True, quantized_prefill=True), device="cpu")
    assert seen["quantized_prefill"] is True and seen["int4_weights"] is True


def test_cli_flag_parses():
    from videollm_online_b200.config import LiveArguments
    from videollm_online_b200.inference import parse_args
    assert LiveArguments().quantized_prefill is False
    assert parse_args([]).quantized_prefill is False
    args = parse_args(["--fp8_weights", "--quantized_prefill"])
    assert args.quantized_prefill is True and args.fp8_weights is True
    assert parse_args(["--int4_weights", "true", "--quantized_prefill", "false"]).quantized_prefill is False


# ============================================================================================ session states
def _state(**kw):
    from videollm_online_b200.inference import SessionState
    return SessionState(kv=None, last_ids=torch.zeros(1), video_time=0.0, last_frame_idx=0, query_queue=[],
                        frame_embeds_queue=[], drafter_ids=None, n_calls=0, started=False, **kw)


def test_session_state_has_no_prefill_field(tmp_path):
    from videollm_online_b200.inference import SessionState
    assert not any("prefill" in f.name for f in dataclasses.fields(SessionState))
    state = _state(int4_weights=True)
    path = tmp_path / "s.pt"
    torch.save(state, path)
    loaded = torch.load(path, weights_only=True)
    assert loaded.int4_weights is True and loaded.fp8_weights is False


class _Accepted(Exception):
    pass


class _FakeEngine:
    fp8_weights, fp8_activations, int4_weights, quantized_vocab = False, False, True, False

    def __init__(self, prefills):
        self.prefills = prefills

    def stream_reset(self, sid):
        raise _Accepted()   # resume got past every check of the state's form


class _FakeKV:
    def __init__(self, engine):
        self.engine, self.stream_id = engine, 0


@pytest.mark.parametrize("ours", [True, False])
def test_resume_accepts_a_state_of_either_prefill_mode(ours):
    from videollm_online_b200.inference import LiveInfer
    live = LiveInfer.__new__(LiveInfer)     # only what resume reads before it touches the stream
    live._lock = threading.RLock()
    live._kv = _FakeKV(_FakeEngine(ours))
    with pytest.raises(_Accepted):
        live.resume(_state(int4_weights=True))
