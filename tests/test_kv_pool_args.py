"""CPU-side: the KV pool size travels from the command line to the engine."""
import pytest


def test_kv_pool_tokens_reaches_the_engine(monkeypatch):
    from videollm_online_b200 import modeling_live
    from videollm_online_b200.config import parse_args
    from videollm_online_b200.inference import LiveInfer

    seen = {}

    class Stop(Exception):
        pass

    def fake_engine(cfg, device, **kw):
        seen.update(kw)
        raise Stop

    monkeypatch.setattr(modeling_live, "Engine", fake_engine)
    args = parse_args(["--kv_pool_tokens", "200000", "--max_streams", "9", "--synthetic_weights", "true"])
    assert args.kv_pool_tokens == 200000
    with pytest.raises(Stop):
        LiveInfer(args)
    assert seen["kv_pool_tokens"] == 200000 and seen["max_streams"] == 9
    assert parse_args([]).kv_pool_tokens == 0   # 0: max_streams x max_kv_tokens, what vlo_engine_create reserves
