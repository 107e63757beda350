"""Int4 (W4A16) layer weights on the host: the quantizer against a numpy restatement of its rule, the engine byte order
of the codes, the weight specs and the flag checks."""
import numpy as np
import pytest
import torch

import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import dist, tiny_config, weights as W


def _bf16_rn(x: np.ndarray) -> np.ndarray:
    """fp32 -> the nearest bf16 (ties to even), as fp32"""
    b = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) >> 16 << 16
    return b.astype(np.uint32).view(np.float32)


def _reference(w: np.ndarray):
    """the rule: s = bf16_rn(fp32(amax) / 7), 1 where 0; q = clamp(rne(fp32(W) / fp32(s)), -8, 7); W4 = bf16_rn(q s)"""
    n, k = w.shape
    g = w.reshape(n, k // 128, 128)
    s = _bf16_rn(np.abs(g).max(axis=2) / np.float32(7))
    s = np.where(s == 0, np.float32(1), s).astype(np.float32)
    q = np.clip(np.rint(g / s[:, :, None]), -8, 7).astype(np.int8)
    w4 = _bf16_rn((q.astype(np.float32) * s[:, :, None]).reshape(n, k))
    return q.reshape(n, k), s, w4


def _check(w: torch.Tensor):
    q, s = W.quantize_int4_groups(w)
    rq, rs, rw4 = _reference(w.float().numpy())
    assert np.array_equal(q.numpy(), rq)
    assert np.array_equal(s.float().numpy(), rs)
    assert np.array_equal(W.dequantize_int4_groups(q, s).float().numpy(), rw4)
    return q, s


@pytest.mark.parametrize("n,k", [(3, 128), (64, 14336), (130, 384)])
def test_quantizer_matches_the_rule(n, k):
    g = torch.Generator().manual_seed(n + k)
    w = (torch.randn(n, k, generator=g) * torch.pow(2.0, torch.randint(-30, 6, (n, 1), generator=g).float())).bfloat16()
    _check(w)


def test_quantizer_edge_cases():
    w = torch.zeros(6, 256)
    w[1, 128:] = torch.linspace(-1, 1, 128)              # a zero group next to a live one
    w[2, :8] = torch.tensor([7, -7, 3.5, -3.5, 0.5, -0.5, 1.5, 2.5])   # amax 7: s = 1, ties at .5 go to even
    w[3, :2] = torch.tensor([-7.0, 7.0])                  # +-amax -> +-7
    w[4, :2] = torch.tensor([1.0, -1.0]) * 7.5            # s = bf16(7.5 / 7) rounds down: 7.5 / s > 7
    w[5, :3] = torch.tensor([-8.0, 8.0, 4.0]) * 3.3
    q, s = _check(w.bfloat16())
    assert s[0].float().tolist() == [1.0, 1.0] and s[1, 0].item() == 1.0
    assert q[2, :8].tolist() == [7, -7, 4, -4, 0, 0, 2, 2]
    assert q[3, :2].tolist() == [-7, 7]
    assert float(s[4, 0]) * 7 < 7.5 and q[4, :2].tolist() == [7, -7]
    assert int(q.min()) >= -8 and int(q.max()) <= 7


def test_quantizer_rejects_bad_shapes():
    with pytest.raises(ValueError, match="multiple of 128"):
        W.quantize_int4_groups(torch.zeros(4, 192, dtype=torch.bfloat16))
    with pytest.raises(ValueError, match="non-finite"):
        W.quantize_int4_groups(torch.full((1, 128), float("inf"), dtype=torch.bfloat16))


@pytest.mark.parametrize("n,k", [(128, 128), (200, 384), (256, 1024)])
def test_pack_round_trip_and_byte_order(n, k):
    g = torch.Generator().manual_seed(k)
    q = torch.randint(-8, 8, (n, k), generator=g, dtype=torch.int8)
    packed = W.pack_int4_codes(q)
    assert packed.dtype == torch.uint8 and packed.numel() == -(-n // 128) * 128 * k // 2
    assert torch.equal(W.unpack_int4_codes(packed, n, k), q)
    # element (row 64h + 16warp + 8e + lane/4, column 64kb + 16kk + 8f + 2(lane%4) + b) of tile 0
    words = packed.view(torch.int32)
    for h, warp, e, lr, kb, kk, f, lc, b in [(0, 0, 0, 0, 0, 0, 0, 0, 0), (1, 3, 1, 7, k // 64 - 1, 3, 1, 3, 1),
                                             (0, 2, 1, 5, 1, 2, 0, 1, 1)]:
        row, col = 64 * h + 16 * warp + 8 * e + lr, 64 * kb + 16 * kk + 8 * f + 2 * lc + b
        t = 32 * warp + 4 * lr + lc
        word = int(words[(kb * 4096 + h * 2048 + t * 16 + kk * 4) // 4]) & 0xFFFFFFFF
        assert (word >> (4 * (e + 2 * f) + 16 * b)) & 0xF == int(q[row, col]) + 8


def test_layer_matrix_and_broadcast_specs():
    spec = W.layer_matrix_spec("L0.o", (200, 384), False, True)
    assert spec == {"L0.o.i4": ((256 * 192,), torch.uint8), "L0.o.gscale": ((200, 3), torch.bfloat16)}
    cfg = tiny_config()
    packed = W.pack_llm_for_engine(cfg, W.synthetic_llm_state(cfg, seed=0), "cpu", 64, int4_weights=True)
    full = dist.engine_weight_spec(cfg, 64, int4_weights=True)
    for name, t in packed.items():
        assert full[name] == (tuple(t.shape), t.dtype), name
    assert not any(k.endswith((".f8", ".scale")) for k in full)
    assert all(f"L{i}.{m}.i4" in full for i in range(cfg.num_hidden_layers) for m in W.LAYER_MATRICES)
    with pytest.raises(ValueError, match="choose one"):
        dist.engine_weight_spec(cfg, 64, fp8_weights=True, int4_weights=True)
    with pytest.raises(ValueError, match="choose one"):
        W.pack_llm_for_engine(cfg, W.synthetic_llm_state(cfg, seed=0), "cpu", 64, fp8_weights=True, int4_weights=True)


@pytest.mark.parametrize("flags", [dict(fp8_weights=True), dict(fp8_activations=True),
                                   dict(fp8_weights=True, fp8_activations=True)])
def test_build_live_rejects_int4_with_fp8(flags):
    from videollm_online_b200.modeling_live import build_live
    with pytest.raises(ValueError, match="int4_weights"):
        build_live(config=tiny_config(), int4_weights=True, synthetic_weights=True, device="cpu", **flags)


def test_cli_flag_parses():
    from videollm_online_b200.config import LiveArguments
    from videollm_online_b200.inference import parse_args
    assert LiveArguments().int4_weights is False
    assert parse_args(["--int4_weights", "true"]).int4_weights is True


def test_old_session_state_loads_as_not_int4(tmp_path):
    from videollm_online_b200.inference import SessionState
    state = SessionState(kv=None, last_ids=torch.zeros(1), video_time=0.0, last_frame_idx=0, query_queue=[],
                         frame_embeds_queue=[], drafter_ids=None, n_calls=0, started=False)
    del state.__dict__["int4_weights"]   # a state written before the field existed
    path = tmp_path / "old.pt"
    torch.save(state, path)
    loaded = torch.load(path, weights_only=True)
    assert loaded.int4_weights is False and loaded.fp8_weights is False
