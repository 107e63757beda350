"""FP8 decoder weights on the CPU: the row quantizer, the engine layout and its broadcast spec, the flag."""
import os
import pathlib
import subprocess
import sys

import pytest
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]


def test_quantizer_agrees_with_torch_e4m3fn():
    from videollm_online_b200 import weights as W
    g = torch.Generator().manual_seed(0)
    w = (torch.randn(64, 256, generator=g) * torch.logspace(-6, 2, 64)[:, None]).bfloat16()
    codes, scale = W.quantize_fp8_rows(w)
    assert codes.dtype == torch.uint8 and codes.shape == w.shape and scale.dtype == torch.float32 and scale.shape == (64,)
    w32 = w.float()
    s = w32.abs().amax(1) / 448.0
    assert torch.equal(scale, s)
    want = (w32 / s[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn)
    assert torch.equal(codes, want.view(torch.uint8))
    # each row reaches the largest code, and the dequantized weight is within half an e4m3 step of W
    assert torch.equal(codes.view(torch.float8_e4m3fn).float().abs().amax(1), torch.full((64,), 448.0))
    err = (W.dequantize_fp8_rows(codes, scale) - w32).abs()
    assert bool((err <= 2.0 ** -4 * w32.abs() + 2.0 ** -10 * scale[:, None] + 1e-30).all())


def test_quantizer_saturation_zero_rows_and_no_nan():
    from videollm_online_b200 import weights as W
    w = torch.zeros(4, 64)
    w[1] = torch.linspace(-3e4, 3e4, 64)
    w[2, 5] = -1e-30
    w[3] = float(torch.finfo(torch.bfloat16).max)
    codes, scale = W.quantize_fp8_rows(w.bfloat16())
    f = codes.view(torch.float8_e4m3fn).float()
    assert scale[0] == 1.0 and bool((codes[0] == 0).all())            # all-zero row: s = 1, codes +0
    assert f[1].max() == 448.0 and f[1].min() == -448.0                 # +-amax saturate to +-448, never past
    assert f[2, 5] == -448.0 and bool((f[2].abs().sum() == 448.0))
    assert bool((f[3] == 448.0).all())
    assert not bool(torch.isnan(f).any())
    assert not bool(((codes & 0x7F) == 0x7F).any())                    # the NaN codes never appear
    with pytest.raises(ValueError):
        W.quantize_fp8_rows(torch.tensor([[1.0, float("inf")]]).bfloat16())


def test_quantized_gate_up_keeps_the_interleaved_row_order():
    from videollm_online_b200 import tiny_config, weights as W
    cfg = tiny_config()
    llm = W.synthetic_llm_state(cfg, seed=3)
    p16 = W.pack_llm_for_engine(cfg, llm, "cpu", 64)
    p8 = W.pack_llm_for_engine(cfg, llm, "cpu", 64, fp8_weights=True)
    for i in range(cfg.num_hidden_layers):
        for m in W.LAYER_MATRICES:
            n = f"L{i}.{m}"
            assert n not in p8
            codes, scale = W.quantize_fp8_rows(p16[n])
            assert torch.equal(p8[n + ".f8"], codes) and torch.equal(p8[n + ".scale"], scale)
        # row r of the packed gate|up is gate row 64 (r // 128) + r % 64 or the matching up row
        gate = llm[f"model.layers.{i}.mlp.gate_proj.weight"]
        c_gate, s_gate = W.quantize_fp8_rows(gate)
        r = torch.arange(2 * cfg.intermediate_size)
        is_gate = (r % 128) < 64
        src = 64 * (r // 128) + r % 64
        assert torch.equal(p8[f"L{i}.gate_up.f8"][r[is_gate]], c_gate[src[is_gate]])
        assert torch.equal(p8[f"L{i}.gate_up.scale"][r[is_gate]], s_gate[src[is_gate]])
    rest = [k for k in p16 if not any(k == f"L{i}.{m}" for i in range(cfg.num_hidden_layers) for m in W.LAYER_MATRICES)]
    assert all(torch.equal(p16[k], p8[k]) for k in rest)


def test_weight_spec_and_flat_layout_with_fp8_weights():
    from videollm_online_b200 import tiny_config, weights as W
    from videollm_online_b200.dist import _flat_layout, engine_weight_spec
    cfg = tiny_config()
    spec16, spec8 = engine_weight_spec(cfg, 64), engine_weight_spec(cfg, 64, fp8_weights=True)
    full = W.pack_llm_for_engine(cfg, W.synthetic_llm_state(cfg), "cpu", 64, fp8_weights=True)
    full.update(W.pack_vision_for_engine(cfg, W.synthetic_vision_state(cfg), "cpu"))
    assert set(spec8) == set(full)
    assert all(tuple(full[k].shape) == tuple(spec8[k][0]) and full[k].dtype == spec8[k][1] for k in spec8)
    for i in range(cfg.num_hidden_layers):
        for m in W.LAYER_MATRICES:
            n = f"L{i}.{m}"
            shape, _ = spec16[n]
            assert spec8[n + ".f8"] == (shape, torch.uint8) and spec8[n + ".scale"] == ((shape[0],), torch.float32)
    layout = _flat_layout(spec8, 4)
    placed = [(name, off, shape, dt) for _, members in layout for name, off, shape, dt in members]
    assert sorted(n for n, *_ in placed) == sorted(spec8) and all(off % 256 == 0 for _, off, *_ in placed)
    b16 = sum(b for b, _ in _flat_layout(spec16, 4))
    b8 = sum(b for b, _ in _flat_layout(spec8, 4))
    assert b8 < b16


def test_fp8_weights_flag_defaults_off():
    from videollm_online_b200 import parse_args
    assert parse_args([]).fp8_weights is False
    assert parse_args(["--fp8_weights"]).fp8_weights is True
    assert parse_args(["--fp8_weights", "true"]).fp8_weights is True


@pytest.mark.timeout(180)
def test_fp8_weight_broadcast_two_ranks_gloo(tmp_path):
    """the FP8 engine layout travels through broadcast_weights unchanged (gloo, two ranks on 127.0.0.1)"""
    script = tmp_path / "bc8.py"
    script.write_text(f"""
import sys, torch, torch.distributed as dist
sys.path.insert(0, {str(ROOT)!r})
import vlo_bootstrap
from videollm_online_b200 import tiny_config, weights as W
from videollm_online_b200.dist import broadcast_weights
dist.init_process_group('gloo')
cfg = tiny_config()
full = W.pack_llm_for_engine(cfg, W.synthetic_llm_state(cfg), 'cpu', 128, fp8_weights=True)
full.update(W.pack_vision_for_engine(cfg, W.synthetic_vision_state(cfg), 'cpu'))
got = broadcast_weights(cfg, full if dist.get_rank() == 0 else None, 'cpu', 128, dist, fp8_weights=True)
assert set(got) == set(full) and all(torch.equal(got[k], full[k]) and got[k].dtype == full[k].dtype for k in full)
assert any(k.endswith('.f8') for k in got) and not any(k == 'L0.qkv' for k in got)
sys.stdout.write('rank %d ok\\n' % dist.get_rank()); sys.stdout.flush()
""")
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    import socket
    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        port = so.getsockname()[1]
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                        "127.0.0.1", "--master-port", str(port), str(script)], capture_output=True, text=True, env=env,
                       timeout=170)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "rank 0 ok" in r.stdout and "rank 1 ok" in r.stdout
