"""Quantized vocabulary matrices (embed, lm_head in the layer matrices' e4m3 or int4 form) on the host: the weight specs
and their byte counts at Llama-3-8B, the embedding rule of each form against a numpy restatement, the flag checks, old
session states and the resume check."""
import threading

import numpy as np
import pytest
import torch

import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import dist, tiny_config, weights as W
from videollm_online_b200.config import llama3_8b_siglip_l

V8B, H8B = 128256, 4096
KV_TOKEN_BYTES = 131072   # one cached token of Llama-3-8B: 32 layers x K and V x 8 heads x 128 x bf16
PAGE_TOKENS = 64


def _bf16_rn(x: np.ndarray) -> np.ndarray:
    """fp32 -> the nearest bf16 (ties to even), as fp32"""
    b = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) >> 16 << 16
    return b.astype(np.uint32).view(np.float32)


def _e4m3_value(code: np.ndarray) -> np.ndarray:
    """e4m3fn byte -> its value (fp32): sign, 4 exponent bits (bias 7), 3 mantissa bits; exponent 0 is subnormal"""
    c = code.astype(np.int64)
    sign = np.where(c & 0x80, -1.0, 1.0)
    e, m = (c >> 3) & 0xF, c & 0x7
    mag = np.where(e == 0, m / 8.0 * 2.0 ** -6, (1 + m / 8.0) * 2.0 ** (e - 7))
    return (sign * mag).astype(np.float32)


def _vocab_bytes(spec):
    return sum(int(np.prod(shape)) * torch.empty((), dtype=dt).element_size()
               for name, (shape, dt) in spec.items() if name.split(".")[0] in ("embed", "lm_head"))


# ============================================================================================ specs
@pytest.mark.parametrize("form,quant_bytes", [("int4", 541_753_344), ("fp8", 1_051_699_200)])
def test_llama3_8b_vocab_bytes(form, quant_bytes):
    """embed + lm_head: 2 101 346 304 B in bf16; the quantized form frees what the table of the design note says, and
    that many bytes hold this many KV pool tokens and pages"""
    cfg = llama3_8b_siglip_l()
    assert (cfg.vocab_size, cfg.hidden_size) == (V8B, H8B)
    flags = dict(int4_weights=True) if form == "int4" else dict(fp8_weights=True)
    bf = dist.engine_weight_spec(cfg, 64, **flags)
    q = dist.engine_weight_spec(cfg, 64, quantize_vocab=True, **flags)
    assert _vocab_bytes(bf) == 2_101_346_304
    assert _vocab_bytes(q) == quant_bytes
    freed = _vocab_bytes(bf) - _vocab_bytes(q)
    tokens = freed // KV_TOKEN_BYTES
    assert (freed, tokens, tokens // PAGE_TOKENS) == {"int4": (1_559_592_960, 11_898, 185),
                                                      "fp8": (1_049_647_104, 8_008, 125)}[form]
    # everything but the vocabulary matrices is the same
    assert {k: v for k, v in bf.items() if k.split(".")[0] not in ("embed", "lm_head")} == \
           {k: v for k, v in q.items() if k.split(".")[0] not in ("embed", "lm_head")}


def test_spec_names_and_shapes():
    cfg = llama3_8b_siglip_l()
    s4 = dist.engine_weight_spec(cfg, 64, int4_weights=True, quantize_vocab=True)
    for m in ("embed", "lm_head"):
        assert m not in s4
        assert s4[m + ".i4"] == ((1002 * 128 * 4096 // 2,), torch.uint8)
        assert s4[m + ".gscale"] == ((V8B, 32), torch.bfloat16)
    s8 = dist.engine_weight_spec(cfg, 64, fp8_weights=True, quantize_vocab=True)
    for m in ("embed", "lm_head"):
        assert m not in s8
        assert s8[m + ".f8"] == ((V8B, H8B), torch.uint8)
        assert s8[m + ".scale"] == ((V8B,), torch.float32)
    assert dist.engine_weight_spec(cfg, 64, int4_weights=True)["lm_head"] == ((V8B, H8B), torch.bfloat16)


@pytest.mark.parametrize("flags", [dict(int4_weights=True), dict(fp8_weights=True)])
def test_packed_tensors_match_the_spec(flags):
    cfg = tiny_config()
    sd = W.synthetic_llm_state(cfg, seed=0)
    packed = W.pack_llm_for_engine(cfg, sd, "cpu", 64, quantize_vocab=True, **flags)
    spec = dist.engine_weight_spec(cfg, 64, quantize_vocab=True, **flags)
    assert {n for n in spec if n.split(".")[0] in ("embed", "lm_head")} <= set(packed)
    for name, t in packed.items():
        assert spec[name] == (tuple(t.shape), t.dtype), name
    # the same layer matrices as without the option
    plain = W.pack_llm_for_engine(cfg, sd, "cpu", 64, **flags)
    for name, t in plain.items():
        if name.split(".")[0] not in ("embed", "lm_head"):
            assert torch.equal(packed[name], t), name


# ============================================================================================ the embedding rules
def test_int4_embedding_rule():
    """row i of the int4 table = bf16_rn((code - 8) * s[i, k / 128]), the code read from the engine byte order"""
    cfg = tiny_config()
    sd = W.synthetic_llm_state(cfg, seed=3)
    packed = W.pack_llm_for_engine(cfg, sd, "cpu", 64, int4_weights=True, quantize_vocab=True)
    V, H = cfg.vocab_size, cfg.hidden_size
    got = W.dequantized_vocab_matrix(packed, "embed", V, H).float().numpy()
    words = packed["embed.i4"].view(torch.int32).numpy().astype(np.int64) & 0xFFFFFFFF
    s = packed["embed.gscale"].float().numpy()
    rows = np.arange(V)[:, None]
    cols = np.arange(H)[None, :]
    tile, rr = rows // 128, rows % 128
    h, warp, e, lr = rr // 64, (rr % 64) // 16, (rr % 16) // 8, rr % 8
    kb, kk, f, lc, b = cols // 64, (cols % 64) // 16, (cols % 16) // 8, (cols % 8) // 2, cols % 2
    byte = (tile * (H // 64) + kb) * 4096 + h * 2048 + (32 * warp + 4 * lr + lc) * 16 + kk * 4
    code = (words[byte // 4] >> (4 * (e + 2 * f) + 16 * b)) & 0xF
    want = _bf16_rn((code - 8).astype(np.float32) * s[rows, cols // 128])
    assert np.array_equal(got, want)
    # and the quantizer's W4 of the bf16 table
    q, sc = W.quantize_int4_groups(sd["model.embed_tokens.weight"])
    assert torch.equal(W.dequantized_vocab_matrix(packed, "embed", V, H), W.dequantize_int4_groups(q, sc))


def test_e4m3_embedding_rule():
    """row i of the e4m3 table = bf16_rn(fp32(q[i, k]) * s[i])"""
    cfg = tiny_config()
    sd = W.synthetic_llm_state(cfg, seed=4)
    packed = W.pack_llm_for_engine(cfg, sd, "cpu", 64, fp8_weights=True, quantize_vocab=True)
    V, H = cfg.vocab_size, cfg.hidden_size
    got = W.dequantized_vocab_matrix(packed, "embed", V, H)
    assert got.dtype == torch.bfloat16
    codes = packed["embed.f8"].numpy()
    s = packed["embed.scale"].numpy()
    want = _bf16_rn(_e4m3_value(codes) * s[:, None])
    assert np.array_equal(got.float().numpy(), want)
    assert torch.equal(got, W.dequantize_fp8_rows_bf16(packed["embed.f8"], packed["embed.scale"]))


def test_bf16_table_is_returned_as_is():
    cfg = tiny_config()
    packed = W.pack_llm_for_engine(cfg, W.synthetic_llm_state(cfg, seed=0), "cpu", 64, int4_weights=True)
    assert W.dequantized_vocab_matrix(packed, "embed", cfg.vocab_size, cfg.hidden_size) is packed["embed"]


# ============================================================================================ flags
def test_flag_needs_a_quantized_layer_form():
    cfg = tiny_config()
    with pytest.raises(ValueError, match="quantize_vocab"):
        dist.engine_weight_spec(cfg, 64, quantize_vocab=True)
    with pytest.raises(ValueError, match="quantize_vocab"):
        W.pack_llm_for_engine(cfg, W.synthetic_llm_state(cfg, seed=0), "cpu", 64, quantize_vocab=True)
    with pytest.raises(ValueError, match="choose one"):
        W.vocab_matrix_spec("embed", (256, 128), True, True, True)
    from videollm_online_b200.modeling_live import build_live
    with pytest.raises(ValueError, match="quantize_vocab"):
        build_live(config=cfg, quantize_vocab=True, synthetic_weights=True, device="cpu")


def test_cli_flag_parses():
    from videollm_online_b200.config import LiveArguments
    from videollm_online_b200.inference import parse_args
    assert LiveArguments().quantize_vocab is False
    args = parse_args(["--int4_weights", "true", "--quantize_vocab", "true"])
    assert args.quantize_vocab is True and args.int4_weights is True


# ============================================================================================ session states
def _state(**kw):
    from videollm_online_b200.inference import SessionState
    return SessionState(kv=None, last_ids=torch.zeros(1), video_time=0.0, last_frame_idx=0, query_queue=[],
                        frame_embeds_queue=[], drafter_ids=None, n_calls=0, started=False, **kw)


def test_old_session_state_loads_as_not_quantized(tmp_path):
    state = _state(int4_weights=True)
    del state.__dict__["quantized_vocab"]   # a state written before the field existed
    path = tmp_path / "old.pt"
    torch.save(state, path)
    loaded = torch.load(path, weights_only=True)
    assert loaded.quantized_vocab is False and loaded.int4_weights is True


class _FakeEngine:
    fp8_weights, fp8_activations = False, False

    def __init__(self, quantized_vocab):
        self.int4_weights = True
        self.quantized_vocab = quantized_vocab

    def stream_reset(self, sid):
        raise AssertionError("resume touched the stream before refusing the state")


class _FakeKV:
    def __init__(self, engine):
        self.engine, self.stream_id = engine, 0


@pytest.mark.parametrize("ours,theirs", [(True, False), (False, True)])
def test_resume_refuses_the_other_vocabulary_form(ours, theirs):
    from videollm_online_b200._lib import VloError
    from videollm_online_b200.inference import LiveInfer
    live = LiveInfer.__new__(LiveInfer)     # only what resume reads before its checks
    live._lock = threading.RLock()
    live._kv = _FakeKV(_FakeEngine(ours))
    with pytest.raises(VloError, match="vocabulary matrices"):
        live.resume(_state(int4_weights=True, quantized_vocab=theirs))
