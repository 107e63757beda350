"""Weights: synthetic HF-style state dicts, LoRA merge, and packing into the engine layout.

The reference loads `meta-llama/Meta-Llama-3-8B-Instruct` + a PEFT adapter (LoRA r=128, alpha=256 on
q,k,v,o,gate,up,down,lm_head plus the `connector` module) + SigLIP-L (models/modeling_live.py:200-220,
models/arguments_live.py:16-19).  No checkpoint is available offline, so tests and benchmarks use
seeded synthetic tensors with the reference's parameter names and shapes (SURVEY.md Appendix A); the
same dict feeds the oracle, the HF reference modules (golden generation) and — after `pack_for_engine`
— the CUDA engine.

Engine layout (name -> tensor), all contiguous on the engine's device:
  embed [V,H] bf16 | final_norm [H] bf16 | lm_head [V,H] bf16 | rope.cos / rope.sin [max_pos,64] bf16
  L{i}.in_norm, L{i}.post_norm [H] bf16 | L{i}.qkv [(nh+2nkv)*128, H] bf16 (q|k|v rows)
  L{i}.o [H, nh*128] | L{i}.gate_up [2I, H] (tile-interleaved: 64 gate rows of features 64j.., then the matching 64 up
  rows, per 128-row tile j - one MMA tile then holds both operands of SwiGLU) | L{i}.down [H, I]   (bf16)
  conn.0.w [H,C] bf16, conn.0.b [H] f32, conn.2.w [H,H] bf16, conn.2.b [H] f32
  vit.patch.w [C, 3*ps*ps] f16, vit.patch.b [C] f32, vit.pos [P,C] f32, vit.post_ln.{w,b} f32
  vit.L{i}.{ln1,ln2}.{w,b} f32, vit.L{i}.qkv.w [3C,C] f16 (+ .b f32), out.w [C,C], fc1.w [M,C], fc2.w [C,M]
  vit.head.q [C] f32 (= in_proj_q(probe), fp16-rounded), vit.head.kv.{w,b}, out.{w,b}, ln.{w,b}, fc1, fc2
16-bit biases are stored as fp32 copies of their 16-bit values (the GEMM epilogue adds them in fp32).
FP8 weights (fp8_weights=True): each layer matrix L{i}.{qkv,o,gate_up,down} [N, K] is replaced by L{i}.{m}.f8 (e4m3fn
bytes [N, K], uint8) and L{i}.{m}.scale (fp32 [N], one scale per output row), quantized by quantize_fp8_rows from the
bf16 matrix above (after the LoRA merge and the gate|up interleave).  Everything else stays 16-bit.
Int4 weights (int4_weights=True, W4A16): each layer matrix [N, K] (K % 128 == 0) is replaced by L{i}.{m}.i4 (the codes
q + 8 in the engine byte order of pack_int4_codes, uint8, ceil(N / 128) * 128 * K / 2 bytes) and L{i}.{m}.gscale (bf16
[N, K / 128]), quantized by quantize_int4_groups from the same bf16 matrix.  The engine multiplies W4 =
dequantize_int4_groups(q, s) exactly, so an int4 engine computes the bits of a bf16 engine loaded with W4.
Quantized vocabulary matrices (quantize_vocab=True, with fp8_weights or int4_weights): embed and lm_head [V, H] are
quantized after the LoRA merge by the same rule as the layer matrices and stored under the same suffixes (embed.f8 +
embed.scale, lm_head.f8 + lm_head.scale; or embed.i4 + embed.gscale, lm_head.i4 + lm_head.gscale).  The engine's
embedding of id i is row i of dequantize_fp8_rows_bf16 / dequantize_int4_groups (dequantized_vocab_matrix).
"""
from __future__ import annotations

import math
import re
from typing import Dict

import torch

from .config import LiveConfig

StateDict = Dict[str, torch.Tensor]


# --------------------------------------------------------------------------- synthetic HF-style
def _gen(shape, std, gen, device, dtype, mean=0.0):
    t = torch.empty(shape, device=device, dtype=torch.float32)
    t.normal_(mean, std, generator=gen)
    return t.to(dtype)


def synthetic_llm_state(cfg: LiveConfig, seed: int = 0, device="cpu", std: float = 0.02) -> StateDict:
    """`LiveLlamaForCausalLM.state_dict()`-shaped random weights (bf16), LoRA already merged."""
    g = torch.Generator(device=device).manual_seed(seed)
    H, I, V = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size
    nh, nkv, hd, C = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim, cfg.vision_hidden_size
    bf = torch.bfloat16
    sd: StateDict = {}
    sd["model.embed_tokens.weight"] = _gen((V, H), 1.0, g, device, bf)
    for i in range(cfg.num_hidden_layers):
        p = f"model.layers.{i}."
        sd[p + "self_attn.q_proj.weight"] = _gen((nh * hd, H), std, g, device, bf)
        sd[p + "self_attn.k_proj.weight"] = _gen((nkv * hd, H), std, g, device, bf)
        sd[p + "self_attn.v_proj.weight"] = _gen((nkv * hd, H), std, g, device, bf)
        sd[p + "self_attn.o_proj.weight"] = _gen((H, nh * hd), std, g, device, bf)
        sd[p + "mlp.gate_proj.weight"] = _gen((I, H), std, g, device, bf)
        sd[p + "mlp.up_proj.weight"] = _gen((I, H), std, g, device, bf)
        sd[p + "mlp.down_proj.weight"] = _gen((H, I), std, g, device, bf)
        sd[p + "input_layernorm.weight"] = _gen((H,), 0.1, g, device, bf, mean=1.0)
        sd[p + "post_attention_layernorm.weight"] = _gen((H,), 0.1, g, device, bf, mean=1.0)
    sd["model.norm.weight"] = _gen((H,), 0.1, g, device, bf, mean=1.0)
    sd["lm_head.weight"] = _gen((V, H), std, g, device, bf)
    sd["connector.0.weight"] = _gen((H, C), std, g, device, bf)
    sd["connector.0.bias"] = _gen((H,), std, g, device, bf)
    sd["connector.2.weight"] = _gen((H, H), std, g, device, bf)
    sd["connector.2.bias"] = _gen((H,), std, g, device, bf)
    return sd


def synthetic_vision_state(cfg: LiveConfig, seed: int = 1, device="cpu", std: float = 0.02) -> StateDict:
    """`SiglipVisionModel(...).vision_model.state_dict()`-shaped random weights (fp32, as loaded by
    build_live_vision, models/vision_live.py:55)."""
    g = torch.Generator(device=device).manual_seed(seed)
    C, M, ps = cfg.vision_hidden_size, cfg.vision_intermediate_size, cfg.vision_patch_size
    P = cfg.num_patches
    f32 = torch.float32
    sd: StateDict = {}
    sd["embeddings.patch_embedding.weight"] = _gen((C, 3, ps, ps), std, g, device, f32)
    sd["embeddings.patch_embedding.bias"] = _gen((C,), std, g, device, f32)
    sd["embeddings.position_embedding.weight"] = _gen((P, C), std, g, device, f32)
    for i in range(cfg.vision_num_hidden_layers):
        p = f"encoder.layers.{i}."
        for ln in ("layer_norm1", "layer_norm2"):
            sd[p + ln + ".weight"] = _gen((C,), 0.1, g, device, f32, mean=1.0)
            sd[p + ln + ".bias"] = _gen((C,), std, g, device, f32)
        for nm in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[p + f"self_attn.{nm}.weight"] = _gen((C, C), std, g, device, f32)
            sd[p + f"self_attn.{nm}.bias"] = _gen((C,), std, g, device, f32)
        sd[p + "mlp.fc1.weight"] = _gen((M, C), std, g, device, f32)
        sd[p + "mlp.fc1.bias"] = _gen((M,), std, g, device, f32)
        sd[p + "mlp.fc2.weight"] = _gen((C, M), std, g, device, f32)
        sd[p + "mlp.fc2.bias"] = _gen((C,), std, g, device, f32)
    sd["post_layernorm.weight"] = _gen((C,), 0.1, g, device, f32, mean=1.0)
    sd["post_layernorm.bias"] = _gen((C,), std, g, device, f32)
    sd["head.probe"] = _gen((1, 1, C), 1.0, g, device, f32)
    sd["head.attention.in_proj_weight"] = _gen((3 * C, C), std, g, device, f32)
    sd["head.attention.in_proj_bias"] = _gen((3 * C,), std, g, device, f32)
    sd["head.attention.out_proj.weight"] = _gen((C, C), std, g, device, f32)
    sd["head.attention.out_proj.bias"] = _gen((C,), std, g, device, f32)
    sd["head.layernorm.weight"] = _gen((C,), 0.1, g, device, f32, mean=1.0)
    sd["head.layernorm.bias"] = _gen((C,), std, g, device, f32)
    sd["head.mlp.fc1.weight"] = _gen((M, C), std, g, device, f32)
    sd["head.mlp.fc1.bias"] = _gen((M,), std, g, device, f32)
    sd["head.mlp.fc2.weight"] = _gen((C, M), std, g, device, f32)
    sd["head.mlp.fc2.bias"] = _gen((C,), std, g, device, f32)
    return sd


# --------------------------------------------------------------------------- LoRA merge (K20)
_LORA_RE = re.compile(r"^(?:base_model\.model\.)?(.*)\.lora_A(?:\.[^.]+)?\.weight$")


def merge_lora(llm_state: StateDict, adapter_state: StateDict, lora_alpha: float = 256, lora_r: int = 128) -> StateDict:
    """W' = W + (alpha/r) * B @ A for every wrapped Linear, plus `modules_to_save` (connector) overrides.

    The reference keeps the adapter unmerged at inference (models/modeling_live.py:216,
    y = W x + 2.0 * B(A(x))); merging at load removes 2 small GEMMs per Linear from the hot path.
    The product is formed in fp32 and rounded once to bf16 (parity note in DESIGN.md)."""
    out = dict(llm_state)
    scaling = float(lora_alpha) / float(lora_r)
    for key, a in adapter_state.items():
        m = _LORA_RE.match(key)
        if m:
            base = m.group(1) + ".weight"
            bkey = key.replace("lora_A", "lora_B")
            if base not in out or bkey not in adapter_state:
                raise KeyError(f"LoRA tensor {key} has no base weight {base} / partner {bkey}")
            w = out[base]
            delta = adapter_state[bkey].float() @ a.float()
            out[base] = (w.float() + scaling * delta.to(w.device)).to(w.dtype)
        elif "modules_to_save" in key or re.match(r"^(?:base_model\.model\.)?connector\.", key):
            name = re.sub(r"^(?:base_model\.model\.)?", "", key)
            name = re.sub(r"\.modules_to_save\.[^.]+", "", name)
            if name.startswith("connector."):
                out[name] = adapter_state[key].to(torch.bfloat16)
    return out


# --------------------------------------------------------------------------- engine layout
def rope_tables(cfg: LiveConfig, n_positions: int, device) -> tuple[torch.Tensor, torch.Tensor]:
    """bf16 cos/sin tables exactly as LlamaRotaryEmbedding.forward produces them for
    position_ids = arange(n) (HF:models/llama/modeling_llama.py:124-135): fp32 outer product,
    fp32 cos/sin, cast to the activation dtype.  Only the first head_dim/2 columns are stored
    (HF concatenates two identical halves)."""
    pos = torch.arange(n_positions, dtype=torch.float32)
    freqs = pos[:, None] * rope_inv_freq(cfg)[None, :]
    return (freqs.cos().to(torch.bfloat16).contiguous().to(device),
            freqs.sin().to(torch.bfloat16).contiguous().to(device))


def rope_inv_freq(cfg: LiveConfig) -> torch.Tensor:
    """fp32 [head_dim / 2]: the RoPE frequencies, as LlamaRotaryEmbedding computes inv_freq (the one definition the
    tables and the eviction's rotation share)."""
    d = cfg.head_dim
    return 1.0 / (cfg.rope_theta ** (torch.arange(0, d, 2, dtype=torch.int64).to(dtype=torch.float) / d))


def rope_rotation(cfg: LiveConfig, delta: int) -> tuple[torch.Tensor, torch.Tensor]:
    """fp32 cos / sin [head_dim / 2] of delta * inv_freq, computed in fp64 from the fp32 inv_freq and rounded once: the
    rotation vlo_kv_evict applies (by -delta) to the keys it moves delta positions down.  Not the bf16 tables, whose
    2^-9 relative error would compound over repeated evictions."""
    ang = rope_inv_freq(cfg).double() * float(delta)
    return ang.cos().float(), ang.sin().float()


def _b32_from16(t: torch.Tensor, dt16) -> torch.Tensor:
    return t.to(dt16).to(torch.float32).contiguous()


def interleave_gate_up(gate: torch.Tensor, up: torch.Tensor) -> torch.Tensor:
    """[I, H] + [I, H] -> [2I, H] with rows ordered per 128-row tile: gate[64j:64j+64] then up[64j:64j+64]."""
    I, H = gate.shape
    if I % 64 != 0:
        raise ValueError("intermediate_size must be a multiple of 64")
    return torch.stack([gate.view(I // 64, 64, H), up.view(I // 64, 64, H)], 1).reshape(2 * I, H).contiguous()


FP8_MAX = 448.0   # largest finite e4m3fn value
LAYER_MATRICES = ("qkv", "o", "gate_up", "down")   # the decoder layer matrices fp8_weights quantizes


def quantize_fp8_rows(w: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """[N, K] weight -> (e4m3fn codes as uint8 [N, K], fp32 scales [N]) on w's device:
    s[n] = fp32(max_k |W[n, k]|) / 448 (1 for an all-zero row), q[n, k] = e4m3fn(clamp(fp32(W[n, k]) / s[n], -448, 448))
    rounded to nearest even, so W[n, k] ~ fp32(q[n, k]) * s[n] and no code is NaN."""
    if w.dim() != 2:
        raise ValueError(f"quantize_fp8_rows: a 2-D weight, got shape {tuple(w.shape)}")
    w32 = w.float()
    if not bool(torch.isfinite(w32).all()):
        raise ValueError("quantize_fp8_rows: the weight holds a non-finite value")
    amax = w32.abs().amax(dim=1)
    scale = torch.where(amax > 0, amax / FP8_MAX, torch.ones_like(amax))
    q = (w32 / scale[:, None]).clamp_(-FP8_MAX, FP8_MAX).to(torch.float8_e4m3fn)
    return q.view(torch.uint8), scale.contiguous()


def dequantize_fp8_rows(codes: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """fp32 [N, K] = fp32(q) * s: the weight the FP8 kernels multiply by (up to where the scale is applied)."""
    return codes.view(torch.float8_e4m3fn).float() * scale[:, None]


def dequantize_fp8_rows_bf16(codes: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """bf16 [N, K] = bf16_rn(fp32(q) * s): the rows of an e4m3 embedding table as the engine's gather returns them (one
    fp32 product, then one rounding to bf16)."""
    return dequantize_fp8_rows(codes, scale).to(torch.bfloat16)


INT4_GROUP = 128   # weights of a row per int4 scale
INT4_TILE = 128    # weight rows per engine tile (the GEMM's 128-row M tile)


def quantize_int4_groups(w: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """[N, K] weight (K % 128 == 0) -> (int8 q [N, K] in [-8, 7], bf16 scales [N, K / 128]) on w's device:
    s[n, g] = bf16_rn(fp32(max_{k in group g} |W[n, k]|) / 7) (1 where that is 0), q[n, k] = clamp(rne(fp32(W[n, k]) /
    fp32(s[n, g])), -8, 7), IEEE fp32 division."""
    if w.dim() != 2:
        raise ValueError(f"quantize_int4_groups: a 2-D weight, got shape {tuple(w.shape)}")
    n, k = w.shape
    if k % INT4_GROUP != 0:
        raise ValueError(f"quantize_int4_groups: K = {k} is not a multiple of {INT4_GROUP}")
    w32 = w.float()
    if not bool(torch.isfinite(w32).all()):
        raise ValueError("quantize_int4_groups: the weight holds a non-finite value")
    g = w32.view(n, k // INT4_GROUP, INT4_GROUP)
    s = (g.abs().amax(dim=2) / 7).to(torch.bfloat16)
    s = torch.where(s == 0, torch.ones_like(s), s)
    q = torch.round(g / s.float()[:, :, None]).clamp_(-8, 7).to(torch.int8)
    return q.view(n, k), s.contiguous()


def dequantize_int4_groups(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """bf16 [N, K] = W4 = bf16_rn(q * s): the weight every int4 kernel multiplies (q * s is exact in fp32)."""
    n, k = q.shape
    return (q.float().view(n, k // INT4_GROUP, INT4_GROUP) * s.float()[:, :, None]).view(n, k).to(torch.bfloat16)


def _int4_code_view(codes: torch.Tensor, n_pad: int, k: int) -> torch.Tensor:
    # [tile][h][warp][e][lane / 4] rows x [k-block][kk][f][lane % 4][b] columns: row = 64h + 16warp + 8e + lane / 4,
    # column = 64 k-block + 16kk + 8f + 2(lane % 4) + b (gemm.cuh, FMT_I4)
    return codes.view(n_pad // INT4_TILE, 2, 4, 2, 8, k // 64, 4, 2, 4, 2)


def pack_int4_codes(q: torch.Tensor) -> torch.Tensor:
    """int8 q [N, K] in [-8, 7] -> uint8 [ceil(N / 128) * 128 * K / 2]: the codes q + 8 in the engine byte order.  One
    4 KB block per (128-row tile, 64-wide k-block), blocks in (tile, k-block) order; inside a block, consumer thread t =
    32 warp + lane has 16 bytes per 64-row half h at h * 2048 + 16 t: one 32-bit word per k16 step kk, holding the code of
    element (row r + 8e, column c + 8f + b) in bits 4(e + 2f) + 16b, r = 64h + 16 warp + lane / 4, c = 16kk + 2(lane % 4).
    Rows past N are padded with code 8 (q = 0)."""
    n, k = q.shape
    n_pad = -(-n // INT4_TILE) * INT4_TILE
    codes = torch.full((n_pad, k), 8, dtype=torch.int64, device=q.device)
    codes[:n] = q.to(torch.int64) + 8
    c = _int4_code_view(codes, n_pad, k)
    # -> [tile, k-block, h, warp, lane / 4, lane % 4, kk, e, f, b]
    c = c.permute(0, 5, 1, 2, 4, 8, 6, 3, 7, 9)
    shift = torch.tensor([[[0, 16], [8, 24]], [[4, 20], [12, 28]]], dtype=torch.int64, device=q.device)   # [e][f][b]
    words = (c << shift).sum(dim=(-3, -2, -1))
    return words.to(torch.int32).contiguous().view(torch.uint8).reshape(-1)


def unpack_int4_codes(packed: torch.Tensor, n: int, k: int) -> torch.Tensor:
    """The inverse of pack_int4_codes: int8 q [N, K]."""
    n_pad = -(-n // INT4_TILE) * INT4_TILE
    words = packed.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    words = words.view(n_pad // INT4_TILE, k // 64, 2, 4, 8, 4, 4)   # [tile, k-block, h, warp, lane/4, lane%4, kk]
    shift = torch.tensor([[[0, 16], [8, 24]], [[4, 20], [12, 28]]], dtype=torch.int64, device=packed.device)
    c = (words[..., None, None, None] >> shift) & 0xF            # [..., kk, e, f, b]
    c = c.permute(0, 2, 3, 7, 4, 1, 6, 8, 5, 9)                  # -> [tile, h, warp, e, lane/4, k-block, kk, f, lane%4, b]
    return (c.reshape(n_pad, k)[:n] - 8).to(torch.int8)


def _weight_form(fp8_weights: bool, int4_weights: bool) -> None:
    if fp8_weights and int4_weights:
        raise ValueError("fp8_weights and int4_weights are two forms of the layer matrices: choose one")


def _vocab_form(fp8_weights: bool, int4_weights: bool, quantize_vocab: bool) -> None:
    _weight_form(fp8_weights, int4_weights)
    if quantize_vocab and not (fp8_weights or int4_weights):
        raise ValueError("quantize_vocab takes the layer matrices' quantized form: it needs fp8_weights or int4_weights")


def layer_matrix_spec(name: str, shape: tuple, fp8_weights: bool, int4_weights: bool = False) -> Dict[str, tuple]:
    """Engine tensor name -> (shape, dtype) of one layer matrix [N, K] in the chosen form."""
    _weight_form(fp8_weights, int4_weights)
    if int4_weights:
        n, k = shape
        n_pad = -(-n // INT4_TILE) * INT4_TILE
        return {name + ".i4": ((n_pad * k // 2,), torch.uint8), name + ".gscale": ((n, k // INT4_GROUP), torch.bfloat16)}
    if not fp8_weights:
        return {name: (shape, torch.bfloat16)}
    return {name + ".f8": (shape, torch.uint8), name + ".scale": ((shape[0],), torch.float32)}


def vocab_matrix_spec(name: str, shape: tuple, fp8_weights: bool, int4_weights: bool = False,
                      quantize_vocab: bool = False) -> Dict[str, tuple]:
    """Engine tensor name -> (shape, dtype) of a vocabulary matrix (embed, lm_head): bf16, or with quantize_vocab in the
    layer matrices' form."""
    _vocab_form(fp8_weights, int4_weights, quantize_vocab)
    return layer_matrix_spec(name, shape, fp8_weights and quantize_vocab, int4_weights and quantize_vocab)


def dequantized_vocab_matrix(weights: StateDict, name: str, n: int, k: int) -> torch.Tensor:
    """bf16 [n, k] of vocabulary matrix `name` in whichever form `weights` holds it: the matrix every engine kernel
    multiplies or gathers (the bf16 tensor itself when it is not quantized; a new tensor otherwise)."""
    if name + ".i4" in weights:
        return dequantize_int4_groups(unpack_int4_codes(weights[name + ".i4"], n, k), weights[name + ".gscale"])
    if name + ".f8" in weights:
        return dequantize_fp8_rows_bf16(weights[name + ".f8"].view(n, k), weights[name + ".scale"])
    return weights[name]


def _put_layer_matrix(out: StateDict, name: str, w: torch.Tensor, fp8_weights: bool, int4_weights: bool = False) -> None:
    # quantized on w's device, one matrix at a time: the bf16 matrix is dropped as soon as its codes exist
    _weight_form(fp8_weights, int4_weights)
    if int4_weights:
        q, s = quantize_int4_groups(w)
        out[name + ".i4"], out[name + ".gscale"] = pack_int4_codes(q), s
    elif fp8_weights:
        out[name + ".f8"], out[name + ".scale"] = quantize_fp8_rows(w)
    else:
        out[name] = w


def pack_llm_for_engine(cfg: LiveConfig, sd: StateDict, device, max_positions: int, fp8_weights: bool = False,
                        int4_weights: bool = False, quantize_vocab: bool = False) -> StateDict:
    """quantize_vocab (with fp8_weights or int4_weights): embed and lm_head in the layer matrices' form too, quantized
    after the LoRA merge (the adapter targets lm_head)."""
    _vocab_form(fp8_weights, int4_weights, quantize_vocab)
    qf8, qi4 = fp8_weights and quantize_vocab, int4_weights and quantize_vocab
    bf = torch.bfloat16
    out: StateDict = {}

    def take(k):
        return sd[k].to(device=device, dtype=bf).contiguous()

    _put_layer_matrix(out, "embed", take("model.embed_tokens.weight"), qf8, qi4)
    out["final_norm"] = take("model.norm.weight")
    _put_layer_matrix(out, "lm_head", take("lm_head.weight"), qf8, qi4)
    cos, sin = rope_tables(cfg, max_positions, device)
    out["rope.cos"], out["rope.sin"] = cos, sin
    for i in range(cfg.num_hidden_layers):
        p = f"model.layers.{i}."
        out[f"L{i}.in_norm"] = take(p + "input_layernorm.weight")
        out[f"L{i}.post_norm"] = take(p + "post_attention_layernorm.weight")
        _put_layer_matrix(out, f"L{i}.qkv", torch.cat([take(p + "self_attn.q_proj.weight"),
                                                       take(p + "self_attn.k_proj.weight"),
                                                       take(p + "self_attn.v_proj.weight")], 0).contiguous(), fp8_weights,
                          int4_weights)
        _put_layer_matrix(out, f"L{i}.o", take(p + "self_attn.o_proj.weight"), fp8_weights, int4_weights)
        _put_layer_matrix(out, f"L{i}.gate_up", interleave_gate_up(take(p + "mlp.gate_proj.weight"),
                                                                   take(p + "mlp.up_proj.weight")), fp8_weights, int4_weights)
        _put_layer_matrix(out, f"L{i}.down", take(p + "mlp.down_proj.weight"), fp8_weights, int4_weights)
    if "connector.0.weight" in sd:
        out["conn.0.w"] = take("connector.0.weight")
        out["conn.0.b"] = _b32_from16(sd["connector.0.bias"].to(device), bf)
        out["conn.2.w"] = take("connector.2.weight")
        out["conn.2.b"] = _b32_from16(sd["connector.2.bias"].to(device), bf)
    return out


def pack_vision_for_engine(cfg: LiveConfig, sd: StateDict, device) -> StateDict:
    f16, f32 = torch.float16, torch.float32
    C = cfg.vision_hidden_size
    out: StateDict = {}

    def w16(k):
        return sd[k].to(device=device, dtype=f16).contiguous()

    def b32(k):  # bias as the fp16 autocast copy would hold it
        return _b32_from16(sd[k].to(device), f16)

    def f(k):
        return sd[k].to(device=device, dtype=f32).contiguous()

    out["vit.patch.w"] = w16("embeddings.patch_embedding.weight").reshape(C, -1).contiguous()
    out["vit.patch.b"] = b32("embeddings.patch_embedding.bias")
    out["vit.pos"] = f("embeddings.position_embedding.weight")
    out["vit.post_ln.w"], out["vit.post_ln.b"] = f("post_layernorm.weight"), f("post_layernorm.bias")
    for i in range(cfg.vision_num_hidden_layers):
        p, q = f"encoder.layers.{i}.", f"vit.L{i}."
        out[q + "ln1.w"], out[q + "ln1.b"] = f(p + "layer_norm1.weight"), f(p + "layer_norm1.bias")
        out[q + "ln2.w"], out[q + "ln2.b"] = f(p + "layer_norm2.weight"), f(p + "layer_norm2.bias")
        out[q + "qkv.w"] = torch.cat([w16(p + f"self_attn.{n}_proj.weight") for n in "qkv"], 0).contiguous()
        out[q + "qkv.b"] = torch.cat([b32(p + f"self_attn.{n}_proj.bias") for n in "qkv"], 0).contiguous()
        out[q + "out.w"], out[q + "out.b"] = w16(p + "self_attn.out_proj.weight"), b32(p + "self_attn.out_proj.bias")
        out[q + "fc1.w"], out[q + "fc1.b"] = w16(p + "mlp.fc1.weight"), b32(p + "mlp.fc1.bias")
        out[q + "fc2.w"], out[q + "fc2.b"] = w16(p + "mlp.fc2.weight"), b32(p + "mlp.fc2.bias")
    if cfg.frame_token_cls:
        ipw, ipb = sd["head.attention.in_proj_weight"].to(device), sd["head.attention.in_proj_bias"].to(device)
        # q of the constant probe, as the fp16 autocast Linear would produce it (fp32 accumulate, one rounding)
        probe16 = sd["head.probe"].to(device).reshape(1, C).to(f16).float()
        q = probe16 @ ipw[:C].to(f16).float().t() + ipb[:C].to(f16).float()
        out["vit.head.q"] = q.reshape(C).to(f16).to(f32).contiguous()
        out["vit.head.kv.w"] = ipw[C:].to(f16).contiguous()
        out["vit.head.kv.b"] = _b32_from16(ipb[C:], f16)
        out["vit.head.out.w"], out["vit.head.out.b"] = w16("head.attention.out_proj.weight"), b32("head.attention.out_proj.bias")
        out["vit.head.ln.w"], out["vit.head.ln.b"] = f("head.layernorm.weight"), f("head.layernorm.bias")
        out["vit.head.fc1.w"], out["vit.head.fc1.b"] = w16("head.mlp.fc1.weight"), b32("head.mlp.fc1.bias")
        out["vit.head.fc2.w"], out["vit.head.fc2.b"] = w16("head.mlp.fc2.weight"), b32("head.mlp.fc2.bias")
    return out


def synthetic_engine_weights(cfg: LiveConfig, device, max_positions: int, seed: int = 0, std: float = 0.02,
                             fp8_weights: bool = False, int4_weights: bool = False, quantize_vocab: bool = False) -> StateDict:
    """Full-size synthetic weights generated directly in the engine layout on `device` (bench path: no
    16 GB host round trip).  Same distributions as synthetic_*_state, different random stream.  fp8_weights /
    int4_weights: the layer matrices of the same seed, quantized; quantize_vocab: embed and lm_head too."""
    _vocab_form(fp8_weights, int4_weights, quantize_vocab)
    qf8, qi4 = fp8_weights and quantize_vocab, int4_weights and quantize_vocab
    g = torch.Generator(device=device).manual_seed(seed)
    bf, f16, f32 = torch.bfloat16, torch.float16, torch.float32
    H, I, V = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size
    nh, nkv, hd = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    C, M, ps, P = cfg.vision_hidden_size, cfg.vision_intermediate_size, cfg.vision_patch_size, cfg.num_patches
    out: StateDict = {}
    _put_layer_matrix(out, "embed", _gen((V, H), 1.0, g, device, bf), qf8, qi4)
    out["final_norm"] = _gen((H,), 0.1, g, device, bf, 1.0)
    _put_layer_matrix(out, "lm_head", _gen((V, H), std, g, device, bf), qf8, qi4)
    out["rope.cos"], out["rope.sin"] = rope_tables(cfg, max_positions, device)
    for i in range(cfg.num_hidden_layers):
        out[f"L{i}.in_norm"] = _gen((H,), 0.1, g, device, bf, 1.0)
        out[f"L{i}.post_norm"] = _gen((H,), 0.1, g, device, bf, 1.0)
        _put_layer_matrix(out, f"L{i}.qkv", _gen(((nh + 2 * nkv) * hd, H), std, g, device, bf), fp8_weights, int4_weights)
        _put_layer_matrix(out, f"L{i}.o", _gen((H, nh * hd), std, g, device, bf), fp8_weights, int4_weights)
        _put_layer_matrix(out, f"L{i}.gate_up", _gen((2 * I, H), std, g, device, bf), fp8_weights, int4_weights)
        _put_layer_matrix(out, f"L{i}.down", _gen((H, I), std, g, device, bf), fp8_weights, int4_weights)
    out["conn.0.w"] = _gen((H, C), std, g, device, bf)
    out["conn.0.b"] = _gen((H,), std, g, device, bf).float()
    out["conn.2.w"] = _gen((H, H), std, g, device, bf)
    out["conn.2.b"] = _gen((H,), std, g, device, bf).float()
    out["vit.patch.w"] = _gen((C, 3 * ps * ps), std, g, device, f16)
    out["vit.patch.b"] = _gen((C,), std, g, device, f16).float()
    out["vit.pos"] = _gen((P, C), std, g, device, f32)
    out["vit.post_ln.w"], out["vit.post_ln.b"] = _gen((C,), 0.1, g, device, f32, 1.0), _gen((C,), std, g, device, f32)
    for i in range(cfg.vision_num_hidden_layers):
        q = f"vit.L{i}."
        for ln in ("ln1", "ln2"):
            out[q + ln + ".w"], out[q + ln + ".b"] = _gen((C,), 0.1, g, device, f32, 1.0), _gen((C,), std, g, device, f32)
        out[q + "qkv.w"], out[q + "qkv.b"] = _gen((3 * C, C), std, g, device, f16), _gen((3 * C,), std, g, device, f16).float()
        out[q + "out.w"], out[q + "out.b"] = _gen((C, C), std, g, device, f16), _gen((C,), std, g, device, f16).float()
        out[q + "fc1.w"], out[q + "fc1.b"] = _gen((M, C), std, g, device, f16), _gen((M,), std, g, device, f16).float()
        out[q + "fc2.w"], out[q + "fc2.b"] = _gen((C, M), std, g, device, f16), _gen((C,), std, g, device, f16).float()
    if cfg.frame_token_cls:
        out["vit.head.q"] = _gen((C,), 0.5, g, device, f16).float()
        out["vit.head.kv.w"], out["vit.head.kv.b"] = _gen((2 * C, C), std, g, device, f16), _gen((2 * C,), std, g, device, f16).float()
        out["vit.head.out.w"], out["vit.head.out.b"] = _gen((C, C), std, g, device, f16), _gen((C,), std, g, device, f16).float()
        out["vit.head.ln.w"], out["vit.head.ln.b"] = _gen((C,), 0.1, g, device, f32, 1.0), _gen((C,), std, g, device, f32)
        out["vit.head.fc1.w"], out["vit.head.fc1.b"] = _gen((M, C), std, g, device, f16), _gen((M,), std, g, device, f16).float()
        out["vit.head.fc2.w"], out["vit.head.fc2.b"] = _gen((C, M), std, g, device, f16), _gen((C,), std, g, device, f16).float()
    return out


def engine_weight_bytes(weights: StateDict) -> int:
    return sum(t.numel() * t.element_size() for t in weights.values())
