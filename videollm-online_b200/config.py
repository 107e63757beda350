"""Configuration surface of the hot path.

Mirrors the fields `LiveInfer` and the builders read from the reference's
`LiveLlamaConfig` (= LlamaConfig + LiveConfigMixin, models/configuration_live.py:5-21,
models/live_llama/configuration_live_llama.py:5-6) and the `live1+` argument preset
(models/arguments_live.py:5-47).  Plain dataclasses: HF `TrainingArguments` cannot even be
instantiated offline (needs `accelerate`), and nothing on this path needs it.
"""
from __future__ import annotations

import argparse
import dataclasses
import math
from dataclasses import dataclass, field
from typing import List, Optional

SYSTEM_PROMPT = (
    "A multimodal AI assistant is helping users with some activities."
    " Below is their conversation, interleaved with the list of video frames received by the assistant."
)


@dataclass
class LiveConfig:
    """Model config: Llama decoder + SigLIP tower + live fields (same attribute names as the reference)."""
    # --- LlamaConfig fields
    hidden_size: int = 4096
    num_hidden_layers: int = 32
    num_attention_heads: int = 32
    num_key_value_heads: int = 8
    head_dim: int = 128
    intermediate_size: int = 14336
    vocab_size: int = 128256
    rms_norm_eps: float = 1e-5
    rope_theta: float = 500000.0
    max_position_embeddings: int = 8192
    bos_token_id: int = 128000
    eos_token_id: int = 128009
    # --- SiglipVisionConfig fields (google/siglip-large-patch16-384)
    vision_pretrained: str = "google/siglip-large-patch16-384"
    vision_hidden_size: int = 1024
    vision_num_hidden_layers: int = 24
    vision_num_attention_heads: int = 16
    vision_intermediate_size: int = 4096
    vision_patch_size: int = 16
    vision_layer_norm_eps: float = 1e-6
    # --- LiveConfigMixin fields (models/configuration_live.py:5-21)
    frame_resolution: int = 384
    frame_token_cls: bool = True
    frame_token_pooled: Optional[List[int]] = field(default_factory=lambda: [3, 3])
    frame_num_tokens: int = 10
    v_placeholder: str = "<v>"
    frame_token_interval: str = ","
    v_placeholder_id: int = 128256
    frame_token_interval_id: int = 11  # "," in the Llama-3 vocabulary
    stream_loss_weight: float = 1.0
    # id of "]\n", asserted by the reference before a streamed response (demo/inference.py:44)
    stream_end_id: int = 933

    def __post_init__(self):
        n = (1 if self.frame_token_cls else 0)
        if self.frame_token_pooled:
            n += self.frame_token_pooled[0] * self.frame_token_pooled[1]
        if self.frame_num_tokens != n:
            raise ValueError(f"frame_num_tokens={self.frame_num_tokens} inconsistent with cls/pooled -> {n}")

    @property
    def num_patches(self) -> int:
        g = self.frame_resolution // self.vision_patch_size
        return g * g

    def to_dict(self):
        return dataclasses.asdict(self)


def llama3_8b_siglip_l() -> LiveConfig:
    """The shipped `live1+` model: Llama-3-8B-Instruct + SigLIP-L/16-384 (BASELINE.json configs)."""
    return LiveConfig()


def tiny_config(**over) -> LiveConfig:
    """Small same-architecture config for parity tests (oracle runs in seconds on CPU)."""
    base = dict(
        hidden_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, head_dim=128,
        intermediate_size=512, vocab_size=1024, max_position_embeddings=512, bos_token_id=1, eos_token_id=2,
        vision_hidden_size=128, vision_num_hidden_layers=2, vision_num_attention_heads=2,
        vision_intermediate_size=256, vision_patch_size=16, frame_resolution=96,
        v_placeholder_id=1024, frame_token_interval_id=11, stream_end_id=933,
    )
    base.update(over)
    return LiveConfig(**base)


@dataclass
class SamplingConfig:
    """How response tokens are picked, with the names and defaults of HF's GenerationConfig.  do_sample False: greedy
    (the argmax, what every response is without a config).  do_sample True: each token is drawn on the device
    (include/vlo_b200.h, vlo_sample) after the repetition penalty over the response's prompt ids and the ids generated
    so far, the temperature, top-k (0: off) and top-p (1: off).  The noise is a function of (seed, KV position), so a
    response is reproducible from the seed and its ids do not depend on drafts, batching or a suspend / resume."""
    do_sample: bool = False
    temperature: float = 1.0
    top_k: int = 50
    top_p: float = 1.0
    repetition_penalty: float = 1.0
    seed: int = 0

    def __post_init__(self):
        if not (math.isfinite(self.temperature) and self.temperature > 0):
            raise ValueError(f"temperature must be finite and > 0, got {self.temperature}")
        if isinstance(self.top_k, bool) or not isinstance(self.top_k, int) or self.top_k < 0:
            raise ValueError(f"top_k must be an int >= 0 (0: off), got {self.top_k!r}")
        if not (0 < self.top_p <= 1):
            raise ValueError(f"top_p must lie in (0, 1], got {self.top_p}")
        if not (math.isfinite(self.repetition_penalty) and self.repetition_penalty > 0):
            raise ValueError(f"repetition_penalty must be finite and > 0, got {self.repetition_penalty}")
        if isinstance(self.seed, bool) or not isinstance(self.seed, int) or not 0 <= self.seed < 1 << 64:
            raise ValueError(f"seed must be an int in [0, 2^64), got {self.seed!r}")
        if not self.do_sample and self.repetition_penalty != 1.0:
            raise ValueError("repetition_penalty applies to sampled responses: set do_sample=True (greedy responses "
                             "take the plain argmax)")

    @classmethod
    def from_args(cls, args: "LiveArguments") -> Optional["SamplingConfig"]:
        """The config the --do_sample / --temperature / --top_k / --top_p / --repetition_penalty / --sample_seed flags
        ask for; None (greedy) without --do_sample."""
        cfg = cls(do_sample=args.do_sample, temperature=args.temperature, top_k=args.top_k, top_p=args.top_p,
                  repetition_penalty=args.repetition_penalty, seed=args.sample_seed)
        return cfg if cfg.do_sample else None


@dataclass
class LiveArguments:
    """Flag surface of `models.parse_args()` that the inference path reads
    (models/arguments_live.py:5-28,40-47; demo/inference.py:14-35)."""
    live_version: str = "live1+"
    system_prompt: str = SYSTEM_PROMPT
    llm_pretrained: str = "meta-llama/Meta-Llama-3-8B-Instruct"
    vision_pretrained: str = "google/siglip-large-patch16-384"
    resume_from_checkpoint: str = ""
    attn_implementation: str = "vlo_b200"  # accepted for CLI compatibility; there is one implementation
    frame_fps: int = 2
    frame_resolution: int = 384
    frame_token_cls: Optional[bool] = None
    frame_token_pooled: Optional[List[int]] = None
    frame_num_tokens: Optional[int] = None
    frame_token_interval: Optional[str] = None
    frame_token_interval_threshold: float = 0.0
    max_num_frames: Optional[int] = None
    lora_r: int = 128
    lora_alpha: int = 256
    # engine-side additions
    device: str = "cuda:0"
    max_streams: int = 1
    kv_pool_tokens: int = 0  # KV page pool shared by the streams, tokens; 0: max_streams x the per-stream cap
    synthetic_weights: bool = False
    seed: int = 0            # of the synthetic weights
    # serve the decoder layers' q|k|v, o, gate|up and down matrices from e4m3 codes with one fp32 scale per row (half the
    # weight bytes per step); changes the model's numbers, so off by default
    fp8_weights: bool = False
    # with fp8_weights: quantize each layer GEMM's activations to e4m3 per token and multiply on the FP8 tensor cores
    # (W8A8); changes the model's numbers again, so off by default
    fp8_activations: bool = False
    # serve the decoder layer matrices from 4-bit codes with one bf16 scale per 128 weights of a row (W4A16, a quarter of
    # the bf16 bytes); changes the model's numbers, so off by default; excludes fp8_weights and fp8_activations
    int4_weights: bool = False
    # with fp8_weights or int4_weights: also serve embed and lm_head in that quantized form (frees 1.05 GB with FP8 and
    # 1.56 GB with int4 weights at Llama-3-8B); changes the model's numbers, so off by default
    quantize_vocab: bool = False
    # with fp8_weights or int4_weights: prefill long single-stream inputs on the quantized layers too, with the bits of
    # max_step_tokens steps; grows the token-row workspaces to 8 x max_step_tokens rows, so off by default
    quantized_prefill: bool = False
    # LiveInfer.context_window, tokens: keep the start prompt and drop the oldest cache pages after it so the session's
    # cache never exceeds this many tokens; 0: off (the cache grows until max_kv_tokens)
    context_window: int = 0
    # LiveInfer.context_keep_turns: with a context window, drop old frames token by token and keep the questions and
    # answers (engine.retain_spans) instead of dropping whole pages; no effect without a window
    context_keep_turns: bool = False
    # response sampling (SamplingConfig; HF GenerationConfig names, sample_seed = its seed); greedy without --do_sample
    do_sample: bool = False
    temperature: float = 1.0
    top_k: int = 50
    top_p: float = 1.0
    repetition_penalty: float = 1.0
    sample_seed: int = 0


def _apply_version(args: LiveArguments) -> LiveArguments:
    if args.live_version == "live1":  # models/arguments_live.py:31-37
        d = dict(frame_token_cls=True, frame_token_pooled=None, frame_num_tokens=1, frame_token_interval="",
                 max_num_frames=7200)
    elif args.live_version == "live1+":  # models/arguments_live.py:40-47
        d = dict(frame_token_cls=True, frame_token_pooled=[3, 3], frame_num_tokens=10, frame_token_interval=",",
                 max_num_frames=1200)
    else:
        raise NotImplementedError(args.live_version)
    for k, v in d.items():
        if getattr(args, k) is None:
            setattr(args, k, v)
    return args


def parse_args(argv=None) -> LiveArguments:
    """Two-pass parse like models/__init__.py:7-10: read live_version, then apply its preset."""
    p = argparse.ArgumentParser(allow_abbrev=False)
    for f in dataclasses.fields(LiveArguments):
        if f.name in ("frame_token_pooled",):
            p.add_argument(f"--{f.name}", type=int, nargs="+", default=None)
        elif f.type in ("bool", "Optional[bool]") or isinstance(f.default, bool):
            # `--flag true|false`, or `--flag` alone for true
            p.add_argument(f"--{f.name}", type=lambda s: s.lower() in ("1", "true", "yes"), nargs="?", const=True,
                           default=f.default)
        elif isinstance(f.default, int):
            p.add_argument(f"--{f.name}", type=int, default=f.default)
        elif isinstance(f.default, float):
            p.add_argument(f"--{f.name}", type=float, default=f.default)
        elif f.name in ("frame_num_tokens", "max_num_frames"):
            p.add_argument(f"--{f.name}", type=int, default=None)
        else:
            p.add_argument(f"--{f.name}", type=str, default=f.default)
    ns, _unknown = p.parse_known_args(argv)
    return _apply_version(LiveArguments(**vars(ns)))
