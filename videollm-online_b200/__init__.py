"""videollm_online_b200 — native CUDA (H100, sm_90a) engine for VideoLLM-online's per-frame hot loop.

The directory is named `videollm-online_b200/`; import it as `videollm_online_b200` via the
repo-root bootstrap (`import vlo_bootstrap`), which registers this package under that name.
"""
from .config import LiveArguments, LiveConfig, SamplingConfig, llama3_8b_siglip_l, parse_args, tiny_config
from ._lib import VloError

__all__ = ["LiveArguments", "LiveConfig", "SamplingConfig", "llama3_8b_siglip_l", "parse_args", "tiny_config", "VloError",
           "build_model_and_tokenizer", "fast_greedy_generate", "LiveInfer", "Engine"]


def __getattr__(name):  # heavy modules (torch + ctypes engine) are imported lazily
    if name in ("build_model_and_tokenizer", "fast_greedy_generate", "build_live", "LiveLlamaForCausalLM", "StreamKV"):
        from . import modeling_live
        return getattr(modeling_live, name)
    if name == "LiveInfer":
        from .inference import LiveInfer
        return LiveInfer
    if name == "Engine":
        from .engine import Engine
        return Engine
    raise AttributeError(name)
