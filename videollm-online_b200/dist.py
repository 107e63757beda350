"""Multi-GPU plumbing: one process per GPU, independent video streams per process, full weight
replica per GPU.  The ONLY collective is the weight broadcast at start-up (NCCL over NVLink 5 /
NVSwitch via torch.distributed); the per-frame path has no cross-GPU step (SURVEY.md §8(e))."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from .config import LiveConfig
from .weights import layer_matrix_spec, vocab_matrix_spec


def engine_weight_spec(cfg: LiveConfig, max_positions: int, fp8_weights: bool = False,
                       int4_weights: bool = False, quantize_vocab: bool = False) -> Dict[str, tuple]:
    """name -> (shape, dtype) of every tensor of the engine layout (weights.py docstring), derivable on
    every rank without materialising anything.  fp8_weights: the layer matrices as e4m3 codes + row scales;
    int4_weights: as packed int4 codes + bf16 group scales; quantize_vocab: embed and lm_head in that form too."""
    bf, f16, f32 = torch.bfloat16, torch.float16, torch.float32
    H, I, V = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size
    nh, nkv, hd = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    C, M, ps, P = cfg.vision_hidden_size, cfg.vision_intermediate_size, cfg.vision_patch_size, cfg.num_patches
    s: Dict[str, tuple] = dict(vocab_matrix_spec("embed", (V, H), fp8_weights, int4_weights, quantize_vocab))
    s["final_norm"] = ((H,), bf)
    s.update(vocab_matrix_spec("lm_head", (V, H), fp8_weights, int4_weights, quantize_vocab))
    s.update({"rope.cos": ((max_positions, hd // 2), bf), "rope.sin": ((max_positions, hd // 2), bf)})
    for i in range(cfg.num_hidden_layers):
        s[f"L{i}.in_norm"] = ((H,), bf)
        s[f"L{i}.post_norm"] = ((H,), bf)
        s.update(layer_matrix_spec(f"L{i}.qkv", ((nh + 2 * nkv) * hd, H), fp8_weights, int4_weights))
        s.update(layer_matrix_spec(f"L{i}.o", (H, nh * hd), fp8_weights, int4_weights))
        s.update(layer_matrix_spec(f"L{i}.gate_up", (2 * I, H), fp8_weights, int4_weights))
        s.update(layer_matrix_spec(f"L{i}.down", (H, I), fp8_weights, int4_weights))
    s.update({"conn.0.w": ((H, C), bf), "conn.0.b": ((H,), f32), "conn.2.w": ((H, H), bf), "conn.2.b": ((H,), f32),
              "vit.patch.w": ((C, 3 * ps * ps), f16), "vit.patch.b": ((C,), f32), "vit.pos": ((P, C), f32),
              "vit.post_ln.w": ((C,), f32), "vit.post_ln.b": ((C,), f32)})
    for i in range(cfg.vision_num_hidden_layers):
        q = f"vit.L{i}."
        for ln in ("ln1", "ln2"):
            s[q + ln + ".w"], s[q + ln + ".b"] = ((C,), f32), ((C,), f32)
        s[q + "qkv.w"], s[q + "qkv.b"] = ((3 * C, C), f16), ((3 * C,), f32)
        s[q + "out.w"], s[q + "out.b"] = ((C, C), f16), ((C,), f32)
        s[q + "fc1.w"], s[q + "fc1.b"] = ((M, C), f16), ((M,), f32)
        s[q + "fc2.w"], s[q + "fc2.b"] = ((C, M), f16), ((C,), f32)
    if cfg.frame_token_cls:
        s.update({"vit.head.q": ((C,), f32), "vit.head.kv.w": ((2 * C, C), f16), "vit.head.kv.b": ((2 * C,), f32),
                  "vit.head.out.w": ((C, C), f16), "vit.head.out.b": ((C,), f32), "vit.head.ln.w": ((C,), f32),
                  "vit.head.ln.b": ((C,), f32), "vit.head.fc1.w": ((M, C), f16), "vit.head.fc1.b": ((M,), f32),
                  "vit.head.fc2.w": ((C, M), f16), "vit.head.fc2.b": ((C,), f32)})
    return s


def _flat_layout(spec: Dict[str, tuple], n_buckets: int):
    """Deal the tensors (sorted by name) into <= n_buckets contiguous byte ranges of similar size.
    Returns [(bucket_bytes, [(name, offset, shape, dtype)])]; offsets are 256-byte aligned (TMA / 16-byte vector loads)."""
    items = []
    for name in sorted(spec):
        shape, dtype = spec[name]
        n = 1
        for d in shape:
            n *= d
        items.append((name, shape, dtype, n * torch.empty(0, dtype=dtype).element_size()))
    total = sum(-(-b // 256) * 256 for *_, b in items)
    target = -(-total // max(1, n_buckets))
    buckets, cur, off = [], [], 0
    for name, shape, dtype, nbytes in items:
        cur.append((name, off, shape, dtype))
        off += -(-nbytes // 256) * 256
        if off >= target and len(buckets) < n_buckets - 1:
            buckets.append((off, cur))
            cur, off = [], 0
    if cur:
        buckets.append((off, cur))
    return buckets


def broadcast_weights(cfg: LiveConfig, weights: Optional[Dict[str, torch.Tensor]], device, max_positions: int,
                      dist=None, src: int = 0, n_buckets: int = 8, release_source: bool = False,
                      fp8_weights: bool = False, int4_weights: bool = False,
                      quantize_vocab: bool = False) -> Dict[str, torch.Tensor]:
    """Rank `src` passes its engine-layout dict, the others pass None; everyone returns the full dict on `device`.
    The ~560 tensors (16.7 GB) travel as <= `n_buckets` flat byte buffers, one NCCL broadcast each over NVLink/NVSwitch
    (per-tensor broadcasts cost 1.2 s at 8 GPUs: launch latency, not bandwidth); the returned tensors are views into
    those buffers (256-byte aligned), on the source rank too, so every rank ends with the same memory layout.
    release_source=True empties the source dict entry by entry while packing.  fp8_weights: every rank expects the layer
    matrices in the FP8 form (engine_weight_spec); int4_weights: in the int4 form; quantize_vocab: embed and lm_head too."""
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        if weights is None:
            raise ValueError("single process: weights must be provided")
        return weights
    spec = engine_weight_spec(cfg, max_positions, fp8_weights, int4_weights, quantize_vocab)
    out: Dict[str, torch.Tensor] = {}
    is_src = dist.get_rank() == src
    if is_src:
        missing = set(spec) - set(weights)
        if missing:
            raise KeyError(f"source rank lacks tensors: {sorted(missing)[:5]}")
    for nbytes, members in _flat_layout(spec, n_buckets):
        flat = torch.empty(nbytes, dtype=torch.uint8, device=device)
        views = []
        for name, off, shape, dtype in members:
            n = 1
            for d in shape:
                n *= d
            esz = torch.empty(0, dtype=dtype).element_size()
            v = flat[off:off + n * esz].view(dtype).view(*shape)
            if is_src:
                t = weights[name]
                if tuple(t.shape) != tuple(shape) or t.dtype != dtype:
                    raise ValueError(f"{name}: {tuple(t.shape)}/{t.dtype} does not match spec {shape}/{dtype}")
                v.copy_(t.to(device), non_blocking=True)
                if release_source:
                    weights[name] = None      # drop the source copy as soon as it is packed (16.7 GB at full size)
            views.append((name, v))
        dist.broadcast(flat, src=src)
        for name, v in views:
            out[name] = v
    return out
