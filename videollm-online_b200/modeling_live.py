"""Host-side mirror of the reference's model API for the inference path.

Keeps the names `demo/inference.py` calls — `build_model_and_tokenizer`, `fast_greedy_generate`,
`model.config`, `model.to`, `model.get_input_embeddings()`, `model.visual_embed`, `model.joint_embed`,
`model(inputs_embeds=..., past_key_values=..., use_cache=True)` — over the CUDA engine
(reference: models/modeling_live.py:11-42,173-222; models/live_llama/modeling_live_llama.py:11-73).
All arithmetic happens in libvlo_b200.so; this file only moves handles around.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

from .config import LiveArguments, LiveConfig, llama3_8b_siglip_l
from .engine import Engine, VloError
from .tokenization_live import build_live_tokenizer_and_update_config
from . import weights as W


class StreamKV:
    """The `past_key_values` object: an opaque handle on one engine-owned KV stream.  Falsy until it
    holds tokens, like `None` / an empty DynamicCache (demo/inference.py:61,98)."""

    def __init__(self, engine: Engine, stream_id: int):
        self.engine, self.stream_id = engine, stream_id

    def get_seq_length(self) -> int:
        return self.engine.kv_len(self.stream_id)

    def __len__(self):
        return self.get_seq_length()

    def __bool__(self):
        return self.get_seq_length() > 0

    def crop(self, max_length: int):
        """trim_past_key_values(0, max_length) (models/modeling_live.py:170-171)."""
        self.engine.kv_truncate(self.stream_id, max_length)
        return self


@dataclass
class LiveOutput:
    """CausalLMOutputWithPast look-alike.  `logits` holds the LAST position only ([B, 1, V]); the
    reference computes all positions but reads only [:, -1:] (demo/inference.py:76,
    models/modeling_live.py:177).  `decisions` is the device-side summary of that row."""
    logits: torch.Tensor
    past_key_values: StreamKV
    decisions: torch.Tensor
    loss: Optional[torch.Tensor] = None


class _Embedding:
    def __init__(self, engine: Engine):
        self.engine = engine

    def __call__(self, ids: torch.Tensor) -> torch.Tensor:
        shape = tuple(ids.shape)
        return self.engine.embed_tokens(ids).view(*shape, self.engine.cfg.hidden_size)

    @property
    def weight(self) -> torch.Tensor:
        """bf16 [V, H], the table the engine gathers from.  With quantized vocabulary matrices it is dequantized on every
        access into a new tensor (1.05 GB at Llama-3-8B's shape): keep it only as long as it is needed."""
        from .weights import dequantized_vocab_matrix
        cfg = self.engine.cfg
        return dequantized_vocab_matrix(self.engine.weights, "embed", cfg.vocab_size, cfg.hidden_size)


class LiveLlamaForCausalLM:
    """Engine-backed stand-in for models.live_llama.LiveLlamaForCausalLM (inference surface only)."""

    def __init__(self, config: LiveConfig, engine: Engine):
        self.config = config
        self.engine = engine
        self.dtype = torch.bfloat16
        self.vocab_size = config.vocab_size
        self._embed = _Embedding(engine)
        self._default_stream: Optional[int] = None
        self.has_vision = any(k.startswith("vit.") for k in engine.weights)

    # --- torch-module idioms the reference uses
    def to(self, device=None, *a, **k):
        if device is not None and torch.device(device) != self.engine.device and torch.device(device).type == "cuda" \
                and torch.device(device).index not in (None, self.engine.index):
            raise VloError("an engine is pinned to its GPU; build another engine for another device")
        return self

    def eval(self):
        return self

    def requires_grad_(self, flag: bool = False):
        return self

    @property
    def device(self):
        return self.engine.device

    def get_input_embeddings(self):
        return self._embed

    # --- LiveMixin
    def set_vision_inside(self):
        if not self.has_vision:
            raise VloError("vision tower weights were not loaded")

    def visual_embed(self, frames: torch.Tensor) -> torch.Tensor:
        """models/modeling_live.py:21-27.  uint8 frames -> ViT + connector; float features
        ([N, frame_num_tokens, vision_hidden], pre-extracted) -> connector only."""
        if frames.dtype == torch.uint8:
            if not self.has_vision:
                raise VloError("visual_embed got raw frames but no vision tower is loaded")
            return self.engine.vit_encode(frames)
        return self.engine.connector(frames)

    def joint_embed(self, input_ids: torch.Tensor = None, frames: torch.Tensor = None) -> torch.Tensor:
        """models/modeling_live.py:29-42."""
        if frames is None:
            return self.get_input_embeddings()(input_ids)
        if input_ids is None:
            return self.visual_embed(frames)
        embeds = self.get_input_embeddings()(input_ids.clamp(max=self.vocab_size - 1))
        v_mask = input_ids.to(embeds.device) == self.config.v_placeholder_id
        if v_mask.any():
            embeds[v_mask] = self.visual_embed(frames)
        return embeds

    def new_stream(self) -> StreamKV:
        return StreamKV(self.engine, self.engine.stream_open())

    # --- evaluation (SURVEY 8(f) row 4)
    def forward_all_logits(self, inputs_embeds: torch.Tensor, past_key_values: StreamKV) -> torch.Tensor:
        """Teacher-forced KV-append forward returning the logits of EVERY position ([L, V] bf16), fed in pieces of
        the engine's one-pass capacity (prefills of max_prefill_tokens, or steps of max_step_tokens; chunked streaming
        == one causal pass): the reference's `self.forward(..., use_cache=True).logits[0]` (models/modeling_live.py:67)
        on the engine's cache."""
        eng = self.engine
        x = inputs_embeds.reshape(-1, self.config.hidden_size).to(torch.bfloat16)
        outs, cap = [], eng.max_pass_tokens
        for lo in range(0, x.shape[0], cap):
            chunk = x[lo:lo + cap].contiguous()
            eng.step([past_key_values.stream_id], [chunk.shape[0]], chunk, want_logits=False)
            outs.append(eng.last_step_logits(chunk.shape[0]))
        return torch.cat(outs, 0)

    @torch.no_grad()
    def stream_evaluate(self, input_ids: torch.LongTensor, labels: torch.LongTensor, frames: torch.Tensor,
                        ignore_token_id: int = -100, frame_token_interval_threshold: float = 0.0, **kwargs):
        """models/modeling_live.py:44-168 on the engine: same metrics, same order of operations.  The full forward runs
        through `forward_all_logits`; the look-ahead of a turn whose frames were all judged "silent" (:110-141) runs on
        a scratch stream holding a copy of the first `stop` cache positions (`vlo_kv_copy_prefix`, the engine's
        trim_past_key_values(pkv, 0, stop)), so the evaluated conversation's own cache survives.
        Returns tensor([lm_ppl, frame_diff, fluency, lm_correctness]) on the engine's device."""
        assert input_ids.size(0) == labels.size(0) == 1
        eng, cfg, dev = self.engine, self.config, self.engine.device
        input_id, label = input_ids[0].to(dev), labels[0].to(dev)
        frames = frames.to(dev)
        zero = torch.tensor(0, dtype=torch.int, device=dev)
        one = torch.tensor(1, dtype=torch.int, device=dev)
        turn_stops = ((input_id == cfg.eos_token_id).nonzero() + 1)[:, 0].tolist()
        turn_starts = [0] + turn_stops[:-1]
        num_turns = len(turn_starts)
        kv, scratch = self.new_stream(), None
        try:
            logit = self.forward_all_logits(self.joint_embed(input_id[None], frames)[0], kv)
            v_id = cfg.v_placeholder_id
            use_interval = cfg.frame_token_interval_id is not None
            interval_id = cfg.frame_token_interval_id if use_interval else cfg.eos_token_id
            fnt = int(cfg.frame_token_cls) + (cfg.frame_token_pooled[0] * cfg.frame_token_pooled[1] if cfg.frame_token_pooled else 0)
            past_num_frames = 0
            lm_ppls, frame_diffs, fluencies, lm_correctness = [], [], [], []
            for r, (turn_start, turn_stop) in enumerate(zip(turn_starts, turn_stops)):
                turn_label = label[turn_start:turn_stop]
                turn_learn_mask = turn_label != ignore_token_id
                if not turn_learn_mask.any():
                    continue
                turn_logit = logit[turn_start:turn_stop]
                turn_input_id = input_id[turn_start:turn_stop]
                turn_v_mask = turn_input_id == v_id
                turn_num_frames = turn_v_mask.sum() // fnt
                turn_stream_mask = turn_v_mask & turn_learn_mask
                turn_lm_mask = turn_learn_mask & ~turn_stream_mask
                if turn_lm_mask.any():
                    ml, mt = turn_logit[turn_lm_mask], turn_label[turn_lm_mask]
                    lm_ppls.append(torch.nn.functional.cross_entropy(ml, mt).exp())
                    wrong = ml.argmax(dim=-1) != mt
                    num_lm_correct_tokens = wrong.nonzero()[0, 0] if wrong.any() else (~wrong).sum()
                    lm_correctness.append(num_lm_correct_tokens / mt.numel())
                if turn_stream_mask.any():
                    score = turn_logit.softmax(dim=-1)[turn_stream_mask]
                    if frame_token_interval_threshold > 0:
                        score[score[:, interval_id] < frame_token_interval_threshold] = 0
                    pred = score.argmax(dim=-1) != interval_id
                    if pred.any():
                        frame_diff = turn_stream_mask.sum() - pred.nonzero()[0, 0] - 1
                    else:
                        last_stream_idx = turn_stream_mask.nonzero()[-1, 0]
                        if r == num_turns - 1:
                            frame_diff = zero
                        else:
                            next_nf = (input_id[turn_starts[r + 1]:turn_stops[r + 1]] == v_id).sum() // fnt
                            n_app = min(next_nf, turn_num_frames - 1)
                            if n_app == 0:
                                frame_diff = zero
                            else:
                                a0 = int(past_num_frames + turn_num_frames)
                                app_frames = frames[a0:a0 + int(n_app)]
                                ph = ([interval_id] if use_interval else []) + [v_id] * fnt
                                app_ids = torch.tensor(ph * int(n_app), dtype=torch.long, device=dev)
                                if scratch is None:
                                    scratch = self.new_stream()
                                eng.kv_copy_prefix(kv.stream_id, scratch.stream_id, int(turn_start + last_stream_idx + 1))
                                app_logit = self.forward_all_logits(self.joint_embed(app_ids[None], app_frames)[0], scratch)
                                idxs = torch.arange(len(ph) - 1, len(app_ids), len(ph), device=dev)
                                app_score = app_logit[idxs].softmax(dim=-1)
                                if frame_token_interval_threshold > 0:
                                    app_score[app_score[:, interval_id] < frame_token_interval_threshold] = 0
                                app_pred = app_score.argmax(dim=-1) != interval_id
                                frame_diff = -(app_pred.nonzero()[0, 0] + 1) if app_pred.any() else -n_app
                    frame_diffs.append(torch.as_tensor(frame_diff, device=dev).abs())
                if turn_lm_mask.any() and turn_stream_mask.any():
                    n_v = turn_stream_mask.sum()
                    n_valid = mt.numel() + n_v
                    if frame_diff == 0:
                        fluency = (n_v + num_lm_correct_tokens) / n_valid
                    elif frame_diff > 0:
                        fluency = (n_v - frame_diff) / n_valid
                    else:
                        fluency = (n_v - 1) / n_valid
                    fluencies.append(fluency)
                past_num_frames += turn_num_frames
        finally:
            eng.stream_close(kv.stream_id)
            if scratch is not None:
                eng.stream_close(scratch.stream_id)
        f32 = lambda t: torch.as_tensor(t, device=dev).float()
        lm_ppl = torch.stack(lm_ppls).mean() if lm_ppls else one
        frame_diff = torch.stack(frame_diffs).float().mean() if frame_diffs else zero
        fluency = torch.stack([f32(x) for x in fluencies]).mean() if fluencies else one
        lm_c = torch.stack([f32(x) for x in lm_correctness]).mean() if lm_correctness else one
        return torch.stack([f32(lm_ppl), f32(frame_diff), f32(fluency), f32(lm_c)])

    def __call__(self, input_ids: torch.Tensor = None, frames: torch.Tensor = None, inputs_embeds: torch.Tensor = None,
                 past_key_values: Optional[StreamKV] = None, use_cache: bool = True, return_dict: bool = True, **_):
        """KV-append forward (models/live_llama/modeling_live_llama.py:24-67), batch 1."""
        if inputs_embeds is None:
            inputs_embeds = self.joint_embed(input_ids, frames)
        if inputs_embeds.dim() == 3:
            if inputs_embeds.shape[0] != 1:
                raise VloError("model(...) is the reference's batch-1 API; use engine.step for ragged batches")
            inputs_embeds = inputs_embeds[0]
        if past_key_values is None:
            past_key_values = self._fresh_default_stream()
        q = inputs_embeds.shape[0]
        logits, dec = self.engine.step([past_key_values.stream_id], [q], inputs_embeds.to(torch.bfloat16))
        return LiveOutput(logits=logits.view(1, 1, -1), past_key_values=past_key_values, decisions=dec)

    forward = __call__

    def _fresh_default_stream(self) -> StreamKV:
        """the stream of a call without past_key_values: opened once, emptied on every such call"""
        if self._default_stream is None:
            self._default_stream = self.engine.stream_open()
        else:
            self.engine.stream_reset(self._default_stream)
        return StreamKV(self.engine, self._default_stream)


def fast_greedy_generate(*, model: LiveLlamaForCausalLM, inputs_embeds: torch.Tensor, past_key_values: StreamKV,
                         eos_token_id: int, inplace_output_ids: torch.Tensor):
    """models/modeling_live.py:173-182: greedy AR until EOS or the buffer is full.  The argmax is taken
    on the device; one 32-byte read-back per step replaces the reference's tensor `if` sync.  Ids the response
    has already produced serve as drafts (speculative.py): a step verifies several of them at once, and the ids and
    the cache are those of one token per step."""
    from .speculative import NgramDrafter, greedy_generate
    eng = model.engine
    if past_key_values is None:
        past_key_values = model._fresh_default_stream()
    sid = past_key_values.stream_id
    zeros = torch.zeros(eng.max_step_tokens, model.config.hidden_size, dtype=torch.bfloat16, device=eng.device)

    def step(ids, drafts):
        if ids is None:   # the caller's embeddings
            model(inputs_embeds=inputs_embeds, past_key_values=past_key_values, use_cache=True)
            return
        rows = ids + drafts
        eng.step([sid], [len(rows)], zeros[:len(rows)], row_ids=torch.tensor(rows, dtype=torch.int64),
                 segments=[[len(ids)] + [1] * len(drafts)] if drafts else None)

    n_first = inputs_embeds.reshape(-1, model.config.hidden_size).shape[0]
    ids = greedy_generate(eng, sid, step, n_first, inplace_output_ids.size(1), eos_token_id, drafter=NgramDrafter(),
                          base=eng.kv_len(sid))
    inplace_output_ids[:, :len(ids)] = torch.tensor(ids, dtype=inplace_output_ids.dtype)
    return inplace_output_ids[:, :len(ids)], past_key_values


def build_live(*, is_training: bool = False, config: Optional[LiveConfig] = None, llm_pretrained: str = None,
               resume_from_checkpoint: str = "", set_vision_inside: bool = False, device: str = "cuda:0",
               synthetic_weights: bool = False, seed: int = 0, max_streams: int = 1, max_kv_tokens: int = 16384,
               max_step_tokens: int = 128, max_vit_batch: int = 8, llm_state=None, vision_state=None,
               lora_r: int = 128, lora_alpha: int = 256, kv_pool_tokens: Optional[int] = None, fp8_weights: bool = False,
               fp8_activations: bool = False, int4_weights: bool = False, quantize_vocab: bool = False,
               quantized_prefill: bool = False, **kwargs):
    """models/modeling_live.py:184-222 for inference: build config + tokenizer, load (or synthesise)
    weights, merge LoRA, hand everything to the engine.  kv_pool_tokens: size of the KV page pool the streams
    share (None or <= 0: max_streams * max_kv_tokens).  fp8_weights: quantize the decoder layer matrices to e4m3 with
    per-row scales after the LoRA merge (weights.quantize_fp8_rows); the engine then runs its FP8-weight GEMMs.
    fp8_activations (needs fp8_weights): the layer GEMMs also quantize their activations to e4m3 per token and run on
    the FP8 tensor cores (W8A8).  int4_weights: quantize the layer matrices to 4-bit codes with one bf16 scale per 128
    weights of a row (weights.quantize_int4_groups, W4A16); the engine computes the bits of a bf16 engine on the
    dequantized weights.  It excludes fp8_weights and fp8_activations.  quantize_vocab (needs fp8_weights or
    int4_weights): embed and lm_head take the layer matrices' quantized form too (weights.pack_llm_for_engine).
    quantized_prefill (needs fp8_weights or int4_weights): long single-stream inputs run as prefills on the quantized
    layers too (Engine(quantized_prefill=True)), with the bits of max_step_tokens steps; it grows the engine's token-row
    workspaces to max_prefill_tokens rows."""
    if is_training:
        raise NotImplementedError("the vlo_b200 engine covers the streaming-inference path only")
    if int4_weights and (fp8_weights or fp8_activations):
        raise ValueError("int4_weights excludes fp8_weights and fp8_activations: the layer matrices take one form, and "
                         "4-bit weights multiply bf16 activations")
    if fp8_activations and not fp8_weights:
        raise ValueError("fp8_activations needs fp8_weights: the FP8 tensor cores take both operands in e4m3")
    if quantize_vocab and not (fp8_weights or int4_weights):
        raise ValueError("quantize_vocab needs fp8_weights or int4_weights: the vocabulary matrices take the layer "
                         "matrices' quantized form")
    if quantized_prefill and not (fp8_weights or int4_weights):
        raise ValueError("quantized_prefill needs fp8_weights or int4_weights: a bf16 engine always prefills")
    cfg = config or llama3_8b_siglip_l()
    for k in ("frame_resolution", "frame_token_cls", "frame_token_pooled", "frame_num_tokens", "frame_token_interval",
              "vision_pretrained"):
        if kwargs.get(k) is not None and hasattr(cfg, k):
            setattr(cfg, k, kwargs[k])
    tokenizer = build_live_tokenizer_and_update_config(llm_pretrained or "", cfg)
    engine = Engine(cfg, device, max_streams=max_streams, max_kv_tokens=max_kv_tokens,
                    max_step_tokens=max_step_tokens, max_vit_batch=max_vit_batch, kv_pool_tokens=kv_pool_tokens,
                    fp8_activations=fp8_activations, quantized_prefill=quantized_prefill)
    if llm_state is not None:
        packed = W.pack_llm_for_engine(cfg, llm_state, engine.device, max_kv_tokens, fp8_weights=fp8_weights,
                                       int4_weights=int4_weights, quantize_vocab=quantize_vocab)
        if set_vision_inside:
            if vision_state is None:
                raise VloError("set_vision_inside=True needs vision_state")
            packed.update(W.pack_vision_for_engine(cfg, vision_state, engine.device))
    elif synthetic_weights:
        packed = W.synthetic_engine_weights(cfg, engine.device, max_kv_tokens, seed=seed, fp8_weights=fp8_weights,
                                            int4_weights=int4_weights, quantize_vocab=quantize_vocab)
        if not set_vision_inside:
            packed = {k: v for k, v in packed.items() if not k.startswith("vit.")}
    else:
        packed = _load_checkpoints(cfg, llm_pretrained, resume_from_checkpoint, set_vision_inside, engine.device,
                                   max_kv_tokens, lora_r, lora_alpha, fp8_weights, int4_weights, quantize_vocab)
    engine.load_weights(packed)
    model = LiveLlamaForCausalLM(cfg, engine)
    return model, tokenizer


def _load_checkpoints(cfg, llm_pretrained, adapter, with_vision, device, max_positions, lora_r, lora_alpha,
                      fp8_weights=False, int4_weights=False, quantize_vocab=False):
    """Real weights: base Llama safetensors + PEFT adapter (+ SigLIP), local files only.  fp8_weights / int4_weights:
    the layer matrices are quantized after the LoRA merge, one at a time on `device`; quantize_vocab: embed and lm_head
    too."""
    import glob
    import os
    try:
        from safetensors.torch import load_file
    except Exception as e:  # pragma: no cover
        raise VloError(f"safetensors unavailable: {e}")
    if not llm_pretrained or not os.path.isdir(llm_pretrained):
        raise VloError(f"checkpoint directory '{llm_pretrained}' not found (no network here); pass "
                       "--synthetic_weights true to run with seeded random weights")
    sd = {}
    for f in sorted(glob.glob(os.path.join(llm_pretrained, "*.safetensors"))):
        sd.update(load_file(f))
    if adapter:
        ad = {}
        for f in sorted(glob.glob(os.path.join(adapter, "*.safetensors"))):
            ad.update(load_file(f))
        # the adapter's own hyper-parameters win over the CLI defaults (PEFT writes them next to the weights)
        acfg = os.path.join(adapter, "adapter_config.json")
        if os.path.isfile(acfg):
            import json
            with open(acfg) as fh:
                aj = json.load(fh)
            lora_r, lora_alpha = int(aj.get("r", lora_r)), float(aj.get("lora_alpha", lora_alpha))
        sd = W.merge_lora(sd, ad, lora_alpha=lora_alpha, lora_r=lora_r)
    packed = W.pack_llm_for_engine(cfg, sd, device, max_positions, fp8_weights=fp8_weights, int4_weights=int4_weights,
                                   quantize_vocab=quantize_vocab)
    if with_vision:
        vdir = cfg.vision_pretrained
        vs = {}
        for f in sorted(glob.glob(os.path.join(vdir, "*.safetensors"))):
            vs.update(load_file(f))
        vs = {k[len("vision_model."):]: v for k, v in vs.items() if k.startswith("vision_model.")}
        packed.update(W.pack_vision_for_engine(cfg, vs, device))
    return packed


def build_live_llama(**kwargs):
    """models/live_llama/modeling_live_llama.py:72-73."""
    return build_live(**kwargs)


build_model_and_tokenizer = build_live_llama
