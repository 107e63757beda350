"""Python handle on one `vlo_engine` (one per GPU / process).

Thin: torch owns the weight storage (so torch.distributed/NCCL can broadcast it) and the
caller-visible tensors; every compute call goes through the C ABI in include/vlo_b200.h.
"""
from __future__ import annotations

import ctypes as C
import threading
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import torch

from . import _lib
from . import weights as W
from ._lib import VloConfig, VloDecision, VloError, VloSampleRow, check
from .config import LiveConfig

DECISION_DTYPE_FIELDS = 8  # 8 x 4 bytes


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


class Decision:
    """Host copy of one `vlo_decision`, plus the id `Engine.step(..., sample=...)` drew for its row (None: not
    sampled)."""
    __slots__ = ("argmax_id", "argmax_excl_id", "p_interval", "max_logit", "top2_margin", "lse", "argmax_prob_id",
                 "sampled_id")

    def __init__(self, row_i32: torch.Tensor, row_f32: torch.Tensor, sampled_id: Optional[int] = None):
        self.argmax_id = int(row_i32[0])
        self.argmax_excl_id = int(row_i32[1])
        self.p_interval = float(row_f32[2])
        self.max_logit = float(row_f32[3])
        self.top2_margin = float(row_f32[4])
        self.lse = float(row_f32[5])
        self.argmax_prob_id = int(row_i32[6])
        self.sampled_id = sampled_id

    def next_id(self, interval_id: int, threshold: float) -> int:
        """The reference's rule (demo/inference.py:76-79) on bf16 probabilities: if p(interval) < threshold the
        interval id is zeroed before the argmax.  torch compares the bf16 tensor with the Python float
        after casting the scalar to bf16, so do the same."""
        thr = float(torch.tensor(threshold, dtype=torch.bfloat16))
        if self.p_interval < thr:
            return self.argmax_excl_id
        return self.argmax_prob_id


class KvImage:
    """A stream's KV cache in pinned host memory (`Engine.kv_swap_out`), to be given back with `Engine.kv_swap_in`.

    `data`: uint8 [vlo_kv_image_bytes(n_tokens)], laid out [page][layer][K|V][kv_head][64][head_dim] bf16.  `layout`:
    (num_layers, num_kv_heads, head_dim, page_tokens), the config fields that layout depends on.  `event`: recorded
    after the copy that fills (or last read) `data`; None once the image is complete on the host.  An image survives
    torch.save / torch.load (the copy is waited for when it is saved, and the data pinned again when it is loaded)."""

    def __init__(self, data: torch.Tensor, n_tokens: int, layout: tuple, event: Optional[torch.cuda.Event] = None):
        self.data, self.n_tokens, self.layout, self.event = data, int(n_tokens), tuple(layout), event

    def synchronize(self) -> "KvImage":
        """Wait for the copy into `data`; it may then be read on the host."""
        if self.event is not None:
            self.event.synchronize()
            self.event = None
        return self

    def __getstate__(self):
        self.synchronize()
        return {"data": self.data.cpu(), "n_tokens": self.n_tokens, "layout": list(self.layout)}

    def __setstate__(self, st):
        data = st["data"]
        if torch.cuda.is_available() and not data.is_pinned():
            data = data.pin_memory()
        self.data, self.n_tokens, self.layout, self.event = data, int(st["n_tokens"]), tuple(st["layout"]), None


torch.serialization.add_safe_globals([KvImage])


def sink_tokens(keep_tokens: int, page: int) -> int:
    """Cache positions a context window never drops: the first ceil(keep_tokens / page) pages."""
    return -(-keep_tokens // page) * page


def evict_span(kv_len: int, need: int, window: int, keep_tokens: int, page: int) -> tuple[int, int]:
    """The one eviction policy of a context window: (first, n) = the cache positions to drop before a stream of kv_len
    positions appends `need` more, n = 0 when kv_len + need <= window.  The sink (`sink_tokens`) stays; after it the
    fewest whole pages that make kv_len + need <= window go, but at least window / 8 tokens' worth rounded up to pages
    (as many full pages as there are, if fewer), so the re-rotation of the tail is paid once per window / 8 tokens.
    Raises VloError when dropping every full page after the sink is not enough."""
    if kv_len + need <= window:
        return 0, 0
    first = sink_tokens(keep_tokens, page)
    avail = max(0, kv_len // page - first // page)          # full pages after the sink
    least = -(-(kv_len + need - window) // page)
    if least > avail:
        raise VloError(f"context window {window}: {kv_len} cached + {need} new tokens do not fit even after dropping "
                       f"every full page after the first {first} positions")
    return first, min(avail, max(least, -(-window // (8 * page)))) * page


def retain_spans(row_ids: Sequence[int], need: int, window: int, keep_tokens: int, interval_id: Optional[int],
                 frame_num_tokens: int) -> List[tuple[int, int]]:
    """The policy of a context window that keeps the conversation (`context_keep_turns`): the spans [(first, n), ...] of
    cache positions to keep before a stream appends `need` more, [] when len(row_ids) + need <= window.

    row_ids holds the id fed at every cache position, -1 for a frame row.  After the start prompt [0, keep_tokens),
    which stays exactly, the history is read as stream messages (frames of frame_num_tokens rows, one interval_id row
    between two frames of a message; none when interval_id is None) and the text between them: a turn is the text from
    the "]" that closes a message to the "\\n[" that reopens one.  What goes, in whole units:
      1. while the turn rows kept after the prompt exceed window / 2: the oldest whole turn, together with the last
         frame of the message before it, so the two messages merge as "... F , G ...";
      2. the oldest frames, each with the interval row after it; the last frame of a message never goes alone;
      3. older turns as in 1, if the frames were not enough.
    It stops once at least max(len(row_ids) + need - window, window / 8) positions go (window / 8 at least, so the
    compaction is paid once per window / 8 tokens), and raises VloError when dropping every unit is not enough.  The
    kept ids are then what the chat template renders for the same conversation with those frames and turns deleted,
    and every message that stays keeps at least one frame.  Text before the first or after the last frame stays."""
    kv_len = len(row_ids)
    excess = kv_len + need - window
    if excess <= 0:
        return []
    fnt, sep = frame_num_tokens, (0 if interval_id is None else 1)
    frames, texts = [], []           # frame starts; text runs (start, end) after the prompt, in order
    i = keep_tokens
    while i < kv_len:
        j = i
        if row_ids[i] < 0:
            while j < kv_len and row_ids[j] < 0:
                j += 1
            if (j - i) % fnt:
                raise VloError(f"context window: {j - i} frame rows at position {i} are not whole frames of {fnt}")
            frames.extend(range(i, j, fnt))
        else:
            while j < kv_len and row_ids[j] >= 0:
                j += 1
            texts.append((i, j))
        i = j
    is_frame = set(frames)
    # a frame continues its message when the next frame follows it after `sep` interval rows
    next_frame = lambda f: f + fnt + sep in is_frame and (not sep or row_ids[f + fnt] == interval_id)
    frame_units = [(f, f + fnt + sep) for f in frames if next_frame(f)]
    seps = {f + fnt for f in frames if sep and next_frame(f)}
    turns = [(s, e) for s, e in texts if s not in seps]          # the text rows the turn budget counts
    # a droppable turn lies between two messages: from the last frame before it to the first frame after it
    turn_units = [(s - fnt, e, e - s) for s, e in turns if s - fnt in is_frame and e in is_frame]
    text_rows = sum(e - s for s, e in turns)
    target = max(excess, -(-window // 8))
    dropped, n_drop, t = [], 0, 0
    while t < len(turn_units) and text_rows > window // 2:      # 1. the turn budget
        dropped.append(turn_units[t][:2])
        n_drop += turn_units[t][1] - turn_units[t][0]
        text_rows -= turn_units[t][2]
        t += 1
    for u in frame_units:                                        # 2. the oldest frames
        if n_drop >= target:
            break
        dropped.append(u)
        n_drop += u[1] - u[0]
    for u in turn_units[t:]:                                     # 3. older turns
        if n_drop >= target:
            break
        dropped.append(u[:2])
        n_drop += u[1] - u[0]
    if n_drop < excess:
        raise VloError(f"context window {window}: {kv_len} cached + {need} new tokens do not fit even after dropping "
                       f"every frame and turn that may go")
    spans, pos = [], 0
    for s, e in sorted(dropped):
        if s > pos:
            spans.append((pos, s - pos))
        pos = e
    if pos < kv_len:
        spans.append((pos, kv_len - pos))
    return spans


def kept_rows(seq: Sequence, spans: Sequence[tuple[int, int]]) -> list:
    """The entries of seq (one per cache position) that `spans` keep, in order."""
    return [x for f, n in spans for x in seq[f:f + n]]


def _check_window_arg(window, max_kv_tokens: int):
    if isinstance(window, bool) or not isinstance(window, int) or window <= 0:
        raise ValueError(f"context_window must be a positive int (tokens), got {window!r}")
    if window > max_kv_tokens:
        raise ValueError(f"context_window {window} exceeds the engine's max_kv_tokens ({max_kv_tokens})")


def check_context_window_turns(window: int, max_kv_tokens: int, keep_tokens: int, largest_need: int):
    """check_context_window for a window that keeps the conversation (`retain_spans`): within max_kv_tokens, and large
    enough for the start prompt, the turn budget (window / 2), one eviction chunk (window / 8) and the largest single
    step or response reserve (`largest_need`)."""
    _check_window_arg(window, max_kv_tokens)
    least = keep_tokens + window // 2 + -(-window // 8) + largest_need
    if window < least:
        raise ValueError(f"context_window {window} cannot hold the {keep_tokens}-token prompt, the turn budget "
                         f"({window // 2}), one eviction chunk and a step of {largest_need} tokens")


def check_context_window(window: int, max_kv_tokens: int, keep_tokens: int, largest_need: int, page: int):
    """Raise ValueError unless a context window of `window` tokens is usable: within max_kv_tokens, and large enough
    for the sink pages, one eviction chunk (window / 8 in whole pages) and the largest single step or response
    reserve (`largest_need`)."""
    _check_window_arg(window, max_kv_tokens)
    least = sink_tokens(keep_tokens, page) + -(-window // (8 * page)) * page + largest_need
    if window < least:
        raise ValueError(f"context_window {window} cannot hold the {sink_tokens(keep_tokens, page)}-token sink, one "
                         f"eviction chunk and a step of {largest_need} tokens: it must be >= {least}")


@dataclass
class SampleRow:
    """What `Engine.step(..., sample=...)` draws one decision row's id with (vlo_sample_row, include/vlo_b200.h).

    position: the KV position of the token whose logits the row holds (the noise depends on it and on the seed only).
    The repetition penalty applies to the first n_penalty ids of penalty_ids (None: all of them); rows of one step
    that pass the same list object share its upload, so the rows of a verify step can use one growing list."""
    seed: int
    position: int
    temperature: float = 1.0
    top_k: int = 0
    top_p: float = 1.0
    repetition_penalty: float = 1.0
    penalty_ids: Sequence[int] = ()
    n_penalty: Optional[int] = None


class Engine:
    def __init__(self, cfg: LiveConfig, device: str | torch.device = "cuda:0", *, max_streams: int = 1,
                 max_kv_tokens: int = 16384, max_step_tokens: int = 128, max_vit_batch: int = 8,
                 kv_pool_tokens: Optional[int] = None, fp8_activations: bool = False, quantized_prefill: bool = False):
        """kv_pool_tokens: size of the KV page pool all streams share (rounded up to 64-token pages); None reserves
        max_streams * max_kv_tokens, so every stream can reach max_kv_tokens at once.  A smaller pool over-subscribes:
        a step that needs more pages than are free raises VloError and leaves every stream as it was.
        fp8_activations: the layer GEMMs quantize their activations to e4m3 per token and multiply on the FP8 tensor
        cores (W8A8, vlo_set_fp8_activations); load_weights then needs FP8 layer weights.
        quantized_prefill: an engine with quantized layer matrices (FP8 weights, W8A8 or int4) prefills long inputs too
        (vlo_set_quantized_prefill), at the cost of token-row workspaces of max_prefill_tokens rows; load_weights then
        needs quantized layer weights."""
        self.lib = _lib.load()
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise VloError("the vlo_b200 engine runs on a CUDA (sm_90a) device only; there is no CPU path")
        if not torch.cuda.is_available():
            raise VloError("no CUDA device visible: the hot path cannot run (no fallback by design)")
        self.index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        c = VloConfig()
        c.hidden_size, c.num_layers = cfg.hidden_size, cfg.num_hidden_layers
        c.num_heads, c.num_kv_heads, c.head_dim = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        c.intermediate_size, c.vocab_size, c.rms_norm_eps = cfg.intermediate_size, cfg.vocab_size, cfg.rms_norm_eps
        c.vit_hidden, c.vit_layers = cfg.vision_hidden_size, cfg.vision_num_hidden_layers
        c.vit_heads, c.vit_mlp = cfg.vision_num_attention_heads, cfg.vision_intermediate_size
        c.image_size, c.patch_size, c.vit_ln_eps = cfg.frame_resolution, cfg.vision_patch_size, cfg.vision_layer_norm_eps
        c.frame_token_cls = 1 if cfg.frame_token_cls else 0
        c.pool_h, c.pool_w = (cfg.frame_token_pooled or [0, 0])
        c.max_streams, c.max_kv_tokens = max_streams, max_kv_tokens
        c.max_step_tokens, c.max_vit_batch = max_step_tokens, max_vit_batch
        self.max_streams, self.max_kv_tokens = max_streams, max_kv_tokens
        self.max_step_tokens, self.max_vit_batch = max_step_tokens, max_vit_batch
        self._cfg_struct = c
        self._h = C.c_void_p()
        self._lock = threading.Lock()
        self._weights: Dict[str, torch.Tensor] = {}
        with torch.cuda.device(self.index):
            check(self.lib.vlo_engine_create_pooled(C.byref(c), int(kv_pool_tokens or 0), self.index, C.byref(self._h)),
                  "vlo_engine_create_pooled")
            self._fp8_act = bool(fp8_activations)
            if self._fp8_act:
                check(self.lib.vlo_set_fp8_activations(self._h, 1), "vlo_set_fp8_activations")
            if quantized_prefill:
                check(self.lib.vlo_set_quantized_prefill(self._h, 1), "vlo_set_quantized_prefill")
        # device scratch for results (decisions, last logits): one row per sequence, or per segment of a segmented step
        # and the sampled ids right behind the decisions, so that one copy brings both back
        rows = max(max_streams, max_step_tokens)
        self._res_dev = torch.zeros(rows * (DECISION_DTYPE_FIELDS + 1), dtype=torch.int32, device=self.device)
        self._res_host = torch.zeros(rows * (DECISION_DTYPE_FIELDS + 1), dtype=torch.int32).pin_memory()
        self._dec_dev = self._res_dev[:rows * DECISION_DTYPE_FIELDS].view(rows, DECISION_DTYPE_FIELDS)
        self._dec_host = self._res_host[:rows * DECISION_DTYPE_FIELDS].view(rows, DECISION_DTYPE_FIELDS)
        self._ids_dev = self._res_dev[rows * DECISION_DTYPE_FIELDS:]
        self._sampled: Optional[List[bool]] = None   # rows of the last step that were sampled (None: no sampling)
        self._logits = torch.zeros(rows, cfg.vocab_size, dtype=torch.bfloat16, device=self.device)
        # pinned image buffers a swap copy may still write or read: kept alive until their event has completed, so the
        # caching host allocator cannot hand them to someone else under a copy
        self._swap_inflight: List[tuple] = []
        self._taps: Dict[tuple, tuple] = {}             # (W, H) -> letterbox tap tables on the device (letterbox)
        self._frame_staging: List[tuple] = []          # (pinned buffer, event after the copy out of it) (letterbox)

    # ------------------------------------------------------------------ life cycle
    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self.lib.vlo_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def load_weights(self, weights: Dict[str, torch.Tensor]):
        """Register tensors already in the engine layout (weights.pack_*_for_engine)."""
        for name, t in weights.items():
            if t.device != self.device:
                t = t.to(self.device)
            t = t.contiguous()
            self._weights[name] = t  # keep the storage alive
            check(self.lib.vlo_load_tensor(self._h, name.encode(), _ptr(t), t.numel() * t.element_size()),
                  f"vlo_load_tensor({name})")
        check(self.lib.vlo_finalize_weights(self._h), "vlo_finalize_weights")

    @property
    def weights(self) -> Dict[str, torch.Tensor]:
        return self._weights

    @property
    def fp8_weights(self) -> bool:
        """True when the decoder layer matrices were loaded as e4m3 codes + row scales (weights.quantize_fp8_rows)."""
        return "L0.qkv.f8" in self._weights

    @property
    def int4_weights(self) -> bool:
        """True when the decoder layer matrices were loaded as int4 codes + bf16 group scales
        (weights.quantize_int4_groups)."""
        return "L0.qkv.i4" in self._weights

    @property
    def quantized_vocab(self) -> bool:
        """True when embed and lm_head were loaded in the layer matrices' quantized form (e4m3 or int4, quantize_vocab)
        rather than in bf16."""
        return "embed.f8" in self._weights or "embed.i4" in self._weights

    @property
    def max_prefill_tokens(self) -> int:
        """rows of one vlo_prefill (8 x max_step_tokens) once bf16 layer weights are loaded, or quantized ones on an
        Engine(quantized_prefill=True); 0 before, and on quantized engines without quantized_prefill"""
        return int(self.lib.vlo_max_prefill_tokens(self._h))

    @property
    def prefills(self) -> bool:
        """True when one stream's input longer than max_step_tokens runs as a prefill (vlo_prefill: tensor-core GEMMs
        over up to max_prefill_tokens rows per call, with the bits of max_step_tokens steps on the same engine): bf16
        engines, and quantized ones built with quantized_prefill.  The other quantized engines chunk such inputs into
        steps instead."""
        return self.max_prefill_tokens > 0

    @property
    def max_pass_tokens(self) -> int:
        """the most rows one single-stream `step` computes in one pass, so that `last_step_logits` /
        `last_step_hidden` cover all of them: max_prefill_tokens on a prefilling engine, else max_step_tokens"""
        return self.max_prefill_tokens if self.prefills else self.max_step_tokens

    @property
    def fp8_activations(self) -> bool:
        """True when the layer GEMMs take e4m3 activations with per-token scales (W8A8; Engine(fp8_activations=True))."""
        return self._fp8_act

    def device_bytes(self) -> int:
        return int(self.lib.vlo_engine_device_bytes(self._h))

    def kv_pool_info(self) -> Dict[str, int]:
        """{"page_tokens", "total_pages", "free_pages"} of the shared KV page pool."""
        pt, total, free = C.c_int(0), C.c_int64(0), C.c_int64(0)
        check(self.lib.vlo_kv_pool_info(self._h, C.byref(pt), C.byref(total), C.byref(free)), "vlo_kv_pool_info")
        return {"page_tokens": pt.value, "total_pages": total.value, "free_pages": free.value}

    # ------------------------------------------------------------------ streams
    def stream_open(self) -> int:
        sid = C.c_int(-1)
        check(self.lib.vlo_stream_open(self._h, C.byref(sid)), "vlo_stream_open")
        return sid.value

    def stream_reset(self, sid: int):
        check(self.lib.vlo_stream_reset(self._h, sid), "vlo_stream_reset")

    def stream_close(self, sid: int):
        check(self.lib.vlo_stream_close(self._h, sid), "vlo_stream_close")

    def kv_len(self, sid: int) -> int:
        n = C.c_int(0)
        check(self.lib.vlo_kv_len(self._h, sid, C.byref(n)), "vlo_kv_len")
        return n.value

    def kv_truncate(self, sid: int, new_len: int):
        check(self.lib.vlo_kv_truncate(self._h, sid, new_len), "vlo_kv_truncate")

    def kv_copy_prefix(self, src_sid: int, dst_sid: int, n_tokens: int):
        check(self.lib.vlo_kv_copy_prefix(self._h, src_sid, dst_sid, n_tokens, self._stream()), "vlo_kv_copy_prefix")

    def kv_evict(self, sid: int, first: int, n: int):
        """Drop cache positions [first, first + n) of stream `sid` (whole, full pages) and move the later ones down by
        n: their keys are re-rotated on the device by -n positions (vlo_kv_evict, current CUDA stream)."""
        cos, sin = W.rope_rotation(self.cfg, n)
        fp = C.POINTER(C.c_float)
        check(self.lib.vlo_kv_evict(self._h, sid, first, n, C.cast(cos.data_ptr(), fp), C.cast(sin.data_ptr(), fp),
                                    self._stream()), "vlo_kv_evict")

    def kv_make_room(self, sid: int, need: int, window: int, keep_tokens: int) -> int:
        """Before stream `sid` appends `need` tokens under a context window: evict what `evict_span` says (the sink of
        keep_tokens positions stays).  Returns the number of positions dropped (0: none); they start at
        sink_tokens(keep_tokens, page)."""
        first, n = evict_span(self.kv_len(sid), need, window, keep_tokens, self.kv_pool_info()["page_tokens"])
        if n:
            self.kv_evict(sid, first, n)
        return n

    def kv_compact(self, sid: int, spans: Sequence[tuple[int, int]]):
        """Keep only the cache positions of stream `sid` in `spans` [(first, n), ...] (sorted, non-overlapping): span i
        moves down to the sum of the earlier spans' lengths and its keys are re-rotated on the device by that shift
        (vlo_kv_compact, current CUDA stream: the one the steps run on)."""
        first = torch.tensor([f for f, _ in spans], dtype=torch.int32)
        lens = torch.tensor([n for _, n in spans], dtype=torch.int32)
        rot, q = [], 0
        for f, n in spans:
            rot.extend(W.rope_rotation(self.cfg, f - q))
            q += n
        rot = torch.cat(rot) if rot else torch.zeros(1)
        i32, fp = C.POINTER(C.c_int32), C.POINTER(C.c_float)
        check(self.lib.vlo_kv_compact(self._h, sid, len(spans), C.cast(first.data_ptr(), i32),
                                      C.cast(lens.data_ptr(), i32), C.cast(rot.data_ptr(), fp), self._stream()),
              "vlo_kv_compact")

    def kv_retain(self, sid: int, row_ids: Sequence[int], need: int, window: int, keep_tokens: int,
                  interval_id: Optional[int], frame_num_tokens: int) -> List[tuple[int, int]]:
        """Before stream `sid` appends `need` tokens under a context window that keeps the conversation: compact the
        cache to what `retain_spans` keeps of its history row_ids.  Returns the spans kept ([]: nothing dropped)."""
        spans = retain_spans(row_ids, need, window, keep_tokens, interval_id, frame_num_tokens)
        if spans:
            self.kv_compact(sid, spans)
        return spans

    def kv_fill_synthetic(self, sid: int, n_tokens: int, seed: int = 0):
        check(self.lib.vlo_kv_fill_synthetic(self._h, sid, n_tokens, seed, self._stream()), "vlo_kv_fill_synthetic")

    def kv_read(self, sid: int, layer: int, is_v: bool) -> torch.Tensor:
        n = self.kv_len(sid)
        out = torch.empty(self.cfg.num_key_value_heads, n, self.cfg.head_dim, dtype=torch.bfloat16, device=self.device)
        check(self.lib.vlo_kv_read(self._h, sid, layer, int(is_v), _ptr(out), self._stream()), "vlo_kv_read")
        return out

    def kv_write(self, sid: int, layer: int, is_v: bool, rows: torch.Tensor):
        rows = rows.to(device=self.device, dtype=torch.bfloat16).contiguous()
        assert rows.shape[0] == self.cfg.num_key_value_heads and rows.shape[2] == self.cfg.head_dim
        check(self.lib.vlo_kv_write(self._h, sid, layer, int(is_v), _ptr(rows), rows.shape[1], self._stream()), "vlo_kv_write")

    # ------------------------------------------------------------------ host images (swap)
    def kv_layout(self) -> tuple:
        """(num_layers, num_kv_heads, head_dim, page_tokens): what the layout of a KvImage depends on"""
        c = self.cfg
        return (c.num_hidden_layers, c.num_key_value_heads, c.head_dim, self.kv_pool_info()["page_tokens"])

    def kv_image_bytes(self, n_tokens: int) -> int:
        return int(self.lib.vlo_kv_image_bytes(self._h, int(n_tokens)))

    def _swap_prune(self):
        self._swap_inflight = [(d, e) for d, e in self._swap_inflight if not e.query()]

    def _swap_hold(self, data: torch.Tensor, ev: torch.cuda.Event):
        self._swap_prune()
        self._swap_inflight.append((data, ev))

    def kv_swap_out(self, sid: int) -> KvImage:
        """Copy stream `sid`'s cache to pinned host memory on the current CUDA stream and empty the stream (its pages go
        back to the pool, its slot stays open).  Nothing is synchronised: the image's event marks the copy's end, and
        the engine orders every later use of the released pages behind it."""
        n = self.kv_len(sid)
        nbytes = self.kv_image_bytes(n)
        self._swap_prune()   # buffers whose copies have ended may be reused by this allocation
        data = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        check(self.lib.vlo_kv_swap_out(self._h, sid, _ptr(data) if nbytes else None, nbytes, self._stream()),
              "vlo_kv_swap_out")
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self._swap_hold(data, ev)
        return KvImage(data, n, self.kv_layout(), ev)

    def kv_swap_in(self, sid: int, image: KvImage):
        """Fill the empty stream `sid` from `image` (current CUDA stream, ordered after the image's own copy).  Fails,
        changing nothing, on a short pool ("KV page pool exhausted"), a non-empty stream, an image of another layout or
        of the wrong size."""
        if tuple(image.layout) != self.kv_layout():
            raise VloError(f"kv_swap_in: the image's layout {tuple(image.layout)} (layers, kv heads, head_dim, page "
                           f"tokens) differs from this engine's {self.kv_layout()}")
        want = self.kv_image_bytes(image.n_tokens)
        data = image.data
        if data.dtype != torch.uint8 or data.device.type != "cpu" or data.numel() != want:
            raise VloError(f"kv_swap_in: an image of {image.n_tokens} tokens is {want} bytes of host uint8, got "
                           f"{data.numel() * data.element_size()} bytes ({data.dtype}, {data.device})")
        if not data.is_pinned():
            data = image.data = data.pin_memory()
        main = torch.cuda.current_stream(self.device)
        if image.event is not None:
            main.wait_event(image.event)
        check(self.lib.vlo_kv_swap_in(self._h, sid, _ptr(data) if want else None, image.n_tokens, self._stream()),
              "vlo_kv_swap_in")
        ev = torch.cuda.Event()
        ev.record(main)
        self._swap_hold(data, ev)

    # ------------------------------------------------------------------ hot path
    def vit_encode(self, frames_u8: torch.Tensor, *, return_vit_tokens: bool = False, connector: bool = True):
        """uint8 [B,3,S,S] -> bf16 [B*frame_num_tokens, hidden] (visual_embed, models/modeling_live.py:21-27)."""
        if frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4:
            raise VloError("vit_encode expects uint8 frames [B,3,S,S]")
        # pinned host frames (a live feed) are copied asynchronously on the caller's stream
        frames_u8 = frames_u8.to(self.device, non_blocking=frames_u8.device.type == "cpu" and frames_u8.is_pinned()).contiguous()
        B = frames_u8.shape[0]
        S = self.cfg.frame_resolution
        if tuple(frames_u8.shape[1:]) != (3, S, S):
            raise VloError(f"frames must be [B,3,{S},{S}], got {tuple(frames_u8.shape)}")
        nt = self.cfg.frame_num_tokens
        outs, toks = [], []
        for b0 in range(0, B, self.max_vit_batch):
            fb = frames_u8[b0:b0 + self.max_vit_batch]
            n = fb.shape[0]
            out = torch.empty(n * nt, self.cfg.hidden_size, dtype=torch.bfloat16, device=self.device) if connector else None
            vt = torch.empty(n, nt, self.cfg.vision_hidden_size, dtype=torch.float32, device=self.device) if return_vit_tokens else None
            check(self.lib.vlo_vit_encode(self._h, _ptr(fb), n, _ptr(out), _ptr(vt), self._stream()), "vlo_vit_encode")
            outs.append(out)
            toks.append(vt)
        out = torch.cat(outs, 0) if connector else None
        if return_vit_tokens:
            return out, torch.cat(toks, 0)
        return out

    def letterbox(self, frames: Sequence, bgr: bool = False, pixel_format: Optional[str] = None) -> torch.Tensor:
        """Native frames -> uint8 [B, 3, R, R] RGB canvases (R = frame_resolution), what vit_encode takes: each frame is
        scaled into the square with the integer INTER_CUBIC of video_ingest.cubic_taps and centred on black bars
        (video_ingest.letterbox_geometry), on the device (vlo_letterbox_planes, current CUDA stream).  frames: HWC uint8
        tensors with 3 channels (RGB, or BGR with bgr=True), each of its own size up to 8192 x 8192, on the CPU or this
        device; or, with pixel_format "nv12", "yuv420p" or "yuyv422" (ffmpeg's names), YUV frames as
        video_ingest.frame_layout describes them, converted to RGB per source pixel with OpenCV's BT.601 integer
        arithmetic, so the canvas is exactly that of cv2.cvtColor's RGB frame.  Device planes are read in place.
        CPU frames are staged through pinned buffers and copied asynchronously; a buffer is reused only once the copy
        out of it has completed.  Every frame is checked before any device work: VloError on a frame of another dtype,
        shape, device, size or format."""
        from .video_ingest import frame_layout
        frames = list(frames)
        if not frames:
            raise VloError("letterbox: no frames")
        try:
            layouts = [frame_layout(f, pixel_format, bgr) for f in frames]
        except ValueError as e:
            raise VloError(f"letterbox: {e}") from None
        for _, _, _, parts, _ in layouts:
            for t in parts:
                if t.device.type == "cuda" and t.device != self.device:
                    raise VloError(f"letterbox: a frame on {t.device}, the engine runs on {self.device}")
        R = self.cfg.frame_resolution
        out = torch.empty(len(frames), 3, R, R, dtype=torch.uint8, device=self.device)
        descs = (_lib.VloFramePlanes * len(frames))()
        held = []   # device frames and tap tables: alive until every launch is enqueued (stream-ordered reuse after it)
        for d, (W, H, fmt, parts, planes) in zip(descs, layouts):
            taps, sw = self._letterbox_taps(W, H)
            # one tensor: its contiguous device copy; planes: read in place (device only, frame_layout)
            parts = [self._frame_on_device(parts[0])] if len(parts) == 1 else parts
            held += [*parts, taps]
            for q, (k, offset, pitch) in enumerate(planes):
                d.d_planes[q], d.pitch[q] = parts[k].data_ptr() + offset, pitch
            d.d_taps, d.format, d.width, d.height, d.x_taps, d.y_taps = taps.data_ptr(), fmt, W, H, 0, sw
        size = C.sizeof(_lib.VloFramePlanes)
        for b0 in range(0, len(frames), self.max_vit_batch):
            n = min(self.max_vit_batch, len(frames) - b0)
            check(self.lib.vlo_letterbox_planes(self._h, C.cast(C.addressof(descs) + b0 * size, C.POINTER(_lib.VloFramePlanes)),
                                                n, _ptr(out[b0:]), self._stream()), "vlo_letterbox_planes")
        return out

    def _letterbox_taps(self, W: int, H: int):
        """(device int32 tap tables of a W x H frame, rows of the horizontal table), built once per size"""
        hit = self._taps.get((W, H))
        if hit is None:
            from .video_ingest import letterbox_geometry, letterbox_taps
            sw = letterbox_geometry(W, H, self.cfg.frame_resolution)[0]
            taps = torch.from_numpy(letterbox_taps(W, H, self.cfg.frame_resolution)).to(self.device)
            # once per frame size: the upload has landed before any stream reads the table; tables are never freed, so no
            # stream can read one after its memory is reused (a table is at most 768 rows of 32 bytes)
            torch.cuda.current_stream(self.device).synchronize()
            hit = self._taps[(W, H)] = (taps, sw)
        return hit

    def _frame_on_device(self, f: torch.Tensor) -> torch.Tensor:
        if f.device.type == "cuda":
            return f.contiguous()
        n = f.numel()
        pool = self._frame_staging
        # Idle buffers (their copy has completed) more than 4x this frame go, and so do the largest idle ones beyond
        # max_vit_batch: after a burst of large frames the pool shrinks to the frames now pushed.  Buffers under a copy
        # stay until their event has completed.
        idle = [i for i, (b, ev) in enumerate(pool) if ev.query()]
        drop = {i for i in idle if pool[i][0].numel() > 4 * n}
        keep = sorted((i for i in idle if i not in drop), key=lambda i: pool[i][0].numel())
        drop |= set(keep[self.max_vit_batch:])
        fit = next((i for i in keep[:self.max_vit_batch] if pool[i][0].numel() >= n), None)   # the smallest that fits
        buf = pool[fit][0] if fit is not None else torch.empty(n, dtype=torch.uint8, pin_memory=True)
        self._frame_staging = pool = [e for i, e in enumerate(pool) if i not in drop and i != fit]
        buf[:n].copy_(f.reshape(-1))
        dev = torch.empty(n, dtype=torch.uint8, device=self.device)
        dev.copy_(buf[:n], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        pool.append((buf, ev))
        return dev.view(f.shape)

    def connector(self, tokens: torch.Tensor) -> torch.Tensor:
        tokens = tokens.to(device=self.device, dtype=torch.bfloat16).contiguous().view(-1, self.cfg.vision_hidden_size)
        out = torch.empty(tokens.shape[0], self.cfg.hidden_size, dtype=torch.bfloat16, device=self.device)
        check(self.lib.vlo_connector(self._h, _ptr(tokens), tokens.shape[0], _ptr(out), self._stream()), "vlo_connector")
        return out

    def embed_tokens(self, ids: torch.Tensor) -> torch.Tensor:
        ids = ids.to(device=self.device, dtype=torch.int64).contiguous().view(-1)
        out = torch.empty(ids.numel(), self.cfg.hidden_size, dtype=torch.bfloat16, device=self.device)
        if ids.numel():
            check(self.lib.vlo_embed_tokens(self._h, _ptr(ids), ids.numel(), _ptr(out), self._stream()), "vlo_embed_tokens")
        return out

    def step(self, stream_ids: Sequence[int], q_lens: Sequence[int], embeds: torch.Tensor, *,
             row_ids: Optional[torch.Tensor] = None, interval_id: Optional[int] = None,
             want_logits: bool = True, segments: Optional[Sequence[Sequence[int]]] = None,
             sample: Optional[Sequence[Optional[SampleRow]]] = None):
        """KV-append forward of a ragged batch.  `row_ids` (int64 [sum q_lens], optional): id >= 0 -> the row is the
        embedding of that token (gathered on the device), id < 0 -> the row of `embeds` is used as is.  Returns (logits [n_seqs, V] bf16 view or None, decisions
        device tensor int32 [n_seqs, 8]).  Nothing is synchronised; call `read_decisions` for host values.

        `segments` (optional): per sequence, the lengths of the consecutive segments its q_len rows are made of (they
        must add up to q_lens[i]).  Then there is one logits row and one decision per segment, in order, read at the
        segment's last row ([n_segments, V] / [n_segments, 8]), and every segment computes the bits the same rows get
        from a step of their own (vlo_step_segments).  A segmented step longer than max_step_tokens is an error.

        `sample` (optional): one SampleRow or None per decision row.  The step then keeps its logits and enqueues
        vlo_sample over them; `read_decisions` returns the drawn ids as `Decision.sampled_id` (None for rows given
        None).  Without it the step runs exactly as before."""
        self._sampled = None
        if sample is None:
            return self._step(stream_ids, q_lens, embeds, row_ids, interval_id, want_logits, segments)
        logits, dec = self._step(stream_ids, q_lens, embeds, row_ids, interval_id, True, segments)
        self._sample(logits, sample)
        return logits, dec

    def _sample(self, logits: torch.Tensor, sample: Sequence[Optional[SampleRow]]):
        if len(sample) != logits.shape[0]:
            raise VloError(f"step: sample needs one entry per decision row ({logits.shape[0]}), got {len(sample)}")
        m = max((i + 1 for i, r in enumerate(sample) if r is not None), default=0)
        if m:
            rows = (VloSampleRow * m)()
            ids: List[int] = []
            at: Dict[int, int] = {}     # id(penalty list) -> its offset in `ids`
            for c, r in zip(rows, sample[:m]):
                if r is None:           # temperature 0: the kernel skips the row
                    continue
                c.seed, c.position, c.temperature = r.seed, r.position, r.temperature
                c.top_k, c.top_p, c.repetition_penalty = r.top_k, r.top_p, r.repetition_penalty
                if r.repetition_penalty != 1.0:
                    n_pen = len(r.penalty_ids) if r.n_penalty is None else r.n_penalty
                    if not 0 <= n_pen <= len(r.penalty_ids):
                        raise VloError(f"step: n_penalty {n_pen} outside the row's {len(r.penalty_ids)} penalty ids")
                    if id(r.penalty_ids) not in at:
                        at[id(r.penalty_ids)] = len(ids)
                        ids.extend(r.penalty_ids)
                    c.penalty_offset, c.penalty_count = at[id(r.penalty_ids)], n_pen
            pen = torch.tensor(ids, dtype=torch.int32) if ids else None
            check(self.lib.vlo_sample(self._h, _ptr(logits), m, rows, _ptr(pen), len(ids), _ptr(self._ids_dev),
                                      self._stream()), "vlo_sample")
        self._sampled = [r is not None for r in sample]

    def _step(self, stream_ids, q_lens, embeds, row_ids, interval_id, want_logits, segments):
        n = len(stream_ids)
        T = int(sum(q_lens))
        embeds = embeds.contiguous()
        if segments is not None:
            return self._step_segments(stream_ids, q_lens, segments, embeds, row_ids, interval_id, want_logits)
        if T > self.max_step_tokens:
            if n == 1 and self.prefills:
                return self._prefill(stream_ids[0], T, embeds, row_ids, interval_id, want_logits)
            return self._step_chunked(stream_ids, q_lens, embeds, row_ids, interval_id, want_logits)
        iid, pid = self._step_inputs(T, embeds, row_ids, interval_id)
        sid = (C.c_int32 * n)(*stream_ids)
        ql = (C.c_int32 * n)(*q_lens)
        logits = self._logits[:n] if want_logits else None
        check(self.lib.vlo_step_ids(self._h, n, sid, ql, _ptr(pid), _ptr(embeds), _ptr(logits), _ptr(self._dec_dev), iid,
                                    self._stream()), "vlo_step")
        return logits, self._dec_dev[:n]

    def _step_inputs(self, T, embeds, row_ids, interval_id):
        """(interval id, device row ids or None) of a step over T packed rows, after checking the inputs"""
        if embeds.dtype != torch.bfloat16 or embeds.device != self.device or embeds.numel() != T * self.cfg.hidden_size:
            raise VloError(f"step: embeds must be bf16 [{T},{self.cfg.hidden_size}] on {self.device}")
        iid = self.cfg.frame_token_interval_id if interval_id is None else interval_id
        if iid is None:
            iid = -1
        pid = None
        if row_ids is not None:
            pid = row_ids.to(device=self.device, dtype=torch.int64).contiguous().view(-1)
            if pid.numel() != T:
                raise VloError(f"step: row_ids must have one entry per packed row ({T}), got {pid.numel()}")
        return iid, pid

    def _step_segments(self, stream_ids, q_lens, segments, embeds, row_ids, interval_id, want_logits):
        n, T = len(stream_ids), int(sum(q_lens))
        if len(segments) != n or any(sum(s) != q for s, q in zip(segments, q_lens)):
            raise VloError("step: segments must give each sequence segment lengths that add up to its q_len")
        if T > self.max_step_tokens:
            raise VloError(f"step: a segmented step of {T} tokens exceeds max_step_tokens ({self.max_step_tokens}); "
                           "segmented steps are not chunked")
        iid, pid = self._step_inputs(T, embeds, row_ids, interval_id)
        lens = [int(x) for s in segments for x in s]
        n_rows = len(lens)
        sid = (C.c_int32 * n)(*stream_ids)
        counts = (C.c_int32 * n)(*[len(s) for s in segments])
        sl = (C.c_int32 * n_rows)(*lens)
        logits = self._logits[:n_rows] if want_logits else None
        check(self.lib.vlo_step_segments(self._h, n, sid, counts, sl, _ptr(pid), _ptr(embeds), _ptr(logits),
                                         _ptr(self._dec_dev), iid, self._stream()), "vlo_step_segments")
        return logits, self._dec_dev[:n_rows]

    def _prefill(self, sid, T, embeds, row_ids, interval_id, want_logits):
        """One stream's input longer than max_step_tokens on a prefilling engine: vlo_prefill calls of up to max_prefill_tokens
        rows, each giving the bits of the same rows fed as max_step_tokens steps.  The logits / decision come from the
        last call; if a later call fails (e.g. on an exhausted KV page pool), the earlier ones are taken back, so the
        call changes nothing and the caller can retry it whole."""
        iid, pid = self._step_inputs(T, embeds, row_ids, interval_id)
        cap = self.max_prefill_tokens
        kv0 = self.kv_len(sid)
        logits = self._logits[:1] if want_logits else None
        try:
            for lo in range(0, T, cap):
                n = min(cap, T - lo)
                last = lo + n == T
                check(self.lib.vlo_prefill(self._h, sid, n, _ptr(None if pid is None else pid[lo:lo + n]),
                                           _ptr(embeds[lo:lo + n]), _ptr(logits if last else None),
                                           _ptr(self._dec_dev[:1]), iid, self._stream()), "vlo_prefill")
        except VloError:
            self.kv_truncate(sid, kv0)
            raise
        return logits, self._dec_dev[:1]

    def _step_chunked(self, stream_ids, q_lens, embeds, row_ids, interval_id, want_logits):
        """Ragged multi-stream inputs longer than max_step_tokens, and long inputs on engines that do not prefill (quantized
        layer matrices without quantized_prefill): feed the KV-append forward in pieces — chunked streaming is exactly one causal pass (SURVEY.md
        Appendix C.1).  Each sequence's logits / decision come from the sub-step that holds its last piece."""
        n, cap, H = len(stream_ids), self.max_step_tokens, self.cfg.hidden_size
        if row_ids is not None:  # materialise the gathered token rows once; the sub-steps then see plain embeddings
            pid = row_ids.to(self.device).view(-1)
            rows = self.embed_tokens(pid.clamp(min=0))
            embeds = torch.where((pid >= 0)[:, None], rows, embeds)
        logits_out = torch.empty(n, self.cfg.vocab_size, dtype=torch.bfloat16, device=self.device) if want_logits else None
        dec_out = torch.empty(n, DECISION_DTYPE_FIELDS, dtype=torch.int32, device=self.device)
        off, done = 0, [0] * n
        starts = [int(sum(q_lens[:i])) for i in range(n)]
        kv0 = [self.kv_len(s) for s in stream_ids]
        try:
            while any(done[i] < q_lens[i] for i in range(n)):
                sub_ids, sub_lens, sub_rows, room = [], [], [], cap
                for i in range(n):
                    left = q_lens[i] - done[i]
                    if left <= 0 or room <= 0:
                        continue
                    take = min(left, room)
                    sub_ids.append(i)
                    sub_lens.append(take)
                    sub_rows.append(embeds[starts[i] + done[i]: starts[i] + done[i] + take])
                    room -= take
                lg, dc = self.step([stream_ids[i] for i in sub_ids], sub_lens, torch.cat(sub_rows, 0),
                                   interval_id=interval_id, want_logits=want_logits)
                for j, i in enumerate(sub_ids):
                    done[i] += sub_lens[j]
                    if done[i] == q_lens[i]:
                        dec_out[i].copy_(dc[j])
                        if want_logits:
                            logits_out[i].copy_(lg[j])
        except VloError:
            # a later piece failed (e.g. on an exhausted KV page pool): undo the earlier pieces, so the call changes
            # no stream and the caller can retry it whole
            for s, k in zip(stream_ids, kv0):
                self.kv_truncate(s, k)
            raise
        self._dec_dev[:n].copy_(dec_out)
        if want_logits:
            self._logits[:n].copy_(logits_out)
        return (self._logits[:n] if want_logits else None), self._dec_dev[:n]

    def read_decisions(self, n: int) -> List[Decision]:
        """One small D2H copy + sync: the only host<->device sync of a frame step.  After a sampling step the same copy
        also carries the sampled ids, which sit behind the decision rows."""
        f32 = self._dec_host.view(torch.float32)
        if self._sampled is None:
            self._dec_host[:n].copy_(self._dec_dev[:n], non_blocking=True)
            torch.cuda.current_stream(self.device).synchronize()
            return [Decision(self._dec_host[i], f32[i]) for i in range(n)]
        end = self._dec_dev.numel() + n
        self._res_host[:end].copy_(self._res_dev[:end], non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        ids = self._res_host[self._dec_dev.numel():end].tolist()
        sampled = self._sampled
        return [Decision(self._dec_host[i], f32[i], ids[i] if i < len(sampled) and sampled[i] else None)
                for i in range(n)]

    def last_step_logits(self, n_tokens: int) -> torch.Tensor:
        out = torch.empty(n_tokens, self.cfg.vocab_size, dtype=torch.bfloat16, device=self.device)
        check(self.lib.vlo_last_step_logits(self._h, _ptr(out), self._stream()), "vlo_last_step_logits")
        return out

    def last_step_hidden(self, n_tokens: int) -> torch.Tensor:
        out = torch.empty(n_tokens, self.cfg.hidden_size, dtype=torch.bfloat16, device=self.device)
        check(self.lib.vlo_last_step_hidden(self._h, _ptr(out), self._stream()), "vlo_last_step_hidden")
        return out

    def launch_count(self) -> int:
        return int(self.lib.vlo_launch_count())
