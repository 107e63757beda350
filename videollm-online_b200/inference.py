"""Streaming session state machine — the engine-backed `LiveInfer`.

Same public surface and protocol as the reference's demo/inference.py:12-124 (`load_video`,
`input_video_stream`, `input_query_stream`, `__call__`, `reset`, `frame_token_interval_threshold`) so
demo/cli.py and demo/app.py can drive it unchanged.  Differences, all behind the same results:
  * the device is a parameter, not a hard-coded 'cuda';
  * the speak/silent decision and the greedy argmax are computed on the device; one 32-byte read-back
    per frame / generated token replaces the reference's two tensor-`if` syncs (demo/inference.py:77,80);
  * the steady-state frame step feeds [interval-token id | 10 frame embeddings] and lets the engine gather
    the token row, so no separate embedding launch or torch.cat is needed;
  * queued frames (a clip processed faster than real time, a seek, a stalled feed) go through one segmented step
    [prefix | F1 | interval | F2 | ...] with one decision per frame, the same bits as one step per frame; where a
    frame speaks or a query is due the stream is cut back to that frame and the rest is queued again.
"""
from __future__ import annotations

import collections
import itertools
import logging
import threading
from dataclasses import asdict, dataclass
from typing import Optional

import torch

from ._lib import VloError
from .config import LiveArguments, SamplingConfig, parse_args
from .engine import KvImage, check_context_window, check_context_window_turns, kept_rows, sink_tokens
from .modeling_live import LiveLlamaForCausalLM, StreamKV, build_model_and_tokenizer, fast_greedy_generate
from .speculative import SEP, NgramDrafter, generate_ids
from .video_ingest import FrameRing

logger = logging.getLogger("liveinfer")


@dataclass
class SessionState:
    """Everything `LiveInfer.__call__` depends on, as `suspend()` returns it: the KV cache as a host image and the
    session's host state, with the queued frame embeddings on the host.  Not the video: load it again after resuming.
    Survives torch.save / torch.load."""
    kv: KvImage
    last_ids: torch.Tensor
    video_time: float
    last_frame_idx: int
    query_queue: list            # [(video_time, query)]
    frame_embeds_queue: list     # [(video_time, bf16 [frame_num_tokens, hidden] on the host)]
    drafter_ids: Optional[list]  # the NgramDrafter's history (SEP for frame rows), None without one
    n_calls: int
    started: bool                # past_key_values was set: a step ran since the last reset
    sampling: Optional[SamplingConfig] = None   # LiveInfer.sampling (None: greedy responses)
    evicted_tokens: int = 0      # cache positions the session's context window dropped so far
    fed_ids: Optional[list] = None   # the id fed at every cache position (-1: frame row) when no NgramDrafter holds them
    fp8_weights: bool = False    # the cache was written by a model with FP8 layer weights (Engine.fp8_weights)
    fp8_activations: bool = False   # ... and with FP8 activations (Engine.fp8_activations)
    int4_weights: bool = False   # ... with int4 layer weights (Engine.int4_weights)
    quantized_vocab: bool = False   # ... with quantized token embeddings and lm_head (Engine.quantized_vocab)


torch.serialization.add_safe_globals([SessionState, SamplingConfig])


class LiveInfer:
    def __init__(self, args: LiveArguments = None, *, model: LiveLlamaForCausalLM = None, tokenizer=None,
                 device: str = None, stream: StreamKV = None) -> None:
        args = args or parse_args()
        if model is None:
            kw = asdict(args)
            kw["device"] = device or args.device
            model, tokenizer = build_model_and_tokenizer(is_training=False, set_vision_inside=True, **kw)
        self.model, self.tokenizer = model, tokenizer
        self.device = model.device
        cfg = model.config
        # visual
        self.hidden_size = cfg.hidden_size
        self.frame_fps = args.frame_fps
        self.frame_interval = 1 / self.frame_fps
        self.frame_resolution = cfg.frame_resolution
        self.frame_num_tokens = cfg.frame_num_tokens
        self.frame_v_placeholder = cfg.v_placeholder * self.frame_num_tokens
        self.frame_token_interval_id = cfg.frame_token_interval_id
        self.frame_placeholder_ids = torch.tensor(cfg.v_placeholder_id).repeat(cfg.frame_num_tokens).reshape(1, -1)
        # generation
        self.system_prompt = args.system_prompt
        self.inplace_output_ids = torch.zeros(1, 100, dtype=torch.long)  # host buffer: ids are decided on device, read back per token
        self.frame_token_interval_threshold = 0.725
        # response tokens: None = greedy (the reference's fast_greedy_generate); a SamplingConfig with do_sample draws
        # them on the device, reproducibly from its seed.  The speak / silent decision is not sampled.
        self.sampling: Optional[SamplingConfig] = SamplingConfig.from_args(args)
        self.eos_token_id = cfg.eos_token_id
        self.stream_end_id = cfg.stream_end_id
        tok = self.tokenizer
        self._start_ids = tok.apply_chat_template([{'role': 'system', 'content': self.system_prompt}], add_stream_prompt=True, return_tensors='pt')
        self._added_stream_prompt_ids = tok.apply_chat_template([{}], add_stream_prompt=True, return_tensors='pt')
        self._added_stream_generation_ids = tok.apply_chat_template([{}], add_stream_generation_prompt=True, return_tensors='pt')
        self._kv = stream if stream is not None else model.new_stream()
        # test seam: decision_hook(decision, call_index) -> decision lets a test script the model's choices
        # (random weights never emit the "]\\n" / EOS protocol ids); None in production.
        self.decision_hook = None
        # drafts for responses: prompt lookup over the session's ids (speculative.py), mirrored with the stream's KV.
        # A test may substitute its own (sync / extend / propose); None answers one token per step.  Either way the
        # response ids, the decisions the hook sees and the cache are those of one token per step.
        self.drafter = NgramDrafter()
        self._n_calls = 0
        # context window (tokens, None: off): the cache keeps the start prompt (the sink) and drops its oldest pages
        # after it, at fixed points only (before a frame step, before a response), so a session runs in bounded memory
        self._context_keep_turns = args.context_keep_turns
        self.context_window = args.context_window or None
        # encode-ahead: with a loaded clip the ViT + connector of the NEXT frame run on a side CUDA stream while the
        # decoder works on the current one (same per-frame arithmetic; a live stream delivers the next frame
        # during the current step anyway).  Set prefetch_next = False for strictly sequential behaviour.
        self.prefetch_next = True
        # frames encoded per encode-ahead call.  1 (default): the next frame only, through the ViT trunk GEMM whose CTAs
        # share the SMs with the decoder step.
        # With a loaded clip a larger depth sends the next `prefetch_depth` frames through ONE batched ViT pass (the
        # reference itself batches every frame between two input_video_stream calls, demo/inference.py:106); from 3 frames
        # on that pass uses the wide-tile tensor-bound GEMM configuration.
        self.prefetch_depth = 1
        self._side = torch.cuda.Stream(self.device)
        # demo/app.py drives input_video_stream and __call__ from separate Gradio callbacks (SURVEY 3.2): both touch the
        # engine's single set of ViT workspaces and the encode-ahead state, so their bodies are serialised.
        self._lock = threading.RLock()
        self._alloc_step_buffers(256)
        self._row_ids_cache = {}
        self._prefetched = {}       # frame_idx -> (embeds [frame_num_tokens, hidden], event)
        self._prefetch_event = None   # last event recorded on the side stream (it owns the engine's ViT workspaces)
        self._want_prefetch = None  # first frame index to encode ahead right after the next decoder step is enqueued
        self.reset()

    def _alloc_step_buffers(self, rows: int):
        self._packed = torch.zeros(rows, self.hidden_size, dtype=torch.bfloat16, device=self.device)
        self._row_ids_host = torch.zeros(rows, dtype=torch.int64).pin_memory()
        self._row_ids_dev = torch.zeros(rows, dtype=torch.int64, device=self.device)

    def _drop_prefetch(self):
        """Forget encoded-ahead frames; an encode-ahead still in flight owns the ViT workspaces: order behind it."""
        if getattr(self, "_prefetch_event", None) is not None:
            torch.cuda.current_stream(self.device).wait_event(self._prefetch_event)
        self._prefetched = {}
        self._prefetch_event = None
        self._want_prefetch = None

    # ------------------------------------------------------------------ context window
    @property
    def context_window(self) -> Optional[int]:
        return self._context_window

    @context_window.setter
    def context_window(self, window: Optional[int]):
        """None: off.  Else it must be <= max_kv_tokens and hold the sink pages, one eviction chunk and the largest
        frame step or response reserve; with context_keep_turns the prompt, the turn budget (window / 2), one eviction
        chunk and that reserve (ValueError otherwise)."""
        if window is not None:
            frame_step = 1 + self._added_stream_prompt_ids.numel() + self.frame_num_tokens
            reserve = self._added_stream_generation_ids.numel() + self.inplace_output_ids.size(1)
            eng = self.model.engine
            if self._context_keep_turns:
                check_context_window_turns(window, eng.max_kv_tokens, self._start_ids.numel(), max(frame_step, reserve))
            else:
                check_context_window(window, eng.max_kv_tokens, self._start_ids.numel(), max(frame_step, reserve),
                                     eng.kv_pool_info()["page_tokens"])
        self._context_window = window

    @property
    def context_keep_turns(self) -> bool:
        return self._context_keep_turns

    @context_keep_turns.setter
    def context_keep_turns(self, keep: bool):
        """With a context window: False (default) drops whole pages after the start prompt (engine.evict_span); True
        drops the oldest frames token by token and keeps the questions and answers (engine.retain_spans)."""
        old, self._context_keep_turns = self._context_keep_turns, bool(keep)
        try:
            self.context_window = self._context_window   # validated for the new mode
        except ValueError:
            self._context_keep_turns = old
            raise

    def _fed_ids(self) -> list:
        """The id fed at every cache position (-1: a frame row): the NgramDrafter's history when the session has one,
        else its own list; both are cut back here to the cache, which a take-back or a rejected draft may have cut."""
        n = self._kv.engine.kv_len(self._kv.stream_id)
        if isinstance(self.drafter, NgramDrafter):
            self.drafter.sync(n)
            return self.drafter.ids
        del self._fed[n:]
        return self._fed

    def _make_room(self, need: int):
        """Under a context window: evict before the stream appends `need` tokens (Engine.kv_make_room, the policy
        StreamScheduler uses as well), and drop the same positions from the drafter's history."""
        if self._context_window is None:
            return
        eng, sid = self._kv.engine, self._kv.stream_id
        if self._context_keep_turns:
            fed = self._fed_ids()
            spans = eng.kv_retain(sid, fed, need, self._context_window, self._start_ids.numel(),
                                  self.frame_token_interval_id, self.frame_num_tokens)
            if spans:
                self.evicted_tokens += len(fed) - sum(n for _, n in spans)
                if self.drafter is not None:
                    self.drafter.keep(spans)
                if not isinstance(self.drafter, NgramDrafter):
                    self._fed = kept_rows(fed, spans)
            return
        n = eng.kv_make_room(sid, need, self._context_window, self._start_ids.numel())
        if n:
            if self.drafter is not None:
                self.drafter.drop(sink_tokens(self._start_ids.numel(), eng.kv_pool_info()["page_tokens"]), n)
            self.evicted_tokens += n

    # ------------------------------------------------------------------ session control
    def reset(self):
        self.query_queue = collections.deque()
        self.frame_embeds_queue = collections.deque()
        self.video_time = 0
        self.last_frame_idx = -1
        self.video_tensor = None
        self.last_ids = torch.tensor([[]], dtype=torch.long)
        self.evicted_tokens = 0
        self._fed = []   # _fed_ids without an NgramDrafter
        self._kv.engine.stream_reset(self._kv.stream_id)
        if self.drafter is not None:
            self.drafter.sync(0)
        self.past_key_values = None
        self._drop_prefetch()

    def suspend(self) -> SessionState:
        """Move the session out of the engine: its KV cache to a pinned host image (its pages go back to the pool) and
        its queued frames to the host.  The session is then reset and its video dropped; `resume(state)` continues it
        exactly where it stopped, here or in another process whose model has the same config."""
        with self._lock:
            self._drop_prefetch()   # encoded-ahead frames are dropped as reset() drops them
            frames = [(t, f.to("cpu")) for t, f in self.frame_embeds_queue]   # before the cache copy: this one syncs
            fed = None if isinstance(self.drafter, NgramDrafter) else list(self._fed_ids())   # before the swap-out too
            state = SessionState(
                kv=self._kv.engine.kv_swap_out(self._kv.stream_id), last_ids=self.last_ids.clone(),
                video_time=self.video_time, last_frame_idx=self.last_frame_idx, query_queue=list(self.query_queue),
                frame_embeds_queue=frames,
                drafter_ids=list(self.drafter.ids) if isinstance(self.drafter, NgramDrafter) else None,
                n_calls=self._n_calls, started=self.past_key_values is not None, sampling=self.sampling,
                evicted_tokens=self.evicted_tokens, fp8_weights=self._kv.engine.fp8_weights,
                fp8_activations=self._kv.engine.fp8_activations, int4_weights=self._kv.engine.int4_weights,
                quantized_vocab=self._kv.engine.quantized_vocab, fed_ids=fed)
            self.reset()
            return state

    def resume(self, state: SessionState):
        """Continue a session `suspend()` returned: the cache is copied back into this session's (emptied) stream and
        every queue and counter `__call__` reads is restored.  The video is not part of the state: load it again
        (before or after resuming).  Raises VloError if the pool is short or the image belongs to another config; the
        session's stream is then empty and the rest of the session unchanged.  A state whose cache was written with the
        other weight form (bf16, FP8 or int4 layer weights: a different model), or with the other activation form (W8A8 or
        not), or with the other form of the vocabulary matrices (quantized or bf16: the cache holds rows computed from
        the text embeddings), is refused before anything changes.  States saved before the int4 form existed load as not
        int4, and states saved before quantized vocabulary matrices existed load as not quantized."""
        with self._lock:
            eng = self._kv.engine
            def weight_form(fp8, int4):
                return "FP8" if fp8 else "int4" if int4 else "bf16"
            theirs = weight_form(state.fp8_weights, state.int4_weights)
            ours = weight_form(eng.fp8_weights, eng.int4_weights)
            if theirs != ours:
                raise VloError(f"resume: the state's cache was written with {theirs} layer weights, this model has {ours} ones")
            if state.fp8_activations != eng.fp8_activations:
                form = {True: "FP8", False: "bf16"}
                raise VloError(f"resume: the state's cache was written with {form[state.fp8_activations]} layer "
                               f"activations, this model has {form[eng.fp8_activations]} ones")
            if state.quantized_vocab != eng.quantized_vocab:
                form = {True: "quantized", False: "bf16"}
                raise VloError(f"resume: the state's cache was written with {form[state.quantized_vocab]} vocabulary "
                               f"matrices, this model has {form[eng.quantized_vocab]} ones")
            self._drop_prefetch()
            eng.stream_reset(self._kv.stream_id)
            eng.kv_swap_in(self._kv.stream_id, state.kv)
            dev = self.device
            self.last_ids = state.last_ids.clone()
            self.video_time, self.last_frame_idx = state.video_time, state.last_frame_idx
            self.query_queue = collections.deque(state.query_queue)
            self.frame_embeds_queue = collections.deque((t, f.to(dev, torch.bfloat16)) for t, f in state.frame_embeds_queue)
            fed = state.drafter_ids if state.drafter_ids is not None else state.fed_ids
            if self.drafter is not None:
                self.drafter.sync(0)
                if fed is not None and isinstance(self.drafter, NgramDrafter):
                    self.drafter.extend(fed)
                else:
                    self.drafter.sync(state.kv.n_tokens)
            if not isinstance(self.drafter, NgramDrafter):
                self._fed = list(fed) if fed is not None else [SEP] * state.kv.n_tokens
            self._n_calls = state.n_calls
            self.sampling = state.sampling
            self.evicted_tokens = state.evicted_tokens
            self.past_key_values = self._kv if state.started else None

    def load_video(self, video_path_or_tensor, keep_on_host: bool = False):
        """Reference: read_video(...)[0].to('cuda') (demo/inference.py:111-115).  Accepts a uint8
        [T,3,H,W] tensor directly (synthetic clips) or a path decodable by torchvision/cv2.
        keep_on_host=True leaves the clip in pinned host memory (a live feed): every frame is then copied to the GPU
        asynchronously by the step that encodes it instead of the whole clip being resident."""
        if isinstance(video_path_or_tensor, torch.Tensor):
            vt = video_path_or_tensor
        else:
            vt = _read_video_tchw(video_path_or_tensor, fps=self.frame_fps, resolution=self.frame_resolution)
        with self._lock:
            # an encode-ahead of the previous clip must neither be consumed nor keep reading the old tensor
            self._drop_prefetch()
            if keep_on_host:
                self.video_tensor = vt if (vt.device.type == "cpu" and vt.is_pinned()) else vt.cpu().pin_memory()
            else:
                self.video_tensor = vt.to(self.device)
        self.num_video_frames = self.video_tensor.size(0)
        self.video_duration = self.video_tensor.size(0) / self.frame_fps
        logger.warning(f'{"tensor" if isinstance(video_path_or_tensor, torch.Tensor) else video_path_or_tensor} -> '
                       f'{tuple(self.video_tensor.shape)}, {self.frame_fps} FPS')

    def push_frames(self, frames, bgr: bool = False, pixel_format: Optional[str] = None):
        """Append live frames to the session's video at frame_fps: frame i of the session is the i-th frame pushed since
        the last reset (counted on from the last frame input_video_stream reached, after a resume), so a camera feeds
        input_video_stream(t) as a loaded clip does.  frames: HWC uint8 tensors at their native sizes (RGB, or BGR with
        bgr=True; CPU or CUDA), or with pixel_format "nv12", "yuv420p" or "yuyv422" the YUV frames of
        video_ingest.frame_layout (a decoder's device planes among them); they are copied, converted and letterboxed to
        frame_resolution on the encode-ahead stream (Engine.letterbox) and held until encoded (video_ingest.FrameRing).
        Bad frames raise VloError before anything is enqueued.  A session plays one source at a time: after load_video,
        reset() before pushing frames (ValueError otherwise); reset and load_video drop the pushed frames."""
        with self._lock:
            ring = self.video_tensor
            if ring is None:
                ring = self.video_tensor = FrameRing(self.model.engine, self._side, first=self.last_frame_idx + 1)
            elif not isinstance(ring, FrameRing):
                raise ValueError("push_frames: the session plays a loaded clip; reset() it before pushing frames")
            ring.push(frames, bgr=bgr, pixel_format=pixel_format)
            self.num_video_frames = ring.size(0)
            self.video_duration = ring.size(0) / self.frame_fps

    def input_query_stream(self, query, history=None, video_time=None):
        self.query_queue.append((self.video_time if video_time is None else video_time, query))
        if not self.past_key_values:
            return f'(NOTE: No video stream here. Please select or upload a video. Then the assistant will answer "{query} (at {self.video_time}s)" in the video stream)'
        return f'(NOTE: Received "{query}" (at {self.video_time}s). Please wait until previous frames have been processed)'

    def input_video_stream(self, video_time):
        with self._lock:
            self._input_video_stream(video_time)

    def _input_video_stream(self, video_time):
        frame_idx = int(video_time * self.frame_fps)
        if frame_idx > self.last_frame_idx and isinstance(self.video_tensor, FrameRing):
            self.video_tensor.check_pushed(frame_idx)   # a camera frame not delivered yet: nothing changes, retry later
        if frame_idx > self.last_frame_idx:
            ranger = range(self.last_frame_idx + 1, frame_idx + 1)
            main = torch.cuda.current_stream(self.device)
            embeds, r = [], ranger.start
            while r < ranger.stop:
                hit = self._prefetched.pop(r, None)
                if hit is not None:                     # encoded ahead on the side stream
                    pe, ev = hit
                    main.wait_event(ev)
                    pe.record_stream(main)
                    embeds.append(pe)
                    r += 1
                    continue
                r2 = r                                  # contiguous run of frames that were not encoded ahead
                while r2 < ranger.stop and r2 not in self._prefetched:
                    r2 += 1
                if self._prefetch_event is not None:    # a side-stream ViT may still own the engine's ViT workspaces
                    main.wait_event(self._prefetch_event)
                embeds.extend(self.model.visual_embed(self.video_tensor[r:r2]).split(self.frame_num_tokens))
                r = r2
            for k in [k for k in self._prefetched if k <= frame_idx]:   # skipped-over frames
                del self._prefetched[k]
            self.frame_embeds_queue.extend([(r / self.frame_fps, e) for r, e in zip(ranger, embeds)])
            nxt = frame_idx + 1
            self._want_prefetch = nxt if (self.prefetch_next and self.video_tensor is not None and nxt not in self._prefetched
                                          and nxt < self.video_tensor.size(0)) else None
        self.last_frame_idx = frame_idx
        self.video_time = video_time

    # ------------------------------------------------------------------ decoder steps
    def _forward(self, ids: torch.Tensor, frame_embeds: torch.Tensor = None):
        """One KV-append step over [embed(ids) ; frame_embeds]; returns the device decision (host copy)."""
        with self._lock:
            return self._forward_locked(ids, frame_embeds)

    def _forward_locked(self, ids: torch.Tensor, frame_embeds: torch.Tensor = None):
        self._enqueue_step(ids, [] if frame_embeds is None else [frame_embeds])
        return self._consume(self.model.engine.read_decisions(1)[0])

    def _consume(self, dec):
        """a decision the session acts on: the test seam sees it and it counts as one call"""
        if self.decision_hook is not None:
            dec = self.decision_hook(dec, self._n_calls)
        self._n_calls += 1
        return dec

    def _enqueue_step(self, ids: torch.Tensor, frames, n_drafts: int = 0, sample=None):
        """Enqueue one KV-append step over [embed(ids) ; frames[0] ; interval id ; frames[1] ; interval id ; ...].
        With more than one frame every frame is a segment with its own decision (the step is the same arithmetic as
        one step per frame, each fed the interval id of a silent predecessor).  n_drafts (no frames): the last n_drafts
        ids are one-token segments, each with its own decision.  sample: Engine.step's, one SampleRow per segment.
        Returns the segment lengths."""
        eng = self.model.engine
        id_list = [int(x) for x in ids.reshape(-1).tolist()]
        n_ids = len(id_list)
        n_frs = tuple(f.shape[0] for f in frames)
        n_fr = sum(n_frs) + len(frames) - 1 if frames else 0   # rows after the prefix ids
        T = n_ids + n_fr
        segs = [n_ids + n_frs[0]] + [1 + n for n in n_frs[1:]] if frames else [T - n_drafts] + [1] * n_drafts
        # pre-allocated step buffers: no per-step torch.empty / torch.cat / pageable H2D on the hot path
        if T > self._packed.shape[0]:
            self._alloc_step_buffers(2 * T)
        packed = self._packed[:T]
        o = n_ids
        for j, f in enumerate(frames):
            o += j > 0          # the interval id row, gathered on the device
            packed[o:o + f.shape[0]] = f.view(-1, self.hidden_size)
            o += f.shape[0]
        key = (tuple(id_list), n_frs)
        row_ids = self._row_ids_cache.get(key) if n_fr else None   # steady state: [interval id | 10 frame rows]
        if row_ids is None:
            host = self._row_ids_host[:T]
            host[:n_ids] = torch.tensor(id_list, dtype=torch.int64)
            host[n_ids:] = -1
            o = n_ids
            for j, n in enumerate(n_frs):
                if j:
                    host[o] = self.frame_token_interval_id
                    o += 1
                o += n
            if n_fr:    # frame steps repeat (same prefix ids): keep their device copy
                row_ids = host.to(self.device, non_blocking=True)
                if len(self._row_ids_cache) < 64:
                    self._row_ids_cache[key] = row_ids
            else:       # prompts / AR tokens: one pinned -> device copy, consumed before the decision read-back below
                row_ids = self._row_ids_dev[:T]
                row_ids.copy_(host, non_blocking=True)
        main = torch.cuda.current_stream(self.device)
        pre = None
        if self._want_prefetch is not None:
            pre = torch.cuda.Event()
            pre.record(main)
        eng.step([self._kv.stream_id], [T], packed, row_ids=row_ids,   # token rows gathered on the device
                 segments=[segs] if len(segs) > 1 else None, sample=sample)
        self.past_key_values = self._kv
        hist = list(id_list)
        for j, n in enumerate(n_frs):
            hist += ([self.frame_token_interval_id] if j else []) + [SEP] * n
        if frames and self.drafter is not None:   # frame rows enter the drafter's history as separators
            self.drafter.sync(eng.kv_len(self._kv.stream_id) - T)
            self.drafter.extend(hist)
        if not isinstance(self.drafter, NgramDrafter):   # the session's own history (_fed_ids)
            del self._fed[eng.kv_len(self._kv.stream_id) - T:]
            self._fed.extend(hist)
        if pre is not None:
            # encode-ahead of the next frame, enqueued AFTER the step's launches (the host is the critical path right
            # after a decision read-back) but ordered only behind what preceded the step: it runs concurrently with it
            nxt, self._want_prefetch = self._want_prefetch, None
            stop = min(nxt + max(1, int(self.prefetch_depth)), self.video_tensor.size(0))
            self._side.wait_event(pre)
            with torch.cuda.stream(self._side):
                pe = self.model.visual_embed(self.video_tensor[nxt:stop]).split(self.frame_num_tokens)
                ev = torch.cuda.Event()
                ev.record(self._side)
            for k, e in zip(range(nxt, stop), pe):
                self._prefetched[k] = (e, ev)
            self._prefetch_event = ev
        return segs

    def _call_for_response(self, video_time, query):
        if query is not None:
            self.last_ids = self.tokenizer.apply_chat_template([{'role': 'user', 'content': query}], add_stream_query_prompt=True, add_generation_prompt=True, return_tensors='pt')
        else:
            assert int(self.last_ids) == self.stream_end_id, f'{self.last_ids} != {self.stream_end_id}'  # "]\n" closes the frame list
            self.last_ids = self._added_stream_generation_ids
        ids = [int(x) for x in self.last_ids.reshape(-1).tolist()]
        # before a response: room for the prompt and every id it may generate.  A verify step's drafts fit in it as
        # well (draft_cap keeps them within the ids still wanted), so the loop below never evicts.
        self._make_room(len(ids) + self.inplace_output_ids.size(1))

        def step(pending, drafts, sample=None):
            with self._lock:
                self._enqueue_step(torch.tensor(pending + drafts, dtype=torch.long), [], n_drafts=len(drafts),
                                   sample=sample)
        # fast_greedy_generate (models/modeling_live.py:173-182), or sampled ids, verifying drafts from the history
        out = generate_ids(self.model.engine, self._kv.stream_id, step, len(ids), self.inplace_output_ids.size(1),
                           self.eos_token_id, first_ids=ids, drafter=self.drafter, consume=self._consume,
                           sampling=self.sampling, position_base=self.evicted_tokens)
        n = len(out)
        self.inplace_output_ids[0, :n] = torch.tensor(out, dtype=torch.long)
        output_ids = self.inplace_output_ids[:, :n]
        self.last_ids = output_ids[:, -1:].clone()
        if query:
            query = f'(Video Time = {video_time}s) User: {query}'
        response = f'(Video Time = {video_time}s) Assistant:{self.tokenizer.decode(output_ids[0], skip_special_tokens=True, clean_up_tokenization_spaces=True)}'
        return query, response

    def _call_for_streaming(self):
        while self.frame_embeds_queue:
            # 1. a query that is due before the next frame is answered first
            if self.query_queue and self.frame_embeds_queue[0][0] > self.query_queue[0][0]:
                video_time, query = self.query_queue.popleft()
                return video_time, query
            if not self.past_key_values:
                self.last_ids = self._start_ids
            elif int(self.last_ids.reshape(-1)[-1]) == self.eos_token_id and self.last_ids.numel() == 1:
                self.last_ids = torch.cat([self.last_ids.reshape(1, -1), self._added_stream_prompt_ids], dim=1)
            self._make_room(self.last_ids.numel() + self.frame_embeds_queue[0][1].shape[0])   # before a frame step
            n = self._backlog_run()
            if n > 1:
                video_time, query, answered = self._stream_backlog(n)
                if answered:
                    return video_time, query
                continue
            video_time, frame_embeds = self.frame_embeds_queue.popleft()
            dec = self._forward(self.last_ids, frame_embeds)
            # 2. a query due at this frame's time is answered right after the frame
            if self.query_queue and video_time >= self.query_queue[0][0]:
                video_time, query = self.query_queue.popleft()
                return video_time, query
            # 3. speak/silent: below-threshold interval probability -> the argmax excludes the interval id
            next_id = dec.next_id(self.frame_token_interval_id, self.frame_token_interval_threshold)
            self.last_ids = torch.tensor([[next_id]], dtype=torch.long)
            if next_id != self.frame_token_interval_id:
                return video_time, None
        return None, None

    def _backlog_run(self) -> int:
        """Queued frames (from the head) that one segmented step can take: the loop above would step them one after
        another, each fed the interval id of a silent predecessor, without a query in between.  So the run stops
        before a frame that rule 1 would precede, after a frame that rule 2 answers, and at max_step_tokens.  Under a
        context window it also stops before a frame whose own step would evict: no segmented step spans an eviction."""
        iid, q = self.frame_token_interval_id, self.frame_embeds_queue
        if iid is None or len(q) < 2:
            return 1
        due = self.query_queue[0][0] if self.query_queue else None
        room = self.model.engine.max_step_tokens - self.last_ids.numel() - q[0][1].shape[0]
        win = self._context_window
        if win is not None:   # window room left after the first frame's step
            kv = self.model.engine.kv_len(self._kv.stream_id)
            room = min(room, win - kv - self.last_ids.numel() - q[0][1].shape[0])
        n, prev = 1, q[0][0]
        # input_video_stream appends to the queue from another thread under the same lock: a deque may not change
        # while it is iterated (only this thread pops, so the n frames counted here stay at the head)
        with self._lock:
            for video_time, frame_embeds in itertools.islice(q, 1, None):
                if due is not None and (prev >= due or video_time > due):   # rule 2 after the previous frame / rule 1 before this one
                    break
                room -= 1 + frame_embeds.shape[0]
                if room < 0:
                    break
                n, prev = n + 1, video_time
        return n

    def _stream_backlog(self, n: int):
        """Step the first n queued frames as one segmented step, then act on their decisions in order exactly as the
        loop above acts on one frame's.  Where that loop would stop (a frame speaks, or a query is due) the stream is
        cut back to the end of that frame and the later frames go back to the head of the queue.
        Returns (video_time, query, stop): stop is False when every frame was silent."""
        with self._lock:
            frames = [self.frame_embeds_queue.popleft() for _ in range(n)]
            eng, sid = self.model.engine, self._kv.stream_id
            kv0 = eng.kv_len(sid)
            segs = self._enqueue_step(self.last_ids, [f for _, f in frames])
            decs = eng.read_decisions(n)

            def take_back(j):   # keep frames [0, j)
                if j < n:
                    eng.kv_truncate(sid, kv0 + sum(segs[:j]))
                    if self.drafter is not None:
                        self.drafter.sync(kv0 + sum(segs[:j]))
                    self.frame_embeds_queue.extendleft(reversed(frames[j:]))

            for j, (video_time, _) in enumerate(frames):
                # 1. a query that is due before this frame is answered first
                if j and self.query_queue and video_time > self.query_queue[0][0]:
                    take_back(j)
                    return (*self.query_queue.popleft(), True)
                dec = self._consume(decs[j])
                # 2. a query due at this frame's time is answered right after the frame
                if self.query_queue and video_time >= self.query_queue[0][0]:
                    take_back(j + 1)
                    return (*self.query_queue.popleft(), True)
                # 3. speak/silent
                next_id = dec.next_id(self.frame_token_interval_id, self.frame_token_interval_threshold)
                self.last_ids = torch.tensor([[next_id]], dtype=torch.long)
                if next_id != self.frame_token_interval_id:
                    take_back(j + 1)
                    return video_time, None, True
            return None, None, False

    def __call__(self):
        while not self.frame_embeds_queue:
            continue
        video_time, query = self._call_for_streaming()
        response = None
        if video_time is not None:
            query, response = self._call_for_response(video_time, query)
        return query, response


def _read_video_tchw(path: str, fps=None, resolution=None) -> torch.Tensor:
    """demo/inference.py:111-115 + the preprocessing demo/cli.py:15-20 does before it (see video_ingest.py)."""
    from .video_ingest import read_video_resampled
    return read_video_resampled(path, fps=fps, resolution=resolution)
