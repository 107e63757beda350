"""Concurrent video streams on one GPU (BASELINE.json configs 3 and 5).

The reference handles one stream per process (demo/inference.py:16; the scalar `if`s at :77,80 raise for
batch > 1).  Here every stream is an independent state machine with the protocol of `LiveInfer`
(demo/inference.py:40-82) and all streams that have work at a tick are advanced by ONE ragged
`vlo_step_ids` launch: frame steps (q = 1 + 10), response prompts (q = 3..40) and autoregressive tokens
(q = 1) ride together, so the 15 GB weight pass is shared.  The ViT runs batched over the frames the
tick needs.  Per tick: one H2D copy (row ids), one D2H copy (decisions), one sync.

Encode-ahead: when at most `encode_ahead_max_frames` (2) streams have a frame pending, those frames are encoded on a
side CUDA stream right after the ragged step of the tick has been enqueued, so the ViT of tick i+1 runs in the shadow
of the HBM-bound decoder step of tick i.  Only that regime pays: the engine's small-batch ViT configuration shares an
SM with a decoder weight-streaming CTA, whereas a batch-8 ViT time-slices the SMs with the persistent decoder kernels
(measured 8 streams: 616 frames/s with the ViT in line, 534 with it on the side stream).

More sessions than the engine holds: a session without work (no pending frame, not responding) may be swapped out to
a pinned host image (`Engine.kv_swap_out`), and then holds neither KV pages nor a stream slot.  Before each tick every
session with work is made resident again if it fits (`StreamScheduler._make_room`); the policy is fixed and
deterministic.

Context window: a session with `context_window` set keeps its cache within that many tokens as `LiveInfer` does, with
the same policy (`engine.evict_span`, or `engine.retain_spans` with `context_keep_turns`) at the same points: before a
frame step and before a response.  A resident session evicts before its pages are counted; a swapped-out one right after
its swap-in.
"""
from __future__ import annotations

import collections
from typing import Callable, Deque, List, Optional, Tuple

import torch

from ._lib import VloError
from .config import SamplingConfig
from .engine import KvImage, SampleRow, evict_span, kept_rows, retain_spans
from .modeling_live import LiveLlamaForCausalLM
from .speculative import sample_rows


class StreamSession:
    """State of one video stream (mirror of the per-instance state of the reference's LiveInfer)."""
    IDLE, RESPOND = 0, 1

    def __init__(self, sched: "StreamScheduler", index: int):
        self.sched, self.index = sched, index
        # swapped out (stream_id None): the cache lives in `image` (None: empty) and the session holds no engine stream
        self.image: Optional[KvImage] = None
        self.last_step = -1   # tick of the session's last step (least recently stepped is swapped out first)
        try:
            self.stream_id: Optional[int] = sched.model.engine.stream_open()
        except VloError:      # more sessions than stream slots: this one starts swapped out
            self.stream_id = None
        self.frame_fps = sched.frame_fps
        self.threshold = 0.725
        # response tokens, as LiveInfer.sampling: None = greedy; each session may have its own config
        self.sampling: Optional[SamplingConfig] = None
        # as LiveInfer.context_window: None = off; the sink is the scheduler's start_ids
        self.context_window: Optional[int] = None
        # as LiveInfer.context_keep_turns: with a window, keep the questions and answers and drop old frames token by token
        self.context_keep_turns = False
        self.reset()

    @property
    def resident(self) -> bool:
        return self.stream_id is not None

    def kv_tokens(self) -> int:
        if self.resident:
            return self.sched.model.engine.kv_len(self.stream_id)
        return self.image.n_tokens if self.image is not None else 0

    def reset(self):
        if self.resident:
            self.sched.model.engine.stream_reset(self.stream_id)
        self.image = None
        getattr(self.sched, "_ahead", {}).pop(self.index, None)   # an encoded-ahead frame of the old clip
        self.query_queue: Deque[Tuple[float, str]] = collections.deque()
        self.pending_frames: Deque[Tuple[float, int]] = collections.deque()   # (video_time, frame index)
        self.video: Optional[torch.Tensor] = None
        self.video_time, self.last_frame_idx = 0.0, -1
        self.last_ids: List[int] = []
        self.started = False
        self.state = self.IDLE
        self.resp: List[int] = []
        self.resp_time, self.resp_query = None, None
        self.outputs: List[Tuple[float, Optional[str], Optional[str]]] = []   # (time, query, response text)
        self.events: List[tuple] = []
        self.n_calls = 0
        self.evicted_tokens = 0   # cache positions the context window dropped (sampled positions count them)
        self.fed_ids: List[int] = []   # the id fed at every cache position, -1 for a frame row (retain_spans reads it)
        self._op = None

    # -- inputs (LiveInfer.load_video / input_video_stream / input_query_stream)
    def load_video(self, video_u8: torch.Tensor):
        self.video = video_u8.to(self.sched.model.device)
        getattr(self.sched, "_ahead", {}).pop(self.index, None)

    def input_video_stream(self, video_time: float):
        idx = int(video_time * self.frame_fps)
        if idx > self.last_frame_idx:
            for r in range(self.last_frame_idx + 1, idx + 1):
                self.pending_frames.append((r / self.frame_fps, r))
        self.last_frame_idx, self.video_time = idx, video_time

    def input_query_stream(self, query: str, video_time: Optional[float] = None):
        self.query_queue.append((self.video_time if video_time is None else video_time, query))

    def has_work(self) -> bool:
        return self.state == self.RESPOND or bool(self.pending_frames)

    # -- planning: which rows does this stream contribute to the next ragged step?
    def plan(self):
        """Returns (row_ids list, frame_index or None).  Sets self._op for `advance`."""
        tk, cfg = self.sched.tokenizer, self.sched.model.config
        if self.state == self.RESPOND:
            ids = self._next_ids
            self._op = ("gen",)
            return ids, None
        # IDLE with a frame pending (demo/inference.py:54-82)
        ft, fidx = self.pending_frames[0]
        if self.query_queue and ft > self.query_queue[0][0]:            # 1. query due before the next frame
            vt, q = self.query_queue.popleft()
            self._begin_response(vt, q)
            return self.plan()
        self.pending_frames.popleft()
        if not self.started:
            ids = list(self.sched.start_ids)
        elif len(self.last_ids) == 1 and self.last_ids[0] == cfg.eos_token_id:
            ids = self.last_ids + list(self.sched.stream_prompt_ids)
        else:
            ids = list(self.last_ids)
        self._op = ("frame", ft)
        return ids, fidx

    def _begin_response(self, video_time, query):
        tk = self.sched.tokenizer
        if query is not None:
            ids = tk.apply_chat_template([{'role': 'user', 'content': query}], add_stream_query_prompt=True,
                                         add_generation_prompt=True)
        else:
            assert self.last_ids == [self.sched.model.config.stream_end_id], f"{self.last_ids} != stream end id"
            ids = list(self.sched.stream_generation_ids)
        self.state, self.resp, self.resp_time, self.resp_query = self.RESPOND, [], video_time, query
        self._next_ids = list(ids)
        self.resp_prompt = list(ids)   # with the response's ids so far: the repetition penalty's set

    def sample_row(self, n: int) -> Optional[SampleRow]:
        """The SampleRow of the session's next step of n rows (None: not sampled): a response token, when the session
        samples.  Position and penalty ids are those LiveInfer gives the same token."""
        s = self.sampling
        if self._op is None or self._op[0] != "gen" or s is None or not s.do_sample:
            return None
        return sample_rows(s, self.evicted_tokens + self.kv_tokens() + n - 1, self.resp_prompt + self.resp,
                           len(self.resp_prompt) + len(self.resp), 0)[0]

    def window_need(self, n: int) -> int:
        """Tokens the context window makes room for before the planned step of n rows: the step itself, or at the start
        of a response its prompt and every id it may generate (as LiveInfer), so no response step evicts."""
        if self._op[0] == "gen" and not self.resp:
            return len(self.resp_prompt) + self.sched.max_new_tokens
        return n

    def _retain(self, need: int):
        cfg = self.sched.model.config
        return retain_spans(self.fed_ids, need, self.context_window, len(self.sched.start_ids),
                            cfg.frame_token_interval_id, cfg.frame_num_tokens)

    def window_drop(self, need: int) -> int:
        """Cache positions the context window would drop before appending `need` tokens (0: none or no window)."""
        if self.context_window is None:
            return 0
        if self.context_keep_turns:
            spans = self._retain(need)
            return len(self.fed_ids) - sum(n for _, n in spans) if spans else 0
        page = self.sched.model.engine.kv_pool_info()["page_tokens"]
        return evict_span(self.kv_tokens(), need, self.context_window, len(self.sched.start_ids), page)[1]

    def make_room(self, need: int):
        """Evict (resident session, context window set) before appending `need` tokens."""
        if self.context_window is None:
            return
        eng = self.sched.model.engine
        if self.context_keep_turns:
            spans = self._retain(need)
            if spans:
                eng.kv_compact(self.stream_id, spans)
                self.evicted_tokens += len(self.fed_ids) - sum(n for _, n in spans)
                self.fed_ids = kept_rows(self.fed_ids, spans)
            return
        self.evicted_tokens += eng.kv_make_room(self.stream_id, need, self.context_window, len(self.sched.start_ids))

    # -- consume the decision of the step this stream took part in
    def advance(self, dec):
        cfg = self.sched.model.config
        if self.sched.decision_hook is not None:
            dec = self.sched.decision_hook(self.index, dec, self.n_calls)
        self.n_calls += 1
        self.started = True
        op, self._op = self._op, None
        if op[0] == "gen":
            tok = dec.argmax_id if dec.sampled_id is None else dec.sampled_id
            self.resp.append(tok)
            if tok == cfg.eos_token_id or len(self.resp) >= self.sched.max_new_tokens:
                text = self.sched.tokenizer.decode(self.resp, skip_special_tokens=True)
                q = f'(Video Time = {self.resp_time}s) User: {self.resp_query}' if self.resp_query else self.resp_query
                self.outputs.append((self.resp_time, q, f'(Video Time = {self.resp_time}s) Assistant:{text}'))
                self.events.append(("response", self.resp_time, list(self.resp)))
                self.last_ids, self.state = [tok], self.IDLE
            else:
                self._next_ids = [tok]
            return
        _, vt = op
        if self.query_queue and vt >= self.query_queue[0][0]:            # 2. query due at this frame's time
            qt, q = self.query_queue.popleft()
            self._begin_response(qt, q)
            return
        nxt = dec.next_id(cfg.frame_token_interval_id, self.threshold)   # 3. speak / silent
        self.last_ids = [nxt]
        self.events.append(("frame", vt, nxt))
        if nxt != cfg.frame_token_interval_id:
            self._begin_response(vt, None)


class StreamScheduler:
    def __init__(self, model: LiveLlamaForCausalLM, tokenizer, n_streams: int, *, frame_fps: int = 2,
                 system_prompt: str = "", max_new_tokens: int = 100):
        self.model, self.tokenizer, self.frame_fps = model, tokenizer, frame_fps
        self.max_new_tokens = max_new_tokens
        self.decision_hook: Optional[Callable] = None
        tk = tokenizer
        self.start_ids = tk.apply_chat_template([{'role': 'system', 'content': system_prompt}], add_stream_prompt=True)
        self.stream_prompt_ids = tk.apply_chat_template([{}], add_stream_prompt=True)
        self.stream_generation_ids = tk.apply_chat_template([{}], add_stream_generation_prompt=True)
        self.swaps_out = self.swaps_in = 0
        self.sessions = [StreamSession(self, i) for i in range(n_streams)]
        self.ticks = 0
        self.frames_done = 0
        self.encode_ahead = True
        self.encode_ahead_max_frames = 2
        self._side = torch.cuda.Stream(model.device)
        self._ahead = {}          # session index -> (frame idx, embeds [frame_num_tokens, hidden], event)
        self._ahead_last = None   # last event recorded on the side stream (it owns the engine's ViT workspaces)

    def tick(self) -> int:
        """Advance every stream that has work by one operation.  Returns the number of streams advanced."""
        eng, cfg = self.model.engine, self.model.config
        active = [s for s in self.sessions if s.has_work()]
        # respect the engine's per-step token budget: long first-frame prompts go alone (the engine chunks them)
        plans, budget = [], eng.max_step_tokens
        for s in active:
            ids, fidx = s.plan()
            n = len(ids) + (cfg.frame_num_tokens if fidx is not None else 0)
            plans.append((s, ids, fidx, n))
        if not plans:
            return 0
        batch, used = [], 0
        busy = {s.index for s in active}
        for p in plans:
            if (batch and used + p[3] > budget) or not self._make_room(p[0], p[3], batch, busy):
                # not in this tick: undo the plan (frame / response prompt stays pending)
                s, ids, fidx, n = p
                if s._op and s._op[0] == "frame":
                    s.pending_frames.appendleft((s._op[1], fidx))
                s._op = None
                continue
            batch.append(p)
            used += p[3]
        # batched ViT over the frames this tick needs that were not encoded ahead
        main = torch.cuda.current_stream(eng.device)
        fr = [(s, fidx) for s, _, fidx, _ in batch if fidx is not None]
        per_frame, waited, todo = {}, set(), []
        for s, fidx in fr:
            a = self._ahead.get(s.index)
            if a is not None and a[0] == fidx:
                if id(a[2]) not in waited:
                    main.wait_event(a[2])
                    waited.add(id(a[2]))
                a[1].record_stream(main)
                per_frame[s.index] = a[1]
                del self._ahead[s.index]
            else:
                todo.append((s, fidx))
        if todo:
            if self._ahead_last is not None:
                main.wait_event(self._ahead_last)     # a side-stream ViT may still own the ViT workspaces
            frames = torch.stack([s.video[fidx] for s, fidx in todo], 0)
            emb = self.model.visual_embed(frames).view(len(todo), cfg.frame_num_tokens, cfg.hidden_size)
            for k, (s, _) in enumerate(todo):
                per_frame[s.index] = emb[k]
        self.frames_done += len(fr)
        T = sum(p[3] for p in batch)
        packed = torch.empty(T, cfg.hidden_size, dtype=torch.bfloat16, device=eng.device)
        row_ids, q_lens, off, k = [], [], 0, 0
        for s, ids, fidx, n in batch:
            row_ids.extend(ids)
            if fidx is not None:
                packed[off + len(ids): off + n] = per_frame[s.index]
                row_ids.extend([-1] * cfg.frame_num_tokens)
            q_lens.append(n)
            off += n
        rid = torch.tensor(row_ids, dtype=torch.int64).to(eng.device, non_blocking=True)
        pre = torch.cuda.Event()
        pre.record(main)
        sample = [s.sample_row(n) for s, _, _, n in batch]   # sampling sessions' response rows: one launch for all
        eng.step([s.stream_id for s, *_ in batch], q_lens, packed, row_ids=rid, want_logits=False,
                 sample=sample if any(r is not None for r in sample) else None)
        if self.encode_ahead:
            self._launch_encode_ahead(pre)        # enqueued after the step's launches, runs concurrently with it
        for s, ids, fidx, _ in batch:
            s.fed_ids.extend(ids + ([-1] * cfg.frame_num_tokens if fidx is not None else []))
        decs = eng.read_decisions(len(batch))
        for (s, *_), d in zip(batch, decs):
            s.last_step = self.ticks
            s.advance(d)
        self.ticks += 1
        return len(batch)

    # -- swapping: a session without work may give its pages and stream slot back (host image) and take them again later
    def _make_room(self, s: StreamSession, n: int, batch, busy) -> bool:
        """Make session `s` resident with room for n more tokens, next to the sessions already in `batch`.  Resident
        sessions outside the batch are swapped out for it: first those without work (not in `busy`), then, only while
        the batch is still empty (so that every tick steps someone), those whose turn is later; least recently stepped
        first, lowest index on a tie.  False: `s` waits for a later tick.  Raises if `s` alone cannot fit in an empty
        pool."""
        eng = self.model.engine
        info = eng.kv_pool_info()
        page, total = info["page_tokens"], info["total_pages"]
        pages = lambda t: -(-t // page)
        w_need = s.window_need(n)
        if s.resident:
            s.make_room(w_need)
        kv = after = s.kv_tokens()
        if not s.resident:   # it evicts right after its swap-in
            after -= s.window_drop(w_need)
        if pages(after + n) > total:
            raise VloError(f"session {s.index}: {after + n} tokens need {pages(after + n)} KV pages, the pool has {total}")
        # pages the sessions already in the batch take in this step
        reserved = sum(pages(q.kv_tokens() + m) - pages(q.kv_tokens()) for q, _, _, m in batch)
        need = pages(kv + n) - pages(kv) if s.resident else max(pages(kv), pages(after + n))
        keep = {q.index for q, *_ in batch} | {s.index}

        def evict() -> bool:
            cands = [q for q in self.sessions if q.resident and q.index not in keep
                     and (q.index not in busy or not batch)]
            if not cands:
                return False
            self._swap_out(min(cands, key=lambda q: (q.index in busy, q.last_step, q.index)))
            return True

        while eng.kv_pool_info()["free_pages"] - reserved < need:
            if not evict():
                return False
        while not s.resident:
            try:
                sid = eng.stream_open()
            except VloError:      # no free stream slot
                if not evict():
                    return False
                continue
            if s.image is not None:
                try:
                    eng.kv_swap_in(sid, s.image)
                except VloError:
                    eng.stream_close(sid)
                    raise
            s.stream_id, s.image = sid, None
            self.swaps_in += 1
            s.make_room(w_need)
        return True

    def _swap_out(self, s: StreamSession):
        eng = self.model.engine
        img = eng.kv_swap_out(s.stream_id)
        eng.stream_close(s.stream_id)
        s.stream_id, s.image = None, (img if img.n_tokens else None)
        self.swaps_out += 1

    def _launch_encode_ahead(self, after: "torch.cuda.Event"):
        """One batched ViT on the side stream over every stream's next pending frame that is not encoded yet."""
        want = []
        for s in self.sessions:
            if s.video is None or not s.pending_frames:
                continue
            fidx = s.pending_frames[0][1]
            a = self._ahead.get(s.index)
            if (a is None or a[0] != fidx) and 0 <= fidx < s.video.size(0):
                want.append((s, fidx))
        if not want or len(want) > self.encode_ahead_max_frames:
            return
        cfg = self.model.config
        self._side.wait_event(after)
        with torch.cuda.stream(self._side):
            frames = torch.stack([s.video[fidx] for s, fidx in want], 0)
            emb = self.model.visual_embed(frames).view(len(want), cfg.frame_num_tokens, cfg.hidden_size)
            ev = torch.cuda.Event()
            ev.record(self._side)
        for k, (s, fidx) in enumerate(want):
            self._ahead[s.index] = (fidx, emb[k], ev)
        self._ahead_last = ev

    def run_until_idle(self, max_ticks: int = 1 << 30) -> int:
        n = 0
        while n < max_ticks and self.tick():
            n += 1
        return n
