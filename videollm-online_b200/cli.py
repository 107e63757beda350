"""Headless driver + FPS measurement: the engine-backed counterpart of demo/cli.py:12-50.

    python -m videollm_online_b200.cli --synthetic_weights true [--frames 100] [--video clip.mp4] [--whole_video]
        [--do_sample --temperature 0.6 --top_p 0.9 --top_k 50 --repetition_penalty 1.1 --sample_seed 0]

Responses are greedy unless --do_sample is given (SamplingConfig; --seed stays the synthetic weights' seed).
--context_window N keeps the session's cache within N tokens (0: off): the start prompt stays, the oldest pages after it
are dropped.
--context_keep_turns (with --context_window) drops the oldest frames token by token instead, and keeps the questions and
answers.
--fp8_weights serves the decoder layers from e4m3 weights with per-row scales (half their bytes per step; the model's
numbers change, so it is off by default).

Loads (or synthesises) a clip, asks for narration at t=0 and runs N iterations of
(encode 1 frame -> KV-append step -> maybe respond), reporting the reference's
"Average Processing FPS" = frames / wall time including responses (demo/cli.py:38)."""
from __future__ import annotations

import json
import os
import sys
import time

import torch

from .config import parse_args
from .inference import LiveInfer


def synthetic_clip(n_frames: int, resolution: int, seed: int = 0) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n_frames, 3, resolution, resolution), dtype=torch.uint8, generator=g)


def main(liveinfer: LiveInfer, video=None, n_iters: int = 100, save_history_path: str = None, quiet: bool = False,
         whole_video: bool = False):
    if video is None:
        video = synthetic_clip(n_iters, liveinfer.frame_resolution)
    liveinfer.load_video(video)
    liveinfer.input_query_stream('Please narrate the video in real time.', video_time=0.0)
    timecosts, history = [], {'frame_fps': liveinfer.frame_fps, 'conversation': []}
    fps = 0.0
    if whole_video:
        return _drain_whole_video(liveinfer, min(n_iters, liveinfer.num_video_frames), history, save_history_path, quiet)
    for i in range(min(n_iters, liveinfer.num_video_frames)):
        start = time.time()
        liveinfer.input_video_stream(i / liveinfer.frame_fps)
        query, response = liveinfer()
        timecosts.append(time.time() - start)
        fps = (i + 1) / sum(timecosts)
        entry = {'time': liveinfer.video_time, 'fps': fps, 'cost': timecosts[-1]}
        if query:
            history['conversation'].append({'role': 'user', 'content': query, **entry})
        if response:
            history['conversation'].append({'role': 'assistant', 'content': response, **entry})
        if not query and not response:
            history['conversation'].append(entry)
        if not quiet and (query or response):
            print(query or '', response or '')
    _finish(history, fps, save_history_path, quiet)
    return fps, history


def _finish(history, fps, save_history_path, quiet):
    if save_history_path:
        os.makedirs(os.path.dirname(save_history_path) or '.', exist_ok=True)
        json.dump(history, open(save_history_path, 'w'), indent=4)
    if not quiet:
        print(f'Average Processing FPS: {fps:.1f}')


def _drain_whole_video(liveinfer: LiveInfer, n_frames: int, history, save_history_path, quiet):
    """Narrate a recorded clip as fast as possible: every frame is queued at t = 0 and the queue is drained, so the
    silent stretches between responses go through segmented steps of several frames each."""
    start = time.time()
    liveinfer.input_video_stream((n_frames - 1) / liveinfer.frame_fps)
    while liveinfer.frame_embeds_queue:
        query, response = liveinfer()
        entry = {'time': liveinfer.video_time, 'elapsed': time.time() - start}
        if query:
            history['conversation'].append({'role': 'user', 'content': query, **entry})
        if response:
            history['conversation'].append({'role': 'assistant', 'content': response, **entry})
        if not quiet and (query or response):
            print(query or '', response or '')
    torch.cuda.synchronize(liveinfer.device)
    fps = n_frames / (time.time() - start)
    _finish(history, fps, save_history_path, quiet)
    return fps, history


if __name__ == '__main__':
    n, video = 100, None
    if '--frames' in sys.argv:
        n = int(sys.argv[sys.argv.index('--frames') + 1])
    if '--video' in sys.argv:   # a clip on disk: resampled to frame_fps and letterboxed to frame_resolution on load
        video = sys.argv[sys.argv.index('--video') + 1]
    # --whole_video: queue the whole clip at t = 0 and drain it (narrate a recorded file as fast as possible)
    main(LiveInfer(parse_args()), video=video, n_iters=n, whole_video='--whole_video' in sys.argv)
