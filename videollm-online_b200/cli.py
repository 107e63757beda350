"""Headless driver + FPS measurement: the engine-backed counterpart of demo/cli.py:12-50.

    python -m videollm_online_b200.cli --synthetic_weights true [--frames 100] [--video clip.mp4] [--whole_video]
        [--live | --live_raw WxH:FORMAT] [--do_sample --temperature 0.6 --top_p 0.9 --top_k 50 --repetition_penalty 1.1 --sample_seed 0]

Responses are greedy unless --do_sample is given (SamplingConfig; --seed stays the synthetic weights' seed).
--context_window N keeps the session's cache within N tokens (0: off): the start prompt stays, the oldest pages after it
are dropped.
--context_keep_turns (with --context_window) drops the oldest frames token by token instead, and keeps the questions and
answers.
--live (with --video) feeds the clip as a camera would: decoded at its native size without a resize, one frame per
1 / frame_fps of video time pushed through LiveInfer.push_frames (BGR, letterboxed on the device), each one frame ahead
of the frame being processed.
--live_raw WxH:FORMAT (with --video PATH, or --video - for stdin) does the same with raw frames, one per frame interval,
in ffmpeg's rawvideo layout: FORMAT is nv12, yuv420p or yuyv422 (ffmpeg's -pix_fmt names), converted to RGB on the
device.  A stream that ends inside a frame drops it with a warning.  A camera at 2 frames/s:
    ffmpeg -i <camera> -r 2 -f rawvideo -pix_fmt nv12 - | python -m videollm_online_b200.cli --live_raw 1920x1080:nv12 --video -
--fp8_weights serves the decoder layers from e4m3 weights with per-row scales (half their bytes per step; the model's
numbers change, so it is off by default).
--fp8_activations (with --fp8_weights) also quantizes the layer GEMMs' activations to e4m3 per token and multiplies them on
the FP8 tensor cores (W8A8); off by default for the same reason.
--int4_weights serves the decoder layers from 4-bit weights with one bf16 scale per 128 weights of a row (W4A16: a
quarter of their bf16 bytes per step); the numbers change, so it is off by default, and it excludes the FP8 flags.
--quantize_vocab (with --fp8_weights or --int4_weights) also serves the token embeddings and lm_head in that quantized
form, which frees their memory for the KV cache; the numbers change, so it is off by default.
--quantized_prefill (with --fp8_weights or --int4_weights) runs long prompts and clips as prefills on the quantized
layers, with the same numbers as without; it grows the engine's token-row workspaces, so it is off by default.

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
         whole_video: bool = False, live: bool = False, live_raw: str = None):
    camera, fmt = None, dict(bgr=True)
    if live and live_raw:
        raise ValueError("--live and --live_raw do not combine")
    if live or live_raw:
        if not isinstance(video, str) or whole_video:
            raise ValueError("--live and --live_raw take a clip (--video) and do not combine with --whole_video")
        from .video_ingest import iter_raw_frames, iter_video_frames, parse_raw_spec
        if live_raw:
            W, H, pixel_format = parse_raw_spec(live_raw)
            camera = iter_raw_frames(sys.stdin.buffer if video == '-' else open(video, 'rb'), W, H, pixel_format)
            fmt = dict(pixel_format=pixel_format)
        else:
            camera = iter_video_frames(video, fps=liveinfer.frame_fps)
        live = True
    else:
        if video is None:
            video = synthetic_clip(n_iters, liveinfer.frame_resolution)
        liveinfer.load_video(video)
    liveinfer.input_query_stream('Please narrate the video in real time.', video_time=0.0)
    timecosts, history = [], {'frame_fps': liveinfer.frame_fps, 'conversation': []}
    fps = 0.0
    if whole_video:
        return _drain_whole_video(liveinfer, min(n_iters, liveinfer.num_video_frames), history, save_history_path, quiet)
    frame = next(camera, None) if live else None   # the camera frame of video time i / frame_fps
    for i in range(n_iters if live else min(n_iters, liveinfer.num_video_frames)):
        if live and frame is None:
            break
        start = time.time()
        if live:
            # frame i + 1 is delivered while frame i is processed, so encode-ahead takes it as it takes a loaded clip's
            if i == 0:
                liveinfer.push_frames([torch.from_numpy(frame)], **fmt)
            frame = next(camera, None)
            if frame is not None and i + 1 < n_iters:
                liveinfer.push_frames([torch.from_numpy(frame)], **fmt)
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
    # --live: push the clip's frames at their native size, one per frame interval (a camera feed)
    # --live_raw WxH:FORMAT: the same from raw YUV frames (--video PATH, or - for stdin)
    live_raw = sys.argv[sys.argv.index('--live_raw') + 1] if '--live_raw' in sys.argv else None
    main(LiveInfer(parse_args()), video=video, n_iters=n, whole_video='--whole_video' in sys.argv, live='--live' in sys.argv,
         live_raw=live_raw)
