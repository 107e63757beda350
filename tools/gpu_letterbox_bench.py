"""Dev tool: live frames at their native size (vlo_letterbox, LiveInfer.push_frames).  One JSON line per measurement:
  card       GPU name and power limit (nvidia-smi), read in the same run
  letterbox  Engine.letterbox us per frame at 640x480, 1280x720, 1920x1080 and 3840x2160, B = 1 and 8 (frames already on
             the device; CUDA events around --iters warm back-to-back calls, so host overhead shows where it exceeds the
             kernel), and the kernel alone: letterbox_kernel's device time per frame from torch.profiler
  host       host-side cost of ingesting one 1920x1080 CPU frame: the copy into pinned staging alone (torch's copy_, which
             Engine.letterbox makes, and one np.copyto for comparison), and a whole LiveInfer.push_frames call (host clock, no synchronisation), both on the thread that drives the session
  h2d        the copy of one native frame from pinned host memory to the device (CUDA events)
  cv2        cv2.resize(INTER_CUBIC) + pad on this host's CPU for the same frames (the read_video_resampled path), per frame
  live       LiveInfer frames/s over --frames 1920x1080 frames, pushed one frame ahead of the one stepped (a camera
             delivers the next frame while the current one is processed) against load_video of the same canvases,
             alternated --reps times; the full-size synthetic model, every frame silent
  backlog    --backlog pushed 1920x1080 frames queued at once and drained (segmented steps), timed from the first push,
             against the same drain from load_video of the same canvases
  python tools/gpu_letterbox_bench.py [--frames 300] [--backlog 110] [--reps 3] [--iters 200]"""
import argparse, json, pathlib, subprocess, sys, time
import numpy as np
import torch
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import llama3_8b_siglip_l, weights as W
from videollm_online_b200.engine import Engine
from videollm_online_b200.video_ingest import letterbox_geometry

ap = argparse.ArgumentParser()
ap.add_argument("--frames", type=int, default=300)
ap.add_argument("--backlog", type=int, default=110)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--iters", type=int, default=200)
args = ap.parse_args()


def emit(kind, rec):
    print(json.dumps({"what": kind, **rec}), flush=True)


smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
emit("card", {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": smi})

dev = torch.device("cuda:0")
cfg = llama3_8b_siglip_l()
R = cfg.frame_resolution
CAP = 11 * (max(args.frames, args.backlog) + 8) + 2048
eng = Engine(cfg, dev, max_streams=1, max_kv_tokens=CAP, max_step_tokens=128, max_vit_batch=8)
eng.load_weights(W.synthetic_engine_weights(cfg, dev, CAP, seed=0))
g = np.random.default_rng(0)


def native(W_, H_, n=8):
    return [torch.from_numpy(g.integers(0, 256, (H_, W_, 3), dtype=np.uint8)) for _ in range(n)]


def timed(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


import cv2  # noqa: E402

for W_, H_ in [(640, 480), (1280, 720), (1920, 1080), (3840, 2160)]:
    host = native(W_, H_)
    on_dev = [f.to(dev) for f in host]
    rec = {f"B{B}_us_per_frame": round(1e3 * timed(lambda: eng.letterbox(on_dev[:B]), args.iters) / B, 2) for B in (1, 8)}
    for B in (1, 8):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(50):
                eng.letterbox(on_dev[:B])
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "letterbox_kernel" in e.key]
        dt = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0) for e in ev)
        rec[f"B{B}_kernel_us_per_frame"] = round(dt / (50 * B), 2) if ev else None
    emit("letterbox", {"size": f"{W_}x{H_}", **rec})
    pinned, dst = host[0].pin_memory(), torch.empty_like(on_dev[0])
    emit("h2d", {"size": f"{W_}x{H_}", "bytes": pinned.numel(),
                 "us_per_frame": round(1e3 * timed(lambda: dst.copy_(pinned, non_blocking=True), args.iters), 2)})
    sw, sh, x0, y0 = letterbox_geometry(W_, H_, R)
    frames_np = [f.numpy() for f in host]

    def host_letterbox(fr):
        canvas = np.zeros((R, R, 3), dtype=np.uint8)
        canvas[y0:y0 + sh, x0:x0 + sw] = cv2.resize(fr, (sw, sh), interpolation=cv2.INTER_CUBIC)
        return canvas
    for fr in frames_np:
        host_letterbox(fr)
    n = max(20, args.iters // 4)
    t0 = time.perf_counter()
    for k in range(n):
        host_letterbox(frames_np[k % len(frames_np)])
    emit("cv2", {"size": f"{W_}x{H_}", "threads": cv2.getNumThreads(),
                 "us_per_frame": round(1e6 * (time.perf_counter() - t0) / n, 1)})

# ---- end to end through LiveInfer
from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT  # noqa: E402
from videollm_online_b200.inference import LiveInfer  # noqa: E402
from videollm_online_b200.modeling_live import LiveLlamaForCausalLM, StreamKV  # noqa: E402
from videollm_online_b200.tokenization_live import ByteTokenizer  # noqa: E402

IID = cfg.frame_token_interval_id
model = LiveLlamaForCausalLM(cfg, eng)
sid = eng.stream_open()
li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT), model=model, tokenizer=ByteTokenizer(cfg),
               stream=StreamKV(eng, sid))


def silent(dec, n):
    dec.argmax_id = dec.argmax_prob_id = IID
    dec.p_interval = 1.0
    return dec


li.decision_hook = silent
cam = native(1920, 1080, 16)
N = max(args.frames, args.backlog)
canvases = torch.cat([eng.letterbox([cam[k % len(cam)]]) for k in range(N)])   # what the pushed frames become


push_s = []   # host seconds of each push_frames call in the timed live runs


def live(push, n):
    li.reset()
    if not push:
        li.load_video(canvases[:n])
    else:
        li.push_frames([cam[0]])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        if push and i + 1 < n:
            t = time.perf_counter()
            li.push_frames([cam[(i + 1) % len(cam)]])
            push_s.append(time.perf_counter() - t)
        li.input_video_stream(i / li.frame_fps)
        li()
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def backlog(push, n):
    li.reset()
    if not push:
        li.load_video(canvases[:n])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if push:
        for b0 in range(0, n, 8):
            li.push_frames([cam[k % len(cam)] for k in range(b0, min(n, b0 + 8))])
    li.input_video_stream((n - 1) / li.frame_fps)
    while li.frame_embeds_queue:
        li()
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


live(True, 20), live(False, 20), backlog(True, 16), backlog(False, 16)   # warm-up
pinned = torch.empty(cam[0].numel(), dtype=torch.uint8, pin_memory=True)


def staging(copy):   # us per copy of a 1080p frame into pinned memory
    for _ in range(3):
        copy(cam[0])
    t0 = time.perf_counter()
    for k in range(50):
        copy(cam[k % len(cam)])
    return round(1e6 * (time.perf_counter() - t0) / 50, 1)


staging_us = {"np_copyto": staging(lambda f: np.copyto(pinned.numpy().reshape(f.shape), f.numpy())),
              "torch_copy_": staging(lambda f: pinned.copy_(f.reshape(-1)))}
push_s.clear()
res = {"push": [], "load_video": []}
for _ in range(args.reps):
    for push in (True, False):
        res["push" if push else "load_video"].append(round(live(push, args.frames), 1))
emit("live", {"frames": args.frames, "size": "1920x1080", "frames_per_s": res})
emit("host", {"size": "1920x1080", "torch_threads": torch.get_num_threads(), "staging_copy_us": staging_us,
              "push_frames_call_us": {"median": round(1e6 * float(np.median(push_s)), 1),
                                      "mean": round(1e6 * float(np.mean(push_s)), 1)}})
res = {"push": [], "load_video": []}
for _ in range(args.reps):
    for push in (True, False):
        res["push" if push else "load_video"].append(round(backlog(push, args.backlog), 1))
emit("backlog", {"frames": args.backlog, "size": "1920x1080", "frames_per_s": res})
