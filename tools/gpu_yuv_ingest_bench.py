"""Dev tool: YUV camera frames letterboxed on the device (vlo_letterbox_planes, push_frames(pixel_format=...)).  One JSON
line per measurement:
  card     GPU name and power limit (nvidia-smi), read in the same run
  kernel   letterbox_kernel's device time per frame (torch.profiler, 50 launches) for packed RGB, NV12, I420 (yuv420p) and
           YUYV (yuyv422) at 640x480, 1280x720, 1920x1080 and 3840x2160, B = 1 and 8, frames already on the device
  h2d      the copy of one 1920x1080 frame from pinned host memory to the device, RGB (6.22 MB) and NV12 (3.11 MB)
           (CUDA events around --iters copies)
  cv2      cv2.cvtColor(COLOR_YUV2RGB_NV12) of one 1920x1080 frame on this host's CPU: the conversion a caller no longer
           makes before pushing
  live     LiveInfer frames/s over --frames 1920x1080 frames pushed from the CPU in NV12 and in RGB (cvtColor's RGB of the
           same frames), one frame ahead of the one stepped, and from load_video of the same canvases; the three
           alternated --reps times in this run; the full-size synthetic model, every frame silent
  push     the host time of each LiveInfer.push_frames call of the live runs, on the thread that drives the session (host
           clock, no synchronisation): median and mean over every call, NV12 against RGB
  python tools/gpu_yuv_ingest_bench.py [--frames 300] [--reps 3] [--iters 200]"""
import argparse, json, pathlib, subprocess, sys, time
import numpy as np
import torch
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import llama3_8b_siglip_l, weights as W
from videollm_online_b200.engine import Engine
from videollm_online_b200.video_ingest import raw_frame_shape

ap = argparse.ArgumentParser()
ap.add_argument("--frames", type=int, default=300)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--iters", type=int, default=200)
args = ap.parse_args()


def emit(kind, rec):
    print(json.dumps({"what": kind, **rec}), flush=True)


smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
emit("card", {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": smi})

import cv2  # noqa: E402

dev = torch.device("cuda:0")
cfg = llama3_8b_siglip_l()
CAP = 11 * (args.frames + 8) + 2048
eng = Engine(cfg, dev, max_streams=1, max_kv_tokens=CAP, max_step_tokens=128, max_vit_batch=8)
eng.load_weights(W.synthetic_engine_weights(cfg, dev, CAP, seed=0))
g = np.random.default_rng(0)
CODES = {"nv12": cv2.COLOR_YUV2RGB_NV12, "yuv420p": cv2.COLOR_YUV2RGB_I420, "yuyv422": cv2.COLOR_YUV2RGB_YUYV}


def frames_of(W_, H_, fmt, n=8):
    """n frames in fmt ("rgb": cvtColor's RGB of NV12 noise, so the picture has a camera's chroma structure)"""
    shape = raw_frame_shape(W_, H_, "nv12" if fmt == "rgb" else fmt)
    raw = [g.integers(0, 256, shape, dtype=np.uint8) for _ in range(n)]
    return [torch.from_numpy(cv2.cvtColor(f, CODES["nv12"]) if fmt == "rgb" else f) for f in raw]


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


def kernel_us(frames, fmt):
    kw = {} if fmt == "rgb" else dict(pixel_format=fmt)
    for _ in range(5):
        eng.letterbox(frames, **kw)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            eng.letterbox(frames, **kw)
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if "letterbox_kernel" in e.key]
    dt = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0) for e in ev)
    return round(dt / (50 * len(frames)), 2) if ev else None


for W_, H_ in [(640, 480), (1280, 720), (1920, 1080), (3840, 2160)]:
    rec = {}
    for fmt in ("rgb", "nv12", "yuv420p", "yuyv422"):
        on_dev = [f.to(dev) for f in frames_of(W_, H_, fmt)]
        rec[fmt] = {f"B{B}_us_per_frame": kernel_us(on_dev[:B], fmt) for B in (1, 8)}
    emit("kernel", {"size": f"{W_}x{H_}", **rec})

rec = {}
for fmt in ("rgb", "nv12"):
    pinned = frames_of(1920, 1080, fmt, 1)[0].pin_memory()
    dst = torch.empty_like(pinned, device=dev)
    rec[fmt] = {"bytes": pinned.numel(),
                "us_per_frame": round(1e3 * timed(lambda: dst.copy_(pinned, non_blocking=True), args.iters), 2)}
emit("h2d", {"size": "1920x1080", **rec})

nv12_np = [f.numpy() for f in frames_of(1920, 1080, "nv12")]
for f in nv12_np:
    cv2.cvtColor(f, CODES["nv12"])
n = max(50, args.iters)
t0 = time.perf_counter()
for k in range(n):
    cv2.cvtColor(nv12_np[k % len(nv12_np)], CODES["nv12"])
emit("cv2", {"size": "1920x1080", "threads": cv2.getNumThreads(), "nv12_to_rgb_us_per_frame":
             round(1e6 * (time.perf_counter() - t0) / n, 1)})

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
cam = {"nv12": frames_of(1920, 1080, "nv12", 16)}
cam["rgb"] = [torch.from_numpy(cv2.cvtColor(f.numpy(), CODES["nv12"])) for f in cam["nv12"]]
canvases = torch.cat([eng.letterbox([cam["rgb"][k % 16]]) for k in range(args.frames)])   # what the pushed frames become
assert torch.equal(canvases[:16], eng.letterbox(cam["nv12"], pixel_format="nv12")[:16])
push_s = {"nv12": [], "rgb": []}


def live(mode, n):
    li.reset()
    kw = dict(pixel_format="nv12") if mode == "nv12" else {}
    if mode == "load_video":
        li.load_video(canvases[:n])
    else:
        li.push_frames([cam[mode][0]], **kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        if mode != "load_video" and i + 1 < n:
            t = time.perf_counter()
            li.push_frames([cam[mode][(i + 1) % 16]], **kw)
            push_s[mode].append(time.perf_counter() - t)
        li.input_video_stream(i / li.frame_fps)
        li()
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


for mode in ("nv12", "rgb", "load_video"):   # warm-up
    live(mode, 20)
push_s = {"nv12": [], "rgb": []}
res = {"nv12": [], "rgb": [], "load_video": []}
for _ in range(args.reps):
    for mode in res:
        res[mode].append(round(live(mode, args.frames), 1))
emit("live", {"frames": args.frames, "size": "1920x1080", "frames_per_s": res})
emit("push", {"size": "1920x1080", "torch_threads": torch.get_num_threads(),
              **{mode: {"calls": len(v), "median_us": round(1e6 * float(np.median(v)), 1),
                        "mean_us": round(1e6 * float(np.mean(v)), 1)} for mode, v in push_s.items()}})
