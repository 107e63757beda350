"""Dev tool: context-window eviction (`vlo_kv_evict`, `Engine.kv_make_room`, `LiveInfer.context_window`) on the
full-size synthetic model.

  card      GPU name and power limit (nvidia-smi), read in the same run
  evict     one vlo_kv_evict at windows of 13 312 (1200 frames) and 66 048 tokens, each dropping window / 8 after a
            one-page sink: device time (CUDA events around the call on its stream) and GB/s of the re-rotation
            (2 x kept tokens x 64 KB of K)
  step      the 11-token frame step at the same kv_len (window - window / 8) on a stream filled in order and on one
            whose table has the hole an eviction leaves: device ms per step, median of STEPS
  host      host time of the Python eviction path (Engine.kv_make_room + NgramDrafter.drop over a window-long history)
  live      LiveInfer frames/s over FRAMES frames with a window of LIVE_WINDOW tokens (several evictions) and without,
            alternated REPEATS times
One JSON line per part."""
import json, pathlib, statistics, subprocess, sys, time
import torch
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import llama3_8b_siglip_l, weights as W
from videollm_online_b200.engine import Engine, evict_span
from videollm_online_b200.speculative import SEP, NgramDrafter

dev = torch.device("cuda:0")
cfg = llama3_8b_siglip_l()
WINDOWS = (13312, 66048)
PAGE, REPEATS, STEPS = 64, 3, 30
FRAMES, LIVE_WINDOW = 600, 2048
K_BYTES = cfg.num_hidden_layers * cfg.num_key_value_heads * cfg.head_dim * 2   # one token's K, all layers


def emit(part, d):
    print(json.dumps({"part": part, **d}), flush=True)


smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
emit("card", {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": smi})

cap = WINDOWS[-1] + 256
w = {k: v for k, v in W.synthetic_engine_weights(cfg, dev, cap, seed=0).items() if not k.startswith("vit.")}
eng = Engine(cfg, dev, max_streams=3, max_kv_tokens=cap, max_step_tokens=128, max_vit_batch=1,
             kv_pool_tokens=3 * cap)
eng.load_weights(w)
a, b = eng.stream_open(), eng.stream_open()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

for win in WINDOWS:
    first, n = evict_span(win, 1, win, PAGE, PAGE)
    kept = win - first - n
    ms = []
    for r in range(REPEATS):
        eng.kv_fill_synthetic(a, win, seed=r)
        torch.cuda.synchronize()
        ev0.record()
        eng.kv_evict(a, first, n)
        ev1.record()
        torch.cuda.synchronize()
        ms.append(ev0.elapsed_time(ev1))
    emit("evict", {"window": win, "dropped": n, "kept_after_drop": kept, "ms": ms,
                   "gbps": [2 * kept * K_BYTES / (t * 1e-3) / 1e9 for t in ms]})

emb = torch.zeros(11, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
ids = torch.tensor([cfg.frame_token_interval_id] + [-1] * 10, dtype=torch.int64, device=dev)


def step_ms(sid):
    kv = eng.kv_len(sid)
    out = []
    for _ in range(STEPS):
        ev0.record()
        eng.step([sid], [11], emb, row_ids=ids, want_logits=False)
        ev1.record()
        eng.read_decisions(1)
        out.append(ev0.elapsed_time(ev1))
        eng.kv_truncate(sid, kv)
    return statistics.median(out)


for win in WINDOWS:
    first, n = evict_span(win, 1, win, PAGE, PAGE)
    eng.kv_fill_synthetic(a, win - n, seed=1)           # in order
    eng.kv_fill_synthetic(b, win, seed=1)
    eng.kv_evict(b, first, n)                            # the same length, with a hole in its table
    assert eng.kv_len(a) == eng.kv_len(b)
    res = {"window": win, "kv_len": win - n, "in_order_ms": [], "after_eviction_ms": []}
    for _ in range(REPEATS):
        res["in_order_ms"].append(step_ms(a))
        res["after_eviction_ms"].append(step_ms(b))
    emit("step", res)

for win in WINDOWS:
    host = []
    for r in range(REPEATS):
        eng.kv_fill_synthetic(a, win, seed=r)
        d = NgramDrafter()
        d.extend(([cfg.frame_token_interval_id] + [SEP] * 10) * (win // 11) + [SEP] * (win % 11))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = eng.kv_make_room(a, 1, win, PAGE)
        d.drop(PAGE, n)
        host.append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize()
    emit("host", {"window": win, "ms": host})

del eng, w
torch.cuda.empty_cache()

from videollm_online_b200.cli import synthetic_clip   # noqa: E402
from videollm_online_b200.config import LiveArguments   # noqa: E402
from videollm_online_b200.inference import LiveInfer   # noqa: E402

li = LiveInfer(LiveArguments(synthetic_weights=True, device="cuda:0"))
# random weights never emit the "]\n" protocol id: frames are kept silent, so the only response is the one the query at
# t = 0 asks for (its ids are the model's own)
responding = [False]
respond = li._call_for_response


def call_for_response(*a):
    responding[0] = True
    try:
        return respond(*a)
    finally:
        responding[0] = False


def silent_frames(dec, n):
    if not responding[0]:
        dec.argmax_prob_id, dec.p_interval = cfg.frame_token_interval_id, 1.0
    return dec


li._call_for_response = call_for_response
li.decision_hook = silent_frames
clip = synthetic_clip(FRAMES, li.frame_resolution)
li.load_video(clip)
res = {"frames": FRAMES, "window": LIVE_WINDOW, "with_window_fps": [], "without_fps": [], "evicted_tokens": []}
for r in range(2 * REPEATS):
    windowed = r % 2 == 1
    li.reset()
    li.load_video(clip)
    li.context_window = LIVE_WINDOW if windowed else None
    li.input_query_stream("Please narrate the video in real time.", video_time=0.0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(FRAMES):
        li.input_video_stream(i / li.frame_fps)
        li()
    torch.cuda.synchronize()
    fps = FRAMES / (time.perf_counter() - t0)
    if windowed:
        res["with_window_fps"].append(fps)
        res["evicted_tokens"].append(li.evicted_tokens)
    else:
        res["without_fps"].append(fps)
emit("live", res)
