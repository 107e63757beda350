"""Dev tool: a context window that keeps the conversation (`vlo_kv_compact`, `engine.retain_spans`,
`LiveInfer.context_keep_turns`) on the full-size synthetic model.

  card      GPU name and power limit (nvidia-smi), read in the same run
  compact   one vlo_kv_compact at windows of 13 312 and 66 048 tokens over a history of stream messages closed by
            TURNS turns of 40 rows spread evenly through it, dropping what retain_spans drops (window / 8 of old frames): device
            time (CUDA events around the call on its stream) and GB/s of the K and V rows moved (read + write, twice:
            through the staging workspace); next to vlo_kv_evict dropping the same count rounded up to whole pages, and
            the host time of the Python path (retain_spans + Engine.kv_compact + the history update)
  live      LiveInfer frames/s over FRAMES frames with keep-turns, the page window (both LIVE_WINDOW tokens) and no
            window, alternated REPEATS times
One JSON line per part."""
import json, pathlib, subprocess, sys, time
import torch
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import llama3_8b_siglip_l, weights as W
from videollm_online_b200.engine import Engine, kept_rows, retain_spans

dev = torch.device("cuda:0")
cfg = llama3_8b_siglip_l()
WINDOWS = (13312, 66048)
PAGE, REPEATS, TURNS, PROMPT = 64, 3, 20, 64
FRAMES, LIVE_WINDOW = 600, 2048
ROW_BYTES = cfg.num_hidden_layers * 2 * cfg.num_key_value_heads * cfg.head_dim * 2   # one token's K and V, all layers
IID, FNT = cfg.frame_token_interval_id, cfg.frame_num_tokens


def emit(part, d):
    print(json.dumps({"part": part, **d}), flush=True)


def history(n):
    """at most n positions: a prompt, then stream messages closed by TURNS 40-row turns spread evenly, then one open
    message; it ends on a whole frame"""
    h = [1] * PROMPT
    every = max(1, (n - PROMPT) // (TURNS + 1) // (FNT + 1))
    frames = turns = 0
    while True:
        nxt = ([IID] if frames and h[-1] == -1 else []) + [-1] * FNT
        if len(h) + len(nxt) > n:
            return h                        # ends on a whole frame, within n
        h += nxt
        frames += 1
        if frames % every == 0 and turns < TURNS:
            h += [cfg.stream_end_id] + [300] * 37 + [40, 41]
            turns += 1


smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
emit("card", {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": smi})

cap = WINDOWS[-1] + 256
w = {k: v for k, v in W.synthetic_engine_weights(cfg, dev, cap, seed=0).items() if not k.startswith("vit.")}
eng = Engine(cfg, dev, max_streams=2, max_kv_tokens=cap, max_step_tokens=128, max_vit_batch=1, kv_pool_tokens=2 * cap)
eng.load_weights(w)
a = eng.stream_open()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def timed(fn):
    torch.cuda.synchronize()
    ev0.record()
    fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1)


for win in WINDOWS:
    h = history(win)
    spans = retain_spans(h, 1, len(h), PROMPT, IID, FNT)
    kept = sum(n for _, n in spans)
    dropped = len(h) - kept
    moved = kept - spans[0][1]                          # positions after the untouched first span
    res = {"window": win, "kv_len": len(h), "turns": h.count(cfg.stream_end_id), "spans": len(spans),
           "dropped": dropped, "moved": moved, "compact_ms": [], "evict_ms": [], "host_ms": []}
    n_ev = -(-dropped // PAGE) * PAGE
    for r in range(REPEATS):
        eng.kv_fill_synthetic(a, len(h), seed=r)
        res["compact_ms"].append(timed(lambda: eng.kv_compact(a, spans)))
        eng.kv_fill_synthetic(a, len(h), seed=r)
        res["evict_ms"].append(timed(lambda: eng.kv_evict(a, PAGE, n_ev)))
        eng.kv_fill_synthetic(a, len(h), seed=r)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s = eng.kv_retain(a, h, 1, len(h), PROMPT, IID, FNT)
        kept_rows(h, s)
        res["host_ms"].append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize()
    res["compact_gbps"] = [4 * moved * ROW_BYTES / (t * 1e-3) / 1e9 for t in res["compact_ms"]]
    emit("compact", res)

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
modes = {"keep_turns_fps": (LIVE_WINDOW, True), "page_window_fps": (LIVE_WINDOW, False), "no_window_fps": (None, False)}
res = {"frames": FRAMES, "window": LIVE_WINDOW, **{m: [] for m in modes}, "evicted_tokens": {m: [] for m in modes}}
for r in range(REPEATS):
    for m, (win, keep) in modes.items():
        li.reset()
        li.load_video(clip)
        li.context_window = None
        li.context_keep_turns = keep
        li.context_window = win
        li.input_query_stream("Please narrate the video in real time.", video_time=0.0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(FRAMES):
            li.input_video_stream(i / li.frame_fps)
            li()
        torch.cuda.synchronize()
        res[m].append(FRAMES / (time.perf_counter() - t0))
        res["evicted_tokens"][m].append(li.evicted_tokens)
emit("live", res)
