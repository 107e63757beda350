"""Dev tool: a backlog of queued frames on one stream of the full-size synthetic model, at 12k and at 66k keys of
context.  One JSON line per measurement:
  card      GPU name and power limit (nvidia-smi), read in the same run
  decoder   decoder ms per frame: one frame per step (11 tokens) against segmented steps of K = 2, 4, 8, 11 frames
            (vlo_step_segments), device-timed back to back with the cache cut back after each step
  attn      the attention of those steps (both attention kernels as one class): per-launch time and algorithmic bytes of the KV-append attention and the merge
            (CUDA-event profiler, which brackets every launch and so removes the PDL overlap of a real step)
  backlog   end to end through LiveInfer with the ViT: the whole backlog queued (input_video_stream of the last frame,
            which encodes every frame), then drained; frames/s with a scripted speak every 20th frame and with none,
            segmented steps against one frame per step
  python tools/gpu_frame_backlog_bench.py [--kv 12000 66000] [--frames 110] [--steps 20]"""
import argparse, ctypes as C, json, pathlib, subprocess, sys, time
import torch
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import llama3_8b_siglip_l, weights as W
from videollm_online_b200.engine import Engine

ap = argparse.ArgumentParser()
ap.add_argument("--kv", type=int, nargs="+", default=[12000, 66000])
ap.add_argument("--frames", type=int, default=110)
ap.add_argument("--steps", type=int, default=20)
args = ap.parse_args()


def emit(kind, rec):
    print(json.dumps({"what": kind, **rec}), flush=True)


smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
emit("card", {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": smi})

dev = torch.device("cuda:0")
cfg = llama3_8b_siglip_l()
IID, FR = cfg.frame_token_interval_id, 10
CAP = max(args.kv) + 11 * (args.frames + 64) + 1024
eng = Engine(cfg, dev, max_streams=1, max_kv_tokens=CAP, max_step_tokens=128, max_vit_batch=8)
eng.load_weights(W.synthetic_engine_weights(cfg, dev, CAP, seed=0))
sid = eng.stream_open()
KS = (1, 2, 4, 8, 11)
emb = torch.randn(11 * 11, cfg.hidden_size, device=dev).bfloat16() * 0.02
ids = torch.tensor(([IID] + [-1] * FR) * 11, dtype=torch.int64, device=dev)
names = ["gemm_weight_stream", "attn_kvappend", "attn_merge", "gemm_vit", "vit_attn", "other"]


def step(k):
    T = 11 * k
    eng.step([sid], [T], emb[:T], row_ids=ids[:T], segments=[[11] * k] if k > 1 else None)


for KV in args.kv:
    eng.kv_fill_synthetic(sid, KV, seed=7)
    rec, attn = {}, {}
    for k in KS:
        for _ in range(3):
            step(k)
            eng.kv_truncate(sid, KV)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.steps):
            step(k)
            eng.kv_truncate(sid, KV)    # host bookkeeping only: every step sees the same context
        b.record()
        torch.cuda.synchronize()
        rec[f"K{k}"] = round(a.elapsed_time(b) / (args.steps * k), 3)
        eng.lib.vlo_profile_enable(1)
        step(k)
        torch.cuda.synchronize()
        ms, n, by = (C.c_double * 6)(), (C.c_longlong * 6)(), (C.c_double * 6)()
        eng.lib.vlo_profile_read(ms, n, by, 6)
        eng.lib.vlo_profile_enable(0)
        eng.kv_truncate(sid, KV)
        attn[f"K{k}"] = {nm: {"us_per_launch": round(1e3 * ms[j] / n[j], 1), "algo_bytes_per_launch": int(by[j] / n[j])}
                         for j, nm in enumerate(names[1:3], 1) if n[j]}
    emit("decoder", {"kv": KV, "ms_per_frame": rec, "speedup_K11": round(rec["K1"] / rec["K11"], 2)})
    emit("attn", {"kv": KV, "per_launch": attn, "note": "one work item per frame segment; pairs with the same split grid share a cache pass (cluster kernel)"})

# ---- end to end through LiveInfer: the ViT of the backlog included
from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT
from videollm_online_b200.inference import LiveInfer
from videollm_online_b200.modeling_live import LiveLlamaForCausalLM, StreamKV
from videollm_online_b200.tokenization_live import ByteTokenizer

model = LiveLlamaForCausalLM(cfg, eng)
S = cfg.frame_resolution
clip = torch.randint(0, 256, (args.frames, 3, S, S), dtype=torch.uint8, device=dev)
li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT), model=model, tokenizer=ByteTokenizer(cfg),
               stream=StreamKV(eng, sid))
state = {"resp": False, "frames": 0, "speak_every": 0}
respond = li._call_for_response


def call_for_response(*a):
    state["resp"] = True
    try:
        return respond(*a)
    finally:
        state["resp"] = False


def hook(dec, n):   # frames speak ("]\n") every `speak_every`-th decision, a response is one EOS token
    if state["resp"]:
        t = cfg.eos_token_id
    else:
        state["frames"] += 1
        every = state["speak_every"]
        t = cfg.stream_end_id if every and state["frames"] % every == 0 else IID
    dec.argmax_id = dec.argmax_prob_id = t
    dec.p_interval = 1.0 if t == IID else 0.0
    if t != IID:
        dec.argmax_excl_id = t
    return dec


li._call_for_response = call_for_response
li.decision_hook = hook
backlog_run = li._backlog_run


def drain(KV, every, segmented):
    li.reset()
    li.load_video(clip)
    eng.kv_fill_synthetic(sid, KV, seed=7)
    li.past_key_values, li.last_ids = li._kv, torch.tensor([[IID]])
    state.update(frames=0, speak_every=every)
    li._backlog_run = backlog_run if segmented else (lambda: 1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    li.input_video_stream((args.frames - 1) / li.frame_fps)
    responses = 0
    while li.frame_embeds_queue:
        responses += li()[1] is not None
    torch.cuda.synchronize()
    return args.frames / (time.perf_counter() - t0), responses


drain(args.kv[0], 0, True)    # warm-up
for KV in args.kv:
    for every in (0, 20):
        r = {}
        for mode, seg in (("one_frame_per_step", False), ("segmented", True), ("one_frame_per_step_2", False),
                          ("segmented_2", True)):
            r[mode] = drain(KV, every, seg)
        emit("backlog", {"kv": KV, "frames": args.frames, "speak_every": every or None,
                         "frames_per_s": {m: round(v[0], 1) for m, v in r.items()},
                         "responses": {m: v[1] for m, v in r.items()}})
