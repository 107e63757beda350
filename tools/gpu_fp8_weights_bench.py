"""Dev tool: FP8 (e4m3) decoder weights, FP8 weights with FP8 activations (W8A8) and int4 weights with per-group scales
(W4A16) against bf16 on the full-size synthetic model (same seed; the quantized engines hold the quantized layer matrices
of the bf16 engine's weights).  The four engines are alternated in one run, REPEATS times.

  card      GPU name and power limit (nvidia-smi), read in the same run
  memory    weight bytes and engine device bytes of each form, and the KV pool tokens / pages the smaller weights free at
            one memory budget (131 072 B per token, 64-token pages), against bf16: one entry per quantized form (these
            fields were scalars for FP8 alone before the int4 arm; nothing in the repository reads the records back)
  gemm      vlo_bench_gemm (the 4 x 32 layer GEMMs, planes only; W8A8: on the e4m3 activation copies; int4: codes and
            group scales) at 11 tokens: ms per pass and algorithmic TB/s
  step      decoder step device ms (CUDA events), median of STEPS, at q = 11 and q = 1, at 12 288 and 66 048 keys
  backlog   one segmented step of 11 frames (11 x 11 rows) at 12 288 keys: decoder ms per frame
  response  1-token steps at 12 288 keys with the host reading each decision (a greedy response's loop): tokens/s
  live      LiveInfer frames/s with the next frame's ViT pipelined, FRAMES frames, silent decisions
One JSON line per part."""
import ctypes as C
import json, pathlib, statistics, subprocess, sys, time
import torch
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import llama3_8b_siglip_l, weights as W
from videollm_online_b200.engine import Engine

dev = torch.device("cuda:0")
cfg = llama3_8b_siglip_l()
KEYS = (12288, 66048)
REPEATS, STEPS, GEMM_ITERS, FRAMES = 3, 30, 20, 300
TOKEN_BYTES, PAGE = 131072, 64
FORMS = ("bf16", "fp8", "w8a8", "int4")


def emit(part, d):
    print(json.dumps({"part": part, **d}), flush=True)


smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
emit("card", {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": smi})

cap = KEYS[-1] + 256
engines, wbytes = {}, {}
for form in FORMS:
    w = {k: v for k, v in W.synthetic_engine_weights(cfg, dev, cap, seed=0, fp8_weights=form in ("fp8", "w8a8"),
                                                     int4_weights=form == "int4").items()
         if not k.startswith("vit.")}
    wbytes[form] = W.engine_weight_bytes(w)
    eng = Engine(cfg, dev, max_streams=1, max_kv_tokens=cap, max_step_tokens=128, max_vit_batch=1,
                 fp8_activations=form == "w8a8")
    eng.load_weights(w)
    assert eng.fp8_weights == (form in ("fp8", "w8a8")) and eng.fp8_activations == (form == "w8a8")
    assert eng.int4_weights == (form == "int4")
    engines[form] = (eng, eng.stream_open())
    del w
    torch.cuda.empty_cache()
freed = {f: wbytes["bf16"] - wbytes[f] for f in FORMS if f != "bf16"}
emit("memory", {"weight_bytes": wbytes, "device_bytes": {f: engines[f][0].device_bytes() for f in FORMS},
                "freed_bytes": freed, "extra_pool_tokens": {f: b // TOKEN_BYTES for f, b in freed.items()},
                "extra_pool_pages": {f: b // (TOKEN_BYTES * PAGE) for f, b in freed.items()}})

ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def timed(fn, n):
    out = []
    for _ in range(n):
        ev0.record()
        fn()
        ev1.record()
        torch.cuda.synchronize()
        out.append(ev0.elapsed_time(ev1))
    return statistics.median(out)


res = {f: [] for f in FORMS}
for _ in range(REPEATS):
    for f in FORMS:
        eng, _sid = engines[f]
        algo, launches = C.c_double(0), C.c_int(0)
        run = lambda: eng.lib.vlo_bench_gemm(eng._h, 11, GEMM_ITERS, C.byref(algo), C.byref(launches), eng._stream())
        run()
        ms = timed(run, 3) / GEMM_ITERS
        res[f].append({"ms_per_pass": ms, "algo_bytes": algo.value, "tb_per_s": algo.value / (ms * 1e-3) / 1e12})
emit("gemm", {"n_tok": 11, "runs": res})


def step_ms(eng, sid, q, kv, segments=None):
    emb = torch.zeros(q, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
    ids = torch.full((q,), -1, dtype=torch.int64, device=dev)
    ids[::11] = cfg.frame_token_interval_id

    def one():
        eng.step([sid], [q], emb, row_ids=ids, want_logits=False, segments=segments)
        eng.kv_truncate(sid, kv)
    one()
    return timed(one, STEPS)


for kv in KEYS:
    res = {f"{f}_q{q}_ms": [] for f in FORMS for q in (11, 1)}
    for f in FORMS:
        eng, sid = engines[f]
        eng.kv_fill_synthetic(sid, kv, seed=1)
    for _ in range(REPEATS):
        for f in FORMS:
            eng, sid = engines[f]
            for q in (11, 1):
                res[f"{f}_q{q}_ms"].append(step_ms(eng, sid, q, kv))
    emit("step", {"keys": kv, **res})

kv = KEYS[0]
res = {f: [] for f in FORMS}
resp = {f: [] for f in FORMS}
for f in FORMS:
    engines[f][0].kv_fill_synthetic(engines[f][1], kv, seed=1)
for _ in range(REPEATS):
    for f in FORMS:
        eng, sid = engines[f]
        res[f].append(step_ms(eng, sid, 121, kv, segments=[[11] * 11]) / 11)
        one = torch.zeros(1, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
        tid = torch.tensor([17], dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(STEPS):
            eng.step([sid], [1], one, row_ids=tid, want_logits=False)
            eng.read_decisions(1)
        resp[f].append(STEPS / (time.perf_counter() - t0))
        eng.kv_truncate(sid, kv)
emit("backlog", {"keys": kv, "frames_per_step": 11, "decoder_ms_per_frame": res})
emit("response", {"keys": kv, "tokens_per_s": resp})

for f in FORMS:
    engines[f][0].close()
del engines
torch.cuda.empty_cache()

from videollm_online_b200.cli import synthetic_clip   # noqa: E402
from videollm_online_b200.config import LiveArguments   # noqa: E402
from videollm_online_b200.inference import LiveInfer   # noqa: E402

lis = {f: LiveInfer(LiveArguments(synthetic_weights=True, device="cuda:0", fp8_weights=f in ("fp8", "w8a8"),
                                  fp8_activations=f == "w8a8", int4_weights=f == "int4")) for f in FORMS}


def silent_frames(dec, n):
    dec.argmax_prob_id, dec.p_interval = cfg.frame_token_interval_id, 1.0
    return dec


clip = synthetic_clip(FRAMES, lis["bf16"].frame_resolution)
res = {f: [] for f in FORMS}
for _ in range(REPEATS):
    for f in FORMS:
        li = lis[f]
        li.decision_hook = silent_frames
        li.reset()
        li.load_video(clip)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(FRAMES):
            li.input_video_stream(i / li.frame_fps)
            li()
        torch.cuda.synchronize()
        res[f].append(FRAMES / (time.perf_counter() - t0))
emit("live", {"frames": FRAMES, "fps": res})
