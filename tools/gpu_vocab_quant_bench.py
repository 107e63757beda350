"""Dev tool: quantized vocabulary matrices (embed and lm_head in the layers' int4 or e4m3 form) against bf16 ones, on the
full-size synthetic model (same seed; the quantized tables are those of the bf16 engine's weights).  The engines are
alternated in one run, REPEATS times.

  card      GPU name and power limit (nvidia-smi), read in the same run
  memory    weight bytes, engine device bytes and the KV pool tokens / pages the quantized vocabulary matrices free
            (131 072 B per token, 64-token pages), per layer form
  lm_head   kernel time of one lm_head launch (torch.profiler, device time of the GEMM kernel over LAUNCHES launches) at
            1, 11 and 128 rows for bf16, e4m3 and int4 weights, and the bytes/s each reaches (weights + activations)
  step      decoder step device ms (CUDA events), median of STEPS, at q = 11 and q = 1, at 12 288 keys
  response  1-token steps at 12 288 keys with the host reading each decision: tokens/s
  stats     64 frame steps of 11 rows at 12 288 keys: logits of each quantized-vocabulary engine against the engine of the
            same layer form with bf16 vocabulary matrices (rms difference, correlation, argmax and speak / silent agreement)
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
KEYS = 12288
REPEATS, STEPS, LAUNCHES, FRAMES, STAT_STEPS = 3, 30, 50, 300, 64
TOKEN_BYTES, PAGE = 131072, 64
FORMS = ("int4", "int4_qv", "fp8", "fp8_qv")


def emit(part, d):
    print(json.dumps({"part": part, **d}), flush=True)


def flags(form):
    return dict(int4_weights=form.startswith("int4"), fp8_weights=form.startswith("fp8"), quantize_vocab=form.endswith("_qv"))


smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
emit("card", {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": smi})

# ---- lm_head kernels alone, on the synthetic lm_head of Llama-3-8B's shape
V, H = cfg.vocab_size, cfg.hidden_size
lib = None
g = torch.Generator(device=dev).manual_seed(0)
w = (torch.randn(V, H, device=dev, generator=g) * 0.02).bfloat16()
q4, s4 = W.quantize_int4_groups(w)
i4 = W.pack_int4_codes(q4)
f8, s8 = W.quantize_fp8_rows(w)
del q4
from videollm_online_b200 import _lib   # noqa: E402
lib = _lib.load()
x_all = torch.randn(128, H, device=dev, generator=g).bfloat16()
out = torch.empty(128, V, dtype=torch.bfloat16, device=dev)
st = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)   # noqa: E731
p = lambda t: C.c_void_p(t.data_ptr())   # noqa: E731


def launch(fmt, T):
    x = x_all[:T]
    if fmt == "bf16":
        return lambda: lib.vlo_op_gemm_ws(1, 1, p(w), V, p(x), T, H, p(out), V, 0, None, 0, 0, 0, None, st())
    wq, sc, f = (i4, s4, 4) if fmt == "int4" else (f8, s8, 2)
    return lambda: lib.vlo_op_gemm_ws_tiles_q(f, p(wq), p(sc), V, p(x), T, H, p(out), V, 0, None, st())


def weight_bytes(fmt):
    return {"bf16": 2.0 * V * H, "e4m3": 1.0 * V * H + 4.0 * V, "int4": i4.numel() + 2.0 * s4.numel()}[fmt]


res = {}
for _ in range(REPEATS):
    for fmt in ("bf16", "e4m3", "int4"):
        for T in (1, 11, 128):
            fn = launch(fmt, T)
            assert fn() == 0
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(LAUNCHES):
                    fn()
                torch.cuda.synchronize()
            ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "gemm_ws" in e.name]
            assert len(ev) == LAUNCHES, len(ev)
            us = statistics.median(e.device_time for e in ev)
            byts = weight_bytes(fmt) + 2.0 * T * H
            res.setdefault(f"{fmt}_T{T}", []).append({"us": us, "gb_per_s": byts / (us * 1e-6) / 1e9})
emit("lm_head", {"launches": LAUNCHES, "runs": res})
del w, i4, s4, f8, s8, out
torch.cuda.empty_cache()

# ---- engines
cap = KEYS + STAT_STEPS * 11 + 256
engines, wbytes = {}, {}
for form in FORMS:
    wt = {k: v for k, v in W.synthetic_engine_weights(cfg, dev, cap, seed=0, **flags(form)).items()
          if not k.startswith("vit.")}
    wbytes[form] = W.engine_weight_bytes(wt)
    eng = Engine(cfg, dev, max_streams=1, max_kv_tokens=cap, max_step_tokens=128, max_vit_batch=1)
    eng.load_weights(wt)
    assert eng.quantized_vocab == form.endswith("_qv")
    engines[form] = (eng, eng.stream_open())
    del wt
    torch.cuda.empty_cache()
freed = {f: wbytes[f.replace("_qv", "")] - wbytes[f] for f in FORMS if f.endswith("_qv")}
emit("memory", {"weight_bytes": wbytes, "device_bytes": {f: engines[f][0].device_bytes() for f in FORMS},
                "freed_bytes": freed, "extra_pool_tokens": {f: b // TOKEN_BYTES for f, b in freed.items()},
                "extra_pool_pages": {f: b // (TOKEN_BYTES * PAGE) for f, b in freed.items()}})

ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def timed(fn, n):
    t = []
    for _ in range(n):
        ev0.record()
        fn()
        ev1.record()
        torch.cuda.synchronize()
        t.append(ev0.elapsed_time(ev1))
    return statistics.median(t)


def step_ms(eng, sid, q, kv):
    emb = torch.zeros(q, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
    ids = torch.full((q,), -1, dtype=torch.int64, device=dev)
    ids[0] = cfg.frame_token_interval_id

    def one():
        eng.step([sid], [q], emb, row_ids=ids, want_logits=False)
        eng.kv_truncate(sid, kv)
    one()
    return timed(one, STEPS)


for f in FORMS:
    engines[f][0].kv_fill_synthetic(engines[f][1], KEYS, seed=1)
res = {f"{f}_q{q}_ms": [] for f in FORMS for q in (11, 1)}
resp = {f: [] for f in FORMS}
for _ in range(REPEATS):
    for f in FORMS:
        eng, sid = engines[f]
        for q in (11, 1):
            res[f"{f}_q{q}_ms"].append(step_ms(eng, sid, q, KEYS))
        one = torch.zeros(1, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
        tid = torch.tensor([17], dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(STEPS):
            eng.step([sid], [1], one, row_ids=tid, want_logits=False)
            eng.read_decisions(1)
        resp[f].append(STEPS / (time.perf_counter() - t0))
        eng.kv_truncate(sid, KEYS)
emit("step", {"keys": KEYS, **res})
emit("response", {"keys": KEYS, "tokens_per_s": resp})

# ---- statistics: the same frame steps on every engine
logits, speak = {}, {}
for f in FORMS:
    eng, sid = engines[f]
    gen = torch.Generator().manual_seed(6)
    lg_all, sp = [], []
    for s in range(STAT_STEPS):
        emb = (torch.randn(11, cfg.hidden_size, generator=gen) * 0.02).bfloat16().to(dev)
        ids = torch.full((11,), -1, dtype=torch.int64)
        ids[0] = cfg.frame_token_interval_id
        lg, _ = eng.step([sid], [11], emb, row_ids=ids)
        lg_all.append(lg[0].float().cpu())
        d = eng.read_decisions(1)[0]
        sp.append(d.next_id(cfg.frame_token_interval_id, 0.725) != cfg.frame_token_interval_id)
    logits[f], speak[f] = torch.stack(lg_all), sp
for f in ("int4", "fp8"):
    a, b = logits[f], logits[f + "_qv"]
    d = b - a
    emit("stats", {"form": f, "steps": STAT_STEPS, "keys": KEYS, "q": 11,
                   "logit_rms_diff": d.pow(2).mean().sqrt().item(), "logit_rms": a.pow(2).mean().sqrt().item(),
                   "corr": torch.corrcoef(torch.stack([a.flatten(), b.flatten()]))[0, 1].item(),
                   "argmax_agree": (a.argmax(-1) == b.argmax(-1)).float().mean().item(),
                   "speak_agree": sum(x == y for x, y in zip(speak[f], speak[f + "_qv"])) / STAT_STEPS,
                   "speak_steps": [sum(speak[f]), sum(speak[f + "_qv"])]})

for f in FORMS:
    engines[f][0].close()
del engines
torch.cuda.empty_cache()

# ---- LiveInfer
from videollm_online_b200.cli import synthetic_clip   # noqa: E402
from videollm_online_b200.config import LiveArguments   # noqa: E402
from videollm_online_b200.inference import LiveInfer   # noqa: E402

lis = {f: LiveInfer(LiveArguments(synthetic_weights=True, device="cuda:0", **flags(f))) for f in FORMS}


def silent_frames(dec, n):
    dec.argmax_prob_id, dec.p_interval = cfg.frame_token_interval_id, 1.0
    return dec


clip = synthetic_clip(FRAMES, lis["int4"].frame_resolution)
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
