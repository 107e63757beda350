"""Dev tool: long teacher-forced inputs on one stream of the full-size synthetic model, prefill (vlo_prefill) against
the chunked path (max_step_tokens steps).  One JSON line per measurement:
  card      GPU name and power limit (nvidia-smi), read in the same run
  gemm128   the layer GEMMs of one 128-token step (vlo_bench_gemm, all 32 layers), device-timed
  pass      T-token input from kv_len `kv`, prefill and chunked alternated, `reps` repeats each: ms, and the layer-GEMM
            TFLOP/s of the whole pass (2 x layer parameters x T over the pass time); the outputs are checked equal
  evaluate  stream_evaluate on a synthetic conversation of `frames` frames, end to end, prefill and chunked alternated
--form picks the layer matrices: bf16 (the default), or fp8 (e4m3 weights), w8a8 (e4m3 weights and activations) or int4,
which run with quantized_prefill; the chunked path is then the same engine's max_step_tokens steps, and the quantized
forms measure the passes of 1024 and 4096 tokens from an empty cache and 4096 after 12k keys.
  python tools/gpu_prefill_bench.py [--form bf16] [--reps 3] [--frames 1200]"""
import argparse, json, pathlib, subprocess, sys, time
import torch
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import llama3_8b_siglip_l
from videollm_online_b200.engine import Engine
from videollm_online_b200.modeling_live import build_live

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--frames", type=int, default=1200)
ap.add_argument("--form", choices=["bf16", "fp8", "w8a8", "int4"], default="bf16")
args = ap.parse_args()


def emit(kind, rec):
    print(json.dumps({"what": kind, **rec}), flush=True)


smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
emit("card", {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": smi, "form": args.form})

dev = torch.device("cuda:0")
cfg = llama3_8b_siglip_l()
CAP = 12000 + 13200 + 1024
quant = args.form != "bf16"
a8 = args.form == "w8a8"
model, _ = build_live(config=cfg, synthetic_weights=True, set_vision_inside=False, device="cuda:0", max_streams=2,
                      max_kv_tokens=CAP, max_step_tokens=128, max_vit_batch=1, fp8_weights=args.form in ("fp8", "w8a8"),
                      fp8_activations=a8, int4_weights=args.form == "int4", quantized_prefill=quant)
eng = model.engine
H, I, A = cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads * cfg.head_dim
QKV = (cfg.num_attention_heads + 2 * cfg.num_key_value_heads) * cfg.head_dim
layer_params = cfg.num_hidden_layers * (QKV * H + H * A + 2 * I * H + H * I)
fresh = Engine(cfg, dev, max_streams=2, max_kv_tokens=CAP, max_step_tokens=128, max_vit_batch=1, fp8_activations=a8)
emit("engine", {"form": args.form, "device_bytes": eng.device_bytes(), "max_prefill_tokens": eng.max_prefill_tokens,
                "prefill_workspace_bytes": eng.device_bytes() - fresh.device_bytes()})   # grown by finalize
fresh.close()
PREFILL = Engine.prefills


def chunked(on):
    Engine.prefills = PREFILL if not on else property(lambda self: False)


def timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


# ---- layer GEMMs of one 128-token step
import ctypes as C  # noqa: E402
bytes_ = C.c_double()
launches = C.c_int()
eng.lib.vlo_bench_gemm(eng._h, 128, 2, C.byref(bytes_), C.byref(launches), eng._stream())
ms, _ = timed(lambda: eng.lib.vlo_bench_gemm(eng._h, 128, 10, C.byref(bytes_), C.byref(launches), eng._stream()))
emit("gemm128", {"form": args.form, "ms_per_step": ms / 10, "algo_GB": bytes_.value / 1e9, "TB_per_s": bytes_.value / (ms / 10) / 1e9})

# ---- whole passes
sid = eng.stream_open()
g = torch.Generator(device=dev).manual_seed(0)
PASSES = [(1024, 0), (4096, 0), (4096, 12000)] + ([] if quant else [(13200, 0), (13200, 12000)])
for T, kv in PASSES:
    emb = (torch.randn(T, H, device=dev, generator=g) * 0.02).bfloat16()
    rec = {"form": args.form, "T": T, "kv": kv, "prefill_ms": [], "chunked_ms": []}
    outs = {}
    for r in range(args.reps + 1):            # the first round warms both paths up
        for mode in ("prefill", "chunked"):
            chunked(mode == "chunked")
            eng.stream_reset(sid)
            if kv:
                eng.kv_fill_synthetic(sid, kv, seed=3)
            ms, (lg, dc) = timed(lambda: eng.step([sid], [T], emb))
            outs[mode] = (lg[0].clone(), dc[0].clone())
            if r:
                rec[mode + "_ms"].append(round(ms, 3))
    chunked(False)
    rec["same_logits_and_decision"] = bool(torch.equal(outs["prefill"][0], outs["chunked"][0]) and
                                           torch.equal(outs["prefill"][1], outs["chunked"][1]))
    for mode in ("prefill", "chunked"):
        best = min(rec[mode + "_ms"])
        rec[mode + "_layer_gemm_TFLOPs_per_s"] = round(2.0 * layer_params * T / (best * 1e-3) / 1e12, 1)
    emit("pass", rec)
eng.stream_close(sid)

# ---- stream_evaluate on a synthetic conversation
fnt, v = cfg.frame_num_tokens, cfg.v_placeholder_id
ids, labels = [], []
gc = torch.Generator().manual_seed(1)
for f in range(args.frames):
    ids += [v] * fnt
    labels += [-100] * (fnt - 1) + [cfg.frame_token_interval_id]
    if f % 100 == 99:
        words = torch.randint(1000, 20000, (15,), generator=gc).tolist() + [cfg.eos_token_id]
        labels[-1] = words[0]
        ids += words
        labels += words[1:] + [-100]
input_ids, label_ids = torch.tensor([ids], device=dev), torch.tensor([labels], device=dev)
feats = (torch.randn(args.frames, fnt, cfg.vision_hidden_size, generator=gc) * 0.5).to(dev)
# the engine's connector takes max_vit_batch frames per call
model.visual_embed = lambda f: torch.cat([eng.connector(f[i:i + eng.max_vit_batch]) for i in range(0, f.shape[0], eng.max_vit_batch)])
rec = {"form": args.form, "frames": args.frames, "tokens": len(ids), "prefill_s": [], "chunked_s": []}
res = {}
for r in range(args.reps + 1):
    for mode in ("prefill", "chunked"):
        chunked(mode == "chunked")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res[mode] = model.stream_evaluate(input_ids, label_ids, feats).cpu()
        torch.cuda.synchronize()
        if r:
            rec[mode + "_s"].append(round(time.perf_counter() - t0, 3))
chunked(False)
rec["same_metrics"] = bool(torch.equal(res["prefill"], res["chunked"]))
emit("evaluate", rec)
