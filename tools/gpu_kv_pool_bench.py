"""Dev tool: 8 streams at 12k tokens + 1 stream at 66k tokens in ONE engine with a shared KV page pool, against the
same two workloads on two engines with the default (max_streams x max_kv_tokens) reservation.  Decoder frame steps
(11 tokens per stream, no ViT), device-timed, pooled and separate setups alternating.  One JSON line."""
import json, pathlib, subprocess, sys
import torch
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import llama3_8b_siglip_l, weights as W
from videollm_online_b200.engine import Engine

dev = torch.device("cuda:0")
cfg = llama3_8b_siglip_l()
KV8, KV66, N8, STEPS, REPEATS = 12000, 66000, 8, 20, 3
CAP8, CAP66 = KV8 + 256, KV66 + 512
w = {k: v for k, v in W.synthetic_engine_weights(cfg, dev, CAP66, seed=0).items() if not k.startswith("vit.")}
free0 = torch.cuda.mem_get_info(dev)[0]


def engine(**kw):
    e = Engine(cfg, dev, max_step_tokens=128, max_vit_batch=1, **kw)
    e.load_weights(w)
    return e


pooled = engine(max_streams=N8 + 1, max_kv_tokens=CAP66, kv_pool_tokens=N8 * CAP8 + CAP66)
sep8, sep66 = engine(max_streams=N8, max_kv_tokens=CAP8), engine(max_streams=1, max_kv_tokens=CAP66)
free1 = torch.cuda.mem_get_info(dev)[0]
# pooled: the 66k stream's pages interleave with the 8 short streams' (fill the 66k stream in slices)
p8 = [pooled.stream_open() for _ in range(N8)]
p66 = pooled.stream_open()
for part in range(1, 13):   # the fill hashes logical positions: growing in slices gives the same contents
    for i, s in enumerate(p8):
        pooled.kv_fill_synthetic(s, KV8 * part // 12, seed=100 + i)
    pooled.kv_fill_synthetic(p66, KV66 * part // 12, seed=66)
s8 = [sep8.stream_open() for _ in range(N8)]
for i, s in enumerate(s8):
    sep8.kv_fill_synthetic(s, KV8, seed=100 + i)
s66 = sep66.stream_open()
sep66.kv_fill_synthetic(s66, KV66, seed=66)

emb8 = torch.zeros(11 * N8, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
emb1 = torch.zeros(11, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
ids8 = torch.tensor(([cfg.frame_token_interval_id] + [-1] * 10) * N8, dtype=torch.int64, device=dev)
ids1 = ids8[:11].clone()


def timed(eng, sids, kv, emb, ids):
    def run():
        eng.step(sids, [11] * len(sids), emb, row_ids=ids, want_logits=True)
    for _ in range(3):
        run()
    for s in sids:
        eng.kv_truncate(s, kv)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(STEPS):
        run()
    b.record()
    torch.cuda.synchronize()
    for s in sids:
        eng.kv_truncate(s, kv)
    return STEPS * len(sids) / (a.elapsed_time(b) / 1e3)


res = {k: [] for k in ("pooled_8x12k", "separate_8x12k", "pooled_66k", "separate_66k")}
for _ in range(REPEATS):
    res["pooled_8x12k"].append(timed(pooled, p8, KV8, emb8, ids8))
    res["separate_8x12k"].append(timed(sep8, s8, KV8, emb8, ids8))
    res["pooled_66k"].append(timed(pooled, [p66], KV66, emb1, ids1))
    res["separate_66k"].append(timed(sep66, [s66], KV66, emb1, ids1))
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({
    "gpu": torch.cuda.get_device_name(dev), "nvidia_smi_name_power_limit": smi,
    "frames_per_s": {k: [round(x, 1) for x in v] for k, v in res.items()},
    "device_bytes": {"pooled": pooled.device_bytes(), "separate": sep8.device_bytes() + sep66.device_bytes()},
    "pool": pooled.kv_pool_info(),
    "free_bytes_after_weights": free0, "free_bytes_after_all_three_engines": free1,
    "note": f"frame step = 11 tokens per stream, decoder only; {STEPS} steps per sample, pooled / separate alternating",
}), flush=True)
