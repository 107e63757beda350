"""Dev tool: the decoder step ALONE (no ViT) at a 12k-token cache: q = 11 frame steps and q = 1 AR steps, device-timed.
One JSON line; run once per library build (VLO_LIB) or environment setting (VLO_NO_PDL)."""
import json, os, pathlib, sys
import torch
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import llama3_8b_siglip_l, weights as W
from videollm_online_b200.engine import Engine
dev = torch.device("cuda:0")
cfg = llama3_8b_siglip_l()
KV = int(os.environ.get("KV", "12000"))
eng = Engine(cfg, dev, max_streams=1, max_kv_tokens=KV + 2048, max_step_tokens=128, max_vit_batch=1)
w = W.synthetic_engine_weights(cfg, dev, KV + 2048, seed=0)
eng.load_weights(w)
sid = eng.stream_open()
eng.kv_fill_synthetic(sid, KV, seed=7)
emb = torch.zeros(11, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
ids = torch.tensor([cfg.frame_token_interval_id] + [-1] * 10, dtype=torch.int64, device=dev)
one = torch.zeros(1, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
tid = torch.tensor([1234], dtype=torch.int64, device=dev)
def timed(fn, n, warm=5):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / n
ms11 = timed(lambda: eng.step([sid], [11], emb, row_ids=ids, want_logits=True), 40)
eng.kv_truncate(sid, KV)
ms1 = timed(lambda: eng.step([sid], [1], one, row_ids=tid), 64)
by = 15009316864 + KV * 131072
env = {k: v for k, v in os.environ.items() if k.startswith("VLO_")}
print(json.dumps({"env": env, "kv": KV, "ms_frame_step": round(ms11, 3), "ms_ar_step": round(ms1, 3), "hbm_frac_frame": round(by / ms11 / 1e6 / 6486.8, 3),
                  "hbm_frac_ar": round(by / ms1 / 1e6 / 6486.8, 3)}), flush=True)
