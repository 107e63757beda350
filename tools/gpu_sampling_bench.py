"""Dev tool: the cost of sampled responses on the full-size synthetic model.  One JSON line per measurement:
  card      GPU name and power limit (nvidia-smi), read in the same run
  kernel    us per vlo_sample call (parameter upload + sample_kernel) for 1 / 8 / 64 rows at vocab 128 256, back to
            back between two CUDA events: temperature only, top-p 0.9, top-k 50 + top-p 0.9, and with the penalty
  tokens    response tokens/s of one stream at 12k and 66k keys, one token per step with the decision read back after
            each (as the generation loop does), greedy and sampled (T 0.6, top_p 0.9, top_k 50) alternating, three repeats
  drafts    verify steps and accepted drafts of a 100-token response with the n-gram drafter, greedy and sampled.  The
            weights are synthetic: this shows the mechanism, not the acceptance real text would get
  python tools/gpu_sampling_bench.py [--kv 12000 66000] [--tokens 48]"""
import argparse, json, pathlib, subprocess, sys, time

ROOT = pathlib.Path(__file__).resolve().parents[1]
ap = argparse.ArgumentParser()
ap.add_argument("--kv", type=int, nargs="+", default=[12000, 66000])
ap.add_argument("--tokens", type=int, default=48)
args = ap.parse_args()

import torch  # noqa: E402

sys.path.insert(0, str(ROOT))
import vlo_bootstrap  # noqa: E402,F401
from videollm_online_b200 import llama3_8b_siglip_l, weights as W  # noqa: E402
from videollm_online_b200.config import SamplingConfig  # noqa: E402
from videollm_online_b200.engine import Engine, SampleRow  # noqa: E402
from videollm_online_b200.speculative import NgramDrafter, generate_ids  # noqa: E402


def emit(kind, rec):
    print(json.dumps({"what": kind, **rec}), flush=True)


smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
emit("card", {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": smi})

dev = torch.device("cuda:0")
cfg = llama3_8b_siglip_l()
CAP = max(args.kv) + 1024
eng = Engine(cfg, dev, max_streams=1, max_kv_tokens=CAP, max_step_tokens=128, max_vit_batch=1)

# ---- the kernel (vlo_sample needs no weights)
g = torch.Generator().manual_seed(0)
logits = (torch.randn(64, cfg.vocab_size, generator=g) * 3).to(torch.bfloat16).to(dev)
hist = torch.randint(0, cfg.vocab_size, (300,), generator=g).tolist()
variants = {"temperature_only": dict(temperature=0.6), "top_p_0.9": dict(temperature=0.6, top_p=0.9),
            "top_k_50_top_p_0.9": dict(temperature=0.6, top_k=50, top_p=0.9),
            "top_p_0.9_penalty_1.2_300_ids": dict(temperature=0.6, top_p=0.9, repetition_penalty=1.2, penalty_ids=hist)}
for n in (1, 8, 64):
    rec = {}
    for name, kw in variants.items():
        rows = [SampleRow(seed=1, position=1000 + i, **kw) for i in range(n)]
        for _ in range(5):
            eng._sample(logits[:n], rows)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = 200
        a.record()
        for _ in range(iters):
            eng._sample(logits[:n], rows)
        b.record()
        torch.cuda.synchronize()
        rec[name] = round(1e3 * a.elapsed_time(b) / iters, 2)
    emit("kernel", {"rows": n, "vocab": cfg.vocab_size, "us_per_call": rec})

# ---- whole response tokens
eng.load_weights(W.synthetic_engine_weights(cfg, dev, CAP, seed=0))
sid = eng.stream_open()
zeros = torch.zeros(16, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
S = SamplingConfig(do_sample=True, temperature=0.6, top_p=0.9, seed=3)


def run(KV, sampled, n):
    eng.kv_truncate(sid, KV)
    tok, out = 1234, []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        pos = eng.kv_len(sid)
        sample = [SampleRow(S.seed, pos, S.temperature, S.top_k, S.top_p)] if sampled else None
        eng.step([sid], [1], zeros[:1], row_ids=torch.tensor([tok], dtype=torch.int64), sample=sample)
        d = eng.read_decisions(1)[0]
        tok = d.sampled_id if sampled else d.argmax_id
        out.append(tok)
    return n / (time.perf_counter() - t0), out


for KV in args.kv:
    eng.kv_fill_synthetic(sid, KV, seed=7)
    run(KV, False, 4)
    run(KV, True, 4)
    rates = {"greedy": [], "sampled": []}
    for _ in range(3):
        for name in ("greedy", "sampled"):
            rates[name].append(round(run(KV, name == "sampled", args.tokens)[0], 1))
    emit("tokens", {"kv": KV, "tokens_per_s_three_reps": rates,
                    "sampled_over_greedy_ms_per_token": round(1e3 / (sum(rates["sampled"]) / 3) -
                                                             1e3 / (sum(rates["greedy"]) / 3), 3)})

# ---- drafts under sampling (synthetic weights)
KV = min(args.kv)
for name, samp in (("greedy", None), ("sampled_T0.6_top_p0.9", S)):
    eng.kv_truncate(sid, KV)
    steps = []

    def step(ids, drafts, rows=None):
        steps.append(len(drafts))
        r = ids + drafts
        eng.step([sid], [len(r)], zeros[:len(r)], row_ids=torch.tensor(r, dtype=torch.int64),
                 segments=[[len(ids)] + [1] * len(drafts)] if drafts else None, sample=rows)
    t0 = time.perf_counter()
    ids = generate_ids(eng, sid, step, 3, 100, -1, first_ids=[1234, 5678, 91], drafter=NgramDrafter(), base=KV,
                       sampling=samp)
    dt = time.perf_counter() - t0
    emit("drafts", {"kv": KV, "mode": name, "tokens": len(ids), "steps": len(steps), "drafts_offered": sum(steps),
                    "tokens_per_s": round(len(ids) / dt, 1), "distinct_ids": len(set(ids)),
                    "note": "synthetic weights: says nothing about acceptance on real text"})
