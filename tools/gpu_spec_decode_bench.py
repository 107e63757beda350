"""Dev tool: the cost side of verifying drafts, on one stream of the full-size synthetic model at 12k and 66k keys.
One JSON line per measurement:
  card      GPU name and power limit (nvidia-smi), read in the same run
  step      decoder ms per step: a one-token step, and verify steps [last | d1 .. dk] (k = 1, 3, 7, 15 one-token
            segments) with every draft accepted and with every draft rejected; the drafts come from a prior greedy run.
            Device-timed back to back, the cache cut back after each step.  tokens/s if a of the k drafts are accepted:
            (a + 1) / (verify ms)
  attn      the attention alone at kv_end 12k / 66k over 32 separate layer caches (CUDA-event profiler around each
            attention call): k + 1 one-token segments in one packed pass, the same as k + 1 one-token launches, and
            with --parent DIR the parent tree's plan of the same segments (pairs in 2-CTA clusters), alternating A/B
  drafter   host time of NgramDrafter.extend + propose per generated token over a repetitive 60-token answer
  python tools/gpu_spec_decode_bench.py [--kv 12000 66000] [--steps 20] [--parent DIR]"""
import argparse, ctypes as C, json, pathlib, subprocess, sys, time

ROOT = pathlib.Path(__file__).resolve().parents[1]
ap = argparse.ArgumentParser()
ap.add_argument("--kv", type=int, nargs="+", default=[12000, 66000])
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--parent", default=None, help="a built tree of the parent commit, for the attention A/B")
ap.add_argument("--attn-only", dest="attn_only", default=None, help=argparse.SUPPRESS)   # child: library path
args = ap.parse_args()
KS = (1, 3, 7, 15)

import torch  # noqa: E402


def emit(kind, rec):
    print(json.dumps({"what": kind, **rec}), flush=True)


# ---------------------------------------------------------------- attention alone (also the child process of the A/B)
def attn_times(lib_path, kvs, ks, layers=32, reps=3):
    """ms per attention call, {kv: {label: ms}}: 'packed' = k + 1 one-token segments in one call, 'solo' = k + 1
    one-token calls.  Only the C ABI of the parent is used, so the parent library loads too."""
    lib = C.CDLL(lib_path)
    P, I = C.c_void_p, C.c_int
    lib.vlo_op_attn_kvappend_segments.argtypes = [P, P, P, P, I, P, I, C.POINTER(C.c_int32), I, I, I, I, P]
    lib.vlo_op_attn_kvappend_segments.restype = I
    lib.vlo_profile_enable.argtypes = [I]
    lib.vlo_profile_read.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_longlong), C.POINTER(C.c_double), I]
    lib.vlo_last_error.restype = C.c_char_p
    Hq, Hk, D = 32, 8, 128
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = {}
    for kv in kvs:
        nblk = (kv + 63) // 64
        kp = [torch.randn(nblk, Hk, 64, D, device="cuda").bfloat16() for _ in range(layers)]
        vp = [torch.randn(nblk, Hk, 64, D, device="cuda").bfloat16() for _ in range(layers)]
        pt = torch.arange(nblk, dtype=torch.int32, device="cuda")
        q = torch.randn(16, Hq, D, device="cuda").bfloat16()
        o = torch.empty(16, Hq * D, device="cuda", dtype=torch.bfloat16)

        def call(l, segs, end):
            n = sum(segs)
            rc = lib.vlo_op_attn_kvappend_segments(P(q.data_ptr()), P(kp[l].data_ptr()), P(vp[l].data_ptr()),
                                                   P(pt.data_ptr()), nblk, P(o.data_ptr()), len(segs),
                                                   (C.c_int32 * len(segs))(*segs), Hq, Hk, D, end, st)
            assert rc == 0, lib.vlo_last_error()
            assert n <= end

        def timed(fn):
            fn()                                # warm
            lib.vlo_profile_enable(1)
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
            ms, n, by = (C.c_double * 6)(), (C.c_longlong * 6)(), (C.c_double * 6)()
            lib.vlo_profile_read(ms, n, by, 6)
            lib.vlo_profile_enable(0)
            return (ms[1] + ms[2]) / (reps * layers)   # main kernels + merge, per layer

        rec = {}
        for k in ks:
            rec[f"packed_k{k}"] = timed(lambda: [call(l, [1] * (k + 1), kv) for l in range(layers)])
            rec[f"solo_k{k}"] = timed(lambda: [call(l, [1], kv - k + i) for l in range(layers) for i in range(k + 1)])
        out[kv] = rec
        del kp, vp
        torch.cuda.empty_cache()
    return out


if args.attn_only:
    print(json.dumps({str(k): v for k, v in attn_times(args.attn_only, args.kv, (0,) + KS).items()}), flush=True)
    sys.exit(0)

sys.path.insert(0, str(ROOT))
import vlo_bootstrap  # noqa: E402,F401
from videollm_online_b200 import llama3_8b_siglip_l, weights as W  # noqa: E402
from videollm_online_b200.engine import Engine  # noqa: E402
from videollm_online_b200.speculative import NgramDrafter  # noqa: E402

smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
emit("card", {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": smi})

# ---- drafter host cost (no GPU work)
d = NgramDrafter()
hist = ([11, 12, 13] + [-1] * 10) * 2000            # a long session of frames between short token runs
d.extend(hist)
answer = [(i * 7) % 23 + 100 for i in range(20)] * 3
t0 = time.perf_counter()
for t in answer:
    d.propose(15)
    d.extend([t])
dt = time.perf_counter() - t0
emit("drafter", {"history": len(hist), "tokens": len(answer), "us_per_token_extend_propose": round(1e6 * dt / len(answer), 2)})

# ---- whole verify steps
dev = torch.device("cuda:0")
cfg = llama3_8b_siglip_l()
CAP = max(args.kv) + 1024
eng = Engine(cfg, dev, max_streams=1, max_kv_tokens=CAP, max_step_tokens=128, max_vit_batch=1)
eng.load_weights(W.synthetic_engine_weights(cfg, dev, CAP, seed=0))
sid = eng.stream_open()
zeros = torch.zeros(16, cfg.hidden_size, dtype=torch.bfloat16, device=dev)


def step(ids, segs=None):
    eng.step([sid], [len(ids)], zeros[:len(ids)], row_ids=torch.tensor(ids, dtype=torch.int64, device=dev),
             segments=segs)


for KV in args.kv:
    eng.kv_fill_synthetic(sid, KV, seed=7)
    greedy = [1234]                                 # a prior greedy run: the drafts every check below accepts
    for _ in range(16):
        step([greedy[-1]])
        greedy.append(eng.read_decisions(1)[0].argmax_id)
    eng.kv_truncate(sid, KV)
    rec = {}

    def timed(ids, segs):
        for _ in range(3):
            step(ids, segs)
            eng.kv_truncate(sid, KV)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.steps):
            step(ids, segs)
            eng.kv_truncate(sid, KV)                # host bookkeeping only: every step sees the same context
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.steps

    rec["one_token"] = timed([greedy[0]], None)
    exact = True
    for k in KS:
        acc = greedy[:k + 1]
        rej = [greedy[0]] + [(t + 1) % cfg.vocab_size for t in greedy[1:k + 1]]
        rec[f"k{k}_accepted"] = timed(acc, [[1] * (k + 1)])
        step(acc, [[1] * (k + 1)])
        exact &= [x.argmax_id for x in eng.read_decisions(k + 1)] == greedy[1:k + 2]
        eng.kv_truncate(sid, KV)
        rec[f"k{k}_rejected"] = timed(rej, [[1] * (k + 1)])
    tps = {f"k{k}": {f"a{a}": round(1e3 * (a + 1) / rec[f"k{k}_accepted"], 1) for a in sorted({0, 1, k // 2, k})}
           for k in KS}
    emit("step", {"kv": KV, "ms_per_step": {n: round(v, 3) for n, v in rec.items()},
                  "tokens_per_s_by_accepted": tps, "one_token_tokens_per_s": round(1e3 / rec["one_token"], 1),
                  "accepted_decisions_equal_greedy": exact})
del eng
torch.cuda.empty_cache()

# ---- attention alone: this build, and alternately the parent's
me = str(ROOT / "videollm-online_b200" / "libvlo_b200.so")
libs = [("this", me)]
if args.parent:
    libs.append(("parent", str(pathlib.Path(args.parent).resolve() / "videollm-online_b200" / "libvlo_b200.so")))
runs = {}
for rep in range(2):
    for name, path in libs:
        r = subprocess.run([sys.executable, __file__, "--attn-only", path, "--kv", *map(str, args.kv)],
                           capture_output=True, text=True)
        if r.returncode != 0:
            raise SystemExit(r.stdout + r.stderr)
        res = json.loads(r.stdout.strip().splitlines()[-1])
        for kv, rec in res.items():
            for lab, ms in rec.items():
                runs.setdefault(kv, {}).setdefault(f"{name}_{lab}", []).append(round(1e3 * ms, 1))
for kv, rec in runs.items():
    emit("attn", {"kv": int(kv), "us_per_layer_call_two_reps": rec,
                  "note": "packed_k = k+1 one-token segments in one call (this: one packed pass; parent: pairs in "
                          "2-CTA clusters); solo_k = k+1 separate one-token calls; main kernels + merge"})
