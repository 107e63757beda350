"""Dev tool: where the time of one frame step goes, device-timed, in one process.  One JSON line per measurement:
  card        GPU name, power limit, max SM clock (nvidia-smi)
  decoder     the decoder step alone at q = 11 (frame step) and q = 1 (AR step), KV tokens of context
  vit         vlo_vit_encode + connector alone at B = 1 and 2, with the engine's gemm_vit kernel class
  gemm        each trunk GEMM shape (QKV 3072x1024, out 1024x1024, fc1 4096x1024, fc2 1024x4096) at 576 and 1152 rows,
              a micro-loop bracketed once by events: gemm_ws_kernel with 64-token tiles, and for QKV / fc1
              vlo_op_gemm_vit (when the library has it), TFLOP/s
  pipelined   frame steps with the ViT of frame i+1 on a side stream during the decoder step of frame i
  python tools/gpu_frame_breakdown.py [--kv 12000] [--steps 40]"""
import argparse, ctypes as C, json, os, pathlib, subprocess, sys
import torch
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import llama3_8b_siglip_l, weights as W
from videollm_online_b200.engine import Engine

ap = argparse.ArgumentParser()
ap.add_argument("--kv", type=int, default=12000)
ap.add_argument("--steps", type=int, default=40)
ap.add_argument("--gemm-iters", type=int, default=200)
args = ap.parse_args()
lib_name = pathlib.Path(os.environ.get("VLO_LIB", "libvlo_b200.so")).name


def emit(kind, rec):
    print(json.dumps({"what": kind, "lib": lib_name, **rec}), flush=True)


def timed(fn, n, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                   capture_output=True, text=True).stdout.strip().splitlines()
emit("card", {"nvidia_smi": q[0] if q else "unavailable"})

dev = torch.device("cuda:0")
cfg = llama3_8b_siglip_l()
KV = args.kv
eng = Engine(cfg, dev, max_streams=1, max_kv_tokens=KV + 11 * (2 * args.steps + 16) + 2048, max_step_tokens=128, max_vit_batch=2)
eng.load_weights(W.synthetic_engine_weights(cfg, dev, KV + 11 * (2 * args.steps + 16) + 2048, seed=0))
sid = eng.stream_open()
eng.kv_fill_synthetic(sid, KV, seed=7)
S = cfg.frame_resolution
frames = torch.randint(0, 256, (2, 3, S, S), dtype=torch.uint8, device=dev)
packed = torch.zeros(11, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
ids = torch.tensor([cfg.frame_token_interval_id] + [-1] * 10, dtype=torch.int64, device=dev)
one = torch.zeros(1, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
tid = torch.tensor([1234], dtype=torch.int64, device=dev)

# ---- decoder alone (the cache grows by 11 per frame step; truncated back before each measurement)
ms11 = timed(lambda: eng.step([sid], [11], packed, row_ids=ids, want_logits=True), args.steps)
eng.kv_truncate(sid, KV)
ms1 = timed(lambda: eng.step([sid], [1], one, row_ids=tid), 64)
eng.kv_truncate(sid, KV)
emit("decoder", {"kv": KV, "ms_frame_step_q11": round(ms11, 3), "ms_ar_step_q1": round(ms1, 3)})

# ---- ViT + connector alone
C_, M_, P = cfg.vision_hidden_size, cfg.vision_intermediate_size, cfg.num_patches
names = ["gemm_weight_stream", "attn_kvappend", "attn_merge", "gemm_vit", "vit_attn", "other"]
for B in (1, 2):
    ms = timed(lambda: eng.vit_encode(frames[:B]), 20)
    eng.lib.vlo_profile_enable(1)
    eng.vit_encode(frames[:B])
    torch.cuda.synchronize()
    msv, n, by = (C.c_double * 6)(), (C.c_longlong * 6)(), (C.c_double * 6)()
    eng.lib.vlo_profile_read(msv, n, by, 6)
    eng.lib.vlo_profile_enable(0)
    trunk_flop = 24 * B * P * (C_ * 3 * C_ + C_ * C_ + 2 * C_ * M_) * 2
    emit("vit", {"batch": B, "ms_per_call": round(ms, 3),
                 "classes_ms_event_bracketed": {nm: round(msv[j], 3) for j, nm in enumerate(names) if n[j]},
                 "classes_n": {nm: int(n[j]) for j, nm in enumerate(names) if n[j]},
                 "trunk_gemm_tflops_event_bracketed": round(trunk_flop / msv[3] / 1e9, 1) if msv[3] > 0 else None})

# ---- trunk GEMM shapes in isolation
lib = eng.lib
has_vit = hasattr(lib, "vlo_op_gemm_vit")
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
for rows in (576, 1152):
    for name, N, K, mode in (("qkv", 3 * C_, C_, 1), ("out", C_, C_, 0), ("fc1", M_, C_, 1), ("fc2", C_, M_, 0)):
        x = torch.randn(rows, K, device=dev).half()
        w = (torch.randn(N, K, device=dev) * 0.05).half()
        bias = torch.randn(N, device=dev)
        out16 = torch.empty(rows, N, device=dev, dtype=torch.float16)
        planes = torch.empty(8, rows, N, device=dev)
        act = 1 if name == "fc1" else 0
        rec = {"shape": name, "rows": rows, "n": N, "k": K}
        flop = 2.0 * rows * N * K
        variants = [("gemm_ws_bn64", lambda: lib.vlo_op_gemm_ws(0, mode, p(w), N, p(x), rows, K, p(out16 if mode else planes), N,
                                                                  rows * N, p(bias) if mode else None, act, 0, 64, None, st))]
        if has_vit and mode == 1:
            variants.insert(0, ("gemm_vit", lambda: lib.vlo_op_gemm_vit(p(w), N, p(x), rows, K, p(out16), N, p(bias), act, 0, st)))
        for vname, fn in variants:
            def call():
                if fn() != 0:
                    raise RuntimeError(lib.vlo_last_error().decode())
            ms = timed(call, args.gemm_iters)
            rec[vname] = {"us": round(ms * 1e3, 2), "tflops": round(flop / ms / 1e9, 1)}
        emit("gemm", rec)

# ---- pipelined frame steps: ViT of frame i+1 on the side stream during the decoder step of frame i
stream = torch.cuda.current_stream(dev)
side = torch.cuda.Stream(dev)
evs = [torch.cuda.Event(), torch.cuda.Event()]
pre = [torch.cuda.Event(), torch.cuda.Event()]
fes = [None, None]


def encode(i, after):
    if after is None:
        side.wait_stream(stream)
    else:
        side.wait_event(after)
    with torch.cuda.stream(side):
        fes[i & 1] = eng.vit_encode(frames[i % 2:i % 2 + 1])
        evs[i & 1].record(side)


def pipelined(n):
    encode(0, None)
    for i in range(n):
        stream.wait_event(evs[i & 1])
        fe = fes[i & 1]
        fe.record_stream(stream)
        pre[i & 1].record(stream)
        packed[1:] = fe
        eng.step([sid], [11], packed, row_ids=ids, want_logits=True)
        if i + 1 < n:
            encode(i + 1, pre[i & 1])


pipelined(5)
eng.kv_truncate(sid, KV)
torch.cuda.synchronize()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record(stream)
pipelined(args.steps)
b.record(stream)
torch.cuda.synchronize()
ms = a.elapsed_time(b) / args.steps
emit("pipelined", {"kv": KV, "ms_per_frame_step": round(ms, 3), "frames_per_s": round(1e3 / ms, 1)})
