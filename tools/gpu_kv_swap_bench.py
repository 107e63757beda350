"""Dev tool: KV swap to pinned host memory (`Engine.kv_swap_out` / `kv_swap_in`) on the full-size synthetic model.

1. Swap-out and swap-in of one stream at 1k, 12k and 66k tokens: device time (CUDA events around the call on its
   stream), GB/s of the image, and the host time of the Python call alone (it returns before the copies end).
2. The 8-stream frame tick at 12k keys (one ragged step of 8 x 11 tokens + the decision read-back, as StreamScheduler
   runs it), alone and while a ninth 12k session swaps out and back in on a side CUDA stream over and over; the two
   alternate, REPEATS samples each.  The 8 streams are truncated back after every tick, so the step never takes a page
   and never waits for a swap-out's copies: the number shows the interference of the copies alone.
One JSON line."""
import json, pathlib, statistics, subprocess, sys, time
import torch
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import llama3_8b_siglip_l, weights as W
from videollm_online_b200.engine import Engine

dev = torch.device("cuda:0")
cfg = llama3_8b_siglip_l()
KV8, N8, TICKS, REPEATS = 12000, 8, 30, 3
SIZES = (1000, 12000, 66000)
CAP8, CAP66 = KV8 + 256, 66000 + 256
w = {k: v for k, v in W.synthetic_engine_weights(cfg, dev, CAP66, seed=0).items() if not k.startswith("vit.")}
eng = Engine(cfg, dev, max_streams=N8 + 2, max_kv_tokens=CAP66, max_step_tokens=128, max_vit_batch=1,
             kv_pool_tokens=(N8 + 1) * CAP8 + CAP66)
eng.load_weights(w)
sids = [eng.stream_open() for _ in range(N8)]
for i, s in enumerate(sids):
    eng.kv_fill_synthetic(s, KV8, seed=100 + i)
swapper, big = eng.stream_open(), eng.stream_open()
eng.kv_fill_synthetic(swapper, KV8, seed=200)
torch.cuda.synchronize()

emb = torch.zeros(11 * N8, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
ids = torch.tensor(([cfg.frame_token_interval_id] + [-1] * 10) * N8, dtype=torch.int64, device=dev)
side = torch.cuda.Stream(dev)


step_ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(TICKS)]


def tick(ev=None):
    if ev is not None:
        ev[0].record()
    eng.step(sids, [11] * N8, emb, row_ids=ids, want_logits=False)
    if ev is not None:
        ev[1].record()
    eng.read_decisions(N8)
    for s in sids:
        eng.kv_truncate(s, KV8)   # 12000 % 64 + 11 <= 64: the step stays inside each stream's last page


def ticks(swapping):
    """(host ms per tick, device ms per step, swap pairs started) over TICKS ticks; swapping: keep a swap-out + swap-in
    pair of the 12k session in flight on `side`"""
    pair = None
    n_pairs = 0

    def feed():
        nonlocal pair, n_pairs
        if pair is None or pair.query():
            with torch.cuda.stream(side):
                eng.kv_swap_in(swapper, eng.kv_swap_out(swapper))
                pair = torch.cuda.Event()
                pair.record(side)
            n_pairs += 1
    if swapping:
        feed()
    t0 = time.perf_counter()
    for i in range(TICKS):
        tick(step_ev[i])
        if swapping:
            feed()
    ms = (time.perf_counter() - t0) * 1e3 / TICKS
    torch.cuda.synchronize()
    return ms, sum(a.elapsed_time(b) for a, b in step_ev) / TICKS, n_pairs


for _ in range(3):
    tick()
ticks(True)   # warm: pinned buffers, events
res = {k: [] for k in ("tick_ms_alone", "step_ms_alone", "tick_ms_swapping", "step_ms_swapping", "swap_pairs_started")}
for _ in range(REPEATS):
    ms, step_ms, _ = ticks(False)
    res["tick_ms_alone"].append(round(ms, 3))
    res["step_ms_alone"].append(round(step_ms, 3))
    ms, step_ms, n = ticks(True)
    res["tick_ms_swapping"].append(round(ms, 3))
    res["step_ms_swapping"].append(round(step_ms, 3))
    res["swap_pairs_started"].append(n)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    t0 = time.perf_counter()
    out = fn()
    host = (time.perf_counter() - t0) * 1e3
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b), host


swap = {}
for n in SIZES:
    eng.kv_fill_synthetic(big, n, seed=300)
    nbytes = eng.kv_image_bytes(n)
    # the first swap-outs of a size allocate their pinned buffers (two are alive at once in the loop below)
    first = []
    for _ in range(2):
        img, ms, host = timed(lambda: eng.kv_swap_out(big))
        first.append(round(host, 1))
        eng.kv_swap_in(big, img)
    rows = {"out_ms": [], "in_ms": [], "out_host_ms": [], "in_host_ms": []}
    for _ in range(REPEATS):
        img, ms, host = timed(lambda: eng.kv_swap_out(big))
        rows["out_ms"].append(ms)
        rows["out_host_ms"].append(host)
        _, ms, host = timed(lambda: eng.kv_swap_in(big, img))
        rows["in_ms"].append(ms)
        rows["in_host_ms"].append(host)
    del img
    eng.stream_reset(big)
    torch._C._host_emptyCache()
    swap[str(n)] = {"image_bytes": nbytes, "first_out_host_ms_incl_pinned_alloc": first,
                    **{k: [round(x, 3) for x in v] for k, v in rows.items()},
                    "out_GB_per_s": round(nbytes / statistics.median(rows["out_ms"]) / 1e6, 2),
                    "in_GB_per_s": round(nbytes / statistics.median(rows["in_ms"]) / 1e6, 2)}

smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
print(json.dumps({
    "gpu": torch.cuda.get_device_name(dev), "nvidia_smi_name_power_limit": smi,
    "swap": swap, "tick_8x12k": res,
    "note": "swap: device ms between CUDA events around one call on its stream, host ms of the Python call; tick: "
            f"host ms per tick (step + decision read-back) over {TICKS} ticks, alone / swapping alternating",
}), flush=True)
