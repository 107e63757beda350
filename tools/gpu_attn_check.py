"""Dev tool: KV-append attention kernel vs torch SDPA on the GPU + bandwidth (run under gpurun)."""
import ctypes as C, pathlib, sys, json, math
import torch

lib = C.CDLL(str(pathlib.Path(__file__).resolve().parents[1] / "videollm-online_b200" / "libvlo_b200.so"))
lib.vlo_last_error.restype = C.c_char_p
P, I, LL = C.c_void_p, C.c_int, C.c_longlong
lib.vlo_op_attn_ws_bytes.argtypes = [I, I, I, I]; lib.vlo_op_attn_ws_bytes.restype = C.c_int64
lib.vlo_op_attn_kvappend.argtypes = [P, P, P, P, P, I, I, I, I, I, LL, P]; lib.vlo_op_attn_kvappend.restype = I
dev = "cuda"
torch.manual_seed(0)
res = []

def run(q, k, v, kv_len, ws):
    n_tok, H, D = q.shape
    Hk, stride, _ = k.shape
    out = torch.empty(n_tok, H * D, device=dev, dtype=torch.bfloat16)
    rc = lib.vlo_op_attn_kvappend(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), ws.data_ptr(), n_tok, H, Hk, D,
                                  kv_len, stride, torch.cuda.current_stream().cuda_stream)
    if rc != 0:
        raise RuntimeError(lib.vlo_last_error().decode())
    return out

def ref(q, k, v, kv_len):
    n_tok, H, D = q.shape
    Hk = k.shape[0]
    G = H // Hk
    kk = k[:, :kv_len].float().repeat_interleave(G, 0)      # [H, kv, D]
    vv = v[:, :kv_len].float().repeat_interleave(G, 0)
    qq = q.float().permute(1, 0, 2)                          # [H, n_tok, D]
    s = qq @ kk.transpose(1, 2) / math.sqrt(D)
    pos = torch.arange(kv_len - n_tok, kv_len, device=dev)[:, None]
    mask = torch.arange(kv_len, device=dev)[None, :] <= pos
    s = s.masked_fill(~mask[None], float("-inf"))
    o = torch.softmax(s, -1) @ vv                            # [H, n_tok, D]
    return o.permute(1, 0, 2).reshape(n_tok, H * D)

for (n_tok, H, Hk, kv_len, stride) in [(11, 32, 8, 28, 64), (1, 32, 8, 1, 64), (11, 32, 8, 1000, 1024), (1, 32, 8, 777, 1024),
                                        (40, 32, 8, 40, 128), (37, 8, 4, 300, 320), (11, 32, 8, 13211, 13312), (3, 4, 2, 130, 192),
                                        (17, 32, 8, 5000, 5056)]:
    D = 128
    q = torch.randn(n_tok, H, D, device=dev).bfloat16()
    k = torch.randn(Hk, stride, D, device=dev).bfloat16()
    v = torch.randn(Hk, stride, D, device=dev).bfloat16()
    ws = torch.empty(lib.vlo_op_attn_ws_bytes(n_tok, H, D, kv_len), device=dev, dtype=torch.uint8)
    out = run(q, k, v, kv_len, ws)
    torch.cuda.synchronize()
    r = ref(q, k, v, kv_len)
    err = (out.float() - r).abs().max().item()
    ok = err < 2e-2 and bool(torch.isfinite(out.float()).all())
    print(f"attn n_tok={n_tok} H={H} Hk={Hk} kv={kv_len}: err={err:.3e} {'OK' if ok else 'FAIL'}", flush=True)
    res.append(dict(name=f"attn_{n_tok}_{H}_{Hk}_{kv_len}", err=err, ok=ok))

# bandwidth at the BASELINE point: q=11, kv=13.2k and q=1
flush = torch.empty(256 * 1024 * 1024, device=dev, dtype=torch.uint8)
for (n_tok, kv_len) in [(11, 13211), (1, 13211), (11, 6000), (11, 66000)]:
    H, Hk, D = 32, 8, 128
    stride = (kv_len + 63) // 64 * 64
    q = torch.randn(n_tok, H, D, device=dev).bfloat16()
    k = torch.randn(Hk, stride, D, device=dev).bfloat16()
    v = torch.randn(Hk, stride, D, device=dev).bfloat16()
    ws = torch.empty(lib.vlo_op_attn_ws_bytes(n_tok, H, D, kv_len), device=dev, dtype=torch.uint8)
    for _ in range(3):
        run(q, k, v, kv_len, ws)
    ts = []
    for _ in range(10):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); run(q, k, v, kv_len, ws); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    t = sorted(ts)[len(ts) // 2]
    byts = kv_len * Hk * D * 2 * 2
    print(f"attn bw n_tok={n_tok} kv={kv_len}: {t*1e3:.1f} us (incl. merge + H2D of items)  {byts/t/1e6:.0f} GB/s", flush=True)
    res.append(dict(name=f"attn_bw_{n_tok}_{kv_len}", us=t * 1e3, gbs=byts / t / 1e6, ok=True))

pathlib.Path("gpurun_out").mkdir(exist_ok=True)
json.dump(res, open("gpurun_out/attn_check.json", "w"), indent=1)
bad = [r for r in res if not r["ok"]]
print("FAILED:" if bad else "ALL OK", bad)
sys.exit(1 if bad else 0)
