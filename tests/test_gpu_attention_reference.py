"""The decoder's KV-append attention and the ViT attention kernels against fp64 references under the error bounds of
attn_reference.py, with inputs that make every key block matter.

Needles.  The query heads of a kv group (a ViT head) share a direction u; a needle key is b u, with a score of about b
against background scores of about 0, so the needles carry nearly all of the softmax mass.  Needles sit where a plan can
go wrong: the first and last key of every split of every work item, the last partial block, and every query row's own
key (its causal limit, and the key just past the limit of the row before it, which that row must mask).  Rows of the
cache past kv_len hold needles with scores above every other key and V values of ~100: they must be masked.  Every case
first checks that the reference without any one needle block violates the bound, so a kernel that drops or misweights
a block cannot pass."""
import ctypes as C
import math

import pytest
import torch

from attn_reference import DECODER, VIT, U, decoder_chain, merge_path, plan_items, reference, vit_chain

pytestmark = pytest.mark.gpu

PAGE = 64
D = 128


@pytest.fixture(scope="module")
def lib():
    from videollm_online_b200 import _lib
    return _lib.load()


def _p(t):
    return C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc, what):
    from videollm_online_b200._lib import check
    check(rc, what)


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _plan_counts(lib, segs, Hq, Hk, kv_end):
    out = (C.c_int32 * 4)()
    _check(lib.vlo_op_attn_plan_counts(len(segs), (C.c_int32 * len(segs))(*segs), Hq, Hk, D, kv_end, out), "plan_counts")
    return {"items": out[0], "clusters": out[1], "packs": out[2], "packed_items": out[3]}


def _items(segs, kv_len, Hq, Hk):
    """the work items of a plan of these segments (each segment planned alone, csrc/attn.cu), rows in absolute order"""
    if len(segs) == 1:
        return plan_items(segs[0], kv_len, Hq, Hk, _n_sm())
    n_tok, o, items = sum(segs), 0, []
    per = 64 // (Hq // Hk)
    for n in segs:
        end = kv_len - n_tok + o + n
        want = max(1, _n_sm() // (Hk * ((n + per - 1) // per)))
        for it in plan_items(n, end, Hq, Hk, _n_sm(), want=want):
            it["t0"] += o
            items.append(it)
        o += n
    return items


# ============================================================================================ decoder
def _needle_keys(items, n_tok, kv_len):
    """split edges of every item, the middle of the last partial block, every row's own key"""
    keys = set(range(kv_len - n_tok, kv_len))
    for it in items:
        end = it["q_pos0"] + it["q_count"]
        for s in range(it["ns"]):
            b0 = s * it["bps"]
            keys.add(b0 * PAGE)
            keys.add(min((b0 + it["bps"]) * PAGE, end) - 1)
    nblk = (kv_len + PAGE - 1) // PAGE
    tail = kv_len - (nblk - 1) * PAGE
    keys.add((nblk - 1) * PAGE + (tail - 1) // 2)
    return sorted(k for k in keys if k < kv_len)


def _decoder_inputs(n_tok, kv_len, Hq, Hk, needles, profile, stride, seed):
    """q [n_tok, Hq, D]; k, v [Hk, stride, D] with needles, a score profile over the background and hostile rows past
    kv_len.  profile: flat (needle scores 16), huge (110: the background underflows to 0), rise (scores grow by 40 over
    the context, so the running max grows in every block), fall (they drop by 95: late splits weigh ~2^-137)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    G = Hq // Hk
    u = torch.randn(Hk, D, device="cuda", generator=g)
    u = u / u.norm(dim=-1, keepdim=True)
    b = 110.0 if profile == "huge" else 16.0
    # the query noise moves a needle's score by about 0.1, whatever b
    q = math.sqrt(D) * u.repeat_interleave(G, 0)[None] + 1.6 / b * torch.randn(n_tok, Hq, D, device="cuda", generator=g)
    k = torch.randn(Hk, stride, D, device="cuda", generator=g)
    v = torch.randn(Hk, stride, D, device="cuda", generator=g)
    j = torch.arange(stride, device="cuda", dtype=torch.float32)
    tau = {"flat": 0 * j, "huge": 0 * j, "rise": 40 * j / kv_len, "fall": -95 * j / kv_len}[profile]
    k += tau[None, :, None] * u[:, None, :]
    nd = torch.tensor(needles, device="cuda", dtype=torch.long)
    k[:, nd] = (b + tau[nd])[None, :, None] * u[:, None, :]
    k[:, kv_len:] = (b + 30.0 + tau[kv_len:])[None, :, None] * u[:, None, :]   # must be masked: would dominate
    v[:, kv_len:] = 100.0 * torch.randn(Hk, stride - kv_len, D, device="cuda", generator=g)
    return q.bfloat16(), k.bfloat16(), v.bfloat16()


def _to_pages(k, v, nblk, seed):
    """scattered pages of a pool with 5 spare NaN pages; returns pools and the page table"""
    Hk = k.shape[0]
    n_pages = nblk + 5
    perm = torch.randperm(n_pages, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))[:nblk]
    kp = torch.full((n_pages, Hk, PAGE, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    vp = torch.full_like(kp, float("nan"))
    kp[perm] = k[:, :nblk * PAGE].reshape(Hk, nblk, PAGE, D).transpose(0, 1)
    vp[perm] = v[:, :nblk * PAGE].reshape(Hk, nblk, PAGE, D).transpose(0, 1)
    return kp, vp, perm.to(torch.int32).contiguous(), n_pages


def _run_decoder(lib, path, segs, kv_len, Hq, Hk, q, k, v, seed):
    n_tok = sum(segs)
    nblk = (kv_len + PAGE - 1) // PAGE
    out = torch.full((n_tok, Hq * D), float("nan"), device="cuda", dtype=torch.bfloat16)
    if path == "contig":
        ws = torch.empty(lib.vlo_op_attn_ws_bytes(n_tok, Hq, D, kv_len), device="cuda", dtype=torch.uint8)
        _check(lib.vlo_op_attn_kvappend(_p(q), _p(k), _p(v), _p(out), _p(ws), n_tok, Hq, Hk, D, kv_len, k.shape[1], _st()),
               "attn")
    else:
        kp, vp, pt, n_pages = _to_pages(k, v, nblk, seed)
        if path == "paged":
            ws = torch.empty(lib.vlo_op_attn_ws_bytes(n_tok, Hq, D, kv_len), device="cuda", dtype=torch.uint8)
            _check(lib.vlo_op_attn_kvappend_paged(_p(q), _p(kp), _p(vp), _p(pt), n_pages, _p(out), _p(ws), n_tok, Hq, Hk,
                                                  D, kv_len, _st()), "attn_paged")
        else:
            lens = (C.c_int32 * len(segs))(*segs)
            _check(lib.vlo_op_attn_kvappend_segments(_p(q), _p(kp), _p(vp), _p(pt), n_pages, _p(out), len(segs), lens, Hq,
                                                     Hk, D, kv_len, _st()), "attn_segments")
    torch.cuda.synchronize()
    return out


# (path, segments, kv_len, Hq, Hk, profile).  "contig" / "paged": one sequence on attn_kvappend_kernel; "cluster": a
# segmented sequence whose items run in 2-CTA clusters; "packed": runs of one-token segments on the packed kernel.
CASES = [
    ("contig", [1], 1, 32, 8, "flat"), ("contig", [1], 63, 32, 8, "flat"), ("contig", [11], 63, 32, 8, "flat"),
    ("contig", [40], 64, 32, 8, "flat"), ("contig", [1], 64, 32, 8, "huge"), ("contig", [11], 65, 32, 8, "flat"),
    ("contig", [40], 65, 32, 8, "rise"),
    ("contig", [11], 260, 32, 8, "flat"),        # 5 blocks: the last split holds block 4 alone, rows 0-6 see none of it
    ("contig", [16], 13211, 32, 8, "flat"), ("contig", [17], 13211, 32, 8, "flat"),   # the 64 / G item boundary
    ("contig", [11], 13211, 32, 8, "rise"), ("contig", [64], 13211, 32, 8, "flat"),   # 15 splits; 4 items of 4 splits
    ("contig", [11], 12288 + 11, 32, 8, "fall"), ("contig", [1], 12288 - 11, 32, 8, "huge"),
    ("contig", [1], 66011, 32, 8, "flat"), ("contig", [11], 66011, 32, 8, "fall"), ("contig", [40], 66011, 32, 8, "huge"),
    ("contig", [11], 3076, 8, 2, "flat"),        # 49 blocks in 25 splits (merge > 20), the last one block past rows 0-6
    ("contig", [11], 13211, 4, 1, "rise"), ("contig", [1], 66011, 64, 1, "flat"),   # 104 and 129 splits, G = 4 and 64
    ("paged", [1], 65, 32, 8, "flat"), ("paged", [11], 13211, 32, 8, "flat"), ("paged", [40], 66011, 32, 8, "flat"),
    ("paged", [11], 3076, 8, 2, "huge"), ("paged", [2], 12288 + 40, 128, 2, "fall"),
    ("cluster", [11] * 4, 12288 + 22, 32, 8, "flat"), ("cluster", [14, 11, 11], 66011, 32, 8, "flat"),
    ("cluster", [11, 11, 11], 3076, 8, 2, "rise"),
    ("packed", [1] * 8, 12288 + 4, 32, 8, "flat"), ("packed", [11, 1, 1, 1, 1], 13211, 32, 8, "huge"),
    ("packed", [1] * 16, 66011, 32, 8, "flat"), ("packed", [1] * 4, 3076, 8, 2, "flat"),
]


def _id(c):
    segs = c[1]
    s = str(segs[0]) if len(segs) == 1 else "+".join(map(str, segs)) if len(segs) <= 4 else f"{segs[0]}+1x{len(segs) - 1}"
    return f"{c[0]}-{s}-kv{c[2]}-{c[3]}x{c[4]}-{c[5]}"


@pytest.mark.parametrize("path,segs,kv_len,Hq,Hk,profile", CASES, ids=[_id(c) for c in CASES])
def test_decoder_attention_within_fp64_bound(lib, path, segs, kv_len, Hq, Hk, profile):
    n_tok = sum(segs)
    seed = kv_len * 31 + n_tok * 7 + Hq + len(segs)
    if path == "cluster":
        assert _plan_counts(lib, segs, Hq, Hk, kv_len)["clusters"] >= 1
    if path == "packed":
        assert _plan_counts(lib, segs, Hq, Hk, kv_len)["packs"] >= 1
    items = _items(segs, kv_len, Hq, Hk)
    needles = _needle_keys(items, n_tok, kv_len)
    stride = (kv_len + PAGE - 1) // PAGE * PAGE + (PAGE if path == "contig" else 0)
    q, k, v = _decoder_inputs(n_tok, kv_len, Hq, Hk, needles, profile, stride, seed)
    q_pos = torch.arange(kv_len - n_tok, kv_len)
    res = reference(q, k[:, :kv_len], v[:, :kv_len], q_pos, DECODER, decoder_chain(kv_len, _n_sm()), blocks=True)
    # self-check: without any one needle block the reference leaves the bound (flat / huge: every needle block; rise /
    # fall: the needles of the blocks that carry the mass)
    blocks = sorted({n // PAGE for n in needles})
    seen = 0
    for b in blocks:
        moved = float(((res.without_block(b) - res.ref).abs() - res.bound).max())
        if profile in ("flat", "huge"):
            assert moved > 0, f"dropping needle block {b} stays within the bound: the case cannot see it"
        seen += moved > 0
    assert seen >= 1
    out = _run_decoder(lib, path, segs, kv_len, Hq, Hk, q, k, v, seed)
    assert torch.isfinite(out.float()).all()
    ex = res.excess(out.view(n_tok, Hq, D))
    assert ex <= 0, f"attention leaves the fp64 bound by {ex}"


def test_cases_reach_every_merge_path(lib):
    """the case list covers attn_merge_kernel's three branches with a real merge (>= 2 splits) and a one-block last split
    that some row of its item cannot see"""
    paths, lone_tail = set(), False
    for _path, segs, kv_len, Hq, Hk, _prof in CASES:
        for it in _items(segs, kv_len, Hq, Hk):
            if it["ns"] >= 2:
                paths.add(merge_path(it["ns"]))
            if it["ns"] >= 2 and it["nblk"] - (it["ns"] - 1) * it["bps"] == 1 and it["q_pos0"] < (it["nblk"] - 1) * PAGE:
                lone_tail = True
    assert paths == {"regs4", "regs20", "smem"}, paths
    assert lone_tail


# ============================================================================================ ViT attention
VIT_HD = 64
SENT16 = 0x7E01      # an fp16 NaN pattern no kernel writes


def _vit_inputs(B, N, heads, seed):
    """qkv fp16 [B N, 3C]: per (frame, head) a direction u, queries ~ 8 u, one needle key (score 12) per 64-key block;
    the first keys of the next frame, which fall into the masked part of this frame's last block, are needles (score 24)
    aligned with THIS frame's queries"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    C_ = heads * VIT_HD
    u = torch.randn(B, heads, VIT_HD, device="cuda", generator=g)
    u = u / u.norm(dim=-1, keepdim=True)
    q = 8.0 * u[:, None] + 0.1 * torch.randn(B, N, heads, VIT_HD, device="cuda", generator=g)
    k = torch.randn(B, N, heads, VIT_HD, device="cuda", generator=g)
    v = torch.randn(B, N, heads, VIT_HD, device="cuda", generator=g)
    nblk = (N + 63) // 64
    spill = nblk * 64 - N     # keys of the next frame inside this frame's last block: block 0's needle lies past them
    needles = []
    for i in range(nblk):
        lo, hi = (spill if i == 0 else 0), min(64, N - 64 * i)
        needles.append(64 * i + int(torch.randint(lo, hi, (1,), generator=g, device="cuda")))
    for n in needles:
        k[:, n] = 12.0 * u
    for f in range(B - 1):
        k[f + 1, :min(spill, N)] = 24.0 * u[f][None]
    qkv = torch.cat([q.reshape(B * N, C_), k.reshape(B * N, C_), v.reshape(B * N, C_)], 1).half().contiguous()
    return qkv, needles


@pytest.mark.parametrize("heads", [2, 16])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("N", [36, 196, 256, 257, 576, 577])
def test_vit_attention_within_fp64_bound(lib, N, B, heads):
    """one block, partial last blocks, the 4-stage ring wrapping past 4 blocks, a one-row last block; frames isolated;
    nothing written outside [0, B N) x [0, C)"""
    C_ = heads * VIT_HD
    qkv, needles = _vit_inputs(B, N, heads, seed=N * 10 + B + heads)
    pad = 64 * C_
    buf = torch.full((pad + B * N * C_ + pad,), SENT16, dtype=torch.int16, device="cuda")
    out = buf[pad:pad + B * N * C_].view(torch.float16)
    _check(lib.vlo_op_vit_attn(_p(qkv), _p(out), B, N, C_, _st()), "vit_attn")
    torch.cuda.synchronize()
    assert bool((buf[:pad] == SENT16).all()) and bool((buf[pad + B * N * C_:] == SENT16).all()), "wrote outside out"
    o = out.view(B, N, heads, VIT_HD)
    assert torch.isfinite(o.float()).all()
    x = qkv.view(B, N, 3, heads, VIT_HD)
    for f in range(B):
        kf, vf = x[f, :, 1].transpose(0, 1), x[f, :, 2].transpose(0, 1)      # [heads, N, 64]
        res = reference(x[f, :, 0], kf, vf, torch.full((N,), N - 1), VIT, vit_chain(N), blocks=True)
        for b in sorted({n // 64 for n in needles}):
            moved = float(((res.without_block(b) - res.ref).abs() - res.bound).max())
            assert moved > 0, f"dropping key block {b} stays within the bound"
        ex = res.excess(o[f])
        assert ex <= 0, f"frame {f}: vit attention leaves the fp64 bound by {ex}"


def test_vit_attention_entry_rejects_bad_sizes(lib):
    x = torch.zeros(64 * 3 * 128, dtype=torch.float16, device="cuda")
    for B, N, C_ in ((0, 36, 128), (1, 0, 128), (1, 36, 96), (1, 36, 0)):
        assert lib.vlo_op_vit_attn(_p(x), _p(x), B, N, C_, _st()) != 0
        assert lib.vlo_op_probe_attn(_p(x), _p(x), _p(x), B, N, C_, _st()) != 0
    assert lib.vlo_op_probe_attn(_p(x), _p(x), _p(x), 1, 12289, 128, _st()) != 0


# ============================================================================================ MAP-head probe attention
def _fp16_range(y, E):
    """the fp16 values the rounding of any value within [y - E, y + E] can give (monotone: the two ends)"""
    return (y - E).float().half().double(), (y + E).float().half().double()


@pytest.mark.parametrize("N", [1, 14, 15, 16, 17, 36, 196, 576])
@pytest.mark.parametrize("B,heads", [(1, 2), (5, 16)])
def test_probe_attention_exact(lib, N, B, heads):
    """fp32 throughout, one fp16 rounding at the end: out = fp16 of the fp64 value, or a neighbour within the derived
    bound.  Scores are exact in fp32 (q integers, k quarters, scale 1/8: every partial sum is a multiple of 1/32 below
    2^10), spread over +-40, so the bound covers expf, the sums and the division only:
      e_n = expf(s_n - max): relative eta = 2^-22 (2 ulp);
      sum e: each thread adds ceil(N / 128) terms, 5 shuffle levels, 3 adds of the warp sums: (ceil(N/128) + 8) u;
      acc: each half adds its keys n = half, half + 2, .. in order with an FMA: u sum_j |partial_j|, then one add;
      the quotient: u.  E = 2 x the sum of these, as an absolute bound on the pre-rounding value."""
    g = torch.Generator(device="cuda").manual_seed(N * 13 + B)
    C_ = heads * VIT_HD
    q = torch.randint(-8, 9, (C_,), device="cuda", generator=g).float()
    k = (torch.randint(-32, 33, (B, N, C_), device="cuda", generator=g).float() / 4).half()
    v = torch.randn(B, N, C_, device="cuda", generator=g).half()
    kv = torch.cat([k, v], -1).reshape(B * N, 2 * C_).contiguous()
    pad = 64
    buf = torch.full((pad + B * C_ + pad,), SENT16, dtype=torch.int16, device="cuda")
    out = buf[pad:pad + B * C_].view(torch.float16)
    _check(lib.vlo_op_probe_attn(_p(kv), _p(q), _p(out), B, N, C_, _st()), "probe_attn")
    torch.cuda.synchronize()
    assert bool((buf[:pad] == SENT16).all()) and bool((buf[pad + B * C_:] == SENT16).all()), "wrote outside out"
    qh = q.double().view(heads, VIT_HD) * 0.125
    kh = k.double().view(B, N, heads, VIT_HD)
    vh = v.double().view(B, N, heads, VIT_HD)
    s = torch.einsum("hd,bnhd->bhn", qh, kh)
    if N >= 14:
        assert float((s.amax(-1) - s.amin(-1)).max()) > 40, "scores must spread over large magnitudes"
    e = torch.exp(s - s.amax(-1, keepdim=True))
    den = e.sum(-1)                                                  # [B, heads]
    ev = e[..., None] * vh.permute(0, 2, 1, 3)                       # [B, heads, N, 64]
    num = ev.sum(2)
    y = num / den[..., None]
    eta = 2.0 ** -22
    n_sum = math.ceil(N / 128) + 8
    partial = sum(ev[:, :, h::2].cumsum(2).abs().sum(2) for h in range(2))
    eva = ev.abs().sum(2)
    # + weights below the fp32 normal range (expf loses their relative accuracy): 2^-126 each at most
    E_num = eta * eva + U * partial + U * num.abs() + 2.0 ** -126 * vh.abs().sum(1)
    E = 2 * (E_num / (den[..., None] * (1 - eta - n_sum * U)) + y.abs() * (eta + n_sum * U + U) * 1.01)
    lo, hi = _fp16_range(y, E)
    o = out.view(B, heads, VIT_HD).double()
    ok = (o >= lo) & (o <= hi)
    assert bool(ok.all()), f"{int((~ok).sum())} of {ok.numel()} outputs outside the fp16 roundings of [y - E, y + E]"
    amb = float((lo != hi).double().mean())
    assert amb <= 0.1, f"{amb:.1%} of the outputs are ambiguous: the bound is too loose"
