"""fp64 references of the attention kernels and the per-element error bounds they are held to.

Causal-with-offset GQA attention (the decoder's KV-append attention, csrc/attn.cuh) and the ViT's non-causal attention
(vit_attn_kernel, csrc/vit_kernels.cuh) are both a softmax over fp32 scores whose probabilities P are rounded to a 16-bit
type before the P V product.  `reference` computes the exact value on the device in fp64 from the kernel's exact 16-bit
inputs, together with a bound on |out - ref| derived from the kernel's rounding points.

Derivation (u = 2^-24, the relative error of one fp32 rounding).  Per row, with p_k = exp(s_k - max s) the exact
weights, A = sum_k p_k |v_k| / sum_k p_k and S = max over the row's visible keys of sum_i |q_i k_i|:
- Q, K and V are exact 16-bit values.
- A score accumulates n_dot = head_dim products in fp32 (the MMA): |ds| <= n_dot u S.
- The exponent t = s c - m c (c = log2(e) / sqrt(head_dim)) takes three more fp32 roundings: 3 u (|s c| + |m c|), and
  exp2f adds 2 ulp = 2^-22 relative.  So every p_k the kernel forms has a relative error
  eps_s = expm1(ln 2 (c n_dot u S + 3 u (|s c|max + |m c|))) + 2^-22.
  The running-max rescales (alpha) and the split-KV merge weights multiply O and l alike, so their errors cancel in O / l
  up to one fp32 rounding per operation.
- P is rounded before PV (relative r_p: bf16 2^-9, fp16 2^-11; below the fp16 normal range an absolute 2^-25 per key
  in units of the running max, which is at most the final max).  The row sum l adds the unrounded P.
  Numerator and denominator together move the quotient by at most (r_p + 2 eps_s) A / (1 - eps_s).
- O and l accumulate in fp32 over `chain` sequential operations (MMA steps, rescales, the merge): 2 chain u A.
- The quotient is one more rounding, and the output is rounded to the 16-bit type: half an ulp of the result,
  at most r_out (|ref| + E) with r_out = 2^-8 (bf16) or 2^-11 (fp16, plus 2^-25 absolute below its normal range).
- Weights that underflow fp32 (p < 2^-126 of the running max) are lost: at most 2^-125 sum_k |v_k| / sum_k p_k.
The bound is  E = 2 (r_p + 2 eps_s) A / (1 - eps_s) + 2 chain u A + abs terms,  |out - ref| <= E + r_out (|ref| + E),
where the factor 2 in front of the first term is headroom.
"""
import math

import torch

U = 2.0 ** -24
LN2 = math.log(2.0)


class Spec:
    """the rounding points of one kernel family"""

    def __init__(self, p_rel, p_abs, out_rel, out_abs):
        self.p_rel, self.p_abs, self.out_rel, self.out_abs = p_rel, p_abs, out_rel, out_abs


DECODER = Spec(p_rel=2.0 ** -9, p_abs=0.0, out_rel=2.0 ** -8, out_abs=0.0)      # bf16 P, bf16 out
VIT = Spec(p_rel=2.0 ** -11, p_abs=2.0 ** -25, out_rel=2.0 ** -11, out_abs=2.0 ** -25)   # fp16 P, fp16 out


class Result:
    """ref / bound [T, H, D] fp64; block_drop(b): the reference without key block b (64 keys), for the self-check"""

    def __init__(self, ref, bound, pv_blocks, l_blocks, pv, l):
        self.ref, self.bound = ref, bound
        self._pvb, self._lb, self._pv, self._l = pv_blocks, l_blocks, pv, l

    def without_block(self, b):
        """the fp64 reference with the keys of 64-key block b removed from every row's softmax"""
        num = self._pv - self._pvb[:, :, b]
        den = self._l - self._lb[:, :, b]
        return num / den.clamp_min(1e-300)[..., None]

    def excess(self, out):
        """max over elements of |out - ref| - bound (<= 0: within the bound)"""
        return float(((out.double() - self.ref).abs() - self.bound).max())


def reference(q, k, v, q_pos, spec, chain, blocks=False):
    """q [T, H, D] 16-bit; k, v [Hk, L, D] 16-bit logical keys (key j of kv head h at k[h, j]); q_pos [T] int: row t
    attends keys 0 .. q_pos[t] (all keys for the ViT: q_pos = L - 1).  chain: fp32 accumulation chain of O / l per row
    (int or tensor [T]).  blocks: keep per-64-key-block partial sums for Result.without_block."""
    T, H, D = q.shape
    Hk, L, _ = k.shape
    G = H // Hk
    dev = q.device
    c = math.log2(math.e) / math.sqrt(D)
    pos = torch.as_tensor(q_pos, device=dev, dtype=torch.long)
    vis = torch.arange(L, device=dev)[None, :] <= pos[:, None]                    # [T, L]
    chain_t = torch.as_tensor(chain, device=dev, dtype=torch.float64).reshape(-1, 1, 1) * torch.ones(T, 1, 1, device=dev,
                                                                                                     dtype=torch.float64)
    nblk = (L + 63) // 64
    ref = torch.empty(T, H, D, dtype=torch.float64, device=dev)
    bound = torch.empty_like(ref)
    pv_all = torch.empty_like(ref) if blocks else None
    l_all = torch.empty(T, H, dtype=torch.float64, device=dev) if blocks else None
    pvb_all = torch.empty(T, H, nblk, D, dtype=torch.float64, device=dev) if blocks else None
    lb_all = torch.empty(T, H, nblk, dtype=torch.float64, device=dev) if blocks else None
    for h in range(Hk):
        qh = q[:, h * G:(h + 1) * G].double()                                       # [T, G, D]
        kh, vh = k[h].double(), v[h].double()                                       # [L, D]
        s = torch.einsum("tgd,ld->tgl", qh, kh) / math.sqrt(D)
        sabs = torch.einsum("tgd,ld->tgl", qh.abs(), kh.abs())
        s = s.masked_fill(~vis[:, None, :], float("-inf"))
        m = s.amax(-1, keepdim=True)
        p = torch.exp(s - m)
        l = p.sum(-1)
        pv = torch.einsum("tgl,ld->tgd", p, vh)
        pav = torch.einsum("tgl,ld->tgd", p, vh.abs())
        vsum = torch.einsum("tl,ld->td", vis.double(), vh.abs())[:, None, :]        # sum over visible keys of |v|
        r = pv / l[..., None]
        A = pav / l[..., None]
        S = sabs.masked_fill(~vis[:, None, :], 0).amax(-1)
        smax = (s.masked_fill(~vis[:, None, :], 0).abs().amax(-1)) * c
        eps_s = torch.expm1(LN2 * (c * D * U * S + 3 * U * (smax + m[..., 0].abs() * c))) + 2.0 ** -22
        E = (2 * (spec.p_rel + 2 * eps_s[..., None]) / (1 - eps_s[..., None]) * A + 2 * chain_t * U * A
             + (spec.p_abs * 2 + 2.0 ** -125) * vsum / l[..., None])
        ref[:, h * G:(h + 1) * G] = r
        bound[:, h * G:(h + 1) * G] = E + spec.out_rel * (r.abs() + E) + spec.out_abs
        if blocks:
            pp = torch.nn.functional.pad(p, (0, nblk * 64 - L)).view(T, G, nblk, 64)
            vv = torch.nn.functional.pad(vh, (0, 0, 0, nblk * 64 - L)).view(nblk, 64, D)
            pvb_all[:, h * G:(h + 1) * G] = torch.einsum("tgbk,bkd->tgbd", pp, vv)
            lb_all[:, h * G:(h + 1) * G] = pp.sum(-1)
            pv_all[:, h * G:(h + 1) * G] = pv
            l_all[:, h * G:(h + 1) * G] = l
    return Result(ref, bound, pvb_all, lb_all, pv_all, l_all)


def decoder_chain(kv_len, n_sm):
    """fp32 chain length of a row's O / l in the decoder attention, whatever the plan: per key block 4 MMA k-steps and
    one rescale (all blocks in one split at worst), the warp-group merge and a split-KV merge of at most n_sm terms,
    plus 32 for the sums inside the MMA"""
    return 5 * ((kv_len + 63) // 64) + n_sm + 32


def vit_chain(n_tok):
    """the same for vit_attn_kernel: one CTA walks all key blocks, no merge"""
    return 5 * ((n_tok + 63) // 64) + 32


def plan_items(n_tok, kv_len, n_heads, n_kv_heads, n_sm, want=None):
    """attn_plan (csrc/attn.cu) for one sequence of one segment: its work items with their split grid.  Rows are chunked
    by 64 / G; the split budget is max(1, n_sm / (n_kv_heads * n_items)) unless `want` is given; blocks_per_split is
    ceil(nblk / want) rounded up to even and >= 2."""
    G = n_heads // n_kv_heads
    per = 64 // G
    n_items = (n_tok + per - 1) // per
    if want is None:
        want = max(1, n_sm // (n_kv_heads * n_items))
    items = []
    for t0 in range(0, n_tok, per):
        qc = min(per, n_tok - t0)
        q_pos0 = kv_len - n_tok + t0
        nblk = (q_pos0 + qc + 63) // 64
        bps = (nblk + want - 1) // want
        bps = max(2, bps + (bps & 1))
        items.append({"t0": t0, "q_count": qc, "q_pos0": q_pos0, "nblk": nblk, "bps": bps, "ns": (nblk + bps - 1) // bps})
    return items


def merge_path(ns):
    """which branch of attn_merge_kernel merges an item of ns splits"""
    return "regs4" if ns <= 4 else ("regs20" if ns <= 20 else "smem")
