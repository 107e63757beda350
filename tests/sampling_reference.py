"""Host restatements of the device sampler (include/vlo_b200.h, vlo_sample): the Philox4x32-10 noise layout, the Gumbel
scores in fp64, and the logits after the penalty and the temperature as the kernel computes them in fp32."""
import numpy as np
import torch

_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 on arrays: ctr = 4 arrays of uint32 values, key = (k0, k1); returns the 4 output words."""
    c = [np.asarray(x, dtype=np.uint64) & _MASK for x in ctr]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _MASK, (k1 + np.uint64(0xBB67AE85)) & _MASK
        p0, p1 = c[0] * np.uint64(0xD2511F53), c[2] * np.uint64(0xCD9E8D57)
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _MASK]
    return c


def gumbel(seed: int, position: int, vocab: int) -> np.ndarray:
    """fp64 g_i = -log(-log(u_i)) of ids 0 .. vocab-1: word i % 4 of Philox(counter (i / 4, position, 0, 0), key =
    (seed low, seed high)), u = ((x >> 8) + 0.5) * 2^-24."""
    i = np.arange(vocab, dtype=np.uint64)
    g = i // np.uint64(4)
    z = np.zeros_like(g)
    words = np.stack(philox4x32_10([g, z + np.uint64(position), z, z], (seed & 0xFFFFFFFF, seed >> 32)))
    x = words[(i % np.uint64(4)).astype(np.int64), np.arange(vocab)]
    u = ((x >> np.uint64(8)).astype(np.float64) + 0.5) * 2.0 ** -24
    return -np.log(-np.log(u))


def penalised(row: torch.Tensor, temperature: float, penalty: float, penalty_ids) -> torch.Tensor:
    """fp32 logits after the repetition penalty (each distinct in-range id once) and the temperature"""
    l = row.float().clone()
    if penalty != 1.0:
        ids = sorted({int(i) for i in penalty_ids if 0 <= int(i) < l.numel()})
        if ids:
            v = l[ids]
            l[ids] = torch.where(v < 0, v * penalty, v / penalty)
    return l / temperature
