"""numpy mirror of keyed dropout (qagnn_keyed_dropout_forward_typed / _backward_typed, qagnn_b200.training.keyed_dropout).

x is [A, G, L]; element (a, g, l) belongs to question qids[g // nc], choice g % nc, with in-graph index e = a L + l.  Its
uniform is word e & 3 of Philox4x32-10(counter = (e >> 2, site + 256 choice, qid lo 32, draw lo 32), key = (seed lo 32,
seed hi 32)); it is kept when u >= min(floor(p 2^32), 2^32 - 1), and never at p = 1."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 of uint32 counters ctr [..., 4] under keys key [..., 2] (broadcast): uint32 [..., 4]."""
    ctr = np.asarray(ctr, dtype=np.uint32)
    key = np.asarray(key, dtype=np.uint32)
    c0, c1, c2, c3 = (ctr[..., i].astype(np.uint64) for i in range(4))
    k0, k1 = key[..., 0].astype(np.uint64), key[..., 1].astype(np.uint64)
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & LO, (k1 + W1) & LO
        p0, p1 = M0 * c0, M1 * c2  # exact: both factors < 2^32
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & LO, p1 >> np.uint64(32), p1 & LO
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def threshold(p):
    return min(int(np.floor(float(p) * 4294967296.0)), 4294967295)


def scale(p):
    return np.float32(1.0 / (1.0 - p)) if p < 1.0 else np.float32(0.0)


def keep_mask(A, G, L, p, seed, draw, qids, nc, site):
    """bool [A, G, L]: which elements are kept."""
    qids = np.asarray(qids, dtype=np.int64)
    a = np.arange(A, dtype=np.int64)[:, None, None]
    g = np.arange(G, dtype=np.int64)[None, :, None]
    l = np.arange(L, dtype=np.int64)[None, None, :]
    e = np.broadcast_to(a * L + l, (A, G, L))
    q = np.broadcast_to(qids[g // nc] & 0xFFFFFFFF, (A, G, L))
    c1 = np.broadcast_to(site + 256 * (g % nc), (A, G, L))
    ctr = np.stack([e >> 2, c1, q, np.full((A, G, L), int(draw) & 0xFFFFFFFF)], axis=-1).astype(np.uint64).astype(np.uint32)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint32)
    u = np.take_along_axis(philox4x32_10(ctr, key), (e & 3)[..., None], axis=-1)[..., 0]
    if p >= 1.0:
        return np.zeros((A, G, L), dtype=bool)
    return u >= np.uint32(threshold(p))


def pack_bits(keep):
    """uint32 words, bit i of word i // 32 = keep.flat[i] (what the forward writes as its mask)."""
    flat = np.asarray(keep, dtype=bool).reshape(-1)
    n = flat.size
    padded = np.zeros((n + 31) // 32 * 32, dtype=np.uint64)
    padded[:n] = flat
    return (padded.reshape(-1, 32) << np.arange(32, dtype=np.uint64)).sum(1).astype(np.uint32)


def apply(x, keep, p, dtype):
    """round_to(dtype, float32(x) * scale) where kept, else 0; x an fp32 array of values representable in dtype, dtype a
    torch dtype.  Returns a torch tensor of that dtype on the CPU."""
    import torch
    x = np.asarray(x, dtype=np.float32)
    y = np.where(keep, x * scale(p), np.float32(0.0)).astype(np.float32)  # one fp32 multiply, then one rounding to dtype
    return torch.from_numpy(y).to(dtype)
