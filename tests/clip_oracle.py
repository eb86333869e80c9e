"""csrc/clip.cu's norm restated in numpy: the fp64 sum of squares in the kernel's order (a thread's elements, the block tree,
the slots), the fp32 norm it rounds to and the clip coefficient torch forms from it.  Test-only reference."""
import numpy as np

THREADS, CHUNK = 256, 8192


def block_tree(v):
    """[..., 256] fp64 -> [...]: each warp's __shfl_down_sync tree at offsets 16, 8, 4, 2, 1, then warp 0's over the 8
    warp sums at 4, 2, 1 (lane 0's sums; the lanes it never reads do not matter)."""
    v = np.array(v, dtype=np.float64).reshape(v.shape[:-1] + (THREADS // 32, 32))
    for o in (16, 8, 4, 2, 1):
        v[..., :o] = v[..., :o] + v[..., o:2 * o]
    w = v[..., 0].copy()
    for o in (4, 2, 1):
        w[..., :o] = w[..., :o] + w[..., o:2 * o]
    return w[..., 0]


def _thread_partials(quads, tail):
    """quads fp64 [chunks, q, 4] of squares, tail [chunks, r] (r < 4): thread t adds quads t, t + 256, ... element by element,
    then tail[t]; [chunks, 256]."""
    c, q = quads.shape[:2]
    m = -(-q // THREADS)
    padded = np.zeros((c, m * THREADS, 4))  # + 0.0 leaves a partial >= +0 as it is
    padded[:, :q] = quads
    padded = padded.reshape(c, m, THREADS, 4)
    acc = np.zeros((c, THREADS))
    for k in range(m):
        for e in range(4):
            acc = acc + padded[:, k, :, e]
    acc[:, :tail.shape[1]] = acc[:, :tail.shape[1]] + tail
    return acc


def chunk_sums(x):
    """The slot of every chunk of one tensor, in order: fp64 [ceil(numel / 8192)]."""
    x = np.asarray(x, dtype=np.float32).reshape(-1)
    full, n = x.size // CHUNK, x.size
    out = []
    if full:
        sq = x[:full * CHUNK].astype(np.float64) ** 2  # exact: a 24-bit significand squared fits in 53 bits
        out.append(block_tree(_thread_partials(sq.reshape(full, CHUNK // 4, 4), np.zeros((full, 0)))))
    if n > full * CHUNK:
        sq = x[full * CHUNK:].astype(np.float64) ** 2
        q = sq.size // 4
        out.append(block_tree(_thread_partials(sq[:4 * q].reshape(1, q, 4), sq[4 * q:].reshape(1, -1))))
    return np.concatenate(out) if out else np.zeros(0)


def sum_squares(tensors):
    """S over a list of tensors in the kernel's order: thread t of the last CTA adds slots t, t + 256, ..., then the tree."""
    slots = np.concatenate([chunk_sums(t) for t in tensors] + [np.zeros(0)])
    m = -(-slots.size // THREADS)
    padded = np.zeros(max(m, 1) * THREADS)
    padded[:slots.size] = slots
    acc = np.zeros(THREADS)
    for row in padded.reshape(-1, THREADS):
        acc = acc + row
    return float(block_tree(acc))


def total_norm(tensors):
    """fp32: sqrt_rn(S) rounded once."""
    return np.float32(np.sqrt(np.float64(sum_squares(tensors))))


def coefficient(norm, max_norm):
    """torch's clip_grad_norm_ coefficient from an fp32 total: clamp(fp32(max_norm) * (1 / (norm + fp32(1e-6))), max=1), one
    fp32 rounding per operation, a NaN kept."""
    with np.errstate(all="ignore"):
        c = np.float32(max_norm) * (np.float32(1.0) / (np.float32(norm) + np.float32(1e-6)))
    return np.float32(1.0) if c > 1 else np.float32(c)
