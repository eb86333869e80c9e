"""fp64 references for the ragged decoder tail (attention_pool_kernel<XT, true>) and its backward
(qagnn_attention_pool_backward_ragged), for the tests of qagnn_b200/csrc/pool.cu's ragged entry points.  Pure torch on the CPU.

A ragged batch keeps graph b's first min(adj_lengths[b], n) positions as packed rows from node_ptr[b] on; rows past
node_ptr[B] up to the node capacity N_cap are tail rows no graph owns.  `ragged_layout` builds node_ptr, `pack` and `repad`
move rows between the packed [N_cap, D] and the padded [B, n, D] layouts, and the references run on the padded one.

`pool_forward` is the pooling of O.multihead_att_pool with the key and value projections folded into the query and out of
the sum, as the kernel does it (exact in fp64, and far cheaper at large n).  `pool_backward` is the closed form in the comment
above PoolBwdScratch in pool.cu, taken in fp64 on exactly the kernel's inputs (its own attn included), together with a
magnitude twin: every sum taken again over absolute values, through the whole chain.  An fp32 evaluation of a chain of L
rounded operations, in any order, is within L * 2^-24 * magnitude of the exact value, so each element gets its own bar
BAR_C * L * 2^-24 * magnitude, with L the operations on the longest chain that feeds it.  A missing or extra term moves an
element by its own size, which is far above that bar wherever the term is not itself negligible.
"""
import math

import torch

from oracle import qagnn_oracle as O

F64 = torch.float64
U32 = 2.0 ** -24  # unit roundoff of fp32
BAR_C = 2.0


def ragged_layout(lens, n, tail_rows, slack=0):
    """(node_ptr [B + 1], N_cap, rows): graph b owns min(max(lens[b], 0) + slack, n) rows (the loader's layout has slack 0;
    with slack > 0 a graph owns rows past its length, which the kernels must ignore); `rows` is the flat [B * n] index of
    every packed row in order, and N_cap = node_ptr[B] + tail_rows."""
    B = lens.numel()
    own = (lens.clamp(min=0) + slack).clamp(max=n)
    node_ptr = torch.zeros(B + 1, dtype=torch.long)
    node_ptr[1:] = own.cumsum(0)
    rows = torch.cat([b * n + torch.arange(int(own[b])) for b in range(B)]) if B else torch.zeros(0, dtype=torch.long)
    return node_ptr, int(node_ptr[-1]) + int(tail_rows), rows


def pack(X, rows, N_cap, tail=None):
    """Packed [N_cap, ...] rows of a padded [B, n, ...] tensor; the tail rows are zero, or `tail` ([N_cap - len(rows), ...])."""
    flat = X.reshape(-1, *X.shape[2:])
    out = torch.zeros((N_cap,) + tuple(flat.shape[1:]), dtype=X.dtype)
    out[:rows.numel()] = flat[rows]
    if tail is not None:
        out[rows.numel():] = tail
    return out


def repad(Xp, rows, B, n, fill=None):
    """The padded [B, n, ...] tensor of packed rows; positions no row maps to are zero, or the same positions of `fill`."""
    shape = (B * n,) + tuple(Xp.shape[1:])
    out = torch.zeros(shape, dtype=Xp.dtype) if fill is None else fill.reshape(shape).clone().to(Xp.dtype)
    out[rows] = Xp[:rows.numel()]
    return out.view((B, n) + tuple(Xp.shape[1:]))


def pool_forward(qs, X, mask, wk, bk, wv, bv, nh):
    """(pooled [B, D], attn [nh * B, n]) of the masked multi-head pooling with query qs [B, D] (w_qs already applied), in
    fp64 with the projections folded: logit_hi = (W_k,h^T qs_h . x_i + qs_h . b_k,h) / sqrt(dk), pooled_h = W_v,h xs_h + b_v,h."""
    B, n, D = X.shape
    dk = D // nh
    qs, X, wk, bk, wv, bv = (t.detach().to(F64) for t in (qs, X, wk, bk, wv, bv))
    qsh = qs.view(B, nh, dk)
    qk = torch.einsum("bhr,hrj->bhj", qsh, wk.view(nh, dk, D))
    cst = (qsh * bk.view(nh, dk)).sum(-1)
    logit = (torch.einsum("bhj,bij->bhi", qk, X) + cst.unsqueeze(-1)) / math.sqrt(dk)
    logit = logit.masked_fill(mask.unsqueeze(1), float("-inf"))
    a = torch.softmax(logit, dim=-1)  # [B, nh, n]
    xs = torch.einsum("bhi,bij->bhj", a, X)
    pooled = torch.einsum("hrj,bhj->bhr", wv.view(nh, dk, D), xs).reshape(B, D) + bv
    return pooled, a.permute(1, 0, 2).reshape(nh * B, n)


def bar(mag, L):
    return BAR_C * L * U32 * mag


def pool_backward(qs, X, attn, dconcat, wk, bk, wv, nh, S, n_rows=None):
    """The ragged pooling backward's closed form in fp64, on the padded layout (X zero past each graph's rows).

    qs [B, D], X [B, n, D], attn [nh * B, n] (the forward's weights, exactly 0 where masked), dconcat [B, 2D + S], wk / wv
    [D, D], bk [D].  `n_rows`: the most rows any graph pools over (default n), the length of the node sums.
    Returns {name: (value, bar)} for dX [B, n, D], dqs [B, D], dwk, dbk, dwv, dbv; `mag` holds each one's magnitude twin and
    `parts` the per-(graph, head) intermediates qk, dxs, xs, g (logit gradient, [B, nh, n]), dqk and dcst."""
    B, n, D = X.shape
    dk = D // nh
    L_n = n if n_rows is None else int(n_rows)
    qs, X, attn, dconcat, wk, bk, wv = (t.detach().to(F64) for t in (qs, X, attn, dconcat, wk, bk, wv))
    Xa = X.abs()
    a = attn.view(nh, B, n).permute(1, 0, 2)  # [B, nh, n], >= 0
    qsh, dp, dZ = qs.view(B, nh, dk), dconcat[:, :D].view(B, nh, dk), dconcat[:, D + S:]
    Wk, Wv, bkh = wk.view(nh, dk, D), wv.view(nh, dk, D), bk.view(nh, dk)
    t = 1.0 / math.sqrt(dk)

    def both(eq, x, y, xm=None, ym=None):
        return torch.einsum(eq, x, y), torch.einsum(eq, x.abs() if xm is None else xm, y.abs() if ym is None else ym)

    qk, qk_m = both("bhr,hrj->bhj", qsh, Wk)
    dxs, dxs_m = both("bhr,hrj->bhj", dp, Wv)
    da, da_m = both("bhj,bij->bhi", dxs, X, dxs_m, Xa)
    sdot, sdot_m = (a * da).sum(-1, keepdim=True), (a * da_m).sum(-1, keepdim=True)
    g, g_m = a * (da - sdot) * t, a * (da_m + sdot_m) * t
    xs, xs_m = both("bhi,bij->bhj", a, X, a, Xa)
    dX = torch.einsum("bhi,bhj->bij", a, dxs) + torch.einsum("bhi,bhj->bij", g, qk)
    dX_m = torch.einsum("bhi,bhj->bij", a, dxs_m) + torch.einsum("bhi,bhj->bij", g_m, qk_m)
    dX[:, 0] += dZ
    dX_m[:, 0] += dZ.abs()
    dqk, dqk_m = both("bhi,bij->bhj", g, X, g_m, Xa)
    dcst, dcst_m = g.sum(-1), g_m.sum(-1)
    dqs = (torch.einsum("hrj,bhj->bhr", Wk, dqk) + bkh * dcst.unsqueeze(-1)).reshape(B, D)
    dqs_m = (torch.einsum("hrj,bhj->bhr", Wk.abs(), dqk_m) + bkh.abs() * dcst_m.unsqueeze(-1)).reshape(B, D)
    dwk, dwk_m = (x.reshape(D, D) for x in both("bhr,bhj->hrj", qsh, dqk, None, dqk_m))
    dbk, dbk_m = (x.reshape(D) for x in both("bhr,bh->hr", qsh, dcst, None, dcst_m))
    dwv, dwv_m = (x.reshape(D, D) for x in both("bhr,bhj->hrj", dp, xs, None, xs_m))
    dbv, dbv_m = dp.reshape(B, D).sum(0), dp.reshape(B, D).abs().sum(0)
    # operations on the longest chain into each result: g_i takes dk (dxs), D (da_i) and n (sdot) sums, plus 3 for the
    # roundings of 1/sqrtf(dk), the subtraction and the products
    L_g = dk + D + L_n + 3
    out = {"dX": (dX, dX_m, L_g + 2 * nh + 1), "dqs": (dqs, dqs_m, L_g + L_n + D + 1), "dwk": (dwk, dwk_m, L_g + L_n + B),
           "dbk": (dbk, dbk_m, L_g + L_n + B), "dwv": (dwv, dwv_m, L_n + B), "dbv": (dbv, dbv_m, B)}
    res = {k: (v, bar(m, L)) for k, (v, m, L) in out.items()}
    res["mag"] = {k: m for k, (v, m, L) in out.items()}
    res["parts"] = {"qk": qk, "dxs": dxs, "xs": xs, "g": g, "dqk": dqk, "dcst": dcst}
    return res


def excess(got, ref, bound):
    """max(|got - ref| - bound): <= 0 within the bar.  Non-finite values fail."""
    got = got.detach().cpu().to(F64)
    assert got.shape == ref.shape, f"shape {tuple(got.shape)} vs {tuple(ref.shape)}"
    if not bool(torch.isfinite(got).all()):
        return float("inf")
    return float(((got - ref).abs() - bound).max()) if ref.numel() else -1.0


def tail_mask(lens, node_type):
    """The decoder tail's pool mask (O.decoder_pool_mask) on padded [B, n] node types."""
    return O.decoder_pool_mask(lens, node_type)
