"""Differentiable forward + backward of the QA-GNN message-passing path (SURVEY.md §8f #3).

What the reference does in `qagnn.py:249-278` (`model.train()`, `loss.backward()`) for this path:
dropout after every layer (`modeling_qagnn.py:49,93`), BatchNorm batch statistics in the shared
`edge_encoder` (`:30`) and in every layer's `mlp` (`:408`), and autograd through
`GATConvE.message` / `propagate` (`:442,455-484`).  The same functions serve an eval-mode module whose caller wants
gradients (fine-tuning the encoder under a frozen decoder, attributions): the modules' own mode then picks the reference's
eval semantics, dropout the identity and every BatchNorm on its running statistics, and no buffer is written.

Split here:
  * the graph part — logits, per-source softmax, out-degree rescale, per-target sum and ITS GRADIENT — runs in the
    hand-written kernels of libqagnn_b200.so (`qagnn_mp_core_forward` / `qagnn_mp_core_backward`, csrc/message_passing.cu,
    csrc/mp_backward.cu) behind one `torch.autograd.Function`;
  * the dense linears, BatchNorm and dropout around it are ordinary PyTorch ops on the GPU (library GEMMs), so their
    gradients come from autograd; the same node-level factorisation as the eval path is used (K/M/Q projections per node,
    the edge encoder evaluated once per distinct one-hot "combo"), which is algebraically the reference's per-edge form.

BatchNorm of the edge encoder: the reference feeds it one row per edge (E+N rows, `:433`), but a row only depends on the
edge's combo, so the batch mean / variance are the combo-histogram-weighted moments of the C distinct rows; the running
statistics receive the k momentum updates the reference's k calls of the shared module apply.
"""
import contextlib
import ctypes as C
import functools
import math
import threading

import torch
import torch.nn.functional as F

from . import _lib


@functools.lru_cache(maxsize=None)
def combo_onehot_table(n_ntype, n_etype, device):
    """[C, R+1+2T] one-hot edge-feature rows, one per combo index used by graph prep
    (c = (etype*T + type_src)*T + type_tgt for real edges, R*T*T + type for the self loop; modeling_qagnn.py:419-432).
    A constant: built once per (T, R, device) and shared, so a training step does not rebuild it (callers only read it)."""
    T, R = n_ntype, n_etype
    Cn = R * T * T + T
    c = torch.arange(Cn, device=device)
    real = c < R * T * T
    et = torch.where(real, c // (T * T), torch.full_like(c, R))
    ts = torch.where(real, (c // T) % T, c - R * T * T)
    tt = torch.where(real, c % T, c - R * T * T)
    tab = torch.zeros(Cn, R + 1 + 2 * T, device=device)
    tab[c, et] = 1.0
    tab[c, R + 1 + ts] = 1.0
    tab[c, R + 1 + T + tt] = 1.0
    return tab


def edge_table_train(enc, onehot_tab, combo_count, k_calls):
    """tab[c] = edge_encoder(onehot(c)) with BATCH statistics over the E' edges (each combo weighted by its edge count),
    plus the running-statistics update of `k_calls` forward calls of the shared module."""
    lin0, bn, lin3 = enc[0], enc[1], enc[3]
    # the moments are fp32 under any autocast: n = E' counts edge positions (> 65504 overflows fp16, bf16 rounds counts to
    # 8 bits), and h widens exactly, so only its own rounding to the autocast dtype remains
    h = lin0(onehot_tab)                                        # [C, D]
    if h.dtype in (torch.float16, torch.bfloat16):
        h = h.float()
    w = combo_count.to(h.dtype)
    n = w.sum()
    mean = (w[:, None] * h).sum(0) / n
    var = (w[:, None] * (h - mean) ** 2).sum(0) / n              # biased, as F.batch_norm normalises with
    y = (h - mean) * torch.rsqrt(var + bn.eps) * bn.weight + bn.bias
    with torch.no_grad():
        if bn.track_running_stats and bn.running_mean is not None:
            m = bn.momentum if bn.momentum is not None else 0.1
            keep = (1.0 - m) ** k_calls
            unbiased = torch.where(n > 1, var * (n / (n - 1.0)), var)  # tensor ops: no host synchronisation
            bn.running_mean.mul_(keep).add_(mean * (1.0 - keep))
            bn.running_var.mul_(keep).add_(unbiased * (1.0 - keep))
            bn.num_batches_tracked += k_calls
    return lin3(F.relu(y))


def edge_table(enc, onehot_tab, prep, k_calls):
    """tab[c] = edge_encoder(onehot(c)) [C, D] in the encoder's own mode: edge_table_train in .train(); in .eval() the module
    itself, whose BatchNorm uses its running statistics, so no combo histogram is needed and no buffer changes."""
    if enc.training:
        return edge_table_train(enc, onehot_tab, prep.combo_count(), k_calls)
    return enc(onehot_tab)


ANSWER_LOSSES = ("cross_entropy", "margin_rank")


def check_answer_loss(loss, num_choice):
    """ValueError unless answer_loss accepts (loss, num_choice)."""
    if loss not in ANSWER_LOSSES:
        raise ValueError(f"qagnn_b200: loss must be one of {ANSWER_LOSSES}, got {loss!r}")
    if loss == "margin_rank" and int(num_choice) < 2:  # the reference would take the mean of no pairs (NaN)
        raise ValueError(f"qagnn_b200: the margin-rank loss needs at least 2 choices, got num_choice = {int(num_choice)}")


def answer_loss(logits, labels, num_choice, loss="cross_entropy"):
    """The answer loss of qagnn.py:208-224 (`--loss cross_entropy` or `--loss margin_rank`) as a 0-dim tensor, from logits
    [bs * nc, 1] or [bs, nc] and labels int64 [bs] on the same device.  Static shapes, no host read and no data-dependent op,
    so it can be captured in a CUDA graph.

    "cross_entropy" is F.cross_entropy(logits.view(-1, nc), labels).  "margin_rank" pairs every question's correct logit
    with each of its nc - 1 wrong ones in the order the reference's boolean masks give (row-major, wrong choices in choice
    order), selected with gathers instead of masks, and calls the op nn.MarginRankingLoss(margin=0.1) calls on them.  Same
    op, same values, same order: the loss and its gradients equal the reference's bit for bit, under autocast too."""
    check_answer_loss(loss, num_choice)
    nc = int(num_choice)
    logits2d = logits.view(-1, nc)
    if loss == "cross_entropy":
        return F.cross_entropy(logits2d, labels)
    lab = labels.view(-1, 1)
    correct = logits2d.gather(1, lab).expand(-1, nc - 1).reshape(-1)
    j = torch.arange(nc - 1, device=logits.device)
    wrong = logits2d.gather(1, j + (j >= lab)).reshape(-1)  # choice j, or j + 1 from the correct one on
    y = wrong.new_ones((wrong.size(0),))
    return F.margin_ranking_loss(correct, wrong, y, margin=0.1)


def _core_dtype(*ts):
    """Storage dtype of one core call: the widest dtype of its operands (fp16 with bf16 widens to fp32).  Under autocast,
    operands of another floating dtype (fp64) are cast to fp32, as torch.amp.custom_fwd(cast_inputs=torch.float32) casts."""
    dt = functools.reduce(torch.promote_types, (t.dtype for t in ts))
    if dt not in _lib.DTYPE_CODES:
        if not torch.is_autocast_enabled("cuda"):
            raise TypeError(f"qagnn_b200: the message-passing core takes float32, float16 or bfloat16 operands (got {dt})")
        dt = torch.float32
    return dt


def _operand(t, dt, name):
    _lib.require_cuda(t, name)
    t = t.detach().to(dt).contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()  # the kernels read rows 4 elements at a time


class _MPCore(torch.autograd.Function):
    """aggr = propagate(...) on node-level projections; forward and backward in libqagnn_b200.so.

    Under torch.autocast (qagnn.py:91 runs the forward in fp16 autocast when --fp16 is set) the dense layers around this
    function hand it qkm / ke / me in the autocast dtype: the kernels read and write that dtype directly (no cast to fp32 and
    back around them) and compute in fp32 inside, like the reference's scatter ops do.  aggr and the three gradients come back
    in that dtype, rounded once from the fp32 results; alpha is fp32.  fp32 operands run the fp32 entry points.

    Under torch.use_deterministic_algorithms(True) the backward runs qagnn_mp_core_backward_det: d_ke / d_me are summed in an
    order fixed by the combo order instead of with float atomics, so every gradient is the same, bit for bit, on every run."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, qkm, ke, me, prep, shape_args, want_alpha):
        lib = _lib.load()
        dt = _core_dtype(qkm, ke, me)
        qkm_c, ke_c, me_c = _operand(qkm, dt, "qkm"), _operand(ke, dt, "ke"), _operand(me, dt, "me")
        N, E, D, H, T, R = shape_args
        dev = qkm_c.device
        shape = _lib.Shape(N, E, D, H, T, R, 1, 0)
        aggr = torch.empty(N, D, dtype=dt, device=dev)
        alpha_s = torch.empty(N + E, H, dtype=torch.float32, device=dev)
        alpha = torch.empty(N + E, H, dtype=torch.float32, device=dev) if want_alpha else None
        scratch = torch.empty(N + E, H, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            if dt == torch.float32:
                st = lib.qagnn_mp_core_forward(C.byref(shape), _lib.ptr(prep.buf), _lib.ptr(qkm_c), _lib.ptr(ke_c), _lib.ptr(me_c),
                                               _lib.ptr(aggr), _lib.ptr(alpha_s), _lib.ptr(alpha), _lib.ptr(scratch),
                                               _lib.stream_ptr(dev))
            else:
                st = lib.qagnn_mp_core_forward_typed(C.byref(shape), _lib.DTYPE_CODES[dt], _lib.ptr(prep.buf), _lib.ptr(qkm_c),
                                                     _lib.ptr(ke_c), _lib.ptr(me_c), _lib.ptr(aggr), _lib.ptr(alpha_s),
                                                     _lib.ptr(alpha), _lib.ptr(scratch), _lib.stream_ptr(dev))
        _lib.check(st, "qagnn_mp_core_forward")
        ctx.save_for_backward(qkm_c, ke_c, me_c, alpha_s)
        ctx.prep, ctx.shape_args = prep, shape_args
        if want_alpha:
            ctx.mark_non_differentiable(alpha)
            return aggr, alpha
        return aggr, None

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, d_aggr, _d_alpha):
        lib = _lib.load()
        qkm, ke, me, alpha_s = ctx.saved_tensors
        N, E, D, H, T, R = ctx.shape_args
        dt, dev = qkm.dtype, qkm.device
        shape = _lib.Shape(N, E, D, H, T, R, 1, 0)
        g = _operand(d_aggr, dt, "d_aggr")
        d_qkm = torch.empty_like(qkm)
        d_ke, d_me = torch.empty_like(ke), torch.empty_like(me)
        count, order = ctx.prep.combo_sort()  # device-side E': valid under an edge capacity without a host read
        with torch.cuda.device(dev):
            if torch.are_deterministic_algorithms_enabled():
                # d_ke / d_me summed in an order fixed by the combo order: the same bits on every run
                code = _lib.DTYPE_CODES[dt]
                nbytes = lib.qagnn_mp_core_backward_det_scratch_bytes(C.byref(shape), code)
                scratch = torch.empty(nbytes // 4, dtype=torch.float32, device=dev)
                st = lib.qagnn_mp_core_backward_det(C.byref(shape), code, _lib.ptr(ctx.prep.buf), _lib.ptr(order), _lib.ptr(count),
                                                    _lib.ptr(qkm), _lib.ptr(ke), _lib.ptr(me), _lib.ptr(alpha_s), _lib.ptr(g),
                                                    _lib.ptr(d_qkm), _lib.ptr(d_ke), _lib.ptr(d_me), _lib.ptr(scratch), nbytes,
                                                    _lib.stream_ptr(dev))
            elif dt == torch.float32:
                scratch = torch.empty(N + E, H, dtype=torch.float32, device=dev)
                st = lib.qagnn_mp_core_backward(C.byref(shape), _lib.ptr(ctx.prep.buf), _lib.ptr(order), _lib.ptr(qkm), _lib.ptr(ke),
                                                _lib.ptr(me), _lib.ptr(alpha_s), _lib.ptr(g), _lib.ptr(d_qkm), _lib.ptr(d_ke),
                                                _lib.ptr(d_me), _lib.ptr(scratch), _lib.stream_ptr(dev))
            else:
                code = _lib.DTYPE_CODES[dt]
                # [E+N, H] fp32 softmax gradients, then the fp32 accumulators of d_ke / d_me
                scratch = torch.empty(lib.qagnn_mp_core_scratch_bytes(C.byref(shape), code) // 4, dtype=torch.float32, device=dev)
                st = lib.qagnn_mp_core_backward_typed(C.byref(shape), code, _lib.ptr(ctx.prep.buf), _lib.ptr(order), _lib.ptr(qkm),
                                                      _lib.ptr(ke), _lib.ptr(me), _lib.ptr(alpha_s), _lib.ptr(g), _lib.ptr(d_qkm),
                                                      _lib.ptr(d_ke), _lib.ptr(d_me), _lib.ptr(scratch), _lib.stream_ptr(dev))
        _lib.check(st, "qagnn_mp_core_backward")
        return d_qkm, d_ke, d_me, None, None, None


def gatconve_autograd(layer, x, extra, node_type, prep, tab, return_attention_weights=False):
    """Differentiable GATConvE.forward (modeling_qagnn.py:411-452) given the edge table `tab` [C, D]; `layer.mlp`'s BatchNorm
    takes batch or running statistics by its mode.  Row-local apart from the message passing, so a ragged prep needs nothing
    more: x / extra are its [N_cap, D] packed rows."""
    D, H = layer.emb_dim, layer.head_count
    d = D // H
    x2 = torch.cat([x, extra], dim=1)                                        # :440
    wk, wm = layer.linear_key.weight, layer.linear_msg.weight
    q = layer.linear_query(x2) / (d ** 0.5)                                  # :466,:469
    kx = F.linear(x2, wk[:, :2 * D])                                         # node part of :464
    mx = F.linear(x2, wm[:, :2 * D])                                         # node part of :465
    ke = F.linear(tab, wk[:, 2 * D:], layer.linear_key.bias)                 # edge part of :464 (+ bias)
    me = F.linear(tab, wm[:, 2 * D:], layer.linear_msg.bias)                 # edge part of :465 (+ bias)
    qkm = torch.cat([q, kx, mx], dim=1)
    aggr, alpha = _MPCore.apply(qkm, ke, me, prep, (x.size(0), prep.E, D, H, layer.n_ntype, layer.n_etype),
                                return_attention_weights)
    out = layer.mlp(aggr)                                                    # :443
    if return_attention_weights:
        return out, (prep.edge_index_prime(), prep.compact_edges(alpha))
    return out


def mp_forward_autograd(mod, H, A, node_type, node_score, prep):
    """Differentiable QAGNN_Message_Passing.forward (modeling_qagnn.py:53-95) with the module's dropout and BatchNorm
    semantics.  H is [B, n, D], or a ragged batch's [N_cap, D] rows: every step around the message passing is row-local."""
    D = H.size(-1)
    nt = node_type.reshape(-1)
    T_ = F.one_hot(nt, mod.n_ntype).to(H.dtype)
    type_emb = mod.activation(mod.emb_node_type(T_))                         # :65-66
    js = mod._score_basis.to(H.device)                                       # 1.1^j, float32 as the reference computes it
    Bs = torch.sin(js.view(1, -1) * node_score.reshape(-1, 1))               # :70-72
    score_emb = mod.activation(mod.emb_score(Bs))                            # :73
    extra = torch.cat([type_emb, score_emb], dim=1)                          # :86
    tab = edge_table(mod.edge_encoder, combo_onehot_table(mod.n_ntype, mod.n_etype, H.device), prep, max(mod.k, 1))
    X = H.reshape(-1, D)
    if mod.training and keyed_active() and len(mod.gnn_layers) > MAX_GNN_LAYERS:
        raise ValueError(f"keyed dropout: {len(mod.gnn_layers)} message-passing layers; the site table has room for "
                         f"{MAX_GNN_LAYERS}")
    for l, layer in enumerate(mod.gnn_layers):                               # mp_helper :45-50
        X = mod.activation(gatconve_autograd(layer, X, extra, nt, prep, tab))
        X = dropout(X.view(H.shape), mod.dropout_rate, mod.training, SITE_GNN_LAYER + l).view(-1, D)
    out = mod.activation(mod.Vh(H) + mod.Vx(X.view(H.shape)))                # :92
    return dropout(out, mod.dropout.p, mod.dropout.training, SITE_GNN_OUT)   # :93


# ---- keyed dropout ------------------------------------------------------------------------------------------------------
# Under keyed_dropout, a training-mode dropout site of the decoder draws its mask from (seed, draw, question id, choice,
# site, element) instead of torch's generator, so a question's masks do not depend on which launches ran before it, on which
# stream or on which rank.  The site ids are part of the mask definition (DESIGN.md §2b).
SITE_EMB = 0          # QAGNN.dropout_e on the GNN input [B, n, D]
SITE_GNN_LAYER = 1    # + l: the dropout after message-passing layer l (l < 31)
SITE_GNN_OUT = 32     # QAGNN_Message_Passing.dropout on its output [B, n, D]
SITE_POOL_ATTN = 33   # MultiheadAttPoolLayer.attn_dropout on the attention [n_head, B, n]
SITE_POOL_OUT = 34    # MultiheadAttPoolLayer.dropout on the pooled [B, n_head d_v]
SITE_FC_IN = 35       # QAGNN.dropout_fc on the concat [B, 2D + S]
SITE_MLP = 36         # + i: the Dropout of MLP block i
MAX_GNN_LAYERS = SITE_GNN_OUT - SITE_GNN_LAYER

_keyed = threading.local()


class DropoutKey:
    """The key of keyed_dropout: a seed (0 <= seed < 2^64) and a device int64 `draw` counter [1] on `device`.  The masks of an
    optimiser batch are those of (seed, draw): advance the key once per optimiser batch, after the optimiser step.
    `advance_()` is one in-place add on the device, so it reads nothing on the host and may be captured; read `draw` on the
    host (int(key.draw)) for logs only.  Every rank of a data-parallel run builds the same key."""

    def __init__(self, seed, device):
        seed = int(seed)
        if not 0 <= seed < 2 ** 64:
            raise ValueError(f"DropoutKey: seed must be in [0, 2^64), got {seed}")
        device = torch.device(device)
        if device.type != "cuda":
            raise ValueError(f"DropoutKey: the key lives on a CUDA device, got {device}")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.seed, self.device = seed, device
        self.draw = torch.zeros(1, dtype=torch.int64, device=device)

    def advance_(self):
        self.draw.add_(1)
        return self


@contextlib.contextmanager
def keyed_dropout(key, question_ids, num_choice):
    """While active, the decoder's training-mode dropout sites draw keyed masks: element e of graph g (choice g % num_choice
    of question question_ids[g // num_choice], device int64 [B / num_choice]) at site s is kept or dropped by
    Philox4x32-10 under `key` (qagnn_keyed_dropout_forward_typed).  Outside it, and in .eval(), dropout is torch's."""
    nc = int(num_choice)
    if nc < 1:
        raise ValueError(f"keyed_dropout: num_choice = {nc}")
    if (not isinstance(question_ids, torch.Tensor) or question_ids.dtype != torch.int64 or question_ids.dim() != 1
            or question_ids.device != key.device):
        raise ValueError(f"keyed_dropout: question_ids must be a 1-d int64 tensor on the key's device {key.device}")
    prev = getattr(_keyed, "ctx", None)
    _keyed.ctx = (key, question_ids, nc)
    try:
        yield
    finally:
        _keyed.ctx = prev


def keyed_active():
    """True inside keyed_dropout."""
    return getattr(_keyed, "ctx", None) is not None


def dropout(x, p, training, site, graph_dim=0):
    """F.dropout(x, p, training); in training under keyed_dropout, the keyed mask of `site` instead.  x's dim `graph_dim` is
    the graph (0 for [B, ...], 1 for the pooler's [n_head, B, n]); the dims before it are A, those after it L."""
    ctx = getattr(_keyed, "ctx", None)
    if ctx is None or not training:
        return F.dropout(x, p, training)
    key, qids, nc = ctx
    p = float(p)
    if not 0.0 <= p <= 1.0:
        raise ValueError(f"keyed dropout: p = {p}; it must be in [0, 1]")
    if not 0 <= site <= 255:
        raise ValueError(f"keyed dropout: site {site} is outside [0, 255]")
    if x.device != key.device:
        raise ValueError(f"keyed dropout: the key is on {key.device}, the batch on {x.device}")
    G = x.size(graph_dim)
    if G != qids.numel() * nc:
        raise ValueError(f"keyed dropout: {qids.numel()} question ids with {nc} choices, the batch has {G} graphs")
    A = math.prod(x.shape[:graph_dim])
    return _KeyedDropout.apply(x, key, qids, nc, p, site, A, G)


class _KeyedDropout(torch.autograd.Function):
    """y = keyed dropout of x (qagnn_keyed_dropout_forward_typed); the backward reads only the forward's 1-bit keep mask."""

    @staticmethod
    def forward(ctx, x, key, qids, nc, p, site, A, G):
        if x.dtype not in _lib.DTYPE_CODES:
            raise TypeError(f"keyed dropout: float32, float16 or bfloat16 input, got {x.dtype}")
        lib = _lib.load()
        xc = x.detach().contiguous()
        n = xc.numel()
        L = n // (A * G) if A * G else 0
        y = torch.empty_like(xc)
        mask = torch.empty((n + 31) // 32, dtype=torch.int32, device=x.device)
        seed = key.seed - 2 ** 64 if key.seed >= 2 ** 63 else key.seed
        with torch.cuda.device(x.device):
            st = lib.qagnn_keyed_dropout_forward_typed(_lib.DTYPE_CODES[xc.dtype], A, G, L, p, seed, _lib.ptr(key.draw),
                                                       _lib.ptr(_lib.i64c(qids, "question_ids")), nc, site, _lib.ptr(xc),
                                                       _lib.ptr(y), _lib.ptr(mask), _lib.stream_ptr(x.device))
        _lib.check(st, "qagnn_keyed_dropout_forward_typed")
        ctx.save_for_backward(mask)
        ctx.p = p
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        lib = _lib.load()
        (mask,) = ctx.saved_tensors
        dyc = dy.contiguous()
        dx = torch.empty_like(dyc)
        with torch.cuda.device(dy.device):
            st = lib.qagnn_keyed_dropout_backward_typed(_lib.DTYPE_CODES[dyc.dtype], dyc.numel(), ctx.p, _lib.ptr(mask),
                                                        _lib.ptr(dyc), _lib.ptr(dx), _lib.stream_ptr(dy.device))
        _lib.check(st, "qagnn_keyed_dropout_backward_typed")
        return dx.view(dy.shape), None, None, None, None, None, None, None
