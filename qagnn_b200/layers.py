"""Small host-side layers around the hot path (the caller side of SURVEY.md §8b), kept as plain
PyTorch.  Constructor arguments and state_dict key names follow the reference's utils/layers.py
so checkpoints load unchanged:
    GELU                    utils/layers.py:10-22   (tanh approximation)
    MLP                     utils/layers.py:47-87   ('layers.{i}-Linear', '{i}-LayerNorm', ...)
    MultiheadAttPoolLayer   utils/layers.py:324-371 (+ MatrixVectorScaledDotProductAttention :276-299)
    CustomizedEmbedding     utils/layers.py:571-607
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import training as _training


# node-feature dtypes the fused pooling kernels read: fp32, and bf16 (the eval forward's output under bf16 autocast)
_POOL_X_DTYPES = (torch.float32, torch.bfloat16)


def gelu(x):
    """tanh-approximation GELU, the form the reference uses everywhere (utils/layers.py:10-14)."""
    return F.gelu(x, approximate="tanh")


class GELU(nn.Module):
    def forward(self, x):
        return gelu(x)


class MLP(nn.Module):
    """num_layers hidden blocks (Linear, Dropout, [BatchNorm1d | LayerNorm], activation) + output Linear."""
    _ACT = {"gelu": GELU, "relu": nn.ReLU, "tanh": nn.Tanh}

    def __init__(self, input_size, hidden_size, output_size, num_layers, dropout, batch_norm=False,
                 init_last_layer_bias_to_zero=False, layer_norm=False, activation="gelu"):
        super().__init__()
        if batch_norm and layer_norm:
            raise ValueError("batch_norm and layer_norm are mutually exclusive")
        self.input_size, self.hidden_size, self.output_size = input_size, hidden_size, output_size
        self.num_layers, self.dropout, self.batch_norm, self.layer_norm = num_layers, dropout, batch_norm, layer_norm
        blocks = nn.Sequential()
        width = input_size
        for i in range(num_layers):
            blocks.add_module(f"{i}-Linear", nn.Linear(width, hidden_size))
            blocks.add_module(f"{i}-Dropout", nn.Dropout(dropout))
            if batch_norm:
                blocks.add_module(f"{i}-BatchNorm1d", nn.BatchNorm1d(hidden_size))
            if layer_norm:
                blocks.add_module(f"{i}-LayerNorm", nn.LayerNorm(hidden_size))
            blocks.add_module(f"{i}-{activation}", self._ACT[activation.lower()]())
            width = hidden_size
        blocks.add_module(f"{num_layers}-Linear", nn.Linear(width, output_size))
        self.layers = blocks
        if init_last_layer_bias_to_zero:
            self.layers[-1].bias.data.zero_()

    def forward(self, x):
        for name, m in self.layers.named_children():  # block i's Dropout is keyed dropout site SITE_MLP + i
            x = (_training.dropout(x, m.p, m.training, _training.SITE_MLP + int(name.split("-")[0]))
                 if isinstance(m, nn.Dropout) else m(x))
        return x


class MultiheadAttPoolLayer(nn.Module):
    """Pools k [b, l, d_k_original] with a query q [b, d_q_original]: n_head scaled dot-product
    attentions over the l positions, masked positions excluded.  Returns (pooled [b, n_head*d_v],
    attn [n_head*b, l]) with the reference's head-major attn layout."""

    def __init__(self, n_head, d_q_original, d_k_original, dropout=0.1):
        super().__init__()
        if d_k_original % n_head != 0:
            raise ValueError("d_k_original must be divisible by n_head")
        self.n_head = n_head
        self.d_k = self.d_v = d_k_original // n_head
        self.w_qs = nn.Linear(d_q_original, n_head * self.d_k)
        self.w_ks = nn.Linear(d_k_original, n_head * self.d_k)
        self.w_vs = nn.Linear(d_k_original, n_head * self.d_v)
        nn.init.normal_(self.w_qs.weight, mean=0, std=math.sqrt(2.0 / (d_q_original + self.d_k)))
        nn.init.normal_(self.w_ks.weight, mean=0, std=math.sqrt(2.0 / (d_k_original + self.d_k)))
        nn.init.normal_(self.w_vs.weight, mean=0, std=math.sqrt(2.0 / (d_k_original + self.d_v)))
        self.temperature = math.sqrt(self.d_k)
        self.attn_dropout = nn.Dropout(0.1)  # MatrixVectorScaledDotProductAttention's own dropout
        self.dropout = nn.Dropout(dropout)
        # fewest nodes per graph the fused kernel has refused (its shared memory grows with the node count): longer inputs
        # go straight to the einsum path, shorter ones still try the kernel
        self._refused_len = None

    def _fused_may_take(self, l):
        return self._refused_len is None or l < self._refused_len

    def _note_refused(self, l):
        self._refused_len = l if self._refused_len is None else min(self._refused_len, l)

    def pool_concat(self, q, k, node_type, adj_lengths):
        """Eval-mode decoder tail in ONE kernel (qagnn_decoder_tail): derives the pool mask from adj_lengths / node_type,
        pools, and returns (cat(pooled, q, k[:, 0]) [b, 2*d_k_original + d_q_original], attn) — modeling_qagnn.py:172-187.
        Returns None when the fused kernel cannot take the shape (caller falls back to mask + forward + cat)."""
        if (self.training or not k.is_cuda or k.dtype not in _POOL_X_DTYPES or not self._fused_may_take(k.size(1))
                or (torch.is_grad_enabled() and (q.requires_grad or k.requires_grad))):
            return None
        from . import _lib
        lib = _lib.load()
        b, l, D = k.shape
        S = q.size(1)
        qc = _lib.f32c(q, "q")
        qs = self.w_qs(qc).detach().float().contiguous()  # fp32 for the kernel, also under autocast
        kc = k.detach().contiguous()  # fp32, or bf16 (the bf16 eval forward's output), widened exactly in the kernel
        concat = torch.empty(b, 2 * D + S, dtype=torch.float32, device=k.device)
        attn = torch.empty(self.n_head * b, l, dtype=torch.float32, device=k.device)
        with torch.cuda.device(k.device):
            st = lib.qagnn_decoder_tail_typed(_lib.DTYPE_CODES[kc.dtype], b, l, D, self.n_head, S, _lib.ptr(kc), _lib.ptr(qs),
                                              _lib.ptr(_lib.i64c(node_type, "node_type")),
                                              _lib.ptr(_lib.i64c(adj_lengths, "adj_lengths")), _lib.ptr(qc),
                                              _lib.ptr(self.w_ks.weight.detach()), _lib.ptr(self.w_ks.bias.detach()),
                                              _lib.ptr(self.w_vs.weight.detach()), _lib.ptr(self.w_vs.bias.detach()),
                                              _lib.ptr(concat), _lib.ptr(attn), _lib.stream_ptr(k.device))
        if st == -5:
            self._note_refused(l)
            return None
        _lib.check(st, "qagnn_decoder_tail")
        return concat, attn

    def pool_concat_ragged(self, q, k, node_ptr, node_type, adj_lengths, n):
        """pool_concat on a ragged batch (qagnn_decoder_tail_ragged): k [N_cap, D] and node_type [N_cap] are packed rows, graph b's
        from node_ptr[b] (device int64 [b + 1]); returns (concat [b, 2D + S], attn [n_head*b, n]) with attn exactly 0 at
        positions >= adj_lengths[b].  Raises where pool_concat would return None: there is no padded fallback.
        Differentiable in q, k and the w_qs / w_ks / w_vs parameters (qagnn_attention_pool_backward_ragged); attn is not."""
        from . import _lib
        if self.training or not k.is_cuda or k.dtype not in _POOL_X_DTYPES + (torch.float16,):
            raise ValueError("pool_concat_ragged: eval mode and a CUDA fp32 / bf16 / fp16 k only")
        if k.dtype == torch.float16:  # only the autograd decoder under fp16 autocast gives one: widened exactly
            k = k.float()
        _lib.f32c(q, "q")  # raises unless q is CUDA fp32: the kernel copies it into concat
        qs = self.w_qs(q).float()
        return _RaggedPoolConcat.apply(qs, k, q, self.w_ks.weight, self.w_ks.bias, self.w_vs.weight, self.w_vs.bias,
                                       (node_ptr, node_type, adj_lengths, n, self.n_head))

    def forward(self, q, k, mask=None):
        b, l, _ = k.shape
        nh, dk, dv = self.n_head, self.d_k, self.d_v
        wants_grad = torch.is_grad_enabled() and (q.requires_grad or k.requires_grad)  # the fused kernel is outside autograd
        if (k.is_cuda and not self.training and not wants_grad and mask is not None and k.dtype in _POOL_X_DTYPES
                and self.w_ks.weight.shape[0] == k.shape[2] and self._fused_may_take(l)):
            # fused kernel (one read of k, no ks/vs GEMMs): qagnn_attention_pool
            from . import _lib
            lib = _lib.load()
            qs = self.w_qs(q).float().contiguous()  # fp32 for the kernel, also under autocast
            kc = k.detach().contiguous()
            m8 = mask.to(torch.uint8).contiguous()
            pooled = torch.empty(b, nh * dv, dtype=torch.float32, device=k.device)
            attn = torch.empty(nh * b, l, dtype=torch.float32, device=k.device)
            with torch.cuda.device(k.device):
                st = lib.qagnn_attention_pool_typed(_lib.DTYPE_CODES[kc.dtype], b, l, k.shape[2], nh, _lib.ptr(kc),
                                                    _lib.ptr(qs.detach()), _lib.ptr(m8),
                                                    _lib.ptr(self.w_ks.weight.detach()), _lib.ptr(self.w_ks.bias.detach()),
                                                    _lib.ptr(self.w_vs.weight.detach()), _lib.ptr(self.w_vs.bias.detach()),
                                                    _lib.ptr(pooled), _lib.ptr(attn), _lib.stream_ptr(k.device))
            if st == -5:  # QAGNN_ERR_UNSUPPORTED (node tile does not fit in shared memory): the einsum path below
                self._note_refused(l)
            else:
                _lib.check(st, "qagnn_attention_pool")
                return pooled, attn
        qs = self.w_qs(q).view(b, nh, dk)
        ks = self.w_ks(k).view(b, l, nh, dk)
        vs = self.w_vs(k).view(b, l, nh, dv)
        logits = torch.einsum("bhd,blhd->hbl", qs, ks) / self.temperature
        if mask is not None:
            logits = logits.masked_fill(mask.unsqueeze(0), float("-inf"))
        attn = _training.dropout(torch.softmax(logits, dim=2), self.attn_dropout.p, self.attn_dropout.training,
                                 _training.SITE_POOL_ATTN, graph_dim=1)
        pooled = torch.einsum("hbl,blhd->bhd", attn, vs).reshape(b, nh * dv)
        return (_training.dropout(pooled, self.dropout.p, self.dropout.training, _training.SITE_POOL_OUT),
                attn.reshape(nh * b, l))


class _RaggedPoolConcat(torch.autograd.Function):
    """concat, attn = the ragged decoder tail (qagnn_decoder_tail_ragged) of qs = w_qs(q); its backward is
    qagnn_attention_pool_backward_ragged, whose sums run in a fixed order, so the gradients are the same bits on every run."""

    @staticmethod
    def forward(ctx, qs, k, q, wk, bk, wv, bv, batch):
        from . import _lib
        lib = _lib.load()
        node_ptr, node_type, adj_lengths, n, nh = batch
        N_cap, D = k.shape
        b, S = q.size(0), q.size(1)
        qc, qsc = _lib.f32c(q, "q"), _lib.f32c(qs, "qs")
        kc = k.detach().contiguous()
        node_ptr, adj_lengths = _lib.i64c(node_ptr, "node_ptr"), _lib.i64c(adj_lengths, "adj_lengths")
        wk, bk, wv, bv = (_lib.f32c(t, "pooler weight") for t in (wk, bk, wv, bv))
        concat = torch.empty(b, 2 * D + S, dtype=torch.float32, device=k.device)
        attn = torch.empty(nh * b, n, dtype=torch.float32, device=k.device)
        with torch.cuda.device(k.device):
            st = lib.qagnn_decoder_tail_ragged(_lib.DTYPE_CODES[kc.dtype], b, n, D, nh, S, N_cap, _lib.ptr(kc), _lib.ptr(node_ptr),
                                               _lib.ptr(qsc), _lib.ptr(_lib.i64c(node_type, "node_type")), _lib.ptr(adj_lengths),
                                               _lib.ptr(qc), _lib.ptr(wk), _lib.ptr(bk), _lib.ptr(wv), _lib.ptr(bv),
                                               _lib.ptr(concat), _lib.ptr(attn), _lib.stream_ptr(k.device))
        _lib.check(st, "qagnn_decoder_tail_ragged")
        if any(ctx.needs_input_grad):
            ctx.save_for_backward(qsc, kc, wk, bk, wv, attn, node_ptr, adj_lengths)
            ctx.dims = (b, n, D, nh, S, N_cap)
        ctx.mark_non_differentiable(attn)
        return concat, attn

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_concat, _d_attn):
        from . import _lib
        lib = _lib.load()
        qs, k, wk, bk, wv, attn, node_ptr, adj_lengths = ctx.saved_tensors
        b, n, D, nh, S, N_cap = ctx.dims
        dev = k.device
        g = d_concat.float().contiguous()
        dk = torch.empty(N_cap, D, dtype=torch.float32, device=dev)
        dqs = torch.empty(b, D, dtype=torch.float32, device=dev)
        dwk, dwv = torch.empty(D, D, dtype=torch.float32, device=dev), torch.empty(D, D, dtype=torch.float32, device=dev)
        dbk, dbv = torch.empty(D, dtype=torch.float32, device=dev), torch.empty(D, dtype=torch.float32, device=dev)
        nbytes = lib.qagnn_attention_pool_backward_ragged_scratch_bytes(b, n, D, nh)
        scratch = torch.empty(max(nbytes // 4, 1), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            st = lib.qagnn_attention_pool_backward_ragged(_lib.DTYPE_CODES[k.dtype], b, n, D, nh, S, N_cap, _lib.ptr(k),
                                                          _lib.ptr(node_ptr), _lib.ptr(adj_lengths), _lib.ptr(qs), _lib.ptr(wk),
                                                          _lib.ptr(bk), _lib.ptr(wv), _lib.ptr(attn), _lib.ptr(g), _lib.ptr(dk),
                                                          _lib.ptr(dqs), _lib.ptr(dwk), _lib.ptr(dbk), _lib.ptr(dwv), _lib.ptr(dbv),
                                                          _lib.ptr(scratch), nbytes, _lib.stream_ptr(dev))
        _lib.check(st, "qagnn_attention_pool_backward_ragged")
        return dqs, dk.to(k.dtype), g[:, D:D + S], dwk, dbk, dwv, dbv, None


class CustomizedEmbedding(nn.Module):
    """Concept embedding table with an optional Linear+GELU projection when the table width differs
    from the GNN width."""

    def __init__(self, concept_num, concept_in_dim, concept_out_dim, use_contextualized=False,
                 pretrained_concept_emb=None, freeze_ent_emb=True, scale=1.0, init_range=0.02):
        super().__init__()
        self.scale = scale
        self.use_contextualized = use_contextualized
        if not use_contextualized:
            self.emb = nn.Embedding(concept_num, concept_in_dim)
            if pretrained_concept_emb is not None:
                self.emb.weight.data.copy_(pretrained_concept_emb)
            else:
                self.emb.weight.data.normal_(mean=0.0, std=init_range)
            if freeze_ent_emb:
                for p in self.emb.parameters():
                    p.requires_grad = False
        if concept_in_dim != concept_out_dim:
            self.cpt_transform = nn.Linear(concept_in_dim, concept_out_dim)
            self.activation = GELU()

    def _project(self, e):
        e = e * self.scale
        if not hasattr(self, "cpt_transform"):
            return e
        lin = self.cpt_transform
        if (e.is_cuda and not self.training and not torch.is_grad_enabled() and e.dtype == torch.float32
                and lin.in_features % 8 == 0 and lin.out_features >= 8):
            # GELU(cpt_transform(e)) on the wgmma split-bf16 GEMM with the activation fused in the epilogue: the
            # [B*(n-1), concept_in_dim] x [concept_in_dim, concept_dim] product is the largest dense op outside the GNN
            from . import ops
            try:
                out = ops.linear_bf16x3(e.reshape(-1, lin.in_features), lin.weight, lin.bias, act="gelu")
                return out.view(*e.shape[:-1], lin.out_features)
            except Exception as exc:  # tensor-core path not available for this shape/driver: plain PyTorch (same math)
                if "unsupported" not in str(exc).lower():
                    raise
        return self.activation(lin(e))

    def projected_table(self):
        """[concept_num, concept_out_dim] = the whole table pushed through scale / cpt_transform / GELU, cached per weight
        version (eval mode: the embedding is frozen and the projection fixed, so a forward becomes a pure row gather).
        `invalidate_table()` after in-place `.data` edits."""
        srcs = [self.emb.weight] + ([self.cpt_transform.weight, self.cpt_transform.bias] if hasattr(self, "cpt_transform") else [])
        key = tuple((t.data_ptr(), t._version, tuple(t.shape)) for t in srcs)
        if getattr(self, "_ptab_key", None) != key:
            # fp32 whatever autocast the caller runs under: the head kernel reads the table as fp32, and the cache outlives
            # the call that fills it
            with torch.no_grad(), torch.autocast("cuda", enabled=False):
                w = self.emb.weight
                rows = [self._project(w[i:i + 65536]) for i in range(0, w.size(0), 65536)]  # chunks bound the GEMM workspace
                self._ptab = torch.cat(rows).contiguous()
            self._ptab_key = key
        return self._ptab

    def invalidate_table(self):
        self._ptab_key = None

    def forward(self, index, contextualized_emb=None):
        if contextualized_emb is not None:
            if index.size(0) != contextualized_emb.size(0):
                raise ValueError("batch size mismatch between index and contextualized_emb")
            table = self._project(contextualized_emb)
            return table.gather(1, index.unsqueeze(-1).expand(-1, -1, table.size(-1)))
        return self._project(self.emb(index))
