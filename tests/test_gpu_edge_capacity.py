"""Packed batches at a fixed edge capacity K on the GPU: graph prep reads the real edge count from graph_ptr on the device,
so a batch in a [3, K] buffer computes exactly what the same batch packed without spare columns computes, and one captured
DecoderStep serves every batch of a split.  Batches come from a loader-shaped synthetic split
(data.synth_adj_pickle -> load_flat_adj_cache).  Needs a GPU: run with -m gpu."""
import copy

import numpy as np
import pytest
import torch

import qagnn_b200
from oracle import qagnn_oracle as O
from qagnn_b200 import data as Dt
from qagnn_b200.modeling_qagnn import GraphPrep
from qagnn_b200.pipeline import DecoderStep, StreamedRunner, packed_host_batch
from tests import helpers as Hh

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N_NODE, NC, BS, D, K_LAYERS, T, R, S = 200, 5, 4, 200, 3, 4, 38, 96


@pytest.fixture(scope="module")
def split(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("split") / "dev.graph.adj.pk")
    Dt.synth_adj_pickle(path, 24 * NC, seed=21)
    cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N_NODE, NC)
    return ntypes, scores, lens, flat


def _batch(split, qs, capacity, seed):
    """(host PackedAdj at `capacity` (None: exact), host dict of the decoder inputs) of questions `qs`."""
    ntypes, scores, lens, flat = split
    adj = flat.pack(np.asarray(qs), pin=False, edge_capacity=capacity)
    B = len(qs) * NC
    g = torch.Generator().manual_seed(seed)
    host = packed_host_batch(adj, torch.randn(B, N_NODE, D, generator=g), ntypes[qs], scores[qs],
                             torch.randn(B, S, generator=g) * 0.5, lens[qs])
    return adj, host


def _dev_adj(adj, max_edges=-1):
    a = adj.to(DEV)
    if max_edges >= 0:
        a.max_edges = max_edges
    return a


def _module(seed=5, dropout=0.1):
    sd = O.random_state_dict(K_LAYERS, D, T, R, "prod", seed=seed)
    mod = qagnn_b200.QAGNN_Message_Passing(None, K_LAYERS, T, R, D, D, D, dropout=dropout).eval()
    mod.load_state_dict(sd)
    return mod.to(DEV), sd


def _tail():
    from qagnn_b200.layers import MLP, MultiheadAttPoolLayer
    torch.manual_seed(4)
    return (MultiheadAttPoolLayer(2, S, D).eval().to(DEV), MLP(D + S + D, D, 1, 0, 0.2, layer_norm=True).eval().to(DEV))


PREP_CSR = ("csr_src_tgt", "csr_src_combo", "csr_tgt_src", "csr_tgt_combo", "csr_tgt_apos", "csr_src_tpos", "pk_src", "pk_tgt")


def _prep(adj_dev, node_type):
    return GraphPrep(adj_dev.edge_index, adj_dev.edge_type, node_type.reshape(-1).to(DEV), T, R, N_NODE,
                     graph_ptr=adj_dev.graph_ptr_dev, max_edges=adj_dev.max_edges)


@pytest.mark.parametrize("spare", [0, 1, 997])
def test_prep_arrays_at_capacity_equal_the_exact_packing(split, spare):
    qs = [3, 7, 11, 19]
    exact, host = _batch(split, qs, None, 0)
    E = exact.n_edges
    cap, _ = _batch(split, qs, E + spare, 0)
    K, N = E + spare, len(qs) * NC * N_NODE
    pe, pc = _prep(_dev_adj(exact), host["node_type"]), _prep(_dev_adj(cap), host["node_type"])
    assert pc.packed and pc.E == K and pc.real_edges() == E
    a = {k: pe.array(k).cpu() for k in ("src", "tgt", "combo", "perm_src", "perm_tgt", "rowptr_src", "rowptr_tgt") + PREP_CSR}
    b = {k: pc.array(k).cpu() for k in a}
    Ep = E + N
    assert int(pc.status_word().item()) == 0
    assert torch.equal(a["rowptr_src"], b["rowptr_src"]) and torch.equal(a["rowptr_tgt"], b["rowptr_tgt"])
    assert int(b["rowptr_src"][N]) == int(b["rowptr_tgt"][N]) == E + N
    for k in PREP_CSR:
        assert torch.equal(a[k][:Ep], b[k][:Ep]), k
    for k in ("perm_src", "perm_tgt"):  # self loops keep the ids E + v with E the capacity
        want = torch.where(a[k][:Ep] >= E, a[k][:Ep] + spare, a[k][:Ep])
        assert torch.equal(b[k][:Ep], want), k
    for k in ("src", "tgt", "combo"):
        assert torch.equal(b[k][:E], a[k][:E]) and torch.equal(b[k][K:], a[k][E:]), k
        assert bool((b[k][E:K] == -1).all()), k
    if spare == 0:  # a full buffer is exactly today's packing, which is the oracle's
        ref = O.graph_prep_oracle(exact.edge_index, exact.edge_type, host["node_type"].reshape(-1), T, R)
        for k in ("src", "tgt", "combo", "rowptr_src", "rowptr_tgt", "perm_src", "perm_tgt"):
            assert np.array_equal(b[k].numpy().astype(np.int64), ref[k]), k
    assert torch.equal(pc.edge_index_prime().cpu(), pe.edge_index_prime().cpu())
    assert torch.equal(pc.combo_count().cpu(), pe.combo_count().cpu())
    assert torch.equal(pc.combo_order().cpu(), pe.combo_order().cpu())


@pytest.mark.parametrize("two_cta", [None, "0"])
@pytest.mark.parametrize("path", [None, "csr", "basic"])
def test_eval_forward_at_capacity_is_bitwise_the_exact_batch(split, monkeypatch, path, two_cta):
    for var, val in (("QAGNN_MP_PATH", path), ("QAGNN_TC_2CTA", two_cta)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, val)
    mod, _ = _module()
    qs = [0, 5, 9, 14]
    exact, host = _batch(split, qs, None, 1)
    cap, _ = _batch(split, qs, exact.n_edges + 613, 1)
    H, nt, sc = host["H"].to(DEV), host["node_type"].to(DEV), host["node_score"].to(DEV)
    with torch.no_grad():
        out_e, lay_e = mod(H, _dev_adj(exact), nt, sc, return_layers=True)
        out_c, lay_c = mod(H, _dev_adj(cap), nt, sc, return_layers=True)
        assert torch.equal(out_e, out_c) and torch.equal(lay_e, lay_c)
        layer = mod.gnn_layers[1]
        extra = mod.node_feature_extra(nt, sc)
        x = lay_e[0]
        ye = layer(x, _dev_adj(exact), None, nt.reshape(-1), extra)
        yc = layer(x, _dev_adj(cap), None, nt.reshape(-1), extra)
        assert torch.equal(ye, yc)
        ye, (eie, ae) = layer(x, _dev_adj(exact), None, nt.reshape(-1), extra, return_attention_weights=True)
        yc, (eic, ac) = layer(x, _dev_adj(cap), None, nt.reshape(-1), extra, return_attention_weights=True)
    E, N = exact.n_edges, nt.numel()
    assert ac.shape == (E + N, layer.head_count) and eic.shape == (2, E + N)
    assert torch.equal(ye, yc) and torch.equal(ae, ac) and torch.equal(eie, eic)


def _split_batches(split, K_seed=0):
    ntypes, scores, lens, flat = split
    rng = np.random.default_rng(K_seed)
    order = rng.permutation(flat.n_questions())
    return [sorted(order[i:i + BS].tolist()) for i in range(0, len(order) - BS + 1, BS)]


def _eager_ref(mod, pooler, fc, host):
    d = {k: v.to(DEV) for k, v in host.items()}
    gp = host["graph_ptr"]
    step = DecoderStep(mod, pooler, fc, d, use_cuda_graph=False, max_edges=int((gp[1:] - gp[:-1]).max()))
    return [t.clone() for t in step.run()]


def test_one_captured_decoder_step_serves_every_batch_of_the_split(split):
    ntypes, scores, lens, flat = split
    mod, sd = _module()
    pooler, fc = _tail()
    K, M = flat.max_batch_edges(BS), flat.max_graph_edges()
    qsets = _split_batches(split)[:5]
    cap_hosts, exact_hosts = [], []
    for i, qs in enumerate(qsets):
        cap_hosts.append(_batch(split, qs, K, 100 + i)[1])
        exact_hosts.append(_batch(split, qs, None, 100 + i)[1])
    assert len({int(h["graph_ptr"][-1]) for h in cap_hosts}) >= 4  # different edge counts, one buffer width
    d = {k: v.to(DEV) for k, v in cap_hosts[0].items()}
    step = DecoderStep(mod, pooler, fc, d, use_cuda_graph=True, max_edges=M)
    assert step.graph is not None
    refs = []
    for i, (hc, he) in enumerate(zip(cap_hosts, exact_hosts)):
        for k in DecoderStep.PACKED_FIELDS:
            d[k].copy_(hc[k])
        got = [t.clone() for t in step.run()]
        ref = _eager_ref(mod, pooler, fc, he)
        refs.append(ref)
        for name, a, b in zip(("logits", "pool_attn", "gnn_out"), got, ref):
            assert torch.equal(a, b), f"batch {i}: {name}"
        if i == 1:  # first and last 4 graphs against the fp64-capable oracle
            B = he["H"].size(0)
            gp = he["graph_ptr"]
            ei = torch.cat([he["edge_index"], he["edge_type"].unsqueeze(0)])
            for g0 in (0, B - 4):
                e0, e1 = int(gp[g0]), int(gp[g0 + 4])
                ref_out = O.message_passing_forward(sd, he["H"][g0:g0 + 4], ei[:2, e0:e1] - g0 * N_NODE, ei[2, e0:e1],
                                                    he["node_type"][g0:g0 + 4], he["node_score"][g0:g0 + 4], K_LAYERS, T, R)
                Hh.assert_close(got[2][g0:g0 + 4], ref_out, f"gnn_out graphs {g0}..{g0 + 3}")
    # the streaming API over the same batches, two buffer sets, one capture each
    runner = StreamedRunner(mod, cap_hosts[0], torch.device(DEV), depth=2, fields=DecoderStep.PACKED_FIELDS,
                            make_step=lambda dv: DecoderStep(mod, pooler, fc, dv, use_cuda_graph=True, max_edges=M),
                            download=(0, 1, 2))
    got = []
    for i, hb in enumerate(cap_hosts):
        runner.submit(hb)
        if i >= 1:
            prev = (i - 1) % 2
            runner.ev_down[prev].synchronize()
            got.append([t.clone() for t in runner.host_out[prev]])
    runner.drain()
    torch.cuda.synchronize()
    got.append([t.clone() for t in runner.host_out[(len(cap_hosts) - 1) % 2]])
    for i, (g, r) in enumerate(zip(got, refs)):
        for a, b in zip(g, r):
            assert torch.equal(a, b.cpu()), f"streamed batch {i}"


def test_replayed_step_reports_bad_indices_and_ignores_the_spare_columns(split):
    mod, _ = _module()
    pooler, fc = _tail()
    ntypes, scores, lens, flat = split
    K, M = flat.max_batch_edges(BS), flat.max_graph_edges()
    qsets = _split_batches(split, 1)
    h0 = _batch(split, qsets[0], K, 7)[1]
    d = {k: v.to(DEV) for k, v in h0.items()}
    step = DecoderStep(mod, pooler, fc, d, use_cuda_graph=True, max_edges=M)
    # garbage past graph_ptr[-1]: never read, no status bit, same results as the exact batch
    hc = _batch(split, qsets[1], K, 8)[1]
    E = int(hc["graph_ptr"][-1])
    assert E < K
    hc["edge_index"][:, E:] = -12345
    hc["edge_type"][E:] = 10 ** 9
    for k in DecoderStep.PACKED_FIELDS:
        d[k].copy_(hc[k])
    got = [t.clone() for t in step.run()]
    torch.cuda.synchronize()
    step.run()  # the previous replay's status word has landed: nothing to report
    torch.cuda.synchronize()
    ref = _eager_ref(mod, pooler, fc, _batch(split, qsets[1], None, 8)[1])
    for a, b in zip(got, ref):
        assert torch.equal(a, b)
    # an out-of-range source inside the real range: IndexError at the next call
    bad = _batch(split, qsets[2], K, 9)[1]
    bad["edge_index"][0, int(bad["graph_ptr"][-1]) // 2] = 10 ** 7
    for k in DecoderStep.PACKED_FIELDS:
        d[k].copy_(bad[k])
    step.run()
    torch.cuda.synchronize()
    with pytest.raises(IndexError):
        step.run()


def test_training_at_capacity_is_bitwise_the_exact_batch(split):
    base, _ = _module(seed=9, dropout=0.0)
    qs = [2, 4, 6, 8]
    exact, host = _batch(split, qs, None, 3)
    cap, _ = _batch(split, qs, exact.n_edges + 301, 3)
    w = torch.randn(len(qs) * NC, N_NODE, D, generator=torch.Generator().manual_seed(1)).to(DEV)

    def run(adj):
        mod = copy.deepcopy(base).train()
        H = host["H"].to(DEV).requires_grad_(True)
        out = mod(H, _dev_adj(adj), host["node_type"].to(DEV), host["node_score"].to(DEV))
        (out * w).sum().backward()
        grads = {n: p.grad.clone() for n, p in mod.named_parameters() if p.grad is not None}
        grads["H"] = H.grad.clone()
        return out.detach(), grads

    out_e, g_e = run(exact)
    out_e2, g_e2 = run(exact)
    out_c, g_c = run(cap)
    assert torch.equal(out_e, out_c)
    assert g_e.keys() == g_c.keys() and len(g_e) > 10
    for name in g_e:
        # the edge-table gradients are summed with float atomics: where the exact batch itself is not run-to-run
        # reproducible, the capacity batch has to stay within that spread
        spread = (g_e[name] - g_e2[name]).abs().max().item()
        err = (g_e[name] - g_c[name]).abs().max().item()
        assert err <= 4 * spread, f"{name}: {err:.3e} vs run-to-run {spread:.3e}"
