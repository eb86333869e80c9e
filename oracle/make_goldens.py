"""TEST INFRASTRUCTURE — mints tests/golden/*.pt from the reference's OWN modules.

Run in the build container only (needs /root/reference):

    python -m oracle.make_goldens            # writes tests/golden/*.pt and the stored reference data under tests/golden/ref/
    python -m oracle.make_goldens --check    # re-mints in memory, compares with the committed files, writes nothing
    python -m oracle.make_goldens --fuzz 24  # reference vs oracle on 24 random cases that are not committed as fixtures

Every fixture is produced by the unmodified `GATConvE` / `QAGNN_Message_Passing` / `QAGNN`
classes of /root/reference/modeling/modeling_qagnn.py (imported through oracle/ref_shim.py),
in eval mode, fp32, on CPU.  Inputs and weights are regenerated deterministically from seeds by
`oracle.qagnn_oracle.synth_graph_batch` / `random_state_dict`, so the fixtures only store the
case description, a fingerprint of the regenerated inputs, and the reference outputs.
"""
import hashlib
import os
import sys

import torch

from oracle import qagnn_oracle as O
from oracle.ref_shim import load_reference

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
# what the tests compare against the reference's own loader / batch generator and its fuzz cases, stored so that the
# tests run without the reference tree (tests/test_loader_cpu.py, tests/test_oracle_golden.py)
REF_DATA_DIR = os.path.join(GOLDEN_DIR, "ref")
FUZZ_FILE = os.path.join(REF_DATA_DIR, "fuzz24.pt")
LOADER_FILE = os.path.join(REF_DATA_DIR, "loader.pt")
FUZZ_SAMPLES = 32  # values kept per compared tensor (a seeded sample: the full outputs would not be small)


def fingerprint(*tensors):
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()[:16]


# ---------------------------------------------------------------------------------------------
# case table (shared with the tests through the saved 'case' dict).  A case without n_ntype / n_etype is minted at the
# reference's (4, 38); the fixture records the pair it was minted at either way.
# ---------------------------------------------------------------------------------------------
MP_CASES = [
    # name, B, n, e/graph, D, k, regime, realistic, seed
    dict(name="cfg1_prod", B=4, n=50, e=200, D=64, k=1, regime="prod", realistic=False, seed=0),
    dict(name="cfg1_peaky_k2", B=4, n=50, e=200, D=64, k=2, regime="peaky", realistic=False, seed=1),
    dict(name="cfg2small_prod", B=3, n=200, e=1000, D=200, k=5, regime="prod", realistic=False, seed=0),
    dict(name="cfg2small_peaky", B=3, n=200, e=1000, D=200, k=5, regime="peaky", realistic=False, seed=2),
    dict(name="cfg2small_realistic", B=5, n=200, e=1000, D=200, k=5, regime="peaky", realistic=True, seed=3),
    dict(name="tiny_realistic_d100", B=6, n=24, e=60, D=100, k=3, regime="peaky", realistic=True, seed=4),
    dict(name="no_edges", B=3, n=10, e=0, D=64, k=2, regime="peaky", realistic=False, seed=5),
    # six node types and five relations (C = R*T*T + T = 186): node types come from all of [0, T)
    dict(name="mp_t6_r5", B=3, n=40, e=150, D=64, k=2, regime="peaky", realistic=False, seed=6, n_ntype=6, n_etype=5),
]

# single-layer GATConvE cases (hand-built graphs and non-default head counts)
LAYER_CASES = [
    dict(name="layer_h8_d1024", N=40, E=300, D=1024, H=8, regime="peaky", seed=10, kind="random"),
    dict(name="layer_h8_d64", N=30, E=200, D=64, H=8, regime="peaky", seed=11, kind="random"),
    dict(name="layer_h4_d200_prod", N=200, E=1000, D=200, H=4, regime="prod", seed=12, kind="random"),
    dict(name="layer_multi_dup", N=12, E=0, D=64, H=4, regime="peaky", seed=13, kind="multi_dup"),
    dict(name="layer_src_only_tgt_only", N=9, E=0, D=64, H=4, regime="peaky", seed=14, kind="bipartite"),
    dict(name="layer_hub", N=300, E=0, D=64, H=4, regime="peaky", seed=15, kind="hub"),
    dict(name="layer_single_node", N=1, E=0, D=64, H=4, regime="peaky", seed=16, kind="random"),
    # other (node type, relation) counts T, R: the combo count C = R*T*T + T sizes every edge table
    dict(name="layer_t1_r5", N=120, E=600, D=64, H=4, regime="peaky", seed=17, kind="random", n_ntype=1, n_etype=5),
    dict(name="layer_t7_r3", N=120, E=600, D=64, H=4, regime="peaky", seed=18, kind="random", n_ntype=7, n_etype=3),
    dict(name="layer_t16_r23", N=120, E=600, D=64, H=4, regime="peaky", seed=19, kind="random", n_ntype=16, n_etype=23),
]


def build_layer_inputs(case, n_ntype=4, n_etype=38):
    g = torch.Generator().manual_seed(500 + case["seed"])
    N, D = case["N"], case["D"]
    x = torch.randn(N, D, generator=g) * 0.5
    extra = torch.randn(N, D, generator=g) * 0.5
    node_type = torch.randint(0, n_ntype, (N,), generator=g)
    kind = case["kind"]
    if kind == "random":
        E = case["E"]
        ei = torch.randint(0, N, (2, E), generator=g)
        et = torch.randint(0, n_etype, (E,), generator=g)
    elif kind == "multi_dup":
        # parallel multi-edges of different type between the same pair, exact duplicates, explicit i->i
        pairs = [(0, 1, 3), (0, 1, 7), (0, 1, 7), (0, 1, 7), (1, 0, 22), (2, 2, 5), (2, 2, 5), (3, 4, 0),
                 (3, 4, 37), (4, 3, 19), (5, 6, 1), (5, 6, 1), (11, 0, 9), (11, 0, 9), (11, 0, 10)]
        ei = torch.tensor([[p[0] for p in pairs], [p[1] for p in pairs]])
        et = torch.tensor([p[2] for p in pairs])
    elif kind == "bipartite":
        # nodes 0-3 only ever sources, 4-7 only ever targets, node 8 isolated (self loop only)
        s = torch.tensor([0, 0, 1, 2, 3, 3, 3, 1])
        t = torch.tensor([4, 5, 5, 6, 7, 4, 5, 7])
        ei = torch.stack([s, t])
        et = torch.randint(0, n_etype, (s.numel(),), generator=g)
    elif kind == "hub":
        # node 0 points at everybody (out-degree N) and half of them point back (in-degree N/2)
        s = torch.cat([torch.zeros(N - 1, dtype=torch.long), torch.arange(1, N, 2)])
        t = torch.cat([torch.arange(1, N), torch.zeros(len(range(1, N, 2)), dtype=torch.long)])
        ei = torch.stack([s, t])
        et = torch.randint(0, n_etype, (s.numel(),), generator=g)
    else:
        raise ValueError(kind)
    return x, extra, node_type, ei.long().contiguous(), et.long().contiguous()


def layer_state_dict(case, n_ntype=4, n_etype=38):
    full = O.random_state_dict(1, case["D"], n_ntype, n_etype, case["regime"], case["seed"])
    return full


@torch.no_grad()
def mint_mp_case(ref, case, n_ntype=4, n_etype=38):
    inp = O.synth_graph_batch(case["B"], case["n"], case["e"], case["D"], n_etype, case["seed"], case["realistic"], n_ntype)
    sd = O.random_state_dict(case["k"], case["D"], n_ntype, n_etype, case["regime"], case["seed"])
    mod = ref.QAGNN_Message_Passing(None, k=case["k"], n_ntype=n_ntype, n_etype=n_etype, input_size=case["D"],
                                    hidden_size=case["D"], output_size=case["D"], dropout=0.2)
    missing = mod.load_state_dict(sd, strict=True)
    mod.eval()
    adj = (inp["edge_index"], inp["edge_type"])
    out = mod(inp["H"], adj, inp["node_type"], inp["node_score"])
    # per-layer trace through the reference's own layers (same code path as mp_helper :45-50)
    T = ref.make_one_hot(inp["node_type"].view(-1), n_ntype).view(case["B"], case["n"], n_ntype)
    type_emb = mod.activation(mod.emb_node_type(T))
    js = torch.pow(1.1, torch.arange(case["D"] // 2).unsqueeze(0).unsqueeze(0).float())
    score_emb = mod.activation(mod.emb_score(torch.sin(js * inp["node_score"])))
    extra = torch.cat([type_emb, score_emb], dim=2).view(case["B"] * case["n"], -1).contiguous()
    X = inp["H"].view(-1, case["D"]).contiguous()
    nt = inp["node_type"].view(-1)
    layers = []
    for l in range(case["k"]):
        X, (ei2, alpha) = mod.gnn_layers[l](X, inp["edge_index"], inp["edge_type"], nt, extra,
                                            return_attention_weights=True)
        X = mod.activation(X)
        layers.append({"x": X.clone(), "alpha": alpha.clone()})
    keep = [0, case["k"] - 1] if case["k"] > 1 else [0]
    fx = {
        "kind": "mp", "case": case, "n_ntype": n_ntype, "n_etype": n_etype,
        "input_fp": fingerprint(inp["H"], inp["edge_index"], inp["edge_type"], inp["node_type"], inp["node_score"]),
        "weight_fp": fingerprint(*[sd[k_] for k_ in sorted(sd) if sd[k_].dtype.is_floating_point]),
        "out": out.clone(), "extra": extra.clone(), "edge_index_prime": ei2.clone(),
        "layers": {l: layers[l] for l in keep},
        "state_dict_keys": sorted(mod.state_dict().keys()),
    }
    return fx


@torch.no_grad()
def mint_layer_case(ref, case, n_ntype=4, n_etype=38):
    x, extra, node_type, ei, et = build_layer_inputs(case, n_ntype, n_etype)
    sd = layer_state_dict(case, n_ntype, n_etype)
    D = case["D"]
    enc = torch.nn.Sequential(torch.nn.Linear(n_etype + 1 + n_ntype * 2, D), torch.nn.BatchNorm1d(D),
                              torch.nn.ReLU(), torch.nn.Linear(D, D))
    layer = ref.GATConvE(None, D, n_ntype, n_etype, enc, head_count=case["H"])
    lsd = {k_[len("gnn_layers.0."):]: v for k_, v in sd.items() if k_.startswith("gnn_layers.0.")}
    layer.load_state_dict(lsd, strict=True)
    layer.eval()
    out, (ei2, alpha) = layer(x, ei, et, node_type, extra, return_attention_weights=True)
    return {"kind": "layer", "case": case, "n_ntype": n_ntype, "n_etype": n_etype,
            "input_fp": fingerprint(x, extra, node_type, ei, et),
            "out": out.clone(), "alpha": alpha.clone(), "edge_index_prime": ei2.clone()}


DEC_CASES = [
    dict(name="decoder_small", B=6, n=30, e=80, D=64, k=2, sent_dim=48, n_concept=500, concept_in_dim=32,
         n_head=2, n_fc_layer=0, regime="peaky", seed=20),
    dict(name="decoder_fc1", B=4, n=20, e=50, D=100, k=2, sent_dim=64, n_concept=300, concept_in_dim=100,
         n_head=2, n_fc_layer=1, regime="peaky", seed=21),
]


def build_decoder_inputs(case, n_etype=38):
    inp = O.synth_graph_batch(case["B"], case["n"], case["e"], case["D"], n_etype, case["seed"], realistic=True)
    g = torch.Generator().manual_seed(700 + case["seed"])
    sent_vecs = torch.randn(case["B"], case["sent_dim"], generator=g)
    concept_ids = torch.randint(1, case["n_concept"] + 1, (case["B"], case["n"]), generator=g)
    concept_ids[:, 0] = 0
    for b in range(case["B"]):
        concept_ids[b, int(inp["adj_lengths"][b]):] = 1
    return inp, sent_vecs, concept_ids


def decoder_state_dict(ref_module, case):
    """Random (seeded) values for every tensor of the reference decoder, 'peaky' style."""
    g = torch.Generator().manual_seed(900 + case["seed"])
    gnn_sd = O.random_state_dict(case["k"], case["D"], 4, 38, case["regime"], case["seed"])
    sd = {}
    for key, v in ref_module.state_dict().items():
        if key.startswith("gnn."):
            sd[key] = gnn_sd[key[4:]].clone()
        elif not v.dtype.is_floating_point:
            sd[key] = v.clone()
        elif key.endswith("running_var"):
            sd[key] = 0.5 + torch.rand(v.shape, generator=g)
        elif v.dim() >= 2:
            sd[key] = torch.randn(v.shape, generator=g) * (1.0 / (v.shape[-1] ** 0.5))
        elif "LayerNorm.weight" in key or key.endswith("1.weight"):
            sd[key] = 1 + 0.3 * torch.randn(v.shape, generator=g)
        else:
            sd[key] = 0.1 * torch.randn(v.shape, generator=g)
    return sd


@torch.no_grad()
def mint_decoder_case(ref, case, n_ntype=4, n_etype=38):
    inp, sent_vecs, concept_ids = build_decoder_inputs(case, n_etype)
    dec = ref.QAGNN(None, case["k"], n_ntype, n_etype, case["sent_dim"], case["n_concept"], case["D"],
                    case["concept_in_dim"], case["n_head"], case["D"], case["n_fc_layer"], 0.2, 0.2, 0.2,
                    pretrained_concept_emb=None, freeze_ent_emb=True, init_range=0.02)
    sd = decoder_state_dict(dec, case)
    dec.load_state_dict(sd, strict=True)
    dec.eval()
    logits, pool_attn = dec(sent_vecs, concept_ids, inp["node_type"], inp["node_score"], inp["adj_lengths"],
                            (inp["edge_index"], inp["edge_type"]))
    return {"kind": "decoder", "case": case, "n_ntype": n_ntype, "n_etype": n_etype,
            "state_dict": {k_: v.clone() for k_, v in sd.items()},
            "logits": logits.clone(), "pool_attn": pool_attn.clone(),
            "input_fp": fingerprint(inp["H"], inp["edge_index"], sent_vecs, concept_ids)}


# training-mode cases (SURVEY.md §8f #3): the reference modules in .train() with dropout 0 (the mask stream of a live
# dropout cannot be reproduced), BatchNorm batch statistics, loss = sum(out * G) for a fixed random G, autograd gradients
TRAIN_CASES = [
    dict(name="train_cfg1_peaky_k2", B=4, n=50, e=200, D=64, k=2, regime="peaky", realistic=False, seed=21),
    dict(name="train_tiny_realistic_d100", B=6, n=24, e=60, D=100, k=3, regime="peaky", realistic=True, seed=22),
    dict(name="train_cfg2tiny_prod", B=2, n=200, e=1000, D=200, k=2, regime="prod", realistic=False, seed=23),
]


def train_loss_weights(case):
    g = torch.Generator().manual_seed(9000 + case["seed"])
    return torch.randn(case["B"], case["n"], case["D"], generator=g)


def mint_train_case(ref, case, n_ntype=4, n_etype=38):
    inp = O.synth_graph_batch(case["B"], case["n"], case["e"], case["D"], n_etype, case["seed"], case["realistic"])
    sd = O.random_state_dict(case["k"], case["D"], n_ntype, n_etype, case["regime"], case["seed"])
    mod = ref.QAGNN_Message_Passing(None, k=case["k"], n_ntype=n_ntype, n_etype=n_etype, input_size=case["D"],
                                    hidden_size=case["D"], output_size=case["D"], dropout=0.0)
    mod.load_state_dict(sd, strict=True)
    mod.train()
    H = inp["H"].clone().requires_grad_(True)
    score = inp["node_score"].clone().requires_grad_(True)
    out = mod(H, (inp["edge_index"], inp["edge_type"]), inp["node_type"], score)
    loss = (out * train_loss_weights(case)).sum()
    loss.backward()
    grads = {}
    seen = set()
    for name, p_ in mod.named_parameters():  # named_parameters de-duplicates the shared edge_encoder
        if id(p_) in seen:
            continue
        seen.add(id(p_))
        grads[name] = p_.grad.detach().clone() if p_.grad is not None else None
    buffers = {name: b.detach().clone() for name, b in mod.named_buffers() if "running" in name or "num_batches" in name}
    return {"kind": "train", "case": case, "n_ntype": n_ntype, "n_etype": n_etype,
            "input_fp": fingerprint(inp["H"], inp["edge_index"], inp["edge_type"], inp["node_type"], inp["node_score"]),
            "weight_fp": fingerprint(*[sd[k_] for k_ in sorted(sd) if sd[k_].dtype.is_floating_point]),
            "out": out.detach().clone(), "loss": float(loss), "grad_H": H.grad.clone(), "grad_score": score.grad.clone(),
            "grads": grads, "buffers_after": buffers}


TRAIN_DEC_CASES = [
    dict(name="train_decoder_small", B=6, n=30, e=80, D=64, k=2, sent_dim=48, n_concept=500, concept_in_dim=32,
         n_head=2, n_fc_layer=1, regime="peaky", seed=24),
]


def mint_train_decoder_case(ref, case, n_ntype=4, n_etype=38):
    """The whole reference decoder (`QAGNN`, modeling_qagnn.py:99-189) in .train(): every nn.Dropout of the instance gets
    p = 0 (a live mask stream cannot be reproduced), BatchNorm batch statistics, loss = sum(logits * g), autograd."""
    inp, sent_vecs, concept_ids = build_decoder_inputs(case, n_etype)
    dec = ref.QAGNN(None, case["k"], n_ntype, n_etype, case["sent_dim"], case["n_concept"], case["D"],
                    case["concept_in_dim"], case["n_head"], case["D"], case["n_fc_layer"], 0.0, 0.0, 0.0,
                    pretrained_concept_emb=None, freeze_ent_emb=True, init_range=0.02)
    sd = decoder_state_dict(dec, case)
    dec.load_state_dict(sd, strict=True)
    dec.train()
    for m in dec.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    dec.gnn.dropout_rate = 0.0
    sv = sent_vecs.clone().requires_grad_(True)
    logits, pool_attn = dec(sv, concept_ids, inp["node_type"], inp["node_score"], inp["adj_lengths"],
                            (inp["edge_index"], inp["edge_type"]))
    g = torch.Generator().manual_seed(9100 + case["seed"])
    w = torch.randn(logits.shape, generator=g)
    loss = (logits * w).sum()
    loss.backward()
    grads, seen = {}, set()
    for name, p_ in dec.named_parameters():
        if id(p_) in seen:
            continue
        seen.add(id(p_))
        grads[name] = p_.grad.detach().clone() if p_.grad is not None else None
    return {"kind": "train_decoder", "case": case, "n_ntype": n_ntype, "n_etype": n_etype,
            "state_dict": {k_: v.clone() for k_, v in sd.items()}, "logits": logits.detach().clone(),
            "pool_attn": pool_attn.detach().clone(), "loss_weights": w, "loss": float(loss.detach()),
            "grad_sent": sv.grad.clone(), "grads": grads,
            "input_fp": fingerprint(inp["H"], inp["edge_index"], sent_vecs, concept_ids)}


def _max_diff(a, b, path=""):
    """Largest absolute difference between two fixtures (nested dicts / lists of tensors and scalars); raises on a
    structural mismatch."""
    if isinstance(a, dict):
        assert isinstance(b, dict) and a.keys() == b.keys(), f"{path}: keys differ"
        return max([_max_diff(a[k_], b[k_], f"{path}.{k_}") for k_ in a] or [0.0])
    if isinstance(a, (list, tuple)):
        assert isinstance(b, (list, tuple)) and len(a) == len(b), f"{path}: lengths differ"
        return max([_max_diff(x, y, f"{path}[{i}]") for i, (x, y) in enumerate(zip(a, b))] or [0.0])
    if torch.is_tensor(a):
        assert torch.is_tensor(b) and a.shape == b.shape and a.dtype == b.dtype, f"{path}: tensor meta differs"
        return float((a.double() - b.double()).abs().max()) if a.numel() else 0.0
    if isinstance(a, float):
        return abs(a - b)
    assert a == b, f"{path}: {a!r} != {b!r}"
    return 0.0


def all_cases():
    return ([(mint_mp_case, c) for c in MP_CASES] + [(mint_layer_case, c) for c in LAYER_CASES] +
            [(mint_train_case, c) for c in TRAIN_CASES] + [(mint_train_decoder_case, c) for c in TRAIN_DEC_CASES] +
            [(mint_decoder_case, c) for c in DEC_CASES])


def mint_case(ref, mint, case):
    """One fixture, at the case's own (n_ntype, n_etype) or the reference's (4, 38)."""
    return mint(ref, case, case.get("n_ntype", 4), case.get("n_etype", 38))


def check(names=None):
    """Re-mints every fixture (or those in `names`) from the reference in memory and returns {name: max |diff|} against the
    committed file — nothing is written.  0.0 everywhere = the fixtures are what the reference's own modules produce here.
    A case whose file is not in the tree maps to None."""
    torch.set_num_threads(8)
    ref = load_reference()
    out = {}
    for mint, case in all_cases():
        if names is not None and case["name"] not in names:
            continue
        path = os.path.join(GOLDEN_DIR, case["name"] + ".pt")
        if not os.path.exists(path):  # nothing committed to compare with (tests/test_oracle_golden.py requires every file)
            out[case["name"]] = None
            continue
        have = torch.load(path, weights_only=False)
        out[case["name"]] = _max_diff(mint_case(ref, mint, case), have, case["name"])
    return out


def fuzz_cases(count):
    """The random small cases of --fuzz, deterministic: 1-4 graphs, 1-30 nodes, 0-80 edges, D 16-100, k 1-3, 6 / 17 / 38
    edge types, 1 / 3 / 4 / 6 node types, both weight regimes."""
    g = torch.Generator().manual_seed(12345)
    ri = lambda lo, hi: int(torch.randint(lo, hi + 1, (1,), generator=g))  # noqa: E731
    cases = []
    for i in range(count):
        n = ri(1, 30)
        R = (38, 38, 6, 17)[ri(0, 3)]
        T = (1, 3, 4, 6)[ri(0, 3)]
        case = dict(name=f"fuzz{i}", B=ri(1, 4), n=n, e=ri(0, 80), D=(16, 32, 64, 100)[ri(0, 3)], k=ri(1, 3),
                    regime=("prod", "peaky")[ri(0, 1)], realistic=bool(ri(0, 1)) and n >= 8 and R >= 6 and T >= 4,
                    seed=100 + i)
        cases.append(dict(case, n_ntype=T, n_etype=R))
    return cases


def fuzz_compared(out, extra, layers, keep):
    """[(name, tensor)] that the fuzz comparison checks: output, node_feature_extra, x and attention of the layers `keep`."""
    ts = [("out", out), ("extra", extra)]
    for l in keep:
        ts += [(f"x{l}", layers[l]["x"]), (f"alpha{l}", layers[l]["alpha"])]
    return ts


def oracle_fuzz_outputs(case):
    T, R = case.get("n_ntype", 4), case["n_etype"]  # fuzz files minted before T varied hold 4-type cases without the key
    inp = O.synth_graph_batch(case["B"], case["n"], case["e"], case["D"], R, case["seed"], case["realistic"], T)
    sd = O.random_state_dict(case["k"], case["D"], T, R, case["regime"], case["seed"])
    return O.message_passing_forward(sd, inp["H"], inp["edge_index"], inp["edge_type"], inp["node_type"], inp["node_score"],
                                     case["k"], T, R, return_layers=True)


def fuzz(count, tol_abs=2e-6, tol_rel=2e-5):
    """Random small cases that are NOT committed as fixtures: the reference's own QAGNN_Message_Passing against the oracle
    (output, node_feature_extra, first / last layer x and attention, edge_index').  Returns [(case, worst excess over the
    tolerance)]; excess <= 0 means inside `tol_abs + tol_rel*|ref|`."""
    torch.set_num_threads(8)
    ref = load_reference()
    results = []
    for case in fuzz_cases(count):
        fx = mint_mp_case(ref, case, case["n_ntype"], case["n_etype"])
        out, extra, layers = oracle_fuzz_outputs(case)
        keep = sorted(fx["layers"])
        got = dict(fuzz_compared(out, extra, layers, keep))
        pairs = [(got[name], want) for name, want in fuzz_compared(fx["out"], fx["extra"], fx["layers"], keep)]
        worst = max(float(((a - b).abs() - tol_abs - tol_rel * b.abs()).max()) if a.numel() else -tol_abs for a, b in pairs)
        results.append((case, worst))
    return results


def mint_fuzz_samples(ref, count=24):
    """The reference's outputs on the fuzz cases: FUZZ_SAMPLES values of each compared tensor at seeded positions, all
    concatenated into one index and one value tensor; `entries` says which slice belongs to which case and tensor."""
    cases, entries, index, value = [], [], [], []
    off = 0
    for ci, case in enumerate(fuzz_cases(count)):
        fx = mint_mp_case(ref, case, case["n_ntype"], case["n_etype"])
        keep = sorted(fx["layers"])
        cases.append(dict(case, keep=keep))
        for name, t in fuzz_compared(fx["out"], fx["extra"], fx["layers"], keep):
            idx = torch.randperm(t.numel(), generator=torch.Generator().manual_seed(case["seed"]))[:FUZZ_SAMPLES].sort().values
            entries.append((ci, name, tuple(t.shape), off, idx.numel()))
            index.append(idx.int())
            value.append(t.reshape(-1)[idx])
            off += idx.numel()
    return {"kind": "fuzz", "cases": cases, "entries": entries, "index": torch.cat(index), "value": torch.cat(value)}


def loader_fingerprint(obj):
    """sha256 of a loader / batch-generator result: tensors by dtype, shape and bytes, lists and tuples element-wise."""
    h = hashlib.sha256()

    def walk(x):
        if torch.is_tensor(x):
            h.update(f"T{x.dtype}{tuple(x.shape)}".encode())
            h.update(x.detach().contiguous().cpu().numpy().tobytes())
        elif isinstance(x, (list, tuple)):
            h.update(f"L{len(x)}".encode())
            for y in x:
                walk(y)
        else:
            h.update(repr(x).encode())
    walk(obj)
    return h.hexdigest()


def loader_generator_case(ei, et, cids, ntypes, scores, lens):
    """The batch-generator case of tests/test_loader_cpu.py: positional args and keywords (bs 4, eval order)."""
    Q = cids.size(0)

    class Args:
        drop_partial_batch = False
        fill_partial_batch = False
    args = (Args(), "eval", "cpu", "cpu", 4, torch.randperm(Q, generator=torch.Generator().manual_seed(0)),
            [f"q{i}" for i in range(Q)], torch.arange(Q) % 5)
    kw = dict(tensors0=[torch.arange(Q * 5 * 7).view(Q, 5, 7)], tensors1=[cids, ntypes, scores, lens])
    return args, kw


def mint_loader_fingerprints():
    """What the reference's own loader and batch generator return on the synthetic adjacency pickles of the loader tests."""
    import tempfile
    from oracle.ref_shim import REFERENCE_ROOT, _install_stubs
    from qagnn_b200 import data as Dt
    sys.path.insert(0, REFERENCE_ROOT)
    try:
        _install_stubs()
        from utils import data_utils as RD
        out = {"kind": "loader", "loader": {}}
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "dev.graph.adj.pk")
            Dt.synth_adj_pickle(path, 20, seed=4)
            for max_node_num in (200, 30):
                res = RD.load_sparse_adj_data_with_contextnode(path, max_node_num, 5, None)
                os.remove(path + ".loaded_cache")
                out["loader"][max_node_num] = loader_fingerprint(list(res[:4]) + [res[4][0], res[4][1]])
            path = os.path.join(tmp, "s.graph.adj.pk")
            Dt.synth_adj_pickle(path, 50, seed=2, max_nodes=60)
            cids, ntypes, scores, lens, (ei, et) = Dt.load_sparse_adj_data_with_contextnode(path, 40, 5, None, use_cache=False,
                                                                                            write_cache=False)
            args, kw = loader_generator_case(ei, et, cids, ntypes, scores, lens)
            out["generator"] = loader_fingerprint(list(RD.MultiGPUSparseAdjDataBatchGenerator(*args, adj_data=(ei, et), **kw)))
    finally:
        sys.path.remove(REFERENCE_ROOT)
    return out


def main():
    if "--fuzz" in sys.argv[1:]:
        count = int(sys.argv[sys.argv.index("--fuzz") + 1])
        bad = 0
        for case, worst in fuzz(count):
            print(f"{case}: {'inside' if worst <= 0 else 'OUTSIDE'} the tolerance (excess {worst:.3g})")
            bad += worst > 0
        sys.exit(1 if bad else 0)
    if "--check" in sys.argv[1:]:
        worst = 0.0
        for name, diff in check().items():
            if diff is None:
                print(f"{name}: no committed fixture")
                continue
            print(f"{name}: max |re-minted - committed| = {diff:.3g}")
            worst = max(worst, diff)
        sys.exit(0 if worst == 0.0 else 1)
    torch.set_num_threads(8)
    ref = load_reference()
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    for mint, case in all_cases():
        fx = mint_case(ref, mint, case)
        torch.save(fx, os.path.join(GOLDEN_DIR, case["name"] + ".pt"))
        print("minted", case["name"], fx.get("kind"))
    os.makedirs(REF_DATA_DIR, exist_ok=True)
    torch.save(mint_fuzz_samples(ref), FUZZ_FILE)
    torch.save(mint_loader_fingerprints(), LOADER_FILE)
    print("minted", FUZZ_FILE, LOADER_FILE)


if __name__ == "__main__":
    main()
