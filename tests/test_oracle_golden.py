"""Pins oracle/qagnn_oracle.py against every golden vector minted from the reference's own
modules (tests/golden/*.pt, made by oracle/make_goldens.py).  CPU only."""
import pytest
import torch

from oracle import qagnn_oracle as O
from tests import helpers as Hh

# the oracle and the reference run the same fp32 op sequence on the same CPU: they agree to
# rounding noise, far inside the 1e-4 parity bar
TIGHT = dict(atol=2e-6, rtol=2e-5)


@pytest.mark.parametrize("name", Hh.golden_names("mp"))
def test_oracle_matches_reference_message_passing(name):
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sd = Hh.regen_mp_inputs(fx)
    out, extra, layers = O.message_passing_forward(sd, inp["H"], inp["edge_index"], inp["edge_type"],
                                                   inp["node_type"], inp["node_score"], c["k"], fx["n_ntype"],
                                                   fx["n_etype"], return_layers=True)
    Hh.assert_close(extra, fx["extra"], "node_feature_extra", **TIGHT)
    for l, ref_l in fx["layers"].items():
        Hh.assert_close(layers[l]["alpha"], ref_l["alpha"], f"alpha[{l}]", **TIGHT)
        Hh.assert_close(layers[l]["x"], ref_l["x"], f"x[{l}]", atol=2e-5, rtol=1e-4)
    Hh.assert_close(out, fx["out"], "out", atol=2e-5, rtol=1e-4)
    # integer side: edge_index' (self loops appended after the real edges) is bit-exact
    prep = O.graph_prep_oracle(inp["edge_index"], inp["edge_type"], inp["node_type"], fx["n_ntype"], fx["n_etype"])
    assert torch.equal(torch.from_numpy(prep["src"]), fx["edge_index_prime"][0])
    assert torch.equal(torch.from_numpy(prep["tgt"]), fx["edge_index_prime"][1])


@pytest.mark.parametrize("name", Hh.golden_names("layer"))
def test_oracle_matches_reference_gatconve(name):
    fx = Hh.load_golden(name)
    c = fx["case"]
    x, extra, node_type, ei, et, sd = Hh.regen_layer_inputs(fx)
    out, ei2, alpha, _ = O.gatconve_forward(sd, "gnn_layers.0", x, ei, et, node_type, extra, fx["n_ntype"],
                                            fx["n_etype"], head_count=c["H"])
    assert torch.equal(ei2, fx["edge_index_prime"])
    Hh.assert_close(alpha, fx["alpha"], "alpha", **TIGHT)
    Hh.assert_close(out, fx["out"], "out", atol=2e-5, rtol=1e-4)


@pytest.mark.parametrize("name", Hh.golden_names("decoder"))
def test_oracle_matches_reference_decoder(name):
    from oracle import make_goldens as MG
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sent_vecs, concept_ids = MG.build_decoder_inputs(c, fx["n_etype"])
    logits, pool_attn, _ = O.qagnn_decoder_forward(fx["state_dict"], sent_vecs, concept_ids, inp["node_type"],
                                                   inp["node_score"], inp["adj_lengths"], inp["edge_index"],
                                                   inp["edge_type"], c["k"], fx["n_ntype"], fx["n_etype"],
                                                   c["n_head"], c["n_fc_layer"])
    Hh.assert_close(pool_attn, fx["pool_attn"], "pool_attn", atol=2e-5, rtol=1e-4)
    Hh.assert_close(logits, fx["logits"], "logits", atol=5e-5, rtol=1e-4)


def test_fp64_oracle_is_the_same_function():
    """fp64 evaluation of the same restatement stays within fp32 noise of the fp32 golden: the
    1e-4 bar is far above the reference's own rounding floor on these cases."""
    fx = Hh.load_golden("cfg2small_peaky")
    c = fx["case"]
    inp, sd = Hh.regen_mp_inputs(fx)
    out64 = O.message_passing_forward(sd, inp["H"], inp["edge_index"], inp["edge_type"], inp["node_type"],
                                      inp["node_score"], c["k"], fx["n_ntype"], fx["n_etype"], dtype=torch.float64)
    Hh.assert_close(out64.float(), fx["out"], "fp64 oracle vs fp32 reference", atol=5e-5, rtol=1e-4)


def test_state_dict_contract():
    """Key names a replacement module must accept (SURVEY.md §8b), incl. the k aliased copies of the
    shared edge encoder."""
    fx = Hh.load_golden("cfg1_peaky_k2")
    keys = fx["state_dict_keys"]
    sd = O.random_state_dict(2, 64)
    assert sorted(sd.keys()) == keys
    assert "gnn_layers.1.edge_encoder.3.weight" in keys and "edge_encoder.3.weight" in keys


def test_committed_goldens_are_what_the_reference_produces_here():
    """Build container only (needs /root/reference): re-mint every fixture in memory from the reference's own modules and
    require it to equal the committed file bit for bit (`python -m oracle.make_goldens --check`, writes nothing)."""
    import os
    import subprocess
    import sys
    if not os.path.isdir("/root/reference/modeling"):
        pytest.skip("the reference tree is not on this machine")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "oracle.make_goldens", "--check"], cwd=root, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [l for l in r.stdout.splitlines() if "max |re-minted - committed|" in l]
    import glob
    assert len(lines) == len(glob.glob(os.path.join(root, "tests", "golden", "*.pt"))) >= 20
    assert all(l.endswith("= 0") for l in lines)


def test_oracle_equals_the_reference_on_uncommitted_random_cases():
    """24 random small cases (1-4 graphs, 1-30 nodes, 0-80 edges, D 16-100, k 1-3, 6 / 17 / 38 edge types, 1 / 3 / 4 / 6 node
    types, both weight regimes) that are not fixtures: the oracle against the reference's own QAGNN_Message_Passing, fp32,
    2e-6 + 2e-5 rel, on a seeded sample of every compared tensor stored by `python -m oracle.make_goldens`
    (tests/golden/ref/fuzz24.pt) — widens the pinned region beyond the committed fixtures."""
    from oracle import make_goldens as MG
    fz = torch.load(MG.FUZZ_FILE, weights_only=False)
    assert len(fz["cases"]) == 24 and [c["name"] for c in fz["cases"]] == [c["name"] for c in MG.fuzz_cases(24)]
    got = {}
    for ci, case in enumerate(fz["cases"]):
        out, extra, layers = MG.oracle_fuzz_outputs(case)
        got[ci] = dict(MG.fuzz_compared(out, extra, layers, case["keep"]))
    assert {(ci, name) for ci, name, *_ in fz["entries"]} == {(ci, name) for ci in got for name in got[ci]}
    for ci, name, shape, off, cnt in fz["entries"]:
        t = got[ci][name]
        assert tuple(t.shape) == shape, (fz["cases"][ci]["name"], name)
        Hh.assert_close(t.reshape(-1)[fz["index"][off:off + cnt].long()], fz["value"][off:off + cnt],
                        f"{fz['cases'][ci]['name']} {name}", **TIGHT)


def test_every_golden_case_has_its_committed_fixture():
    """`make_goldens --check` reports a case whose fixture is not in the tree without comparing it: every case of the table
    must have its file here."""
    import os
    from oracle import make_goldens as MG
    missing = [c["name"] for _, c in MG.all_cases() if not os.path.exists(os.path.join(MG.GOLDEN_DIR, c["name"] + ".pt"))]
    assert not missing, f"cases without a committed fixture: {missing}"
