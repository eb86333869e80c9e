"""world_size=2 gloo test of the sharding + all-gather host logic (CPU; the GNN itself needs a GPU, so the decoder's
message-passing module is replaced by the CPU oracle here — tests may use the oracle as a stand-in checker)."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import qagnn_b200
from oracle import make_goldens as MG
from oracle import qagnn_oracle as O
from qagnn_b200 import distributed as D


class OracleGNN(torch.nn.Module):
    """Stand-in for QAGNN_Message_Passing on CPU: evaluates the oracle with the module's own weights."""

    def __init__(self, mod):
        super().__init__()
        self.mod = mod

    def forward(self, H, A, node_type, node_score):
        sd = {k: v for k, v in self.mod.state_dict().items()}
        return O.message_passing_forward(sd, H, A[0], A[1], node_type, node_score, self.mod.k, self.mod.n_ntype,
                                         self.mod.n_etype)


def _decoder(case):
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", case + ".pt"), weights_only=False)
    c = fx["case"]
    dec = qagnn_b200.QAGNN(None, c["k"], 4, 38, c["sent_dim"], c["n_concept"], c["D"], c["concept_in_dim"], c["n_head"],
                           c["D"], c["n_fc_layer"], 0.2, 0.2, 0.2).eval()
    dec.load_state_dict(fx["state_dict"])
    dec.gnn = OracleGNN(dec.gnn)
    return fx, c, dec


def _worker(rank, world, port, case, out_q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    fx, c, dec = _decoder(case)
    inp, sent_vecs, concept_ids = MG.build_decoder_inputs(c, 38)
    B, n = c["B"], c["n"]
    lo, hi = D.shard_bounds(B, rank, world)
    sel = (inp["edge_index"][0] >= lo * n) & (inp["edge_index"][0] < hi * n)
    ei = inp["edge_index"][:, sel] - lo * n
    with torch.no_grad():
        logits, _ = D.decoder_forward_sharded(dec, sent_vecs[lo:hi], concept_ids[lo:hi], inp["node_type"][lo:hi],
                                              inp["node_score"][lo:hi], inp["adj_lengths"][lo:hi],
                                              (ei, inp["edge_type"][sel]), world)
    # by value: a tensor would travel as a file descriptor served by this process, which may have exited by the time the
    # parent unpickles it
    out_q.put((rank, logits.numpy()))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_shard_and_all_gather_matches_reference_logits():
    case = "decoder_small"
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, case, q)) for r in range(2)]
    [p.start() for p in procs]
    got = {r: torch.from_numpy(a) for r, a in (q.get(timeout=120) for _ in range(2))}
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", case + ".pt"), weights_only=False)
    for r in (0, 1):  # every rank holds the logits of the whole batch, equal to the reference's
        assert torch.allclose(got[r], fx["logits"], atol=1e-4, rtol=1e-4), (got[r] - fx["logits"]).abs().max()


def test_shard_bounds_cover_the_batch():
    for B in (1, 5, 64, 65):
        for w in (1, 2, 4, 8):
            spans = [D.shard_bounds(B, r, w) for r in range(w)]
            assert spans[0][0] == 0 and spans[-1][1] == B
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))


def test_numa_binding_is_a_no_op_without_a_gpu():
    """bind_to_gpu_numa_node is an optimisation: on a host without CUDA devices (or without NUMA information) it must return
    None and leave the process affinity alone."""
    before = os.sched_getaffinity(0)
    assert D.bind_to_gpu_numa_node(0) is None or isinstance(D.bind_to_gpu_numa_node(0), int)
    if not torch.cuda.is_available():
        assert os.sched_getaffinity(0) == before
