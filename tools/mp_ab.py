"""In-process A/B of the tiled message-passing kernel's launch-time switches on the GPU (the library reads them at every
launch): bit-equality of the outputs across settings and the message-passing stage time of each.

    python tools/mp_ab.py QAGNN_MP_WARPS=24 QAGNN_MP_WARPS=28 QAGNN_MP_WARPS=31      # -> gpurun_out/mp_ab.txt
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "gpurun_out", "mp_ab.txt")
os.makedirs(os.path.dirname(OUT), exist_ok=True)


def say(*a):
    with open(OUT, "a") as f:
        f.write(" ".join(str(x) for x in a) + "\n")
    print(*a, flush=True)


def main():
    import torch
    import qagnn_b200
    from qagnn_b200 import _lib
    from oracle import qagnn_oracle as O
    settings = [dict(kv.split("=") for kv in arg.split(",")) for arg in sys.argv[1:]] or [{}]
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    t00 = time.time()
    for name, B, n, e, D, k, realistic in (("cfg2", 320, 200, 1000, 200, 5, False), ("cfg2-loader-shaped", 320, 200, 1000, 200, 5, True),
                                           ("hubs", 32, 40, 1400, 200, 1, False), ("cfg1", 4, 50, 200, 64, 1, False)):
        inp = O.synth_graph_batch(B, n, e, D, 38, 7, realistic)
        sd = O.random_state_dict(k, D, 4, 38, "peaky", 7)
        mod = qagnn_b200.QAGNN_Message_Passing(None, k, 4, 38, D, D, D).eval()
        mod.load_state_dict(sd)
        mod = mod.to(dev)
        d = {k_: v.to(dev) for k_, v in inp.items() if k_ != "adj_lengths"}
        first = None
        for st in settings + settings[:1]:
            for k_ in list(os.environ):
                if k_.startswith("QAGNN_MP_"):
                    del os.environ[k_]
            os.environ.update(st)
            for _ in range(2):
                out = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"])
            torch.cuda.synchronize()
            lib.qagnn_profile_enable(1)
            for _ in range(10):
                out = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"])
            torch.cuda.synchronize()
            prof = _lib.profile_read()
            lib.qagnn_profile_enable(0)
            us = prof["message_passing"][0] / 10 / k * 1e3
            o = out.cpu()
            if first is None:
                first = o
            say(name, st, "mp us/layer", round(us, 1), "bit-identical to first:", torch.equal(first, o),
                "finite:", bool(torch.isfinite(o).all()), "t", round(time.time() - t00, 1))
    say("done")


if __name__ == "__main__":
    main()
