"""Timings of the dense model's adjacency on the device (prepare_graph_dense_device / set_message_weights / backward with
d_message_weights) against today's host path (set_graph_dense: the host scan of the matrix into a CSR and its upload).

Workload: the dense model (one layer of 4 timesteps, GRU, edge bias) on 256 synthetic molecules in bucket 29 (7 424 rows, 4 edge types) at
hidden 100, 256 and 512; forward on --precision (bf16x3 by default), backward on --bwd-precision (bf16x3 by default).  Arms:
  host-binary     set_graph_dense of the 0/1 matrix once (its host prepare timed on its own, wall clock to the end of the upload), then
                  the forward of that batch
  device-binary   prepare_graph_dense_device + set_message_weights of the same 0/1 matrix as a CUDA tensor, then the forward
  device-soft     the same with a full soft matrix (a row softmax of random scores: no zero entry)
Each arm reports forward, forward + backward, and forward + backward with dA (the device arms only): the device time between two CUDA
events around the calls, the L2 flushed before each run, median of --steps runs after --warmup; the arms alternate, --rounds times, and the
figure is the median of the round medians.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/dense_adjacency_bench.py [--steps 30] [--warmup 5] [--rounds 3] [--hidden 100,256,512] [--json OUT]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.wide_hidden_bench import Timer, gpu_info  # noqa: E402

GRAPHS, BUCKET, T, STEPS = 256, 29, 4, 4
ARMS = ("host-binary", "device-binary", "device-soft")


def workload(D):
    """(engine params, 0/1 matrix, soft matrix, h0 [b*v, D]) of the molecules."""
    from gated_graph_neural_network_samples_b200 import packing, synthetic, workloads
    mols = synthetic.make_molecules(GRAPHS, seed=0, num_bond_types=T)
    b = packing.pack_dense_batch(mols, BUCKET, D, T)
    binary = np.ascontiguousarray(b["adjacency_matrix"], np.float32)
    s = np.random.default_rng(3).normal(0, 1, binary.shape)
    e = np.exp(s - s.max(-1, keepdims=True))
    soft = (e / e.sum(-1, keepdims=True)).astype(np.float32)
    h0 = np.ascontiguousarray(b["initial_node_representation"], np.float32).reshape(-1, D)
    params = workloads.dense_engine_params({"hidden_size": D, "num_timesteps": STEPS, "use_edge_bias": True})
    return params, binary, soft, h0


def host_prepare_ms(eng, A, reps):
    """Median wall time of set_graph_dense (host scan, CSR build, upload) + synchronize."""
    import torch
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.set_graph_dense(A)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times)


def run_hidden(timer, D, precision, bwd_precision, rounds):
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    from oracle import ggnn_oracle as O
    params, binary, soft, h0_np = workload(D)
    b, v = binary.shape[0], binary.shape[2]
    w = O.init_dense_weights(dict(params, hidden_size=D), T, np.random.default_rng(1))
    w["edge_biases"] = w["edge_biases"].reshape(T, D)
    dev_w = [{k: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda() for k, x in w.items()}]
    h0 = torch.from_numpy(h0_np).cuda()
    g_out = torch.randn_like(h0)

    def engine():
        eng = PropagationEngine(params, T, precision=precision)
        eng.set_weights(dev_w)
        eng.set_save_for_backward(True)
        eng.set_backward_precision(bwd_precision)
        return eng

    engines, mats = {}, {"device-binary": torch.from_numpy(binary).cuda(), "device-soft": torch.from_numpy(soft).cuda()}
    host = engines["host-binary"] = engine()
    prep_ms = host_prepare_ms(host, binary, timer.steps)
    for a in ("device-binary", "device-soft"):
        eng = engines[a] = engine()
        eng.set_graph_prepared(eng.prepare_graph_dense_device(b, v))
        eng.set_message_weights(mats[a])
    out = {a: torch.empty_like(h0) for a in ARMS}
    grads = {a: [{k: torch.zeros_like(t) for k, t in dev_w[0].items()}] for a in ARMS}
    dh0 = {a: torch.zeros_like(h0) for a in ARMS}
    dA = {a: torch.zeros_like(m) for a, m in mats.items()}

    def fwd(a):
        return lambda: engines[a].forward(h0, out[a])

    def fwd_bwd(a, with_dA):
        def fn():
            engines[a].forward(h0, out[a])
            engines[a].backward(g_out, grads[a], dh0[a], d_message_weights=dA[a] if with_dA else None)
        return fn

    cols = {"fwd": lambda a: fwd(a), "fwd+bwd": lambda a: fwd_bwd(a, False), "fwd+bwd+dA": lambda a: fwd_bwd(a, True)}
    per = {(a, c): [] for a in ARMS for c in cols if not (a == "host-binary" and c == "fwd+bwd+dA")}
    for _ in range(rounds):
        for a in ARMS:
            for c, make in cols.items():
                if (a, c) in per:
                    per[(a, c)].append(timer.median_ms(make(a), flush=True))
    for eng in engines.values():
        eng.sync_check()
    res = {"%s %s" % k: round(statistics.median(v), 4) for k, v in per.items()}
    same = float((engines["host-binary"].forward(h0, out["host-binary"]) - engines["device-binary"].forward(h0, out["device-binary"]))
                 .abs().max() / out["host-binary"].abs().max())
    return {"D": D, "V": b * v, "graphs": b, "bucket": v, "T": T, "steps": STEPS, "precision": precision, "bwd_precision": bwd_precision,
            "plan_host": host.plan, "plan_device": engines["device-binary"].plan, "host_prepare_ms": round(prep_ms, 4), "ms": res,
            "round_medians_ms": {"%s %s" % k: [round(x, 4) for x in v] for k, v in per.items()},
            "binary_paths_max_rel_diff": same}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--precision", default="bf16x3", choices=("fp32", "bf16x3", "bf16"))
    ap.add_argument("--bwd-precision", default="bf16x3", choices=("fp32", "bf16x3"))
    ap.add_argument("--hidden", default="100,256,512")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    timer = Timer(args.steps, args.warmup)
    card = gpu_info()
    print("card: %s" % card)
    rows = []
    for D in (int(x) for x in args.hidden.split(",")):
        row = run_hidden(timer, D, args.precision, args.bwd_precision, args.rounds)
        row["card"] = card
        rows.append(row)
        print(json.dumps(row))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
