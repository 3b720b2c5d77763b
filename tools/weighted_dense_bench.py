"""Timings of a weighted dense adjacency on the tensor-core kernels (and on fp32), every nonzero entry of the matrix drawn from
U(0.25, 1.75); the dense model with 4 edge types, 4 timesteps and edge bias.

Workload "molecules": 256 molecules in bucket 29 at hidden 256 and 512, above the tile-local kernel's hidden sizes.  Arms per hidden size:
  weighted-bf16x3  the weighted matrix on the streaming wgmma kernels through set_graph_dense_weighted (every (target, type) pair with
                   messages is a virtual row, summed by each gather launch)
  binary-bf16x3    the same matrix as 0/1 on the streaming kernels (only pairs with several messages are virtual rows)
  weighted-fp32    the weighted matrix on the fp32 path (the only way to run it above hidden 128 before the streaming gather took weights)
Workload "big-components": 64 graphs of v = 200, each one connected 200-node component (a random spanning tree and 200 more undirected
edges, types uniform), at hidden 100 and 128: within the tile kernel's hidden sizes, but every component is larger than its 128-row
tile, so the weighted batch runs the tile kernel's GLOBAL plan (one launch per timestep).  One arm, weighted-bf16x3.
Each arm times the forward and forward + backward (save_for_backward, every weight gradient and d h0) with CUDA events, after a warm-up,
as the median of --steps runs with the L2 flushed before each run.  The arms run in turn, --reps times, and each number is the median over
the repetitions.  The card's name, power limit and maximum SM clock are read in the same run (an nvidia-smi query).

    python tools/weighted_dense_bench.py [--steps 30] [--warmup 5] [--reps 3] [--workloads molecules,big-components] [--json OUT]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.wide_hidden_bench import Timer, gpu_info  # noqa: E402

ARMS = (("weighted-bf16x3", True, "bf16x3"), ("binary-bf16x3", False, "bf16x3"), ("weighted-fp32", True, "fp32"))
GRAPHS, BUCKET, T, STEPS = 256, 29, 4, 4
BIG_GRAPHS, BIG_NODES = 64, 200


def _weigh(binary):
    rng = np.random.default_rng(2)
    return np.where(binary != 0, rng.uniform(0.25, 1.75, binary.shape), 0.0).astype(np.float32)


def _params(D):
    from gated_graph_neural_network_samples_b200 import workloads
    return workloads.dense_engine_params({"hidden_size": D, "num_timesteps": STEPS, "use_edge_bias": True})


def workload(D):
    """(engine params, weighted matrix, its 0/1 twin, h0 [b*v, D]) of the molecules."""
    from gated_graph_neural_network_samples_b200 import packing, synthetic
    mols = synthetic.make_molecules(GRAPHS, seed=0, num_bond_types=T)
    b = packing.pack_dense_batch(mols, BUCKET, D, T)
    binary = np.asarray(b["adjacency_matrix"], np.float32)
    h0 = np.asarray(b["initial_node_representation"], np.float32).reshape(-1, D)
    return _params(D), _weigh(binary), binary, h0


def big_component_workload(D):
    """(engine params, weighted matrix, its 0/1 twin, h0 [b*v, D]) of the 200-node components."""
    rng = np.random.default_rng(41)
    n = BIG_NODES
    binary = np.zeros((BIG_GRAPHS, T, n, n), np.float32)
    for g in range(BIG_GRAPHS):
        pairs = {(int(rng.integers(0, i)), i) for i in range(1, n)}
        while len(pairs) < 2 * n - 1:
            a, c = sorted(int(x) for x in rng.choice(n, 2, replace=False))
            pairs.add((a, c))
        for k, (a, c) in enumerate(sorted(pairs)):
            t = k % T if k < T else int(rng.integers(0, T))
            binary[g, t, a, c] = binary[g, t, c, a] = 1.0
    h0 = rng.normal(0, 1, (BIG_GRAPHS * n, D)).astype(np.float32)
    return _params(D), _weigh(binary), binary, h0


# name: (hidden sizes, batch builder, arms)
WORKLOADS = {"molecules": ((256, 512), workload, ARMS),
             "big-components": ((100, 128), big_component_workload, ARMS[:1])}


def arm(timer, D, A, precision, params, h0_np):
    import torch
    from gated_graph_neural_network_samples_b200 import workloads
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph, PropagationEngine
    w = workloads.init_weights(params, T, seed=1)
    dev_w = [{k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in lw.items()} for lw in w]
    eng = PropagationEngine(params, T, precision=precision)
    eng.set_weights(dev_w)
    eng.set_save_for_backward(True)
    eng.set_graph_dense_weighted(A)
    h0 = torch.from_numpy(h0_np).cuda()
    out = torch.empty_like(h0)
    g = PreparedGraph.host_only_dense_weighted(params, T, A, precision=precision)
    rows = {"plan": eng.plan, "V": int(h0.shape[0]), "messages": g.info()["num_messages"]}
    if g.info()["streaming"]:
        rows["virtual_rows"] = int(len(g.stream_tables()["vrow_ptr"]) - 1)
    rows["forward_ms"] = timer.median_ms(lambda: eng.forward(h0, out), True)
    grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in dev_w]
    d_out = torch.randn_like(h0)
    d_h0 = torch.empty_like(h0)

    def fwd_bwd():
        eng.forward(h0, out)
        eng.backward(d_out, grads, d_h0)

    rows["fwd_bwd_ms"] = timer.median_ms(fwd_bwd, True)
    eng.sync_check()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed runs per number (the median is reported; at least 20)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3, help="rounds over the arms (each number is the median over the rounds)")
    ap.add_argument("--workloads", default=",".join(WORKLOADS), help="comma-separated, of: %s" % ", ".join(WORKLOADS))
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    args = ap.parse_args()
    chosen = args.workloads.split(",")
    unknown = sorted(set(chosen) - set(WORKLOADS))
    if unknown:
        raise SystemExit("unknown workloads: %s" % unknown)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("weighted_dense_bench.py needs a CUDA device")
    steps = max(args.steps, 20)
    timer = Timer(steps, args.warmup)
    result = {"gpu": gpu_info(), "steps": steps, "warmup": args.warmup, "reps": args.reps, "rows": []}
    print("GPU (name, power limit, max SM clock): %s" % result["gpu"])
    print("%-15s %-7s %-16s %10s %10s %8s   plan" % ("workload", "hidden", "arm", "fwd ms", "fwd+bwd ms", "vrows"))
    for wl, D in ((k, D) for k in chosen for D in WORKLOADS[k][0]):
        _, build, arms = WORKLOADS[wl]
        params, weighted, binary, h0 = build(D)
        runs = {name: [] for name, _, _ in arms}
        for _ in range(args.reps):
            for name, is_weighted, precision in arms:
                runs[name].append(arm(timer, D, weighted if is_weighted else binary, precision, params, h0))
        for name, _, _ in arms:
            rs = runs[name]
            r = dict(rs[0], workload=wl, hidden=D, arm=name, forward_ms=statistics.median(x["forward_ms"] for x in rs),
                     fwd_bwd_ms=statistics.median(x["fwd_bwd_ms"] for x in rs), forward_ms_all=[x["forward_ms"] for x in rs],
                     fwd_bwd_ms_all=[x["fwd_bwd_ms"] for x in rs])
            result["rows"].append(r)
            print("%-15s %-7d %-16s %10.3f %10.3f %8s   %s" % (wl, D, name, r["forward_ms"], r["fwd_bwd_ms"], r.get("virtual_rows", "-"),
                                                                r["plan"]), flush=True)
    print(json.dumps(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
