"""Timings of a weighted dense adjacency above hidden 128: the dense model on 256 molecules in bucket 29 (4 edge types, 4 timesteps, edge
bias), every nonzero entry of the matrix drawn from U(0.25, 1.75), at hidden 256 and 512.

Arms per hidden size:
  weighted-bf16x3  the weighted matrix on the streaming wgmma kernels through set_graph_dense_weighted (every (target, type) pair with
                   messages is a virtual row, summed by each gather launch)
  binary-bf16x3    the same matrix as 0/1 on the streaming kernels (only pairs with several messages are virtual rows)
  weighted-fp32    the weighted matrix on the fp32 path (the only way to run it above hidden 128 before the streaming gather took weights)
Each arm times the forward and forward + backward (save_for_backward, every weight gradient and d h0) with CUDA events, after a warm-up,
as the median of --steps runs with the L2 flushed before each run.  The arms run in turn, --reps times, and each number is the median over
the repetitions.  The card's name, power limit and maximum SM clock are read in the same run (an nvidia-smi query).

    python tools/weighted_dense_bench.py [--steps 30] [--warmup 5] [--reps 3] [--json OUT]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.wide_hidden_bench import Timer, gpu_info  # noqa: E402

WIDTHS = (256, 512)
ARMS = (("weighted-bf16x3", True, "bf16x3"), ("binary-bf16x3", False, "bf16x3"), ("weighted-fp32", True, "fp32"))
GRAPHS, BUCKET, T, STEPS = 256, 29, 4, 4


def workload(D):
    """(engine params, weighted matrix, its 0/1 twin, h0 [b*v, D])."""
    from gated_graph_neural_network_samples_b200 import packing, synthetic, workloads
    mols = synthetic.make_molecules(GRAPHS, seed=0, num_bond_types=T)
    b = packing.pack_dense_batch(mols, BUCKET, D, T)
    binary = np.asarray(b["adjacency_matrix"], np.float32)
    rng = np.random.default_rng(2)
    weighted = np.where(binary != 0, rng.uniform(0.25, 1.75, binary.shape), 0.0).astype(np.float32)
    params = workloads.dense_engine_params({"hidden_size": D, "num_timesteps": STEPS, "use_edge_bias": True})
    h0 = np.asarray(b["initial_node_representation"], np.float32).reshape(-1, D)
    return params, weighted, binary, h0


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
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("weighted_dense_bench.py needs a CUDA device")
    steps = max(args.steps, 20)
    timer = Timer(steps, args.warmup)
    result = {"gpu": gpu_info(), "steps": steps, "warmup": args.warmup, "reps": args.reps, "rows": []}
    print("GPU (name, power limit, max SM clock): %s" % result["gpu"])
    print("%-7s %-16s %10s %10s %8s   plan" % ("hidden", "arm", "fwd ms", "fwd+bwd ms", "vrows"))
    for D in WIDTHS:
        params, weighted, binary, h0 = workload(D)
        runs = {name: [] for name, _, _ in ARMS}
        for _ in range(args.reps):
            for name, is_weighted, precision in ARMS:
                runs[name].append(arm(timer, D, weighted if is_weighted else binary, precision, params, h0))
        for name, _, _ in ARMS:
            rs = runs[name]
            r = dict(rs[0], hidden=D, arm=name, forward_ms=statistics.median(x["forward_ms"] for x in rs),
                     fwd_bwd_ms=statistics.median(x["fwd_bwd_ms"] for x in rs), forward_ms_all=[x["forward_ms"] for x in rs],
                     fwd_bwd_ms_all=[x["fwd_bwd_ms"] for x in rs])
            result["rows"].append(r)
            print("%-7d %-16s %10.3f %10.3f %8s   %s" % (D, name, r["forward_ms"], r["fwd_bwd_ms"], r.get("virtual_rows", "-"), r["plan"]),
                  flush=True)
    print(json.dumps(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
