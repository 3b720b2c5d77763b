"""Timings of propagation attention on the streaming wgmma kernels (GGNN_ATT_TENSOR_CORES) against the fp32 kernels it ran on before.

Workloads (seeded, workloads.py), every one with use_propagation_attention and a_t = 1 (the plug-in's initialiser):
  cfg2        256 molecules, hidden 100, 4 edge types, layer_timesteps [4]
  100k        the reference's default batch of about 100 000 nodes (default_batch_100k_nodes), hidden 100, [4]
  cfg4        1024 molecules, hidden 256, 8 edge types, [2, 2, 2, 2] with a residual input
  cfg4-h512   the same batch and model at hidden 512
Arms per workload:
  att-fp32         attention on the fp32 kernels (GGNN_ATT_FP32, the only way to run it before)
  att-tc-bf16x3    attention on the streaming wgmma kernels at bf16x3 (GGNN_ATT_TENSOR_CORES)
  noatt-bf16x3     the same model without attention at bf16x3 (its own plan): what attention itself costs
Each arm times the forward and forward + backward (save_for_backward, every weight gradient and d h0) with CUDA events after --warmup
runs, as the median of --steps runs with the L2 flushed before each run.  The arms run in turn, --reps times, and each number is the
median over the repetitions.  The att-tc-bf16x3 output of the timed forward is compared with float64 (oracle.sparse_propagation_torch on
the GPU) against the bf16x3 forward bar, 1e-4 of max|ref|, so that a fast wrong answer fails the run.  The card's name, power limit and
maximum SM clock are read in the same run (an nvidia-smi query).

    python tools/attention_bench.py [--steps 30] [--warmup 5] [--reps 3] [--json OUT]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.wide_hidden_bench import Timer, gpu_info  # noqa: E402

WORKLOADS = (("cfg2", "cfg2", None), ("100k", "default_batch_100k_nodes", None), ("cfg4", "cfg4", None), ("cfg4-h512", "cfg4", 512))
ARMS = (("att-fp32", True, False, "fp32"), ("att-tc-bf16x3", True, True, "bf16x3"), ("noatt-bf16x3", False, False, "bf16x3"))
BAR_FORWARD = 1e-4


def workload(config, hidden):
    """(params with attention, T, adjacency lists, in-degrees, h0, weights with a_t = 1)."""
    from gated_graph_neural_network_samples_b200 import workloads
    w = workloads.build(config)
    params = dict(w["engine_params"], use_propagation_attention=True)
    h0 = np.asarray(w["h0"], np.float32)
    if hidden is not None:   # the same molecules at another width: the annotations zero-padded, as the packer pads them
        params["hidden_size"] = hidden
        h0 = np.pad(h0, ((0, 0), (0, hidden - h0.shape[1])))
    T = w["num_edge_types"]
    weights = workloads.init_weights(params, T, seed=1)
    for lw in weights:
        lw["edge_type_attention_weights"] = np.ones(T, np.float32)
    return params, T, w["adjacency_lists"], np.asarray(w["num_incoming_edges_per_type"], np.float32), h0, weights


def float64_forward(params, T, adj, indeg, h0, weights):
    import torch
    from oracle import ggnn_oracle as O
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    with torch.device("cuda"):   # the oracle's own tensors on the GPU too
        out = O.sparse_propagation_torch(d(h0), [d(np.asarray(a, np.int64).reshape(-1, 2)) for a in adj], d(indeg),
                                         [{k: d(v) for k, v in lw.items()} for lw in weights], params, dtype=torch.float64)
    return out.cpu().numpy()


def arm(timer, params, T, adj, indeg, h0_np, weights, attention, tensor_cores, precision):
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    p = dict(params, use_propagation_attention=attention)
    ws = [{k: v for k, v in lw.items() if attention or k != "edge_type_attention_weights"} for lw in weights]
    dev_w = [{k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in lw.items()} for lw in ws]
    eng = PropagationEngine(p, T, precision=precision, attention_tensor_cores=tensor_cores)
    eng.set_weights(dev_w)
    eng.set_save_for_backward(True)
    eng.set_graph_sparse(adj, indeg)
    h0 = torch.from_numpy(h0_np).cuda()
    out = torch.empty_like(h0)
    rows = {"plan": eng.plan, "V": int(h0.shape[0]), "messages": int(sum(np.asarray(a).reshape(-1, 2).shape[0] for a in adj))}
    rows["forward_ms"] = timer.median_ms(lambda: eng.forward(h0, out), True)
    result = out.cpu().numpy()
    grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in dev_w]
    d_out = torch.randn_like(h0)
    d_h0 = torch.empty_like(h0)

    def fwd_bwd():
        eng.forward(h0, out)
        eng.backward(d_out, grads, d_h0)

    rows["fwd_bwd_ms"] = timer.median_ms(fwd_bwd, True)
    eng.sync_check()
    return rows, result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed runs per number (the median is reported; at least 20)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3, help="rounds over the arms (each number is the median over the rounds)")
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("attention_bench.py needs a CUDA device")
    steps = max(args.steps, 20)
    timer = Timer(steps, args.warmup)
    result = {"gpu": gpu_info(), "steps": steps, "warmup": args.warmup, "reps": args.reps, "rows": []}
    print("GPU (name, power limit, max SM clock): %s" % result["gpu"])
    print("%-10s %-14s %10s %10s   plan" % ("workload", "arm", "fwd ms", "fwd+bwd ms"))
    failed = []
    for name, config, hidden in WORKLOADS:
        params, T, adj, indeg, h0, weights = workload(config, hidden)
        runs = {a[0]: [] for a in ARMS}
        check = None
        for _ in range(args.reps):
            for arm_name, attention, tc, precision in ARMS:
                rows, out = arm(timer, params, T, adj, indeg, h0, weights, attention, tc, precision)
                runs[arm_name].append(rows)
                if arm_name == "att-tc-bf16x3":
                    check = out
        ref = float64_forward(params, T, adj, indeg, h0, weights)
        err = float(np.max(np.abs(check - ref)) / np.max(np.abs(ref)))
        if not err < BAR_FORWARD:
            failed.append((name, err))
        for arm_name, _, _, _ in ARMS:
            rs = runs[arm_name]
            r = dict(rs[0], workload=name, hidden=params["hidden_size"], arm=arm_name,
                     forward_ms=statistics.median(x["forward_ms"] for x in rs), fwd_bwd_ms=statistics.median(x["fwd_bwd_ms"] for x in rs),
                     forward_ms_all=[x["forward_ms"] for x in rs], fwd_bwd_ms_all=[x["fwd_bwd_ms"] for x in rs])
            if arm_name == "att-tc-bf16x3":
                r["forward_rel_err_vs_float64"] = err
            result["rows"].append(r)
            print("%-10s %-14s %10.3f %10.3f   %s" % (name, arm_name, r["forward_ms"], r["fwd_bwd_ms"], r["plan"]), flush=True)
        print("%-10s att-tc-bf16x3 forward max|err|/max|ref| against float64: %.2e" % (name, err), flush=True)
    print(json.dumps(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)
    if failed:
        raise SystemExit("att-tc-bf16x3 outputs outside the %.0e bar: %s" % (BAR_FORWARD, failed))


if __name__ == "__main__":
    main()
