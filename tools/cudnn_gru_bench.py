"""Timings of CudnnCompatibleGRUCell on the streaming wgmma kernels (GGNN_CELL_CUDNN_GRU_TENSOR_CORES) against the fp32 kernels it ran on
before, with the GRU cell at bf16x3 as the yardstick (it does the same MACs per step).

Workloads (seeded, workloads.py):
  cfg2        256 molecules, hidden 100, 4 edge types, layer_timesteps [4]
  100k        the reference's default batch of about 100 000 nodes (default_batch_100k_nodes), hidden 100, [4]
  cfg4        1024 molecules, hidden 256, 8 edge types, [2, 2, 2, 2] with a residual input
  cfg4-h512   the same batch and model at hidden 512
Arms per workload:
  cudnn-fp32        CudnnCompatibleGRUCell on the fp32 kernels (GGNN_CELL_CUDNN_GRU, the only way to run it before)
  cudnn-tc-bf16x3   CudnnCompatibleGRUCell on the streaming wgmma kernels at bf16x3 (GGNN_CELL_CUDNN_GRU_TENSOR_CORES)
  gru-bf16x3        the GRU cell at bf16x3 (its own plan: the tile-local kernel up to hidden 128, the streaming kernels above)
Each arm times the forward and forward + backward (save_for_backward, every weight gradient and d h0) with CUDA events after --warmup
runs, as the median of --steps runs with the L2 flushed before each run.  The arms run in turn, --reps times, and each number is the
median over the repetitions.  The timed forward of both CudnnCompatibleGRUCell arms is compared with float64
(oracle.sparse_propagation_torch on the GPU) against the forward bar, 1e-4 of max|ref|, so that a fast wrong answer fails the run.  The
card's name, power limit and maximum SM clock are read in the same run (an nvidia-smi query).

    python tools/cudnn_gru_bench.py [--steps 30] [--warmup 5] [--reps 3] [--json OUT]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.attention_bench import float64_forward  # noqa: E402
from tools.wide_hidden_bench import Timer, gpu_info  # noqa: E402

WORKLOADS = (("cfg2", "cfg2", None), ("100k", "default_batch_100k_nodes", None), ("cfg4", "cfg4", None), ("cfg4-h512", "cfg4", 512))
# (name, cell, precision, cudnn_gru_tensor_cores)
ARMS = (("cudnn-fp32", "CudnnCompatibleGRUCell", "fp32", False), ("cudnn-tc-bf16x3", "CudnnCompatibleGRUCell", "bf16x3", True),
        ("gru-bf16x3", "GRU", "bf16x3", False))
BAR_FORWARD = 1e-4


def workload(config, hidden):
    """(params, T, adjacency lists, in-degrees, h0)."""
    from gated_graph_neural_network_samples_b200 import workloads
    w = workloads.build(config)
    params = dict(w["engine_params"], graph_rnn_activation="tanh")
    h0 = np.asarray(w["h0"], np.float32)
    if hidden is not None:   # the same molecules at another width: the annotations zero-padded, as the packer pads them
        params["hidden_size"] = hidden
        h0 = np.pad(h0, ((0, 0), (0, hidden - h0.shape[1])))
    return params, w["num_edge_types"], w["adjacency_lists"], np.asarray(w["num_incoming_edges_per_type"], np.float32), h0


def weights_of(params, T, cell):
    """Seeded weights of the cell: the oracle's initialisers (CudnnCompatibleGRUCell's two candidate biases drawn), fp32."""
    from oracle import ggnn_oracle as O
    w = O.init_sparse_weights(dict(params, graph_rnn_cell=cell), T, np.random.default_rng(1))
    return [{k: np.ascontiguousarray(v, np.float32) for k, v in lw.items()} for lw in w]


def arm(timer, params, T, adj, indeg, h0_np, weights, precision, tensor_cores):
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    dev_w = [{k: torch.from_numpy(v).cuda() for k, v in lw.items()} for lw in weights]
    eng = PropagationEngine(params, T, precision=precision, cudnn_gru_tensor_cores=tensor_cores)
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
        raise SystemExit("cudnn_gru_bench.py needs a CUDA device")
    steps = max(args.steps, 20)
    timer = Timer(steps, args.warmup)
    result = {"gpu": gpu_info(), "steps": steps, "warmup": args.warmup, "reps": args.reps, "rows": []}
    print("GPU (name, power limit, max SM clock): %s" % result["gpu"])
    print("%-10s %-16s %10s %10s   plan" % ("workload", "arm", "fwd ms", "fwd+bwd ms"))
    failed = []
    for name, config, hidden in WORKLOADS:
        params, T, adj, indeg, h0 = workload(config, hidden)
        weights = {cell: weights_of(params, T, cell) for cell in ("CudnnCompatibleGRUCell", "GRU")}
        runs = {a[0]: [] for a in ARMS}
        outs = {}
        for _ in range(args.reps):
            for arm_name, cell, precision, tc in ARMS:
                rows, out = arm(timer, dict(params, graph_rnn_cell=cell), T, adj, indeg, h0, weights[cell], precision, tc)
                runs[arm_name].append(rows)
                outs[arm_name] = out
        cp = dict(params, graph_rnn_cell="CudnnCompatibleGRUCell")
        ref = float64_forward(cp, T, adj, indeg, h0, weights["CudnnCompatibleGRUCell"])
        errs = {a: float(np.max(np.abs(outs[a] - ref)) / np.max(np.abs(ref))) for a in ("cudnn-fp32", "cudnn-tc-bf16x3")}
        failed += [(name, a, e) for a, e in errs.items() if not e < BAR_FORWARD]
        for arm_name, _, _, _ in ARMS:
            rs = runs[arm_name]
            r = dict(rs[0], workload=name, hidden=params["hidden_size"], arm=arm_name,
                     forward_ms=statistics.median(x["forward_ms"] for x in rs), fwd_bwd_ms=statistics.median(x["fwd_bwd_ms"] for x in rs),
                     forward_ms_all=[x["forward_ms"] for x in rs], fwd_bwd_ms_all=[x["fwd_bwd_ms"] for x in rs])
            if arm_name in errs:
                r["forward_rel_err_vs_float64"] = errs[arm_name]
            result["rows"].append(r)
            print("%-10s %-16s %10.3f %10.3f   %s" % (name, arm_name, r["forward_ms"], r["fwd_bwd_ms"], r["plan"]), flush=True)
        print("%-10s forward max|err|/max|ref| against float64: fp32 %.2e, bf16x3 streaming %.2e" % (name, errs["cudnn-fp32"],
                                                                                                   errs["cudnn-tc-bf16x3"]), flush=True)
    print(json.dumps(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)
    if failed:
        raise SystemExit("outputs outside the %.0e bar: %s" % (BAR_FORWARD, failed))


if __name__ == "__main__":
    main()
