"""Timings of message weights in the sparse GGNN model (prepare_graph_sparse_weighted / set_message_weights / backward with
d_message_weights), every weight drawn from U(0.25, 1.75).

Workloads: cfg2 (256 molecules, hidden 100, [4] timesteps, 4 edge types), the 100 000-node batch (5500 molecules, cfg2's model) and cfg4's
model (1024 molecules, 8 edge types, [2, 2, 2, 2] with a residual input) at hidden 256 and 512.  Forward on --precision (bf16x3 by
default: the tile-local wgmma kernel at hidden 100, the streaming kernels above 128), backward on --bwd-precision (bf16x3 by default).
Arms:
  unweighted       forward of the batch through set_graph_sparse
  weighted         forward of the message-weighted batch (on the streaming plan every (target, type) pair with messages is a virtual row)
  weighted+bwd     forward + backward of the message-weighted batch without d w (every weight gradient and d h0)
  weighted+bwd+dw  the same with d w (one P = dx' . W^T GEMM and one per-slot dot-product launch per timestep)
Each arm's number is the device time between two CUDA events around one call, the L2 flushed before each run, median of --steps runs after
--warmup; the arms alternate, --rounds times, and the reported figure is the median of the round medians.  The card's name, power limit and
maximum SM clock are read in the same run (an nvidia-smi query).

    python tools/message_weights_bench.py [--steps 30] [--warmup 5] [--rounds 3] [--workloads cfg2,100k,cfg4-256,cfg4-512] [--json OUT]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.wide_hidden_bench import Timer, gpu_info  # noqa: E402

WORKLOADS = {"cfg2": ("cfg2", None), "100k": ("default_batch_100k_nodes", None), "cfg4-256": ("cfg4", 256), "cfg4-512": ("cfg4", 512)}
ARMS = ("unweighted", "weighted", "weighted+bwd", "weighted+bwd+dw")


def load(name):
    from gated_graph_neural_network_samples_b200 import workloads
    cfg, D = WORKLOADS[name]
    if D is not None:
        saved = dict(workloads.CONFIGS[cfg]["params"])
        workloads.CONFIGS[cfg]["params"]["hidden_size"] = D
        try:
            return workloads.build(cfg)
        finally:
            workloads.CONFIGS[cfg]["params"] = saved
    return workloads.build(cfg)


def run_workload(timer, name, precision, bwd_precision, rounds):
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    wl = load(name)
    p, T = wl["engine_params"], wl["num_edge_types"]
    D = int(p["hidden_size"])
    dev_w = [{("cand_kernel" if k == "rnn_kernel" else "cand_bias" if k == "rnn_bias" else k): torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda()
              for k, v in lw.items()} for lw in wl["weights"]]
    h0 = torch.from_numpy(np.ascontiguousarray(wl["h0"], np.float32)).cuda()
    M = wl["M"]
    mw = torch.from_numpy(np.random.default_rng(2).uniform(0.25, 1.75, M).astype(np.float32)).cuda()
    g_out = torch.randn_like(h0)

    def engine(weighted):
        eng = PropagationEngine(p, T, precision=precision)
        eng.set_weights(dev_w)
        eng.set_save_for_backward(True)
        eng.set_backward_precision(bwd_precision)
        if weighted:
            eng.set_graph_prepared(eng.prepare_graph_sparse_weighted(wl["adjacency_lists"], wl["num_incoming_edges_per_type"]))
            eng.set_message_weights(mw)
        else:
            eng.set_graph_sparse(wl["adjacency_lists"], wl["num_incoming_edges_per_type"])
        return eng

    plain, weighted = engine(False), engine(True)
    out_p, out_w = torch.empty_like(h0), torch.empty_like(h0)
    grads = [{k: torch.zeros_like(t) for k, t in lw.items()} for lw in dev_w]
    dh0, dmw = torch.zeros_like(h0), torch.zeros(M, device="cuda")

    def fwd(eng, out):
        return lambda: eng.forward(h0, out)

    def fwd_bwd(with_dw):
        def f():
            weighted.forward(h0, out_w)
            weighted.backward(g_out, grads, dh0, d_message_weights=dmw if with_dw else None)
        return f

    fns = {"unweighted": fwd(plain, out_p), "weighted": fwd(weighted, out_w), "weighted+bwd": fwd_bwd(False), "weighted+bwd+dw": fwd_bwd(True)}
    per = {a: [] for a in ARMS}
    for _ in range(rounds):
        for a in ARMS:
            per[a].append(timer.median_ms(fns[a], flush=True))
    plain.sync_check(); weighted.sync_check()
    res = {a: statistics.median(v) for a, v in per.items()}
    row = {"workload": name, "V": wl["V"], "M": M, "D": D, "T": T, "timesteps": wl["timesteps"], "precision": precision,
           "bwd_precision": bwd_precision, "plan_unweighted": plain.plan, "plan_weighted": weighted.plan,
           "ms": {a: round(v, 4) for a, v in res.items()}, "round_medians_ms": {a: [round(x, 4) for x in v] for a, v in per.items()},
           "weighted_forward_cost": round(res["weighted"] / res["unweighted"] - 1.0, 4),
           "dw_cost_of_fwd_bwd": round(res["weighted+bwd+dw"] / res["weighted+bwd"] - 1.0, 4),
           "extra_P_scratch_bytes": wl["V"] * T * D * 4, "extra_gemm_flops_per_step": 2 * wl["V"] * T * D * D}
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--precision", default="bf16x3", choices=("fp32", "bf16x3", "bf16"))
    ap.add_argument("--bwd-precision", default="bf16x3", choices=("fp32", "bf16x3"))
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    timer = Timer(args.steps, args.warmup)
    card = gpu_info()
    print("card: %s" % card)
    rows = []
    for name in args.workloads.split(","):
        row = run_workload(timer, name, args.precision, args.bwd_precision, args.rounds)
        row["card"] = card
        rows.append(row)
        print(json.dumps(row))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
