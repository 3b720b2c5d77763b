"""Timings of adjacency weights on the device in the sparse GCN model (prepare_graph_gcn_message_weighted / set_message_weights / backward
with d_adjacency_weights), against the host-weighted batch (set_graph_gcn) with the same weights: the packer's D^-1/2 (A+I) D^-1/2.

Workloads (chem_tensorflow_gcn.py defaults: 4 layers, no bias): 256 synthetic molecules at hidden 100, the plug-in's 100 000-node batch
(5 500 molecules) at hidden 100, and that batch at hidden 512 with wide_hidden.  Forward on --precision (bf16x3 by default: the LOCAL wgmma
kernel at hidden 100, the streaming plan at 512), backward on --bwd-precision (bf16x3 by default).  Arms:
  host             forward of the host-weighted batch
  device           forward of the message-weighted batch, its weights set once
  fwd+bwd          forward + backward of the message-weighted batch without d w (every kernel gradient and d h0)
  fwd+bwd+dw       the same with d w (dS on layer 0 too, and the source-row pass that also forms d w, in place of the dH gather)
  reprepare        DropEdge with per-step renormalization the host way: ggnn_prepare_graph_gcn of the batch with new weights and its
                   upload (set_graph_prepared), host time to the end of the upload
  set_weights      the same the device way: one set_message_weights of new weights on the prepared batch
Each arm's number is the device time between two CUDA events around one call (reprepare: wall time around the host prepare and the
upload, then a synchronize), the L2 flushed before each run, median of --steps runs after --warmup; the arms alternate, --rounds times, and
the reported figure is the median of the round medians.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/gcn_message_weights_bench.py [--steps 30] [--warmup 5] [--rounds 3] [--workloads mol256,100k,100k-512] [--json OUT]
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

LAYERS = 4
WORKLOADS = {"mol256": (256, 100), "100k": (5500, 100), "100k-512": (5500, 512)}
ARMS = ("host", "device", "fwd+bwd", "fwd+bwd+dw", "reprepare", "set_weights")


def feed(molecules, D):
    from gated_graph_neural_network_samples_b200 import packing, synthetic
    return packing.pack_gcn_batch(packing.process_raw_graphs_gcn(synthetic.make_molecules(molecules, seed=0)), D)


def wall_ms(timer, fn):
    """Median wall time of fn() + synchronize over timer.steps runs after timer.warmup, the L2 flushed (untimed) before each."""
    import torch
    for _ in range(timer.warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(timer.steps):
        timer.flush_buf.fill_(1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times)


def run_workload(timer, name, precision, bwd_precision, rounds):
    import torch
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    molecules, D = WORKLOADS[name]
    f = feed(molecules, D)
    V = f["initial_node_representation"].shape[0]
    lst = np.ascontiguousarray(f["adjacency_list"], np.int64)
    w = np.ascontiguousarray(f["adjacency_weights"], np.float32)
    nnz = lst.shape[0]
    rng = np.random.default_rng(1)
    r = np.sqrt(6.0 / (2 * D))
    kernels = [torch.from_numpy(rng.uniform(-r, r, (D, D)).astype(np.float32)).cuda() for _ in range(LAYERS)]
    h0 = torch.from_numpy(rng.normal(0, 1, (V, D)).astype(np.float32)).cuda()
    g_out = torch.randn_like(h0)
    dev_w = torch.from_numpy(w).cuda()
    wide = D > 256

    def engine():
        eng = GCNEngine(D, LAYERS, precision=precision, wide_hidden=wide)
        eng.set_weights(kernels)
        eng.set_save_for_backward(True)
        eng.set_backward_precision(bwd_precision)
        return eng

    host, dev = engine(), engine()
    host.set_graph_gcn(V, lst, w)
    prepared = dev.prepare_graph_gcn_message_weighted(V, lst)
    dev.set_graph_prepared(prepared)
    dev.set_message_weights(dev_w)
    out_h, out_d = torch.empty_like(h0), torch.empty_like(h0)
    grads = [{"kernel": torch.zeros_like(k)} for k in kernels]
    dh0, dw = torch.zeros_like(h0), torch.zeros(nnz, device="cuda")
    # DropEdge: a fresh mask and renormalization per step; the timed arms take turns over a few precomputed weight vectors
    drops = [np.where(np.random.default_rng(10 + i).random(nnz) < 0.9, w, 0.0).astype(np.float32) for i in range(4)]
    drops_dev = [torch.from_numpy(x).cuda() for x in drops]
    rep = engine()
    rep_graph = [None]
    k = [0]

    def fwd_bwd(with_dw):
        def fn():
            dev.forward(h0, out_d)
            dev.backward(g_out, grads, dh0, d_adjacency_weights=dw if with_dw else None)
        return fn

    def reprepare():
        k[0] = (k[0] + 1) % len(drops)
        rep_graph[0] = rep.prepare_graph_gcn(V, lst, drops[k[0]], reuse=rep_graph[0])
        rep.set_graph_prepared(rep_graph[0])

    def set_weights():
        k[0] = (k[0] + 1) % len(drops)
        dev.set_message_weights(drops_dev[k[0]])

    fns = {"host": lambda: host.forward(h0, out_h), "device": lambda: dev.forward(h0, out_d), "fwd+bwd": fwd_bwd(False),
           "fwd+bwd+dw": fwd_bwd(True), "set_weights": set_weights}
    per = {a: [] for a in ARMS}
    for _ in range(rounds):
        for a in ARMS:
            if a == "reprepare":
                per[a].append(wall_ms(timer, reprepare))
            else:
                if a in ("device", "fwd+bwd", "fwd+bwd+dw"):
                    dev.set_message_weights(dev_w)
                per[a].append(timer.median_ms(fns[a], flush=True))
    host.sync_check(); dev.sync_check(); rep.sync_check()
    dev.set_message_weights(dev_w)
    bit_identical = bool(torch.equal(host.forward(h0, out_h), dev.forward(h0, out_d)))
    res = {a: statistics.median(v) for a, v in per.items()}
    return {"workload": name, "V": V, "nnz": nnz, "D": D, "layers": LAYERS, "precision": precision, "bwd_precision": bwd_precision,
            "plan_host": host.plan, "plan_device": dev.plan, "forward_bit_identical": bit_identical,
            "ms": {a: round(v, 4) for a, v in res.items()}, "round_medians_ms": {a: [round(x, 4) for x in v] for a, v in per.items()},
            "device_forward_cost": round(res["device"] / res["host"] - 1.0, 4),
            "dw_cost_of_fwd_bwd": round(res["fwd+bwd+dw"] / res["fwd+bwd"] - 1.0, 4),
            "reprepare_over_set_weights": round(res["reprepare"] / res["set_weights"], 1)}


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
