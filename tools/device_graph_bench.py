"""Timings of sparse batches built on the device (set_graph_sparse_device, set_graph_gcn_device) against the host route a caller with
GPU-resident adjacency lists has without them: copy the lists to the host (.cpu()) and build there.

GGNN rows (--models ggnn): cfg2's 256 molecules (its model, hidden 100: the tile-local wgmma plan), the 100 000-node batch (its model,
hidden 100), and cfg4's 1 024 molecules with cfg4's model at hidden 256 (the streaming plan).  Arms:
  host     lists on the GPU -> .cpu() + set_graph_sparse (validation, CSR, tile plan, pinned image, upload)
  device   set_graph_sparse_device on the same CUDA tensors
GCN rows (--models gcn; 4 layers as the plug-in's default, adjacency weights on the device): 256 molecules at hidden 100 (the LOCAL wgmma
plan), the 100 000-node batch at hidden 100 (LOCAL) and at hidden 512 with wide_hidden (the streaming plan).  Arms:
  host     list on the GPU -> .cpu() + prepare_graph_gcn_message_weighted (one prepared graph, rebuilt in place) + set_graph_prepared +
           set_message_weights
  device   set_graph_gcn_device + set_message_weights on the same CUDA tensors
Every workload runs with save_for_backward off and on; forward on --precision (bf16x3 by default).  "build" is the host wall clock from the call to the end of a stream synchronise (median of --steps after --warmup); "forward" the device
time between two CUDA events around one forward with the L2 flushed before it, the median of --steps runs after --warmup.  The arms
alternate --rounds times and the figure is the median of the round medians.  Each row also checks that the two arms' graph images are
identical, and that the two forwards are bit-identical.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/device_graph_bench.py [--models ggnn,gcn] [--steps 30] [--warmup 5] [--rounds 3] [--json OUT]
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

WORKLOADS = (("cfg2", "cfg2", None), ("100k", "default_batch_100k_nodes", None), ("cfg4-h256", "cfg4", 256))
# GCN: tag -> (molecules, hidden size); 5 500 molecules are the plug-in's 100 000-node batch (99 046 nodes)
GCN_WORKLOADS = (("gcn-mol256", 256, 100), ("gcn-100k", 5500, 100), ("gcn-100k-h512", 5500, 512))
GCN_LAYERS = 4
ARMS = ("host", "device")


def build_ms(fn, steps, warmup):
    """Median host wall time of fn() up to the end of a synchronise of the current stream."""
    import torch
    times = []
    for i in range(warmup + steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.current_stream().synchronize()
        if i >= warmup:
            times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times)


def run_workload(timer, tag, name, hidden, precision, save, rounds):
    import torch
    from gated_graph_neural_network_samples_b200 import workloads
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    wl = workloads.build(name)
    T = wl["num_edge_types"]
    params = dict(wl["engine_params"])
    if hidden:
        params["hidden_size"] = hidden
    D = int(params["hidden_size"])
    w = workloads.init_weights(params, T, seed=1)
    dev_w = [{{"rnn_kernel": "cand_kernel", "rnn_bias": "cand_bias"}.get(k, k): torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
              for k, x in lw.items()} for lw in w]
    lists = [torch.from_numpy(np.asarray(a, np.int32).reshape(-1, 2)).cuda() for a in wl["adjacency_lists"]]
    indeg = torch.from_numpy(np.asarray(wl["num_incoming_edges_per_type"], np.float32)).cuda()
    V = indeg.shape[0]
    h0 = torch.from_numpy(np.random.default_rng(2).normal(0, 0.1, (V, D)).astype(np.float32)).cuda()
    engines = {}
    for a in ARMS:
        eng = engines[a] = PropagationEngine(params, T, precision=precision)
        eng.set_weights(dev_w)
        eng.set_save_for_backward(save)
    builds = {
        "host": lambda: engines["host"].set_graph_sparse([x.cpu().numpy() for x in lists], indeg.cpu().numpy()),
        "device": lambda: engines["device"].set_graph_sparse_device(V, lists, indeg),
    }
    row = {"model": "ggnn", "workload": tag, "V": V, "M": sum(int(x.shape[0]) for x in lists), "T": T, "D": D, "precision": precision,
           "save": save}
    return dict(row, **compare_arms(timer, engines, builds, h0, rounds))


def compare_arms(timer, engines, builds, h0, rounds):
    """The two arms' build and forward times, alternating over `rounds`, and whether their plans, images and forward bits agree."""
    import torch
    out = {a: torch.empty_like(h0) for a in ARMS}
    per = {(a, c): [] for a in ARMS for c in ("build", "forward")}
    for _ in range(rounds):
        for a in ARMS:
            per[(a, "build")].append(build_ms(builds[a], timer.steps, timer.warmup))
            per[(a, "forward")].append(timer.median_ms(lambda a=a: engines[a].forward(h0, out[a]), flush=True))
    for eng in engines.values():
        eng.sync_check()
    same_image = bool(np.array_equal(engines["host"].graph_image(), engines["device"].graph_image()))
    same_out = bool(torch.equal(engines["host"].forward(h0, out["host"]), engines["device"].forward(h0, out["device"])))
    return {"plan": engines["device"].plan, "same_plan": engines["host"].plan == engines["device"].plan, "same_image": same_image,
            "same_forward_bits": same_out, "ms": {"%s %s" % k: round(statistics.median(v), 4) for k, v in per.items()},
            "round_medians_ms": {"%s %s" % k: [round(x, 4) for x in v] for k, v in per.items()}}


def run_gcn_workload(timer, tag, molecules, hidden, precision, save, rounds):
    import torch
    from gated_graph_neural_network_samples_b200 import packing, synthetic
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    f = packing.pack_gcn_batch(packing.process_raw_graphs_gcn(synthetic.make_molecules(molecules, seed=0)), hidden)
    V = f["initial_node_representation"].shape[0]
    lst = torch.from_numpy(np.ascontiguousarray(f["adjacency_list"], np.int64)).cuda()     # the caller's GPU-resident feed
    w = torch.from_numpy(np.ascontiguousarray(f["adjacency_weights"], np.float32)).cuda()
    rng = np.random.default_rng(1)
    r = np.sqrt(6.0 / (2 * hidden))
    kernels = [torch.from_numpy(rng.uniform(-r, r, (hidden, hidden)).astype(np.float32)).cuda() for _ in range(GCN_LAYERS)]
    h0 = torch.from_numpy(rng.normal(0, 1, (V, hidden)).astype(np.float32)).cuda()
    engines = {}
    for a in ARMS:
        eng = engines[a] = GCNEngine(hidden, GCN_LAYERS, precision=precision, wide_hidden=hidden > 128)
        eng.set_weights(kernels)
        eng.set_save_for_backward(save)

    prepared = [None]   # one prepared graph rebuilt in place, as a producer thread keeps one

    def host():
        eng = engines["host"]
        prepared[0] = eng.prepare_graph_gcn_message_weighted(V, lst.cpu().numpy(), reuse=prepared[0])
        eng.set_graph_prepared(prepared[0])
        eng.set_message_weights(w)

    def device():
        engines["device"].set_graph_gcn_device(V, lst)
        engines["device"].set_message_weights(w)

    row = {"model": "gcn", "workload": tag, "V": V, "M": int(lst.shape[0]), "T": 1, "D": hidden, "precision": precision, "save": save}
    return dict(row, **compare_arms(timer, engines, {"host": host, "device": device}, h0, rounds))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--precision", default="bf16x3", choices=("fp32", "bf16x3", "bf16"))
    ap.add_argument("--models", default="ggnn,gcn", help="comma-separated: ggnn, gcn")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    models = args.models.split(",")
    import torch
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    timer = Timer(args.steps, args.warmup)
    card = gpu_info()
    print("card: %s" % card)
    runs = []
    if "ggnn" in models:
        runs += [lambda save, w=w: run_workload(timer, *w, args.precision, save, args.rounds) for w in WORKLOADS]
    if "gcn" in models:
        runs += [lambda save, w=w: run_gcn_workload(timer, *w, args.precision, save, args.rounds) for w in GCN_WORKLOADS]
    rows = []
    for run in runs:
        for save in (False, True):
            row = run(save)
            row["card"] = card
            rows.append(row)
            print(json.dumps(row))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
