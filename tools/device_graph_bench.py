"""Timings of sparse batches built on the device (set_graph_sparse_device) against the host route a caller with GPU-resident adjacency
lists has without it: copy the lists and the in-degree table to the host (.cpu()) and call set_graph_sparse.

Workloads: cfg2's 256 molecules (its model, hidden 100: the tile-local wgmma plan), the 100 000-node batch (its model, hidden 100), and
cfg4's 1 024 molecules with cfg4's model at hidden 256 (the streaming plan); each with save_for_backward off and on; forward on --precision
(bf16x3 by default).  Arms:
  host     lists on the GPU -> .cpu() + set_graph_sparse (validation, CSR, tile plan, pinned image, upload)
  device   set_graph_sparse_device on the same CUDA tensors
"build" is the host wall clock from the call to the end of a stream synchronise (median of --steps after --warmup); "forward" the device
time between two CUDA events around one forward with the L2 flushed before it, the median of --steps runs after --warmup.  The arms
alternate --rounds times and the figure is the median of the round medians.  Each row also checks that the two arms' graph images are
identical.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/device_graph_bench.py [--steps 30] [--warmup 5] [--rounds 3] [--json OUT]
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
    return {"workload": tag, "V": V, "M": sum(int(x.shape[0]) for x in lists), "T": T, "D": D, "precision": precision, "save": save,
            "plan": engines["device"].plan, "same_plan": engines["host"].plan == engines["device"].plan, "same_image": same_image,
            "same_forward_bits": same_out, "ms": {"%s %s" % k: round(statistics.median(v), 4) for k, v in per.items()},
            "round_medians_ms": {"%s %s" % k: [round(x, 4) for x in v] for k, v in per.items()}}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--precision", default="bf16x3", choices=("fp32", "bf16x3", "bf16"))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    timer = Timer(args.steps, args.warmup)
    card = gpu_info()
    print("card: %s" % card)
    rows = []
    for tag, name, hidden in WORKLOADS:
        for save in (False, True):
            row = run_workload(timer, tag, name, hidden, args.precision, save, args.rounds)
            row["card"] = card
            rows.append(row)
            print(json.dumps(row))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
