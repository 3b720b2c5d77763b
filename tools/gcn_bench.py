#!/usr/bin/env python
"""Timings of the sparse GCN model (SparseGCNChemModel, chem_tensorflow_gcn.py defaults: hidden 100, 4 layers, no bias) on one GPU.

    python tools/gcn_bench.py [--steps 30] [--warmup 5]

Workloads: 256 synthetic molecules in one batch (the GCN counterpart of bench.py's cfg2) and one batch at the plug-in's default
100 000-node budget (5 500 molecules).  Per workload and precision (bf16x3, fp32):

* ``forward``: one propagation (ggnn_forward) with graph, states and weights resident, CUDA events around every run, median and min, with
  L2 flushed (256 MiB write, untimed) before every run and with a hot L2;
* ``train_step``: ``forward_batch`` + ``train_step`` of the plug-in on a prepared graph (upload, forward with saved states, fused readout,
  loss, backward, per-variable clip, Adam), CUDA events, L2 flushed before every step;
* node updates/s = V * layers / time;
* ``host``: per-batch host cost of the flat packer (packing.FlatGCNGraphs.pack), the per-graph packer (packing.pack_gcn_batch) and the
  prepare call (ggnn_prepare_graph_gcn, the producer thread's share), best of several runs on this host's CPU;
* ``cpu_torch_fp32``: the fp32 torch-CPU restatement of the reference graph (tests/gcn_oracle.gcn_propagation_torch) on this host's cores,
  timed beside it -- a CPU baseline, not the reference itself (TensorFlow 1.3 cannot be installed).

The device name, power limit and max SM clock are read in the same run (read-only nvidia-smi query).  Prints one JSON line.  Needs a
CUDA device: there is no fallback.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HIDDEN, LAYERS = 100, 4
WORKLOADS = {"gcn_256_molecules": 256, "gcn_default_batch_100k_nodes": 5500}
PRECISIONS = ("bf16x3", "fp32")


def gpu_info():
    import torch
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=" + q, "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        fields = [x.strip() for x in r.stdout.strip().split(",")]
        smi = dict(zip(q.split(","), fields)) if len(fields) == 3 else {"error": (r.stderr or r.stdout).strip()[-200:]}
    except Exception as exc:   # noqa: BLE001 -- reported, the timings still stand
        smi = {"error": str(exc)}
    return dict(smi, torch_device_name=torch.cuda.get_device_name())


def best_ms(fn, runs):
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return min(times)


def event_times(fn, steps, flush=None):
    import torch
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for a, b in ev:
        if flush is not None:
            flush()
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    t = [a.elapsed_time(b) for a, b in ev]
    return {"median_ms": statistics.median(t), "min_ms": min(t), "runs": steps}


def cpu_restatement(feed, kernels, budget_s=10.0, max_runs=20):
    import torch
    from tests import gcn_oracle as G
    h0 = torch.from_numpy(feed["initial_node_representation"])
    w = torch.from_numpy(feed["adjacency_weights"].astype(np.float32))
    ks = [torch.from_numpy(k) for k in kernels]
    with torch.no_grad():
        out = G.gcn_propagation_torch(h0, feed["adjacency_list"], w, ks)       # warm-up (thread pool, allocator)
        times, t_start = [], time.perf_counter()
        while len(times) < max_runs and (len(times) < 3 or time.perf_counter() - t_start < budget_s):
            t0 = time.perf_counter()
            G.gcn_propagation_torch(h0, feed["adjacency_list"], w, ks)
            times.append((time.perf_counter() - t0) * 1e3)
    return out.numpy(), {"median_ms": statistics.median(times), "min_ms": min(times), "runs": len(times),
                         "threads": torch.get_num_threads(),
                         "what": "fp32 torch-CPU restatement of gcn:59-82 (tests/gcn_oracle.gcn_propagation_torch) on this host, no_grad"}


def run_workload(name, n_mols, args, flush):
    import torch
    from gated_graph_neural_network_samples_b200 import packing, synthetic
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    mols = synthetic.make_molecules(n_mols, seed=0)
    res = {"precisions": {}}
    for prec in PRECISIONS:
        with tempfile.TemporaryDirectory() as log_dir:
            m = SparseGCNChemModel({"--log_dir": log_dir, "--precision": prec, "--train_data": mols, "--valid_data": mols[:4],
                                    "--config": {"batch_size": 100000, "hidden_size": HIDDEN, "num_timesteps": LAYERS, "gcn_use_bias": False,
                                                 "random_seed": 0}})
        m.prepare_graphs_in_producer = False
        feed = next(iter(m.make_minibatch_iterator(m.train_data, False)))
        V, nnz = feed["initial_node_representation"].shape[0], feed["adjacency_list"].shape[0]
        if "host" not in res:
            graphs = list(m.train_data[:feed["num_graphs"]])
            t0 = time.perf_counter()
            flat = packing.FlatGCNGraphs(graphs)
            flatten_ms = (time.perf_counter() - t0) * 1e3
            idx = np.arange(len(graphs))
            res.update(V=V, nnz=nnz, graphs=feed["num_graphs"], hidden=HIDDEN, layers=LAYERS, use_bias=False)
            res["host"] = {"flat_pack_ms": best_ms(lambda: flat.pack(idx, HIDDEN), 5),
                           "per_graph_pack_ms": best_ms(lambda: packing.pack_gcn_batch(graphs, HIDDEN), 3),
                           "flatten_once_ms": flatten_ms, "cpu_count": len(os.sched_getaffinity(0))}
        eng = m.engine
        kernels = [k.detach().contiguous() for k in m.weights["edge_weights"]]
        eng.set_weights(kernels)
        eng.set_save_for_backward(False)
        eng.set_graph_gcn(V, feed["adjacency_list"], feed["adjacency_weights"])
        eng.set_state_dropout(1.0, 0)
        h0 = torch.from_numpy(feed["initial_node_representation"]).cuda()
        out = torch.empty_like(h0)
        for _ in range(args.warmup):
            eng.forward(h0, out)
        torch.cuda.synchronize()
        fwd = {"l2_flushed": event_times(lambda: eng.forward(h0, out), args.steps, flush),
               "l2_hot": event_times(lambda: eng.forward(h0, out), args.steps)}
        eng.sync_check()
        plan = eng.plan
        if "cpu_torch_fp32" not in res:
            cpu_out, res["cpu_torch_fp32"] = cpu_restatement(feed, [k.cpu().numpy() for k in kernels])
            res["cpu_torch_fp32"]["node_updates_per_s"] = V * LAYERS / (res["cpu_torch_fp32"]["median_ms"] * 1e-3)
        err = float(np.max(np.abs(out.cpu().numpy() - cpu_out)) / np.max(np.abs(cpu_out)))
        # the training step of the plug-in on a prepared graph (built once here; in training the producer thread builds one per batch)
        g = eng.prepare_graph_gcn(V, feed["adjacency_list"], feed["adjacency_weights"], save_for_backward=True)
        prepare_ms = best_ms(lambda: eng.prepare_graph_gcn(V, feed["adjacency_list"], feed["adjacency_weights"], save_for_backward=True,
                                                           reuse=g), 5)
        g.for_training = True
        tfeed = dict(feed, _prepared_graph=g, out_layer_dropout_keep_prob=1.0)
        losses = []

        def train_step():
            loss, _ = m.forward_batch(tfeed)
            m.train_step(loss)
            m._prepared_pool.clear()
            losses.append(loss.detach())

        for _ in range(args.warmup):
            train_step()
        torch.cuda.synchronize()
        tr = event_times(train_step, args.steps, flush)
        eng.sync_check()
        assert all(bool(torch.isfinite(x)) for x in losses), "non-finite training loss"
        res["host"]["prepare_ms_" + prec] = prepare_ms
        res["precisions"][prec] = {
            "plan": plan, "forward": fwd, "max_rel_err_vs_cpu_restatement": err,
            "forward_node_updates_per_s": V * LAYERS / (fwd["l2_flushed"]["median_ms"] * 1e-3),
            "forward_node_updates_per_s_hot_l2": V * LAYERS / (fwd["l2_hot"]["median_ms"] * 1e-3),
            "train_step": tr, "train_step_node_updates_per_s": V * LAYERS / (tr["median_ms"] * 1e-3)}
        m.engine.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if args.steps < 20:
        raise SystemExit("--steps must be at least 20")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("gcn_bench.py needs a CUDA device (the GCN engine has no CPU path)")
    torch.cuda.set_device(0)
    flush_buf = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    line = {"metric": "sparse GCN (SparseGCNChemModel) node updates/s", "gpu": gpu_info(),
            "model": {"hidden_size": HIDDEN, "num_timesteps": LAYERS, "gcn_use_bias": False},
            "workloads": {name: run_workload(name, n, args, lambda: flush_buf.fill_(1)) for name, n in WORKLOADS.items()}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
