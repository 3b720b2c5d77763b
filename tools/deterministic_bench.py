#!/usr/bin/env python
"""The cost of deterministic mode (ggnn_set_deterministic / torch.use_deterministic_algorithms) on one GPU.

    python tools/deterministic_bench.py [--steps 20] [--warmup 3]

Per workload, both modes alternate call by call in one process, CUDA events around every call, median (and min) over ``--steps`` calls of
each mode after ``--warmup`` calls of each:

* ``backward``: one ggnn_backward (GCN: ggnn_gcn_backward) of a resident forward with saved activations, all weight and bias gradients
  requested (bf16x3 forward plans; the backward is fp32 either way);
* ``train_step``: one step of the plug-in (forward_batch + train_step on a prepared graph: upload, forward, readout, loss, backward, clip,
  Adam), with ``torch.use_deterministic_algorithms`` switched with the mode -- the plug-in sets the engine's flag from it.

Workloads: bench.py's cfg2, cfg1_true_default, cfg4 (1024 molecules, hidden 256, 8 edge types) and the 100 000-node batch for the sparse
GGNN, and tools/gcn_bench.py's 100 000-node batch for the GCN.  Also times ggnn_readout_set_graphs on a shuffled node list of the 100 000-node
batch (where the by-graph permutation is built) against the grouped list.  The device name, power limit and max SM clock are read in the
same run.  Prints one JSON line.  Needs a CUDA device: there is no fallback.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")   # cuBLAS is deterministic under torch's flag only with a fixed workspace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gcn_bench import gpu_info  # noqa: E402

GGNN_WORKLOADS = ("cfg2", "cfg1_true_default", "cfg4", "default_batch_100k_nodes")


def alternate(run_off, run_on, steps, warmup):
    """CUDA-event times of run_off / run_on, called alternately."""
    import torch
    for _ in range(warmup):
        run_off()
        run_on()
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for _ in range(steps):
        for det, fn in ((False, run_off), (True, run_on)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            times[det].append(a.elapsed_time(b))
    out = {}
    for det, name in ((False, "atomic"), (True, "deterministic")):
        out[name] = {"median_ms": statistics.median(times[det]), "min_ms": min(times[det]), "runs": steps}
    out["ratio_median"] = out["deterministic"]["median_ms"] / out["atomic"]["median_ms"]
    return out


def ggnn_backward(wl, args):
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    eng = PropagationEngine(wl["engine_params"], wl["num_edge_types"], precision="bf16x3")
    w = [{k: torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda() for k, v in lw.items()} for lw in wl["weights"]]
    eng.set_weights(w)
    eng.set_save_for_backward(True)
    eng.set_graph_sparse(wl["adjacency_lists"], wl["num_incoming_edges_per_type"])
    h0 = torch.from_numpy(wl["h0"]).cuda()
    out = eng.forward(h0)   # kept alive: the backward reads the forward's states
    g = torch.from_numpy(np.random.default_rng(5).normal(size=wl["h0"].shape).astype(np.float32)).cuda()
    grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in w]
    dh0 = torch.zeros_like(h0)

    def run(det):
        eng.set_deterministic(det)
        eng.backward(g, grads, dh0)

    res = alternate(lambda: run(False), lambda: run(True), args.steps, args.warmup)
    eng.sync_check()
    del out
    res["plan"] = eng.plan
    eng.close()
    return res


def train_step(model_cls, mols, cfg, args, precision="bf16x3"):
    import torch
    with tempfile.TemporaryDirectory() as log_dir:
        m = model_cls({"--log_dir": log_dir, "--precision": precision, "--train_data": mols, "--valid_data": mols[:4],
                       "--config": dict(cfg, batch_size=100000, random_seed=0)})
    m.prepare_graphs_in_producer = False
    feed = next(iter(m.make_minibatch_iterator(m.train_data, True)))
    eng = m.engine
    if hasattr(eng, "prepare_graph_gcn"):
        g = eng.prepare_graph_gcn(feed["initial_node_representation"].shape[0], feed["adjacency_list"], feed["adjacency_weights"],
                                  save_for_backward=True)
    else:
        g = eng.prepare_graph_sparse([feed[k] for k in m.placeholders["adjacency_lists"]], feed["num_incoming_edges_per_type"],
                                     save_for_backward=True)
    g.for_training = True
    tfeed = dict(feed, _prepared_graph=g)
    losses = []

    def step(det):
        torch.use_deterministic_algorithms(det)
        loss, _ = m.forward_batch(tfeed)
        m.train_step(loss)
        m._prepared_pool.clear()
        losses.append(loss.detach())

    res = alternate(lambda: step(False), lambda: step(True), args.steps, args.warmup)
    torch.use_deterministic_algorithms(False)
    eng.sync_check()
    assert all(bool(torch.isfinite(x)) for x in losses), "non-finite training loss"
    res.update(V=int(feed["initial_node_representation"].shape[0]), plan=eng.plan)
    eng.close()
    return res


def gcn_backward(mols, args):
    import torch
    from gated_graph_neural_network_samples_b200 import packing
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    from gcn_bench import HIDDEN, LAYERS
    b = packing.pack_gcn_batch(packing.process_raw_graphs_gcn(mols), HIDDEN)
    V = b["initial_node_representation"].shape[0]
    rng = np.random.default_rng(1)
    eng = GCNEngine(HIDDEN, LAYERS, use_bias=True, precision="bf16x3")
    ks = [torch.from_numpy(rng.uniform(-0.17, 0.17, (HIDDEN, HIDDEN)).astype(np.float32)).cuda() for _ in range(LAYERS)]
    bs = [torch.zeros(HIDDEN, device="cuda") for _ in range(LAYERS)]
    eng.set_weights(ks, bs)
    eng.set_save_for_backward(True)
    eng.set_graph_gcn(V, b["adjacency_list"], b["adjacency_weights"])
    h0 = torch.from_numpy(b["initial_node_representation"]).cuda()
    out = eng.forward(h0)   # kept alive: the backward reads the forward's states
    g = torch.from_numpy(np.random.default_rng(5).normal(size=(V, HIDDEN)).astype(np.float32)).cuda()
    grads = [{"kernel": torch.zeros_like(k), "bias": torch.zeros_like(c)} for k, c in zip(ks, bs)]
    dh0 = torch.zeros_like(h0)

    def run(det):
        eng.set_deterministic(det)
        eng.backward(g, grads, dh0)

    res = alternate(lambda: run(False), lambda: run(True), args.steps, args.warmup)
    eng.sync_check()
    del out
    res.update(V=V, plan=eng.plan)
    eng.close()
    return res


def readout_set_graphs_host(wl):
    """Host time of ggnn_readout_set_graphs (synchronised) on the batch's grouped node list and on a shuffled one (permutation built)."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    eng = PropagationEngine(wl["engine_params"], wl["num_edge_types"])
    gnl = np.asarray(wl["graph_nodes_list"], np.int32)
    out = {}
    for name, lst in (("grouped", gnl), ("shuffled", np.random.default_rng(0).permutation(gnl))):
        times = []
        for _ in range(10):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.readout_set_graphs(wl["num_graphs"], graph_nodes_list=lst)
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
        out[name + "_ms"] = {"median": statistics.median(times), "min": min(times)}
    out["V"] = int(gnl.shape[0])
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("deterministic_bench.py needs a CUDA device")
    from gated_graph_neural_network_samples_b200 import synthetic, workloads
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    only = set(filter(None, args.only.split(",")))
    res = {"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, "workloads": {}}
    for name in GGNN_WORKLOADS:
        if only and name not in only:
            continue
        wl = workloads.build(name)
        cfg = dict(wl["params"])
        r = {"V": wl["V"], "backward": ggnn_backward(wl, args)}
        r["train_step"] = train_step(SparseGGNNChemModel, wl["molecules"], cfg, args)
        if name == "default_batch_100k_nodes":
            r["readout_set_graphs_host"] = readout_set_graphs_host(wl)
        res["workloads"][name] = r
        print(json.dumps({name: r}), file=sys.stderr, flush=True)
    if not only or "gcn_default_batch_100k_nodes" in only:
        from gcn_bench import HIDDEN, LAYERS, WORKLOADS
        mols = synthetic.make_molecules(WORKLOADS["gcn_default_batch_100k_nodes"], seed=0)
        r = {"backward": gcn_backward(mols, args),
             "train_step": train_step(SparseGCNChemModel, mols, {"hidden_size": HIDDEN, "num_timesteps": LAYERS, "gcn_use_bias": True}, args)}
        res["workloads"]["gcn_default_batch_100k_nodes"] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
