#!/usr/bin/env python
"""The fp32 (FFMA) against the bf16x3 (wgmma) backward, ggnn_set_backward_precision, on one GPU.

    python tools/tc_backward_bench.py [--steps 20] [--warmup 3] [--only cfg4,...]

Per workload and per mode (atomic, and deterministic: ggnn_set_deterministic / torch.use_deterministic_algorithms), the two backward
precisions alternate call by call in one process, CUDA events around every call, median (and min) over ``--steps`` calls of each after
``--warmup`` calls of each:

* ``backward``: one ggnn_backward (GCN: ggnn_gcn_backward) of a resident bf16x3 forward with saved activations, every weight and bias
  gradient and d h0 requested;
* ``train_step``: one step of the plug-in (forward_batch + train_step: forward, readout, loss, backward, clip, Adam), the engine's backward
  precision switched before each step.  Sparse GGNN and GCN run the whole batch on a prepared graph (as tools/deterministic_bench.py); the
  dense plug-in runs one 64-graph batch and sets its graph inside the step.

Workloads: bench.py's cfg2, cfg1_true_default, cfg3_dense and cfg4, cfg4's model at hidden 512, the 100 000-node batch, and
tools/gcn_bench.py's 100 000-node GCN batch.  The device name, power limit and max SM clock are read in the same run.  Prints one JSON line.
Needs a CUDA device: there is no fallback.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")   # cuBLAS is deterministic under torch's flag only with a fixed workspace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gcn_bench import gpu_info  # noqa: E402

WORKLOADS = ("cfg2", "cfg1_true_default", "cfg3_dense", "cfg4", "cfg4_hidden512", "default_batch_100k_nodes", "gcn_default_batch_100k_nodes")
PRECS = ("fp32", "bf16x3")
DENSE_BATCH = 64   # graphs per dense training step: the dense plug-in yields only full batches of one size bucket


def alternate(run, steps, warmup):
    """CUDA-event times of run("fp32") / run("bf16x3"), called alternately."""
    import torch
    for _ in range(warmup):
        for p in PRECS:
            run(p)
    torch.cuda.synchronize()
    times = {p: [] for p in PRECS}
    for _ in range(steps):
        for p in PRECS:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            run(p)
            b.record()
            b.synchronize()
            times[p].append(a.elapsed_time(b))
    out = {p: {"median_ms": statistics.median(times[p]), "min_ms": min(times[p]), "runs": steps} for p in PRECS}
    out["speedup_median"] = out["fp32"]["median_ms"] / out["bf16x3"]["median_ms"]
    return out


def build(name):
    """The workload dict of workloads.build (cfg4_hidden512: cfg4's molecules and model at hidden 512)."""
    from gated_graph_neural_network_samples_b200 import workloads
    if name != "cfg4_hidden512":
        return workloads.build(name)
    from wide_hidden_bench import cfg4_at
    params, T, mols, b = cfg4_at(512)
    return {"kind": "sparse", "params": params, "engine_params": params, "num_edge_types": T, "molecules": mols,
            "adjacency_lists": b["adjacency_lists"], "num_incoming_edges_per_type": b["num_incoming_edges_per_type"],
            "h0": b["initial_node_representation"], "weights": workloads.init_weights(params, T, seed=1),
            "V": int(b["initial_node_representation"].shape[0])}


def ggnn_backward(wl, det, args):
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    eng = PropagationEngine(wl["engine_params"], wl["num_edge_types"], precision="bf16x3")
    w = [{k: torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda() for k, v in lw.items()} for lw in wl["weights"]]
    eng.set_weights(w)
    eng.set_save_for_backward(True)
    if wl["kind"] == "dense":
        eng.set_graph_dense(wl["adjacency_matrix"])
    else:
        eng.set_graph_sparse(wl["adjacency_lists"], wl["num_incoming_edges_per_type"])
    eng.set_deterministic(det)
    h0 = torch.from_numpy(np.ascontiguousarray(wl["h0"], np.float32)).cuda()
    out = eng.forward(h0)   # kept alive: the backward reads the forward's states
    g = torch.from_numpy(np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)).cuda()
    grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in w]
    dh0 = torch.zeros_like(h0)

    def run(prec):
        eng.set_backward_precision(prec)
        eng.backward(g, grads, dh0)

    res = alternate(run, args.steps, args.warmup)
    eng.sync_check()
    del out
    res["plan"] = eng.plan
    eng.close()
    return res


def gcn_backward(mols, det, args):
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
    eng.set_deterministic(det)
    h0 = torch.from_numpy(b["initial_node_representation"]).cuda()
    out = eng.forward(h0)
    g = torch.from_numpy(np.random.default_rng(5).normal(size=(V, HIDDEN)).astype(np.float32)).cuda()
    grads = [{"kernel": torch.zeros_like(k), "bias": torch.zeros_like(c)} for k, c in zip(ks, bs)]
    dh0 = torch.zeros_like(h0)

    def run(prec):
        eng.set_backward_precision(prec)
        eng.backward(g, grads, dh0)

    res = alternate(run, args.steps, args.warmup)
    eng.sync_check()
    del out
    res.update(V=V, plan=eng.plan)
    eng.close()
    return res


def train_step(model_cls, mols, cfg, det, args):
    import torch
    with tempfile.TemporaryDirectory() as log_dir:
        m = model_cls({"--log_dir": log_dir, "--precision": "bf16x3", "--train_data": mols, "--valid_data": mols[:4],
                       "--config": dict(cfg, random_seed=0)})
    m.prepare_graphs_in_producer = False
    feed = next(iter(m.make_minibatch_iterator(m.train_data, True)))
    eng = m.engine
    if hasattr(eng, "prepare_graph_gcn"):
        g = eng.prepare_graph_gcn(feed["initial_node_representation"].shape[0], feed["adjacency_list"], feed["adjacency_weights"],
                                  save_for_backward=True)
    elif "adjacency_lists" in m.placeholders:
        g = eng.prepare_graph_sparse([feed[k] for k in m.placeholders["adjacency_lists"]], feed["num_incoming_edges_per_type"],
                                     save_for_backward=True)
    else:
        g = None   # the dense plug-in sets its graph in hook 2
    if g is not None:
        g.for_training = True
        feed = dict(feed, _prepared_graph=g)
    torch.use_deterministic_algorithms(det)
    losses = []

    def step(prec):
        eng.set_backward_precision(prec)
        loss, _ = m.forward_batch(feed)
        m.train_step(loss)
        if g is not None:
            m._prepared_pool.clear()
        losses.append(loss.detach())

    try:
        res = alternate(step, args.steps, args.warmup)
    finally:
        torch.use_deterministic_algorithms(False)
    eng.sync_check()
    assert all(bool(torch.isfinite(x)) for x in losses), "non-finite training loss"
    res.update(V=int(feed["initial_node_representation"].reshape(-1, eng.D).shape[0]), plan=eng.plan)
    eng.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tc_backward_bench.py needs a CUDA device")
    from gated_graph_neural_network_samples_b200 import synthetic
    from gated_graph_neural_network_samples_b200.chem_dense import DenseGGNNChemModel
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    only = set(filter(None, args.only.split(",")))
    res = {"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, "workloads": {}}
    for name in WORKLOADS:
        if only and name not in only:
            continue
        r = {}
        if name == "gcn_default_batch_100k_nodes":
            from gcn_bench import HIDDEN, LAYERS, WORKLOADS as GCN_WORKLOADS
            mols = synthetic.make_molecules(GCN_WORKLOADS[name], seed=0)
            cfg = {"hidden_size": HIDDEN, "num_timesteps": LAYERS, "gcn_use_bias": True, "batch_size": 100000}
            for det, mode in ((False, "atomic"), (True, "deterministic")):
                r[mode] = {"backward": gcn_backward(mols, det, args), "train_step": train_step(SparseGCNChemModel, mols, cfg, det, args)}
        else:
            wl = build(name)
            r["V"] = wl["V"]
            mols = wl.get("molecules") or synthetic.make_molecules(wl["num_graphs"], seed=0, num_bond_types=wl["num_edge_types"])
            if wl["kind"] == "dense":
                cls, cfg = DenseGGNNChemModel, dict(wl["params"], batch_size=DENSE_BATCH)
            else:
                cls, cfg = SparseGGNNChemModel, dict(wl["params"], batch_size=10 ** 6)
            for det, mode in ((False, "atomic"), (True, "deterministic")):
                r[mode] = {"backward": ggnn_backward(wl, det, args), "train_step": train_step(cls, mols, cfg, det, args)}
        res["workloads"][name] = r
        print(json.dumps({name: r}), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
