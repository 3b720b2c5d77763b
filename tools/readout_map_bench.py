"""Timings of the readout map built from a CUDA graph_nodes_list (readout_set_graphs with a CUDA tensor, ggnn_readout_set_graphs_device)
against the host route a caller with a GPU-resident list has without it: copy the list to the host (.cpu()) and build there.

Map rows: cfg2's 256 molecules and the 100 000-node batch (5 500 molecules, 99 046 nodes), each with the packer's grouped list and with a
shuffled one.  Arms:
  host     list on the GPU -> .cpu() + readout_set_graphs (the host builder and its upload)
  device   readout_set_graphs on the same CUDA tensor
Each is the host wall clock from the call to the end of a stream synchronise, the median of --steps after --warmup, the arms alternating
call by call.  Each row also checks that the two arms leave the same map (ggnn_readout_map).

Step rows: one training step (forward_batch, then train_step: backward, clip and Adam, to the end of a device synchronise) of
SparseGGNNChemModel (hidden 100, layer_timesteps [4], 4 edge types) and SparseGCNChemModel (hidden 100, 4 layers) on the 100 000-node batch,
bf16x3, in atomic mode.  Arms, alternating step by step:
  host        the packer's NumPy feed (the plug-in builds the graph and the map on the host in the step)
  cuda-list   every array a CUDA tensor but graph_nodes_list, which is .cpu()'d in the step (the best a GPU pipeline had before)
  cuda        every array a CUDA tensor
The card's name, power limit and maximum SM clock are read in the same run.

    python tools/readout_map_bench.py [--steps 20] [--warmup 5] [--json OUT]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.wide_hidden_bench import gpu_info  # noqa: E402

MAP_WORKLOADS = (("cfg2", "cfg2"), ("100k", "default_batch_100k_nodes"))
MAP_ARMS = ("host", "device")
STEP_ARMS = ("host", "cuda-list", "cuda")


def wall_ms(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.current_stream().synchronize()
    return (time.perf_counter() - t0) * 1e3


def alternate(fns, steps, warmup):
    """Median wall time of each of `fns` (name -> callable), called in turn `warmup + steps` times."""
    per = {a: [] for a in fns}
    for i in range(warmup + steps):
        for a, fn in fns.items():
            t = wall_ms(fn)
            if i >= warmup:
                per[a].append(t)
    return {a: round(statistics.median(v), 4) for a, v in per.items()}


def same_map(a, b):
    return all(np.array_equal(a[k], b[k]) if a[k] is not None and b[k] is not None else a[k] is b[k]
               for k in ("graph_of", "start", "perm", "node_mask")) and a["grouped"] == b["grouped"]


def map_row(tag, name, shuffled, steps, warmup):
    import torch
    from gated_graph_neural_network_samples_b200 import workloads
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    wl = workloads.build(name)
    gnl = np.asarray(wl["graph_nodes_list"], np.int32)
    if shuffled:
        gnl = np.random.default_rng(0).permutation(gnl).astype(np.int32)
    G = int(wl["num_graphs"])
    dl = torch.from_numpy(gnl).cuda()   # the caller's GPU-resident list
    engines = {a: PropagationEngine(wl["engine_params"], wl["num_edge_types"], precision="bf16x3") for a in MAP_ARMS}
    fns = {"host": lambda: engines["host"].readout_set_graphs(G, graph_nodes_list=dl.cpu()),
           "device": lambda: engines["device"].readout_set_graphs(G, graph_nodes_list=dl)}
    ms = alternate(fns, steps, warmup)
    return {"rows": "map", "workload": tag, "list": "shuffled" if shuffled else "grouped", "V": int(gnl.shape[0]), "G": G, "ms": ms,
            "same_map": same_map(engines["host"].readout_map(), engines["device"].readout_map())}


def _cuda_feed(feed):
    """The feed with every array a CUDA tensor of its dtype (the GGNN's int32 lists as [E, 2])."""
    import torch
    out = {}
    for k, v in feed.items():
        if not isinstance(v, np.ndarray):
            out[k] = v
        else:
            a = np.ascontiguousarray(v)
            out[k] = torch.from_numpy(a.reshape(-1, 2) if k.startswith("adjacency_e") else a).cuda()
    return out


def step_row(model_name, steps, warmup, tmp):
    import torch
    from gated_graph_neural_network_samples_b200 import synthetic
    mols = synthetic.make_molecules(5500, seed=0, num_bond_types=4)
    if model_name == "ggnn":
        from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel as M
        cfg = dict(hidden_size=100, layer_timesteps=[4], batch_size=100000, random_seed=3)
    else:
        from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel as M
        cfg = dict(hidden_size=100, num_timesteps=4, batch_size=100000, random_seed=3)
    m = M({"--log_dir": tmp, "--precision": "bf16x3", "--train_data": mols, "--valid_data": mols[:10], "--config": cfg})
    m.make_train_step()
    feed = dict(next(iter(m.make_minibatch_iterator(m.train_data, True))))
    feed.pop("_prepared_graph", None)
    for k in ("graph_state_keep_prob", "edge_weight_dropout_keep_prob", "out_layer_dropout_keep_prob"):
        if k in m.placeholders:
            feed[m.placeholders[k]] = 1.0
    feeds = {"host": feed, "cuda": _cuda_feed(feed)}

    def step(arm):
        f = dict(feeds["host" if arm == "host" else "cuda"])
        if arm == "cuda-list":
            f["graph_nodes_list"] = f["graph_nodes_list"].cpu()
        loss = m.forward_batch(f)[0]
        m.train_step(loss)

    ms = alternate({a: (lambda a=a: step(a)) for a in STEP_ARMS}, steps, warmup)
    return {"rows": "step", "model": model_name, "V": int(feed["initial_node_representation"].shape[0]), "G": int(feed["num_graphs"]),
            "ms": ms}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import tempfile
    import torch
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    card = gpu_info()
    print("card: %s" % card)
    rows = []
    for tag, name in MAP_WORKLOADS:
        for shuffled in (False, True):
            rows.append(map_row(tag, name, shuffled, args.steps, args.warmup))
            print(json.dumps(rows[-1]))
    with tempfile.TemporaryDirectory() as tmp:
        for model_name in ("ggnn", "gcn"):
            rows.append(step_row(model_name, args.steps, args.warmup, tmp))
            print(json.dumps(rows[-1]))
    print("\n| rows | workload | V | host ms | device ms |")
    print("|---|---|---|---|---|")
    for r in rows:
        if r["rows"] == "map":
            print("| map | %s %s | %d | %.3f | %.3f |" % (r["workload"], r["list"], r["V"], r["ms"]["host"], r["ms"]["device"]))
    print("\n| step | V | host feed ms | CUDA feed, list .cpu() ms | all-CUDA feed ms |")
    print("|---|---|---|---|---|")
    for r in rows:
        if r["rows"] == "step":
            print("| %s | %d | %.2f | %.2f | %.2f |" % (r["model"], r["V"], r["ms"]["host"], r["ms"]["cuda-list"], r["ms"]["cuda"]))
    for r in rows:
        r["card"] = card
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
