"""Host-packed batches against device-resident datasets (``--device-data``) in the three plug-ins, in one process.

    python tools/device_data_bench.py [--molecules N] [--reps R] [--models ggnn,gcn,dense] [--out FILE]

For SparseGGNNChemModel and SparseGCNChemModel (bf16x3, the reference's default shapes), at a batch of about 256 molecules and at the
reference's 100 000-node batch, and for DenseGGNNChemModel (bf16x3) at BASELINE cfg3's 64-graph batch and the reference's default of 256
graphs per bucketed batch, the two paths are measured alternately, R times each, and the medians printed as one JSON line:
  producer_ms_per_batch  host time of the batch producer (make_minibatch_iterator) per batch, the dataset upload excluded (done once before)
  step_ms                one training step on the consumer thread (forward_batch + train_step) between CUDA events
  instances_per_s        run_epoch (training) over the whole synthetic set, the producer thread overlapping the GPU as in training
The GPU's name and power limit are printed beside the numbers.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as ex:   # the numbers are still printed; the card is then named by torch only
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown (%s)" % ex}


def make_model(kind: str, mols, batch_size: int, device_data: bool):
    from gated_graph_neural_network_samples_b200.chem_dense import DenseGGNNChemModel
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    model = {"ggnn": SparseGGNNChemModel, "gcn": SparseGCNChemModel, "dense": DenseGGNNChemModel}[kind]
    args = {"--log_dir": "/tmp/device_data_bench", "--train_data": mols, "--valid_data": mols[:64], "--precision": "bf16x3",
            "--config": {"batch_size": batch_size, "random_seed": 0}}
    if device_data:
        args["--device-data"] = True
    return model(args)


def producer_ms(m) -> float:
    """Host time per batch of one pass of the batch producer (no GPU work is waited for)."""
    t0 = time.perf_counter()
    n = sum(1 for _ in m.make_minibatch_iterator(m.train_data, True))
    return (time.perf_counter() - t0) * 1e3 / max(n, 1)


def step_ms(m, steps: int = 8) -> float:
    """Median of `steps` training steps (forward_batch + train_step) between CUDA events, feeds produced beforehand."""
    import torch
    feeds = []
    for f in m.make_minibatch_iterator(m.train_data, True):
        f['out_layer_dropout_keep_prob'] = m.params['out_layer_dropout_keep_prob']
        feeds.append(f)
        if len(feeds) == steps:
            break
    times = []
    for f in feeds:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        loss, _ = m.forward_batch(f)
        m.train_step(loss)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--molecules", type=int, default=60000, help="synthetic training molecules (~18 nodes each)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--models", default="ggnn,gcn,dense", help="comma-separated subset of ggnn, gcn, dense")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("device_data_bench needs a CUDA device")
    from gated_graph_neural_network_samples_b200 import synthetic
    mols = synthetic.make_molecules(a.molecules, seed=0)
    mean_nodes = float(np.mean([len(m["node_features"]) for m in mols]))
    result = {"bench": "device_data", "molecules": a.molecules, **gpu_info(), "rows": []}
    sizes = {"ggnn": (("256 molecules", int(256 * mean_nodes)), ("100000 nodes", 100000)),   # batch_size: a node budget
             "gcn": (("256 molecules", int(256 * mean_nodes)), ("100000 nodes", 100000)),
             "dense": (("64 graphs", 64), ("256 graphs", 256))}                            # batch_size: graphs per bucketed batch
    for kind in a.models.split(","):
        for label, batch_size in sizes[kind]:
            models = {dd: make_model(kind, mols, batch_size, dd) for dd in (False, True)}
            for m in models.values():   # warm-up: flattening, the dataset upload, kernel first launches
                m.run_epoch("warm-up", m.train_data, True)
            samples = {dd: {"producer_ms_per_batch": [], "step_ms": [], "instances_per_s": []} for dd in models}
            for _ in range(a.reps):
                for dd, m in models.items():   # alternating
                    samples[dd]["producer_ms_per_batch"].append(producer_ms(m))
                    samples[dd]["step_ms"].append(step_ms(m))
                    samples[dd]["instances_per_s"].append(m.run_epoch("bench", m.train_data, True)[3])
            for dd in models:
                result["rows"].append({"model": kind, "batch": label, "batch_size": batch_size,
                                       "path": "device-data" if dd else "host-packed",
                                       **{k: round(statistics.median(v), 3) for k, v in samples[dd].items()}})
            del models
            torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
