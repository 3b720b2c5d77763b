"""Prediction throughput of the sparse GGNN model: ``ChemModel.predict`` (host-packed and ``device_data=True``) against the loop a user would
write without it -- ``forward_batch`` under ``torch.no_grad()`` with the molecules' targets as dummy targets, reading ``model.output`` after
each batch -- at two batch sizes and with 1 and 13 tasks, over synthetic QM9-like molecules.

Every arm is one whole pass over the molecule list (processing, batching, propagation, readout, the copy back), timed with CUDA events
around a call that ends in a device synchronise.  Every arm is run once untimed first (module loads, allocations, every batch shape), then
the arms are timed in rotation, ``--repeats`` times each, and the median pass is reported as molecules per second.  The GPU's name and power
limit are read in the same run.

    python tools/predict_bench.py [--molecules 60000] [--repeats 3] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# batch sizes of the sparse model are node budgets: ~256 molecules (QM9's mean of 18 atoms) and the reference's default of 100 000 nodes
BATCHES = {"256 mol": 256 * 18, "100k nodes": 100000}
TASK_COUNTS = (1, 13)


def gpu_info() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001 -- the name still comes from torch below
        return "power limit not read (%s)" % ex


def molecules(n, seed=0):
    from gated_graph_neural_network_samples_b200 import synthetic
    rng = np.random.default_rng(seed)
    mols = synthetic.make_molecules(n, seed=seed)
    for m in mols:
        m["targets"] = [[float(rng.normal())] for _ in range(13)]
    return mols


def make_model(mols, batch_size, tasks, log_dir):
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    return SparseGGNNChemModel({"--log_dir": log_dir, "--train_data": mols[:200], "--valid_data": mols[200:400], "--precision": "bf16x3",
                                "--config": {"batch_size": batch_size, "task_ids": list(range(tasks))}})


def dummy_target_loop(m, mols):
    """What predicting takes without ChemModel.predict: validation batches through forward_batch, model.output (the last task) per batch."""
    import torch
    outs = []
    data = m.process_raw_graphs(mols, False)
    with torch.no_grad():
        for feed in m.make_minibatch_iterator(data, False):
            feed[m.placeholders['out_layer_dropout_keep_prob']] = 1.0
            m.forward_batch(feed)
            outs.append(m.output)
    return torch.cat(outs).cpu().numpy()


def timed(fn):
    import torch
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--molecules", type=int, default=60000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("predict_bench measures the GPU: no CUDA device")
    info = "%s | %s" % (torch.cuda.get_device_name(0), gpu_info())
    print("GPU: %s" % info)
    mols = molecules(args.molecules)
    N = len(mols)
    log_dir = tempfile.mkdtemp(prefix="predict_bench_")
    arms = {}
    for bname, bs in BATCHES.items():
        for K in TASK_COUNTS:
            m = make_model(mols, bs, K, log_dir)
            arms[(bname, K, "predict host")] = lambda m=m: m.predict(mols)
            arms[(bname, K, "predict device_data")] = lambda m=m: m.predict(mols, device_data=True)
            arms[(bname, K, "forward_batch loop")] = lambda m=m: dummy_target_loop(m, mols)
    for key, fn in arms.items():   # warm-up: every shape, every module
        print("warm-up %s: %.1f s" % (key, timed(fn)), flush=True)
    times = {k: [] for k in arms}
    for r in range(args.repeats):
        for key, fn in arms.items():
            times[key].append(timed(fn))
    rows = []
    print("\n%-11s %3s  %-20s %12s %10s" % ("batch", "K", "arm", "molecules/s", "median s"))
    for key in arms:
        med = float(np.median(times[key]))
        rows.append({"batch": key[0], "tasks": key[1], "arm": key[2], "molecules_per_s": N / med, "median_s": med, "times_s": times[key]})
        print("%-11s %3d  %-20s %12.0f %10.3f" % (key[0], key[1], key[2], N / med, med))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"gpu": info, "molecules": N, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
