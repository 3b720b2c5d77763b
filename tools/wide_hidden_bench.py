"""Timings of the GGNN engine at hidden 256, 384 and 512 on bf16x3 and fp32: BASELINE config 4's model and molecules (1024 molecules, 8
edge types, layer_timesteps [2, 2, 2, 2], a residual input into layer 2) with only the hidden size changed.

Per (hidden, precision): the propagation forward, forward + backward (save_for_backward, every weight gradient and d h0), and one
SparseGGNNChemModel training step (forward_batch on the whole batch, loss.backward(), clip + Adam).  Each is timed with CUDA events, after
a warm-up, as the median of --steps runs, with the 50 MB L2 flushed before every run and without.  The card's name, power limit and
maximum SM clock are read in the same run (an nvidia-smi query).  At hidden 256 on bf16x3 the flushed forward is the number
``bench.py --config cfg4`` reports as ms_per_step.

    python tools/wide_hidden_bench.py [--steps 30] [--warmup 5] [--json OUT]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WIDTHS = (256, 384, 512)
PRECISIONS = ("bf16x3", "fp32")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


class Timer:
    def __init__(self, steps, warmup):
        import torch
        self.steps, self.warmup = steps, warmup
        self.flush_buf = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")

    def median_ms(self, fn, flush):
        """Median over self.steps runs of fn (device time between two events around it); flush: L2 flushed before every run."""
        import torch
        for _ in range(self.warmup):
            fn()
        torch.cuda.synchronize()
        times = []
        for _ in range(self.steps):
            if flush:
                self.flush_buf.fill_(1)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b))
        return statistics.median(times)


def cfg4_at(D):
    """cfg4's molecules and model at hidden D: (params, T, molecules, packed batch)."""
    from gated_graph_neural_network_samples_b200 import packing, synthetic, workloads
    cfg = workloads.CONFIGS["cfg4"]
    T = cfg["edge_types"]
    params = dict(cfg["params"], hidden_size=D)
    mols = synthetic.make_molecules(cfg["molecules"], seed=0, num_bond_types=T)
    b = packing.pack_sparse_batch(packing.process_raw_graphs_sparse(mols), D, T)
    return params, T, mols, b


def engine_rows(timer, D, precision):
    import torch
    from gated_graph_neural_network_samples_b200 import workloads
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    params, T, _, b = cfg4_at(D)
    w = workloads.init_weights(params, T, seed=1)
    dev_w = [{k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in lw.items()} for lw in w]
    eng = PropagationEngine(params, T, precision=precision)
    eng.set_weights(dev_w)
    eng.set_graph_sparse(b["adjacency_lists"], b["num_incoming_edges_per_type"])
    h0 = torch.from_numpy(b["initial_node_representation"]).cuda()
    out = torch.empty_like(h0)
    rows = {"plan": eng.plan, "V": int(h0.shape[0])}
    for flush in (True, False):
        rows["forward_ms" + ("" if flush else "_hot_l2")] = timer.median_ms(lambda: eng.forward(h0, out), flush)
    eng.set_save_for_backward(True)
    eng.set_graph_sparse(b["adjacency_lists"], b["num_incoming_edges_per_type"])
    grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in dev_w]
    d_out = torch.randn_like(h0)
    d_h0 = torch.empty_like(h0)

    def fwd_bwd():
        eng.forward(h0, out)
        eng.backward(d_out, grads, d_h0)

    for flush in (True, False):
        rows["fwd_bwd_ms" + ("" if flush else "_hot_l2")] = timer.median_ms(fwd_bwd, flush)
    eng.sync_check()
    return rows


def train_step_rows(timer, D, precision, log_dir):
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    params, _, mols, _ = cfg4_at(D)
    cfg = {k: params[k] for k in ("hidden_size", "layer_timesteps", "residual_connections", "use_edge_bias", "use_edge_msg_avg_aggregation",
                                  "graph_rnn_cell", "graph_rnn_activation")}
    cfg.update(batch_size=10 ** 6, num_epochs=1)
    m = SparseGGNNChemModel({"--log_dir": log_dir, "--precision": precision, "--train_data": mols, "--valid_data": mols[:8], "--config": cfg})
    feed = next(iter(m.make_minibatch_iterator(m.train_data, True)))
    feed[m.placeholders["out_layer_dropout_keep_prob"]] = m.params["out_layer_dropout_keep_prob"]
    assert feed[m.placeholders["num_graphs"]] == len(mols), "the whole batch in one step"

    def step():
        loss, _ = m.forward_batch(feed)
        m.train_step(loss)

    rows = {}
    for flush in (True, False):
        rows["train_step_ms" + ("" if flush else "_hot_l2")] = timer.median_ms(step, flush)
    m.engine.sync_check()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed runs per number (the median is reported; at least 20)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    args = ap.parse_args()
    import tempfile
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("wide_hidden_bench.py needs a CUDA device")
    steps = max(args.steps, 20)
    timer = Timer(steps, args.warmup)
    result = {"gpu": gpu_info(), "steps": steps, "warmup": args.warmup, "rows": []}
    print("GPU (name, power limit, max SM clock): %s" % result["gpu"])
    print("%-7s %-7s %10s %10s %10s %10s %10s %10s   plan" % ("hidden", "prec", "fwd", "fwd hot", "fwd+bwd", "f+b hot", "train", "train hot"))
    with tempfile.TemporaryDirectory() as log_dir:
        for D in WIDTHS:
            for precision in PRECISIONS:
                r = dict(hidden=D, precision=precision)
                r.update(engine_rows(timer, D, precision))
                r.update(train_step_rows(timer, D, precision, log_dir))
                result["rows"].append(r)
                print("%-7d %-7s %10.3f %10.3f %10.3f %10.3f %10.3f %10.3f   %s" % (
                    D, precision, r["forward_ms"], r["forward_ms_hot_l2"], r["fwd_bwd_ms"], r["fwd_bwd_ms_hot_l2"], r["train_step_ms"],
                    r["train_step_ms_hot_l2"], r["plan"]), flush=True)
    print(json.dumps(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
