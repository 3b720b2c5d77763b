#!/usr/bin/env python
"""Timings of the sparse GCN above hidden 128: the fp32 CUDA-core kernel against the streaming wgmma plan (GCNEngine(wide_hidden=True),
SparseGCNChemModel --gcn-wide-hidden) on one GPU.

    python tools/gcn_wide_bench.py [--hidden 256 384 512] [--steps 30] [--warmup 5] [--rounds 3]

Workloads: 256 synthetic molecules in one batch, and one batch at the plug-in's default 100 000-node budget (5 500 molecules); four
layers, no bias (the reference's defaults but the width).  Arms per hidden size:

* 256: precision bf16x3 without wide_hidden (the fp32 kernel, as before the option) against bf16x3 with it (the streaming plan);
* 384, 512 (refused without the option): precision fp32 with wide_hidden (the fp32 kernel) against bf16x3 with it (the streaming plan).

Per arm: ``forward`` (ggnn_forward, graph and weights resident), ``forward_backward`` (forward with saved states + ggnn_gcn_backward of
every weight and d h0, fp32 backward GEMMs in both arms), ``train_step`` (the plug-in's forward_batch + train_step on a prepared graph:
upload, forward, fused readout, loss, backward, clip, Adam).  CUDA events around every run, L2 flushed (256 MiB write, untimed) before
every run, ``--steps`` timed runs after ``--warmup``; the arms alternate, ``--rounds`` times, and the median of the rounds' medians is
reported.  The card's name, power limit and max SM clock are read in the same run.  Prints one JSON line.  Needs a CUDA device.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.gcn_bench import event_times, gpu_info   # noqa: E402

LAYERS = 4
WORKLOADS = {"gcn_256_molecules": 256, "gcn_default_batch_100k_nodes": 5500}


def arms(D):
    """(label, precision, wide_hidden) of the two arms at hidden D."""
    slow = ("fp32-kernel (bf16x3, no wide_hidden)", "bf16x3", False) if D <= 256 else ("fp32-kernel (fp32, wide_hidden)", "fp32", True)
    return [slow, ("stream (bf16x3, wide_hidden)", "bf16x3", True)]


class Arm:
    """A SparseGCNChemModel at hidden D with its first batch prepared for training, and the three timed calls."""

    def __init__(self, mols, D, precision, wide, log_dir):
        import torch
        from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
        args = {"--log_dir": log_dir, "--precision": precision, "--train_data": mols, "--valid_data": mols[:4],
                "--config": {"batch_size": 100000, "hidden_size": D, "num_timesteps": LAYERS, "gcn_use_bias": False, "random_seed": 0}}
        if wide:
            args["--gcn-wide-hidden"] = True
        self.m = m = SparseGCNChemModel(args)
        m.prepare_graphs_in_producer = False
        feed = next(iter(m.make_minibatch_iterator(m.train_data, False)))
        self.V = feed["initial_node_representation"].shape[0]
        self.nnz = feed["adjacency_list"].shape[0]
        self.eng = eng = m.engine
        self.g = eng.prepare_graph_gcn(self.V, feed["adjacency_list"], feed["adjacency_weights"], save_for_backward=True)
        self.g.for_training = True
        self.tfeed = dict(feed, _prepared_graph=self.g, out_layer_dropout_keep_prob=1.0)
        self.h0 = torch.from_numpy(feed["initial_node_representation"]).cuda()
        self.out = torch.empty_like(self.h0)
        self.d_out = torch.randn_like(self.h0)
        self.d_h0 = torch.empty_like(self.h0)
        self.grads = [{"kernel": torch.zeros(D, D, device="cuda")} for _ in range(LAYERS)]
        self.losses = []
        self.plan = None

    def resident(self):
        """Graph and weights on the engine for the forward / forward_backward timings (a train step re-adopts its prepared graph)."""
        self.eng.set_weights([k.detach().contiguous() for k in self.m.weights["edge_weights"]])
        self.eng.set_save_for_backward(True)
        self.eng.set_state_dropout(1.0, 0)
        self.eng.set_graph_prepared(self.g)
        self.plan = self.eng.plan

    def forward(self):
        self.eng.forward(self.h0, self.out)

    def forward_backward(self):
        self.eng.forward(self.h0, self.out)
        self.eng.backward(self.d_out, self.grads, d_h0=self.d_h0)

    def train_step(self):
        loss, _ = self.m.forward_batch(self.tfeed)
        self.m.train_step(loss)
        self.m._prepared_pool.clear()
        self.losses.append(loss.detach())


def run_workload(n_mols, widths, args, flush):
    import torch
    from gated_graph_neural_network_samples_b200 import synthetic
    mols = synthetic.make_molecules(n_mols, seed=0)
    out = {}
    for D in widths:
        with tempfile.TemporaryDirectory() as log_dir:
            built = [(label, Arm(mols, D, prec, wide, log_dir)) for label, prec, wide in arms(D)]
        rounds = {label: {"forward": [], "forward_backward": [], "train_step": []} for label, _ in built}
        for r in range(args.rounds):
            for label, a in (built if r % 2 == 0 else built[::-1]):   # alternate the arms' order from round to round
                a.resident()
                for what in ("forward", "forward_backward"):
                    fn = getattr(a, what)
                    for _ in range(args.warmup):
                        fn()
                    rounds[label][what].append(event_times(fn, args.steps, flush)["median_ms"])
                a.eng.sync_check()
                for _ in range(args.warmup):
                    a.train_step()
                rounds[label]["train_step"].append(event_times(a.train_step, args.steps, flush)["median_ms"])
                a.eng.sync_check()
        torch.cuda.synchronize()
        res = {}
        for label, a in built:
            assert all(bool(torch.isfinite(x)) for x in a.losses), "non-finite training loss"
            res[label] = {"plan": a.plan, "V": a.V, "nnz": a.nnz,
                          **{what: {"median_of_round_medians_ms": statistics.median(v), "round_medians_ms": v} for what, v in rounds[label].items()}}
            res[label]["forward_node_updates_per_s"] = a.V * LAYERS / (res[label]["forward"]["median_of_round_medians_ms"] * 1e-3)
            # the layer GEMMs alone, 2 V D^2 per layer: what the forward's FLOP rate is counted on
            res[label]["forward_gemm_tflops"] = 2.0 * a.V * D * D * LAYERS / (res[label]["forward"]["median_of_round_medians_ms"] * 1e-3) / 1e12
            a.eng.close()
        out["hidden_%d" % D] = res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hidden", type=int, nargs="+", default=[256, 384, 512])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    args = ap.parse_args()
    if any(D <= 128 or D > 512 or D % 4 for D in args.hidden):
        raise SystemExit("--hidden: multiples of 4 in 132 .. 512")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("gcn_wide_bench.py needs a CUDA device (the GCN engine has no CPU path)")
    torch.cuda.set_device(0)
    flush_buf = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    line = {"metric": "sparse GCN above hidden 128: fp32 kernel vs streaming wgmma plan, median ms", "gpu": gpu_info(),
            "model": {"num_timesteps": LAYERS, "gcn_use_bias": False, "backward_precision": "fp32"},
            "method": {"steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "l2_flushed": True},
            "workloads": {name: run_workload(WORKLOADS[name], args.hidden, args, lambda: flush_buf.fill_(1)) for name in args.workloads}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
