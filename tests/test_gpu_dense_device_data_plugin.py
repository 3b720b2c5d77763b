"""GPU: ``--device-data`` in DenseGGNNChemModel, whose batches are bucketed by graph size.

The plug-in trains two epochs from one seed under ``torch.use_deterministic_algorithms(True)``, once with batches packed on the host
(``pack_dense_batch``, the ``[b, T, v, v]`` matrix) and once with batches assembled on the device from a dense dataset.  The runs use state,
edge-weight and out-layer dropout, two tasks with ``task_sample_ratios``, the fused readout (hidden 100, bf16x3) and the torch readout
(hidden 30, zero-padded to 32).  Both give the same per-epoch losses and the same checkpoint, Adam slots included, bit for bit.  A
checkpoint written without the option restores into a model with it."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_CHILD = r"""
import json, sys
import numpy as np
import torch
torch.use_deterministic_algorithms(True)
from gated_graph_neural_network_samples_b200 import synthetic
from gated_graph_neural_network_samples_b200.chem_dense import DenseGGNNChemModel
cfg, out_dir, ckpt, device_data = json.loads(sys.argv[1]), sys.argv[2], sys.argv[3], sys.argv[4] == "1"
mols = synthetic.make_molecules(160, seed=11)
rng = np.random.default_rng(12)
for m in mols:                                # two tasks
    m["targets"] = [m["targets"][0], [float(rng.normal())]]
args = {"--log_dir": out_dir, "--train_data": mols[:128], "--valid_data": mols[128:], "--precision": cfg.pop("precision", "fp32"),
        "--config": dict(cfg, task_ids=[0, 1], task_sample_ratios={"1": 0.5}, learning_rate=0.01, num_epochs=2, random_seed=3)}
if device_data:
    args["--device-data"] = True
m = DenseGGNNChemModel(args)
losses = []
for ep in range(2):
    losses.append(float(m.run_epoch("train%d" % ep, m.train_data, True)[0]))
    losses.append(float(m.run_epoch("valid%d" % ep, m.valid_data, False)[0]))
m.save_progress(ckpt, 2, 0)
if device_data:                               # a checkpoint of the host-packed run restores into a device-data model
    m2 = DenseGGNNChemModel(args)
    assert m2.restore_progress(sys.argv[5]) == (2, 0)
print("LOSSES " + json.dumps(losses))
"""

TRAIN = {"batch_size": 4, "num_timesteps": 3, "graph_state_dropout_keep_prob": 0.9, "out_layer_dropout_keep_prob": 0.9}
CASES = {
    "dense-bf16x3-D100": dict(TRAIN, hidden_size=100, precision="bf16x3"),
    "dense-padded-D30-torch-readout": dict(TRAIN, hidden_size=30),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_dense_device_data_trains_bit_for_bit_like_host_packing(name, tmp_path):
    cfg = CASES[name]
    runs = []
    for device_data in (0, 1):
        ckpt = str(tmp_path / ("run%d.pickle" % device_data))
        env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8", PYTHONPATH=REPO)
        res = subprocess.run([sys.executable, "-c", _CHILD, json.dumps(cfg), str(tmp_path / ("log%d" % device_data)), ckpt, str(device_data),
                              str(tmp_path / "run0.pickle")], env=env, cwd=REPO, capture_output=True, text=True, timeout=900)
        assert res.returncode == 0, res.stderr[-3000:]
        losses = json.loads(next(l for l in res.stdout.splitlines() if l.startswith("LOSSES "))[7:])
        runs.append((losses, pickle.load(open(ckpt, "rb"))))
    (la, ca), (lb, cb) = runs
    assert all(np.isfinite(la))
    assert la == lb, (la, lb)
    assert ca["params"] == cb["params"]
    wa, wb = ca["weights"], cb["weights"]
    assert sorted(wa) == sorted(wb)
    assert any(k.endswith("/Adam:0") for k in wa) and any(k.endswith("/Adam_1:0") for k in wa)
    for k in wa:
        assert np.array_equal(np.asarray(wa[k]), np.asarray(wb[k])), k
