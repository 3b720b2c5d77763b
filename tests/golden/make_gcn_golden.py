#!/usr/bin/env python
"""GCN fixtures computed by the REFERENCE'S OWN code (run in a checkout next to the reference sources; only the committed .npz travel).

``chem_tensorflow_gcn.py`` is imported unmodified with ``tests/golden/tf_shim.py`` registered as ``tensorflow``.  The shim gains, in this
script only, the three pieces of the TF-1 API that the GCN model uses and the GGNN models do not: ``tf.int64``, ``tf.SparseTensor`` and
``tf.sparse_tensor_dense_matmul``.  The sparse product adds ``w * H[j]`` into row ``i`` with ``np.add.at`` in list order, the serial order of
TF 1.3's CPU functor as we recall it from TF's source.  Writes only new files; every other fixture is left untouched.

    packing_gcn.npz          batches of the reference's process_raw_graphs + make_minibatch_iterator (chem_tensorflow_gcn.py:96-199)
    refgraph_gcn_<case>.npz  the reference's make_model (both hooks, gated_regression, masked loss and MAE) evaluated in float64 on one of
                             those batches: inputs, the weights the model created (float32-rounded), final node states, readout, loss, MAE

Usage:  python tests/golden/make_gcn_golden.py [path to the reference sources]
"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import tf_shim  # noqa: E402
from gated_graph_neural_network_samples_b200 import synthetic  # noqa: E402


def extend_shim():
    class SparseTensor:
        def __init__(self, indices, values, dense_shape):
            self.indices, self.values, self.dense_shape = indices, values, dense_shape

    def sparse_tensor_dense_matmul(sp, dense):
        def f(idx, vals, h, shape):
            idx = np.asarray(idx, np.int64).reshape(-1, 2)
            out = np.zeros((int(shape[0]), h.shape[1]), np.float64)
            np.add.at(out, idx[:, 0], np.asarray(vals, np.float64)[:, None] * h[idx[:, 1]])   # list order
            return out
        return tf_shim.Node(f, sp.indices, sp.values, dense, tf_shim.Node(lambda *s: np.array(s), *sp.dense_shape))

    tf_shim.int64 = "int64"
    tf_shim.SparseTensor = SparseTensor
    tf_shim.sparse_tensor_dense_matmul = sparse_tensor_dense_matmul


def import_reference(ref_dir):
    extend_shim()
    sys.modules["tensorflow"] = tf_shim
    tf_shim.register_submodules(sys.modules)
    d = types.ModuleType("docopt")
    d.docopt = lambda *a, **k: {}
    sys.modules["docopt"] = d
    sys.path.insert(0, ref_dir)
    import chem_tensorflow_gcn as ref_gcn  # noqa
    return ref_gcn


def new_model(ref_gcn, cfg, batch_size):
    m = object.__new__(ref_gcn.SparseGCNChemModel)
    m.params = dict(ref_gcn.SparseGCNChemModel.default_params())
    m.params.update({"task_ids": [0], "batch_size": batch_size, "use_graph": True})
    m.params.update(cfg)
    m.annotation_size = 0
    return m


def packing_fixture(ref_gcn, mols):
    m = new_model(ref_gcn, {"hidden_size": 8}, 200)
    m.annotation_size = len(mols[0]["node_features"][0])
    keys = ["initial_node_representation", "adjacency_list", "adjacency_weights", "graph_nodes_list", "target_values", "target_mask",
            "num_graphs", "graph_state_keep_prob"]
    m.placeholders = {k: k for k in keys}
    data = m.process_raw_graphs(mols, is_training_data=False)
    batches = list(m.make_minibatch_iterator(data, is_training=False))
    out = {"num_batches": np.int64(len(batches))}
    for bi, b in enumerate(batches):
        out["b%d_init" % bi] = np.asarray(b["initial_node_representation"], np.float32)
        out["b%d_adj" % bi] = np.asarray(b["adjacency_list"], np.int64).reshape(-1, 2)
        out["b%d_w" % bi] = np.asarray(b["adjacency_weights"], np.float64)
        out["b%d_gnl" % bi] = np.asarray(b["graph_nodes_list"], np.int32)
        out["b%d_targets" % bi] = np.asarray(b["target_values"], np.float32)
        out["b%d_mask" % bi] = np.asarray(b["target_mask"], np.float32)
        out["b%d_num_graphs" % bi] = np.int64(b["num_graphs"])
        out["b%d_keep" % bi] = np.float64(b["graph_state_keep_prob"])
    np.savez_compressed(os.path.join(HERE, "packing_gcn.npz"), **out)
    print("packing_gcn: %d batches" % len(batches))


def refgraph_case(ref_gcn, name, cfg, mols, seed):
    m = new_model(ref_gcn, cfg, 100000)
    m.annotation_size = len(mols[0]["node_features"][0])
    m.placeholders, m.weights, m.ops = {}, {}, {}
    np.random.seed(seed)
    m.make_model()                                                # chem_tensorflow.py:133-170 -> gcn:42-57, 59-82, 84-93, unmodified
    f32 = lambda a: np.asarray(a, np.float64).astype(np.float32).astype(np.float64)
    L = cfg["num_timesteps"]
    rng = np.random.RandomState(seed + 1)
    for v in m.weights["edge_weights"]:
        v.value = f32(v.value)
    if cfg.get("gcn_use_bias"):
        for v in m.weights["edge_biases"]:                        # the reference initialises zeros: perturb so the bias path is exercised
            v.value = f32(rng.uniform(-0.2, 0.2, v.value.shape))
    gate, trans = m.weights["regression_gate_task0"], m.weights["regression_transform_task0"]
    for mlp in (gate, trans):
        mlp.params["weights"][0].value = f32(mlp.params["weights"][0].value)
        mlp.params["biases"][0].value = f32(rng.uniform(-0.2, 0.2, mlp.params["biases"][0].value.shape))
    readout = m.gated_regression(m.ops["final_node_representations"], gate, trans)   # the node the loss is built on (gcn:84-93)
    data = m.process_raw_graphs(mols, is_training_data=False)
    feed = next(iter(m.make_minibatch_iterator(data, is_training=False)))
    h0 = np.asarray(feed[m.placeholders["initial_node_representation"]], np.float64)
    h0 = f32(h0 + np.random.RandomState(seed + 2).normal(0, 0.3, h0.shape))   # every column live, exactly representable in fp32
    feed[m.placeholders["initial_node_representation"]] = h0
    feed[m.placeholders["out_layer_dropout_keep_prob"]] = 1.0
    final, ro, loss, mae = tf_shim.evaluate([m.ops["final_node_representations"], readout, m.ops["loss"], m.ops["accuracy_task0"]], feed)
    out = {"params_json": np.asarray(json.dumps(cfg)), "h0": h0.astype(np.float32), "final": final, "readout": ro,
           "loss": np.float64(loss), "accuracy": np.float64(mae),
           "adjacency_list": np.asarray(feed[m.placeholders["adjacency_list"]], np.int64).reshape(-1, 2),
           "adjacency_weights": np.asarray(feed[m.placeholders["adjacency_weights"]], np.float64),
           "adjacency_weights_f32": np.asarray(feed[m.placeholders["adjacency_weights"]], np.float32),
           "graph_nodes_list": np.asarray(feed[m.placeholders["graph_nodes_list"]], np.int32),
           "num_graphs": np.int64(feed[m.placeholders["num_graphs"]]),
           "target_values": np.asarray(feed[m.placeholders["target_values"]], np.float64),
           "target_mask": np.asarray(feed[m.placeholders["target_mask"]], np.float64)}
    for l in range(L):
        out["w%d_kernel" % l] = m.weights["edge_weights"][l].value.astype(np.float32)
        if cfg.get("gcn_use_bias"):
            out["w%d_bias" % l] = m.weights["edge_biases"][l].value.astype(np.float32)
    for k, mlp in (("gate", gate), ("trans", trans)):
        out["ro_w_" + k] = mlp.params["weights"][0].value.astype(np.float32)
        out["ro_b_" + k] = mlp.params["biases"][0].value.astype(np.float32)
    np.savez_compressed(os.path.join(HERE, "refgraph_gcn_%s.npz" % name), **out)
    print(name, "V=%d nnz=%d final max %.3f loss %.5f mae %.5f" % (h0.shape[0], out["adjacency_list"].shape[0], np.abs(final).max(), loss, mae))


def main():
    ref_gcn = import_reference(sys.argv[1] if len(sys.argv) > 1 else os.environ.get("GGNN_REFERENCE_DIR", "../reference"))
    packing_fixture(ref_gcn, synthetic.make_molecules(40, seed=123))
    mols = synthetic.make_molecules(12, seed=321)
    mols[4]["targets"][0][0] = None                              # one unlabeled graph: the loss mask is exercised
    refgraph_case(ref_gcn, "h12_l3", {"hidden_size": 12, "num_timesteps": 3, "gcn_use_bias": False}, mols, 31)
    refgraph_case(ref_gcn, "h100_l4_bias", {"hidden_size": 100, "num_timesteps": 4, "gcn_use_bias": True}, synthetic.make_molecules(24, seed=77), 32)
    refgraph_case(ref_gcn, "h12_l1", {"hidden_size": 12, "num_timesteps": 1, "gcn_use_bias": True}, mols, 33)
    print("GCN fixtures written to", HERE)


if __name__ == "__main__":
    main()
