"""CPU: the host-side logic of prediction -- ChemModel.predict, evaluate_one_batch and example_evaluation of the three plug-ins, the
target-free packing paths and the target-free dataset -- driven end to end with the stand-in engines of the plug-in tests (propagation
answered by the oracle), and the new ABI symbols."""
import json
import os
import re

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import _lib, chem_dense, chem_gcn, chem_sparse, packing, synthetic
from tests.test_chem_gcn_cpu import StandInGCNEngine, StandInPropagation as StandInGCNPropagation
from tests.test_chem_model_cpu import StandInEngine, StandInPropagation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TASKS = [0, 2, 3]


@pytest.fixture
def stand_in(monkeypatch):
    for mod in (chem_sparse, chem_dense):
        monkeypatch.setattr(mod, "PropagationEngine", StandInEngine)
        monkeypatch.setattr(mod, "_propagation_function", lambda: StandInPropagation)
    monkeypatch.setattr(chem_gcn, "GCNEngine", StandInGCNEngine)
    monkeypatch.setattr(chem_gcn, "_propagation_function", lambda: StandInGCNPropagation)


def molecules(n, seed):
    """Synthetic molecules with four targets each (QM9 files carry 13)."""
    rng = np.random.default_rng(seed)
    mols = synthetic.make_molecules(n, seed=seed)
    for m in mols:
        m["targets"] = [[float(rng.normal())] for _ in range(4)]
    return mols


PLUGINS = {
    "sparse": (chem_sparse.SparseGGNNChemModel, {"batch_size": 120, "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}}),
    "gcn": (chem_gcn.SparseGCNChemModel, {"batch_size": 120, "num_timesteps": 2}),
    "dense": (chem_dense.DenseGGNNChemModel, {"batch_size": 3, "num_timesteps": 2}),
}


def make(name, tmp_path, mols, hidden=16, **extra):
    cls, cfg = PLUGINS[name]
    config = dict(cfg, hidden_size=hidden, task_ids=TASKS, num_epochs=1, learning_rate=0.01)
    args = {"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:24], "--valid_data": mols[24:], "--config": config}
    args.update(extra)
    return cls(args)


def validation_outputs(m, name, mols):
    """Every task's gated_regression after a validation forward_batch, [tasks, N] in the order of ``mols``."""
    import torch
    out = np.zeros((len(TASKS), len(mols)), np.float32)
    if name == "dense":
        batches = [(ids, packing.pack_dense_batch([mols[i] for i in ids], v, m.params["hidden_size"], m.num_edge_types, TASKS))
                   for v, ids in packing.bucket_batches(mols, m.params["batch_size"])]
    else:
        feeds, start = m.make_minibatch_iterator(m.process_raw_graphs(mols, False), False), 0
        batches = []
        for feed in feeds:
            batches.append((np.arange(start, start + feed["num_graphs"]), feed))
            start += feed["num_graphs"]
        assert start == len(mols)
    assert len(batches) >= 3
    for ids, feed in batches:
        feed = dict(feed, out_layer_dropout_keep_prob=1.0, graph_state_keep_prob=1.0, edge_weight_dropout_keep_prob=1.0)
        with torch.no_grad():
            m.forward_batch(feed)
            final = m.ops["final_node_representations"]
            for k, t in enumerate(TASKS):
                out[k, ids] = m.gated_regression(final, m.weights["regression_gate_task%i" % t].bind(1.0),
                                                 m.weights["regression_transform_task%i" % t].bind(1.0)).numpy()
    return out


@pytest.mark.parametrize("name", sorted(PLUGINS))
def test_predict_rows_follow_the_input_order_and_match_the_validation_forward(tmp_path, stand_in, name):
    mols = molecules(48, seed=3)
    m = make(name, tmp_path, mols)
    shuffled = [mols[i] for i in np.random.default_rng(0).permutation(len(mols))]
    got = m.predict(shuffled)
    assert got.shape == (len(TASKS), len(mols)) and got.dtype == np.float32
    np.testing.assert_allclose(got, validation_outputs(m, name, shuffled), rtol=1e-5, atol=1e-6)
    # target-free graphs are accepted and predict the same
    bare = [{k: v for k, v in g.items() if k != "targets"} for g in shuffled]
    np.testing.assert_array_equal(m.predict(bare), got)
    # another batch size cuts other batches: the columns still follow the input
    np.testing.assert_allclose(m.predict(shuffled, batch_size=60 if name != "dense" else 5), got, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("name", ["sparse", "gcn"])
def test_evaluate_one_batch_returns_the_last_task(tmp_path, stand_in, name, capsys):
    mols = molecules(40, seed=4)
    m = make(name, tmp_path, mols)
    got = m.evaluate_one_batch(m.process_raw_graphs(mols, False))
    np.testing.assert_allclose(got, m.predict(mols)[-1], rtol=1e-5, atol=1e-6)
    assert capsys.readouterr().out.count("[") >= 3          # one printed array per batch, as the reference's loop prints them


def test_dense_evaluate_one_batch_builds_the_reference_default_mask(tmp_path, stand_in):
    mols = molecules(40, seed=5)
    m = make("dense", tmp_path, mols)
    rng = np.random.default_rng(1)
    ann = [rng.normal(size=(29, 5)).astype(np.float32), rng.normal(size=(7, 5)).astype(np.float32), rng.normal(size=(12, 5)).astype(np.float32)]
    adj = (rng.random((3, m.num_edge_types, 29, 29)) < 0.05).astype(np.float32)
    got = m.evaluate_one_batch([a.tolist() for a in ann], adj)
    mask = np.zeros((3, 29), np.float32)
    mask[0, :29], mask[1, :7], mask[2, :12] = 1, 1, 1              # dense:232-235: 1 for each graph's rows, 0 up to the first graph's count
    np.testing.assert_array_equal(m.feed["node_mask"], mask)
    assert got.shape == (3,)
    np.testing.assert_array_equal(m.evaluate_one_batch([a.tolist() for a in ann], adj, mask), got)
    assert not np.allclose(m.evaluate_one_batch([a.tolist() for a in ann], adj, np.ones((3, 29), np.float32)), got)


def test_dense_evaluate_one_batch_returns_the_last_task(tmp_path, stand_in):
    mols = molecules(40, seed=6)
    m = make("dense", tmp_path, mols)
    v, ids = next(packing.bucket_batches(mols, 4))
    b = packing.pack_dense_batch([mols[i] for i in ids], v, m.annotation_size, m.num_edge_types, ())
    got = m.evaluate_one_batch(list(b["initial_node_representation"]), b["adjacency_matrix"], b["node_mask"])
    np.testing.assert_allclose(got, m.predict([mols[i] for i in ids], batch_size=4)[-1], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("name", ["sparse", "dense"])
def test_example_evaluation_prints_targets_then_predictions(tmp_path, stand_in, name, capsys):
    mols = molecules(40, seed=7)
    m = make(name, tmp_path, mols)
    path = tmp_path / "valid.json"
    path.write_text(json.dumps(mols[:12]))
    out = m.example_evaluation(str(path), n=10)
    assert out.shape == (10,)
    text = capsys.readouterr().out
    assert text.index(str(mols[0]["targets"])) < text.index(str(mols[9]["targets"])) < text.rindex("[")


@pytest.mark.parametrize("name", sorted(PLUGINS))
def test_a_restored_model_predicts_what_the_saved_one_did(tmp_path, stand_in, name):
    mols = molecules(48, seed=8)
    m = make(name, tmp_path, mols)
    m.run_epoch("train", m.train_data, True)
    path = str(tmp_path / "model.pickle")
    m.save_progress(path, 1, 1)
    m2 = make(name, tmp_path, mols, **{"--restore": path})
    np.testing.assert_array_equal(m2.predict(mols), m.predict(mols))


@pytest.mark.parametrize("name", sorted(PLUGINS))
def test_hidden_sizes_that_are_not_multiples_of_4_predict(tmp_path, stand_in, name):
    mols = molecules(40, seed=9)
    m = make(name, tmp_path, mols, hidden=18)
    np.testing.assert_allclose(m.predict(mols), validation_outputs(m, name, mols), rtol=1e-5, atol=1e-6)


def test_target_free_packing_and_labelled_packing_unchanged():
    mols = molecules(12, seed=10)
    bare = [{k: v for k, v in g.items() if k != "targets"} for g in mols]
    for proc, kw in ((packing.process_raw_graphs_sparse, {}), (packing.process_raw_graphs_gcn, {})):
        labelled, default = proc(mols, TASKS, **kw), proc(mols, TASKS, labels=True, **kw)
        for a, b in zip(labelled, default):
            assert a["labels"] == b["labels"] and len(a["labels"]) == len(TASKS)
        free = proc(bare, TASKS, labels=False, **kw)
        assert all(g["labels"] == [] for g in free)
    flat = packing.FlatSparseGraphs(packing.process_raw_graphs_sparse(bare, TASKS, labels=False), 4)
    b = flat.pack(np.arange(5), 16)
    assert b["target_values"].shape == (0, 5) and b["target_mask"].shape == (0, 5)
    d = packing.pack_dense_batch(bare[:3], 29, 16, 4, ())
    assert d["target_values"].shape == (0, 3)
    # the dense batches of a prediction: every graph exactly once, each bucket's graphs in input order, at most batch_size per batch
    seen = []
    for v, ids in packing.bucket_batches(bare, 2):
        assert 1 <= len(ids) <= 2 and list(ids) == sorted(ids)
        assert all(packing.DEFAULT_BUCKET_SIZES[packing.choose_bucket(bare[i]["graph"])] == v for i in ids)
        seen += list(ids)
    assert sorted(seen) == list(range(len(bare)))


def test_a_target_free_dataset_is_refused_for_a_training_batch():
    from gated_graph_neural_network_samples_b200.engine import DeviceDataset, GgnnError
    mols = [{k: v for k, v in g.items() if k != "targets"} for g in synthetic.make_molecules(10, seed=11)]
    flat = packing.FlatSparseGraphs(packing.process_raw_graphs_sparse(mols, [0], labels=False), 4)
    params = {"hidden_size": 16, "layer_timesteps": [1], "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh"}
    ds = DeviceDataset.host_only(params, 4, flat, for_training=True)
    assert ds.num_tasks == 0
    ds.prepare_batch(np.arange(10), save_for_backward=False)
    with pytest.raises(GgnnError, match="no targets") as ex:
        ds.prepare_batch(np.arange(10), save_for_backward=True)
    assert ex.value.code == -1   # GGNN_EINVAL
    labelled = DeviceDataset.host_only(params, 4, packing.FlatSparseGraphs(packing.process_raw_graphs_sparse(synthetic.make_molecules(10, seed=11)), 4))
    labelled.prepare_batch(np.arange(10), save_for_backward=True)


def test_the_prediction_calls_are_in_the_header_and_the_binding():
    header = open(os.path.join(ROOT, "include", "ggnn_b200.h")).read()
    declared = set(re.findall(r"\b(ggnn_\w+)\s*\(", header))
    for name in ("ggnn_readout_predict", "ggnn_dataset_batch_slots", "ggnn_run_sparse_host_predict", "ggnn_run_dense_host_predict"):
        assert name in declared and name in _lib.SYMBOLS, name
    assert _lib.SYMBOLS["ggnn_readout_predict"][1][4] is not None
