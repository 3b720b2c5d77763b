"""CPU: the host-side logic of the SparseGCNChemModel plug-in (chem_tensorflow_gcn.py) driven end to end with a STAND-IN engine whose
propagation is the fp32 torch restatement of the reference graph (tests/gcn_oracle.gcn_propagation_torch) with the engine's state-dropout
masks (oracle.state_dropout_mask): feeds, padding, readout, loss, training, checkpoints, data parallelism, and the flattened packer."""
import json
import os
import pickle
import socket

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import chem_gcn, packing, synthetic
from oracle import ggnn_oracle as O
from tests import gcn_oracle as G


class StandInGCNEngine:
    def __init__(self, hidden_size, num_layers, use_bias=False, device=0, precision="fp32"):
        self.D, self.L, self.use_bias = int(hidden_size), int(num_layers), bool(use_bias)
        self.drop = (1.0, 0)
        self.seen = []

    def set_save_for_backward(self, enable):
        pass

    def set_graph_gcn(self, num_nodes, adjacency_list, adjacency_weights):
        self.V = int(num_nodes)
        self.lst = np.asarray(adjacency_list, np.int64).reshape(-1, 2)
        self.w = np.asarray(adjacency_weights, np.float32)      # the engine's float32 feed, as the reference's placeholder casts it

    def set_state_dropout(self, keep, seed=0):
        self.drop = (float(keep), int(seed))


class StandInPropagation:
    @staticmethod
    def apply(engine, h0, *weights):
        import torch
        L = engine.L
        keep, seed = engine.drop
        masks = [O.state_dropout_mask(seed, l, engine.V, engine.D, keep) for l in range(L - 1)] if keep < 1.0 else None
        engine.seen.append((tuple(h0.shape), [tuple(w.shape) for w in weights]))
        return G.gcn_propagation_torch(h0, engine.lst, torch.from_numpy(engine.w), list(weights[:L]), list(weights[L:]) or None, masks, keep)


@pytest.fixture
def stand_in(monkeypatch):
    monkeypatch.setattr(chem_gcn, "GCNEngine", StandInGCNEngine)
    monkeypatch.setattr(chem_gcn, "_propagation_function", lambda: StandInPropagation)


def _args(tmp_path, mols, n_train=48, **cfg):
    base = {"hidden_size": 16, "batch_size": 300, "num_timesteps": 3, "learning_rate": 0.01, "num_epochs": 2}
    base.update(cfg)
    return {"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:n_train], "--valid_data": mols[n_train:], "--config": base}


def _load_fixture_weights(m, z, cfg):
    import torch
    with torch.no_grad():
        for l in range(cfg["num_timesteps"]):
            m.weights["edge_weights"][l].copy_(torch.from_numpy(z["w%d_kernel" % l]))
            if cfg["gcn_use_bias"]:
                m.weights["edge_biases"][l].copy_(torch.from_numpy(z["w%d_bias" % l]))
        gate, trans = m.weights["regression_gate_task0"], m.weights["regression_transform_task0"]
        gate.weights[0].copy_(torch.from_numpy(z["ro_w_gate"])); gate.biases[0].copy_(torch.from_numpy(z["ro_b_gate"]))
        trans.weights[0].copy_(torch.from_numpy(z["ro_w_trans"])); trans.biases[0].copy_(torch.from_numpy(z["ro_b_trans"]))


def fixture_feed(z):
    return {"initial_node_representation": z["h0"], "adjacency_list": z["adjacency_list"], "adjacency_weights": z["adjacency_weights"],
            "graph_nodes_list": z["graph_nodes_list"], "num_graphs": int(z["num_graphs"]), "target_values": z["target_values"],
            "target_mask": z["target_mask"], "graph_state_keep_prob": 1.0, "out_layer_dropout_keep_prob": 1.0}


def fixture_model(tmp_path, z):
    cfg = json.loads(str(z["params_json"]))
    mols = synthetic.make_molecules(8, seed=1)                    # only sets the dataset's shape facts; the feed comes from the fixture
    m = chem_gcn.SparseGCNChemModel({"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:4], "--valid_data": mols[4:],
                                     "--config": dict(cfg, batch_size=100000)})
    _load_fixture_weights(m, z, cfg)
    return m


@pytest.mark.parametrize("name", ["h12_l3", "h100_l4_bias", "h12_l1"])
def test_forward_batch_matches_the_reference_make_model(tmp_path, golden_dir, stand_in, name):
    """refgraph_gcn_*.npz hold the final states, readout, loss and MAE of the reference's OWN make_model (both GCN hooks, gated_regression,
    masked loss): with the fixture's weights loaded, forward_batch on the fixture's feed returns them."""
    import torch
    z = np.load(os.path.join(golden_dir, "refgraph_gcn_%s.npz" % name))
    m = fixture_model(tmp_path, z)
    with torch.no_grad():
        loss, accs = m.forward_batch(fixture_feed(z))
    final = m.ops["final_node_representations"].numpy()
    np.testing.assert_allclose(final, z["final"], rtol=1e-4, atol=1e-5 * float(np.abs(z["final"]).max()))
    np.testing.assert_allclose(m.output.numpy(), z["readout"], rtol=1e-4, atol=1e-5 * float(np.abs(z["readout"]).max()))
    assert abs(float(loss) - float(z["loss"])) < 1e-4 * abs(float(z["loss"]))
    assert abs(float(accs[0]) - float(z["accuracy"])) < 1e-4 * abs(float(z["accuracy"]))


def test_default_params_and_variables(tmp_path, stand_in):
    p = chem_gcn.SparseGCNChemModel.default_params()
    assert (p["batch_size"], p["task_sample_ratios"], p["gcn_use_bias"], p["graph_state_dropout_keep_prob"], p["num_timesteps"]) == (100000, {}, False, 1.0, 4)
    mols = synthetic.make_molecules(64, seed=1)
    m = chem_gcn.SparseGCNChemModel(_args(tmp_path, mols, gcn_use_bias=True))
    names = [n for n, _ in m.graph_model_variables()]
    assert names == ["graph_model/gcn_scope/gcn_weights_%d:0" % l for l in range(3)] + ["graph_model/gcn_scope/gcn_bias_%d:0" % l for l in range(3)]
    assert all(tuple(v.shape) == (16, 16) for v in m.weights["edge_weights"]) and all(float(b.detach().abs().sum()) == 0 for b in m.weights["edge_biases"])
    assert (m.engine.D, m.engine.L, m.engine.use_bias) == (16, 3, True)


def _assert_same_batch(f, r):
    for k in ("initial_node_representation", "adjacency_list", "adjacency_weights", "graph_nodes_list", "target_values", "target_mask"):
        assert f[k].dtype == r[k].dtype and f[k].shape == r[k].shape and np.array_equal(f[k], r[k]), k
    assert f["num_graphs"] == r["num_graphs"]


def test_plugin_batches_equal_the_per_graph_packer_across_epochs():
    """make_minibatch_iterator (host logic only; built without an engine) over a list that is shuffled in place every epoch, copied and
    shortened: every feed equals iter_gcn_minibatches' batch of the same graphs, bit for bit."""
    m = object.__new__(chem_gcn.SparseGCNChemModel)
    m.params = {"batch_size": 600, "hidden_size": 100, "graph_state_dropout_keep_prob": 0.7}
    data = packing.process_raw_graphs_gcn(synthetic.make_molecules(150, seed=9))

    def check(lst, training):
        state = np.random.get_state()
        feeds = list(m.make_minibatch_iterator(lst, training))          # shuffles lst in place when training
        np.random.set_state(state)
        ref = list(packing.iter_gcn_minibatches(lst, 600, 100))         # same (already shuffled) order
        assert len(feeds) == len(ref) > 2
        for f, r in zip(feeds, ref):
            _assert_same_batch(f, r)
            assert f["graph_state_keep_prob"] == (0.7 if training else 1.0)
            assert "_prepared_graph" not in f

    np.random.seed(3)
    for _ in range(3):
        check(data, True)
    check(list(data), False)
    check(data, True)
    del data[10:40]
    check(data, False)
    assert len(m._flat_cache) <= 4
    with pytest.raises(Exception, match="does not fit"):
        m.params["batch_size"] = 5                                   # gcn:162 loops forever on a graph larger than the budget
        list(m.make_minibatch_iterator(data, False))


def test_flat_packer_equals_pack_gcn_batch_on_shuffled_orders():
    mols = synthetic.make_molecules(300, seed=4)
    proc = packing.process_raw_graphs_gcn(mols)
    for i in range(0, 300, 7):
        proc[i]["labels"][0] = None
    flat = packing.FlatGCNGraphs(proc)
    rng = np.random.default_rng(0)
    for _ in range(6):
        idx = rng.permutation(300)[:int(rng.integers(1, 300))]
        got, ref = flat.pack(idx, 24), packing.pack_gcn_batch([proc[i] for i in idx], 24)
        assert got.keys() == ref.keys()
        _assert_same_batch(got, ref)
    order = rng.permutation(300)
    A = list(packing.iter_gcn_minibatches([proc[i] for i in order], 700, 16))
    B = list(flat.iter_minibatches(order, 700, 16))
    assert len(A) == len(B) > 3
    for a, b in zip(A, B):
        _assert_same_batch(b, a)


def test_flat_packer_reproduces_the_reference_batches(golden_dir):
    """packing_gcn.npz: batches of the reference's own process_raw_graphs + make_minibatch_iterator."""
    z = np.load(os.path.join(golden_dir, "packing_gcn.npz"))
    flat = packing.FlatGCNGraphs(packing.process_raw_graphs_gcn(synthetic.make_molecules(40, seed=123)))
    batches = list(flat.iter_minibatches(np.arange(40), 200, 8))
    assert len(batches) == int(z["num_batches"])
    for bi, b in enumerate(batches):
        np.testing.assert_array_equal(b["initial_node_representation"], z["b%d_init" % bi])
        np.testing.assert_array_equal(b["adjacency_list"], z["b%d_adj" % bi])
        np.testing.assert_array_equal(b["adjacency_weights"], z["b%d_w" % bi])
        np.testing.assert_array_equal(b["graph_nodes_list"], z["b%d_gnl" % bi])
        np.testing.assert_array_equal(b["target_values"], z["b%d_targets" % bi])
        np.testing.assert_array_equal(b["target_mask"], z["b%d_mask" % bi])
        assert b["num_graphs"] == int(z["b%d_num_graphs" % bi])


@pytest.mark.parametrize("cfg", [{}, {"gcn_use_bias": True, "graph_state_dropout_keep_prob": 0.8}])
def test_model_trains_saves_and_restores_on_the_host(tmp_path, stand_in, cfg):
    mols = synthetic.make_molecules(64, seed=1)
    m = chem_gcn.SparseGCNChemModel(_args(tmp_path, mols, **cfg))
    l0 = m.run_epoch("valid0", m.valid_data, False)[0]
    for ep in range(5):
        train_loss, accs, errs, speed, steps = m.run_epoch("train%d" % ep, m.train_data, True)
        assert steps >= 3 and np.isfinite(train_loss)
    l1 = m.run_epoch("valid1", m.valid_data, False)[0]
    assert np.isfinite(l1) and l1 < l0
    path = str(tmp_path / "ckpt.pickle")
    m.save_progress(path, 3, 1)
    saved = pickle.load(open(path, "rb"))["weights"]
    for n, _ in m.graph_model_variables():
        assert n in saved and n[:-2] + "/Adam:0" in saved and n[:-2] + "/Adam_1:0" in saved
    assert saved["graph_model/gcn_scope/gcn_weights_0:0"].shape == (16, 16) and "beta1_power:0" in saved
    assert ("graph_model/gcn_scope/gcn_bias_2:0" in saved) == bool(cfg.get("gcn_use_bias"))
    m2 = chem_gcn.SparseGCNChemModel(_args(tmp_path, mols, **cfg))
    assert m2.restore_progress(path) == (3, 1)
    for (n, a), (_, b) in zip(m.trainable_variables(), m2.trainable_variables()):
        np.testing.assert_array_equal(a.detach().numpy(), b.detach().numpy(), err_msg=n)
    assert abs(m2.run_epoch("valid2", m2.valid_data, False)[0] - l1) < 1e-5 * max(1.0, abs(l1))
    m.train()
    assert pickle.load(open(m.best_model_file, "rb"))["params"]["hidden_size"] == 16


def test_freeze_graph_model_drops_exactly_the_gcn_variables(tmp_path, stand_in):
    mols = synthetic.make_molecules(64, seed=1)
    args = _args(tmp_path, mols, gcn_use_bias=True)
    args["--freeze-graph-model"] = True
    m = chem_gcn.SparseGCNChemModel(args)
    trained = {n for n, _ in m._train_vars}
    graph = {n for n, _ in m.graph_model_variables()}
    assert trained == {n for n, _ in m.trainable_variables()} - graph and len(graph) == 6
    before = [w.detach().clone() for w in m.weights["edge_weights"]]
    m.run_epoch("train", m.train_data, True)
    for a, b in zip(before, m.weights["edge_weights"]):
        np.testing.assert_array_equal(a.numpy(), b.detach().numpy())


def test_task_sample_ratios_and_keep_prob_in_training_only(tmp_path, stand_in):
    """gcn:105-112 drops labels beyond the ratio of the shuffled TRAINING graphs only; gcn:149 feeds the keep probability in training and
    1 in validation -- and the stand-in engine receives it, with a fresh seed per training run."""
    mols = synthetic.make_molecules(96, seed=5)
    m = chem_gcn.SparseGCNChemModel(_args(tmp_path, mols, n_train=80, task_sample_ratios={"0": 0.5}, graph_state_dropout_keep_prob=0.75))
    labelled = total = 0
    for feed in m.make_minibatch_iterator(m.train_data, is_training=True):
        labelled += float(np.sum(feed["target_mask"]))
        total += feed["num_graphs"]
        assert feed["graph_state_keep_prob"] == 0.75
    assert total == 80 and labelled == 40
    for feed in m.make_minibatch_iterator(m.valid_data, is_training=False):
        assert np.all(feed["target_mask"] == 1.0) and feed["graph_state_keep_prob"] == 1.0
    seeds = set()
    for feed in m.make_minibatch_iterator(m.train_data, is_training=True):
        feed["out_layer_dropout_keep_prob"] = 1.0
        m.forward_batch(feed)
        assert m.engine.drop[0] == 0.75
        seeds.add(m.engine.drop[1])
    assert len(seeds) > 1
    m.run_epoch("valid", m.valid_data, False)
    assert m.engine.drop[0] == 1.0


@pytest.mark.parametrize("D", [10, 30])
def test_hidden_sizes_that_are_not_multiples_of_4_run_zero_padded(tmp_path, stand_in, D):
    """The engine wants multiples of 4; the plug-in zero-pads h0, kernels and biases and slices the result.  The stand-in receives the
    PADDED problem; the result matches the oracle on the UNPADDED one, and training flows back to the D-wide variables."""
    import torch
    mols = synthetic.make_molecules(64, seed=3)
    m = chem_gcn.SparseGCNChemModel(_args(tmp_path, mols, hidden_size=D, gcn_use_bias=True))
    DP = (D + 3) // 4 * 4
    assert m._padded_hidden == DP != D and m.engine.D == DP
    with torch.no_grad():
        for b in m.weights["edge_biases"]:
            b.uniform_(-0.2, 0.2)
    feed = next(iter(m.make_minibatch_iterator(m.valid_data, False)))
    m.feed = feed
    with torch.no_grad():
        got = m.compute_final_node_representations().numpy()
    V = feed["initial_node_representation"].shape[0]
    assert m.engine.seen[-1] == ((V, DP), [(DP, DP)] * 3 + [(DP,)] * 3)
    assert got.shape == (V, D)
    ref = G.gcn_propagation_loops(feed["initial_node_representation"], feed["adjacency_list"], feed["adjacency_weights"].astype(np.float32),
                                  [k.detach().numpy() for k in m.weights["edge_weights"]], [b.detach().numpy() for b in m.weights["edge_biases"]])
    np.testing.assert_allclose(got, ref, rtol=2e-5, atol=2e-6 * max(1.0, float(np.abs(ref).max())))
    # gradients flow back through pad / slice to the D-wide variables: the same as float64 autograd of the unpadded problem
    R = torch.from_numpy(np.random.default_rng(1).normal(0, 1, (V, D)))
    (m.compute_final_node_representations().double() * R).sum().backward()
    tk = [k.detach().double().requires_grad_() for k in m.weights["edge_weights"]]
    tb = [b.detach().double().requires_grad_() for b in m.weights["edge_biases"]]
    out = G.gcn_propagation_torch(torch.from_numpy(feed["initial_node_representation"]).double(), feed["adjacency_list"],
                                  torch.from_numpy(feed["adjacency_weights"]), tk, tb)
    (out * R).sum().backward()
    for var, t in zip(m.weights["edge_weights"] + m.weights["edge_biases"], tk + tb):
        assert var.grad.shape == t.shape
        np.testing.assert_allclose(var.grad.numpy(), t.grad.numpy(), rtol=1e-4, atol=1e-5 * float(t.grad.abs().max()))
    m.run_epoch("train", m.train_data, True)
    assert tuple(m.weights["edge_weights"][0].shape) == (D, D) and tuple(m.weights["edge_biases"][0].shape) == (D,)


def test_the_real_engine_refuses_the_cpu(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    with pytest.raises(Exception, match="CUDA|cuda|device"):
        chem_gcn.SparseGCNChemModel(_args(tmp_path, synthetic.make_molecules(64, seed=1)))


def _dp_worker(rank, world, port, tmp, out_q):
    """One data-parallel step of the GCN plug-in (stand-in engine) on this rank's shard of graphs, ONE all-reduce, compared with the
    gradient of the union batch computed locally."""
    import torch.distributed as dist
    from gated_graph_neural_network_samples_b200 import chem_gcn, parallel, synthetic
    from tests.test_chem_gcn_cpu import StandInGCNEngine, StandInPropagation
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    chem_gcn.GCNEngine = StandInGCNEngine
    chem_gcn._propagation_function = lambda: StandInPropagation
    mols = synthetic.make_molecules(40, seed=11)
    args = {"--log_dir": os.path.join(tmp, "r%d" % rank), "--device": "cpu", "--train_data": mols, "--valid_data": mols[:4],
            "--config": {"hidden_size": 12, "batch_size": 100000, "num_timesteps": 3, "gcn_use_bias": True, "random_seed": 3}}
    model = chem_gcn.SparseGCNChemModel(args)               # same seed on every rank -> identical replicas

    def feed_of(graphs):
        proc = model.process_raw_graphs(graphs, is_training_data=False)
        batch = next(iter(model.make_minibatch_iterator(proc, is_training=False)))
        batch["out_layer_dropout_keep_prob"] = 1.0
        return batch

    variables = [v for _, v in model._train_vars]
    model.forward_batch(feed_of(parallel.shard_graphs(mols, rank, world)))
    active = model.reduce_gradients(True)
    got = [v.grad.clone() for v in variables]
    for v in variables:
        v.grad = None
    loss, _ = model.forward_batch(feed_of(mols))            # the union batch on one rank
    loss.backward()
    worst = max(float((g - v.grad).abs().max()) / (float(v.grad.abs().max()) + 1e-12) for g, v in zip(got, variables))
    out_q.put((rank, active, worst))
    dist.barrier()
    dist.destroy_process_group()


def test_data_parallel_step_equals_the_union_batch(tmp_path):
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, str(tmp_path), q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in range(2)]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for rank, active, worst in res:
        assert active == 2 and worst < 1e-4, (rank, active, worst)
