"""GPU: prediction.  The K-task readout kernel (ggnn_readout_predict) against a float64 restatement and against its own K = 1 bits, the
one-call host predictions against the fixtures of the reference's own graph code, the plug-ins' ``predict`` against their validation
forward, the device-data and target-free paths, and guard bands around every buffer the kernel touches."""
import json
import os

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing, synthetic
from gated_graph_neural_network_samples_b200.engine import GgnnError, PropagationEngine
from tests import _util as U
from tests import test_canaries_cpu as K
from tests.test_chem_gcn_cpu import _load_fixture_weights, fixture_feed

pytestmark = pytest.mark.gpu

MAX_TASKS = 16


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _engine(D):
    return PropagationEngine({"hidden_size": D, "layer_timesteps": [1], "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh"}, 2)


def _problem(D, Dreal, K, sizes, seed):
    """Node states and K tasks' weights at width D whose columns from Dreal on are zero (a padded hidden size)."""
    rng = np.random.default_rng(seed)
    V = int(sum(sizes))
    h, h0 = rng.normal(0, 0.5, (V, D)).astype(np.float32), rng.normal(0, 0.5, (V, D)).astype(np.float32)
    h[:, Dreal:] = 0
    h0[:, Dreal:] = 0
    tasks = []
    for _ in range(K):
        wg, wt = rng.normal(0, 0.3, (2, D)).astype(np.float32), rng.normal(0, 0.3, D).astype(np.float32)
        wg[:, Dreal:] = 0
        wt[Dreal:] = 0
        tasks.append((wg.reshape(-1), rng.normal(0, 0.3, 1).astype(np.float32), wt, rng.normal(0, 0.3, 1).astype(np.float32)))
    return h, h0, tasks


def _float64(h, h0, tasks, gnl, G, mask=None):
    """[K, G]: sum over graph g's nodes of sigmoid([h|h0] . w_gate + b_gate) * (h . w_trans + b_trans) * mask."""
    h, h0 = h.astype(np.float64), h0.astype(np.float64)
    D = h.shape[1]
    out = np.zeros((len(tasks), G))
    for k, (wg, bg, wt, bt) in enumerate(tasks):
        gate = h @ wg[:D].astype(np.float64) + h0 @ wg[D:].astype(np.float64) + float(bg[0])
        val = 1.0 / (1.0 + np.exp(-gate)) * (h @ wt.astype(np.float64) + float(bt[0]))
        if mask is not None:
            val = val * mask
        np.add.at(out[k], gnl, val)
    return out


def _sizes(case, rng):
    if case == "one":
        return [int(rng.integers(1, 30))]
    if case == "empty":
        return []
    s = rng.integers(0, 30, 203)          # graphs of zero nodes among them
    s[:3] = 0
    return [int(x) for x in s]


@pytest.mark.parametrize("D,Dreal", [(4, 4), (100, 100), (128, 128), (256, 256), (260, 260), (512, 512), (20, 18), (512, 510)])
@pytest.mark.parametrize("K", [1, 2, 13, MAX_TASKS])
@pytest.mark.parametrize("mode", ["grouped", "atomic", "deterministic"])
@pytest.mark.parametrize("case", ["many", "one", "empty"])
def test_k_task_kernel_against_float64(D, Dreal, K, mode, case):
    import torch
    rng = np.random.default_rng(D * 131 + K * 7 + len(mode) + len(case))
    sizes = _sizes(case, rng)
    G = len(sizes)
    gnl = np.repeat(np.arange(G, dtype=np.int32), sizes)
    if mode != "grouped":
        gnl = gnl[rng.permutation(gnl.shape[0])]
    h, h0, tasks = _problem(D, Dreal, K, sizes, seed=D + K)
    eng = _engine(D)
    eng.set_deterministic(mode == "deterministic")
    eng.readout_set_graphs(G, graph_nodes_list=gnl)
    stride = 2 * G + 7                     # a slot map with gaps: graph g at slot[g], the other columns untouched
    slot = np.sort(rng.choice(stride, G, replace=False)).astype(np.int32)[rng.permutation(G)] if G else np.zeros(0, np.int32)
    out = torch.full((K, stride), -7.0, device="cuda")
    dev_tasks = [tuple(_cuda(a) for a in t) for t in tasks]
    eng.readout_predict(_cuda(h), _cuda(h0), dev_tasks, slot=torch.from_numpy(slot).cuda(), out=out, out_stride=stride)
    got = out.cpu().numpy()
    eng.sync_check()
    ref = _float64(h, h0, tasks, gnl, G)
    rest = np.ones(stride, bool)
    rest[slot] = False
    assert np.all(got[:, rest] == -7.0)
    if G:
        scale = max(np.abs(ref).max(), 1e-3)
        assert np.abs(got[:, slot] - ref).max() / scale < 2e-6 * max(1, max(sizes)) ** 0.5 + 1e-6
    # without a slot map: [K, G]
    plain = eng.readout_predict(_cuda(h), _cuda(h0), dev_tasks).cpu().numpy()
    if mode != "atomic":
        np.testing.assert_array_equal(plain, got[:, slot])


def test_more_tasks_than_the_kernel_holds_are_refused():
    eng = _engine(8)
    eng.readout_set_graphs(2, graph_nodes_list=np.array([0, 0, 1], np.int32))
    h, h0, tasks = _problem(8, 8, MAX_TASKS + 1, [2, 1], seed=1)
    with pytest.raises(GgnnError, match="tasks") as ex:
        eng.readout_predict(_cuda(h), _cuda(h0), [tuple(_cuda(a) for a in t) for t in tasks])
    assert ex.value.code == -1


@pytest.mark.parametrize("D", [100, 512])
@pytest.mark.parametrize("grouped", [True, False])
def test_each_task_column_has_the_bits_of_a_single_task_call(D, grouped):
    """Deterministic mode or a grouped list: task k of a K-task call is bit-identical to a K = 1 call and to ggnn_readout_forward."""
    rng = np.random.default_rng(D)
    sizes = [int(x) for x in rng.integers(1, 30, 500)]
    gnl = np.repeat(np.arange(len(sizes), dtype=np.int32), sizes)
    if not grouped:
        gnl = gnl[rng.permutation(gnl.shape[0])]
    h, h0, tasks = _problem(D, D, 13, sizes, seed=3)
    eng = _engine(D)
    eng.set_deterministic(True)
    eng.readout_set_graphs(len(sizes), graph_nodes_list=gnl)
    dh, dh0 = _cuda(h), _cuda(h0)
    dev_tasks = [tuple(_cuda(a) for a in t) for t in tasks]
    all_k = eng.readout_predict(dh, dh0, dev_tasks).cpu().numpy()
    for k, t in enumerate(dev_tasks):
        np.testing.assert_array_equal(all_k[k], eng.readout_predict(dh, dh0, [t]).cpu().numpy()[0])
        np.testing.assert_array_equal(all_k[k], eng.readout_forward(dh, dh0, *t).cpu().numpy())


# ------------------------------------------------------------------------------------------------ the reference's own graph code
@pytest.mark.parametrize("precision,bar", [("bf16x3", 1e-4), ("fp32", 1e-5)])
@pytest.mark.parametrize("name", ["true_default_shape", "rnn_relu_bias_sum", "attention_bias_avg", "cudnn_gru"])
def test_sparse_host_predict_reproduces_the_reference_readout(golden_dir, name, precision, bar):
    z = np.load(os.path.join(golden_dir, "refgraph_sparse_%s.npz" % name))
    p = json.loads(str(z["params_json"]))
    w = [{k[len("w%d_" % l):]: z[k] for k in z.files if k.startswith("w%d_" % l)} for l in range(len(p["layer_timesteps"]))]
    adj = [z["adj%d" % e] for e in range(4)]
    _, eng = U.engine_sparse(p, 4, w, adj, z["indeg"].astype(np.float32), z["h0"].astype(np.float32), precision=precision, return_engine=True)
    task = tuple(_cuda(z[k]).reshape(-1) for k in ("ro_w_gate", "ro_b_gate", "ro_w_trans", "ro_b_trans"))
    got = eng.run_sparse_host_predict(adj, z["indeg"], z["h0"], z["graph_nodes_list"], int(z["num_graphs"]), [task, task])
    assert got.shape == (2, int(z["num_graphs"]))
    np.testing.assert_array_equal(got[0], got[1])
    assert U.max_rel_err(got[0], z["readout"]) < bar


@pytest.mark.parametrize("precision,bar", [("bf16x3", 1e-4), ("fp32", 1e-5)])
@pytest.mark.parametrize("fixture", ["refgraph_dense.npz", "refgraph_dense_cfg3_shape.npz"])
def test_dense_host_predict_reproduces_the_reference_readout(golden_dir, fixture, precision, bar):
    z = np.load(os.path.join(golden_dir, fixture))
    p = json.loads(str(z["params_json"]))
    b, v, D = z["h0"].shape
    T = z["adj"].shape[1]
    eng = PropagationEngine(U.dense_params_as_engine_params(p, D), T, precision=precision)
    w = {k[2:]: z[k] for k in z.files if k.startswith("w_")}
    if "edge_biases" in w:
        w["edge_biases"] = np.asarray(w["edge_biases"]).reshape(T, D)
    eng.set_weights(U.to_cuda_weights([w]))
    task = tuple(_cuda(z[k]).reshape(-1) for k in ("ro_w_gate", "ro_b_gate", "ro_w_trans", "ro_b_trans"))
    got = eng.run_dense_host_predict(z["adj"], z["h0"].reshape(b * v, D), z["node_mask"], [task])
    assert U.max_rel_err(got[0], z["readout"]) < bar


@pytest.mark.parametrize("precision,bar", [("bf16x3", 1e-4), ("fp32", 1e-5)])
@pytest.mark.parametrize("name", ["h12_l3", "h100_l4_bias", "h12_l1"])
def test_gcn_readout_predict_reproduces_the_reference_readout(tmp_path, golden_dir, name, precision, bar):
    import torch
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    z = np.load(os.path.join(golden_dir, "refgraph_gcn_%s.npz" % name))
    cfg = json.loads(str(z["params_json"]))
    mols = synthetic.make_molecules(8, seed=1)
    m = SparseGCNChemModel({"--log_dir": str(tmp_path), "--precision": precision, "--train_data": mols[:4], "--valid_data": mols[4:],
                            "--config": dict(cfg, batch_size=100000)})
    _load_fixture_weights(m, z, cfg)
    with torch.inference_mode():
        final = m._final_node_representations(fixture_feed(z))
        m._set_readout_map()
        got = m.engine.readout_predict(*m._readout_inputs(final), m._readout_task_weights()).cpu().numpy()
    assert U.max_rel_err(got[0], z["readout"]) < bar


# ------------------------------------------------------------------------------------------------ the plug-ins
def _molecules(n, seed, ntargets=13):
    rng = np.random.default_rng(seed)
    mols = synthetic.make_molecules(n, seed=seed)
    for m in mols:
        m["targets"] = [[float(rng.normal())] for _ in range(ntargets)]
    return mols


TASKS = list(range(13))
PLUGINS = {"sparse": {"batch_size": 2000, "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}},
           "gcn": {"batch_size": 2000, "num_timesteps": 2},
           "dense": {"batch_size": 16, "num_timesteps": 2}}


def _model(name, tmp_path, mols, hidden, precision="fp32"):
    from gated_graph_neural_network_samples_b200.chem_dense import DenseGGNNChemModel
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    cls = {"sparse": SparseGGNNChemModel, "gcn": SparseGCNChemModel, "dense": DenseGGNNChemModel}[name]
    return cls({"--log_dir": str(tmp_path), "--precision": precision, "--train_data": mols[:40], "--valid_data": mols[40:],
                "--config": dict(PLUGINS[name], hidden_size=hidden, task_ids=TASKS)})


def _validation_outputs(m, name, mols):
    """Every task's readout (the fused kernel of gated_regression) after the validation epoch's forward_batch, [tasks, N]."""
    import torch
    out = np.zeros((len(TASKS), len(mols)), np.float32)
    if name == "dense":
        batches = [(ids, packing.pack_dense_batch([mols[i] for i in ids], v, m.params["hidden_size"], m.num_edge_types, TASKS))
                   for v, ids in packing.bucket_batches(mols, m.params["batch_size"])]
    else:
        batches, start = [], 0
        for feed in m.make_minibatch_iterator(m.process_raw_graphs(mols, False), False):
            batches.append((np.arange(start, start + feed["num_graphs"]), feed))
            start += feed["num_graphs"]
    for ids, feed in batches:
        with torch.no_grad():
            m.forward_batch(dict(feed, out_layer_dropout_keep_prob=1.0))
            final = m.ops["final_node_representations"]
            for k, t in enumerate(TASKS):
                out[k, ids] = m.gated_regression(final, m.weights["regression_gate_task%i" % t].bind(1.0),
                                                 m.weights["regression_transform_task%i" % t].bind(1.0)).cpu().numpy()
    return out


@pytest.mark.parametrize("name", sorted(PLUGINS))
@pytest.mark.parametrize("hidden", [100, 18])
def test_plugin_predict_matches_the_validation_forward_and_device_data(tmp_path, name, hidden):
    import torch
    mols = _molecules(300, seed=5)
    m = _model(name, tmp_path, mols, hidden, precision="bf16x3" if hidden == 100 else "fp32")
    shuffled = [mols[i] for i in np.random.default_rng(2).permutation(len(mols))]
    torch.use_deterministic_algorithms(True)
    try:
        host = m.predict(shuffled)
        dev = m.predict(shuffled, device_data=True)
        bare = m.predict([{k: v for k, v in g.items() if k != "targets"} for g in shuffled], device_data=True)
    finally:
        torch.use_deterministic_algorithms(False)
    ref = _validation_outputs(m, name, shuffled)
    assert host.shape == (len(TASKS), len(mols))
    np.testing.assert_array_equal(dev, host)
    np.testing.assert_array_equal(bare, host)
    if hidden == 100:            # the plug-in's validation forward runs the same fused readout: same bits
        np.testing.assert_array_equal(host, ref)
    else:                        # ... its eager fall-back at padded widths: the same sums in another order
        np.testing.assert_allclose(host, ref, rtol=1e-5, atol=1e-5)


def test_a_labelled_device_dataset_predicts_like_a_target_free_one(tmp_path):
    import torch
    from gated_graph_neural_network_samples_b200.engine import DeviceDataset
    mols = _molecules(120, seed=6)
    m = _model("sparse", tmp_path, mols, 100)
    outs = []
    for labels in (True, False):
        flat = packing.FlatSparseGraphs(packing.process_raw_graphs_sparse(mols, TASKS, labels=labels), m.num_edge_types)
        ds = DeviceDataset.for_engine(m.engine, flat, for_training=False)
        assert ds.num_tasks == (len(TASKS) if labels else 0)
        out = torch.zeros(len(TASKS), len(mols), device="cuda")
        with torch.inference_mode():
            for ids in flat.iter_batch_ids(np.arange(len(mols)), 1500):
                batch = ds.prepare_batch(ids, save_for_backward=False)
                final = m._final_node_representations({"num_graphs": len(ids), "_graph_sizes": flat.n_nodes[ids], "_dataset_batch": batch})
                m.engine.readout_predict(*m._readout_inputs(final), m._readout_task_weights(), slot=batch.slot_table, out=out,
                                         out_stride=len(mols))
        outs.append(out.cpu().numpy())
    np.testing.assert_array_equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------------ canaries
@pytest.mark.parametrize("grouped", [True, False])
@pytest.mark.parametrize("ntasks", [1, 13])
def test_guard_bands_around_the_k_task_readout(grouped, ntasks):
    """Every pointer of ggnn_readout_predict guarded (node states, each task's four weights, the slot map, the output): the same bits as on
    plain buffers, no payload read into a result, both bands intact, and no write outside out[k * stride + slot[g]]."""
    import torch
    D, Gn = 36, 300
    rng = np.random.default_rng(ntasks)
    sizes = [int(x) for x in rng.integers(1, 9, Gn)]
    gnl = np.repeat(np.arange(Gn, dtype=np.int32), sizes)
    if not grouped:
        gnl = gnl[rng.permutation(gnl.shape[0])]
    h, h0, tasks = _problem(D, D, ntasks, sizes, seed=9)
    stride = 2 * Gn + 3
    slot = rng.choice(stride, Gn, replace=False).astype(np.int32)
    eng = _engine(D)
    eng.set_deterministic(True)
    eng.readout_set_graphs(Gn, graph_nodes_list=gnl)
    res = {}
    for guard in (True, False):
        def mk(a, dtype=np.float32):
            if not guard:
                return None, torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()
            g = K.guarded(a.size)
            g.view.copy_(torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1)).cuda() if dtype == np.float32
                         else torch.from_numpy(np.ascontiguousarray(a, dtype).reshape(-1)).cuda().view(torch.float32))
            return g, g.view if dtype == np.float32 else g.view.view(torch.int32)
        bufs = [mk(h), mk(h0)] + [mk(a) for t in tasks for a in t] + [mk(slot, np.int32)]
        if guard:
            og = K.guarded(ntasks * stride)
            out = og.view
        else:
            og, out = None, torch.full((ntasks * stride,), float("nan"), device="cuda")
        ts = [b[1] for b in bufs]
        dev_tasks = [tuple(ts[2 + 4 * k:6 + 4 * k]) for k in range(ntasks)]
        eng.readout_predict(ts[0], ts[1], dev_tasks, slot=ts[-1], out=out, out_stride=stride)
        eng.sync_check()
        got = out.view(ntasks, stride)[:, torch.from_numpy(slot).long().cuda()]
        assert not (guard and K.has_payload(got))
        assert all(b[0].bands_intact() for b in bufs if b[0] is not None) and (og is None or og.bands_intact())
        if guard:   # nothing written outside the slots: those words still hold the payload
            rest = np.ones(stride, bool)
            rest[slot] = False
            untouched = og.raw[K.BAND:K.BAND + ntasks * stride].view(ntasks, stride)[:, torch.from_numpy(rest).cuda()]
            assert bool(torch.all(untouched == og.raw[0]).item())
        res[guard] = got.cpu().numpy()
    np.testing.assert_array_equal(res[True], res[False])
