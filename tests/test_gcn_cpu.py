"""Sparse GCN on the CPU: the packer, the two oracles against each other, and the host half of the engine (ggnn_host_prepare_graph_gcn)
pinned against NumPy -- stable CSR by output row, per-slot weights, index validation, tile plans."""
import json
import os

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing, synthetic
from gated_graph_neural_network_samples_b200.engine import GgnnError, PreparedGraph
from tests import gcn_oracle as G


def reference_gcn_adjacency(graph, num_nodes):
    """chem_tensorflow_gcn.py:116-142 written out as the reference's loops."""
    adj = np.zeros((num_nodes, num_nodes))
    for src, _, dest in graph:
        adj[src, dest] = 1
        adj[dest, src] = 1
    adj += np.eye(num_nodes)
    d = np.diag(np.power(np.sum(adj, axis=-1), -0.5).flatten() + 1e-7)
    adj = d.dot(adj).dot(d)
    lst, ws = [], []
    for i in range(num_nodes):
        for j in range(num_nodes):
            if adj[i, j] != 0:
                lst.append([i, j])
                ws.append(adj[i, j])
    return np.array(lst), np.array(ws)


def test_packer_matches_the_reference_loops_bit_for_bit():
    mols = synthetic.make_molecules(20, seed=7)
    mols[0]["graph"] = list(mols[0]["graph"]) + [list(mols[0]["graph"][0])]   # a duplicate bond collapses
    for d in mols:
        lst, w = packing.graph_to_gcn_adjacency(d["graph"], len(d["node_features"]))
        rl, rw = reference_gcn_adjacency(d["graph"], len(d["node_features"]))
        assert lst.dtype == np.int64 and w.dtype == np.float64
        np.testing.assert_array_equal(lst, rl)
        np.testing.assert_array_equal(w, rw)


def test_batches_concatenate_with_node_offsets():
    mols = synthetic.make_molecules(30, seed=3)
    data = packing.process_raw_graphs_gcn(mols)
    batches = list(packing.iter_gcn_minibatches(data, 200, 16))
    assert sum(b["num_graphs"] for b in batches) == 30
    off = 0
    first = batches[0]
    for gi in range(first["num_graphs"]):
        n = len(data[gi]["init"])
        assert off + n < 200
        off += n
    assert first["initial_node_representation"].shape == (off, 16)
    np.testing.assert_array_equal(first["adjacency_list"][:len(data[0]["adjacency_list"])], data[0]["adjacency_list"])
    n0 = len(data[0]["init"])
    np.testing.assert_array_equal(first["adjacency_list"][len(data[0]["adjacency_list"]):][:len(data[1]["adjacency_list"])],
                                  data[1]["adjacency_list"] + n0)
    assert first["adjacency_weights"].dtype == np.float64
    assert first["target_values"].shape == (1, first["num_graphs"])


def test_loop_and_torch_oracles_agree():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(1)
    V, D = 40, 12
    lst, w = G.random_gcn_list(V, 150, rng, isolated=(3, 17))
    ks = [G.glorot((D, D), rng) for _ in range(3)]
    bs = [rng.normal(0, 0.1, D).astype(np.float32) for _ in range(3)]
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    masks = [rng.random((V, D)) < 0.7 for _ in range(2)]
    ref = G.gcn_propagation_loops(h0, lst, w, ks, bs, masks, 0.7)
    got = G.gcn_propagation_torch(torch.from_numpy(h0).double(), lst, torch.from_numpy(w).double(), [torch.from_numpy(k).double() for k in ks],
                                  [torch.from_numpy(b).double() for b in bs], masks, 0.7)
    np.testing.assert_allclose(got.numpy(), ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("threads", ["1", "2", "5", "8"])
def test_host_csr_is_numpy_stable_sort_with_slot_weights(monkeypatch, threads):
    monkeypatch.setenv("GGNN_HOST_THREADS", threads)
    rng = np.random.default_rng(int(threads))
    V = 300
    lst, w = G.random_gcn_list(V, 30000, rng, isolated=(0, 299, 150))
    g = PreparedGraph.host_only_gcn(32, 2, V, lst, w, precision="bf16x3", save_for_backward=True)
    a = g.arrays(1)
    order = np.argsort(lst[:, 0], kind="stable")
    np.testing.assert_array_equal(a["row_ptr"], np.concatenate([[0], np.cumsum(np.bincount(lst[:, 0], minlength=V))]))
    np.testing.assert_array_equal(a["msg"], order)
    np.testing.assert_array_equal(a["src"], lst[order, 1])
    np.testing.assert_array_equal(g.slot_weights(), w[a["msg"]])
    np.testing.assert_array_equal(g.slot_weights(source_order=True), w[np.argsort(lst[:, 1], kind="stable")])
    assert g.info()["num_messages"] == lst.shape[0]


def test_image_bytes_do_not_depend_on_the_thread_count(monkeypatch):
    rng = np.random.default_rng(5)
    V = 500
    lst, w = G.random_gcn_list(V, 40000, rng)
    images = []
    for t in ("1", "3", "8"):
        monkeypatch.setenv("GGNN_HOST_THREADS", t)
        images.append(PreparedGraph.host_only_gcn(64, 3, V, lst, w, precision="fp32", save_for_backward=True).image())
    for img in images[1:]:
        np.testing.assert_array_equal(img, images[0])


@pytest.mark.parametrize("bad", [(5, 0), (0, 5), (-1, 0), (0, -1), (2 ** 33, 0)])
def test_out_of_range_index_is_refused(bad):
    lst = np.array([[0, 1], [1, 2], list(bad)], np.int64)
    with pytest.raises(GgnnError, match="out of range"):
        PreparedGraph.host_only_gcn(16, 2, 5, lst, np.ones(3, np.float32))


def test_empty_list_and_empty_batch():
    g = PreparedGraph.host_only_gcn(16, 2, 7, np.zeros((0, 2), np.int64), np.zeros(0, np.float32), save_for_backward=True)
    a = g.arrays(1)
    assert g.info()["num_messages"] == 0 and np.all(a["row_ptr"] == 0)
    g = PreparedGraph.host_only_gcn(16, 2, 0, np.zeros((0, 2), np.int64), np.zeros(0, np.float32))
    assert g.info()["num_nodes"] == 0


def test_plans_name_the_kernel_that_runs(monkeypatch):
    monkeypatch.delenv("GGNN_FORCE_GLOBAL", raising=False)
    rng = np.random.default_rng(2)
    V, lst, w = G.component_list([20] * 50, rng)
    plan = PreparedGraph.host_only_gcn(100, 4, V, lst, w, precision="bf16x3").info()["plan"]
    assert plan.startswith("gcn-wgmma-bf16x3 LOCAL"), plan
    tiles = PreparedGraph.host_only_gcn(100, 4, V, lst, w, precision="bf16x3").arrays(1)["tile_start"]
    # tiles are unions of whole components
    assert all(t % 20 == 0 for t in tiles) and tiles[-1] == V
    V2, lst2, w2 = G.component_list([300, 10], rng)
    assert "GLOBAL" in PreparedGraph.host_only_gcn(100, 4, V2, lst2, w2, precision="bf16").info()["plan"]
    assert PreparedGraph.host_only_gcn(100, 4, V, lst, w, precision="fp32").info()["plan"].startswith("gcn-fp32")
    assert PreparedGraph.host_only_gcn(256, 4, V, lst, w, precision="bf16x3").info()["plan"].startswith("gcn-fp32")


def test_limits_are_refused():
    lst, w = np.zeros((0, 2), np.int64), np.zeros(0, np.float32)
    for D, L in ((10, 2), (260, 2), (16, 0), (16, 17)):
        with pytest.raises(GgnnError):
            PreparedGraph.host_only_gcn(D, L, 4, lst, w)


def test_ggnn_prepared_graphs_have_no_slot_weights():
    from gated_graph_neural_network_samples_b200 import workloads
    params = dict(workloads.SPARSE_BASE, hidden_size=16, layer_timesteps=[1])
    g = PreparedGraph.host_only(params, 1, [np.array([[0, 1]], np.int32)], np.array([[0.0], [1.0]], np.float32))
    with pytest.raises(GgnnError):
        g.slot_weights()


def test_packer_reproduces_the_reference_batches(golden_dir):
    """packing_gcn.npz: batches of the reference's own process_raw_graphs + make_minibatch_iterator (tests/golden/make_gcn_golden.py)."""
    z = np.load(os.path.join(golden_dir, "packing_gcn.npz"))
    data = packing.process_raw_graphs_gcn(synthetic.make_molecules(40, seed=123))
    batches = list(packing.iter_gcn_minibatches(data, 200, 8))
    assert len(batches) == int(z["num_batches"])
    for bi, b in enumerate(batches):
        np.testing.assert_array_equal(b["initial_node_representation"], z["b%d_init" % bi])
        np.testing.assert_array_equal(b["adjacency_list"], z["b%d_adj" % bi])
        np.testing.assert_array_equal(b["adjacency_weights"], z["b%d_w" % bi])      # float64, bit for bit
        np.testing.assert_array_equal(b["graph_nodes_list"], z["b%d_gnl" % bi])
        np.testing.assert_array_equal(b["target_values"], z["b%d_targets" % bi])
        np.testing.assert_array_equal(b["target_mask"], z["b%d_mask" % bi])
        assert b["num_graphs"] == int(z["b%d_num_graphs" % bi])


def gated_regression_loss(final, z):
    """gcn:84-93 + chem_tensorflow.py:158-166 in float64: per-graph readout, masked 1/2-MSE loss and MAE of task 0."""
    h0 = np.asarray(z["h0"], np.float64)
    gate = 1.0 / (1.0 + np.exp(-(np.concatenate([final, h0], 1) @ z["ro_w_gate"].astype(np.float64) + z["ro_b_gate"].astype(np.float64))))
    vals = gate * (final @ z["ro_w_trans"].astype(np.float64) + z["ro_b_trans"].astype(np.float64))
    ro = np.zeros(int(z["num_graphs"]))
    np.add.at(ro, z["graph_nodes_list"], vals[:, 0])
    diff = (ro - z["target_values"][0]) * z["target_mask"][0]
    n = z["target_mask"][0].sum() + 1e-7
    return ro, np.sum(0.5 * diff ** 2) / n, np.sum(np.abs(diff)) / n


@pytest.mark.parametrize("name", ["h12_l3", "h100_l4_bias", "h12_l1"])
def test_oracles_reproduce_the_reference_graph(golden_dir, name):
    """refgraph_gcn_*.npz: the reference's unmodified make_model evaluated in float64 -- final states, readout, loss and MAE."""
    torch = pytest.importorskip("torch")
    z = np.load(os.path.join(golden_dir, "refgraph_gcn_%s.npz" % name))
    cfg = json.loads(str(z["params_json"]))
    L = cfg["num_timesteps"]
    ks = [z["w%d_kernel" % l] for l in range(L)]
    bs = [z["w%d_bias" % l] for l in range(L)] if cfg["gcn_use_bias"] else None
    final = G.gcn_propagation_loops(z["h0"], z["adjacency_list"], z["adjacency_weights"], ks, bs)
    np.testing.assert_allclose(final, z["final"], rtol=1e-12, atol=1e-12)
    ro, loss, mae = gated_regression_loss(final, z)
    np.testing.assert_allclose(ro, z["readout"], rtol=1e-12, atol=1e-12)
    assert abs(loss - float(z["loss"])) <= 1e-12 * abs(float(z["loss"])) and abs(mae - float(z["accuracy"])) <= 1e-12 * abs(float(z["accuracy"]))
    t = G.gcn_propagation_torch(torch.from_numpy(z["h0"]), z["adjacency_list"], torch.from_numpy(z["adjacency_weights_f32"]),
                                [torch.from_numpy(k) for k in ks], None if bs is None else [torch.from_numpy(b) for b in bs])
    assert float(np.max(np.abs(t.numpy() - z["final"])) / np.max(np.abs(z["final"]))) < 1e-6


@pytest.mark.parametrize("bad", [np.zeros(6, np.int64), np.zeros((2, 3), np.int64), np.zeros((3, 2, 1), np.int64)])
def test_misshaped_lists_are_refused(bad):
    with pytest.raises(GgnnError, match=r"\[nnz, 2\]"):
        PreparedGraph.host_only_gcn(16, 2, 5, bad, np.ones(3, np.float32))
