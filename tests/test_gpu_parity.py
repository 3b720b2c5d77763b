"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs."""
import json
import os

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing, synthetic
from oracle import ggnn_oracle as O
from tests import _util as U

pytestmark = pytest.mark.gpu

CFG2 = {"hidden_size": 100, "layer_timesteps": [4], "residual_connections": {}, "use_edge_bias": False,
        "use_edge_msg_avg_aggregation": True, "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh"}
CFG1_TRUE = dict(CFG2, layer_timesteps=[2, 2, 1, 2, 1], residual_connections={"2": [0], "4": [0, 2]})
CFG4 = {"hidden_size": 256, "layer_timesteps": [2, 2, 2, 2], "residual_connections": {"2": [0]}, "use_edge_bias": False,
        "use_edge_msg_avg_aggregation": True, "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh"}
CFG5 = {"hidden_size": 100, "layer_timesteps": [1] * 8, "residual_connections": {}, "use_edge_bias": False,
        "use_edge_msg_avg_aggregation": True, "graph_rnn_cell": "RNN", "graph_rnn_activation": "ReLU"}


def _check(got, ref, rtol=U.RTOL, atol=U.ATOL):
    assert np.all(np.isfinite(got))
    np.testing.assert_allclose(got, ref, rtol=rtol, atol=atol)
    assert U.max_rel_err(got, ref) < 1e-4


@pytest.mark.parametrize("name", ["gru_bias_avg_res", "gru_plain", "rgcn_relu"])
def test_golden_sparse(golden_dir, name):
    z, p, w, adj = U.load_golden_sparse(golden_dir, name)
    got, eng = U.engine_sparse(p, 4, w, adj, z["indeg"], z["h0"], return_engine=True)
    _check(got, z["final"])
    for li in range(len(p["layer_timesteps"]) + 1):   # node_states_per_layer, every entry
        _check(eng.layer_state(li).cpu().numpy(), z["state%d" % li])


def test_golden_dense(golden_dir):
    z = np.load(os.path.join(golden_dir, "prop_dense.npz"))
    p = json.loads(str(z["params_json"]))
    w = {k[2:]: z[k] for k in z.files if k.startswith("w_")}
    _check(U.engine_dense(p, 4, w, z["adj"], z["h0"]), z["final"])


@pytest.mark.parametrize("params,n,T", [(CFG2, 256, 4), (CFG1_TRUE, 256, 4), (CFG4, 128, 8),
                                        (dict(CFG2, use_edge_bias=True, graph_rnn_activation="relu"), 64, 4)])
def test_molecule_batches_vs_oracle(params, n, T):
    _, b = U.molecule_batch(n, params["hidden_size"], T=T, seed=5)
    w = O.init_sparse_weights(params, T, np.random.default_rng(1))
    args = (b["initial_node_representation"], b["adjacency_lists"], b["num_incoming_edges_per_type"], w, params)
    ref = O.sparse_propagation_np(*args, dtype=np.float64)
    got = U.engine_sparse(params, T, w, b["adjacency_lists"], b["num_incoming_edges_per_type"],
                          b["initial_node_representation"])
    _check(got, ref)


@pytest.mark.parametrize("variant", ["0", "1"])
@pytest.mark.parametrize("force_global", ["0", "1"])
def test_tile_variants_and_global_mode_agree(monkeypatch, variant, force_global):
    monkeypatch.setenv("GGNN_FFMA_VARIANT", variant)
    monkeypatch.setenv("GGNN_FORCE_GLOBAL", force_global)
    params = dict(CFG1_TRUE, hidden_size=64, use_edge_bias=True)
    _, b = U.molecule_batch(40, 64, seed=9)
    w = O.init_sparse_weights(params, 4, np.random.default_rng(3))
    ref = O.sparse_propagation_np(b["initial_node_representation"], b["adjacency_lists"],
                                  b["num_incoming_edges_per_type"], w, params, dtype=np.float64)
    got, eng = U.engine_sparse(params, 4, w, b["adjacency_lists"], b["num_incoming_edges_per_type"],
                               b["initial_node_representation"], return_engine=True)
    assert ("GLOBAL" in eng.plan) == (force_global == "1")
    _check(got, ref)


def test_single_large_graph_rgcn_global_mode():
    """cfg5 shape: one 10 000-node graph, 80 000 messages, RNN/ReLU, 8 layers of 1 step (README.md:48-52)."""
    adj, indeg = synthetic.random_sparse_graph(10000, 40000, 4, seed=2)
    rng = np.random.default_rng(4)
    h0 = (rng.normal(0, 0.1, (10000, 100))).astype(np.float32)
    w = O.init_sparse_weights(CFG5, 4, np.random.default_rng(1))
    ref = O.sparse_propagation_np(h0, adj, indeg, w, CFG5, dtype=np.float64)
    got, eng = U.engine_sparse(CFG5, 4, w, adj, indeg, h0, return_engine=True)
    assert "GLOBAL" in eng.plan and eng.last_launch_count == 8
    _check(got, ref)


def test_dense_cfg3_shape_and_sparse_dense_cross_check():
    D, T, steps = 100, 4, 4
    mols = synthetic.make_molecules(64, seed=21)
    db = packing.pack_dense_batch(mols, 32, D, T)
    rng = np.random.default_rng(2)
    h0 = (db["initial_node_representation"] + rng.normal(0, 0.1, db["initial_node_representation"].shape)).astype(np.float32)
    dw = O.init_dense_weights({"hidden_size": D}, T, np.random.default_rng(5))
    dp = {"num_timesteps": steps, "use_edge_bias": True}
    ref = O.dense_propagation_loops(h0, db["adjacency_matrix"], dw, dp)
    got = U.engine_dense(dp, T, dw, db["adjacency_matrix"], h0)
    _check(got, ref)
    # the sparse engine on the same molecules reproduces the dense engine on the real nodes
    sb = packing.pack_sparse_batch(packing.process_raw_graphs_sparse(mols), D, T)
    real = db["node_mask"].astype(bool)
    sw = [dict(dw, edge_biases=dw["edge_biases"].reshape(T, D))]
    sp = U.dense_params_as_engine_params(dp, D)
    got_s = U.engine_sparse(sp, T, sw, sb["adjacency_lists"], sb["num_incoming_edges_per_type"], h0[real])
    np.testing.assert_allclose(got_s, got[real], rtol=1e-4, atol=1e-5)


def test_edge_cases_empty_types_isolated_nodes_tiny_batches():
    params = dict(CFG2, hidden_size=8, layer_timesteps=[2], use_edge_bias=True)
    w = O.init_sparse_weights(params, 4, np.random.default_rng(0))
    rng = np.random.default_rng(1)
    # (a) a single isolated node, no edges at all
    h0 = rng.normal(size=(1, 8)).astype(np.float32)
    adj = [np.zeros((0, 2), np.int32)] * 4
    indeg = np.zeros((1, 4), np.float32)
    _check(U.engine_sparse(params, 4, w, adj, indeg, h0), O.sparse_propagation_loops(h0, adj, indeg, w, params))
    # (b) only edge type 2 present, plus isolated nodes in the middle, plus a self loop and a duplicate edge
    h0 = rng.normal(size=(7, 8)).astype(np.float32)
    a2 = np.array([[0, 1], [1, 0], [1, 0], [3, 3], [5, 6], [6, 5]], np.int32)
    adj = [np.zeros((0, 2), np.int32), np.zeros((0, 2), np.int32), a2, np.zeros((0, 2), np.int32)]
    indeg = np.zeros((7, 4), np.float32)
    np.add.at(indeg[:, 2], a2[:, 1], 1)
    _check(U.engine_sparse(params, 4, w, adj, indeg, h0), O.sparse_propagation_loops(h0, adj, indeg, w, params))
    # (c) zero timesteps: result is the input (sparse:152 with empty loops)
    p0 = dict(params, layer_timesteps=[0])
    got = U.engine_sparse(p0, 4, O.init_sparse_weights(p0, 4, np.random.default_rng(0)), adj, indeg, h0)
    np.testing.assert_array_equal(got, h0)


def test_csr_and_gather_are_bit_exact():
    """Integer path: the device CSR equals NumPy's stable sort of the type-major message list, and with
    W = I, a zero-weight cell and one message per target the gather itself is a bit-exact copy."""
    _, b = U.molecule_batch(50, 12, seed=13)
    params = dict(CFG2, hidden_size=12, layer_timesteps=[1])
    w = O.init_sparse_weights(params, 4, np.random.default_rng(0))
    V = b["initial_node_representation"].shape[0]
    _, eng = U.engine_sparse(params, 4, w, b["adjacency_lists"], b["num_incoming_edges_per_type"],
                             b["initial_node_representation"], return_engine=True)
    row_ptr, src, msg = eng.csr()
    ref_ptr, ref_src, _, ref_order = O.stable_target_csr(b["adjacency_lists"], V)
    np.testing.assert_array_equal(row_ptr[::4], ref_ptr)
    np.testing.assert_array_equal(src, ref_src)
    np.testing.assert_array_equal(msg, ref_order)
    # bit-exact gather: a permutation graph (every node receives exactly one message), RNN/ReLU with
    # kernel [I; 0], W = I, no averaging -> h'[tgt] = relu(h[src]) exactly
    D, n = 12, 37
    perm = np.random.default_rng(3).permutation(n).astype(np.int32)
    adj = [np.stack([perm, np.arange(n, dtype=np.int32)], 1)]
    h0 = np.abs(np.random.default_rng(4).normal(size=(n, D))).astype(np.float32)
    p = {"hidden_size": D, "layer_timesteps": [1], "residual_connections": {}, "use_edge_bias": False,
         "use_edge_msg_avg_aggregation": False, "graph_rnn_cell": "RNN", "graph_rnn_activation": "relu"}
    k = np.concatenate([np.eye(D), np.zeros((D, D))]).astype(np.float32)
    ww = [{"edge_weights": np.eye(D, dtype=np.float32)[None], "rnn_kernel": k, "rnn_bias": np.zeros(D, np.float32)}]
    got = U.engine_sparse(p, 1, ww, adj, np.ones((n, 1), np.float32), h0)
    np.testing.assert_array_equal(got, h0[perm])


def test_host_buffer_call_matches_device_call():
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    _, b = U.molecule_batch(32, 100, seed=3)
    w = O.init_sparse_weights(CFG2, 4, np.random.default_rng(1))
    eng = PropagationEngine(CFG2, 4)
    eng.set_weights(U.to_cuda_weights(w))
    eng.set_graph_sparse(b["adjacency_lists"], b["num_incoming_edges_per_type"])
    dev = eng.forward(torch.from_numpy(b["initial_node_representation"]).cuda()).cpu().numpy()
    host = eng.forward_host(b["initial_node_representation"])
    np.testing.assert_array_equal(dev, host)
    one_call = eng.run_sparse_host(b["adjacency_lists"], b["num_incoming_edges_per_type"], b["initial_node_representation"])
    np.testing.assert_allclose(one_call, host, rtol=1e-4, atol=1e-5)
    assert eng.last_launch_count == 1 and "LOCAL" in eng.plan


def test_two_batches_in_flight_on_two_engines():
    """forward_host(sync=False) on two engines / two streams: both results equal the synchronous call."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    w = U.to_cuda_weights(O.init_sparse_weights(CFG2, 4, np.random.default_rng(1)))
    batches = [U.molecule_batch(24 + 8 * k, 100, seed=5 + k)[1] for k in range(2)]
    engs, streams, outs, ins = [], [], [], []
    for b in batches:
        e = PropagationEngine(CFG2, 4)
        e.set_weights(w)
        engs.append(e)
        streams.append(torch.cuda.Stream())
        ins.append(torch.from_numpy(b["initial_node_representation"]).pin_memory())
        outs.append(torch.empty_like(ins[-1]).pin_memory())
    for rep in range(3):
        for k, b in enumerate(batches):
            with torch.cuda.stream(streams[k]):
                engs[k].set_graph_sparse(b["adjacency_lists"], b["num_incoming_edges_per_type"])
                engs[k].forward_host(ins[k].numpy(), outs[k].numpy(), sync=False)
        for k in range(2):
            with torch.cuda.stream(streams[k]):
                engs[k].sync_check()
    for k, b in enumerate(batches):
        ref = engs[k].forward_host(b["initial_node_representation"])
        np.testing.assert_allclose(outs[k].numpy(), ref, rtol=1e-4, atol=1e-5)


def test_error_behaviour_matches_reference():
    from gated_graph_neural_network_samples_b200.engine import GgnnError, PropagationEngine
    with pytest.raises(Exception, match="Unknown activation"):
        PropagationEngine(dict(CFG2, graph_rnn_activation="gelu"), 4)                 # sparse:81
    with pytest.raises(Exception, match="Unknown RNN cell"):
        PropagationEngine(dict(CFG2, graph_rnn_cell="lstm"), 4)                       # sparse:112
    with pytest.raises(GgnnError, match="multiple of 4"):
        PropagationEngine(dict(CFG2, hidden_size=10), 4)
    eng = PropagationEngine(dict(CFG2, hidden_size=8), 2)
    with pytest.raises(GgnnError, match="out of range"):                              # TF-CPU gather raises on OOB ids
        eng.set_graph_sparse([np.array([[0, 3]], np.int32), np.zeros((0, 2), np.int32)], np.zeros((3, 2), np.float32))
    import torch
    with pytest.raises(GgnnError, match="set_weights"):
        eng.set_graph_sparse([np.array([[0, 1]], np.int32), np.zeros((0, 2), np.int32)], np.zeros((3, 2), np.float32))
        eng.forward(torch.zeros(3, 8, device="cuda"))


def test_full_size_cfg4_properties():
    """BASELINE config 4 at full size (1024 molecules, D=256, T=8): direct comparison with the fp32 torch
    restatement plus a size-independent property: permuting the graphs of the batch permutes the output."""
    mols, b = U.molecule_batch(1024, 256, T=8, seed=0)
    w = O.init_sparse_weights(CFG4, 8, np.random.default_rng(1))
    h0, adj, indeg = b["initial_node_representation"], b["adjacency_lists"], b["num_incoming_edges_per_type"]
    got = U.engine_sparse(CFG4, 8, w, adj, indeg, h0)
    ref = O.sparse_propagation_torch(h0, adj, indeg, w, CFG4).numpy()
    np.testing.assert_allclose(got, ref, rtol=2e-4, atol=2e-5)
    # reverse the order of the molecules in the batch
    proc = packing.process_raw_graphs_sparse(mols)[::-1]
    b2 = packing.pack_sparse_batch(proc, 256, 8)
    sizes = [len(m["node_features"]) for m in mols]
    starts = np.concatenate([[0], np.cumsum(sizes)])
    idx = np.concatenate([np.arange(starts[i], starts[i + 1]) for i in range(len(mols) - 1, -1, -1)])
    got2 = U.engine_sparse(CFG4, 8, w, b2["adjacency_lists"], b2["num_incoming_edges_per_type"], h0[idx])
    np.testing.assert_allclose(got2, got[idx], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_dense_weighted_adjacency_weights_its_messages(precision):
    """A non-binary adjacency is converted to a CSR that carries its entries as per-message weights (the reference's matmul
    semantics, dense:110-112); a binary one to a plain CSR -- both must agree with the oracle."""
    D, T, steps, b, v = 24, 3, 2, 5, 16
    rng = np.random.default_rng(11)
    A = (rng.random((b, T, v, v)) < 0.15).astype(np.float32)
    Aw = A * rng.uniform(0.25, 1.5, size=A.shape).astype(np.float32)
    h0 = rng.normal(0, 0.3, (b, v, D)).astype(np.float32)
    dw = O.init_dense_weights({"hidden_size": D}, T, np.random.default_rng(5))
    dp = {"num_timesteps": steps, "use_edge_bias": True}
    for adj in (Aw, A):
        ref = O.dense_propagation_loops(h0, adj, dw, dp)
        got = U.engine_dense(dp, T, dw, adj, h0, precision=precision)
        assert U.max_rel_err(got, ref) < 1e-4
