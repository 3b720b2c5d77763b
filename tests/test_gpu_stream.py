"""GPU parity of the STREAMING wgmma path (ggnn_fwd_stream.cuh: hidden sizes > 128, BASELINE config 4, and -- forced with
GGNN_TC_STREAM=1 -- any CSR batch) against the float64 oracle at the north-star tolerance (1e-4 relative)."""
import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import packing, synthetic
from oracle import ggnn_oracle as O
from tests import _util as U
from tests.test_gpu_parity import CFG1_TRUE, CFG2, CFG4, CFG5

pytestmark = pytest.mark.gpu
PREC = "bf16x3"


def _check(got, ref, tag=""):
    assert np.all(np.isfinite(got))
    err = U.max_rel_err(got, ref)
    print("[stream %s] %s max|err|/max|ref| = %.3e" % (PREC, tag, err))
    assert err < 1e-4
    np.testing.assert_allclose(got, ref, rtol=1e-4, atol=1e-4 * float(np.max(np.abs(ref))))


def _run(params, T, w, b, tag, precision=PREC):
    ref = O.sparse_propagation_np(b["initial_node_representation"], b["adjacency_lists"], b["num_incoming_edges_per_type"], w, params,
                                  dtype=np.float64)
    got, eng = U.engine_sparse(params, T, w, b["adjacency_lists"], b["num_incoming_edges_per_type"], b["initial_node_representation"],
                               precision=precision, return_engine=True)
    assert "STREAM" in eng.plan, eng.plan
    _check(got, ref, tag)
    return got, eng, ref


@pytest.mark.parametrize("n", [20, 128, 300])
def test_cfg4_shape_hidden_256_eight_edge_types(n):
    """BASELINE config 4's model (D=256, T=8, [2,2,2,2], residual {"2":[0]}) on 20 / 128 / 300 molecules: fewer tiles than SMs
    (N-split gate), a ragged last tile, and more than one tile per SM pair."""
    _, b = U.molecule_batch(n, 256, T=8, seed=5)
    w = O.init_sparse_weights(CFG4, 8, np.random.default_rng(1))
    got, eng, _ = _run(CFG4, 8, w, b, "cfg4 n=%d" % n)
    steps = sum(CFG4["layer_timesteps"])
    assert eng.last_launch_count >= 3 * steps


def test_hidden_256_layer_states_bias_relu_rnn():
    p = dict(CFG4, layer_timesteps=[1, 2], residual_connections={"1": [0]}, use_edge_bias=True, graph_rnn_cell="RNN", graph_rnn_activation="relu")
    _, b = U.molecule_batch(40, 256, T=8, seed=11)
    w = O.init_sparse_weights(p, 8, np.random.default_rng(2))
    for lw in w:
        lw["edge_biases"] = np.random.default_rng(3).uniform(-0.1, 0.1, lw["edge_biases"].shape).astype(np.float32)
    _run(p, 8, w, b, "rnn relu bias D=256")


def test_hidden_192_and_132_are_padded_inside_the_kernel():
    for D in (192, 132):
        p = dict(CFG2, hidden_size=D, layer_timesteps=[2], use_edge_bias=True)
        _, b = U.molecule_batch(30, D, T=4, seed=7)
        w = O.init_sparse_weights(p, 4, np.random.default_rng(1))
        _run(p, 4, w, b, "D=%d" % D)


@pytest.mark.parametrize("params,n", [(CFG2, 256), (CFG1_TRUE, 100), (dict(CFG2, use_edge_bias=True, graph_rnn_activation="relu", hidden_size=64), 64),
                                      (dict(CFG1_TRUE, hidden_size=128, graph_rnn_cell="RNN"), 100)])
def test_forced_stream_matches_oracle_at_small_hidden_sizes(monkeypatch, params, n):
    monkeypatch.setenv("GGNN_TC_STREAM", "1")
    _, b = U.molecule_batch(n, params["hidden_size"], T=4, seed=5)
    w = O.init_sparse_weights(params, 4, np.random.default_rng(1))
    _, eng, _ = _run(params, 4, w, b, "forced stream D=%d" % params["hidden_size"])
    assert eng.last_launch_count > 1


def test_forced_stream_golden_layer_states(monkeypatch, golden_dir):
    monkeypatch.setenv("GGNN_TC_STREAM", "1")
    for name in ("gru_bias_avg_res", "gru_plain", "rgcn_relu"):
        z, p, w, adj = U.load_golden_sparse(golden_dir, name)
        got, eng = U.engine_sparse(p, 4, w, adj, z["indeg"], z["h0"], precision=PREC, return_engine=True)
        assert "STREAM" in eng.plan
        _check(got, z["final"], name)
        for li in range(len(p["layer_timesteps"]) + 1):
            _check(eng.layer_state(li).cpu().numpy(), z["state%d" % li], "%s layer %d" % (name, li))


def test_forced_stream_single_large_graph(monkeypatch):
    monkeypatch.setenv("GGNN_TC_STREAM", "1")
    adj, indeg = synthetic.random_sparse_graph(10000, 40000, 4, seed=2)
    h0 = np.random.default_rng(4).normal(0, 0.1, (10000, 100)).astype(np.float32)
    w = O.init_sparse_weights(CFG5, 4, np.random.default_rng(1))
    ref = O.sparse_propagation_np(h0, adj, indeg, w, CFG5, dtype=np.float64)
    got, eng = U.engine_sparse(CFG5, 4, w, adj, indeg, h0, precision=PREC, return_engine=True)
    assert "STREAM" in eng.plan
    _check(got, ref, "cfg5 forced stream")


def test_edge_cases_hidden_256():
    params = dict(CFG4, layer_timesteps=[2], residual_connections={}, use_edge_bias=True)
    w = O.init_sparse_weights(params, 8, np.random.default_rng(0))
    rng = np.random.default_rng(1)
    none = np.zeros((0, 2), np.int32)
    # a single isolated node, no edges at all (no K-steps in the gather GEMM)
    h0 = rng.normal(size=(1, 256)).astype(np.float32)
    adj = [none] * 8
    indeg = np.zeros((1, 8), np.float32)
    _check(U.engine_sparse(params, 8, w, adj, indeg, h0, precision=PREC), O.sparse_propagation_loops(h0, adj, indeg, w, params), "isolated")
    # one edge type present, isolated nodes, a self loop, a duplicate edge, 130 nodes (second tile has 2 rows and no messages)
    h0 = rng.normal(size=(130, 256)).astype(np.float32)
    a5 = np.array([[0, 1], [1, 0], [1, 0], [3, 3], [5, 6], [6, 5], [100, 2]], np.int32)
    adj = [none] * 5 + [a5] + [none] * 2
    indeg = np.zeros((130, 8), np.float32)
    np.add.at(indeg[:, 5], a5[:, 1], 1)
    _check(U.engine_sparse(params, 8, w, adj, indeg, h0, precision=PREC), O.sparse_propagation_loops(h0, adj, indeg, w, params), "one type, two tiles")
    # zero timesteps in the middle layer: that layer aliases its input (sparse:152)
    p0 = dict(CFG4, layer_timesteps=[1, 0, 1], residual_connections={"2": [1]})
    w0 = O.init_sparse_weights(p0, 8, np.random.default_rng(0))
    _, b = U.molecule_batch(9, 256, T=8, seed=2)
    _run(p0, 8, w0, b, "zero-step layer")


def test_fast_single_bf16_mode_hidden_256():
    _, b = U.molecule_batch(64, 256, T=8, seed=5)
    w = O.init_sparse_weights(CFG4, 8, np.random.default_rng(1))
    ref = O.sparse_propagation_np(b["initial_node_representation"], b["adjacency_lists"], b["num_incoming_edges_per_type"], w, CFG4, dtype=np.float64)
    got = U.engine_sparse(CFG4, 8, w, b["adjacency_lists"], b["num_incoming_edges_per_type"], b["initial_node_representation"], precision="bf16")
    err = U.max_rel_err(got, ref)
    print("[stream bf16] max|err|/max|ref| = %.3e" % err)
    assert err < 3e-2


def test_full_size_cfg4_stream_properties():
    """BASELINE config 4 at full size (1024 molecules): vs the fp32 torch restatement, run-to-run bit-identical (one issuer, fixed
    order), and permuting the graphs of the batch permutes the output."""
    mols, b = U.molecule_batch(1024, 256, T=8, seed=0)
    w = O.init_sparse_weights(CFG4, 8, np.random.default_rng(1))
    h0, adj, indeg = b["initial_node_representation"], b["adjacency_lists"], b["num_incoming_edges_per_type"]
    got = U.engine_sparse(CFG4, 8, w, adj, indeg, h0, precision=PREC)
    ref = O.sparse_propagation_torch(h0, adj, indeg, w, CFG4).numpy()
    np.testing.assert_allclose(got, ref, rtol=2e-4, atol=2e-5)
    again = U.engine_sparse(CFG4, 8, w, adj, indeg, h0, precision=PREC)
    np.testing.assert_array_equal(got, again)
    proc = packing.process_raw_graphs_sparse(mols)[::-1]
    b2 = packing.pack_sparse_batch(proc, 256, 8)
    sizes = [len(m["node_features"]) for m in mols]
    starts = np.concatenate([[0], np.cumsum(sizes)])
    idx = np.concatenate([np.arange(starts[i], starts[i + 1]) for i in range(len(mols) - 1, -1, -1)])
    got2 = U.engine_sparse(CFG4, 8, w, b2["adjacency_lists"], b2["num_incoming_edges_per_type"], h0[idx], precision=PREC)
    np.testing.assert_allclose(got2, got[idx], rtol=1e-5, atol=1e-6)


def test_gradients_hidden_256_stream_forward_saved_states():
    """Forward on the streaming path with save_for_backward, backward through ggnn_backward: every gradient against float64 autograd."""
    from tests.test_gpu_backward import _autograd_reference, _cmp, _engine_grads
    p = dict(CFG4, layer_timesteps=[2, 1], residual_connections={"1": [0]}, use_edge_bias=True)
    T = 8
    _, b = U.molecule_batch(12, 256, T=T, seed=3)
    w = O.init_sparse_weights(p, T, np.random.default_rng(1))
    h0, adj, indeg = b["initial_node_representation"], b["adjacency_lists"], b["num_incoming_edges_per_type"]
    G = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    ref_out, ref_dh0, ref_gw = _autograd_reference(p, T, w, adj, indeg, h0, G)
    out, dh0, gw = _engine_grads(p, T, w, lambda e: e.set_graph_sparse(adj, indeg), h0, G, PREC)
    _cmp(out, ref_out, "forward")
    _cmp(dh0, ref_dh0, "d h0")
    for l, (a, r) in enumerate(zip(gw, ref_gw)):
        for k in r:
            _cmp(a[k], r[k], "layer %d %s" % (l, k))


def test_state_dropout_on_the_streaming_path():
    p = dict(CFG4, layer_timesteps=[2], residual_connections={})
    T, keep, seed = 8, 0.8, 1234
    _, b = U.molecule_batch(10, 256, T=T, seed=4)
    w = O.init_sparse_weights(p, T, np.random.default_rng(1))
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    eng = PropagationEngine(p, T, precision=PREC)
    eng.set_weights(U.to_cuda_weights(w))
    eng.set_state_dropout(keep, seed)
    eng.set_graph_sparse(b["adjacency_lists"], b["num_incoming_edges_per_type"])
    h0 = b["initial_node_representation"]
    got = eng.forward(torch.from_numpy(h0).cuda()).cpu().numpy()
    eng.sync_check()
    ref = O.sparse_propagation_torch(h0, b["adjacency_lists"], b["num_incoming_edges_per_type"], w, p,
                                     dtype=torch.float64, state_dropout=(keep, seed)).numpy()
    _check(got, ref, "state dropout")
    np.testing.assert_array_equal(got != 0.0, eng.state_dropout_mask(1, keep, seed).astype(bool) & (ref != 0.0))


@pytest.mark.parametrize("D,T,plan", [(100, 4, "LOCAL"), (256, 8, "STREAM")])
def test_error_growth_over_32_timesteps_stays_inside_the_bar(D, T, plan):
    """The epilogues use ex2-based sigmoid / tanh and the operands carry 16 mantissa bits: 32 recurrent timesteps (8x the deepest BASELINE
    configuration) bound how those errors accumulate on both tensor-core plans."""
    p = dict(CFG2, hidden_size=D, layer_timesteps=[32])
    _, b = U.molecule_batch(24, D, T=T, seed=17)
    w = O.init_sparse_weights(p, T, np.random.default_rng(1))
    ref = O.sparse_propagation_np(b["initial_node_representation"], b["adjacency_lists"], b["num_incoming_edges_per_type"], w, p, dtype=np.float64)
    got, eng = U.engine_sparse(p, T, w, b["adjacency_lists"], b["num_incoming_edges_per_type"], b["initial_node_representation"],
                               precision=PREC, return_engine=True)
    assert plan in eng.plan
    _check(got, ref, "32 timesteps D=%d" % D)


def test_hub_nodes_with_many_messages_per_type():
    """Virtual rows of every length: a hub receiving 40 messages of one type (the source list continues past the 7 inline entries of
    vinfo), nodes with 3..12 messages, duplicates and self loops -- summed in message order like TF's CPU unsorted_segment_sum."""
    rng = np.random.default_rng(7)
    V, T, D = 300, 3, 256
    p = dict(CFG4, layer_timesteps=[2], residual_connections={}, use_edge_bias=True)
    adj = []
    for t in range(T):
        e = [(int(s), 0) for s in rng.integers(1, V, size=40)] if t == 1 else []          # the hub (node 0), type 1
        for tgt in range(5, 120, 5):                                                       # 3 .. 12 messages into a few nodes
            e += [(int(s), tgt) for s in rng.integers(0, V, size=3 + (tgt // 5) % 10)]
        e += [(10, 10), (10, 10), (200, 299), (299, 200)]                                  # self loop twice, a pair across the tile boundary
        e = np.asarray(sorted(e), np.int32).reshape(-1, 2)
        adj.append(e)
    indeg = np.zeros((V, T), np.float32)
    for t in range(T):
        np.add.at(indeg[:, t], adj[t][:, 1], 1)
    h0 = rng.normal(0, 0.3, (V, D)).astype(np.float32)
    w = O.init_sparse_weights(p, T, np.random.default_rng(1))
    ref = O.sparse_propagation_np(h0, adj, indeg, w, p, dtype=np.float64)
    got, eng = U.engine_sparse(p, T, w, adj, indeg, h0, precision=PREC, return_engine=True)
    assert "STREAM" in eng.plan
    _check(got, ref, "hub nodes")


@pytest.mark.parametrize("ksteps,stages", [("1", "8"), ("1", "2"), ("2", "3"), ("4", "2"), ("4", "3"), ("3", "5")])
def test_ring_geometry_does_not_change_the_result(monkeypatch, ksteps, stages):
    """K-steps per stage and ring depth (incl. the shallowest ring, one stage per gather group, and partial last stages of a K segment)
    only change the schedule and -- because the gather GEMM walks K group by K group -- the fp32 summation order: the result stays within
    rounding of the default geometry and is bit-identical from run to run for a fixed geometry."""
    _, b = U.molecule_batch(40, 256, T=8, seed=21)
    w = O.init_sparse_weights(CFG4, 8, np.random.default_rng(1))
    args = (CFG4, 8, w, b["adjacency_lists"], b["num_incoming_edges_per_type"], b["initial_node_representation"])
    base = U.engine_sparse(*args, precision=PREC)
    monkeypatch.setenv("GGNN_TS_KSTEPS", ksteps)
    monkeypatch.setenv("GGNN_TS_STAGES", stages)
    got = U.engine_sparse(*args, precision=PREC)
    np.testing.assert_allclose(got, base, rtol=2e-5, atol=2e-6)
    np.testing.assert_array_equal(got, U.engine_sparse(*args, precision=PREC))


@pytest.mark.parametrize("first", ["1", "0"])
def test_set_weights_once_reaches_both_plans_of_one_engine(monkeypatch, first):
    """One engine, weights set once per update, batches alternating between the streaming and the tile-local plan: each plan keeps its
    own tiled copy of the weights, and a forward after set_weights must run on the new weights whichever plan tiled them last."""
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    _, b = U.molecule_batch(40, 100, T=4, seed=13)
    h0, adj, indeg = b["initial_node_representation"], b["adjacency_lists"], b["num_incoming_edges_per_type"]
    w1, w2 = (O.init_sparse_weights(CFG2, 4, np.random.default_rng(s)) for s in (1, 2))
    eng = PropagationEngine(CFG2, 4, precision=PREC)
    h0_dev = torch.from_numpy(h0).cuda()

    def forward(stream):
        monkeypatch.setenv("GGNN_TC_STREAM", stream)   # read when the batch is prepared
        eng.set_graph_sparse(adj, indeg)
        assert ("STREAM" in eng.plan) == (stream == "1"), eng.plan
        out = eng.forward(h0_dev).cpu().numpy()
        eng.sync_check()
        return out

    other = "0" if first == "1" else "1"
    eng.set_weights(U.to_cuda_weights(w1))
    forward(first)
    eng.set_weights(U.to_cuda_weights(w2))
    forward(other)
    _check(forward(first), O.sparse_propagation_np(h0, adj, indeg, w2, CFG2, dtype=np.float64), "plan %s after the other plan re-tiled" % first)


def test_twelve_edge_types_and_hidden_100_padding(monkeypatch):
    """More edge types than any BASELINE configuration (tile masks, K segments) on the forced streaming plan at a hidden size that is
    not a multiple of 16 (DP = 112: seven K-steps per segment, a partial last stage)."""
    monkeypatch.setenv("GGNN_TC_STREAM", "1")
    rng = np.random.default_rng(3)
    V, T, D = 500, 12, 100
    p = dict(CFG2, hidden_size=D, layer_timesteps=[2, 1], residual_connections={"1": [0]})
    adj = []
    for t in range(T):
        n = 0 if t == 5 else int(rng.integers(20, 400))                                    # one type without any edge
        e = np.stack([rng.integers(0, V, n), rng.integers(0, V, n)], 1).astype(np.int32).reshape(-1, 2)
        adj.append(e[np.lexsort((e[:, 1], e[:, 0]))] if n else e)
    indeg = np.zeros((V, T), np.float32)
    for t in range(T):
        np.add.at(indeg[:, t], adj[t][:, 1], 1)
    h0 = rng.normal(0, 0.3, (V, D)).astype(np.float32)
    w = O.init_sparse_weights(p, T, np.random.default_rng(2))
    ref = O.sparse_propagation_np(h0, adj, indeg, w, p, dtype=np.float64)
    got, eng = U.engine_sparse(p, T, w, adj, indeg, h0, precision=PREC, return_engine=True)
    assert "STREAM" in eng.plan
    _check(got, ref, "12 edge types")


def test_dense_binary_adjacency_at_hidden_256_and_weighted_refusal():
    """The dense plug-in at hidden 256: a 0/1 adjacency becomes a CSR and streams; a weighted one has no tensor-core path above
    hidden 128 and says so (it runs on GGNN_PREC_FP32)."""
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    D, T, steps = 256, 4, 2
    mols = synthetic.make_molecules(20, seed=9)
    db = packing.pack_dense_batch(mols, 32, D, T)
    h0 = (db["initial_node_representation"] + np.random.default_rng(2).normal(0, 0.1, db["initial_node_representation"].shape)).astype(np.float32)
    dw = O.init_dense_weights({"hidden_size": D}, T, np.random.default_rng(5))
    dp = {"num_timesteps": steps, "use_edge_bias": True}
    _check(U.engine_dense(dp, T, dw, db["adjacency_matrix"], h0, precision=PREC), O.dense_propagation_loops(h0, db["adjacency_matrix"], dw, dp), "dense D=256")
    weighted = db["adjacency_matrix"] * 0.5
    with pytest.raises(GgnnError, match="weighted dense adjacency"):
        U.engine_dense(dp, T, dw, weighted, h0, precision=PREC)
    got = U.engine_dense(dp, T, dw, weighted, h0, precision="fp32")
    assert U.max_rel_err(got, O.dense_propagation_loops(h0, weighted, dw, dp)) < 1e-4
