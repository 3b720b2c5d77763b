"""CPU: hidden sizes 260 .. 512 on the GGNN engine, without a GPU.

* The width limit: 512 is accepted by the host-only prepare calls, 516 is refused with ``hidden_size > 512``, the GCN still refuses 260.
* The plans at 132 SMs (an H100 SXM): the tensor-core precisions stream (``wgmma-* STREAM``) with the K-steps per ring stage each padded
  width implies (DP 272: 1, 288: 2, 320 / 384 / 512: 4, so all six streaming instances run), and fp32, propagation attention and
  CudnnCompatibleGRUCell take the per-timestep fp32 path (``fp32-stepwise``).  A binary dense adjacency lands on both families.  (The
  weighted dense matrix cannot be pinned here: the host-only dense prepare refuses weighted matrices; tests/test_gpu_wide_hidden.py checks
  its plan on the device.)
* The four oracle statements (float64 loops, NumPy, torch, plain C) agree at D = 512, T = 8 with four residual inputs into one layer.
* The sparse and dense plug-ins at hidden 510 run zero-padded to 512 through the stand-in engine.
"""
import re

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import chem_dense, chem_sparse, synthetic
from oracle import ggnn_oracle as O
from tests.test_backward_plans_cpu import component_graph, dense_batch, dense_params, model, sparse_batch
from tests.test_chem_model_cpu import _args, stand_in  # noqa: F401  (stand_in: a fixture)
from tests.test_forward_plans_cpu import instance_of_plan, pad16, stream_ksteps

NUM_SMS = 132
STREAM_WIDTHS = (260, 272, 288, 320, 384, 512)
STEPWISE_WIDTHS = (260, 512)


def host_plan(params, T=4, precision="fp32", batch="mol24", save=False):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    adj, indeg, _ = sparse_batch(batch, params["hidden_size"], T)
    return PreparedGraph.host_only(params, T, adj, indeg, precision=precision, num_sms=NUM_SMS, save_for_backward=save).info()["plan"]


# ---------------------------------------------------------------------------------------------------------------- limits
def test_512_is_accepted_and_516_refused():
    from gated_graph_neural_network_samples_b200.engine import GgnnError, PreparedGraph
    assert host_plan(model("GRU", 512)).startswith("fp32-stepwise ")
    for prec in ("fp32", "bf16x3"):
        with pytest.raises(GgnnError, match=r"hidden_size > 512 is not supported"):
            host_plan(model("GRU", 516), precision=prec)
    rng = np.random.default_rng(0)
    lst = rng.integers(0, 20, (40, 2))
    with pytest.raises(GgnnError, match=r"hidden_size > 256 is not supported"):
        PreparedGraph.host_only_gcn(260, 2, 20, lst, np.ones(40, np.float32), precision="fp32", num_sms=NUM_SMS)


# ---------------------------------------------------------------------------------------------------------------- plans
@pytest.mark.parametrize("D", STREAM_WIDTHS)
@pytest.mark.parametrize("precision", ("bf16x3", "bf16"))
@pytest.mark.parametrize("cell", ("GRU", "RNN"))
def test_tensor_core_precisions_stream(D, precision, cell):
    DP = pad16(D)
    plan = host_plan(model(cell, D, act="tanh"), precision=precision, save=True)
    blocks = lambda w: (w + 127) // 128
    assert re.match(r"^wgmma-%s STREAM\(3 launches per step: .*\) tiles=\d+ DP=%d N-blocks agg/cand=%dx128 gate=%dx128$"
                    % (precision, DP, blocks(DP), blocks(2 * DP)), plan), plan
    ks = {272: 1, 288: 2, 320: 4, 384: 4, 512: 4}[DP]
    assert stream_ksteps(DP, {}) == ks
    assert instance_of_plan(plan, {}) == ("stream", precision == "bf16x3", ks)


STEPWISE_MODELS = {   # name: (params at hidden D, launches per step)
    "gru": (lambda D: model("GRU", D, act="tanh", avg=True), 7),
    "rnn": (lambda D: model("RNN", D, act="ReLU"), 5),
    "cudnn": (lambda D: model("CudnnCompatibleGRUCell", D, act="tanh"), 8),
    "attention": (lambda D: model("GRU", D, act="tanh", attention=True), 8),
    "attention-rnn": (lambda D: model("RNN", D, act="tanh", attention=True), 6),
}


@pytest.mark.parametrize("D", STEPWISE_WIDTHS)
@pytest.mark.parametrize("name", sorted(STEPWISE_MODELS))
def test_fp32_attention_and_cudnn_run_stepwise(name, D):
    """fp32 at any cell, and attention / CudnnCompatibleGRUCell at every precision (the engine moves them onto fp32)."""
    make, launches = STEPWISE_MODELS[name]
    p = make(D)
    tag = ("+attention" if p["use_propagation_attention"] else "") + ("+cudnn-gru" if p["graph_rnn_cell"] != "GRU" and p["graph_rnn_cell"] != "RNN" else "")
    for prec in ("fp32", "bf16x3") if tag else ("fp32",):
        plan = host_plan(p, precision=prec, save=True)
        adj, indeg, _ = sparse_batch("mol24", D, 4)
        assert plan == "fp32-stepwise%s (%d launches per step) V=%d D=%d T=4" % (tag, launches, indeg.shape[0], D), plan


def test_plans_up_to_256_are_not_stepwise():
    assert host_plan(model("GRU", 256, act="tanh")).startswith("fp32-ffma LOCAL(")
    assert host_plan(model("GRU", 256, act="tanh"), precision="bf16x3").startswith("wgmma-bf16x3 STREAM(")


@pytest.mark.parametrize("precision,pattern", [("fp32", r"^fp32-stepwise \(7 launches per step\) V=\d+ D=512 T=4 \[binary dense adjacency -> CSR\]$"),
                                               ("bf16x3", r"^wgmma-bf16x3 STREAM\(.* DP=512 .*\[binary dense adjacency -> CSR\]$")])
def test_binary_dense_matrix_on_both_families(precision, pattern):
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    A, _ = dense_batch(512, False)
    plan = PreparedGraph.host_only_dense(dense_params(512), 4, A, precision=precision, num_sms=NUM_SMS, save_for_backward=True).info()["plan"]
    assert re.match(pattern, plan), plan


def test_a_10k_node_component_and_an_empty_batch_plan_stepwise():
    from gated_graph_neural_network_samples_b200.engine import PreparedGraph
    rng = np.random.default_rng(1)
    V = 10000
    chain = np.stack([np.arange(V - 1), np.arange(1, V)], 1)
    extra = rng.integers(0, V, (5000, 2))
    adj = [np.concatenate([chain, chain[:, ::-1]]).astype(np.int32), extra.astype(np.int32)]
    indeg = np.zeros((V, 2), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    g = PreparedGraph.host_only(model("GRU", 512), 2, adj, indeg, num_sms=NUM_SMS, save_for_backward=True)
    assert g.info()["plan"] == "fp32-stepwise (7 launches per step) V=10000 D=512 T=2"
    empty = PreparedGraph.host_only(model("GRU", 512), 2, [np.zeros((0, 2), np.int32)] * 2, np.zeros((0, 2), np.float32), num_sms=NUM_SMS)
    assert empty.info()["plan"] == "fp32-stepwise (7 launches per step) V=0 D=512 T=2"


# ---------------------------------------------------------------------------------------------------------------- oracle
def test_oracle_statements_agree_at_512():
    import torch
    from oracle import c_oracle
    T, D = 8, 512
    p = model("GRU", D, layer_timesteps=(1, 1, 1, 2), residual_connections={"3": [0, 1, 2, 3]}, act="tanh", avg=True)
    adj, indeg = component_graph(T, V_target=40, seed=11)
    h0 = np.random.default_rng(4).normal(0, 1, (indeg.shape[0], D))
    w = O.init_sparse_weights(p, T, np.random.default_rng(5))
    loops = O.sparse_propagation_loops(h0, adj, indeg, w, p, dtype=np.float64, return_all_layers=True)
    vec = O.sparse_propagation_np(h0, adj, indeg, w, p, dtype=np.float64, return_all_layers=True)
    tor = O.sparse_propagation_torch(h0, adj, indeg, w, p, dtype=torch.float64, return_all_layers=True)
    c = c_oracle.sparse_propagation_c(h0, adj, indeg, w, p)
    for l, (a, b, t) in enumerate(zip(loops, vec, tor)):
        scale = max(np.max(np.abs(a)), 1e-30)
        assert np.max(np.abs(a - b)) / scale < 1e-12, l
        assert np.max(np.abs(a - t.numpy())) / scale < 1e-12, l
    assert np.max(np.abs(loops[-1] - c)) / np.max(np.abs(loops[-1])) < 1e-12


# ---------------------------------------------------------------------------------------------------------------- plug-ins
def test_sparse_plugin_at_hidden_510_runs_padded_to_512(tmp_path, stand_in):  # noqa: F811
    import torch
    mols = synthetic.make_molecules(56, seed=3)
    m = chem_sparse.SparseGGNNChemModel(_args(tmp_path, mols, hidden_size=510, batch_size=150, edge_weight_dropout_keep_prob=1.0,
                                              graph_state_dropout_keep_prob=1.0, num_epochs=1))
    assert m._padded_hidden == 512 and m.engine.D == 512
    feed = next(iter(m.make_minibatch_iterator(m.valid_data, False)))
    m.feed = feed
    with torch.no_grad():
        got = m.compute_final_node_representations().numpy()
    assert got.shape[1] == 510
    weights = []
    for l in range(len(m.params["layer_timesteps"])):
        w = {"edge_weights": m.gnn_weights.edge_weights[l].detach().numpy().reshape(m.num_edge_types, 510, 510),
             "edge_biases": m.gnn_weights.edge_biases[l].detach().numpy()}
        w.update({k: v.detach().numpy() for k, v in m.gnn_weights.rnn_cells[l].items()})
        weights.append(w)
    ref = O.sparse_propagation_np(feed["initial_node_representation"], [feed[k] for k in m.placeholders["adjacency_lists"]],
                                  feed["num_incoming_edges_per_type"], weights, m.params, dtype=np.float64)
    np.testing.assert_allclose(got, ref, rtol=2e-5, atol=2e-6)
    train_loss = m.run_epoch("train", m.train_data, True)[0]
    assert np.isfinite(train_loss)
    assert tuple(m.gnn_weights.edge_weights[0].shape) == (m.num_edge_types * 510, 510)


def test_dense_plugin_at_hidden_510_runs_padded_to_512(tmp_path, stand_in):  # noqa: F811
    import torch
    mols = synthetic.make_molecules(24, seed=4)
    args = {"--log_dir": str(tmp_path), "--device": "cpu", "--train_data": mols[:16], "--valid_data": mols[16:],
            "--config": {"hidden_size": 510, "batch_size": 4, "num_timesteps": 2, "learning_rate": 0.01, "num_epochs": 1}}
    m = chem_dense.DenseGGNNChemModel(args)
    assert m._padded_hidden == 512 and m.engine.D == 512
    feed = next(iter(m.make_minibatch_iterator(m.valid_data, False)))
    m.feed = feed
    with torch.no_grad():
        got = m.compute_final_node_representations().numpy()
    w = {"edge_weights": m.weights["edge_weights"].detach().numpy(), "edge_biases": m.weights["edge_biases"].detach().numpy()}
    w.update({k: v.detach().numpy() for k, v in m.weights["node_gru"].items()})
    ref = O.dense_propagation_loops(feed["initial_node_representation"], feed["adjacency_matrix"], w, {"num_timesteps": 2, "use_edge_bias": True})
    assert got.shape == ref.shape and got.shape[-1] == 510
    np.testing.assert_allclose(got, ref, rtol=2e-5, atol=2e-6)
    assert np.isfinite(m.run_epoch("train", m.train_data, True)[0])
