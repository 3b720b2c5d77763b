"""SparseGCNChemModel on the H100: the plug-in's forward, fused readout, loss and gradients against the reference's own make_model and
float64 autograd, training, checkpoints, prepared graphs from the batch producer thread, and a padded hidden size."""
import json
import os

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import synthetic
from gated_graph_neural_network_samples_b200.utils import SMALL_NUMBER
from tests import gcn_oracle as G
from tests._util import max_rel_err
from tests.test_chem_gcn_cpu import _load_fixture_weights, fixture_feed

pytestmark = pytest.mark.gpu

PLANS = {"bf16x3": "gcn-wgmma-bf16x3 LOCAL", "fp32": "gcn-fp32-ffma"}


def model(tmp_path, precision, mols, n_train, **cfg):
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    return SparseGCNChemModel({"--log_dir": str(tmp_path), "--precision": precision, "--train_data": mols[:n_train],
                               "--valid_data": mols[n_train:], "--config": cfg})


def fixture_model(tmp_path, golden_dir, precision, name):
    z = np.load(os.path.join(golden_dir, "refgraph_gcn_%s.npz" % name))
    cfg = json.loads(str(z["params_json"]))
    m = model(tmp_path, precision, synthetic.make_molecules(8, seed=1), 4, batch_size=100000, **cfg)
    _load_fixture_weights(m, z, cfg)
    return m, z, cfg


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
@pytest.mark.parametrize("name", ["h12_l3", "h100_l4_bias", "h12_l1"])
def test_reference_graph_fixtures_through_the_plugin(tmp_path, golden_dir, precision, name):
    import torch
    m, z, _ = fixture_model(tmp_path, golden_dir, precision, name)
    with torch.no_grad():
        loss, accs = m.forward_batch(fixture_feed(z))
    assert m.engine.plan.startswith(PLANS[precision]), m.engine.plan
    assert max_rel_err(m.ops["final_node_representations"].cpu().numpy(), z["final"]) < 1e-4
    assert max_rel_err(m.output.cpu().numpy(), z["readout"]) < 1e-4
    assert abs(float(loss) - float(z["loss"])) < 1e-4 * abs(float(z["loss"]))
    assert abs(float(accs[0]) - float(z["accuracy"])) < 1e-4 * abs(float(z["accuracy"]))


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
@pytest.mark.parametrize("keep", [1.0, 0.8])
def test_gradients_of_every_trainable_match_float64_autograd(tmp_path, golden_dir, precision, keep):
    """loss.backward() through the fused readout and ggnn_gcn_backward: GCN kernels and biases and both readout MLPs against float64
    autograd of oracle -> readout -> masked loss, with the state-dropout mask regenerated from the seed the plug-in passed to the engine."""
    import torch
    m, z, cfg = fixture_model(tmp_path, golden_dir, precision, "h100_l4_bias")
    seeds = []
    set_dropout = m.engine.set_state_dropout
    m.engine.set_state_dropout = lambda k, seed=0: (seeds.append((k, seed)), set_dropout(k, seed))
    feed = dict(fixture_feed(z), graph_state_keep_prob=keep)
    loss, _ = m.forward_batch(feed)
    loss.backward()
    torch.cuda.synchronize()
    assert seeds[-1][0] == keep
    L, V, D = cfg["num_timesteps"], z["h0"].shape[0], cfg["hidden_size"]
    masks = [m.engine.state_dropout_mask(l, keep, seeds[-1][1], V) for l in range(L - 1)] if keep < 1.0 else None
    named = dict(m.trainable_variables())
    ref = {n: v.detach().cpu().double().requires_grad_() for n, v in named.items()}
    ks = [ref["graph_model/gcn_scope/gcn_weights_%d:0" % l] for l in range(L)]
    bs = [ref["graph_model/gcn_scope/gcn_bias_%d:0" % l] for l in range(L)]
    h0 = torch.from_numpy(z["h0"]).double()
    final = G.gcn_propagation_torch(h0, z["adjacency_list"], torch.from_numpy(z["adjacency_weights_f32"]).double(), ks, bs, masks, keep)
    wg, bg = ref["out_layer_task0/regression_gate/MLP_W_layer0:0"], ref["out_layer_task0/regression_gate/MLP_b_layer0:0"]
    wt, bt = ref["out_layer_task0/regression/MLP_W_layer0:0"], ref["out_layer_task0/regression/MLP_b_layer0:0"]
    gated = torch.sigmoid(torch.cat([final, h0], 1) @ wg + bg) * (final @ wt + bt)
    ro = torch.zeros(int(z["num_graphs"]), 1, dtype=torch.float64).index_add_(0, torch.from_numpy(z["graph_nodes_list"]).long(), gated).squeeze(-1)
    tv, tm = torch.from_numpy(z["target_values"][0]), torch.from_numpy(z["target_mask"][0])
    diff = (ro - tv) * tm
    ((0.5 * diff * diff).sum() / (tm.sum() + SMALL_NUMBER)).backward()
    assert len(named) == 2 * L + 4
    for n, v in named.items():
        assert v.grad is not None, n
        assert max_rel_err(v.grad.cpu().numpy(), ref[n].grad.numpy()) < 2.5e-5, (n, max_rel_err(v.grad.cpu().numpy(), ref[n].grad.numpy()))


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_training_lowers_the_validation_loss_and_a_checkpoint_restores_it(tmp_path, precision):
    mols = synthetic.make_molecules(64, seed=1)
    cfg = dict(hidden_size=16, batch_size=300, num_timesteps=3, learning_rate=0.01, num_epochs=1)
    m = model(tmp_path, precision, mols, 48, **cfg)
    l0 = m.run_epoch("valid0", m.valid_data, False)[0]
    for ep in range(5):
        loss, _, _, _, steps = m.run_epoch("train%d" % ep, m.train_data, True)
        assert steps >= 3 and np.isfinite(loss)
    l1 = m.run_epoch("valid1", m.valid_data, False)[0]
    assert np.isfinite(l1) and l1 < l0
    assert m.engine.plan.startswith(PLANS[precision]), m.engine.plan
    path = str(tmp_path / "ckpt.pickle")
    m.save_progress(path, 5, 1)
    m2 = model(tmp_path, precision, mols, 48, **cfg)
    m2.restore_progress(path)
    assert abs(m2.run_epoch("valid2", m2.valid_data, False)[0] - l1) < 1e-5 * max(1.0, abs(l1))


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_producer_thread_prepared_graphs_match_the_one_call_path(tmp_path, precision):
    """Batches prepared in the ThreadedIterator's producer thread (ggnn_prepare_graph_gcn) against a model that sets every graph inside
    hook 2 (ggnn_set_graph_gcn): the same validation loss, and weights after one training epoch that agree to 1e-6 (not bit for bit: the
    weight-gradient GEMM accumulates with atomics)."""
    mols = synthetic.make_molecules(96, seed=1)
    cfg = dict(hidden_size=32, batch_size=300, num_timesteps=3, gcn_use_bias=True, learning_rate=0.01, num_epochs=1, random_seed=3)

    def make():
        np.random.seed(0)
        return model(tmp_path, precision, mols, 64, **cfg)

    a, b = make(), make()
    b.prepare_graphs_in_producer = False
    feeds = list(a.make_minibatch_iterator(a.valid_data, False))
    assert all(f.get("_prepared_graph") is not None and not f["_prepared_graph"].for_training for f in feeds)
    assert all("_prepared_graph" not in f for f in b.make_minibatch_iterator(b.valid_data, False))
    for (_, va), (_, vb) in zip(a.trainable_variables(), b.trainable_variables()):
        np.testing.assert_array_equal(va.detach().cpu().numpy(), vb.detach().cpu().numpy())
    la, lb = a.run_epoch("valid", a.valid_data, False)[0], b.run_epoch("valid", b.valid_data, False)[0]
    assert abs(la - lb) < 1e-5 * max(1.0, abs(la))
    np.random.seed(5); ta = a.run_epoch("train", a.train_data, True)
    np.random.seed(5); tb = b.run_epoch("train", b.train_data, True)
    assert ta[4] == tb[4] >= 3
    for (n, va), (_, vb) in zip(a.trainable_variables(), b.trainable_variables()):
        x, y = va.detach().cpu().numpy(), vb.detach().cpu().numpy()
        assert float(np.max(np.abs(x - y))) <= 1e-6 * max(1.0, float(np.max(np.abs(y)))), n
    assert len(a._prepared_pool) >= 1


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_padded_hidden_size_matches_the_oracle(tmp_path, precision):
    import torch
    mols = synthetic.make_molecules(40, seed=3)
    m = model(tmp_path, precision, mols, 24, hidden_size=30, batch_size=100000, num_timesteps=3, gcn_use_bias=True)
    assert m._padded_hidden == 32 and m.engine.D == 32
    with torch.no_grad():
        for b in m.weights["edge_biases"]:
            b.uniform_(-0.2, 0.2)
    feed = next(iter(m.make_minibatch_iterator(m.valid_data, False)))
    m.feed = feed
    with torch.no_grad():
        got = m.compute_final_node_representations().cpu().numpy()
    ref = G.gcn_propagation_loops(feed["initial_node_representation"], feed["adjacency_list"], feed["adjacency_weights"].astype(np.float32),
                                  [k.detach().cpu().numpy() for k in m.weights["edge_weights"]],
                                  [b.detach().cpu().numpy() for b in m.weights["edge_biases"]])
    assert got.shape == ref.shape == (feed["initial_node_representation"].shape[0], 30)
    assert max_rel_err(got, ref) < 1e-4, (m.engine.plan, max_rel_err(got, ref))
    assert m.engine.plan.startswith(PLANS[precision]), m.engine.plan
