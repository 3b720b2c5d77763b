"""GPU: the gradients at EVERY step of real training epochs, against float64 autograd at that step's parameters.

tests/test_gpu_chem_ggnn_gradients.py checks one forward_batch of a fresh model.  Here the plug-ins run what training runs: a training
epoch of several steps, a validation epoch, and a second training epoch, on one engine whose batches differ in size and plan (the
dataset holds two raw graphs of 200+ nodes, so the batches holding one take STREAM on bf16x3 and GLOBAL on fp32; the dataset and the
plans are pinned in tests/test_engine_lifetime_cpu.py).  ``train_step`` is wrapped: before the optimizer's clip and step, every
trainable's gradient is compared with float64 autograd of the same model at the current parameters, with that step's random draws
replayed (state-dropout seed, edge-weight and out-layer weight-dropout masks).  Bars as in that file: fp32 2.5e-5, bf16x3 2e-4, each
variable's scale floored at 1 % of the model's largest gradient; the GCN the same, with 2.5e-5 on fp32.
"""
import re

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import synthetic
from gated_graph_neural_network_samples_b200.utils import SMALL_NUMBER
from tests import gcn_oracle as G
from tests.test_engine_lifetime_cpu import TRAIN_MODEL, training_molecules
from tests.test_gpu_chem_ggnn_gradients import BARS, FLOOR, Draws, _compare, _reference

pytestmark = pytest.mark.gpu

# The GCN: 2.5e-5 on the fp32 kernel; on bf16x3 the bar of the GGNN tensor-core plans, 2e-4 (a few Adam steps into training the readout
# gate's gradient behind the bf16x3 forward measured 3.7e-5)
GCN_BARS = {"fp32": 2.5e-5, "bf16x3": 2e-4}
TRAINING = dict(edge_weight_dropout_keep_prob=0.8, graph_state_dropout_keep_prob=0.9, out_layer_dropout_keep_prob=0.9, task_ids=[0, 1],
                task_sample_ratios={"1": 0.5}, random_seed=3, learning_rate=0.01)


def _two_task_molecules(n=30, seed=9):
    mols = synthetic.make_molecules(n, seed=seed)
    rng = np.random.default_rng(seed)
    return [dict(m, targets=[m["targets"][0], [float(rng.normal())]]) for m in mols]


def _epochs(m):
    """A training epoch, a validation epoch, a second training epoch; returns the numbers of steps of the two training epochs (the
    shuffle of the second may batch the graphs differently)."""
    first = m.run_epoch("train 1", m.train_data, True)[4]
    m.run_epoch("valid", m.valid_data, False)
    return first, m.run_epoch("train 2", m.train_data, True)[4]


def _plan_kind(plan):
    return re.search(r" (LOCAL|GLOBAL|STREAM)\(", plan).group(1)


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_sparse_ggnn_gradients_at_every_training_step(tmp_path, monkeypatch, precision):
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    m = SparseGGNNChemModel({"--log_dir": str(tmp_path), "--precision": precision, "--train_data": training_molecules(),
                             "--valid_data": _two_task_molecules(), "--config": dict(TRAIN_MODEL, **TRAINING)})
    draws = Draws(m, monkeypatch)
    forward_batch, train_step = m.forward_batch, m.train_step
    plans = []

    def fresh_draws_forward(feed):   # Draws holds one forward's draws: one mask per weight
        draws.state.clear()
        draws.weight_masks.clear()
        return forward_batch(feed)

    def checked_train_step(loss):
        import torch
        m.optimizer.zero_grad(set_to_none=True)
        loss.backward(retain_graph=True)   # train_step runs the backward again: a second backward of the same forward
        torch.cuda.synchronize()
        plans.append(m.engine.plan)
        ref, ref_loss = _reference(m, m.feed, draws)
        ref_loss.backward()
        bar = BARS["fp32" if m.engine.plan.startswith("fp32") else precision]
        _compare("training step %d %s" % (len(plans), precision), m, {n: v.grad for n, v in m.trainable_variables()}, ref, bar)
        return train_step(loss)

    m.forward_batch, m.train_step = fresh_draws_forward, checked_train_step
    steps, second = _epochs(m)
    assert steps >= 6 and len(plans) == steps + second, (steps, second, len(plans))
    kinds = [_plan_kind(p) for p in plans[:steps]]
    assert {"LOCAL", "STREAM" if precision == "bf16x3" else "GLOBAL"} <= set(kinds), kinds


def test_dense_ggnn_gradients_at_every_training_step(tmp_path, monkeypatch):
    from gated_graph_neural_network_samples_b200.chem_dense import DenseGGNNChemModel
    cfg = dict(TRAINING, hidden_size=32, num_timesteps=3, batch_size=8)
    m = DenseGGNNChemModel({"--log_dir": str(tmp_path), "--precision": "bf16x3", "--train_data": _two_task_molecules(60, seed=10),
                            "--valid_data": _two_task_molecules(10), "--config": cfg})
    draws = Draws(m, monkeypatch)
    forward_batch, train_step = m.forward_batch, m.train_step
    n = []

    def fresh_draws_forward(feed):
        draws.state.clear()
        draws.weight_masks.clear()
        return forward_batch(feed)

    def checked_train_step(loss):
        import torch
        m.optimizer.zero_grad(set_to_none=True)
        loss.backward(retain_graph=True)
        torch.cuda.synchronize()
        n.append(1)
        ref, ref_loss = _reference(m, m.feed, draws)
        ref_loss.backward()
        _compare("dense training step %d" % len(n), m, {k: v.grad for k, v in m.trainable_variables()}, ref,
                 BARS["fp32" if m.engine.plan.startswith("fp32") else "bf16x3"])
        return train_step(loss)

    m.forward_batch, m.train_step = fresh_draws_forward, checked_train_step
    steps, second = _epochs(m)
    assert steps >= 6 and len(n) == steps + second, (steps, second, len(n))


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_gcn_gradients_at_every_training_step(tmp_path, precision):
    import torch
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    cfg = dict(hidden_size=32, num_timesteps=3, gcn_use_bias=True, batch_size=TRAIN_MODEL["batch_size"], graph_state_dropout_keep_prob=0.9,
               task_ids=[0], random_seed=3, learning_rate=0.01)
    m = SparseGCNChemModel({"--log_dir": str(tmp_path), "--precision": precision, "--train_data": training_molecules(),
                            "--valid_data": _two_task_molecules(), "--config": cfg})
    seeds, plans = [], []
    set_dropout = m.engine.set_state_dropout
    m.engine.set_state_dropout = lambda k, seed=0: (seeds.append((k, seed)), set_dropout(k, seed))
    train_step = m.train_step
    L = cfg["num_timesteps"]
    bar = GCN_BARS[precision]

    def checked_train_step(loss):
        m.optimizer.zero_grad(set_to_none=True)
        loss.backward(retain_graph=True)
        torch.cuda.synchronize()
        plans.append(m.engine.plan)
        feed, (keep, seed) = m.feed, seeds[-1]
        V = feed["initial_node_representation"].shape[0]
        masks = [m.engine.state_dropout_mask(l, keep, seed, V) for l in range(L - 1)] if keep < 1.0 else None
        named = dict(m.trainable_variables())
        ref = {n: v.detach().cpu().double().requires_grad_() for n, v in named.items()}
        ks = [ref["graph_model/gcn_scope/gcn_weights_%d:0" % l] for l in range(L)]
        bs = [ref["graph_model/gcn_scope/gcn_bias_%d:0" % l] for l in range(L)]
        h0 = torch.from_numpy(np.asarray(feed["initial_node_representation"], np.float64))
        adj_w = torch.from_numpy(np.asarray(feed["adjacency_weights"], np.float32)).double()
        final = G.gcn_propagation_torch(h0, feed["adjacency_list"], adj_w, ks, bs, masks, keep)
        wg, bg = ref["out_layer_task0/regression_gate/MLP_W_layer0:0"], ref["out_layer_task0/regression_gate/MLP_b_layer0:0"]
        wt, bt = ref["out_layer_task0/regression/MLP_W_layer0:0"], ref["out_layer_task0/regression/MLP_b_layer0:0"]
        gated = torch.sigmoid(torch.cat([final, h0], 1) @ wg + bg) * (final @ wt + bt)
        gnl = torch.from_numpy(np.asarray(feed["graph_nodes_list"])).long()
        ro = torch.zeros(int(feed["num_graphs"]), 1, dtype=torch.float64).index_add_(0, gnl, gated).squeeze(-1)
        tv = torch.from_numpy(np.asarray(feed["target_values"], np.float64)[0])
        tm = torch.from_numpy(np.asarray(feed["target_mask"], np.float64)[0])
        diff = (ro - tv) * tm
        ((0.5 * diff * diff).sum() / (tm.sum() + SMALL_NUMBER)).backward()
        assert len(named) == 2 * L + 4
        floor = FLOOR * max(float(ref[n].grad.abs().max()) for n in named)
        for n, v in named.items():
            got, r = v.grad.cpu().numpy(), ref[n].grad.numpy()
            err = float(np.max(np.abs(got - r))) / max(float(np.max(np.abs(r))), floor)
            assert err < bar, ("gcn step %d %s" % (len(plans), precision), n, err)
        return train_step(loss)

    m.train_step = checked_train_step
    steps, second = _epochs(m)
    assert steps >= 6 and len(plans) == steps + second, (steps, second, len(plans))
    kinds = [_plan_kind(p) for p in plans[:steps]]
    if precision == "bf16x3":
        assert {"LOCAL", "GLOBAL"} <= set(kinds), kinds
