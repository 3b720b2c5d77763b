"""GPU: the gradients the two GGNN plug-ins hand to the optimizer, against float64 autograd of the same model.

What trains is ``ChemModel.forward_batch`` -> ``loss.backward()``: the plug-in's glue around the checked kernels -- the flat weight layout
handed to ``ggnn_backward`` and the gradients mapped back to the variables, CudnnCompatibleGRUCell's stacked candidate kernel, the
edge-weight dropout drawn in torch (sparse: one mask per layer; dense: the state keep fed into the weight slot, dense:222), state dropout
seeded per run, zero padding of hidden sizes that are not multiples of 4 (the torch readout), the dense [T, 1, D] bias view and masked
fused readout, the out-layer weight dropout and the multi-task masked loss, and the data-parallel path ``reduce_gradients``.  Every case
compares EVERY trainable's gradient with float64 autograd of oracle propagation -> ``gated_regression_torch`` -> the loss of
chem_tensorflow.py:161-170, with the random parts reproduced: the state-dropout seed the plug-in passed to the engine, and the weight-
dropout masks the plug-in drew (``output != 0`` of each ``torch.nn.functional.dropout`` call, scaled by 1/keep in float64).  Each case
also asserts the plan text, so that it stays on the kernel family it was written for.

Bars (max|err| / max|ref| per variable): 2.5e-5 on the fp32 kernels, 2e-4 on the bf16x3 tensor-core plans.  The bf16x3 cases use tanh:
ReLU's kink makes float64 and the engine take opposite sides of 0 at some nodes (tests/test_backward_plans_cpu.py,
smooth_on_tensor_cores)."""
import json
import os
import re

import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import synthetic
from gated_graph_neural_network_samples_b200.utils import SMALL_NUMBER
from oracle import ggnn_oracle as O
from tests import _util as U

pytestmark = pytest.mark.gpu

BARS = {"fp32": 2.5e-5, "bf16x3": 2e-4}
# A variable whose gradient is far below the model's largest is a sum with cancellation: on the training batch the task-1 gate bias is
# 1e-4 of the largest gradient, and fp32 rounding alone (the plug-in's Python around an oracle-backed fp32 engine) puts it 1e-4 off
# relative to itself.  So each variable's error is taken relative to max(max|its ref|, FLOOR * max|ref| over all variables).
FLOOR = 1e-2
FFMA = r"^fp32-ffma[ +]"
TC_LOCAL = r"^wgmma-bf16x3 LOCAL\("
TC_STREAM = r"^wgmma-bf16x3 STREAM\("


# ---------------------------------------------------------------------------------------------------------------- models and feeds
def _sparse_model(tmp_path, precision, mols, **cfg):
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    return SparseGGNNChemModel({"--log_dir": str(tmp_path), "--precision": precision, "--train_data": mols[:48], "--valid_data": mols[48:],
                                "--config": cfg})


def _dense_model(tmp_path, precision, mols, **cfg):
    from gated_graph_neural_network_samples_b200.chem_dense import DenseGGNNChemModel
    return DenseGGNNChemModel({"--log_dir": str(tmp_path), "--precision": precision, "--train_data": mols[:48], "--valid_data": mols[48:],
                               "--config": cfg})


def _two_task_molecules(n, seed, T=4):
    mols = synthetic.make_molecules(n, seed=seed, num_bond_types=T)
    rng = np.random.default_rng(seed)
    return [dict(mol, targets=[mol["targets"][0], [float(rng.normal())]]) for mol in mols]


# the training settings: edge-weight, state and out-layer dropout on, two tasks, task 1 labelled on half of the training graphs (its ratio
# is looked up with the int task id in the loss, chem_tensorflow.py:168, so it drops labels without rescaling the loss)
TRAINING = dict(edge_weight_dropout_keep_prob=0.8, graph_state_dropout_keep_prob=0.9, out_layer_dropout_keep_prob=0.9, task_ids=[0, 1],
                task_sample_ratios={"1": 0.5}, random_seed=3)
SPARSE_TRAINING = dict(TRAINING, hidden_size=32, layer_timesteps=[2, 1], residual_connections={"1": [0]}, use_edge_bias=True, batch_size=400)
DENSE_TRAINING = dict(TRAINING, hidden_size=32, num_timesteps=3, batch_size=8, graph_state_dropout_keep_prob=0.9)


def _training_feed(m):
    """The first training batch as run_epoch gets it: the graph prepared with save=True by the batch iterator, the dropout keeps set."""
    feed = next(iter(m.make_minibatch_iterator(m.train_data, True)))
    assert feed["_prepared_graph"].for_training
    feed["out_layer_dropout_keep_prob"] = m.params["out_layer_dropout_keep_prob"]
    tm = np.asarray(feed["target_mask"])
    assert tm.shape[0] == 2 and tm[0].all() and 0 < tm[1].sum() < tm.shape[1], tm    # task 1 has unlabelled graphs in the batch
    return feed


def _load_sparse_weights(m, layers, z):
    """Fixture weights (oracle keys per layer) into the plug-in's variables; CudnnCompatibleGRUCell's stacked candidate kernel is split
    into its input and hidden projections."""
    import torch
    T, D = m.num_edge_types, m.params["hidden_size"]
    g = m.gnn_weights
    f32 = lambda a: torch.from_numpy(np.asarray(a, np.float32))
    with torch.no_grad():
        for l, lw in enumerate(layers):
            cell = g.rnn_cells[l]
            for k, a in lw.items():
                if k == "edge_weights":
                    g.edge_weights[l].copy_(f32(a).reshape(T * D, D))
                elif k == "edge_biases":
                    g.edge_biases[l].copy_(f32(a))
                elif k == "edge_type_attention_weights":
                    g.edge_type_attention_weights[l].copy_(f32(a))
                elif k == "cand_kernel" and "cand_input_kernel" in cell:
                    din = cell["cand_input_kernel"].shape[0]
                    cell["cand_input_kernel"].copy_(f32(a)[:din])
                    cell["cand_hidden_kernel"].copy_(f32(a)[din:])
                else:
                    cell[{"rnn_kernel": "cand_kernel", "rnn_bias": "cand_bias"}.get(k, k)].copy_(f32(a))
        _load_readout(m, z)


def _load_readout(m, z):
    import torch
    gate, trans = m.weights["regression_gate_task0"], m.weights["regression_transform_task0"]
    for t, k in ((gate.weights[0], "ro_w_gate"), (gate.biases[0], "ro_b_gate"), (trans.weights[0], "ro_w_trans"), (trans.biases[0], "ro_b_trans")):
        with torch.no_grad():
            t.copy_(torch.from_numpy(np.asarray(z[k], np.float32)))


def _targets(z, num_graphs):
    """The fixture's targets; the BASELINE-width fixtures carry none, so those get seeded targets with every label present."""
    if "target_values" in z.files:
        return z["target_values"], z["target_mask"]
    return np.random.default_rng(11).normal(size=(1, num_graphs)), np.ones((1, num_graphs))


def _sparse_fixture(tmp_path, golden_dir, name, precision):
    if name in ("cfg2_shape", "cfg4_shape"):
        z, p, layers, adj, T = U.load_refgraph_wide(golden_dir, name)
    else:
        z = np.load(os.path.join(golden_dir, "refgraph_sparse_%s.npz" % name))
        p = json.loads(str(z["params_json"]))
        layers = [{k[len("w%d_" % l):]: z[k] for k in z.files if k.startswith("w%d_" % l)} for l in range(len(p["layer_timesteps"]))]
        T = 4
        adj = [z["adj%d" % e] for e in range(T)]
    m = _sparse_model(tmp_path, precision, synthetic.make_molecules(56, seed=1, num_bond_types=T), **dict(p, batch_size=100000))
    assert m.num_edge_types == T
    _load_sparse_weights(m, layers, z)
    tv, tm = _targets(z, int(z["num_graphs"]))
    feed = {"initial_node_representation": z["h0"].astype(np.float32), "num_incoming_edges_per_type": z["indeg"].astype(np.float32),
            "graph_nodes_list": z["graph_nodes_list"], "num_graphs": int(z["num_graphs"]), "target_values": tv, "target_mask": tm,
            "graph_state_keep_prob": 1.0, "edge_weight_dropout_keep_prob": 1.0, "out_layer_dropout_keep_prob": 1.0}
    for e in range(T):
        feed["adjacency_e%d" % e] = adj[e]
    return m, z, feed


def _dense_fixture(tmp_path, golden_dir, name, precision):
    import torch
    z = np.load(os.path.join(golden_dir, "%s.npz" % name))
    p = json.loads(str(z["params_json"]))
    m = _dense_model(tmp_path, precision, synthetic.make_molecules(56, seed=1), **dict(p, batch_size=8))
    assert m.num_edge_types == 4
    with torch.no_grad():
        m.weights["edge_weights"].copy_(torch.from_numpy(z["w_edge_weights"].astype(np.float32)))
        m.weights["edge_biases"].copy_(torch.from_numpy(z["w_edge_biases"].astype(np.float32)))
        for k, t in m.weights["node_gru"].items():
            t.copy_(torch.from_numpy(z["w_" + k].astype(np.float32)))
    _load_readout(m, z)
    b, v = z["h0"].shape[:2]
    tv, tm = _targets(z, b)
    feed = {"initial_node_representation": z["h0"].astype(np.float32), "adjacency_matrix": z["adj"].astype(np.float32),
            "node_mask": z["node_mask"].astype(np.float32), "num_vertices": v, "num_graphs": b, "target_values": tv, "target_mask": tm,
            "graph_state_keep_prob": 1.0, "edge_weight_dropout_keep_prob": 1.0, "out_layer_dropout_keep_prob": 1.0}
    return m, z, feed


# ---------------------------------------------------------------------------------------------------------------- the random parts
class Draws:
    """What the plug-in drew in one forward: the (keep, seed) it handed to ``engine.set_state_dropout``, and per weight-dropout call the
    input's storage and the kept positions of the output."""

    def __init__(self, m, monkeypatch):
        import torch
        self.state, self.weight_masks = [], {}
        set_state_dropout = m.engine.set_state_dropout

        def recording_set_state_dropout(keep, seed=0):
            self.state.append((keep, seed))
            return set_state_dropout(keep, seed)

        m.engine.set_state_dropout = recording_set_state_dropout
        dropout = torch.nn.functional.dropout

        def recording_dropout(input, p=0.5, training=True, inplace=False):
            out = dropout(input, p=p, training=training, inplace=inplace)
            assert input.data_ptr() not in self.weight_masks, "one weight dropped twice in one forward"
            self.weight_masks[input.data_ptr()] = ((out != 0).detach().cpu().double(), 1.0 - p)
            return out

        monkeypatch.setattr(torch.nn.functional, "dropout", recording_dropout)

    def weight(self, var, ref):
        """``ref`` (the float64 copy of ``var``) with the mask the plug-in drew for ``var`` applied, if it drew one."""
        drawn = self.weight_masks.get(var.data_ptr())
        if drawn is None:
            return ref
        mask, keep = drawn
        return ref * mask.reshape(ref.shape) / keep

    def state_dropout(self):
        keep, seed = self.state[-1]
        return (keep, seed) if keep < 1.0 else None


# ---------------------------------------------------------------------------------------------------------------- the float64 model
def _loss(m, feed, draws, R, readout):
    """chem_tensorflow.py:161-170 in float64: per task the masked squared error over (mask sum + 1e-7), times 1 / ratio with the
    reference's int-key lookup of task_sample_ratios, summed over tasks."""
    import torch
    tv = torch.as_tensor(np.asarray(feed["target_values"], np.float64))
    tm = torch.as_tensor(np.asarray(feed["target_mask"], np.float64))
    total = 0.0
    for i, task_id in enumerate(m.params["task_ids"]):
        gate, trans = m.weights["regression_gate_task%i" % task_id], m.weights["regression_transform_task%i" % task_id]
        computed = readout(draws.weight(gate.weights[0], R[id(gate.weights[0])]), R[id(gate.biases[0])],
                           draws.weight(trans.weights[0], R[id(trans.weights[0])]), R[id(trans.biases[0])])
        diff = (computed - tv[i]) * tm[i]
        task_loss = (0.5 * diff * diff).sum() / (tm[i].sum() + SMALL_NUMBER)
        total = total + task_loss * (1.0 / (m.params["task_sample_ratios"].get(task_id) or 1.0))
    return total


def _reference(m, feed, draws):
    """(float64 leaves by variable name, float64 loss) of the plug-in's model on ``feed`` with the plug-in's draws."""
    import torch
    named = m.trainable_variables()
    ref = {n: v.detach().cpu().double().requires_grad_() for n, v in named}
    R = {id(v): ref[n] for n, v in named}
    T, D, DP = m.num_edge_types, m.params["hidden_size"], m._padded_hidden
    h0 = torch.from_numpy(np.asarray(feed["initial_node_representation"], np.float64))
    if hasattr(m, "gnn_weights"):
        g, layers = m.gnn_weights, []
        rnn = m.params["graph_rnn_cell"].lower() == "rnn"
        for l in range(len(m.params["layer_timesteps"])):
            w = {"edge_weights": draws.weight(g.edge_weights[l], R[id(g.edge_weights[l])]).reshape(T, D, D)}
            if m.params["use_edge_bias"]:
                w["edge_biases"] = R[id(g.edge_biases[l])]
            if m.params["use_propagation_attention"]:
                w["edge_type_attention_weights"] = R[id(g.edge_type_attention_weights[l])]
            cell = {k: R[id(v)] for k, v in g.rnn_cells[l].items()}
            if "cand_input_kernel" in cell:
                cell["cand_kernel"] = torch.cat([cell.pop("cand_input_kernel"), cell.pop("cand_hidden_kernel")], dim=0)
            w.update({({"cand_kernel": "rnn_kernel", "cand_bias": "rnn_bias"}.get(k, k) if rnn else k): v for k, v in cell.items()})
            layers.append(w)
        adj = [feed[k] for k in m.placeholders["adjacency_lists"]]
        final = O.sparse_propagation_torch(h0, adj, feed["num_incoming_edges_per_type"], layers, m.params, dtype=torch.float64,
                                           state_dropout=draws.state_dropout(), mask_width=DP)
        readout = lambda wg, bg, wt, bt: O.gated_regression_torch(final, h0, wg, bg, wt, bt, graph_nodes_list=feed["graph_nodes_list"],
                                                                  num_graphs=feed["num_graphs"], dtype=torch.float64)
    else:
        w = {"edge_weights": draws.weight(m.weights["edge_weights"], R[id(m.weights["edge_weights"])])}
        if "edge_biases" in m.weights:
            w["edge_biases"] = R[id(m.weights["edge_biases"])]
        w.update({k: R[id(v)] for k, v in m.weights["node_gru"].items()})
        final = O.dense_propagation_torch(h0, feed["adjacency_matrix"], w, {"num_timesteps": m.params["num_timesteps"],
                                                                             "use_edge_bias": "edge_biases" in w},
                                          dtype=torch.float64, state_dropout=draws.state_dropout(), mask_width=DP)
        readout = lambda wg, bg, wt, bt: O.gated_regression_torch(final, h0, wg, bg, wt, bt, node_mask=feed["node_mask"], dtype=torch.float64)
    return ref, _loss(m, feed, draws, R, readout)


def _expected_variable_count(p, dense):
    per_task = 4 * len(p["task_ids"])       # gate and transform: one weight, one bias each
    if dense:
        return 1 + int(p["use_edge_bias"]) + 4 + per_task
    cell = {"gru": 4, "rnn": 2, "cudnncompatiblegrucell": 6}[p["graph_rnn_cell"].lower()]
    return len(p["layer_timesteps"]) * (1 + int(p["use_edge_bias"]) + int(p["use_propagation_attention"]) + cell) + per_task


def _compare(tag, m, grads, ref, bar):
    """Every trainable's gradient (``grads``: name -> CUDA tensor) against float64 autograd; prints the worst variable."""
    named = m.trainable_variables()
    assert len(named) == _expected_variable_count(m.params, not hasattr(m, "gnn_weights")), [n for n, _ in named]
    refs = {n: np.zeros(tuple(v.shape)) if ref[n].grad is None else ref[n].grad.numpy().reshape(tuple(v.shape)) for n, v in named}
    floor = FLOOR * max(float(np.max(np.abs(r))) for r in refs.values())
    errs = []
    for n, _ in named:
        assert grads[n] is not None, "%s: no gradient for %s" % (tag, n)
        got, r = grads[n].detach().cpu().numpy(), refs[n]
        errs.append((float(np.max(np.abs(got - r))) / max(float(np.max(np.abs(r))), floor), n))
    worst = max(errs)
    print("\n%-40s [%s] worst gradient %.2e on %s" % (tag, m.engine.plan[:32], worst[0], worst[1]))
    bad = [(n, e) for e, n in errs if not e < bar]
    assert not bad, (tag, bar, bad)


def _check(tag, m, feed, monkeypatch, plan, precision):
    """forward_batch + loss.backward() through the plug-in, then every gradient against float64 autograd.  Returns the model's loss and
    the reference loss."""
    import torch
    draws = Draws(m, monkeypatch)
    loss, _ = m.forward_batch(feed)
    loss.backward()
    torch.cuda.synchronize()
    assert re.search(plan, m.engine.plan), (plan, m.engine.plan)
    ref, ref_loss = _reference(m, feed, draws)
    ref_loss.backward()
    loss, ref_loss = float(loss.detach()), float(ref_loss.detach())
    assert abs(loss - ref_loss) <= 1e-4 * abs(ref_loss), (loss, ref_loss)
    bar = BARS["fp32" if m.engine.plan.startswith("fp32") else precision]     # the fp32 kernel serves attention and CudnnCompatibleGRUCell at every precision
    _compare(tag, m, {n: v.grad for n, v in m.trainable_variables()}, ref, bar)
    return loss


# ---------------------------------------------------------------------------------------------------------------- reference fixtures
@pytest.mark.parametrize("name,precision,plan", [
    ("true_default_shape", "fp32", FFMA), ("true_default_shape", "bf16x3", TC_LOCAL),
    ("rnn_relu_bias_sum", "fp32", FFMA),
    ("attention_bias_avg", "fp32", r"^fp32-ffma\+attention"), ("attention_bias_avg", "bf16x3", r"^fp32-ffma\+attention"),
    ("cudnn_gru", "fp32", r"^fp32-ffma\+cudnn-gru"), ("cudnn_gru", "bf16x3", r"^fp32-ffma\+cudnn-gru"),
    ("cfg2_shape", "bf16x3", TC_LOCAL), ("cfg4_shape", "bf16x3", TC_STREAM)])
def test_sparse_reference_fixtures_through_the_plugin(tmp_path, golden_dir, monkeypatch, name, precision, plan):
    """The reference graph code's fixtures with their weights loaded into the plug-in: the loss anchors the forward to the fixture, the
    gradients of every trainable are checked.  Attention and CudnnCompatibleGRUCell run on the fp32 kernel at every precision."""
    m, z, feed = _sparse_fixture(tmp_path, golden_dir, name, precision)
    loss = _check("refgraph %s %s" % (name, precision), m, feed, monkeypatch, plan, precision)
    if "target_values" in z.files:
        assert abs(loss - float(z["loss"])) < 1e-4 * abs(float(z["loss"])), (loss, float(z["loss"]))
    else:
        assert U.max_rel_err(m.output.detach().cpu().numpy(), z["readout"]) < 1e-4


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
@pytest.mark.parametrize("name", ["refgraph_dense", "refgraph_dense_cfg3_shape"])
def test_dense_reference_fixtures_through_the_plugin(tmp_path, golden_dir, monkeypatch, name, precision):
    """The dense fixtures: [T, 1, D] bias view, fused masked readout."""
    m, z, feed = _dense_fixture(tmp_path, golden_dir, name, precision)
    loss = _check("%s %s" % (name, precision), m, feed, monkeypatch, FFMA if precision == "fp32" else TC_LOCAL, precision)
    if "target_values" in z.files:
        assert abs(loss - float(z["loss"])) < 1e-4 * abs(float(z["loss"])), (loss, float(z["loss"]))
    else:
        assert U.max_rel_err(m.output.detach().cpu().numpy(), z["readout"]) < 1e-4


# ---------------------------------------------------------------------------------------------------------------- training feeds
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_sparse_gru_training_batch(tmp_path, monkeypatch, precision):
    """Edge-weight dropout 0.8 (one mask per layer), state dropout 0.9, out-layer weight dropout 0.9, two tasks with missing labels, the
    graph prepared by the batch iterator."""
    m = _sparse_model(tmp_path, precision, _two_task_molecules(64, seed=1), **SPARSE_TRAINING)
    _check("sparse gru training %s" % precision, m, _training_feed(m), monkeypatch, FFMA if precision == "fp32" else TC_LOCAL, precision)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_dense_training_batch(tmp_path, monkeypatch, precision):
    """The dense plug-in at keep 0.9: the state keep drives both the state dropout and the edge-weight dropout (dense:222)."""
    m = _dense_model(tmp_path, precision, _two_task_molecules(64, seed=2), **DENSE_TRAINING)
    _check("dense training %s" % precision, m, _training_feed(m), monkeypatch, FFMA if precision == "fp32" else TC_LOCAL, precision)


# ---------------------------------------------------------------------------------------------------------------- padded hidden sizes
@pytest.mark.parametrize("cfg,precision,plan", [
    (dict(hidden_size=30), "fp32", FFMA), (dict(hidden_size=30), "bf16x3", TC_LOCAL),
    (dict(hidden_size=10, graph_rnn_cell="RNN", graph_rnn_activation="tanh"), "fp32", FFMA)], ids=["gru30-fp32", "gru30-bf16x3", "rnn10-fp32"])
def test_sparse_padded_hidden_size_training_batch(tmp_path, monkeypatch, cfg, precision, plan):
    """Zero-padded to the next multiple of 4 at the engine boundary, the torch readout; the state-dropout mask is drawn at the padded
    width."""
    m = _sparse_model(tmp_path, precision, _two_task_molecules(64, seed=1), **dict(SPARSE_TRAINING, **cfg))
    assert m._padded_hidden != m.params["hidden_size"]
    _check("sparse padded %s %s" % (cfg, precision), m, _training_feed(m), monkeypatch, plan, precision)


def test_dense_padded_hidden_size_training_batch(tmp_path, monkeypatch):
    m = _dense_model(tmp_path, "fp32", _two_task_molecules(64, seed=2), **dict(DENSE_TRAINING, hidden_size=10))
    assert m._padded_hidden == 12
    _check("dense padded 10 fp32", m, _training_feed(m), monkeypatch, FFMA, "fp32")


# ---------------------------------------------------------------------------------------------------------------- data-parallel path
def test_reduce_gradients_at_world_size_one_matches_loss_backward_and_float64(tmp_path, monkeypatch):
    """``reduce_gradients`` back-propagates each task's numerator separately through the same engine forward and fused readout
    (retain_graph) into FlatGradients views and divides by the mask sums; the all-reduce is a no-op at world size 1.  It must give the
    gradients of loss.backward() and of float64 autograd."""
    import torch
    m = _sparse_model(tmp_path, "fp32", _two_task_molecules(64, seed=1), **SPARSE_TRAINING)
    feed = _training_feed(m)
    draws = Draws(m, monkeypatch)
    loss, _ = m.forward_batch(feed)
    loss.backward(retain_graph=True)
    direct = {n: v.grad.clone() for n, v in m.trainable_variables()}
    for _, v in m.trainable_variables():
        v.grad = None
    assert m.reduce_gradients() == 1
    torch.cuda.synchronize()
    reduced = {n: v.grad for n, v in m.trainable_variables()}
    for n in direct:
        assert reduced[n] is not None and reduced[n].data_ptr() != direct[n].data_ptr(), n
        err = U.max_rel_err(reduced[n].cpu().numpy(), direct[n].cpu().numpy())
        assert err < 1e-6, (n, err)
    ref, ref_loss = _reference(m, feed, draws)
    ref_loss.backward()
    _compare("reduce_gradients fp32", m, reduced, ref, BARS["fp32"])
