"""GPU: CudnnCompatibleGRUCell on the streaming wgmma kernels (GGNN_CELL_CUDNN_GRU_TENSOR_CORES), forward and every gradient against float64.

The cell applies the reset gate after the recurrent product, ``c = tanh(x.K_in + b_in + r*(h.K_hid + b_hid))``; on the streaming plan a
timestep is the gather-GEMM, the gate GEMM, the hidden-projection GEMM (q = h.K_hid + b_hid, then r*q) and the candidate GEMM over
[res.. | agg].  Each case runs a forward with save_for_backward and ``ggnn_backward`` on an engine created with
``cudnn_gru_tensor_cores=True`` and compares the forward and every ``node_states_per_layer`` entry with float64, and ``d h0`` and every
weight gradient of every layer, ``cand_hidden_bias`` included, with float64 autograd of ``oracle.sparse_propagation_torch``.  Bars,
max|err| / max|ref| per tensor: bf16x3 1e-4 forward and 2e-4 gradients, bf16 2e-2 forward (the bars of the other streaming tests).
"""
import json
import os
import pickle

import numpy as np
import pytest

from oracle import ggnn_oracle as O
from tests import _util as U
from tests.test_gpu_backward import _autograd_reference

pytestmark = pytest.mark.gpu

CELL = "CudnnCompatibleGRUCell"
BARS = {"bf16x3": (1e-4, 2e-4), "bf16": (2e-2, 2e-2)}
STREAM = "wgmma-%s STREAM+cudnn-gru(4 launches per step"
DROP_SEED = 4321


def cudnn_model(D, layer_timesteps=(2, 1), residual_connections=None, bias=True, avg=True, attention=False):
    return {"hidden_size": D, "layer_timesteps": list(layer_timesteps),
            "residual_connections": {"1": [0]} if residual_connections is None else residual_connections,
            "use_edge_bias": bias, "use_edge_msg_avg_aggregation": avg, "graph_rnn_cell": CELL, "graph_rnn_activation": "tanh",
            "use_propagation_attention": attention}


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _rel(got, ref):
    return U.max_rel_err(got, ref)


class Run:
    """One engine with CudnnCompatibleGRUCell at the configured precision, its weights bound and save_for_backward on."""

    def __init__(self, params, T, w, precision="bf16x3", bwd_precision=None, det=False, keep=1.0, attention=False):
        from gated_graph_neural_network_samples_b200.engine import PropagationEngine
        self.eng = PropagationEngine(params, T, precision=precision, cudnn_gru_tensor_cores=True, attention_tensor_cores=attention)
        self.dev_w = [{k: _cuda(v) for k, v in lw.items()} for lw in w]
        self.eng.set_weights(self.dev_w)
        self.eng.set_save_for_backward(True)
        if bwd_precision:
            self.eng.set_backward_precision(bwd_precision)
        self.eng.set_deterministic(det)
        if keep < 1.0:
            self.eng.set_state_dropout(keep, DROP_SEED)

    def forward(self, h0):
        self.th0 = _cuda(h0)
        self.out = self.eng.forward(self.th0)
        self.eng.sync_check()
        return self.out.cpu().numpy()

    def backward(self, g):
        import torch
        grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in self.dev_w]
        dh0 = torch.zeros_like(self.th0)
        self.eng.backward(_cuda(g), grads, dh0)
        self.eng.sync_check()
        return dh0.cpu().numpy(), [{k: v.cpu().numpy() for k, v in lw.items()} for lw in grads]


def molecules(n, D, T=4, seed=11):
    _, b = U.molecule_batch(n, D, T=T, seed=seed)
    return b["adjacency_lists"], np.asarray(b["num_incoming_edges_per_type"], np.float32), b["initial_node_representation"]


def one_component(V=3000, T=3, D=64, seed=7):
    """One connected component of V nodes (a path plus random nearby edges): larger than any tile."""
    rng = np.random.default_rng(seed)
    adj = []
    for t in range(T):
        src = rng.integers(0, V, 4000)
        tgt = (src + rng.integers(1, 50, 4000)) % V
        adj.append(np.stack([src, tgt], 1).astype(np.int32))
    adj[0] = np.concatenate([adj[0], np.stack([np.arange(V - 1), np.arange(1, V)], 1).astype(np.int32)])
    indeg = np.zeros((V, T), np.float32)
    for t in range(T):
        np.add.at(indeg[:, t], adj[t][:, 1], 1.0)
    return adj, indeg, rng.normal(0, 0.5, (V, D)).astype(np.float32)


def check(name, params, T, adj, indeg, h0, precision="bf16x3", bwd_precision=None, det=False, keep=1.0, attention=False, w=None):
    w = O.init_sparse_weights(params, T, np.random.default_rng(2), attention_scale=0.5) if w is None else w
    g = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    drop = (keep, DROP_SEED) if keep < 1.0 else None
    ref_out, ref_dh0, ref_gw = _autograd_reference(params, T, w, adj, indeg, h0, g, state_dropout=drop)
    r = Run(params, T, w, precision, bwd_precision, det, keep, attention)
    r.eng.set_graph_sparse(adj, indeg)
    want = ("wgmma-%s STREAM+attention+cudnn-gru(5 launches per step" if attention else STREAM) % precision
    assert r.eng.plan.startswith(want), r.eng.plan
    out = r.forward(h0)
    bar_f, bar_g = BARS[precision]
    errs = {"forward": _rel(out, ref_out)}
    if drop is None:   # every node_states_per_layer entry (residual sources, the layers' outputs)
        ref_layers = O.sparse_propagation_np(h0, adj, indeg, w, params, dtype=np.float64, return_all_layers=True)
        for l in range(1, len(params["layer_timesteps"])):
            errs["layer %d" % l] = _rel(r.eng.layer_state(l).cpu().numpy(), ref_layers[l])
    bad = {k: e for k, e in errs.items() if not e < bar_f}
    if precision == "bf16x3":
        dh0, gw = r.backward(g)
        errs["d h0"] = _rel(dh0, ref_dh0)
        bad.update({k: e for k, e in (("d h0", errs["d h0"]),) if not e < bar_g})
        for l, (a, rf) in enumerate(zip(gw, ref_gw)):
            assert set(rf) == set(a) and "cand_hidden_bias" in rf
            for k in rf:
                e = _rel(a[k], rf[k])
                errs["layer %d %s" % (l, k)] = e
                if not e < bar_g:
                    bad["layer %d %s" % (l, k)] = e
    print("cudnn-gru tensor cores %-24s worst %.2e  [%s]" % (name, max(errs.values()), r.eng.plan[:70]))
    assert np.all(np.isfinite(out)) and not bad, bad
    return r, out


WIDTHS = (20, 64, 100, 128, 132, 256, 384, 512)


@pytest.mark.parametrize("D", WIDTHS)
def test_every_width(D):
    adj, indeg, h0 = molecules(24, D)
    check("width-D%d" % D, cudnn_model(D), 4, adj, indeg, h0)


@pytest.mark.parametrize("D", [100, 256])
def test_single_bf16_mma(D):
    adj, indeg, h0 = molecules(24, D)
    check("bf16-D%d" % D, cudnn_model(D), 4, adj, indeg, h0, precision="bf16")


@pytest.mark.parametrize("T", [1, 4, 8])
@pytest.mark.parametrize("steps", [(1,), (4,), (8,)], ids=lambda s: "steps%d" % s[0])
def test_edge_types_and_timesteps(steps, T):
    adj, indeg, h0 = molecules(20, 100, T=T, seed=3)
    check("T%d-steps%d" % (T, steps[0]), cudnn_model(100, layer_timesteps=steps, residual_connections={}), T, adj, indeg, h0)


VARIANTS = {
    "bias-avg": lambda D: cudnn_model(D, bias=True, avg=True),
    "sum-nobias": lambda D: cudnn_model(D, bias=False, avg=False),
    "zero-step": lambda D: cudnn_model(D, layer_timesteps=(2, 0, 1), residual_connections={"2": [1, 2]}),
    "res4": lambda D: cudnn_model(D, layer_timesteps=(1, 1, 1, 2), residual_connections={"3": [0, 1, 2, 3]}),
}


@pytest.mark.parametrize("D", [36, 260])
@pytest.mark.parametrize("variant", sorted(VARIANTS) + ["dropout"])
def test_model_variants(variant, D):
    adj, indeg, h0 = molecules(20, D, seed=4)
    if variant == "dropout":   # forward and gradients under the same regenerated mask
        check("dropout-D%d" % D, cudnn_model(D), 4, adj, indeg, h0, keep=0.8)
    else:
        check("%s-D%d" % (variant, D), VARIANTS[variant](D), 4, adj, indeg, h0)


@pytest.mark.parametrize("D", [100, 260])
def test_tensor_core_backward_and_deterministic_mode(D):
    adj, indeg, h0 = molecules(20, D, seed=6)
    check("bwd-bf16x3-D%d" % D, cudnn_model(D), 4, adj, indeg, h0, bwd_precision="bf16x3")
    check("det-D%d" % D, cudnn_model(D), 4, adj, indeg, h0, det=True)


def test_one_large_component():
    adj, indeg, h0 = one_component()
    check("3000-node component", cudnn_model(64), 3, adj, indeg, h0)


@pytest.mark.parametrize("D", [36, 256])
def test_with_tensor_core_attention_at_16_edge_types(D):
    from tests.test_attention_edges_cpu import batch, regime_h0
    adj, indeg, T = batch("t16_all")
    assert T == 16
    check("attention-t16-D%d" % D, cudnn_model(D, attention=True), T, adj, indeg, regime_h0("mild", indeg.shape[0], D), attention=True)


def test_matches_the_reference_graph_code_fixture(golden_dir):
    z = np.load(os.path.join(golden_dir, "refgraph_sparse_cudnn_gru.npz"))
    p = json.loads(str(z["params_json"]))
    w = [{k[len("w%d_" % l):]: z[k] for k in z.files if k.startswith("w%d_" % l)} for l in range(len(p["layer_timesteps"]))]
    adj = [z["adj%d" % e] for e in range(4)]
    r = Run(p, 4, w)
    r.eng.set_graph_sparse(adj, z["indeg"].astype(np.float32))
    assert r.eng.plan.startswith(STREAM % "bf16x3"), r.eng.plan
    err = _rel(r.forward(z["h0"].astype(np.float32)), z["final"])
    print("refgraph cudnn_gru through the streaming plan: max rel err %.2e" % err)
    assert err < 1e-4


@pytest.mark.parametrize("D", [100, 260])
def test_repeats_and_feeds_agree(D):
    """Two forwards give identical bits (1 + 4 launches per step); set_graph_sparse, a prepared graph and a device-dataset batch of the
    same graphs give identical images and bit-identical final states."""
    from gated_graph_neural_network_samples_b200 import packing
    from gated_graph_neural_network_samples_b200.engine import DeviceDataset
    from tests.test_device_data_cpu import packed_graph, sparse_graph_set
    T = 4
    flat = packing.FlatSparseGraphs(sparse_graph_set(), T)
    ids = np.array([5, 2, 9, 0, 31, 17, 40, 3], np.int64)
    pk = packed_graph(flat, ids, D)
    adj, indeg = pk["adjacency_lists"], pk["num_incoming_edges_per_type"]
    params = cudnn_model(D)
    r = Run(params, T, O.init_sparse_weights(params, T, np.random.default_rng(2)))
    ds = DeviceDataset.for_engine(r.eng, flat, for_training=True)
    b = ds.prepare_batch(ids, save_for_backward=True)
    h0, _, _ = r.eng.set_graph_from_dataset(b)
    h0 = h0.cpu().numpy()
    img_ds = r.eng.graph_image()
    out_ds = r.forward(h0)
    r.eng.set_graph_sparse(adj, indeg)
    img_sp = r.eng.graph_image()
    out_sp = r.forward(h0)
    assert r.eng.last_launch_count == 1 + 3 * 4
    np.testing.assert_array_equal(r.forward(h0), out_sp)
    g = r.eng.prepare_graph_sparse(adj, indeg)
    r.eng.set_graph_prepared(g)
    out_pg = r.forward(h0)
    assert r.eng.plan.startswith(STREAM % "bf16x3"), r.eng.plan
    assert img_ds.shape == img_sp.shape and np.array_equal(img_ds, img_sp), np.flatnonzero(img_ds != img_sp)[:32]
    np.testing.assert_array_equal(g.image(), img_sp)
    np.testing.assert_array_equal(out_ds, out_sp)
    np.testing.assert_array_equal(out_pg, out_sp)


# ---------------------------------------------------------------------------------------------------------------- through the plug-in
def test_plugin_trains_and_checkpoints_like_the_fp32_cell(tmp_path):
    """SparseGGNNChemModel with --precision bf16x3 --cudnn-gru-tensor-cores: the engine runs the streaming plan, the validation loss
    falls, the checkpoint has the fp32 run's variable names and shapes, and it restores into a model without the option."""
    from gated_graph_neural_network_samples_b200 import synthetic
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    mols = synthetic.make_molecules(96, seed=1)

    def model(**opts):
        return SparseGGNNChemModel(dict({"--log_dir": str(tmp_path), "--train_data": mols[:64], "--valid_data": mols[64:],
                                         "--config": {"hidden_size": 32, "batch_size": 400, "layer_timesteps": [2, 1],
                                                      "residual_connections": {"1": [0]}, "edge_weight_dropout_keep_prob": 1.0,
                                                      "learning_rate": 0.01, "num_epochs": 1, "graph_rnn_cell": CELL}}, **opts))
    m = model(**{"--precision": "bf16x3", "--cudnn-gru-tensor-cores": True})
    l0 = m.run_epoch("valid0", m.valid_data, False)[0]
    assert m.engine.plan.startswith(STREAM % "bf16x3"), m.engine.plan
    for ep in range(6):
        m.run_epoch("train%d" % ep, m.train_data, True)
    l1 = m.run_epoch("valid1", m.valid_data, False)[0]
    print("cudnn-gru tensor cores validation loss %.4f -> %.4f" % (l0, l1))
    assert np.isfinite(l1) and l1 < l0
    path = str(tmp_path / "ckpt.pickle")
    m.save_progress(path, 2, 1)
    ref_path = str(tmp_path / "ckpt_fp32.pickle")
    f = model()   # an fp32 run of the same model: one epoch, so that its checkpoint holds the optimizer's slots too
    f.run_epoch("train-fp32", f.train_data, True)
    f.save_progress(ref_path, 0, 0)
    got, want = pickle.load(open(path, "rb"))["weights"], pickle.load(open(ref_path, "rb"))["weights"]
    assert sorted(got) == sorted(want)
    assert all(np.shape(got[k]) == np.shape(want[k]) for k in got)
    m2 = model(**{"--precision": "bf16x3"})   # without the option: the fp32 cell
    assert m2.restore_progress(path) == (2, 1)
    l2 = m2.run_epoch("valid2", m2.valid_data, False)[0]
    assert m2.engine.plan.startswith("fp32-") and "+cudnn-gru" in m2.engine.plan, m2.engine.plan
    assert abs(l2 - l1) < 1e-3 * max(1.0, abs(l1)), (l1, l2)
