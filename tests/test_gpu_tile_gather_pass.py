"""GPU: the compact tile kernel's gather pass.

On compact tiles (<= 64 rows) ``ggnn_fwd_tc_kernel`` gathers the A_t of several edge types into separate gather tiles in one pass and
then runs their MMAs back to back, one barrier per group of types.  ``GGNN_TC_GATHER_TILES=<n>`` sets the number of gather tiles (by
default the most edge types present in one tile, as many as shared memory holds while the weight ring keeps four slots); with 2 the
kernel gathers one type at a time, each followed by its MMAs.  Every accumulator sums the same products in the same order either way, so:

* the final states and every ``node_states_per_layer`` entry are the same bits with the default and with two gather tiles;
* both are within the 1e-4 bar of the float64 oracle;
* with save-for-backward on, ``d h0`` and every weight gradient (fixed-order sums, ``set_deterministic``) are the same bits.

Cases: cfg2, cfg1 true default (residuals), cfg3 dense (binary adjacency -> CSR, edge bias), and a 17-edge-type batch, where the gather
tiles do not hold every type of a tile (groups of half the tiles, rotating) and the tile's CSR slice is read from global memory.
"""
import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import workloads
from oracle import ggnn_oracle as O
from tests import _util as U
from tests.test_backward_plans_cpu import component_graph

pytestmark = pytest.mark.gpu

BAR = 1e-4
T17_PARAMS = dict(workloads.SPARSE_BASE, hidden_size=100, layer_timesteps=[2, 1], residual_connections={"1": [0]}, use_edge_bias=True)


def _workload(name):
    if name != "T17":
        w = workloads.build(name)
        w["params_oracle"] = w["params"]
        return w
    adj, indeg = component_graph(17, V_target=2000, seed=17)
    h0 = np.random.default_rng(17).normal(0, 1, (indeg.shape[0], 100)).astype(np.float32)
    return {"kind": "sparse", "num_edge_types": 17, "engine_params": T17_PARAMS, "params_oracle": T17_PARAMS, "adjacency_lists": adj,
            "num_incoming_edges_per_type": indeg, "h0": h0, "weights": workloads.init_weights(T17_PARAMS, 17, seed=5)}


def _oracle(w):
    if w["kind"] == "dense":
        b, v = w["dense_shape"]
        return O.dense_propagation_loops(w["h0"].reshape(b, v, -1), w["adjacency_matrix"], w["weights"][0],
                                         w["params_oracle"]).reshape(b * v, -1)
    return O.sparse_propagation_np(w["h0"], w["adjacency_lists"], w["num_incoming_edges_per_type"], w["weights"], w["engine_params"],
                                   dtype=np.float64)


def _run(w, monkeypatch, tiles, save):
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    for k in ("GGNN_FORCE_GLOBAL", "GGNN_TC_STREAM"):
        monkeypatch.delenv(k, raising=False)
    if tiles is None:
        monkeypatch.delenv("GGNN_TC_GATHER_TILES", raising=False)
    else:
        monkeypatch.setenv("GGNN_TC_GATHER_TILES", str(tiles))
    eng = PropagationEngine(w["engine_params"], w["num_edge_types"], precision="bf16x3")
    dev_w = U.to_cuda_weights(w["weights"])
    eng.set_weights(dev_w)
    eng.set_save_for_backward(save)
    eng.set_deterministic(True)   # fixed-order weight-gradient sums: the same saved states give the same gradient bits
    if w["kind"] == "dense":
        eng.set_graph_dense(w["adjacency_matrix"])
    else:
        eng.set_graph_sparse(w["adjacency_lists"], w["num_incoming_edges_per_type"])
    h0 = torch.from_numpy(np.ascontiguousarray(w["h0"])).cuda()
    out = eng.forward(h0)
    eng.sync_check()
    assert "compact 64-row operand tiles" in eng.plan and eng.plan.startswith("wgmma-bf16x3 LOCAL("), eng.plan
    L = len(w["engine_params"]["layer_timesteps"])
    res = {"out": out.cpu().numpy(), "layers": [eng.layer_state(l).cpu().numpy() for l in range(L + 1)]}
    if save:
        g_out = torch.from_numpy(np.random.default_rng(3).normal(size=w["h0"].shape).astype(np.float32)).cuda()
        grads = [{k: torch.zeros_like(v) for k, v in lw.items()} for lw in dev_w]
        dh0 = torch.zeros_like(h0)
        eng.backward(g_out, grads, dh0)
        eng.sync_check()
        res["dh0"] = dh0.cpu().numpy()
        res["grads"] = [{k: v.cpu().numpy() for k, v in lw.items()} for lw in grads]
    return res


@pytest.mark.parametrize("name", ["cfg2", "cfg1_true_default", "cfg3_dense", "T17"])
@pytest.mark.parametrize("save", [False, True])
def test_gather_pass_gives_the_same_bits_as_one_type_at_a_time(name, save, monkeypatch):
    w = _workload(name)
    ref = _oracle(w)
    two = _run(w, monkeypatch, 2, save)
    for tiles in (None, 3):
        got = _run(w, monkeypatch, tiles, save)
        tag = "%s tiles=%s save=%s" % (name, tiles, save)
        np.testing.assert_array_equal(got["out"], two["out"], err_msg=tag)
        for l, (a, b) in enumerate(zip(got["layers"], two["layers"])):
            np.testing.assert_array_equal(a, b, err_msg="%s layer %d" % (tag, l))
        if save:
            np.testing.assert_array_equal(got["dh0"], two["dh0"], err_msg=tag + " d h0")
            for l, (ga, gb) in enumerate(zip(got["grads"], two["grads"])):
                for k in ga:
                    np.testing.assert_array_equal(ga[k], gb[k], err_msg="%s layer %d d %s" % (tag, l, k))
    err = U.max_rel_err(two["out"], ref)
    assert err < BAR, (name, err)
