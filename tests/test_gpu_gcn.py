"""Sparse GCN on the H100: the wgmma (bf16x3 / bf16) and fp32 kernels against the float64 list-order oracle, the backward pass against
float64 autograd, prepared graphs, refusals of the other model's calls."""
import threading

import numpy as np
import pytest

from tests import gcn_oracle as G
from tests._util import max_rel_err

pytestmark = pytest.mark.gpu


def run(D, L, V, lst, w, h0, ks, bs=None, precision="bf16x3", keep=1.0, seed=0, save=False):
    import torch
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    eng = GCNEngine(D, L, use_bias=bs is not None, precision=precision)
    dk = [torch.from_numpy(k).cuda() for k in ks]
    db = None if bs is None else [torch.from_numpy(b).cuda() for b in bs]
    eng.set_weights(dk, db)
    eng.set_save_for_backward(save)
    eng.set_graph_gcn(V, lst, w)
    eng.set_state_dropout(keep, seed)
    h = torch.from_numpy(np.ascontiguousarray(h0, np.float32)).cuda()
    out = eng.forward(h)
    eng.sync_check()
    eng._keep = (dk, db, h, out)
    return out.cpu().numpy(), eng


def case(D, L, V, nnz, seed, bias=False, isolated=()):
    rng = np.random.default_rng(seed)
    lst, w = G.random_gcn_list(V, nnz, rng, isolated=isolated)
    ks = [G.glorot((D, D), rng) for _ in range(L)]
    bs = [rng.normal(0, 0.2, D).astype(np.float32) for _ in range(L)] if bias else None
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    return lst, w, ks, bs, h0


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
@pytest.mark.parametrize("D", [12, 100, 128, 256])
def test_forward_matches_list_order_oracle(precision, D):
    V = 300
    lst, w, ks, bs, h0 = case(D, 3, V, 2000, D, bias=True, isolated=(0, 7, 299))
    got, eng = run(D, 3, V, lst, w, h0, ks, bs, precision)
    ref = G.gcn_propagation_loops(h0, lst, w, ks, bs)
    assert max_rel_err(got, ref) < 1e-4, (eng.plan, max_rel_err(got, ref))
    if precision == "bf16x3" and D <= 128:
        assert eng.plan.startswith("gcn-wgmma-bf16x3 GLOBAL"), eng.plan   # one random graph over all nodes: a single big component
    else:
        assert eng.plan.startswith("gcn-fp32"), eng.plan


def test_orientation_is_pinned_by_a_non_symmetric_list():
    # (i, j) = (output, input): node 0 receives 2 * h[1]; node 1 receives nothing
    import torch  # noqa: F401
    D = 16
    lst = np.array([[0, 1]], np.int64)
    w = np.array([2.0], np.float32)
    h0 = np.zeros((2, D), np.float32)
    h0[1] = 1.0
    k = np.eye(D, dtype=np.float32)
    for precision in ("bf16x3", "fp32"):
        got, _ = run(D, 1, 2, lst, w, h0, [k], precision=precision)
        np.testing.assert_allclose(got[0], 2.0, rtol=1e-6)
        np.testing.assert_array_equal(got[1], 0.0)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16", "fp32"])
def test_local_plan_on_molecule_sized_components(precision):
    rng = np.random.default_rng(11)
    D, L = 100, 4
    V, lst, w = G.component_list(list(rng.integers(5, 30, 200)), rng)
    ks = [G.glorot((D, D), rng) for _ in range(L)]
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    got, eng = run(D, L, V, lst, w, h0, ks, precision=precision)
    ref = G.gcn_propagation_loops(h0, lst, w, ks)
    tol = 1e-2 if precision == "bf16" else 1e-4
    assert max_rel_err(got, ref) < tol, (eng.plan, max_rel_err(got, ref))
    if precision != "fp32":
        assert "LOCAL" in eng.plan and eng.last_launch_count <= 1 + L, (eng.plan, eng.last_launch_count)


def test_local_equals_global(monkeypatch):
    rng = np.random.default_rng(12)
    D, L = 64, 3
    V, lst, w = G.component_list(list(rng.integers(5, 40, 100)), rng)
    ks = [G.glorot((D, D), rng) for _ in range(L)]
    bs = [rng.normal(0, 0.2, D).astype(np.float32) for _ in range(L)]
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    loc, e1 = run(D, L, V, lst, w, h0, ks, bs)
    monkeypatch.setenv("GGNN_FORCE_GLOBAL", "1")
    glo, e2 = run(D, L, V, lst, w, h0, ks, bs)
    assert "LOCAL" in e1.plan and "GLOBAL" in e2.plan
    # same gather order, same operand split, same MMAs and epilogue: only where the previous layer's state is read from differs
    np.testing.assert_array_equal(loc, glo)


def test_run_to_run_bit_identity():
    lst, w, ks, bs, h0 = case(100, 4, 500, 4000, 3)
    a, eng = run(100, 4, 500, lst, w, h0, ks)
    import torch
    h = torch.from_numpy(h0).cuda()
    for _ in range(3):
        b = eng.forward(h).cpu().numpy()
        np.testing.assert_array_equal(a, b)


def test_empty_lists_and_isolated_nodes():
    D = 32
    rng = np.random.default_rng(4)
    ks = [G.glorot((D, D), rng) for _ in range(2)]
    bs = [rng.normal(0, 0.2, D).astype(np.float32) for _ in range(2)]
    h0 = rng.normal(0, 1, (10, D)).astype(np.float32)
    for precision in ("bf16x3", "fp32"):
        got, _ = run(D, 2, 10, np.zeros((0, 2), np.int64), np.zeros(0, np.float32), h0, ks, bs, precision)
        ref = G.gcn_propagation_loops(h0, np.zeros((0, 2)), np.zeros(0), ks, bs)
        np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-6)


def test_dropout_forward_matches_the_oracle_with_the_engine_mask():
    D, L, V = 48, 3, 200
    lst, w, ks, bs, h0 = case(D, L, V, 1500, 8, bias=True)
    keep, seed = 0.75, 1234
    for precision in ("bf16x3", "fp32"):
        got, eng = run(D, L, V, lst, w, h0, ks, bs, precision, keep=keep, seed=seed)
        masks = [eng.state_dropout_mask(l, keep, seed) for l in range(L - 1)]
        ref = G.gcn_propagation_loops(h0, lst, w, ks, bs, masks, keep)
        assert max_rel_err(got, ref) < 1e-4


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
@pytest.mark.parametrize("keep", [1.0, 0.8])
def test_gradients_match_float64_autograd(precision, keep):
    import torch
    D, L, V = 40, 3, 150
    lst, w, ks, bs, h0 = case(D, L, V, 900, 21, bias=True, isolated=(5,))
    seed = 77
    got, eng = run(D, L, V, lst, w, h0, ks, bs, precision, keep=keep, seed=seed, save=True)
    rng = np.random.default_rng(5)
    g_out = rng.normal(0, 1, (V, D)).astype(np.float32)
    gk = [torch.zeros(D, D, device="cuda") for _ in range(L)]
    gb = [torch.zeros(D, device="cuda") for _ in range(L)]
    dh0 = torch.empty(V, D, device="cuda")
    eng.backward(torch.from_numpy(g_out).cuda(), [{"kernel": a, "bias": b} for a, b in zip(gk, gb)], d_h0=dh0)
    eng.sync_check()
    masks = [eng.state_dropout_mask(l, keep, seed) for l in range(L - 1)] if keep < 1 else None
    th0 = torch.from_numpy(h0).double().requires_grad_()
    tk = [torch.from_numpy(k).double().requires_grad_() for k in ks]
    tb = [torch.from_numpy(b).double().requires_grad_() for b in bs]
    out = G.gcn_propagation_torch(th0, lst, torch.from_numpy(w).double(), tk, tb, masks, keep)
    out.backward(torch.from_numpy(g_out).double())
    for l in range(L):
        assert max_rel_err(gk[l].cpu().numpy(), tk[l].grad.numpy()) < 2.5e-5, l
        assert max_rel_err(gb[l].cpu().numpy(), tb[l].grad.numpy()) < 2.5e-5, l
    assert max_rel_err(dh0.cpu().numpy(), th0.grad.numpy()) < 2.5e-5


def test_prepared_graph_built_in_a_producer_thread():
    import torch
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    D, L = 100, 4
    lst, w, ks, bs, h0 = case(D, L, 400, 3000, 9)
    eng = GCNEngine(D, L, precision="bf16x3")
    dk = [torch.from_numpy(k).cuda() for k in ks]
    eng.set_weights(dk)
    box = {}
    t = threading.Thread(target=lambda: box.setdefault("g", eng.prepare_graph_gcn(400, lst, w)))
    t.start()
    t.join()
    eng.set_graph_prepared(box["g"])
    got = eng.forward(torch.from_numpy(h0).cuda()).cpu().numpy()
    eng.sync_check()
    assert max_rel_err(got, G.gcn_propagation_loops(h0, lst, w, ks)) < 1e-4


def test_readout_on_a_gcn_engine():
    import torch
    D, L = 32, 2
    rng = np.random.default_rng(6)
    V, lst, w = G.component_list([10, 12, 8], rng)
    ks = [G.glorot((D, D), rng) for _ in range(L)]
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    got, eng = run(D, L, V, lst, w, h0, ks)
    gnl = np.repeat(np.arange(3, dtype=np.int32), [10, 12, 8])
    eng.readout_set_graphs(3, gnl)
    wg, bg, wt, bt = (torch.from_numpy(rng.normal(0, 0.3, n).astype(np.float32)).cuda() for n in (2 * D, 1, D, 1))
    hl, hz = torch.from_numpy(got).cuda(), torch.from_numpy(h0).cuda()
    out = eng.readout_forward(hl, hz, wg, bg, wt, bt).cpu().numpy()
    gate = torch.sigmoid(torch.cat([hl, hz], 1) @ wg + bg) * (hl @ wt + bt)
    ref = torch.zeros(3, device="cuda").index_add_(0, torch.from_numpy(gnl).long().cuda(), gate).cpu().numpy()
    np.testing.assert_allclose(out, ref, rtol=1e-4, atol=1e-5)


def test_mismatched_calls_are_refused():
    import torch
    from gated_graph_neural_network_samples_b200 import _lib, workloads
    from gated_graph_neural_network_samples_b200.engine import GCNEngine, GgnnError, PropagationEngine
    gcn = GCNEngine(16, 2)
    with pytest.raises(GgnnError, match="GGNN call"):
        gcn.set_graph_sparse([np.array([[0, 1]], np.int32)], np.array([[0.0], [1.0]], np.float32))
    with pytest.raises(GgnnError, match="GGNN call"):
        gcn.set_graph_dense(np.zeros((1, 1, 2, 2), np.float32))
    ggnn = PropagationEngine(dict(workloads.SPARSE_BASE, hidden_size=16, layer_timesteps=[1]), 1)
    with pytest.raises(GgnnError, match="GCN call"):
        GCNEngine.set_graph_gcn(ggnn, 2, np.array([[0, 1]]), np.ones(1, np.float32))
    with pytest.raises(GgnnError, match="GCN call"):
        GCNEngine.backward(ggnn, torch.zeros(2, 16, device="cuda"), [{}])
    k = torch.zeros(16, 16, device="cuda")
    arr = (_lib.GcnLayerWeights * 1)()
    arr[0].kernel = k.data_ptr()
    assert ggnn.lib.ggnn_gcn_set_weights(ggnn._h, arr, 1) == -3   # GGNN_ESTATE
    assert "GCN call" in ggnn.lib.ggnn_last_error(ggnn._h).decode()
    with pytest.raises(GgnnError, match="GGNN call"):
        PropagationEngine.backward(gcn, torch.zeros(2, 16, device="cuda"), [{}, {}])
    with pytest.raises(GgnnError):
        gcn.set_graph_prepared(ggnn.prepare_graph_sparse([np.array([[0, 1]], np.int32)], np.array([[0.0], [1.0]], np.float32)))
    gcn.set_graph_gcn(2, np.array([[0, 1]]), np.ones(1, np.float32))
    with pytest.raises(GgnnError, match="out of range"):
        gcn.set_graph_gcn(2, np.array([[0, 2]]), np.ones(1, np.float32))


def test_hidden_sizes_through_padding():
    """A hidden size that is not a multiple of 4, zero-padded by the caller to the next multiple: the padded columns stay zero and the real
    ones match the unpadded oracle."""
    D, Dp, L, V = 10, 12, 3, 120
    rng = np.random.default_rng(13)
    lst, w = G.random_gcn_list(V, 700, rng)
    ks = [G.glorot((D, D), rng) for _ in range(L)]
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    kp = [np.pad(k, ((0, Dp - D), (0, Dp - D))) for k in ks]
    got, _ = run(Dp, L, V, lst, w, np.pad(h0, ((0, 0), (0, Dp - D))), kp)
    assert np.all(got[:, D:] == 0)
    assert max_rel_err(got[:, :D], G.gcn_propagation_loops(h0, lst, w, ks)) < 1e-4


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
@pytest.mark.parametrize("name", ["h12_l3", "h100_l4_bias", "h12_l1"])
def test_reference_graph_fixtures(golden_dir, precision, name):
    """refgraph_gcn_*.npz: the reference's own make_model (both hooks, gated_regression) evaluated in float64; the engine's propagation and
    its fused readout reproduce the final states and the per-graph outputs at 1e-4."""
    import json
    import os
    import torch
    z = np.load(os.path.join(golden_dir, "refgraph_gcn_%s.npz" % name))
    cfg = json.loads(str(z["params_json"]))
    D, L = cfg["hidden_size"], cfg["num_timesteps"]
    ks = [z["w%d_kernel" % l] for l in range(L)]
    bs = [z["w%d_bias" % l] for l in range(L)] if cfg["gcn_use_bias"] else None
    h0 = z["h0"]
    got, eng = run(D, L, h0.shape[0], z["adjacency_list"], z["adjacency_weights_f32"], h0, ks, bs, precision)
    assert max_rel_err(got, z["final"]) < 1e-4, (eng.plan, max_rel_err(got, z["final"]))
    eng.readout_set_graphs(int(z["num_graphs"]), z["graph_nodes_list"])
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1)).cuda()
    ro = eng.readout_forward(dev(got), dev(h0), dev(z["ro_w_gate"]), dev(z["ro_b_gate"]), dev(z["ro_w_trans"]), dev(z["ro_b_trans"]))
    assert max_rel_err(ro.cpu().numpy(), z["readout"]) < 1e-4
