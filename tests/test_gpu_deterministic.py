"""GPU: deterministic mode (``ggnn_set_deterministic``).  With it on, every output and every accumulated gradient must be the same bits
from call to call, engine to engine and process to process, and still meet the float64 bars of the gradient tests.

* Forward: the tile-local and GCN wgmma kernels (the default plans for hidden <= 128) give the same bits twice on one engine and once on a
  fresh engine, for every tile-local and GCN-wgmma case of tests/test_forward_plans_cpu.py -- so deterministic mode needs no forward change.
* Backward, on the case lists of tests/test_backward_plans_cpu.py: forward, ``d h0`` and every weight / bias gradient are identical across
  two backward calls of one forward, a fresh engine, and a different prefill of the caller's buffers (result = prefill + G, G identical),
  and G meets the float64 bar; partial requests; attention with 16 types, absent types exactly 0.
* Readout: forward and all five gradients on grouped, shuffled and masked node lists, with the mode set before or after
  ``readout_set_graphs``.
* cfg4 and the 100 000-node batch: gradients identical across two engines; there and on batches whose splits are not capped by the row
  count (GRU, RNN, CudnnCompatibleGRUCell, attention; layers with different residual counts), within ordering noise of the atomic path.
* End to end: two training runs of each plug-in in fresh processes under ``torch.use_deterministic_algorithms(True)`` give identical
  per-epoch losses and identical checkpoints (weights and both Adam slots).
"""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from oracle import ggnn_oracle as O
from tests import _util as U
from tests import gcn_oracle as G
from tests.test_backward_plans_cpu import (DENSE_CASES, DENSE_T, EDGE_SHAPES, GCN_CASES, GCN_LAYERS, PARTIAL_CASES, PLAN_MATRIX, SPARSE_CASES,
                                           dense_batch, dense_params, gcn_batch, plan_matches, sparse_batch)
from tests.test_forward_plans_cpu import CASES as FWD_CASES
from tests.test_gpu_backward import _autograd_reference

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REN = {"rnn_kernel": "cand_kernel", "rnn_bias": "cand_bias"}


def _set_env(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _same(a, b, tag):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.tobytes() == b.tobytes(), (tag, float(np.max(np.abs(a.astype(np.float64) - b))))


# ---------------------------------------------------------------------------------------------------------------- forward
TC_FWD = sorted(n for n, c in FWD_CASES.items() if c.instance[0] in ("tc", "gcn"))


@pytest.mark.parametrize("case", TC_FWD)
def test_wgmma_forward_is_bit_identical_run_to_run_and_engine_to_engine(case, monkeypatch):
    import torch
    from gated_graph_neural_network_samples_b200.engine import PropagationEngine
    from tests.test_forward_plans_cpu import dense_batch as fwd_dense_batch, gcn_graph, graph, h0_for
    from tests.test_gpu_forward_plans import DROP_SEED, _weights
    from tests.test_gpu_gcn import run
    c = FWD_CASES[case]
    _set_env(monkeypatch, c.env)
    if c.kind == "gcn":
        V, lst, w = gcn_graph(c.D, c.batch)
        rng = np.random.default_rng(c.D)
        ks = [G.glorot((c.D, c.D), rng) for _ in range(GCN_LAYERS)]
        bs = [rng.normal(0, 0.2, c.D).astype(np.float32) for _ in range(GCN_LAYERS)]
        h0 = rng.normal(0, 1, (V, c.D)).astype(np.float32)
        a, eng = run(c.D, GCN_LAYERS, V, lst, w, h0, ks, bs, c.precision, keep=c.keep, seed=DROP_SEED)
        b = eng.forward(torch.from_numpy(h0).cuda()).cpu().numpy()
        fresh, _ = run(c.D, GCN_LAYERS, V, lst, w, h0, ks, bs, c.precision, keep=c.keep, seed=DROP_SEED)
    else:
        if c.kind == "dense":
            A, h0 = fwd_dense_batch(c.D, True)
            h0 = h0.reshape(-1, c.D)
            dw = O.init_dense_weights({"hidden_size": c.D}, c.T, np.random.default_rng(5))
            w = [dict(dw, edge_biases=dw["edge_biases"].reshape(c.T, c.D))]
        else:
            adj, indeg = graph(c.batch, c.T)
            h0 = h0_for(indeg.shape[0], c.D)
            w = _weights(c.params, c.T)

        def engine():
            e = PropagationEngine(c.params, c.T, precision=c.precision)
            e.set_weights(U.to_cuda_weights(w))
            if c.keep < 1.0:
                e.set_state_dropout(c.keep, DROP_SEED)
            e.set_graph_dense(A) if c.kind == "dense" else e.set_graph_sparse(adj, indeg)
            return e

        th0 = torch.from_numpy(h0).cuda()
        eng = engine()
        a = eng.forward(th0).cpu().numpy()
        b = eng.forward(th0).cpu().numpy()
        fresh = engine().forward(th0).cpu().numpy()
    torch.cuda.synchronize()
    print("\nFWDBITS %-40s %s" % (case, "identical" if a.tobytes() == b.tobytes() == fresh.tobytes() else "DIFFERENT"))
    _same(b, a, case + " second forward")
    _same(fresh, a, case + " fresh engine")


# ---------------------------------------------------------------------------------------------------------------- GGNN backward
def _weights(p, T, seed=1):
    from tests.test_gpu_backward_plans import _weights as w
    return w(p, T, seed)


class _Det:
    """One deterministic engine after a forward with save_for_backward; ``backward(prefill)`` accumulates into buffers holding
    ``prefill`` (per layer {field: array}, None: zeros) and returns (d h0, per-layer gradients) as NumPy."""

    def __init__(self, params, T, w, set_graph, h0, g_out, precision, fields=None):
        import torch
        from gated_graph_neural_network_samples_b200.engine import PropagationEngine
        self.eng = PropagationEngine(params, T, precision=precision)
        self.eng.set_deterministic(True)
        self.dev_w = [{REN.get(k, k): torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda() for k, v in lw.items()} for lw in w]
        self.eng.set_weights(self.dev_w)
        self.eng.set_save_for_backward(True)
        set_graph(self.eng)
        self.plan = self.eng.plan
        self.h0 = torch.from_numpy(np.ascontiguousarray(h0, np.float32)).cuda()
        self.out_t = self.eng.forward(self.h0)   # the backward reads the forward's output again (the RNN cell's last step)
        self.out = self.out_t.cpu().numpy()
        self.g_out = torch.from_numpy(np.ascontiguousarray(g_out, np.float32)).cuda()
        self.fields = sorted(self.dev_w[0]) if fields is None else fields

    def backward(self, prefill=None, want_dh0=True):
        import torch
        grads = [{k: (torch.zeros_like(lw[k]) if prefill is None else torch.from_numpy(prefill[l][k]).cuda()) for k in self.fields if k in lw}
                 for l, lw in enumerate(self.dev_w)]
        dh0 = torch.zeros_like(self.h0) if want_dh0 else None
        self.eng.backward(self.g_out, grads, dh0)
        self.eng.sync_check()
        return (None if dh0 is None else dh0.cpu().numpy()), [{k: v.cpu().numpy() for k, v in lw.items()} for lw in grads]


def _check_repeatable(make, ref=None, tag=""):
    """Two backward calls of one forward, a fresh engine, and a random prefill: identical bits.  Returns the first engine's results."""
    t = make()
    dh0, g = t.backward()
    dh0_b, g_b = t.backward()
    t2 = make()
    _same(t2.out, t.out, tag + " forward, fresh engine")
    dh0_c, g_c = t2.backward()
    rng = np.random.default_rng(9)
    prefill = [{k: rng.normal(0, 1, v.shape).astype(np.float32) for k, v in lw.items()} for lw in g]
    _, g_p = t.backward(prefill)
    for other, odh0, name in ((g_b, dh0_b, "second call"), (g_c, dh0_c, "fresh engine")):
        _same(odh0, dh0, "%s d h0 %s" % (tag, name))
        for l, (x, y) in enumerate(zip(g, other)):
            for k in x:
                _same(y[k], x[k], "%s layer %d %s %s" % (tag, l, k, name))
    for l, (x, y, p) in enumerate(zip(g, g_p, prefill)):
        for k in x:
            _same(y[k], p[k] + x[k], "%s layer %d %s prefill" % (tag, l, k))
    if ref is not None:
        from tests.test_gpu_backward_plans import _compare
        inv = {v: k for k, v in REN.items()} if "rnn_kernel" in ref[2][0] else {}
        _compare(tag, (t.out, dh0, [{inv.get(k, k): v for k, v in lw.items()} for lw in g]), ref)
    return t, dh0, g


def _sparse_case(c, monkeypatch):
    _set_env(monkeypatch, c.env)
    adj, indeg, h0 = sparse_batch(c.batch, c.params["hidden_size"], c.T)
    w = _weights(c.params, c.T)
    g_out = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    ref = _autograd_reference(c.params, c.T, w, adj, indeg, h0, g_out)
    t, _, _ = _check_repeatable(lambda: _Det(c.params, c.T, w, lambda e: e.set_graph_sparse(adj, indeg), h0, g_out, c.precision), ref, c.name)
    assert plan_matches(t.plan, c.plan), (c.plan, t.plan)


@pytest.mark.parametrize("case", [c.name for c in PLAN_MATRIX + EDGE_SHAPES])
def test_gradients_are_bit_identical_and_meet_float64(case, monkeypatch):
    """Every forward plan, T = 1 / 3 / 17 / 32, four residuals, zero-step layers, CudnnCompatibleGRUCell and attention."""
    _sparse_case(SPARSE_CASES[case], monkeypatch)


@pytest.mark.parametrize("case", PARTIAL_CASES)
def test_partial_requests_are_bit_identical(case, monkeypatch):
    """Only the edge weights, only the biases (kernels null: the column-sum splits), only d h0: each twice, identical, and within fp32
    rounding of the same fields of a full request."""
    c = SPARSE_CASES[case]
    _set_env(monkeypatch, c.env)
    adj, indeg, h0 = sparse_batch(c.batch, c.params["hidden_size"], c.T)
    w = _weights(c.params, c.T)
    g_out = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    full = _Det(c.params, c.T, w, lambda e: e.set_graph_sparse(adj, indeg), h0, g_out, c.precision)
    full_dh0, full_g = full.backward()
    for request in (["edge_weights"], [k for k in full.fields if "bias" in k], []):
        t = _Det(c.params, c.T, w, lambda e: e.set_graph_sparse(adj, indeg), h0, g_out, c.precision, fields=request)
        dh0, a = t.backward()
        dh0_b, b = t.backward()
        _same(dh0, full_dh0, "d h0")
        _same(dh0_b, dh0, "d h0 twice")
        for l, (x, y, f) in enumerate(zip(a, b, full_g)):
            assert sorted(x) == sorted(request)
            for k in x:
                _same(y[k], x[k], "layer %d %s twice" % (l, k))
                assert U.max_rel_err(x[k], f[k]) < 1e-5, (l, k)


def test_attention_with_16_types_and_absent_types(monkeypatch):
    """d a_t summed per warp slot and per block in a fixed order; types without messages get exactly 0 (the prefill stays)."""
    T = 16
    p = {"hidden_size": 36, "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}, "use_edge_bias": True,
         "use_edge_msg_avg_aggregation": False, "graph_rnn_cell": "GRU", "graph_rnn_activation": "tanh", "use_propagation_attention": True}
    adj4, indeg4, h0 = sparse_batch("mol24", 36, 4)
    # types 0-3 from the molecules, 4-9 copies of them, 10-15 absent
    adj = list(adj4) + [a[::2].copy() for a in adj4] + [a[1::2].copy() for a in adj4[:2]] + [np.zeros((0, 2), np.int32)] * 6
    indeg = np.zeros((h0.shape[0], T), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    w = _weights(p, T)
    g_out = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    ref = _autograd_reference(p, T, w, adj, indeg, h0, g_out)
    t, _, g = _check_repeatable(lambda: _Det(p, T, w, lambda e: e.set_graph_sparse(adj, indeg), h0, g_out, "fp32"), ref, "attention-T16")
    for lw in g:
        assert np.all(lw["edge_type_attention_weights"][10:] == 0.0)
        assert np.all(lw["edge_type_attention_weights"][:10] != 0.0)


@pytest.mark.parametrize("name,precision,D,weighted,pattern", DENSE_CASES, ids=[c[0] for c in DENSE_CASES])
def test_dense_gradients_are_bit_identical(name, precision, D, weighted, pattern):
    import torch
    A, h0 = dense_batch(D, weighted)
    b, v = h0.shape[:2]
    dw = O.init_dense_weights({"hidden_size": D}, DENSE_T, np.random.default_rng(5))
    dw["cand_bias"] = np.random.default_rng(6).normal(0, 0.1, D).astype(np.float32)
    g_out = np.random.default_rng(7).normal(size=h0.shape).astype(np.float32)
    tw = {k: torch.tensor(x, dtype=torch.float64, requires_grad=True) for k, x in dw.items()}
    th0 = torch.tensor(h0, dtype=torch.float64, requires_grad=True)
    out = O.dense_propagation_torch(th0, A, tw, {"num_timesteps": 3, "use_edge_bias": True}, dtype=torch.float64)
    (out * torch.tensor(g_out, dtype=torch.float64)).sum().backward()
    w_eng = [dict(dw, edge_biases=dw["edge_biases"].reshape(DENSE_T, D))]
    ref = (out.detach().numpy().reshape(b * v, D), th0.grad.numpy().reshape(b * v, D),
           [{k: tw[k].grad.numpy().reshape(w_eng[0][k].shape) for k in tw}])
    t, _, _ = _check_repeatable(lambda: _Det(dense_params(D), DENSE_T, w_eng, lambda e: e.set_graph_dense(A), h0.reshape(b * v, D),
                                             g_out.reshape(b * v, D), precision), ref, "dense " + name)
    assert plan_matches(t.plan, pattern), (pattern, t.plan)


# ---------------------------------------------------------------------------------------------------------------- GCN backward
@pytest.mark.parametrize("name,precision,D,kind,keep,env,pattern", GCN_CASES, ids=[c[0] for c in GCN_CASES])
@pytest.mark.parametrize("bias_only", [False, True], ids=["full", "bias-only"])
def test_gcn_gradients_are_bit_identical(name, precision, D, kind, keep, env, pattern, bias_only, monkeypatch):
    import torch
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    _set_env(monkeypatch, env)
    V, lst, w, ks, bs, h0 = gcn_batch(D, kind)
    g_out = torch.from_numpy(np.random.default_rng(5).normal(0, 1, (V, D)).astype(np.float32)).cuda()

    def engine():
        e = GCNEngine(D, GCN_LAYERS, use_bias=True, precision=precision)
        e.set_deterministic(True)
        e.set_weights([torch.from_numpy(k).cuda() for k in ks], [torch.from_numpy(b).cuda() for b in bs])
        e.set_save_for_backward(True)
        e.set_state_dropout(keep, 77)
        e.set_graph_gcn(V, lst, w)
        e.h0_keepalive = torch.from_numpy(h0).cuda()   # the backward reads the forward's input again
        out = e.forward(e.h0_keepalive)
        assert plan_matches(e.plan, pattern), (pattern, e.plan)
        return e, out.cpu().numpy()

    def backward(e, prefill):
        gk = [torch.from_numpy(p[0]).cuda() for p in prefill]
        gb = [torch.from_numpy(p[1]).cuda() for p in prefill]
        dh0 = torch.empty(V, D, device="cuda")
        e.backward(g_out, [{"kernel": None if bias_only else a, "bias": b} for a, b in zip(gk, gb)], d_h0=dh0)
        e.sync_check()
        return [dh0.cpu().numpy()] + [x.cpu().numpy() for x in gk + gb]

    zero = [(np.zeros((D, D), np.float32), np.zeros(D, np.float32)) for _ in range(GCN_LAYERS)]
    rng = np.random.default_rng(9)
    pre = [(rng.normal(0, 1, (D, D)).astype(np.float32), rng.normal(0, 1, D).astype(np.float32)) for _ in range(GCN_LAYERS)]
    e1, out1 = engine()
    a = backward(e1, zero)
    b = backward(e1, zero)
    e2, out2 = engine()
    c = backward(e2, zero)
    p = backward(e1, pre)
    _same(out2, out1, name + " forward")
    flat_pre = [np.zeros((V, D), np.float32)] + [x[0] for x in pre] + [x[1] for x in pre]
    for i, (x, y, z, q, f) in enumerate(zip(a, b, c, p, flat_pre)):
        _same(y, x, "%s array %d second call" % (name, i))
        _same(z, x, "%s array %d fresh engine" % (name, i))
        if i > 0:
            _same(q, (f if bias_only and i <= GCN_LAYERS else f + x), "%s array %d prefill" % (name, i))
    if not bias_only:   # the float64 bar of the GCN gradient test
        masks = [e1.state_dropout_mask(l, keep, 77) for l in range(GCN_LAYERS - 1)] if keep < 1 else None
        th0 = torch.from_numpy(h0).double().requires_grad_()
        tk = [torch.from_numpy(k).double().requires_grad_() for k in ks]
        tb = [torch.from_numpy(b).double().requires_grad_() for b in bs]
        out = G.gcn_propagation_torch(th0, lst, torch.from_numpy(w).double(), tk, tb, masks, keep)
        out.backward(g_out.cpu().double())
        refs = [th0.grad.numpy()] + [t.grad.numpy() for t in tk + tb]
        for i, (x, r) in enumerate(zip(a, refs)):
            assert U.max_rel_err(x, r) < 2.5e-5, (name, i, U.max_rel_err(x, r))


# ---------------------------------------------------------------------------------------------------------------- readout
def _readout_direct(eng, last_h, h0, w, Gw):
    """ggnn_readout_forward / _backward without the autograd node (which sets the mode from torch's flag)."""
    import torch
    args = [torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in (last_h, h0, w["w_gate"], w["b_gate"], w["w_trans"],
                                                                                    w["b_trans"])]
    out = eng.readout_forward(*args)
    d_h, d_wg, d_bg, d_wt, d_bt = eng.readout_backward(*args, torch.from_numpy(Gw).cuda())
    eng.sync_check()
    g = {"w_gate": d_wg.view(-1, 1), "b_gate": d_bg, "w_trans": d_wt.view(-1, 1), "b_trans": d_bt}
    return out.cpu().numpy(), d_h.cpu().numpy(), {k: v.cpu().numpy() for k, v in g.items()}


@pytest.mark.parametrize("layout", ["grouped", "shuffled", "masked"])
@pytest.mark.parametrize("D", [20, 100, 256])
def test_readout_is_bit_identical_in_either_call_order(layout, D):
    from tests.test_gpu_readout import _case, _engine, _ref
    Gn = 37
    mask = None
    if layout == "masked":
        Gn, v = 9, 16
        last_h, h0, w, Gw = _case(Gn * v, D, Gn, 5)
        mask = (np.random.default_rng(6).random((Gn, v)) < 0.7).astype(np.float32)
        kw, ref_kw = dict(nodes_per_graph=v, node_mask=mask), dict(node_mask=mask)
    else:
        sizes = np.random.default_rng(3 + D).integers(1, 30, Gn)
        sizes[5] = 0
        gnl = np.repeat(np.arange(Gn, dtype=np.int32), sizes)
        if layout == "shuffled":
            gnl = np.random.default_rng(4 + D).permutation(gnl)
        last_h, h0, w, Gw = _case(gnl.shape[0], D, Gn, 11 + D)
        kw, ref_kw = dict(graph_nodes_list=gnl), dict(graph_nodes_list=gnl, num_graphs=Gn)
    results = []
    for before in (True, False, True):
        eng = _engine(D)
        if before:
            eng.set_deterministic(True)
        eng.readout_set_graphs(Gn, **kw)
        eng.set_deterministic(True)
        results.append(_readout_direct(eng, last_h, h0, w, Gw))
        results.append(_readout_direct(eng, last_h, h0, w, Gw))
    out, dh, dw = results[0]
    for o, d, g in results[1:]:
        _same(o, out, "forward")
        _same(d, dh, "d h_last")
        for k in dw:
            _same(g[k], dw[k], "d " + k)
    if layout == "masked":
        b = Gn
        r_out, r_dh, r_dw = _ref(last_h.reshape(b, -1, D), h0.reshape(b, -1, D), w, Gw, **ref_kw)
        r_dh = r_dh.reshape(-1, D)
    else:
        r_out, r_dh, r_dw = _ref(last_h, h0, w, Gw, **ref_kw)
    assert U.max_rel_err(out, r_out) < 1e-4 and U.max_rel_err(dh, r_dh) < 1e-4   # the bar of tests/test_gpu_readout.py
    for k in r_dw:
        assert U.max_rel_err(dw[k], r_dw[k]) < 1e-4, k


# ---------------------------------------------------------------------------------------------------------------- benchmark batches
ORDER_NOISE = 5e-5   # the atomic path's run-to-run ordering noise is ~1e-6 of the largest entry; a dropped or overwritten partial is >1e-3


def _agree_with_atomic(t, dh0, g, tag):
    """The same engine's atomic backward (ggnn_set_deterministic off) on the same forward: d h0 bit-identical, every weight and bias
    gradient within the ordering noise of the atomic sums."""
    t.eng.set_deterministic(False)
    dh0_a, ga = t.backward()
    t.eng.set_deterministic(True)
    _same(dh0_a, dh0, tag + " d h0 atomic")
    worst = (0.0, "")
    for l, (x, y) in enumerate(zip(g, ga)):
        for k in x:
            err = U.max_rel_err(x[k], y[k]) if np.any(y[k]) else float(np.max(np.abs(x[k])))
            worst = max(worst, (err, "layer %d %s" % (l, k)))
            assert err < ORDER_NOISE, (tag, l, k, err)
    print("\n%-44s deterministic vs atomic: worst %.2e on %s" % (tag, worst[0], worst[1]))


@pytest.mark.parametrize("name,precision", [("cfg4", "bf16x3"), ("default_batch_100k_nodes", "bf16x3")])
def test_benchmark_batches_give_identical_gradients_on_two_engines(name, precision):
    """Two engines agree bit for bit, and both agree with the atomic path (a systematic error would reproduce on both engines)."""
    from gated_graph_neural_network_samples_b200 import workloads
    wl = workloads.build(name)
    p, T = wl["engine_params"], wl["num_edge_types"]
    g_out = np.random.default_rng(5).normal(size=wl["h0"].shape).astype(np.float32)
    make = lambda: _Det(p, T, wl["weights"], lambda e: e.set_graph_sparse(wl["adjacency_lists"], wl["num_incoming_edges_per_type"]),
                        wl["h0"], g_out, precision)
    a, b = make(), make()
    _same(b.out, a.out, name + " forward")
    dh0_a, ga = a.backward()
    dh0_b, gb = b.backward()
    _same(dh0_b, dh0_a, name + " d h0")
    for l, (x, y) in enumerate(zip(ga, gb)):
        for k in x:
            _same(y[k], x[k], "%s layer %d %s" % (name, l, k))
    _agree_with_atomic(a, dh0_a, ga, name)


# Batches large enough that the deterministic split count is not capped by the row count (ceil(V/64)), with layers of different
# residual counts: the workspace a launch needs is not monotone in its segment count (fewer segments get more splits), so each layer's
# launches must be sized on their own.  The plug-in's default residuals {"2": [0], "4": [0, 2]} on the 256-molecule batch and on the
# 100 000-node batch; GRU and RNN on the tile-local kernel, CudnnCompatibleGRUCell (which adds the R+1- and 1-segment projection
# launches) and attention on the fp32 kernel.
DEFAULT_RES = {"layer_timesteps": [2, 2, 1, 2, 1], "residual_connections": {"2": [0], "4": [0, 2]}}
UNCAPPED = {
    "cfg1-gru": ("cfg1_true_default", dict(DEFAULT_RES, graph_rnn_cell="GRU", graph_rnn_activation="tanh"), "bf16x3"),
    "cfg1-rnn": ("cfg1_true_default", dict(DEFAULT_RES, graph_rnn_cell="RNN", graph_rnn_activation="tanh", use_edge_bias=True), "bf16x3"),
    "cfg1-cudnn": ("cfg1_true_default", dict(DEFAULT_RES, graph_rnn_cell="CudnnCompatibleGRUCell", graph_rnn_activation="tanh"), "fp32"),
    "cfg1-attention": ("cfg1_true_default", dict(DEFAULT_RES, use_propagation_attention=True, use_edge_bias=True), "fp32"),
    "100k-default-residuals-gru": ("default_batch_100k_nodes", DEFAULT_RES, "bf16x3"),
}


@pytest.mark.parametrize("case", sorted(UNCAPPED))
def test_uncapped_splits_agree_with_the_atomic_path(case):
    from gated_graph_neural_network_samples_b200 import workloads
    name, over, precision = UNCAPPED[case]
    wl = workloads.build(name)
    p, T = dict(wl["engine_params"], **over), wl["num_edge_types"]
    w = _weights(p, T)
    g_out = np.random.default_rng(5).normal(size=wl["h0"].shape).astype(np.float32)
    t = _Det(p, T, w, lambda e: e.set_graph_sparse(wl["adjacency_lists"], wl["num_incoming_edges_per_type"]), wl["h0"], g_out, precision)
    dh0, g = t.backward()
    dh0_b, g_b = t.backward()
    _same(dh0_b, dh0, case + " d h0 twice")
    for l, (x, y) in enumerate(zip(g, g_b)):
        for k in x:
            _same(y[k], x[k], "%s layer %d %s twice" % (case, l, k))
    _agree_with_atomic(t, dh0, g, case)


# ---------------------------------------------------------------------------------------------------------------- end to end
_CHILD = r"""
import json, pickle, sys
import numpy as np
import torch
torch.use_deterministic_algorithms(True)
from gated_graph_neural_network_samples_b200 import synthetic
from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
from gated_graph_neural_network_samples_b200.chem_dense import DenseGGNNChemModel
from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
kind, cfg, out_dir, ckpt = sys.argv[1], json.loads(sys.argv[2]), sys.argv[3], sys.argv[4]
mols = synthetic.make_molecules(96, seed=11, num_bond_types=cfg.pop("bond_types", 4))
rng = np.random.default_rng(12)
for m in mols:                                # two tasks
    m["targets"] = [m["targets"][0], [float(rng.normal())]]
model = {"sparse": SparseGGNNChemModel, "dense": DenseGGNNChemModel, "gcn": SparseGCNChemModel}[kind]
m = model({"--log_dir": out_dir, "--train_data": mols[:80], "--valid_data": mols[80:], "--precision": cfg.pop("precision", "fp32"),
           "--config": dict(cfg, task_ids=[0, 1], task_sample_ratios={"1": 0.5}, learning_rate=0.01, num_epochs=2, random_seed=3)})
losses = []
for ep in range(2):
    losses.append(float(m.run_epoch("train%d" % ep, m.train_data, True)[0]))
    losses.append(float(m.run_epoch("valid%d" % ep, m.valid_data, False)[0]))
m.save_progress(ckpt, 2, 0)
print("LOSSES " + json.dumps(losses))
"""

SPARSE_TRAIN = {"batch_size": 400, "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}, "edge_weight_dropout_keep_prob": 0.8,
                "graph_state_dropout_keep_prob": 0.9, "out_layer_dropout_keep_prob": 0.9}
E2E = {
    "sparse-bf16x3-tile-local-D100": ("sparse", dict(SPARSE_TRAIN, hidden_size=100, precision="bf16x3")),
    "sparse-bf16x3-streaming-D256-T8": ("sparse", dict(SPARSE_TRAIN, hidden_size=256, precision="bf16x3", bond_types=8)),
    "sparse-fp32-attention": ("sparse", dict(SPARSE_TRAIN, hidden_size=36, use_propagation_attention=True, use_edge_bias=True)),
    "sparse-padded-D30-torch-readout": ("sparse", dict(SPARSE_TRAIN, hidden_size=30)),
    "dense": ("dense", {"hidden_size": 32, "batch_size": 8, "num_timesteps": 3, "graph_state_dropout_keep_prob": 0.9,
                        "out_layer_dropout_keep_prob": 0.9}),
    "gcn": ("gcn", {"hidden_size": 64, "batch_size": 400, "num_timesteps": 3, "gcn_use_bias": True, "graph_state_dropout_keep_prob": 0.9,
                    "out_layer_dropout_keep_prob": 0.9}),
}


@pytest.mark.parametrize("name", sorted(E2E))
def test_training_runs_repeat_bit_for_bit(name, tmp_path):
    kind, cfg = E2E[name]
    runs = []
    for i in range(2):
        ckpt = str(tmp_path / ("run%d.pickle" % i))
        env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8", PYTHONPATH=REPO)
        res = subprocess.run([sys.executable, "-c", _CHILD, kind, json.dumps(cfg), str(tmp_path / ("log%d" % i)), ckpt], env=env, cwd=REPO,
                             capture_output=True, text=True, timeout=900)
        assert res.returncode == 0, res.stderr[-3000:]
        losses = json.loads(next(l for l in res.stdout.splitlines() if l.startswith("LOSSES "))[7:])
        runs.append((losses, pickle.load(open(ckpt, "rb"))["weights"]))
    (la, wa), (lb, wb) = runs
    print("\n%s losses %s" % (name, la))
    assert all(np.isfinite(la))
    assert la == lb, (la, lb)
    assert sorted(wa) == sorted(wb)
    assert any(k.endswith("/Adam:0") for k in wa) and any(k.endswith("/Adam_1:0") for k in wa)
    for k in wa:
        _same(wb[k], wa[k], k)
