"""GPU: the bf16x3 tensor-core backward (``ggnn_set_backward_precision(GGNN_PREC_BF16X3)``) against float64 autograd.

Every GEMM of ``ggnn_backward`` / ``ggnn_gcn_backward`` but the edge-bias gradient runs on the wgmma kernels of ggnn_bwd_tc.cuh with this
setting.  Each case runs a forward with save_for_backward, sets the backward precision in the graph callback (after engine creation,
before the forward), runs the backward and compares the forward, ``d h0`` and every weight and bias gradient with float64 autograd at
max|err| / max|ref| < 2e-4 per tensor (the bf16x3 bar of the other gradient files).  The cases are those of
tests/test_gpu_backward_plans.py, each with the forward precision of its plan and with the other one; the tile tails of the two kernels
(hidden sizes, node counts, an empty batch); the long reductions of the benchmark batches; partial requests, prefilled buffers and
determinism; switching the setting on one saved forward; refusals; and the three plug-ins with ``--backward-precision bf16x3``.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import ggnn_oracle as O
from tests import _util as U
from tests import gcn_oracle as G
from tests.test_backward_plans_cpu import (DENSE_CASES, DETERMINISM_CASES, EDGE_SHAPES, GCN_CASES, GCN_LAYERS, PARTIAL_CASES, PLAN_MATRIX,
                                           SPARSE_CASES, dense_batch, dense_params, gcn_batch, plan_matches, smooth_on_tensor_cores,
                                           sparse_batch)
from tests.test_gpu_backward import _autograd_reference, _cmp, _engine_grads

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REN = {"rnn_kernel": "cand_kernel", "rnn_bias": "cand_bias"}
BAR = 2e-4


def _weights(p, T, seed=1):
    from tests.test_gpu_backward_plans import _weights as w
    return w(p, T, seed)


def _compare(tag, got, ref):
    from tests.test_gpu_backward_plans import _compare as c
    c(tag + " [bwd bf16x3]", got, ref)


def _same(a, b, tag):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes(), (tag, U.max_rel_err(a, b) if b.size else 0.0)


def _bf16x3_graph(set_graph):
    def f(e):
        e.set_backward_precision("bf16x3")
        set_graph(e)
    return f


def _flip(c):
    """The case with the other forward precision: the plan family follows the precision (attention and CudnnCompatibleGRUCell stay on the
    fp32 kernel), tanh on the tensor-core forward (smooth_on_tensor_cores), no plan-forcing environment."""
    prec = "fp32" if c.precision == "bf16x3" else "bf16x3"
    p = dict(c.params)
    if prec == "bf16x3":
        p["graph_rnn_activation"] = smooth_on_tensor_cores(prec)
    fp32_only = p.get("use_propagation_attention") or p["graph_rnn_cell"] == "CudnnCompatibleGRUCell"
    plan = r"^fp32-ffma" if prec == "fp32" or fp32_only else r"^wgmma-bf16x3 "
    return p, prec, {}, plan


def _run_sparse(tag, params, T, batch, precision, env, plan, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    adj, indeg, h0 = sparse_batch(batch, params["hidden_size"], T)
    w = _weights(params, T)
    g_out = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    ref = _autograd_reference(params, T, w, adj, indeg, h0, g_out)
    plans = []

    def set_graph(e):
        e.set_graph_sparse(adj, indeg)
        plans.append(e.plan)

    got = _engine_grads(params, T, w, _bf16x3_graph(set_graph), h0, g_out, precision)
    assert plan_matches(plans[0], plan), (plan, plans[0])
    _compare(tag, got, ref)


@pytest.mark.parametrize("forward", ["plan", "flipped"])
@pytest.mark.parametrize("case", [c.name for c in PLAN_MATRIX + EDGE_SHAPES])
def test_gradients_on_every_plan_and_edge_shape(case, forward, monkeypatch):
    """Every forward plan (GRU, RNN, CudnnCompatibleGRUCell, attention), T = 1 / 3 / 17 / 32, four residuals, a zero-step layer; each
    with the plan's forward precision and with the other one (the backward setting is independent of the forward)."""
    c = SPARSE_CASES[case]
    if forward == "plan":
        _run_sparse(c.name, c.params, c.T, c.batch, c.precision, c.env, c.plan, monkeypatch)
    else:
        p, prec, env, plan = _flip(c)
        _run_sparse(c.name + " flipped", p, c.T, c.batch, prec, env, plan, monkeypatch)


# ---------------------------------------------------------------------------------------------------------------- tile tails
def _model(D, cell="GRU", T=4):
    return {"hidden_size": D, "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}, "use_edge_bias": True,
            "use_edge_msg_avg_aggregation": True, "graph_rnn_cell": cell, "graph_rnn_activation": "tanh"}


@pytest.mark.parametrize("D", [4, 12, 36, 100, 128, 132, 256, 260, 512])
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_hidden_size_tails(D, precision, monkeypatch):
    """K and N tails of both kernels: N = D, 2D, (R+2)D, K = D; hidden 4 (one 4-wide k-chunk) to 512 (four 128-wide data-gradient
    tiles, eight 64-wide weight-gradient tiles)."""
    _run_sparse("D%d %s" % (D, precision), _model(D), 4, "mol24", precision, {}, r"^(fp32-ffma|fp32-stepwise|wgmma-bf16x3) ", monkeypatch)


def _random_graph(V, T, seed):
    rng = np.random.default_rng(seed)
    adj = []
    for t in range(T):
        E = int(rng.integers(0, 2 * V + 1)) if V > 0 else 0
        adj.append(rng.integers(0, max(V, 1), (E, 2)).astype(np.int32) if V > 0 else np.zeros((0, 2), np.int32))
    indeg = np.zeros((V, T), np.float32)
    for t, a in enumerate(adj):
        np.add.at(indeg[:, t], a[:, 1], 1.0)
    return adj, indeg


@pytest.mark.parametrize("V", [1, 15, 17, 63, 65, 129])
@pytest.mark.parametrize("cell", ["GRU", "RNN"])
def test_node_count_tails(V, cell):
    """M tails of the data-gradient tile (128 rows) and the row tails of the weight-gradient slabs (32 rows), V < 16 included."""
    T, D = 3, 20
    p = _model(D, cell)
    adj, indeg = _random_graph(V, T, V)
    h0 = np.random.default_rng(V).normal(0, 1, (V, D)).astype(np.float32)
    w = _weights(p, T)
    g_out = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    ref = _autograd_reference(p, T, w, adj, indeg, h0, g_out)
    got = _engine_grads(p, T, w, _bf16x3_graph(lambda e: e.set_graph_sparse(adj, indeg)), h0, g_out, "fp32")
    _compare("V%d %s" % (V, cell), got, ref)


def test_empty_batch():
    T, D = 3, 20
    p = _model(D)
    adj, indeg = _random_graph(0, T, 0)
    h0 = np.zeros((0, D), np.float32)
    out, dh0, gw = _engine_grads(p, T, _weights(p, T), _bf16x3_graph(lambda e: e.set_graph_sparse(adj, indeg)), h0, h0, "bf16x3")
    assert out.shape == dh0.shape == (0, D)
    assert all(not np.any(a) for lw in gw for a in lw.values())


# ---------------------------------------------------------------------------------------------------------------- dense and GCN
@pytest.mark.parametrize("name,precision,D,weighted,pattern", DENSE_CASES, ids=[c[0] for c in DENSE_CASES])
def test_dense_gradients(name, precision, D, weighted, pattern):
    import torch
    A, h0 = dense_batch(D, weighted)
    b, v = h0.shape[:2]
    dw = O.init_dense_weights({"hidden_size": D}, 4, np.random.default_rng(5))
    dw["cand_bias"] = np.random.default_rng(6).normal(0, 0.1, D).astype(np.float32)
    g_out = np.random.default_rng(7).normal(size=h0.shape).astype(np.float32)
    tw = {k: torch.tensor(x, dtype=torch.float64, requires_grad=True) for k, x in dw.items()}
    th0 = torch.tensor(h0, dtype=torch.float64, requires_grad=True)
    out = O.dense_propagation_torch(th0, A, tw, {"num_timesteps": 3, "use_edge_bias": True}, dtype=torch.float64)
    (out * torch.tensor(g_out, dtype=torch.float64)).sum().backward()
    plans = []

    def set_graph(e):
        e.set_graph_dense(A)
        plans.append(e.plan)

    w_eng = [dict(dw, edge_biases=dw["edge_biases"].reshape(4, D))]
    o2, dh0, gw = _engine_grads(dense_params(D), 4, w_eng, _bf16x3_graph(set_graph), h0.reshape(b * v, D), g_out.reshape(b * v, D), precision)
    assert plan_matches(plans[0], pattern), (pattern, plans[0])
    ref_gw = [{k: tw[k].grad.numpy().reshape(gw[0][k].shape) for k in tw}]
    _compare("dense " + name, (o2.reshape(b, v, D), dh0.reshape(b, v, D), gw), (out.detach().numpy(), th0.grad.numpy(), ref_gw))


def _gcn_check(tag, eng, V, D, L, lst, w, h0, ks, bs, got, keep, seed):
    import torch
    g_out = np.random.default_rng(5).normal(0, 1, (V, D)).astype(np.float32)
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
    errs = [("forward", U.max_rel_err(got, out.detach().numpy())), ("d h0", U.max_rel_err(dh0.cpu().numpy(), th0.grad.numpy()))]
    for l in range(L):
        errs += [("layer %d kernel" % l, U.max_rel_err(gk[l].cpu().numpy(), tk[l].grad.numpy())),
                 ("layer %d bias" % l, U.max_rel_err(gb[l].cpu().numpy(), tb[l].grad.numpy()))]
    worst = max((e, n) for n, e in errs[1:])
    print("\n%-36s forward %.2e  worst gradient %.2e on %s" % ("gcn " + tag, errs[0][1], worst[0], worst[1]))
    for n, e in errs:
        assert e < (1e-4 if n == "forward" else BAR), (tag, n, e)


@pytest.mark.parametrize("name,precision,D,kind,keep,env,pattern", GCN_CASES, ids=[c[0] for c in GCN_CASES])
def test_gcn_gradients(name, precision, D, kind, keep, env, pattern, monkeypatch):
    from tests.test_gpu_gcn import run
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    V, lst, w, ks, bs, h0 = gcn_batch(D, kind)
    got, eng = run(D, GCN_LAYERS, V, lst, w, h0, ks, bs, precision, keep=keep, seed=77, save=True)
    assert plan_matches(eng.plan, pattern), (pattern, eng.plan)
    eng.set_backward_precision("bf16x3")
    _gcn_check(name, eng, V, D, GCN_LAYERS, lst, w, h0, ks, bs, got, keep, 77)


# ---------------------------------------------------------------------------------------------------------------- long reductions
def _workload_case(name, over=None, D=None, T=None):
    from gated_graph_neural_network_samples_b200 import workloads
    wl = workloads.build(name)
    p = dict(wl["engine_params"], **(over or {}))
    if D is not None:
        p["hidden_size"] = D
    T = T or wl["num_edge_types"]
    return p, T, wl


@pytest.mark.parametrize("name", ["cfg4", "default_batch_100k_nodes"])
def test_long_reductions_on_benchmark_batches(name):
    """cfg4 (hidden 256, 8 edge types, 18 481 nodes) and the 100 000-node batch: weight-gradient splits of thousands of rows, the
    data-gradient sum over 8 edge types."""
    p, T, wl = _workload_case(name, {"graph_rnn_activation": "tanh"})
    w = _weights(p, T)
    adj, indeg, h0 = wl["adjacency_lists"], wl["num_incoming_edges_per_type"], wl["h0"]
    g_out = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    ref = _autograd_reference(p, T, w, adj, indeg, h0, g_out)
    got = _engine_grads(p, T, w, _bf16x3_graph(lambda e: e.set_graph_sparse(adj, indeg)), h0, g_out, "bf16x3")
    _compare(name, got, ref)


def test_long_reductions_hidden_512_with_32_edge_types():
    """dh += sum_t G_t . W_t^T over T*D = 16 384: the longest data-gradient reduction one CTA owns."""
    from tests.test_backward_plans_cpu import component_graph
    T, D = 32, 512
    p = _model(D)
    adj, indeg = component_graph(T, seed=T)
    h0 = np.random.default_rng(3).normal(0, 1, (indeg.shape[0], D)).astype(np.float32)
    w = _weights(p, T)
    g_out = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    ref = _autograd_reference(p, T, w, adj, indeg, h0, g_out)
    got = _engine_grads(p, T, w, _bf16x3_graph(lambda e: e.set_graph_sparse(adj, indeg)), h0, g_out, "bf16x3")
    _compare("D512 T32", got, ref)


def test_long_reductions_gcn_100k_nodes():
    """dW = S^T . dPre over 99 046 rows.  One layer, which is linear: with relu between layers, pre-activations within the forward's
    rounding of 0 can take the other side of the kink than in float64 at some of the 6.3 million units (smooth_on_tensor_cores), and
    that node's d h0 then differs by O(1) -- the activation, not a GEMM."""
    from gated_graph_neural_network_samples_b200 import packing, synthetic
    from gated_graph_neural_network_samples_b200.engine import GCNEngine
    import torch
    D, L = 64, 1
    mols = synthetic.make_molecules(5500, seed=0)
    b = packing.pack_gcn_batch(packing.process_raw_graphs_gcn(mols), D)
    V = b["initial_node_representation"].shape[0]
    assert V > 99000   # the 100 000-node batch of tools/gcn_bench.py: 99 046 nodes
    rng = np.random.default_rng(1)
    ks = [G.glorot((D, D), rng) for _ in range(L)]
    bs = [rng.normal(0, 0.2, D).astype(np.float32) for _ in range(L)]
    h0 = rng.normal(0, 1, (V, D)).astype(np.float32)
    eng = GCNEngine(D, L, use_bias=True, precision="bf16x3")
    eng.set_backward_precision("bf16x3")
    eng.set_weights([torch.from_numpy(k).cuda() for k in ks], [torch.from_numpy(x).cuda() for x in bs])
    eng.set_save_for_backward(True)
    eng.set_graph_gcn(V, b["adjacency_list"], b["adjacency_weights"])
    h0_dev = torch.from_numpy(h0).cuda()   # kept alive: the backward recomputes S from the forward's input
    got = eng.forward(h0_dev).cpu().numpy()
    _gcn_check("100k", eng, V, D, L, b["adjacency_list"], np.asarray(b["adjacency_weights"], np.float32), h0, ks, bs, got, 1.0, 0)


# ---------------------------------------------------------------------------------------------------------------- one engine, many calls
class _Trained:
    """One engine after a forward with save_for_backward, bf16x3 backward; ``backward(fields, prefill)`` accumulates into buffers holding
    ``prefill`` (None: zeros) and returns (d h0, per-layer gradients) as NumPy."""

    def __init__(self, params, T, w, set_graph, h0, g_out, precision, det=False):
        import torch
        from gated_graph_neural_network_samples_b200.engine import PropagationEngine
        self.eng = PropagationEngine(params, T, precision=precision)
        self.eng.set_deterministic(det)
        self.eng.set_backward_precision("bf16x3")
        self.dev_w = [{REN.get(k, k): torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda() for k, v in lw.items()} for lw in w]
        self.eng.set_weights(self.dev_w)
        self.eng.set_save_for_backward(True)
        set_graph(self.eng)
        self.plan = self.eng.plan
        self.h0 = torch.from_numpy(np.ascontiguousarray(h0, np.float32)).cuda()
        self.out_t = self.eng.forward(self.h0)
        self.g_out = torch.from_numpy(np.ascontiguousarray(g_out, np.float32)).cuda()
        self.fields = sorted(self.dev_w[0])

    def backward(self, fields=None, prefill=None, want_dh0=True):
        import torch
        fields = self.fields if fields is None else fields
        grads = [{k: (torch.zeros_like(lw[k]) if prefill is None else torch.from_numpy(prefill[l][k]).cuda()) for k in fields if k in lw}
                 for l, lw in enumerate(self.dev_w)]
        dh0 = torch.zeros_like(self.h0) if want_dh0 else None
        self.eng.backward(self.g_out, grads, dh0)
        self.eng.sync_check()
        return (None if dh0 is None else dh0.cpu().numpy()), [{k: v.cpu().numpy() for k, v in lw.items()} for lw in grads]


def _trained(case, monkeypatch, det=False):
    c = SPARSE_CASES[case]
    for k, v in c.env.items():
        monkeypatch.setenv(k, v)
    adj, indeg, h0 = sparse_batch(c.batch, c.params["hidden_size"], c.T)
    w = _weights(c.params, c.T)
    g_out = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    make = lambda: _Trained(c.params, c.T, w, lambda e: e.set_graph_sparse(adj, indeg), h0, g_out, c.precision, det)
    return make


NOISE = 1e-5   # atomic-order noise of the weight-gradient sums, relative to the largest entry


def _close(a, b, tag):
    err = U.max_rel_err(a, b) if np.any(b) else float(np.max(np.abs(a)))
    assert err < NOISE, (tag, err)


@pytest.mark.parametrize("case", PARTIAL_CASES)
def test_partial_requests_and_prefilled_buffers(case, monkeypatch):
    """Only d h0, only the edge weights, only the biases (kernels null: the column sums) against a full request; buffers prefilled with
    P end as P + G."""
    t = _trained(case, monkeypatch)()
    full_dh0, full = t.backward()
    dh0, none = t.backward([])
    _same(dh0, full_dh0, "d h0 alone")
    assert all(not lw for lw in none)
    for request in (["edge_weights"], [k for k in t.fields if "bias" in k]):
        dh0, part = t.backward(request, want_dh0=False)
        assert dh0 is None
        for l, (p, f) in enumerate(zip(part, full)):
            assert sorted(p) == sorted(request), (p.keys(), request)
            for k in p:
                _close(p[k], f[k], "layer %d %s" % (l, k))
    rng = np.random.default_rng(9)
    prefill = [{k: rng.normal(0, 1, v.shape).astype(np.float32) for k, v in lw.items()} for lw in full]
    dh0, pre = t.backward(prefill=prefill)
    _same(dh0, full_dh0, "d h0 prefilled")
    for l, (x, y, p) in enumerate(zip(full, pre, prefill)):
        for k in x:
            _close(y[k], p[k] + x[k], "layer %d %s prefill" % (l, k))


def _check_repeatable(make, tag):
    """Deterministic mode: two calls, a fresh engine and a prefilled buffer give identical bits."""
    t = make()
    dh0, g = t.backward()
    dh0_b, g_b = t.backward()
    dh0_c, g_c = make().backward()
    rng = np.random.default_rng(9)
    prefill = [{k: rng.normal(0, 1, v.shape).astype(np.float32) for k, v in lw.items()} for lw in g]
    _, g_p = t.backward(prefill=prefill)
    for other, odh0, name in ((g_b, dh0_b, "second call"), (g_c, dh0_c, "fresh engine")):
        _same(odh0, dh0, "%s d h0 %s" % (tag, name))
        for l, (x, y) in enumerate(zip(g, other)):
            for k in x:
                _same(y[k], x[k], "%s layer %d %s %s" % (tag, l, k, name))
    for l, (x, y, p) in enumerate(zip(g, g_p, prefill)):
        for k in x:
            _same(y[k], p[k] + x[k], "%s layer %d %s prefill" % (tag, l, k))
    return t, dh0


@pytest.mark.parametrize("case", DETERMINISM_CASES)
def test_deterministic_mode_is_bit_identical(case, monkeypatch):
    _check_repeatable(_trained(case, monkeypatch, det=True), case)


@pytest.mark.parametrize("case", DETERMINISM_CASES)
def test_d_h0_is_bit_identical_run_to_run_in_atomic_mode(case, monkeypatch):
    t = _trained(case, monkeypatch)()
    a, _ = t.backward()
    for _ in range(2):
        _same(t.backward()[0], a, case + " d h0")


DEFAULT_RES = {"layer_timesteps": [2, 2, 1, 2, 1], "residual_connections": {"2": [0], "4": [0, 2]}, "graph_rnn_activation": "tanh"}


@pytest.mark.parametrize("name", ["cfg1_true_default", "default_batch_100k_nodes"])
def test_uncapped_splits_are_bit_identical(name):
    """The plug-in's default residuals on 256 molecules and on the 100 000-node batch: split counts not capped by the row count, layers
    of different segment counts sharing one workspace."""
    p, T, wl = _workload_case(name, DEFAULT_RES)
    w = _weights(p, T)
    g_out = np.random.default_rng(5).normal(size=wl["h0"].shape).astype(np.float32)
    set_graph = lambda e: e.set_graph_sparse(wl["adjacency_lists"], wl["num_incoming_edges_per_type"])
    _check_repeatable(lambda: _Trained(p, T, w, set_graph, wl["h0"], g_out, "bf16x3", det=True), name)


@pytest.mark.parametrize("case", ["tc-local64-gru-D100", "ffma-global-cudnn-D100", "ffma-global-attention-D36"])
def test_switching_precision_between_backward_calls(case, monkeypatch):
    """fp32 -> bf16x3 -> fp32 -> bf16x3 on one saved forward, deterministic mode: each result equals a fresh engine's at that setting,
    bit for bit; the plan text is not touched."""
    make = _trained(case, monkeypatch, det=True)
    t = make()
    plan = t.plan
    fresh_tc = make().backward()
    f = make()
    f.eng.set_backward_precision("fp32")
    fresh_fp = f.backward()
    for prec in ("fp32", "bf16x3", "fp32", "bf16x3"):
        t.eng.set_backward_precision(prec)
        dh0, g = t.backward()
        rdh0, rg = fresh_tc if prec == "bf16x3" else fresh_fp
        _same(dh0, rdh0, "%s d h0" % prec)
        for l, (x, y) in enumerate(zip(g, rg)):
            for k in x:
                _same(x[k], y[k], "%s layer %d %s" % (prec, l, k))
    assert t.eng.plan == plan


def test_refused_values_keep_the_setting(monkeypatch):
    from gated_graph_neural_network_samples_b200 import _lib
    from gated_graph_neural_network_samples_b200.engine import GgnnError
    make = _trained("tc-local64-gru-D20", monkeypatch, det=True)
    t = make()
    ref = t.backward()
    for bad in (2, 3, -1, 1 << 20):   # GGNN_PREC_BF16 and out-of-range values
        assert t.eng.lib.ggnn_set_backward_precision(t.eng._h, bad) == -1, bad
    with pytest.raises(ValueError):
        t.eng.set_backward_precision("bf16")
    with pytest.raises(GgnnError):
        t.eng._check(t.eng.lib.ggnn_set_backward_precision(t.eng._h, 2))
    got = t.backward()
    _same(got[0], ref[0], "d h0 after refusals")
    for l, (x, y) in enumerate(zip(got[1], ref[1])):
        for k in x:
            _same(x[k], y[k], "layer %d %s after refusals" % (l, k))
    assert _lib.load().ggnn_set_backward_precision(None, 1) == -1


# ---------------------------------------------------------------------------------------------------------------- the plug-ins
def _plugin_check(tag, m, feed, monkeypatch, plan):
    """forward_batch + loss.backward() through the plug-in, every trainable's gradient against float64 autograd at 2e-4."""
    import re
    import torch
    from tests.test_gpu_chem_ggnn_gradients import Draws, _compare as cmp, _reference
    draws = Draws(m, monkeypatch)
    loss, _ = m.forward_batch(feed)
    loss.backward()
    torch.cuda.synchronize()
    assert re.search(plan, m.engine.plan), (plan, m.engine.plan)
    ref, ref_loss = _reference(m, feed, draws)
    ref_loss.backward()
    assert abs(float(loss.detach()) - float(ref_loss.detach())) <= 1e-4 * abs(float(ref_loss.detach()))
    cmp(tag, m, {n: v.grad for n, v in m.trainable_variables()}, ref, BAR)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
@pytest.mark.parametrize("kind", ["sparse", "dense"])
def test_ggnn_plugins_with_tensor_core_backward(kind, precision, tmp_path, monkeypatch):
    from gated_graph_neural_network_samples_b200.chem_dense import DenseGGNNChemModel
    from gated_graph_neural_network_samples_b200.chem_sparse import SparseGGNNChemModel
    from tests.test_gpu_chem_ggnn_gradients import DENSE_TRAINING, SPARSE_TRAINING, _training_feed, _two_task_molecules
    cls, cfg, seed = (SparseGGNNChemModel, SPARSE_TRAINING, 1) if kind == "sparse" else (DenseGGNNChemModel, DENSE_TRAINING, 2)
    cfg = dict(cfg, graph_rnn_activation="tanh")
    mols = _two_task_molecules(64, seed=seed)
    m = cls({"--log_dir": str(tmp_path), "--precision": precision, "--backward-precision": "bf16x3", "--train_data": mols[:48],
             "--valid_data": mols[48:], "--config": cfg})
    _plugin_check("%s plug-in %s forward" % (kind, precision), m, _training_feed(m), monkeypatch,
                  r"^fp32-ffma" if precision == "fp32" else r"^wgmma-bf16x3 LOCAL")


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
@pytest.mark.parametrize("keep", [1.0, 0.8])
def test_gcn_plugin_with_tensor_core_backward(tmp_path, golden_dir, precision, keep):
    """SparseGCNChemModel with --backward-precision bf16x3 on the h100_l4_bias fixture: GCN kernels and biases and both readout MLPs
    against float64 autograd."""
    import torch
    from gated_graph_neural_network_samples_b200 import synthetic
    from gated_graph_neural_network_samples_b200.chem_gcn import SparseGCNChemModel
    from gated_graph_neural_network_samples_b200.utils import SMALL_NUMBER
    from tests.test_chem_gcn_cpu import _load_fixture_weights, fixture_feed
    z = np.load(os.path.join(golden_dir, "refgraph_gcn_h100_l4_bias.npz"))
    cfg = json.loads(str(z["params_json"]))
    mols = synthetic.make_molecules(8, seed=1)
    m = SparseGCNChemModel({"--log_dir": str(tmp_path), "--precision": precision, "--backward-precision": "bf16x3", "--train_data": mols[:4],
                            "--valid_data": mols[4:], "--config": dict(cfg, batch_size=100000)})
    _load_fixture_weights(m, z, cfg)
    seeds = []
    set_dropout = m.engine.set_state_dropout
    m.engine.set_state_dropout = lambda k, seed=0: (seeds.append((k, seed)), set_dropout(k, seed))
    loss, _ = m.forward_batch(dict(fixture_feed(z), graph_state_keep_prob=keep))
    loss.backward()
    torch.cuda.synchronize()
    L, V = cfg["num_timesteps"], z["h0"].shape[0]
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
    for n, v in named.items():
        err = U.max_rel_err(v.grad.cpu().numpy(), ref[n].grad.numpy())
        assert err < BAR, (n, err)


E2E = {
    "sparse": ("sparse", {"batch_size": 400, "layer_timesteps": [2, 1], "residual_connections": {"1": [0]}, "hidden_size": 100,
                          "precision": "bf16x3", "edge_weight_dropout_keep_prob": 0.8, "graph_state_dropout_keep_prob": 0.9,
                          "out_layer_dropout_keep_prob": 0.9}),
    "dense": ("dense", {"hidden_size": 32, "batch_size": 8, "num_timesteps": 3, "graph_state_dropout_keep_prob": 0.9,
                        "out_layer_dropout_keep_prob": 0.9}),
    "gcn": ("gcn", {"hidden_size": 64, "batch_size": 400, "num_timesteps": 3, "gcn_use_bias": True, "graph_state_dropout_keep_prob": 0.9,
                    "out_layer_dropout_keep_prob": 0.9}),
}


@pytest.mark.parametrize("name", sorted(E2E))
def test_deterministic_training_runs_repeat_bit_for_bit(name, tmp_path):
    """Two deterministic two-epoch runs in fresh processes with --backward-precision bf16x3: identical losses and checkpoints."""
    import pickle
    from tests.test_gpu_deterministic import _CHILD
    child = _CHILD.replace('"--precision": cfg.pop("precision", "fp32"),', '"--precision": cfg.pop("precision", "fp32"), "--backward-precision": "bf16x3",')
    assert child != _CHILD
    kind, cfg = E2E[name]
    runs = []
    for i in range(2):
        ckpt = str(tmp_path / ("run%d.pickle" % i))
        env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8", PYTHONPATH=REPO)
        res = subprocess.run([sys.executable, "-c", child, kind, json.dumps(cfg), str(tmp_path / ("log%d" % i)), ckpt], env=env, cwd=REPO,
                             capture_output=True, text=True, timeout=900)
        assert res.returncode == 0, res.stderr[-3000:]
        losses = json.loads(next(l for l in res.stdout.splitlines() if l.startswith("LOSSES "))[7:])
        with open(ckpt, "rb") as f:
            runs.append((losses, pickle.load(f)["weights"]))
    (la, wa), (lb, wb) = runs
    print("\n%s losses %s" % (name, la))
    assert all(np.isfinite(la)) and la == lb, (la, lb)
    assert sorted(wa) == sorted(wb)
    for k in wa:
        _same(np.asarray(wb[k]), np.asarray(wa[k]), k)
