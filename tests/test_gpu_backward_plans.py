"""GPU: gradients against float64 autograd on every forward plan, and at the backward kernels' edge shapes.

``ggnn_backward`` reads the activations the forward saved (``h_in``, ``agg``, ``r``, ``u``, ``c``, and ``q`` for CudnnCompatibleGRUCell),
and each forward plan stores them with its own code: the tile-local wgmma kernel from its accumulator fragments (rows 64-127 of a tile by
the second pair of warpgroups), the streaming kernels through a column-guarded store, the fp32 kernel per row in either tile variant,
and the GCN kernels per layer.  Only a gradient test can see a wrong store, so every case here runs a forward with save_for_backward,
the backward, and compares the forward, ``d h0`` and every weight and bias gradient with float64 autograd of the oracle
(max|err| / max|ref| < 2e-4; the GCN at 2.5e-5).  Each case also asserts the plan text, so that a planner change cannot move it onto
another kernel; tests/test_backward_plans_cpu.py pins the same plans without a GPU.

Further: partial gradient requests (null ``ggnn_layer_grads`` fields, a bias without its kernel) against a full request, accumulation
into the caller's buffers, run-to-run bit identity of ``d h0`` (no float atomics on node states), the dense model on weighted and
binary matrices, and the GCN on its LOCAL-with-save, GLOBAL and fp32 plans.
"""
import numpy as np
import pytest

from oracle import ggnn_oracle as O
from tests import _util as U
from tests import gcn_oracle as G
from tests.test_backward_plans_cpu import (DENSE_CASES, DENSE_STEPS, DENSE_T, DETERMINISM_CASES, EDGE_SHAPES, GCN_CASES, GCN_LAYERS,
                                           PARTIAL_CASES, PLAN_MATRIX, SPARSE_CASES, dense_batch, dense_params, gcn_batch, plan_matches,
                                           sparse_batch)
from tests.test_gpu_backward import _autograd_reference, _cmp, _engine_grads

pytestmark = pytest.mark.gpu

REN = {"rnn_kernel": "cand_kernel", "rnn_bias": "cand_bias"}


def _weights(p, T, seed=1):
    """The oracle's initialisers, with the zero candidate biases drawn instead, so that every bias enters the forward."""
    rng = np.random.default_rng(seed)
    w = O.init_sparse_weights(p, T, rng, attention_scale=0.5)
    for lw in w:
        for k in ("cand_bias", "rnn_bias"):
            if k in lw:
                lw[k] = rng.normal(0, 0.1, lw[k].shape).astype(np.float32)
    return w


def _compare(tag, got, ref):
    """Every array of (forward, d h0, per-layer weight gradients) against the reference at the bar of _cmp; prints the forward's error
    and the worst gradient's."""
    (out, dh0, gw), (rout, rdh0, rgw) = got, ref
    pairs = [("forward", out, rout), ("d h0", dh0, rdh0)]
    pairs += [("layer %d %s" % (l, k), a[k], r[k]) for l, (a, r) in enumerate(zip(gw, rgw)) for k in sorted(r)]
    worst = max((U.max_rel_err(g, r) if np.any(r) else float(np.max(np.abs(g))), n) for n, g, r in pairs[1:])
    print("\n%-36s forward %.2e  worst gradient %.2e on %s" % (tag, U.max_rel_err(out, rout), worst[0], worst[1]))
    for n, g, r in pairs:
        _cmp(g, r, "%s %s" % (tag, n))


def _set_env(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _check_sparse_case(c, monkeypatch):
    _set_env(monkeypatch, c.env)
    D = c.params["hidden_size"]
    adj, indeg, h0 = sparse_batch(c.batch, D, c.T)
    w = _weights(c.params, c.T)
    g_out = np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)
    ref = _autograd_reference(c.params, c.T, w, adj, indeg, h0, g_out)
    plan = []

    def set_graph(e):
        e.set_graph_sparse(adj, indeg)
        plan.append(e.plan)

    got = _engine_grads(c.params, c.T, w, set_graph, h0, g_out, c.precision)
    assert plan_matches(plan[0], c.plan), (c.plan, plan[0])
    _compare(c.name, got, ref)


@pytest.mark.parametrize("case", [c.name for c in PLAN_MATRIX])
def test_gradients_on_every_forward_plan(case, monkeypatch):
    """GRU and RNN (edge bias, sum aggregation, two layers and a residual; ReLU on fp32, tanh on bf16x3: smooth_on_tensor_cores says
    why) on every plan: both fp32 tile variants LOCAL, fp32
    GLOBAL, tile-local wgmma on compact 64-row and on 128-row tiles (1024 molecules: more tiles than SMs), wgmma GLOBAL, forced and
    natural streaming (hidden 132 / 204 / 256: the column tail of the saved-state stores).  CudnnCompatibleGRUCell on fp32 LOCAL and
    GLOBAL, attention on fp32 GLOBAL."""
    _check_sparse_case(SPARSE_CASES[case], monkeypatch)


@pytest.mark.parametrize("case", [c.name for c in EDGE_SHAPES])
def test_gradients_at_backward_edge_shapes(case, monkeypatch):
    """T = 1 / 3 / 17 / 32 edge types with edge bias and avg aggregation over components with isolated nodes and single-type nodes; four
    residual inputs into one layer, one of them the layer's own input; a zero-step layer read through a residual."""
    _check_sparse_case(SPARSE_CASES[case], monkeypatch)


# ---------------------------------------------------------------------------------------------------------------- one engine, many backward calls
class _Trained:
    """One engine after a forward with save_for_backward; ``backward(fields)`` runs ggnn_backward into fresh zeroed buffers for the
    requested weight fields of every layer (plus ``d h0`` when asked) and returns them as NumPy."""

    def __init__(self, c, monkeypatch):
        import torch
        from gated_graph_neural_network_samples_b200.engine import PropagationEngine
        _set_env(monkeypatch, c.env)
        D = c.params["hidden_size"]
        adj, indeg, h0 = sparse_batch(c.batch, D, c.T)
        w = _weights(c.params, c.T)
        self.eng = PropagationEngine(c.params, c.T, precision=c.precision)
        self.dev_w = [{REN.get(k, k): torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda() for k, v in lw.items()} for lw in w]
        self.eng.set_weights(self.dev_w)
        self.eng.set_save_for_backward(True)
        self.eng.set_graph_sparse(adj, indeg)
        assert plan_matches(self.eng.plan, c.plan), (c.plan, self.eng.plan)
        self.h0 = torch.from_numpy(h0).cuda()
        self.out = self.eng.forward(self.h0)
        self.g_out = torch.from_numpy(np.random.default_rng(5).normal(size=h0.shape).astype(np.float32)).cuda()

    def fields(self):
        return sorted(self.dev_w[0])

    def zeros(self, fields):
        import torch
        return [{k: torch.zeros_like(lw[k]) for k in fields if k in lw} for lw in self.dev_w]

    def backward(self, fields, want_dh0=True, into=None):
        import torch
        grads = self.zeros(fields) if into is None else into
        dh0 = torch.zeros_like(self.h0) if want_dh0 else None
        self.eng.backward(self.g_out, grads, dh0)
        self.eng.sync_check()
        return (None if dh0 is None else dh0.cpu().numpy()), [{k: v.cpu().numpy() for k, v in lw.items()} for lw in grads]


NOISE = 1e-5   # atomic-order noise of the fp32 weight-gradient sums, relative to the largest entry


def _close(a, b, tag):
    err = U.max_rel_err(a, b) if np.any(b) else float(np.max(np.abs(a)))
    assert err < NOISE, (tag, err)


@pytest.mark.parametrize("case", PARTIAL_CASES)
def test_partial_requests_match_a_full_request(case, monkeypatch):
    """``ggnn_backward`` with only ``d h0``, only the edge weights, or only the biases (``gate_bias`` / ``cand_bias`` with their kernels
    null: the column-sum kernel), against the same fields of a full request.  A second call accumulates exactly one more gradient."""
    t = _Trained(SPARSE_CASES[case], monkeypatch)
    full_dh0, full = t.backward(t.fields())
    dh0, none = t.backward([])
    np.testing.assert_array_equal(dh0, full_dh0)
    assert all(not lw for lw in none)
    for request in (["edge_weights"], [k for k in t.fields() if "bias" in k]):
        dh0, part = t.backward(request, want_dh0=False)
        assert dh0 is None
        for l, (p, f) in enumerate(zip(part, full)):
            assert sorted(p) == sorted(request), (p.keys(), request)
            for k in p:
                _close(p[k], f[k], "layer %d %s" % (l, k))
    # accumulation: the weight gradients are added into the caller's buffers, d h0 is overwritten
    bufs = t.zeros(t.fields())
    _, once = t.backward(t.fields(), into=bufs)
    dh0, twice = t.backward(t.fields(), into=bufs)
    np.testing.assert_array_equal(dh0, full_dh0)
    for l, (a, b) in enumerate(zip(once, twice)):
        for k in a:
            _close(b[k], 2.0 * a[k], "layer %d %s twice" % (l, k))


@pytest.mark.parametrize("case", DETERMINISM_CASES)
def test_d_h0_is_bit_identical_run_to_run(case, monkeypatch):
    """No float atomics on node states (the scatter of the backward is a gather through the source-keyed CSR): ``d h0`` is the same bits
    on every call.  The weight gradients are split-row sums with atomics: equal within their ordering noise."""
    t = _Trained(SPARSE_CASES[case], monkeypatch)
    a_dh0, a = t.backward(t.fields())
    for _ in range(2):
        b_dh0, b = t.backward(t.fields())
        np.testing.assert_array_equal(b_dh0, a_dh0)
        for l, (x, y) in enumerate(zip(a, b)):
            for k in x:
                _close(y[k], x[k], "layer %d %s" % (l, k))


# ---------------------------------------------------------------------------------------------------------------- dense
@pytest.mark.parametrize("name,precision,D,weighted,pattern", DENSE_CASES, ids=[c[0] for c in DENSE_CASES])
def test_dense_gradients_on_weighted_and_binary_matrices(name, precision, D, weighted, pattern):
    """A weighted ``[b, T, v, v]`` matrix goes through the CSR builder with its entries as slot weights, which weight both gathers of the
    backward (target- and source-keyed CSR); a binary one goes through it unweighted.  Reference: the dense oracle in float64, which takes
    weighted matrices."""
    import torch
    A, h0 = dense_batch(D, weighted)
    b, v = h0.shape[:2]
    dw = O.init_dense_weights({"hidden_size": D}, DENSE_T, np.random.default_rng(5))
    dw["cand_bias"] = np.random.default_rng(6).normal(0, 0.1, D).astype(np.float32)
    g_out = np.random.default_rng(7).normal(size=h0.shape).astype(np.float32)
    tw = {k: torch.tensor(x, dtype=torch.float64, requires_grad=True) for k, x in dw.items()}
    th0 = torch.tensor(h0, dtype=torch.float64, requires_grad=True)
    out = O.dense_propagation_torch(th0, A, tw, {"num_timesteps": DENSE_STEPS, "use_edge_bias": True}, dtype=torch.float64)
    (out * torch.tensor(g_out, dtype=torch.float64)).sum().backward()
    plan = []

    def set_graph(e):
        e.set_graph_dense(A)
        plan.append(e.plan)

    w_eng = [dict(dw, edge_biases=dw["edge_biases"].reshape(DENSE_T, D))]
    o2, dh0, gw = _engine_grads(dense_params(D), DENSE_T, w_eng, set_graph, h0.reshape(b * v, D), g_out.reshape(b * v, D), precision)
    assert plan_matches(plan[0], pattern), (pattern, plan[0])
    ref_gw = [{k: tw[k].grad.numpy().reshape(gw[0][k].shape) for k in tw}]
    _compare("dense " + name, (o2.reshape(b, v, D), dh0.reshape(b, v, D), gw), (out.detach().numpy(), th0.grad.numpy(), ref_gw))


# ---------------------------------------------------------------------------------------------------------------- GCN
@pytest.mark.parametrize("name,precision,D,kind,keep,env,pattern", GCN_CASES, ids=[c[0] for c in GCN_CASES])
def test_gcn_gradients_on_every_plan(name, precision, D, kind, keep, env, pattern, monkeypatch):
    """The GCN's saves on the LOCAL wgmma kernel (all layers fused, every layer written when save is set), its GLOBAL plan and the fp32
    kernel above hidden 128, with and without state dropout, against float64 autograd at 2.5e-5."""
    import torch
    from tests.test_gpu_gcn import run
    _set_env(monkeypatch, env)
    V, lst, w, ks, bs, h0 = gcn_batch(D, kind)
    seed = 77
    got, eng = run(D, GCN_LAYERS, V, lst, w, h0, ks, bs, precision, keep=keep, seed=seed, save=True)
    assert plan_matches(eng.plan, pattern), (pattern, eng.plan)
    g_out = np.random.default_rng(5).normal(0, 1, (V, D)).astype(np.float32)
    gk = [torch.zeros(D, D, device="cuda") for _ in range(GCN_LAYERS)]
    gb = [torch.zeros(D, device="cuda") for _ in range(GCN_LAYERS)]
    dh0 = torch.empty(V, D, device="cuda")
    eng.backward(torch.from_numpy(g_out).cuda(), [{"kernel": a, "bias": b} for a, b in zip(gk, gb)], d_h0=dh0)
    eng.sync_check()
    masks = [eng.state_dropout_mask(l, keep, seed) for l in range(GCN_LAYERS - 1)] if keep < 1 else None
    th0 = torch.from_numpy(h0).double().requires_grad_()
    tk = [torch.from_numpy(k).double().requires_grad_() for k in ks]
    tb = [torch.from_numpy(b).double().requires_grad_() for b in bs]
    out = G.gcn_propagation_torch(th0, lst, torch.from_numpy(w).double(), tk, tb, masks, keep)
    out.backward(torch.from_numpy(g_out).double())
    errs = [("forward", U.max_rel_err(got, out.detach().numpy())), ("d h0", U.max_rel_err(dh0.cpu().numpy(), th0.grad.numpy()))]
    for l in range(GCN_LAYERS):
        errs += [("layer %d kernel" % l, U.max_rel_err(gk[l].cpu().numpy(), tk[l].grad.numpy())),
                 ("layer %d bias" % l, U.max_rel_err(gb[l].cpu().numpy(), tb[l].grad.numpy()))]
    worst = max((e, n) for n, e in errs[1:])
    print("\n%-36s forward %.2e  worst gradient %.2e on %s" % ("gcn " + name, errs[0][1], worst[0], worst[1]))
    for n, e in errs:
        assert e < (1e-4 if n == "forward" else 2.5e-5), (name, n, e)
